"""The propagation scans' gather kernels against float64, element by element (references and bounds: scan_gather_ref).

pp_deform_gather, pp_deform_align, pp_flow_warp_fbcheck, pp_prop_cond and pp_img_prop_scan run in every step of the
flow-completion scans, the generator's feature scans and the image scan of stage 3.  Here:

  * sampling positions of a flow warp are restated bit for bit; continuous outputs are within their own per-element
    bound E of float64; TF32 outputs are rounded to nearest, ties away (low bits, ulp/2 + E, equality with rna(ref) where
    the rounding is decided, mean signed rounding error), with crafted midpoint ties;
  * the validity flags and the 0.1 binarisations are compared by margin: decided where the float64 quantity lies further
    than its fp32 evaluation bound from the threshold, and exactly (numpy float32 restatement) on crafted integer-flow
    cases that put lhs == thr and masks of exactly 0.1f under the strict comparisons;
  * the image scan is checked one step at a time, each step from the kernel's own previous state (the workspace holds
    the backward scan);
  * operands and outputs are channel slices of NaN-filled buffers laid out as production lays them out, and nothing
    outside the written slices changes;
  * each bound rejects a reference that is wrong the way a kernel goes wrong;
  * the cases cover every signature the models and stage 3 call these entry points with.
"""
import collections
import ctypes
import gc

import numpy as np
import pytest
import torch

from tests import scan_gather_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda"
UNDECIDED_MAX = 1e-3


def _nan(*shape):
    return torch.full(shape, float("nan"), device=DEV)


def _free():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _midpoints(t):
    """fp32 values whose low 13 bits are 0x1000: exactly halfway between TF32 neighbours"""
    i = t.contiguous().view(torch.int32)
    return ((i & ~0x1FFF) | R.TF32_MID).view(torch.float32)


# ================================================================================================ pp_deform_gather
GCase = collections.namedtuple("GCase", "label Cin x2 flow obias max_res n H W kind")
GATHER_CASES = [
    GCase("generator, bias folded (hoisted plan)", 128, False, True, True, 3.0, 1, 60, 108, "rand"),
    GCase("generator, bias in o (wgmma plan)", 128, False, True, False, 3.0, 1, 60, 108, "rand"),
    GCase("flow completion, first order", 256, False, False, True, 5.0, 1, 30, 54, "rand"),
    GCase("flow completion, second order x2 split", 256, True, False, False, 5.0, 1, 30, 54, "rand"),
    GCase("x2 + flow, n=3, 231 pixels (partial last block)", 128, True, True, True, 5.0, 3, 7, 11, "rand"),
    GCase("1-pixel-high map, n=2", 256, False, True, False, 3.0, 2, 1, 13, "rand"),
    GCase("1-pixel-wide map", 128, False, False, True, 5.0, 1, 9, 1, "rand"),
    GCase("n=2 flow completion batch", 256, False, False, True, 5.0, 2, 30, 54, "rand"),
    GCase("exact: integer flow across every border, TF32 ties, x2, n=2", 256, True, True, False, 3.0, 2, 9, 13, "exact"),
    GCase("exact: integer flow, bias", 128, False, True, True, 5.0, 1, 5, 7, "exact"),
]


def _gather_inputs(c, gen):
    n, H, W, Cin = c.n, c.H, c.W, c.Cin
    if c.kind == "exact":
        xv = _midpoints(torch.randn(n, H, W, Cin, generator=gen) * 3)
        o = torch.zeros(n, H, W, 432)
        o[..., 288:] = 200.0                                  # sigmoid(200) == 1 in fp32: the modulation is exactly 1
        ob = torch.zeros(432) if c.obias else None            # an all-zero bias keeps the offsets exactly 0
        flow = torch.randint(-3, 4, (n, H, W, 2), generator=gen).float() if c.flow else None
    else:
        xv = torch.randn(n, H, W, Cin, generator=gen)
        o = torch.randn(n, H, W, 432, generator=gen) * 1.5
        ob = torch.randn(432, generator=gen) * 0.3 if c.obias else None
        flow = torch.randn(n, H, W, 2, generator=gen) * 2 if c.flow else None
    return xv, o, ob, flow


def _run_gather(c, xv, o, ob, flow):
    """production layouts: x (and x2) channel slices of wider NaN buffers, o [..., :432] of a 436-wide one, cols between
    NaN guard regions"""
    n, H, W, Cin = c.n, c.H, c.W, c.Cin
    half = Cin // 2
    if c.x2:
        xb1, xb2 = _nan(n, H, W, Cin + 8), _nan(n, H, W, Cin + 8)    # ld >= Cin: a late split would read NaN, in bounds
        xb1[..., :half] = xv[..., :half].to(DEV)
        xb2[..., 4:4 + half] = xv[..., half:].to(DEV)
        x, x2 = xb1[..., :half], xb2[..., 4:4 + half]
    else:
        xb1 = _nan(n, H, W, Cin + 8)
        xb1[..., 4:4 + Cin] = xv.to(DEV)
        x, x2 = xb1[..., 4:4 + Cin], None
    obuf = _nan(n, H, W, 436)
    obuf[..., :432] = o.to(DEV)
    N, pad = n * H * W * 9 * Cin, 64
    flat = _nan(N + 2 * pad)
    cols = flat[pad:pad + N].view(n, H, W, 9 * Cin)
    from propainter_b200 import ops
    ops.deform_gather(x, obuf[..., :432], flow.to(DEV) if flow is not None else None, c.max_res, cols,
                      o_bias=ob.to(DEV) if ob is not None else None, x2=x2)
    torch.cuda.synchronize()
    assert torch.isnan(flat[:pad]).all() and torch.isnan(flat[pad + N:]).all(), "pp_deform_gather wrote outside cols"
    return cols


def _o_eff(o, ob):
    """the raw offset-net output as the kernels see it: o + o_bias added once in fp32"""
    o = o.to(DEV)
    return o + ob.to(DEV) if ob is not None else o


def _exact_cols(xv, flow, n, H, W, Cin):
    """integer flow, zero offsets, modulation 1: every tap reads one pixel exactly (0 outside), rounded rna to TF32"""
    from propainter_b200 import ops
    ys, xs = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    out = torch.zeros(n, H * W, 9, Cin)
    xr = ops.tf32_round(xv.to(DEV)).cpu()
    for k in range(9):
        py = (ys - 1 + k // 3)[None] + flow[..., 1].long()
        px = (xs - 1 + k % 3)[None] + flow[..., 0].long()
        ok = (py > -1) & (py < H) & (px > -1) & (px < W)
        for b in range(n):
            v = xr[b][py[b].clamp(0, H - 1), px[b].clamp(0, W - 1)]
            out[b, :, k] = torch.where(ok[b].reshape(-1, 1), v.reshape(H * W, Cin), torch.zeros(()))
    return out


def test_deform_gather_f64():
    gen = torch.Generator().manual_seed(40)
    bias = {}
    for c in GATHER_CASES:
        xv, o, ob, flow = _gather_inputs(c, gen)
        cols = _run_gather(c, xv, o, ob, flow)
        n, H, W, Cin = c.n, c.H, c.W, c.Cin
        got = cols.view(n, H * W, 9, Cin)
        if c.kind == "exact":
            exp = _exact_cols(xv, flow, n, H, W, Cin)
            assert torch.equal(got.cpu(), exp), c.label
            outside = (exp == 0).float().mean().item()
            assert 0.05 < outside < 0.6, outside                  # taps do cross the borders
            print(f"[deform_gather] {c.label}: bit-exact, {outside:.2%} of the taps outside the map")
            continue
        x64 = xv.to(DEV).double()
        o32 = _o_eff(o, ob)
        fl = flow.to(DEV) if flow is not None else None
        st = {}
        for k in range(9):
            ref, E = R.deform_cols_ref(x64, o32, fl, c.max_res, k)
            R.check_tf32(got[:, :, k], ref, E, st)
            if k == 4 and c.label.startswith("generator, bias folded"):
                for fault in ("swap", "noflip", "corner", "group", "shift"):
                    wr, _ = R.deform_cols_ref(x64, o32, fl, c.max_res, k, fault)
                    assert R.bound_rejects(got[:, :, k], wr, E + 0.5 * R.tf32_ulp(wr.abs() + E)), fault
                ulp = R.tf32_ulp(ref)
                trunc = torch.sign(ref) * torch.floor(ref.abs() / torch.where(ulp == 0, torch.ones_like(ulp), ulp)) * ulp
                assert (got[:, :, k].double() != trunc).any()                     # columns truncated: rejected
            del ref, E
        for key in ("n", "sum", "total"):
            bias[key] = bias.get(key, 0) + st[key]
        print(f"[deform_gather] {c.label}: worst |err|/(ulp/2+E) {st['worst']:.3f}, decided {st['n'] / st['total']:.4f}, "
              f"mean rounding error {st['sum'] / max(st['n'], 1):+.4f} ulp")
        del x64, o32, cols, got
        _free()
    mean = bias["sum"] / bias["n"]
    print(f"[deform_gather] mean TF32 rounding error {mean:+.5f} ulp over {bias['n']} decided columns")
    assert bias["n"] >= 10 ** 5 and abs(mean) < 0.02


# ================================================================================================ pp_deform_align
ACase = collections.namedtuple("ACase", "label Cin flow obias max_res H W")
ALIGN_CASES = [
    ACase("generator C2 map", 128, True, True, 3.0, 60, 108),
    ACase("flow completion C2 map", 256, False, True, 5.0, 30, 54),
    ACase("one full wave of CTAs", 128, True, False, 3.0, 128, 132),
    ACase("small ragged map", 256, True, True, 5.0, 7, 10),
]


def _align_ref(x64, o32, fl, mr, wk, fault=None):
    """float64 deform_conv3x3 without bias: sum_k cols_k @ W_k, plus S = sum |cols||W| and ES = sum E |W|"""
    out = S = ES = 0
    for k in range(9):
        ref, E = R.deform_cols_ref(x64, o32, fl, mr, k, fault)
        out = out + ref[0] @ wk[k]
        if fault is None:
            S = S + ref[0].abs() @ wk[k].abs()
            ES = ES + E[0] @ wk[k].abs()
        del ref, E
    return out, S, ES


def test_deform_align_f64():
    from propainter_b200 import ops
    gen = torch.Generator().manual_seed(41)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    seen = set()
    for c in ALIGN_CASES:
        H, W, Cin, npix = c.H, c.W, c.Cin, c.H * c.W
        splits = R.da_splits(npix, 9 * (Cin // 32), sms)
        seen.add(("split1" if splits == 1 else "splitN", "ragged" if npix % 32 else "even", Cin))
        xv = torch.randn(1, H, W, Cin, generator=gen)
        o = torch.randn(1, H, W, 432, generator=gen) * 1.5
        ob = torch.randn(432, generator=gen) * 0.3 if c.obias else None
        flow = torch.randn(1, H, W, 2, generator=gen) * 2 if c.flow else None
        wgt = torch.randn(128, Cin, 3, 3, generator=gen) / (Cin * 9) ** 0.5
        bias = torch.randn(128, generator=gen)
        xb = _nan(H, W, Cin + 128)
        xb[..., :Cin] = xv[0].to(DEV)
        outb = _nan(H, W, 260)
        fl = flow[0].contiguous().to(DEV) if flow is not None else None
        ops.deform_align(xb[..., :Cin], o[0].contiguous().to(DEV), fl, c.max_res, ops.pack_deform_weight(wgt).to(DEV),
                         bias.to(DEV), outb[..., 128:256], o_bias=ob.to(DEV) if ob is not None else None)
        torch.cuda.synchronize()
        assert torch.isnan(outb[..., :128]).all() and torch.isnan(outb[..., 256:]).all()
        got = outb[..., 128:256].reshape(npix, 128).double()
        x64, o32 = xv.to(DEV).double(), _o_eff(o, ob)
        wk = wgt.to(DEV).double().permute(2, 3, 1, 0).reshape(9, Cin, 128)
        out, S, ES = _align_ref(x64, o32, fl, c.max_res, wk)
        ref = out + bias.to(DEV).double()
        K = 9 * Cin
        # rna operands (2 x 2^-11 relative per product, of the sample within ES), the samples' own bound, fp32 accumulation
        # of K products over `splits` partial sums (2^-23 per step), the bias add
        bound = (2 * 2.0 ** -11 + 2.0 ** -22) * (S + ES) + ES + (K + splits + 2) * 2.0 ** -23 * (S + ES) \
            + 2 * R.U * (bias.to(DEV).double().abs() + ref.abs()) + R.TINY
        worst = R.check_bound(got, ref, bound, c.label)
        for fault in ("corner", "group"):
            wr, _, _ = _align_ref(x64, o32, fl, c.max_res, wk, fault)
            assert R.bound_rejects(got, wr + bias.to(DEV).double(), bound), fault
        print(f"[deform_align] {c.label} ({H}x{W}, Cin {Cin}): split factor {splits}, worst err/E {worst:.4f}, "
              f"worst err/S {((got - ref).abs() / (S + R.TINY)).max().item():.2e}")
        del x64, o32, out, S, ES, ref, got, xb, outb
        _free()
    for need in (("split1",), ("splitN",), ("ragged",), (128,), (256,)):
        assert any(all(v in s for v in need) for s in seen), need


# ================================================================================================ validity by margin
def _valid_decision(fprop, fcheck64, ix, iy, stats=None):
    """float64 fb check of every pixel: fprop [n,h,w,2] fp32 (CPU), fcheck64 [n,h,w,2] float64 (device), exact
    positions [n,P].  Returns (valid, decided) [n,P] on the device; where the position is integral the check-flow samples
    are exact and the decision is pp_fb_valid's own fp32 arithmetic (numpy), exact ties included."""
    b, e = R.warp_sample(fcheck64, ix, iy)
    f = fprop.reshape(fprop.shape[0], -1, 2)
    fx, fy = f[..., 0].to(DEV).double(), f[..., 1].to(DEV).double()
    valid, decided = R.fb_margin(fx, fy, b[..., 0], b[..., 1], e[..., 0], e[..., 1])
    integral = (ix == np.rint(ix)) & (iy == np.rint(iy))
    if integral.any():
        v32, tie = R.fb_valid32(f[..., 0].numpy(), f[..., 1].numpy(), b[..., 0].float().cpu().numpy(), b[..., 1].float().cpu().numpy())
        it = torch.from_numpy(integral).to(DEV)
        valid = torch.where(it, torch.from_numpy(v32).to(DEV), valid)
        decided = decided | it
        if stats is not None:
            stats["ties"] = stats.get("ties", 0) + int((tie & integral).sum())
    if stats is not None:
        stats["und"] = stats.get("und", 0) + int((~decided).sum())
        stats["cnt"] = stats.get("cnt", 0) + decided.numel()
    return valid, decided


def _tie_field(n, h, w, fx, fy, gen):
    """integer flow (fx, fy) everywhere on an h x w map with power-of-two denominators (exact positions), and a check flow
    whose value at each in-image target is one of the (bx, by) that put pp_fb_valid's lhs exactly on its threshold (every
    other target: a random nearby value)"""
    assert ((h - 1) & (h - 2)) == 0 and ((w - 1) & (w - 2)) == 0
    ties = R.fb_ties(fx, fy, 6)
    assert len(ties) >= 3
    fprop = torch.empty(n, h, w, 2)
    fprop[..., 0], fprop[..., 1] = float(fx), float(fy)
    fcheck = torch.randn(n, h, w, 2, generator=gen) * 0.3 - torch.tensor([fx, fy], dtype=torch.float32)
    sel = torch.rand(n, h, w, generator=gen) < 0.7
    idx = torch.randint(0, len(ties), (n, h, w), generator=gen)
    tv = torch.tensor(ties, dtype=torch.float32)[idx]
    fcheck = torch.where(sel[..., None], tv, fcheck)
    return fprop, fcheck.contiguous()


# ================================================================================================ pp_flow_warp_fbcheck
WCase = collections.namedtuple("WCase", "label n h w C want_warp round_tf32 aux_ld kind")
WARP_CASES = [
    WCase("generator (fx, fy, valid) of all frames, aux of the 8-channel buffer", 4, 60, 108, 128, False, False, 8, "rand"),
    WCase("hoisted plan: aux inside the 136-channel scan input", 4, 60, 108, 128, False, False, 136, "rand"),
    WCase("wgmma plan: warped, TF32-rounded", 1, 60, 108, 128, True, True, None, "rand"),
    WCase("hoisted plan: warped", 1, 60, 108, 128, True, False, None, "rand"),
    WCase("1-pixel-high maps, warp + aux", 3, 1, 13, 128, True, False, 8, "rand"),
    WCase("1-pixel-wide maps, warp + aux, TF32", 2, 9, 1, 64, True, True, 8, "rand"),
    WCase("exact ties: integer flow, lhs == thr", 2, 9, 17, 16, True, False, 8, "tie"),
]


def _smooth_flow(gen, n, h, w, amp):
    import torch.nn.functional as F
    z = torch.randn(n, 2, h // 4 + 2, w // 4 + 2, generator=gen) * amp
    return F.interpolate(z, size=(h, w), mode="bilinear", align_corners=False).permute(0, 2, 3, 1).contiguous()


def _flow_pair(gen, n, h, w):
    fprop = _smooth_flow(gen, n, h, w, 3.0)
    fcheck = (-fprop + 0.5 * torch.randn(n, h, w, 2, generator=gen)).contiguous()
    return fprop, fcheck


def test_flow_warp_fbcheck_f64():
    from propainter_b200 import ops
    gen = torch.Generator().manual_seed(42)
    tfst = {}
    for c in WARP_CASES:
        n, h, w, C = c.n, c.h, c.w, c.C
        if c.kind == "tie":
            fprop, fcheck = _tie_field(n, h, w, 3, -2, gen)
        else:
            fprop, fcheck = _flow_pair(gen, n, h, w)
        feat = torch.randn(n, h, w, C, generator=gen)
        fb = _nan(n, h, w, C + 8)
        fb[..., 4:4 + C] = feat.to(DEV)
        wb = _nan(n, h, w, C + 8)
        aux_b = _nan(n, h, w, c.aux_ld) if c.aux_ld else None
        warped, aux = ops.flow_warp_fbcheck(fb[..., 4:4 + C] if c.want_warp else None, fprop.to(DEV),
                                            fcheck.to(DEV) if c.aux_ld else None, warped=wb[..., :C] if c.want_warp else None,
                                            aux=aux_b[..., :3] if c.aux_ld else None, want_warp=c.want_warp, round_tf32=c.round_tf32)
        torch.cuda.synchronize()
        ix, iy = R.warp_positions(fprop)
        msg = [c.label]
        if c.want_warp:
            assert torch.isnan(wb[..., C:]).all()
            ref, E = R.warp_sample(feat.to(DEV).double(), ix, iy)
            got = warped.reshape(n, h * w, C)
            if c.round_tf32:
                plain, _ = ops.flow_warp_fbcheck(fb[..., 4:4 + C], fprop.to(DEV))
                assert torch.equal(got, ops.tf32_round(plain).reshape(n, h * w, C))
                R.check_tf32(got, ref, E, tfst)
                got = plain.reshape(n, h * w, C)
            worst = R.check_bound(got, ref, E, c.label)
            # integral positions or a 1-pixel axis: no lower-right corner to drop
            for fault in ("corner", "shift") if h > 1 and w > 1 and c.kind == "rand" else ("shift",):
                wr, _ = R.warp_sample(feat.to(DEV).double(), ix, iy, fault)
                assert R.bound_rejects(got, wr, E), fault
            wx, wy = R.warp_positions(fprop, "swap")
            wr, _ = R.warp_sample(feat.to(DEV).double(), wx, wy)
            assert (n * h * w < 32) or R.bound_rejects(got, wr, E), "swap"
            msg.append(f"warped worst err/E {worst:.3f}")
        if c.aux_ld:
            assert torch.isnan(aux_b[..., 3:]).all()
            assert torch.equal(aux[..., :2].cpu(), fprop)                   # fx, fy: bit-exact copies
            st = {}
            valid, decided = _valid_decision(fprop, fcheck.to(DEV).double(), ix, iy, st)
            gv = aux[..., 2].reshape(n, h * w)
            assert ((gv == 0) | (gv == 1)).all()
            assert torch.equal(gv.bool()[decided], valid[decided]), c.label
            frac = st["und"] / st["cnt"]
            assert frac < UNDECIDED_MAX, frac
            if c.kind == "tie":
                assert st["ties"] >= 10 and st["und"] == 0
            msg.append(f"valid undecided {frac:.2e} ({st.get('ties', 0)} exact ties)")
        print("[flow_warp_fbcheck] " + ", ".join(msg))
        _free()
    print(f"[flow_warp_fbcheck] TF32 mean rounding error {tfst['sum'] / tfst['n']:+.4f} ulp over {tfst['n']} values")
    assert abs(tfst["sum"] / tfst["n"]) < 0.02
    # want_warp=False needs no feature map; fcheck=None skips the validity
    with pytest.raises(RuntimeError):
        ops.flow_warp_fbcheck(None, torch.zeros(1, 4, 4, 2, device=DEV), None, want_warp=False)


# ================================================================================================ pp_prop_cond
PCase = collections.namedtuple("PCase", "label h w C first ld_cond ld_bb kind")
COND_CASES = [
    PCase("generator step (library-conv plan)", 60, 108, 128, False, 264, 260, "rand"),
    PCase("generator first step", 60, 108, 128, True, 264, 260, "rand"),
    PCase("1-pixel-high map", 1, 13, 64, False, 136, 132, "rand"),
    PCase("1-pixel-wide map", 9, 1, 64, False, 136, 132, "rand"),
    PCase("exact ties", 9, 17, 32, False, 72, 68, "tie"),
]


def test_prop_cond_f64():
    from propainter_b200 import ops
    gen = torch.Generator().manual_seed(43)
    for c in COND_CASES:
        h, w, C = c.h, c.w, c.C
        if c.kind == "tie":
            fprop, fcheck = _tie_field(1, h, w, -2, 1, gen)
        else:
            fprop, fcheck = _flow_pair(gen, 1, h, w)
        fprop, fcheck = fprop[0], fcheck[0]
        cur, prop = torch.randn(h, w, C, generator=gen), torch.randn(h, w, C, generator=gen)
        m = (torch.rand(h, w, 2, generator=gen) > 0.5).float()
        cb, pb = _nan(h, w, C + 8), _nan(h, w, C + 8)
        cb[..., 4:4 + C], pb[..., :C] = cur.to(DEV), prop.to(DEV)
        cond, bb = _nan(h, w, c.ld_cond), _nan(h, w, c.ld_bb)
        if c.first:
            ops.prop_cond(cb[..., 4:4 + C], None, None, None, m.to(DEV), None, bb, True)
        else:
            ops.prop_cond(cb[..., 4:4 + C], pb[..., :C], fprop.to(DEV), fcheck.to(DEV), m.to(DEV), cond, bb, False)
        torch.cuda.synchronize()
        b = bb.cpu()
        assert torch.equal(b[..., :C], cur) and torch.equal(b[..., 2 * C:2 * C + 2], m) and (b[..., 2 * C + 2:] == 0).all()
        if c.first:
            assert torch.equal(b[..., C:2 * C], cur) and torch.isnan(cond).all()
            print(f"[prop_cond] {c.label}: copies exact")
            continue
        assert torch.isnan(b[..., C:2 * C]).all()                                   # the aligned-feature slot is left alone
        cd = cond.cpu()
        assert torch.equal(cd[..., :C], cur) and torch.equal(cd[..., 2 * C:2 * C + 2], fprop)
        assert torch.equal(cd[..., 2 * C + 3:2 * C + 5], m) and (cd[..., 2 * C + 5:] == 0).all()
        ix, iy = R.warp_positions(fprop[None])
        ref, E = R.warp_sample(prop[None].to(DEV).double(), ix, iy)
        got = cond[..., C:2 * C].reshape(1, h * w, C)
        worst = R.check_bound(got, ref, E, c.label)
        if h > 1 and w > 1 and c.kind == "rand":
            wr, _ = R.warp_sample(prop[None].to(DEV).double(), ix, iy, "corner")
            assert R.bound_rejects(got, wr, E)
        st = {}
        valid, decided = _valid_decision(fprop[None], fcheck[None].to(DEV).double(), ix, iy, st)
        gv = cond[..., 2 * C + 2].reshape(1, h * w)
        assert torch.equal(gv.bool()[decided], valid[decided]) and ((gv == 0) | (gv == 1)).all()
        frac = st["und"] / st["cnt"]
        assert frac < UNDECIDED_MAX
        if c.kind == "tie":
            assert st["ties"] >= 10 and st["und"] == 0
        print(f"[prop_cond] {c.label}: warped worst err/E {worst:.3f}, valid undecided {frac:.2e} ({st.get('ties', 0)} exact ties)")
        _free()


# ================================================================================================ pp_img_prop_scan
def _step_bad(cur, mc, prev, mprev, fprop, fcheck, got_f, got_m, nearest, st=None, fault=None):
    """one scan step (pp_imgprop_values over the map), all planar fp32 device tensors: cur/prev/got_f [3,H,W],
    mc/mprev/got_m [H,W], flows [2,H,W].  Returns the number of pixels whose (frame, mask) matches no combination of
    the decisions the margins leave open (valid, mw), each evaluated in float64."""
    H, W = mc.shape
    fpm = fprop.permute(1, 2, 0).contiguous().cpu()[None]
    ix, iy = R.warp_positions(fpm, fault if fault == "swap" else None)
    valid, vdec = _valid_decision(fpm, fcheck.permute(1, 2, 0)[None].double(), ix, iy, st)
    sm, em = R.warp_sample(mprev.reshape(1, H, W, 1).double(), ix, iy)
    mw, mdec = R.threshold_margin(sm[0, :, 0], em[0, :, 0])
    integral = torch.from_numpy((ix == np.rint(ix)) & (iy == np.rint(iy))).to(DEV)[0]
    mdec = mdec | integral                                             # exact sample: the fp32 comparison itself
    valid, vdec = valid[0], vdec[0]
    if st is not None:
        st["mw_und"] = st.get("mw_und", 0) + int((~mdec).sum())
        st["mw_tenth"] = st.get("mw_tenth", 0) + int((integral & (sm[0, :, 0] == R.F_TENTH)).sum())
    p64 = prev.permute(1, 2, 0)[None].double()
    if nearest:
        wv, ew = R.nearest_sample(p64, ix, iy)[0], None
    else:
        s, e = R.warp_sample(p64, ix, iy, fault if fault in ("corner", "shift") else None)
        wv, ew = s[0], e[0]
    c64 = cur.reshape(3, -1).t().double()
    g64 = got_f.reshape(3, -1).t().double()
    mc64 = mc.reshape(-1).double()
    gm = got_m.reshape(-1)
    ok = torch.zeros_like(gm, dtype=torch.bool)
    worst = 0.0
    for v_c in (False, True):
        for w_c in (False, True):
            allowed = torch.where(vdec, valid == v_c, torch.ones_like(vdec)) & torch.where(mdec, mw == w_c, torch.ones_like(mdec))
            moved = v_c and not w_c                                   # valid * (1 - mw) == 1
            use = (mc64 > R.F_TENTH) & moved
            m2 = (mc64 > R.F_TENTH) & (not moved)
            fr_ok = torch.where(use[:, None], (g64 - wv).abs() <= (ew if ew is not None else 0), g64 == c64).all(1)
            if ew is not None and allowed.any():
                r = torch.where(use[:, None] & allowed[:, None], (g64 - wv).abs() / ew, torch.zeros_like(g64))
                worst = max(worst, float(r.max()))
            ok |= allowed & fr_ok & (gm == m2.float())
    if st is not None:
        st["worst"] = max(st.get("worst", 0.0), worst)
        st["use"] = st.get("use", 0) + int(((mc64 > R.F_TENTH) & valid & ~mw).sum())
    return int((~ok).sum())


def _scan(frames, ff, fb, masks, nearest):
    """pp_img_prop_scan through the C ABI with a workspace the test owns: returns (out, out_masks, bf, bm)"""
    from propainter_b200 import _lib
    L = _lib.lib()
    t, _, H, W = frames.shape
    HW = H * W
    wsb = L.pp_img_prop_scan_workspace_bytes(t, H, W)
    ws = _nan(wsb // 4 + 64)
    of, om = _nan(t, 3, H, W), _nan(t, 1, H, W)
    p = lambda a: ctypes.c_void_p(a.data_ptr())                      # noqa: E731
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(L.pp_img_prop_scan(p(frames), p(ff), p(fb), p(masks), p(of), p(om), p(ws), wsb, t, H, W, int(nearest), stream),
               "pp_img_prop_scan")
    torch.cuda.synchronize()
    assert torch.isnan(ws[wsb // 4:]).all()
    return of, om[:, 0], ws[:t * 3 * HW].view(t, 3, H, W), ws[t * 3 * HW:t * 4 * HW].view(t, H, W)


def _scan_inputs(gen, t, H, W, kind):
    """frames in [-1, 1]; a hole that moves from frame to frame, with 3-8 % of the mask values exactly 0.1f"""
    frames = (torch.rand(t, 3, H, W, generator=gen) * 2 - 1)
    masks = torch.zeros(t, 1, H, W)
    for i in range(t):
        x0 = (W // 8) * (i % 4)
        masks[i, :, H // 4:3 * H // 4, x0:x0 + W // 2] = 1
    tenth = torch.rand(t, 1, H, W, generator=gen) < (0.08 if kind == "exact" else 0.03)
    masks = torch.where(tenth, torch.full((), R.F_TENTH), masks)                  # masks of exactly 0.1f
    if kind == "exact":
        # integer and half-integer flows on power-of-two grids: exact positions, nearest ties, exact fb ties
        ff = torch.randint(-2, 3, (max(t - 1, 1), 2, H, W), generator=gen).float()
        ff = ff + 0.5 * (torch.rand(ff.shape, generator=gen) < 0.3).float()
        fb = -ff + torch.randn(ff.shape, generator=gen) * 0.4
        ties = R.fb_ties(2.0, -1.0, 6)
        sel = (ff[:, 0] == 2.0) & (ff[:, 1] == -1.0)
        tv = torch.tensor(ties, dtype=torch.float32)[torch.randint(0, len(ties), sel.shape, generator=gen)].permute(0, 3, 1, 2)
        # the check flow at the target of a (2, -1) source pixel: shift the tie values by the flow
        tgt = torch.zeros_like(sel)
        tgt[:, :-1, 2:] = sel[:, 1:, :-2]
        fb = torch.where(tgt[:, None], tv, fb)
        if t > 1:
            # the first backward step samples masks[t-1] at integer positions: put exactly 0.1f under half of the hole
            # pixels of frame t-2 whose flow is integral, so `mw > 0.1` decides whether they are filled
            f = ff[t - 2]
            ys, xs = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
            tx, ty = (xs + f[0]).long(), (ys + f[1]).long()
            ok = (masks[t - 2, 0] == 1) & (f == f.round()).all(0) & (tx >= 0) & (tx < W) & (ty >= 0) & (ty < H)
            ok &= torch.rand(H, W, generator=gen) < 0.5
            masks[t - 1, 0][ty[ok], tx[ok]] = R.F_TENTH
        return frames[:t], ff[:t - 1].contiguous(), fb[:t - 1].contiguous(), masks
    # flows of up to ~40 pixels
    ff = _smooth_flow(gen, max(t - 1, 1), H, W, 16.0).permute(0, 3, 1, 2)[:t - 1].contiguous()
    fb = (-ff + 0.3 * _smooth_flow(gen, max(t - 1, 1), H, W, 4.0).permute(0, 3, 1, 2)[:t - 1]).contiguous()
    return frames, ff, fb, masks


SCAN_CASES = [(1, 240, 432, "rand"), (2, 240, 432, "rand"), (9, 240, 432, "rand"), (10, 9, 17, "exact"), (2, 17, 33, "exact")]


def test_img_prop_scan_stepwise_f64():
    gen = torch.Generator().manual_seed(44)
    for (t, H, W, kind) in SCAN_CASES:
        frames, ff, fb, masks = (a.to(DEV) for a in _scan_inputs(gen, t, H, W, kind))
        masked = (frames * (1 - masks)).contiguous()
        for nearest in (True, False):
            of, om, bf, bm = _scan(masked, ff, fb, masks, nearest)
            assert torch.equal(bf[t - 1], masked[t - 1]) and torch.equal(bm[t - 1], masks[t - 1, 0])
            assert torch.equal(of[0], bf[0]) and torch.equal(om[0], bm[0])
            st = {}
            for i in range(t - 2, -1, -1):                                # backward: frames[i] from bf[i+1] along ff[i]
                bad = _step_bad(masked[i], masks[i, 0], bf[i + 1], bm[i + 1], ff[i], fb[i], bf[i], bm[i], nearest, st)
                assert bad == 0, (t, H, W, nearest, "backward", i, bad)
            for i in range(1, t):                                         # forward: bf[i] from out[i-1] along fb[i-1]
                bad = _step_bad(bf[i], bm[i], of[i - 1], om[i - 1], fb[i - 1], ff[i - 1], of[i], om[i], nearest, st)
                assert bad == 0, (t, H, W, nearest, "forward", i, bad)
            if t > 1:
                vfrac, mfrac = st["und"] / st["cnt"], st["mw_und"] / st["cnt"]
                if kind == "exact":                  # half-integer samples of 0.1f masks may sit exactly on the threshold
                    assert st["ties"] > 0 and st["mw_tenth"] > 0
                else:
                    assert vfrac < UNDECIDED_MAX and mfrac < UNDECIDED_MAX, (vfrac, mfrac)
                if kind == "rand" and t >= 9 and not nearest:             # the bound rejects wrong step references
                    for fault in ("swap", "corner", "shift"):
                        assert _step_bad(bf[1], bm[1], of[0], om[0], fb[0], ff[0], of[1], om[1], False, None, fault) > 0, fault
                print(f"[img_prop_scan] t={t} {H}x{W} {'nearest' if nearest else 'bilinear'} ({kind}): valid undecided "
                      f"{vfrac:.2e}, mw undecided {mfrac:.2e}, warped pixels {st['use']}, worst err/E {st['worst']:.3f}, "
                      f"{st.get('ties', 0)} exact fb ties, {st['mw_tenth']} mw samples of exactly 0.1f")
            del of, om, bf, bm
        _free()


# ================================================================================================ production signatures
def _record(monkeypatch):
    """signatures of every call of the five entry points from RecurrentFlowCompleteNet.forward_bidirect_flow,
    InpaintGenerator.forward_parts (each scan plan forced) and stage 3 (ProPainterPipeline.propagate_images)"""
    import types
    from propainter_b200 import autotune, config, ops
    from propainter_b200.inference_propainter import InferenceConfig, ProPainterPipeline
    from propainter_b200.model.propainter import InpaintGenerator
    from propainter_b200.model.recurrent_flow_completion import RecurrentFlowCompleteNet
    monkeypatch.setattr(config, "UMMA_CONV", "auto")
    seen = collections.defaultdict(set)
    plan = {"i": 0}
    real_pick = autotune.pick

    def forced(key, variants, *a, **k):
        if key[0] in ("rfc_prop", "gen_prop"):
            return variants[min(plan["i"], len(variants) - 1)](*a)
        return real_pick(key, variants, *a, **k)

    def wrap(name, sig):
        real = getattr(ops, name)

        def rec(*a, **k):
            seen[name].add(sig(*a, **k))
            return real(*a, **k)
        monkeypatch.setattr(ops, name, rec)

    wrap("deform_gather", lambda x, o, flow, max_res, cols=None, o_bias=None, x2=None:
         (x.shape[-1] * (2 if x2 is not None else 1), x2 is not None, flow is not None, o_bias is not None, float(max_res),
          x.shape[0] > 1))
    wrap("deform_align", lambda x, o, flow, max_res, w_packed, bias, out, o_bias=None:
         (x.shape[-1], flow is not None, o_bias is not None, float(max_res)))
    wrap("flow_warp_fbcheck", lambda feat, fprop, fcheck=None, warped=None, aux=None, want_warp=True, round_tf32=False:
         (bool(want_warp), bool(round_tf32), aux.stride(-2) if aux is not None else None, fprop.shape[0] > 1))
    wrap("prop_cond", lambda cur, prop, fprop, fcheck, mcur, cond, bb, first:
         (bool(first), cur.shape[-1], cond.stride(-2) if cond is not None else None, bb.stride(-2)))
    wrap("img_prop_scan", lambda frames, flows_f, flows_b, masks, nearest=True: (bool(nearest),))
    monkeypatch.setattr(autotune, "pick", forced)
    gen = torch.Generator().manual_seed(0)
    T, H, W = 5, 64, 96
    flows = tuple((torch.randn(1, T - 1, 2, H, W, generator=gen) * 3).to(DEV) for _ in range(2))
    masks = torch.zeros(1, T, 1, H, W, device=DEV)
    masks[..., 16:48, 24:72] = 1
    Hg, Wg, t, lt = 128, 128, 5, 3
    frames = (torch.rand(1, t, 3, Hg, Wg, generator=gen) * 2 - 1).to(DEV)
    fl = tuple((torch.randn(1, lt - 1, 2, Hg, Wg, generator=gen) * 4).to(DEV) for _ in range(2))
    m = torch.zeros(1, t, 1, Hg, Wg, device=DEV)
    m[..., Hg // 4:Hg // 2, Wg // 3:2 * Wg // 3] = 1
    for i in range(5):
        plan["i"] = i
        RecurrentFlowCompleteNet(None, seed=2).to(DEV).forward_bidirect_flow(flows, masks)
        InpaintGenerator(seed=3).to(DEV).forward_parts(frames * (1 - m), fl, m, m, lt)
    fl3 = tuple((torch.randn(1, t - 1, 2, Hg, Wg, generator=gen) * 4).to(DEV) for _ in range(2))
    stage3 = types.SimpleNamespace(model=InpaintGenerator(seed=3).to(DEV))
    ProPainterPipeline.propagate_images(stage3, frames, m, fl3, InferenceConfig())
    torch.cuda.synchronize()
    return seen


def test_cases_cover_production_signatures(monkeypatch):
    seen = _record(monkeypatch)
    _free()
    print("[signatures] " + "; ".join(f"{k}: {sorted(v, key=str)}" for k, v in sorted(seen.items())))
    for name in ("deform_gather", "flow_warp_fbcheck", "prop_cond", "img_prop_scan"):
        assert seen[name], name
    have = {(c.Cin, c.x2, c.flow, c.obias, c.max_res, c.n > 1) for c in GATHER_CASES if c.kind == "rand"}
    assert seen["deform_gather"] <= have, seen["deform_gather"] - have
    have = {(c.Cin, c.flow, c.obias, c.max_res) for c in ALIGN_CASES}
    assert seen["deform_align"] <= have, seen["deform_align"] - have
    have = {(c.want_warp, c.round_tf32, c.aux_ld, c.n > 1) for c in WARP_CASES if c.kind == "rand"}
    assert seen["flow_warp_fbcheck"] <= have, seen["flow_warp_fbcheck"] - have
    have = {(c.first, c.C, c.ld_cond if not c.first else None, c.ld_bb) for c in COND_CASES if c.kind == "rand"}
    assert seen["prop_cond"] <= have, seen["prop_cond"] - have
    assert seen["img_prop_scan"] <= {(True,), (False,)}
