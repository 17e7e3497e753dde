"""The recurrent propagation scans on fp16 operands (config.half_convs): the fp16 instance of pp_conv2d_umma, the fp16 outputs
of pp_deform_gather and pp_flow_warp_fbcheck, and both scans and nets against the fp32 oracle.

  * conv_umma_f16 against a float64 conv of the same fp16 operands, element by element, over its tile plans (M 64 / 128,
    8- / 16-wide tiles, BN 32 / 64 / 128), KH 1 / 3, grouped 1x1 GEMMs, 1-4 segments, ragged maps, n > 1, every epilogue
    and every output mode (fp32 out, fp16 out16, both in one pass), and every conv signature the fp16 scans issue at the
    production map sizes.  Bound: the fp32 accumulation error, plus 1/2 fp16 ulp where it stores fp16.  Columns of the
    output buffers past Cout hold NaN and must keep it.
  * the fp16 gather and warp against the float64 references of tests/scan_gather_ref.py: 1/2 fp16 ulp plus the fp32 sum error.
  * both nets with their scans on fp16 (plan 0 forced) against the oracle: within 1.5x the error of the TF32 plan 0 on the
    same inputs, with the largest |value| of every fp16 tensor recorded; in strict fp32 the switch changes nothing.
"""
import collections
import contextlib
import gc
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import scan_gather_ref as R
from tests.test_gpu_scan_gather_f64 import GATHER_CASES, WARP_CASES, _flow_pair, _gather_inputs, _o_eff

pytestmark = pytest.mark.gpu
DEV = "cuda"
TAU = 2.0 ** -16          # fp32 accumulation, relative to sum |x| |w| (as in test_gpu_tensor_core_f64.py)
ACTS = {"none": (lambda v, s: v), "relu": (lambda v, s: v.clamp_min(0)), "leaky": (lambda v, s: torch.where(v > 0, v, v * s)),
        "sigmoid": (lambda v, s: torch.sigmoid(v)), "tanh": (lambda v, s: torch.tanh(v))}


@pytest.fixture(autouse=True)
def _release():
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _nan(shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), device=DEV, dtype=dtype)


def _r8(c):
    return (c + 7) // 8 * 8


def _ulp16(a):
    """fp16 ulp of |a| (float64 tensor)"""
    return torch.from_numpy(np.spacing(np.abs(a.cpu().numpy()).astype(np.float16)).astype(np.float64)).to(a.device)


def _ulp32(a):
    _, e = torch.frexp(a)
    return torch.where(a > 0, torch.ldexp(torch.ones_like(a), (e - 24).clamp_min(-149)), torch.full_like(a, 2.0 ** -149))


# ================================================================================================ conv_umma_f16
C16 = collections.namedtuple("C16", "name n H W segC Cout KH KW act pre res post bn tile_w tile_m mode")
CASES = [
    C16("scan 3x3, M128 16x8, BN128, out16", 1, 30, 54, [128], 128, 3, 3, "leaky", True, False, False, 128, 8, 128, "out16"),
    C16("scan 3x3, M128 8x16, BN64, dual store + res", 1, 60, 108, [128], 128, 3, 3, "none", False, True, False, 64, 16, 128, "dual"),
    C16("conv_offset.6: Cout 432 (ragged N tile), fp32 out", 1, 20, 27, [128], 432, 3, 3, "none", False, False, False, 128, 16, 128, "out"),
    C16("two state segments, M64 8x8, BN32", 2, 17, 23, [128, 128], 128, 3, 3, "leaky", True, False, False, 32, 8, 64, "out16"),
    C16("four segments 72/56/8/1, n=3, ragged rows", 3, 19, 13, [72, 56, 8, 1], 36, 3, 3, "relu", True, True, True, 32, 8, 64, "dual"),
    C16("three segments, M64 4x16, BN64, sigmoid", 2, 9, 37, [128, 128, 2], 64, 3, 3, "sigmoid", False, True, False, 64, 16, 64, "dual"),
    C16("deformable GEMM 1152 cols: grouped", 2, 13, 11, [1152], 128, 1, 1, "none", False, False, False, 128, 8, 128, "dual"),
    C16("deformable GEMM 2304 cols: grouped", 1, 21, 19, [2304], 128, 1, 1, "none", False, False, False, 128, 16, 128, "dual"),
    C16("1x1 ungrouped 2 blocks, tanh", 1, 9, 37, [128], 132, 1, 1, "tanh", True, False, False, 64, 8, 128, "out"),
    C16("1x1 grouped ragged segments [520, 96]", 1, 30, 54, [520, 96], 128, 1, 1, "leaky", False, True, True, 128, 8, 64, "out16"),
    C16("map smaller than one tile", 1, 5, 6, [40], 128, 3, 3, "none", True, True, True, 128, 8, 128, "dual"),
    C16("1x1 map, BN32", 2, 1, 1, [24], 36, 3, 3, "leaky", False, True, True, 32, 8, 64, "out16"),
]


def check_conv16(c, gen, slope=0.1):
    """run case c through conv_umma_f16 and bound every element by the float64 conv of the same fp16 operands; returns the
    worst err / bound"""
    from propainter_b200 import ops
    n, H, W, Cout = c.n, c.H, c.W, c.Cout
    plan = ops.conv_plan([(n, H, W, C) for C in c.segC], c.KH, c.KW, Cout, bn=c.bn, tile_w=c.tile_w, tile_m=c.tile_m, half=True)
    if c.bn:
        assert plan.bn == c.bn and plan.tile_w == c.tile_w and plan.tile_h * plan.tile_w == c.tile_m, (c.name, plan)
    segs, xs = [], []
    for C in c.segC:                                      # channel slices of wider NaN buffers, 16-byte aligned
        b = _nan((n, H, W, _r8(C) + 16), torch.float16)
        x = (torch.randn(n, H, W, C, generator=gen) * 2).half()
        b[..., 8:8 + C] = x.to(DEV)
        segs.append(b[..., 8:8 + C])
        xs.append(x.to(DEV).double())
    Cin = sum(c.segC)
    w = torch.randn(Cout, Cin, c.KH, c.KW, generator=gen) / (Cin * c.KH * c.KW) ** 0.5
    wp = ops.pack_conv_weight_f16(w.to(DEV), c.segC)
    w64 = w.half().double().to(DEV)
    bias = (torch.randn(Cout, generator=gen) * 0.5).to(DEV)
    pre = _nan((n, H, W, Cout + 4))
    pre[..., :Cout] = torch.randn(n, H, W, Cout, generator=gen).to(DEV)
    res = _nan((n, H, W, Cout + 4))
    res[..., :Cout] = torch.randn(n, H, W, Cout, generator=gen).to(DEV)
    out = _nan((n, H, W, Cout + 4)) if c.mode in ("out", "dual") else None
    out16 = _nan((n, H, W, _r8(Cout) + 8), torch.float16) if c.mode in ("out16", "dual") else None
    ops.conv_umma_f16(segs, wp, c.KH, c.KW, Cout, bias=bias, act=c.act, slope=slope, pre=pre[..., :Cout] if c.pre else None,
                      res=res[..., :Cout] if c.res else None, post_relu=c.post, out=out[..., :Cout] if out is not None else None,
                      out16=out16[..., :Cout] if out16 is not None else None)
    torch.cuda.synchronize()
    pad = (c.KH // 2, c.KW // 2)
    x64 = torch.cat(xs, -1).permute(0, 3, 1, 2)
    conv = F.conv2d(x64, w64, padding=pad).permute(0, 2, 3, 1) + bias.double()
    S = F.conv2d(x64.abs(), w64.abs(), padding=pad).permute(0, 2, 3, 1) + bias.double().abs()
    if c.pre:
        conv = conv + pre[..., :Cout].double()
        S = S + pre[..., :Cout].double().abs()
    a = ACTS[c.act](conv, slope)
    ref = a + res[..., :Cout].double() if c.res else a
    if c.post:
        ref = ref.clamp_min(0)
    lip = 0.25 if c.act == "sigmoid" else 1.0
    mag = a.abs() + (res[..., :Cout].double().abs() if c.res else 0) + ref.abs()
    bound = lip * TAU * S + 4 * _ulp32(mag)
    worst = 0.0
    for got, extra in ((out, 0), (out16, 0.5)):
        if got is None:
            continue
        assert torch.isnan(got[..., Cout:]).all(), f"{c.name}: wrote past Cout"
        b = bound + (extra * _ulp16(ref.abs() + bound) if extra else 0)
        err = (got[..., :Cout].double() - ref).abs()
        assert bool((err <= b).all()), (c.name, (err - b).max().item())
        worst = max(worst, (err / b).max().item())
    return worst, plan


@pytest.mark.parametrize("c", CASES, ids=[c.name for c in CASES])
def test_conv_umma_f16_f64(c):
    gen = torch.Generator().manual_seed(zlib.crc32(c.name.encode()) & 0xFFFF)
    worst, plan = check_conv16(c, gen)
    print(f"[conv_umma_f16] {c.name}: plan {plan}, worst err/bound {worst:.3f}")


def test_conv_umma_f16_every_act():
    gen = torch.Generator().manual_seed(7)
    for act in ACTS:
        c = C16(f"act {act}", 1, 11, 19, [64], 64, 3, 3, act, True, True, act == "tanh", 0, 0, 0, "dual")
        check_conv16(c, gen, slope=0.2)


def test_conv_umma_f16_refuses_misaligned():
    from propainter_b200 import ops
    x = torch.zeros(1, 4, 4, 72, device=DEV, dtype=torch.float16)
    wp = torch.zeros(8, 9 * 64, device=DEV, dtype=torch.float16)
    with pytest.raises(RuntimeError):                                 # ld 72 is fine, a 4-element offset is not 16-byte aligned
        ops.conv_umma_f16([x[..., 4:68]], wp, 3, 3, 8)
    with pytest.raises(RuntimeError):                                 # fp32 segments are refused by the fp16 entry
        ops.conv_umma_f16([x[..., :64].float()], wp, 3, 3, 8)


def _record_f16_convs(monkeypatch):
    """signatures of every conv_umma_f16 call of both nets with plan 0 forced under half_convs"""
    from propainter_b200 import config, ops
    from propainter_b200.model.propainter import InpaintGenerator
    from propainter_b200.model.recurrent_flow_completion import RecurrentFlowCompleteNet
    monkeypatch.setattr(config, "UMMA_CONV", True)
    monkeypatch.setattr(config, "HALF_OPERANDS", True)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", True)
    real = ops.conv_umma_f16
    seen = {"rfc": set(), "gen": set()}
    now = {"net": None}

    def rec(segs, w_packed, KH, KW, Cout, bias=None, act="none", slope=0.0, pre=None, res=None, post_relu=False, out=None,
            out16=None, **kw):
        seen[now["net"]].add((tuple(s.shape[-1] for s in segs), Cout, KH, KW, act, float(slope), pre is not None, res is not None,
                              bool(post_relu), bias is not None, out is not None, out16 is not None))
        return real(segs, w_packed, KH, KW, Cout, bias, act, slope, pre, res, post_relu, out, out16, **kw)
    monkeypatch.setattr(ops, "conv_umma_f16", rec)
    gen = torch.Generator().manual_seed(0)
    T, H, W = 5, 64, 96
    flows = tuple((torch.randn(1, T - 1, 2, H, W, generator=gen) * 3).to(DEV) for _ in range(2))
    masks = torch.zeros(1, T, 1, H, W, device=DEV)
    masks[..., 16:48, 24:72] = 1
    now["net"] = "rfc"
    RecurrentFlowCompleteNet(None, seed=2).to(DEV).forward_bidirect_flow(flows, masks)
    Hg, Wg, t, lt = 128, 128, 5, 3
    frames = (torch.rand(1, t, 3, Hg, Wg, generator=gen) * 2 - 1).to(DEV)
    fl = tuple((torch.randn(1, lt - 1, 2, Hg, Wg, generator=gen) * 4).to(DEV) for _ in range(2))
    m = torch.zeros(1, t, 1, Hg, Wg, device=DEV)
    m[..., Hg // 4:Hg // 2, Wg // 3:2 * Wg // 3] = 1
    now["net"] = "gen"
    InpaintGenerator(seed=3).to(DEV).forward_parts(frames * (1 - m), fl, m, m, lt)
    monkeypatch.setattr(ops, "conv_umma_f16", real)
    return seen


def test_production_f16_conv_shapes(monkeypatch):
    """every conv signature the fp16 scans issue, at the C2 map sizes (flow completion 30x54, generator 60x108) with the
    plan the planner picks there"""
    seen = _record_f16_convs(monkeypatch)
    assert len(seen["rfc"]) >= 6 and len(seen["gen"]) >= 6, seen
    assert any(s[0] == (2304,) for s in seen["rfc"]) and any(s[0] == (1152,) for s in seen["gen"])
    assert any(s[0] == (128, 128) for s in seen["rfc"])                       # conv_offset.0 over the two fp16 states
    gen = torch.Generator().manual_seed(11)
    for net, (H, W) in (("rfc", (30, 54)), ("gen", (60, 108))):
        for segC, Cout, KH, KW, act, slope, pre, res, post, bias, o32, o16 in sorted(seen[net]):
            mode = "dual" if o32 and o16 else "out" if o32 else "out16"
            c = C16(f"{net} {segC}->{Cout} {KH}x{KW} {act}", 1, H, W, list(segC), Cout, KH, KW, act, pre, res, post, 0, 0, 0, mode)
            worst, plan = check_conv16(c, gen, slope=slope or 0.1)
            print(f"[production f16] {c.name} {mode}: plan {plan}, worst err/bound {worst:.3f}")


# ================================================================================================ fp16 gather and warp
def _check_rn16(got, ref, E, what):
    """fp16 `got` is the float64 `ref` (within the fp32 sum error E) rounded to nearest once"""
    bound = E + 0.5 * _ulp16(ref.abs() + E)
    err = (got.double() - ref).abs()
    assert bool((err <= bound).all()), (what, (err - bound).max().item())
    return (err / bound.clamp_min(1e-30)).max().item()


def test_deform_gather_f16_f64():
    from propainter_b200 import ops
    gen = torch.Generator().manual_seed(40)
    for c in GATHER_CASES:
        if c.kind != "rand":
            continue
        xv, o, ob, flow = _gather_inputs(c, gen)
        n, H, W, Cin = c.n, c.H, c.W, c.Cin
        hc = Cin // 2
        xb1, xb2 = _nan((n, H, W, Cin + 8)), _nan((n, H, W, Cin + 8))
        if c.x2:
            xb1[..., :hc] = xv[..., :hc].to(DEV)
            xb2[..., 4:4 + hc] = xv[..., hc:].to(DEV)
            x, x2 = xb1[..., :hc], xb2[..., 4:4 + hc]
        else:
            xb1[..., 4:4 + Cin] = xv.to(DEV)
            x, x2 = xb1[..., 4:4 + Cin], None
        obuf = _nan((n, H, W, 436))
        obuf[..., :432] = o.to(DEV)
        N, pad = n * H * W * 9 * Cin, 64
        flat = _nan((N + 2 * pad,), torch.float16)
        cols = flat[pad:pad + N].view(n, H, W, 9 * Cin)
        fl = flow.to(DEV) if flow is not None else None
        ops.deform_gather(x, obuf[..., :432], fl, c.max_res, cols, o_bias=ob.to(DEV) if ob is not None else None, x2=x2)
        torch.cuda.synchronize()
        assert torch.isnan(flat[:pad]).all() and torch.isnan(flat[pad + N:]).all(), "pp_deform_gather_f16 wrote outside cols"
        got = cols.view(n, H * W, 9, Cin)
        x64, o32 = xv.to(DEV).double(), _o_eff(o, ob)
        worst = 0.0
        for k in range(9):
            ref, E = R.deform_cols_ref(x64, o32, fl, c.max_res, k)
            worst = max(worst, _check_rn16(got[:, :, k], ref, E, c.label))
        print(f"[deform_gather_f16] {c.label}: worst err/(E + ulp/2) {worst:.3f}")


def test_flow_warp_f16_f64():
    from propainter_b200 import ops
    gen = torch.Generator().manual_seed(42)
    for c in WARP_CASES:
        if not c.want_warp or c.kind != "rand":
            continue
        n, h, w, C = c.n, c.h, c.w, c.C
        fprop, fcheck = _flow_pair(gen, n, h, w)
        feat = torch.randn(n, h, w, C, generator=gen)
        fb = _nan((n, h, w, C + 8))
        fb[..., 4:4 + C] = feat.to(DEV)
        wb = _nan((n, h, w, C + 8), torch.float16)
        aux_b = _nan((n, h, w, c.aux_ld)) if c.aux_ld else None
        _, aux = ops.flow_warp_fbcheck(fb[..., 4:4 + C], fprop.to(DEV), fcheck.to(DEV) if c.aux_ld else None, warped=wb[..., :C],
                                       aux=aux_b[..., :3] if c.aux_ld else None)
        torch.cuda.synchronize()
        assert torch.isnan(wb[..., C:]).all()
        ix, iy = R.warp_positions(fprop)
        ref, E = R.warp_sample(feat.to(DEV).double(), ix, iy)
        worst = _check_rn16(wb[..., :C].reshape(n, h * w, C), ref, E, c.label)
        if c.aux_ld:                                                   # the validity is the fp32 entry's, bit for bit
            a32 = _nan((n, h, w, c.aux_ld))
            ops.flow_warp_fbcheck(None, fprop.to(DEV), fcheck.to(DEV), aux=a32[..., :3], want_warp=False)
            assert torch.equal(aux, a32[..., :3])
        print(f"[flow_warp_f16] {c.label}: worst err/(E + ulp/2) {worst:.3f}")


# ================================================================================================ scans and nets
@contextlib.contextmanager
def _switches(half, tf32=True):
    """plan 0 (the wgmma scan) forced, run eagerly (the fp16 range probes read values back); half: fp16 operands"""
    from propainter_b200 import config
    prev = (config.HALF_OPERANDS, config.UMMA_CONV, config.LINEAR_TF32, config.CUDA_GRAPHS, torch.backends.cuda.matmul.allow_tf32,
            torch.backends.cudnn.allow_tf32)
    config.HALF_OPERANDS, config.UMMA_CONV, config.LINEAR_TF32, config.CUDA_GRAPHS = half, True, tf32, False
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = tf32
    try:
        yield
    finally:
        (config.HALF_OPERANDS, config.UMMA_CONV, config.LINEAR_TF32, config.CUDA_GRAPHS, torch.backends.cuda.matmul.allow_tf32,
         torch.backends.cudnn.allow_tf32) = prev


def rel_err(a, b):
    return (a.float() - b.float()).abs().max().item() / max(b.abs().max().item(), 1e-12)


@contextlib.contextmanager
def _peaks():
    """largest |value| of every fp16 tensor the scans hand to a kernel (conv operands and outputs, columns, warped maps)"""
    from propainter_b200 import ops
    peak = collections.defaultdict(float)
    real = {k: getattr(ops, k) for k in ("conv_umma_f16", "deform_gather", "flow_warp_fbcheck")}

    def note(k, t):
        if t is not None and t.dtype == torch.float16:
            assert bool(torch.isfinite(t).all()), k
            peak[k] = max(peak[k], t.float().abs().max().item())

    def conv(segs, w, KH, KW, Cout, *a, **k):
        r = real["conv_umma_f16"](segs, w, KH, KW, Cout, *a, **k)
        for i, s in enumerate(segs):
            note(f"conv operand {tuple(x.shape[-1] for x in segs)}->{Cout}", s)
        note(f"conv out16 ->{Cout} {KH}x{KW}", k.get("out16"))
        return r

    def gather(*a, **k):
        r = real["deform_gather"](*a, **k)
        note("deform columns", r)
        return r

    def warp(*a, **k):
        r = real["flow_warp_fbcheck"](*a, **k)
        note("warped features", r[0])
        return r
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(ops, "conv_umma_f16", conv)
        mp.setattr(ops, "deform_gather", gather)
        mp.setattr(ops, "flow_warp_fbcheck", warp)
        yield peak


def _rfc_inputs(T, H, W, seed=0):
    gen = torch.Generator().manual_seed(seed)
    sm = lambda z: F.avg_pool2d(z.reshape(-1, 2, H, W), 9, 1, 4).view(z.shape)
    flows = tuple(sm(torch.randn(1, T - 1, 2, H, W, generator=gen) * 12).to(DEV) for _ in range(2))
    masks = torch.zeros(1, T, 1, H, W)
    masks[..., H // 4:H // 2, W // 3:2 * W // 3] = 1
    return flows, masks.to(DEV)


def test_flow_completion_half_scan_vs_tf32():
    """an RFC clip of C2 size (80 frames of 240x432: 30x54 scan maps)"""
    from oracle import flowcomp_ref
    from propainter_b200.model.recurrent_flow_completion import RecurrentFlowCompleteNet
    net = RecurrentFlowCompleteNet(None, seed=2).to(DEV)
    flows, masks = _rfc_inputs(80, 240, 432)
    sd = {k: v.detach() for k, v in net.state_dict().items()}
    with _switches(False, tf32=False):
        ref = flowcomp_ref.forward_bidirect_flow(sd, flows, masks)
    errs = {}
    for half in (False, True):
        with _switches(half), (_peaks() if half else contextlib.nullcontext({})) as peak:
            pred, _ = net.forward_bidirect_flow(flows, masks)
        errs[half] = max(rel_err(a, b) for a, b in zip(pred, ref))
        if half:
            print("[rfc] max |fp16 tensor|:", {k: round(v, 2) for k, v in sorted(peak.items())})
            assert peak and max(peak.values()) < 6e4
    print(f"[rfc] C2 clip rel err vs oracle: TF32 plan 0 {errs[False]:.3e}, fp16 plan 0 {errs[True]:.3e}")
    assert errs[True] < 2e-3
    assert errs[True] <= 1.5 * errs[False] + 1e-6


def test_generator_half_scan_vs_tf32():
    """a synthetic C2 window (18 frames, 11 local, 240x432: 60x108 scan maps).  The 1.5x bar is on the scan's output (the
    propagated local features, which nothing else under the switch touches); the generator's output also carries the
    fp16 trunk and transformer and is held to the generator's own bound"""
    from oracle import generator_ref
    from propainter_b200.model.propainter import InpaintGenerator
    H, W, t, lt = 240, 432, 18, 11
    gen = torch.Generator().manual_seed(1)
    frames = (torch.rand(1, t, 3, H, W, generator=gen) * 2 - 1).to(DEV)
    flows, _ = _rfc_inputs(lt, H, W, seed=3)
    masks = torch.zeros(1, t, 1, H, W, device=DEV)
    masks[..., H // 4:H // 2, W // 3:2 * W // 3] = 1
    mf = frames * (1 - masks)
    net = InpaintGenerator(seed=3).to(DEV)
    sd = {k: v.detach() for k, v in net.state_dict().items()}
    with _switches(False, tf32=False):
        ref, rparts = generator_ref.generator_forward(sd, mf, flows, masks, masks, lt, return_parts=True)
    rp = rparts["prop_feat"][0]
    errs = {}
    for half in (False, True):
        with _switches(half), (_peaks() if half else contextlib.nullcontext({})) as peak:
            out, parts = net.forward_parts(mf, flows, masks, masks, lt)
        pf = parts["prop_feat"]
        assert pf.numel() == rp.numel()
        errs[half] = {"scan": rel_err(pf.reshape(rp.shape), rp), "out": rel_err(out, ref)}
        if half:
            print("[gen] max |fp16 tensor|:", {k: round(v, 2) for k, v in sorted(peak.items())})
            assert peak and max(peak.values()) < 6e4
    print(f"[gen] C2 window rel err vs oracle: TF32 {errs[False]}, fp16 {errs[True]}")
    assert errs[True]["out"] < 5e-3 and errs[True]["scan"] < 5e-3
    assert errs[True]["scan"] <= 1.5 * errs[False]["scan"] + 1e-5


def test_strict_fp32_scans_unchanged():
    """with cuDNN TF32 off the switch changes nothing: both scans bit for bit with HALF_OPERANDS on and off"""
    from propainter_b200.model.propainter import InpaintGenerator
    from propainter_b200.model.recurrent_flow_completion import RecurrentFlowCompleteNet
    gen = torch.Generator(device=DEV).manual_seed(0)
    rfc, g = RecurrentFlowCompleteNet(None, seed=2).to(DEV), InpaintGenerator(seed=3).to(DEV)
    x = torch.randn(20, 128, 30, 54, device=DEV, generator=gen).contiguous(memory_format=torch.channels_last)
    xl = torch.randn(6, 60, 108, 128, device=DEV, generator=gen)
    ds = [torch.randn(5, 60, 108, 2, device=DEV, generator=gen) * 3 for _ in range(2)]
    pm = (torch.rand(6, 60, 108, 2, device=DEV, generator=gen) > 0.5).float()
    res = {}
    for half in (False, True):
        with _switches(half, tf32=False):
            res[half] = (rfc._propagate_umma(x), g._feat_propagation_umma(xl, ds[0], ds[1], pm))
    assert all(torch.equal(a, b) for a, b in zip(res[False], res[True]))
