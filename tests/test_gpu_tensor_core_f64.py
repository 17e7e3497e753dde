"""The two wgmma kernels against float64 references, per element, over their tile plans and the model's call shapes.

pp_conv2d_umma (implicit-GEMM convolution) and pp_sparse_window_attn (masked-window attention) are the TF32 tensor-core
hot paths of both propagation scans and of every transformer block.  Their older tests (test_gpu_ops.py) compare a few
hand-picked shapes at a fraction of the output maximum.  Here:

  * every conv case names the tile / ring plan it exercises, checks it against ops.conv_plan and a restatement of the
    ring-depth rule, and bounds every element by its own float64 error budget; altered copies of the reference (one tap
    dropped, a one-pixel shift, a zeroed channel tile or tile row) must fail that same bound, so the bound is not vacuous;
  * the convolutions the generator and the flow-completion net actually launch are recorded, planned at production map
    sizes and batch counts, and every distinct plan is run through the same check;
  * the attention runs on both implementations against oracle/attn_table_ref over the kernels' edges (ragged query and
    key tiles, the key-table limit, window sizes that select the fallback kernels, empty key sets, flag patterns), with
    diffuse and with peaked softmaxes whose winning key sits where a gather mistake would move it.
"""
import collections
import math
import zlib

import pytest
import torch
import torch.nn.functional as F

from oracle import attn_table_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"

# ================================================================================================ convolution
SMEM_BUDGET = 216 * 1024           # CV_SMEM_BUDGET (conv_umma.cu): both rings together
SENTINEL = -12345.5
# Per-element bound |out - ref_out| <= L_act * TAU * S + 4 ulp, with ref_out the float64 epilogue of the float64 conv of
# the operands the tensor core reads (TF32 weights, activations with the low 13 mantissa bits cleared: wgmma kind tf32
# truncates fp32 operands), S the same conv of |x| |w| plus |bias| + |pre|, L_act the Lipschitz constant of the
# activation (1/4 for sigmoid).  The 4 ulp are of |act| + |res| + |ref_out|: the fp32 epilogue rounds each of them.
# On an H100 the largest err / (L_act * S) is about 1e-6 (fp32 accumulation), 15x under TAU; against round-to-nearest
# operands it is about 1e-4, so a kernel that rounded instead of truncating, or dropped one k-block, fails.
TAU = 2.0 ** -16


@pytest.fixture(autouse=True)
def _exact_library_math():
    """torch's float32 convs / matmuls without TF32 (the references below are float64 anyway)."""
    a, b = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = a, b


def ring_plan(segC, KH, KW, bn, tile_h, tile_w):
    """cv_plan's ring-depth rule (conv_umma.cu) restated: A ring of na slots (one per 32-channel block, or per group of 4
    blocks for a 1x1 conv with >= 8 blocks), B ring of nb slots (one per (block, dy)), deferred slot release only when both
    rings have two or more slots.  None where the rings do not fit."""
    kb = [(c + 31) // 32 for c in segC]
    group = KH == 1 and KW == 1 and sum(kb) >= 8
    kw = 4 if group else KW
    nblk = sum((k + 3) // 4 for k in kb) if group else sum(kb)
    a_slot, b_slot = kw * (tile_h + KH - 1) * tile_w * 128, kw * bn * 128
    na = min(4 if KH * KW == 1 and not group else 2, nblk)
    if na * a_slot + b_slot > SMEM_BUDGET:
        na = 1
    if na * a_slot + b_slot > SMEM_BUDGET:
        return None
    nb = min((SMEM_BUDGET - na * a_slot) // b_slot, 8, nblk * KH)
    while na < 6 and na < nblk and (na + 1) * a_slot + nb * b_slot <= SMEM_BUDGET:
        na += 1
    return dict(na=na, nb=nb, group=group, defer=na >= 2 and nb >= 2, smem=na * a_slot + nb * b_slot + 1536)


Case = collections.namedtuple("Case", "name n H W segC Cout KH KW act pre res post bn tile_w tile_m slope plan")
ACTS = {"none": (lambda v, s: v), "relu": (lambda v, s: v.clamp_min(0)), "leaky": (lambda v, s: torch.where(v > 0, v, v * s)),
        "sigmoid": (lambda v, s: torch.sigmoid(v)), "tanh": (lambda v, s: torch.tanh(v))}
P, R, X = True, True, False
# plan: (tile_h, tile_w, bn, na, nb, grouped, deferred)
CASES = [
    Case("scan 3x3 conv, 16x8 tiles, deferred release", 1, 30, 54, [128], 128, 3, 3, "leaky", P, R, X, 128, 8, 128, 0.1,
         (16, 8, 128, 2, 2, False, True)),
    Case("conv_offset.6: ragged last N tile (Cout 432)", 1, 20, 27, [128], 432, 3, 3, "none", X, X, X, 128, 16, 128, 0.1,
         (8, 16, 128, 2, 2, False, True)),
    Case("fuse.0: three segments [128, 128, 2]", 2, 17, 23, [128, 128, 2], 128, 3, 3, "leaky", X, X, X, 64, 16, 128, 0.2,
         (8, 16, 64, 2, 4, False, True)),
    Case("four segments of 33/31/5/1 channels, n = 3 with ragged tile rows", 3, 19, 13, [33, 31, 5, 1], 36, 3, 3, "relu", P, R, P,
         32, 8, 64, 0.1, (8, 8, 32, 4, 8, False, True)),
    Case("deformable GEMM over 2304 columns: grouped, one-slot B ring", 1, 21, 19, [2304], 128, 1, 1, "none", X, X, X, 128, 8, 128,
         0.1, (16, 8, 128, 2, 1, True, False)),
    Case("deformable GEMM over 1152 columns: grouped, one-slot B ring", 2, 13, 11, [1152], 128, 1, 1, "none", X, X, X, 128, 16,
         128, 0.1, (8, 16, 128, 2, 1, True, False)),
    Case("1x1 with 4 k-blocks: ungrouped 4-slot A ring (Cout 132)", 1, 9, 37, [128], 132, 1, 1, "tanh", P, X, X, 64, 8, 128, 0.1,
         (16, 8, 64, 4, 4, False, True)),
    Case("1x1 grouped with ragged segment ends [160, 96]", 1, 30, 54, [160, 96], 128, 1, 1, "sigmoid", X, R, X, 128, 8, 128, 0.1,
         (16, 8, 128, 2, 1, True, False)),
    Case("5x5: one-slot A ring (Cout 4)", 2, 17, 9, [32], 4, 5, 5, "sigmoid", P, X, P, 32, 8, 128, 0.1,
         (16, 8, 32, 1, 5, False, False)),
    Case("7x7 on a 37x1 map: one-slot A ring, 2-channel segment", 1, 37, 1, [2], 128, 7, 7, "tanh", X, R, P, 32, 8, 128, 0.1,
         (16, 8, 32, 1, 2, False, False)),
    Case("1x37 map, 4x16 tiles", 1, 1, 37, [5], 128, 3, 3, "relu", X, X, X, 64, 16, 64, 0.1, (4, 16, 64, 1, 3, False, False)),
    Case("1x1 maps, 8x8 tiles", 2, 1, 1, [31], 36, 3, 3, "leaky", X, R, P, 32, 8, 64, 0.1, (8, 8, 32, 1, 3, False, False)),
    Case("map smaller than one tile", 1, 5, 6, [33], 128, 3, 3, "none", P, R, P, 128, 8, 128, 0.1, (16, 8, 128, 2, 2, False, True)),
    Case("map one pixel past a tile edge", 1, 17, 9, [128], 128, 3, 3, "none", X, X, X, 128, 8, 128, 0.1,
         (16, 8, 128, 2, 2, False, True)),
    Case("two state segments, 8x16 tiles", 2, 30, 54, [128, 128], 128, 3, 3, "leaky", P, X, X, 64, 16, 128, 0.1,
         (8, 16, 64, 2, 4, False, True)),
    Case("SepConvGRU 1x5: one slot in both rings", 2, 12, 20, [256], 128, 1, 5, "tanh", X, X, X, 128, 16, 128, 0.1, (8, 16, 128, 1, 1, False, False)),
]


def _ulp32(a):
    """ulp of the float32 values of magnitude `a` (float64 tensor)."""
    _, e = torch.frexp(a)
    return torch.where(a > 0, torch.ldexp(torch.ones_like(a), (e - 24).clamp_min(-149)), torch.full_like(a, 2.0 ** -149))


def _trunc13(x):
    """what the tensor core reads of an fp32 operand: the low 13 mantissa bits cleared."""
    return (x.contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


def _epilogue(pre_act, c, res, act, slope):
    a = ACTS[act](pre_act, slope)
    out = a + res if res is not None else a
    return (out.clamp_min(0) if c.post else out), a


def _conv64(xs, w):
    """float64 conv of the channel-concatenated [n,H,W,C] input with w [Cout,Cin,KH,KW] -> [n,H,W,Cout]."""
    KH, KW = w.shape[-2:]
    return F.conv2d(torch.cat(xs, -1).permute(0, 3, 1, 2), w, padding=(KH // 2, KW // 2)).permute(0, 2, 3, 1)


def check_conv(c, gen, label=None):
    """Run case `c` through conv_umma and bound every element by the float64 reference.  Returns the plan line printed."""
    from propainter_b200 import ops
    n, H, W, Cout = c.n, c.H, c.W, c.Cout
    Cin = sum(c.segC)
    plan = ops.conv_plan([(n, H, W, C) for C in c.segC], c.KH, c.KW, Cout, bn=c.bn, tile_w=c.tile_w, tile_m=c.tile_m)
    ring = ring_plan(c.segC, c.KH, c.KW, plan.bn, plan.tile_h, plan.tile_w)
    tiles_y = (H + plan.tile_h - 1) // plan.tile_h
    ctas = ((W + plan.tile_w - 1) // plan.tile_w) * tiles_y * n * ((Cout + plan.bn - 1) // plan.bn)
    assert ring is not None and ring["smem"] == plan.smem_bytes and ctas == plan.ctas, (c.name, plan, ring)
    got_plan = (plan.tile_h, plan.tile_w, plan.bn, ring["na"], ring["nb"], ring["group"], ring["defer"])
    if c.plan is not None:
        assert got_plan == tuple(c.plan), (c.name, got_plan)
    slope = float(torch.tensor(c.slope, dtype=torch.float32))          # the kernel multiplies by the fp32 slope
    w = torch.randn(Cout, Cin, c.KH, c.KW, generator=gen) / math.sqrt(Cin * c.KH * c.KW)
    wr = ops.tf32_round(w).to(DEV)
    wp = ops.pack_conv_weight(w, c.segC).to(DEV)
    bias = torch.randn(Cout, generator=gen).to(DEV)
    # operands live in wider buffers whose extra channels are NaN: the kernel must read exactly C channels of each
    def poisoned(C, lo=0):
        buf = torch.full((n, H, W, lo + (C + 7) // 4 * 4), float("nan"), device=DEV)
        buf[..., lo:lo + C] = torch.randn(n, H, W, C, generator=gen).to(DEV)
        return buf[..., lo:lo + C]
    pre = poisoned(Cout) if c.pre else None
    res = poisoned(Cout, 4) if c.res else None
    worst = {}
    for mode in ("exact", "plain"):
        xs = [poisoned(C) for C in c.segC]
        if mode == "exact":
            for x in xs:
                x.copy_(ops.tf32_round(x))
        outs = {}
        for rnd in (False, True):
            obuf = torch.full((n, H, W, Cout + 12), SENTINEL, device=DEV)
            outs[rnd] = ops.conv_umma(xs, wp, c.KH, c.KW, Cout, bias=bias, act=c.act, slope=c.slope, pre=pre, res=res,
                                      post_relu=c.post, out=obuf[..., 8:8 + Cout], round_tf32=rnd, bn=c.bn, tile_w=c.tile_w,
                                      tile_m=c.tile_m)
            assert (obuf[..., :8] == SENTINEL).all() and (obuf[..., 8 + Cout:] == SENTINEL).all(), (c.name, "wrote outside out")
            assert torch.isfinite(outs[rnd]).all(), (c.name, mode, "non-finite output")
        assert torch.equal(outs[True], ops.tf32_round(outs[False])), (c.name, mode, "round_tf32 is not tf32_round of the output")
        out = outs[False].double()
        add = bias.double() + (pre.double() if pre is not None else 0)
        res64 = res.double() if res is not None else None
        xt = [_trunc13(x).double() for x in xs]
        S = _conv64([x.abs() for x in xt], wr.double().abs()) + bias.double().abs() + (pre.double().abs() if pre is not None else 0)
        L = 0.25 if c.act == "sigmoid" else 1.0

        def bound_of(ref_out, a):
            return L * TAU * S + 4 * _ulp32(a.abs() + (res64.abs() if res64 is not None else 0) + ref_out.abs())
        ref_pre = _conv64(xt, wr.double()) + add
        ref_out, a = _epilogue(ref_pre, c, res64, c.act, slope)
        bound = bound_of(ref_out, a)
        err = (out - ref_out).abs()
        worst[mode] = (err / (L * S)).max().item()
        if mode == "plain":        # the same comparison against round-to-nearest operands, for the record
            xr = [ops.tf32_round(x).double() for x in xs]
            rr, _ = _epilogue(_conv64(xr, wr.double()) + add, c, res64, c.act, slope)
            worst["plain, rounded operands"] = ((out - rr).abs() / (L * S)).max().item()
        assert (err <= bound).all(), (c.name, mode, worst[mode], (err / bound).max().item())
        # the same bound rejects a reference that is wrong in the ways a kernel goes wrong
        blk = torch.zeros_like(wr)
        blk[:, :min(32, c.segC[0]), c.KH // 2, c.KW // 2] = wr[:, :min(32, c.segC[0]), c.KH // 2, c.KW // 2]
        alts = {"one tap of one 32-channel block dropped": _epilogue(ref_pre - _conv64(xt, blk.double()), c, res64, c.act, slope)[0],
                "shifted by one pixel": ref_out.reshape(-1, Cout).roll(1, 0).view_as(ref_out)}
        z = ref_out.clone()
        z[..., (Cout - 1) // plan.bn * plan.bn:] = 0
        alts["last channel tile zeroed"] = z
        if n > 1:
            z = ref_out.clone()
            z[-1, (tiles_y - 1) * plan.tile_h:] = 0
            alts["last tile row of the last image zeroed"] = z
        for what, alt in alts.items():
            assert ((out - alt).abs() > bound).any(), (c.name, mode, f"bound accepts the reference with {what}")
    line = (f"{label or c.name}: BN {plan.bn}, tile {plan.tile_h}x{plan.tile_w}, na {ring['na']} nb {ring['nb']}, "
            f"{'grouped, ' if ring['group'] else ''}{'deferred' if ring['defer'] else 'immediate'} release; max err/(L*S): "
            + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()) + f" (tau = {TAU:.2e})")
    print(line)
    return line


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_conv_umma_f64(case):
    check_conv(case, torch.Generator().manual_seed(zlib.crc32(case.name.encode())))


def test_conv_cases_cover_the_plans():
    plans = []
    for c in CASES:
        th = (128 if c.tile_m != 64 else 64) // c.tile_w
        r = ring_plan(c.segC, c.KH, c.KW, c.bn, th, c.tile_w)
        assert r is not None and (th, c.tile_w, c.bn, r["na"], r["nb"], r["group"], r["defer"]) == tuple(c.plan), c.name
        plans.append((c, th, r))
    assert {c.bn for c in CASES} >= {32, 64, 128}
    assert {(th, c.tile_w) for c, th, _ in plans} >= {(16, 8), (8, 16), (8, 8), (4, 16)}
    assert any(r["defer"] for *_, r in plans)
    assert any(not r["defer"] and r["nb"] == 1 for *_, r in plans)
    assert any(r["na"] == 1 for *_, r in plans)
    ones = [(c, r) for c, _, r in plans if c.KH == c.KW == 1]
    assert any(r["group"] for _, r in ones) and any(not r["group"] for _, r in ones)
    assert any(r["group"] and len(c.segC) > 1 and any(C % 128 for C in c.segC) for c, r in ones)   # ragged group ends
    assert {len(c.segC) for c in CASES} >= {1, 2, 3, 4}
    assert {C for c in CASES for C in c.segC} >= {1, 2, 5, 31, 32, 33, 128, 1152, 2304}
    assert {c.KH * 10 + c.KW for c in CASES} >= {11, 33, 55, 77, 15}
    maps = {(c.H, c.W) for c in CASES}
    assert {(1, 1), (1, 37), (37, 1)} <= maps
    assert any(c.H < th and c.W < c.tile_w for c, th, _ in plans)
    assert any(c.H % th == 1 and c.W % c.tile_w == 1 for c, th, _ in plans)
    assert any(c.n == 3 and c.H % th for c, th, _ in plans)
    assert {c.Cout for c in CASES} >= {4, 36, 128, 132, 432}
    for act in ACTS:
        mine = [c for c in CASES if c.act == act]
        for flag in ("pre", "res", "post"):
            assert {getattr(c, flag) for c in mine} == {True, False}, (act, flag)


def test_conv_plan_refusals():
    from propainter_b200 import ops
    x = torch.zeros(1, 8, 8, 32, device=DEV)
    shp = [(1, 8, 8, 32)]
    for KH, KW in ((2, 3), (3, 4), (9, 9), (1, 9)):
        with pytest.raises(RuntimeError):
            ops.conv_plan(shp, KH, KW, 32)
        with pytest.raises(RuntimeError):
            ops.conv_umma([x], torch.zeros(32, KH * KW * 32, device=DEV), KH, KW, 32)
    with pytest.raises(RuntimeError):
        ops.conv_plan(shp, 3, 3, 6)                                                    # Cout not a multiple of 4
    with pytest.raises(RuntimeError):
        ops.conv_umma([x], torch.zeros(6, 288, device=DEV), 3, 3, 6)
    with pytest.raises(RuntimeError):
        ops.conv_plan(shp * 5, 3, 3, 32)                                               # 5 segments
    with pytest.raises(RuntimeError):
        ops.conv_umma([x] * 5, torch.zeros(32, 5 * 288, device=DEV), 3, 3, 32)
    with pytest.raises(RuntimeError):
        ops.conv_umma([], torch.zeros(32, 0, device=DEV), 3, 3, 32)
    wide = torch.zeros(1, 8, 8, 38, device=DEV)[..., :32]                              # ld = 38: rows not 16-byte aligned
    with pytest.raises(RuntimeError):
        ops.conv_plan([wide], 3, 3, 32)
    with pytest.raises(RuntimeError):
        ops.conv_umma([wide], torch.zeros(32, 288, device=DEV), 3, 3, 32)
    assert ring_plan([32], 7, 7, 128, 8, 16) is None                                   # rings larger than shared memory
    with pytest.raises(RuntimeError):
        ops.conv_plan(shp, 7, 7, 128, bn=128, tile_w=16)
    with pytest.raises(RuntimeError):
        ops.conv_umma([x], torch.zeros(128, 49 * 32, device=DEV), 7, 7, 128, bn=128, tile_w=16)
    assert ops.conv_plan(shp, 7, 7, 128, bn=32, tile_w=8).smem_bytes == ring_plan([32], 7, 7, 32, 16, 8)["smem"]


# ------------------------------------------------------------------------------------------------ production call shapes
Sig = collections.namedtuple("Sig", "KH KW segC Cout act slope pre res post round_tf32 bias")
GEN_MAPS = [(s[0] // 4, s[1] // 4) for s in ((128, 128), (240, 432), (720, 1280), (1080, 1920), (2160, 3840))]
RFC_MAPS = [(s[0] // 8, s[1] // 8) for s in ((128, 128), (240, 432), (720, 1280), (1080, 1920), (2160, 3840))]
BATCHES = (1, 2, 5, 10, 20, 80)


def _record_model_convs(monkeypatch):
    """Signatures of every conv_umma call of RecurrentFlowCompleteNet and InpaintGenerator forward, each scan plan forced."""
    from propainter_b200 import autotune, config, ops
    from propainter_b200.model.propainter import InpaintGenerator
    from propainter_b200.model.recurrent_flow_completion import RecurrentFlowCompleteNet
    monkeypatch.setattr(config, "UMMA_CONV", "auto")
    real_pick, real_conv = autotune.pick, ops.conv_umma
    seen = {"rfc": set(), "gen": set()}
    net_of = {"now": None}
    plan = {"i": 0}

    def forced(key, variants, *a, **k):
        if key[0] in ("rfc_prop", "gen_prop"):
            return variants[min(plan["i"], len(variants) - 1)](*a)
        return real_pick(key, variants, *a, **k)

    def recording(segs, w_packed, KH, KW, Cout, bias=None, act="none", slope=0.0, pre=None, res=None, post_relu=False, out=None,
                  round_tf32=False, **kw):
        seen[net_of["now"]].add(Sig(KH, KW, tuple(s.shape[-1] for s in segs), Cout, act, float(slope), pre is not None,
                                    res is not None, bool(post_relu), bool(round_tf32), bias is not None))
        return real_conv(segs, w_packed, KH, KW, Cout, bias, act, slope, pre, res, post_relu, out, round_tf32, **kw)

    monkeypatch.setattr(autotune, "pick", forced)
    monkeypatch.setattr(ops, "conv_umma", recording)
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
        net_of["now"] = "rfc"
        RecurrentFlowCompleteNet(None, seed=2).to(DEV).forward_bidirect_flow(flows, masks)
        net_of["now"] = "gen"
        InpaintGenerator(seed=3).to(DEV).forward_parts(frames * (1 - m), fl, m, m, lt)
    monkeypatch.setattr(ops, "conv_umma", real_conv)
    monkeypatch.setattr(autotune, "pick", real_pick)
    return seen


def test_production_conv_shapes(monkeypatch):
    """Every distinct plan the planner picks for the model's conv signatures at production map sizes runs the float64
    check.  Ring depths depend on BN, the tile and K only, so a small ragged map with bn / tile forced runs the same
    pipeline as the large map."""
    from propainter_b200 import ops
    seen = _record_model_convs(monkeypatch)
    allsig = seen["rfc"] | seen["gen"]
    assert any(s.KH == 3 and s.segC == (128, 128, 2) for s in seen["gen"])            # fuse.0
    assert any(s.KH == 1 and s.segC == (1152,) and s.Cout == 128 for s in seen["gen"])  # generator deformable GEMM
    assert any(s.KH == 1 and s.segC == (2304,) and s.Cout == 128 for s in seen["rfc"])  # flow-completion deformable GEMM
    assert any(s.KH == 3 and s.Cout == 432 for s in allsig)                            # conv_offset.6
    todo = {}
    for net, maps in (("rfc", RFC_MAPS), ("gen", GEN_MAPS)):
        for s in seen[net]:
            for (h, w) in maps:
                for nb in BATCHES:
                    p = ops.conv_plan([(nb, h, w, C) for C in s.segC], s.KH, s.KW, s.Cout)
                    todo.setdefault((s, p.bn, p.tile_h, p.tile_w), (h, w, nb))
    # the one-slot B ring of the deformable GEMMs is what production runs at 720p and above
    deferred = {k: ring_plan(k[0].segC, k[0].KH, k[0].KW, k[1], k[2], k[3])["defer"] for k in todo}
    assert any(k[0].segC == (2304,) and not d for k, d in deferred.items())
    assert any(k[0].segC == (1152,) and not d for k, d in deferred.items())
    gen = torch.Generator().manual_seed(1)
    for (s, bn, th, tw), where in sorted(todo.items(), key=str):
        c = Case(f"{s}", 2, 2 * th + 1, 2 * tw + 3, list(s.segC), s.Cout, s.KH, s.KW, s.act, s.pre, s.res, s.post, bn, tw, 128,
                 s.slope or 0.1, None)
        check_conv(c, gen, label=f"{s.KH}x{s.KW} {list(s.segC)}->{s.Cout} {s.act} (first seen at {where[0]}x{where[1]}, n={where[2]})")


# ================================================================================================ attention
C_ATT = 512
# per query row and head, relative to the largest |v| of the row's key set.  The kernels round P and the scaled q to
# TF32; on an H100 the largest error is about 2^-12.5 of that |v|.
ATT_TOL = 2.0 ** -10
Att = collections.namedtuple("Att", "name t nwin WN NKO NP flags kf_start kf_step")
ATT_CASES = [
    Att("t=37 WN=45: last query tile has one row", 37, 2, 45, 45, 4, "alt", 0, 2),
    Att("257 keys (NKO 193 + 64 pooled, one key frame): last key tile has one key", 2, 5, 45, 193, 64, "all1", 1, 2),
    Att("255 keys, WN=48", 3, 5, 48, 193, 62, "alt", 2, 1),
    Att("NKO=224, WN=49 (fallback unmasked kernel), 4 key frames step 1", 4, 5, 49, 224, 16, "alt", 0, 1),
    Att("WN=64, 3 key frames step 2", 5, 3, 64, 100, 8, "alt", 0, 2),
    Att("WN=1", 6, 8, 1, 7, 5, "alt", 0, 2),
    Att("one-frame clip on an odd layer: no key frame", 1, 5, 45, 193, 12, "alt", 1, 2),
    Att("flags all 0", 3, 5, 45, 193, 12, "all0", 0, 2),
    Att("unmasked: 8 frames per CTA, t=13", 13, 36, 45, 45, 4, "alt", 1, 2),
]


def _att_problem(a, gen):
    """TF32-representable qkv / pool_kv and a key table whose own-token blocks partition the NT tokens; the rest of a
    window's table is other windows' tokens, each at most once (a repeated key would share the peak of a peaked row)."""
    from propainter_b200 import ops
    NT = a.nwin * a.WN
    perm = torch.randperm(NT, generator=gen)
    tab = torch.empty(a.nwin, a.NKO, dtype=torch.int32)
    for w in range(a.nwin):
        own = perm[w * a.WN:(w + 1) * a.WN]
        rest = perm[torch.randperm(NT, generator=gen)]
        rest = rest[~torch.isin(rest, own)][:a.NKO - a.WN]
        assert len(rest) == a.NKO - a.WN, "not enough tokens for a table without repeats"
        tab[w] = torch.cat([own, rest]).int()
    flags = {"all0": torch.zeros(a.nwin), "all1": torch.ones(a.nwin), "alt": torch.arange(a.nwin) % 2 == 0}[a.flags].int()
    qkv = ops.tf32_round(torch.randn(a.t, NT, 3 * C_ATT, generator=gen))
    pool = ops.tf32_round(torch.randn(a.t, a.NP, 2 * C_ATT, generator=gen))
    return qkv.to(DEV), pool.to(DEV), tab.to(DEV), flags.to(DEV)


def _peak(qkv, pool, tab, flags, t, WN, kf_start, kf_step, targets):
    """Make the softmax of every masked query row peaked on one key: q row = 2 * (the target's k row), so the target
    carries >= 0.9 of the weight in every head.  targets(nkeys, tab_row, window) -> candidate key indices; the rows of a
    window cycle through them.  Returns [(window, frames, tokens, key index)], one entry per (window, target)."""
    from propainter_b200 import ops
    kfs = list(range(kf_start, t, kf_step))
    peaks = []
    if not kfs:
        return peaks
    for w in torch.nonzero(flags).view(-1).tolist():
        K, _ = attn_table_ref.masked_keys(qkv, pool, tab[w].long(), kfs)
        cand = targets(K.shape[0], tab[w], w)
        own = tab[w, :WN].long()
        r = torch.arange(t * WN, device=qkv.device)
        for k, j in enumerate(cand):
            sel = r[r % len(cand) == k]
            f, tok = sel // WN, own[sel % WN]
            qkv[f, tok, :C_ATT] = ops.tf32_round(2 * K[j])[None]
            peaks.append((w, f, tok, j))
    return peaks


def _generic_targets(t, WN, NKO, NP, kf_start, kf_step):
    kfs = list(range(kf_start, t, kf_step))
    kpf = NKO + NP

    def f(nkeys, _row, _w):
        c = {0, nkeys - 1, (nkeys - 1) // 64 * 64, (len(kfs) - 1) * kpf, (len(kfs) - 1) * kpf + NKO - 1, NKO - 1}
        if NP:
            c |= {NKO, (len(kfs) - 1) * kpf + NKO}
        return sorted(c)
    return f


def _row_scale(qkv, pool, tab, flags, t, WN, kfs):
    """[t, NT, heads]: largest |v| of each query row's key set, per head."""
    v, pv = qkv[..., 2 * C_ATT:].abs().double(), pool[..., C_ATT:].abs().double()
    sc = torch.zeros(t, qkv.shape[1], C_ATT // 128, dtype=torch.float64, device=qkv.device)
    for w, flag in enumerate(flags.tolist()):
        own = tab[w, :WN].long()
        if not flag:
            sc[:, own] = v[:, own].unflatten(-1, (-1, 128)).amax(dim=(1, 3))[:, None]
        elif kfs:
            rows = torch.cat([torch.cat([v[f, tab[w].long()], pv[f]], 0) for f in kfs], 0)
            sc[:, own] = rows.unflatten(-1, (-1, 128)).amax(dim=(0, 2))
    return sc


def _row_err(got, ref):
    return (got.double() - ref).abs().unflatten(-1, (-1, 128)).amax(-1)            # [t, NT, heads]


def check_attention(qkv, pool, tab, flags, t, WN, kf_start, kf_step, peaks=None, label=""):
    from propainter_b200 import ops
    kfs = list(range(kf_start, t, kf_step))
    ref = attn_table_ref.window_attention_table(qkv, pool, tab, flags, t, WN, kf_start, kf_step)
    bound = ATT_TOL * _row_scale(qkv, pool, tab, flags, t, WN, kfs)
    NT = qkv.shape[1]
    if peaks:                     # precondition, and the alteration the bound must reject
        q64, p64 = qkv.double(), pool.double()
        alt = ref.clone()
        for w, f, tok, j in peaks:
            K, V = attn_table_ref.masked_keys(q64, p64, tab[w].long(), kfs)
            q = q64[f, tok, :C_ATT].unflatten(-1, (-1, 128)).transpose(0, 1)                 # [heads, rows, 128]
            wts = torch.softmax(q @ K.unflatten(-1, (-1, 128)).permute(1, 2, 0) / math.sqrt(128), -1)
            assert (wts[..., j] >= 0.9).all(), (label, w, j, wts[..., j].min().item())
            nb = j + 1 if j + 1 < K.shape[0] else j - 1                                      # the target's neighbour
            K[j], V[j] = K[nb], V[nb]
            alt[f, tok] = attn_table_ref._attend(q64[f, tok, :C_ATT], K, V)
    impls = ("umma", "mma") if tab.shape[1] <= 224 else ("mma",)
    for impl in impls:
        obuf = torch.full((t, NT, C_ATT + 8), SENTINEL, device=DEV)
        out = ops.sparse_window_attn(qkv, pool, tab, flags, t, NT, kf_start, kf_step, out=obuf[..., 4:4 + C_ATT], WN=WN, impl=impl)
        assert (obuf[..., :4] == SENTINEL).all() and (obuf[..., 4 + C_ATT:] == SENTINEL).all(), (label, impl, "wrote outside out")
        assert torch.isfinite(out).all(), (label, impl)
        err = _row_err(out, ref)
        ratio = (err / bound.clamp_min(1e-300)).max().item()
        print(f"attention {label} [{impl}]: max row err / bound = {ratio:.3f}")
        assert (err <= bound).all(), (label, impl, ratio)
        if peaks:
            bad = _row_err(out, alt) > bound
            for w, f, tok, j in peaks:
                assert bad[f, tok].any(-1).all(), (label, impl, w, j, "bound accepts a neighbouring key as the target")


ATT_RUNS = [(a, "diffuse") for a in ATT_CASES] + [(a, "peaked") for a in ATT_CASES
                                                   if a.flags != "all0" and a.t > a.kf_start]


@pytest.mark.parametrize("a,family", ATT_RUNS, ids=[f"{a.name}, {fam}" for a, fam in ATT_RUNS])
def test_sparse_window_attn_f64(a, family):
    qkv, pool, tab, flags = _att_problem(a, torch.Generator().manual_seed(zlib.crc32(a.name.encode())))
    peaks = None
    if family == "peaked":
        peaks = _peak(qkv, pool, tab, flags, a.t, a.WN, a.kf_start, a.kf_step,
                      _generic_targets(a.t, a.WN, a.NKO, a.NP, a.kf_start, a.kf_step))
        assert peaks
    check_attention(qkv, pool, tab, flags, a.t, a.WN, a.kf_start, a.kf_step, peaks, label=f"{a.name}, {family}")


def test_sparse_window_attn_key_table_limit():
    """The wgmma kernel stages the key table in 224 entries of shared memory: 225 is refused, the mma.sync kernel runs it."""
    from propainter_b200 import ops
    a = Att("NKO=225", 2, 5, 45, 225, 8, "alt", 0, 1)
    qkv, pool, tab, flags = _att_problem(a, torch.Generator().manual_seed(7))
    with pytest.raises(RuntimeError):
        ops.sparse_window_attn(qkv, pool, tab, flags, a.t, qkv.shape[1], 0, 1, WN=45, impl="umma")
    check_attention(qkv, pool, tab, flags, a.t, a.WN, 0, 1, label=a.name)


@pytest.mark.parametrize("layer", [0, 1])
def test_sparse_window_attn_model_table_peaked(layer):
    """The model's own key table (window_index.window_key_table) on a padded 20x36 grid, peaked on keys that a gather
    mistake would move: rolled tokens that wrap around the grid, pooled tokens, both ends of the last key tile and the
    last key frame."""
    from propainter_b200 import ops
    from propainter_b200.window_index import window_key_table
    H2, W2, t = 20, 36, 5
    gen = torch.Generator().manual_seed(20 + layer)
    tab = torch.from_numpy(window_key_table(H2, W2)).to(DEV)
    nwin, NKO = tab.shape
    NP = (H2 // 4) * (W2 // 4)
    flags = (torch.arange(nwin) % 3 != 1).int().to(DEV)
    qkv = ops.tf32_round(torch.randn(t, H2 * W2, 3 * C_ATT, generator=gen)).to(DEV)
    pool = ops.tf32_round(torch.randn(t, NP, 2 * C_ATT, generator=gen)).to(DEV)
    kf_start, kf_step = layer % 2, 2
    nkf = len(range(kf_start, t, kf_step))
    kpf = NKO + NP
    generic = _generic_targets(t, 45, NKO, NP, kf_start, kf_step)

    def targets(nkeys, row, w):
        wy, wx = divmod(w, W2 // 9)
        ys, xs = row.long() // W2, row.long() % W2
        far = ((ys - wy * 5).abs() > 8) | ((xs - wx * 9).abs() > 14)        # wrapped around the grid by torch.roll
        wrapped = torch.nonzero(far[45:]).view(-1) + 45
        return sorted(set(generic(nkeys, row, w)) | {int(s) for s in wrapped[:4]} | {(nkf - 1) * kpf + int(s) for s in wrapped[-2:]})
    assert bool(flags[0]) and len(targets(nkf * kpf, tab[0], 0)) > len(generic(nkf * kpf, tab[0], 0))
    peaks = _peak(qkv, pool, tab, flags, t, 45, kf_start, kf_step, targets)
    check_attention(qkv, pool, tab, flags, t, 45, kf_start, kf_step, peaks, label=f"model table, layer {layer}")


def test_attention_cases_cover_the_edges():
    t_wn = {(a.t * a.WN) % 128 for a in ATT_CASES}
    assert 1 in t_wn
    nkeys = {len(range(a.kf_start, a.t, a.kf_step)) * (a.NKO + a.NP) % 64 for a in ATT_CASES if a.t > a.kf_start}
    assert {1, 63} <= nkeys
    assert {a.NKO for a in ATT_CASES} >= {45, 193, 224}
    assert {a.WN for a in ATT_CASES} >= {1, 45, 48, 49, 64}
    nkf = {(len(range(a.kf_start, a.t, a.kf_step)), a.kf_step) for a in ATT_CASES}
    assert {n for n, _ in nkf} >= {0, 1} and any(n >= 3 and s == 1 for n, s in nkf) and any(n >= 3 and s == 2 for n, s in nkf)
    assert {a.flags for a in ATT_CASES} == {"all0", "all1", "alt"}
    fpc = [min(8, max(1, -(-a.t * 4 * a.nwin // 264))) for a in ATT_CASES if a.WN <= 48]
    assert any(f == 8 and a.t % 8 for f, a in zip(fpc, [a for a in ATT_CASES if a.WN <= 48]))
