"""RAFT's fp32 front end against float64, element by element (references and bounds: tests/raft_front_ref.py):

- pp_corr_build (3xTF32 all-pairs volume) within c 2^-22 sum_k |a_k b_k| / sqrt(D); crafted operands whose TF32 low parts
  all have one sign make a 2xTF32 or plain-TF32 build miss by ~2^-12 of that sum, so the bound rejects both;
- pp_corr_pool_pyramid and pp_corr_fmap_pyramid bit-exact with numpy float32 in pp_pool4's order, each level from the
  device's own previous level, and within a pooling bound of float64;
- the lookups (TMA and plain-load at radius 4 and 3, on the fly at (D, R) = (256, 4) and (128, 3)) within their blend
  bound of float64 taps, on pyramids built into NaN-filled buffers (the row padding is NaN), with finite, NaN and
  infinite centres, into NaN-filled output buffers whose neighbours must stay intact;
- pp_convex_upsample within its softmax-and-blend bound, logits up to +-400 after the 0.25 scale;
- pp_instance_norm within c1 u (|y| + 1) + c2 u |mean| / std of float64 statistics, |mean| / std up to 1000, constant
  channels exactly 0, and on the real fnet conv outputs of the seeded RAFT on the synthetic C2 clip.
Each bound is also shown to reject a wrong reference."""
import collections
import math
import types

import numpy as np
import pytest
import torch

from tests import raft_front_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAN32 = 0x7FC5A5A5          # NaN payload of the sentinel fills
WORST = collections.defaultdict(float)


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _note(kernel, worst):
    WORST[kernel] = max(WORST[kernel], worst)
    print(f"  {kernel}: worst err/E {worst:.3g}")


def _nan(*shape):
    t = torch.empty(*shape, device=DEV, dtype=torch.float32)
    t.view(torch.int32).fill_(NAN32)
    return t


def _nan_levels(B, h, w):
    """the pyramid of ops.corr_alloc, but NaN-filled: the row padding is never written, so it stays NaN"""
    from propainter_b200 import ops
    lv, hl, wl = [], h, w
    for _ in range(4):
        lv.append(_nan(B * h * w, hl, ops.corr_ld(wl)))
        hl, wl = hl // 2, wl // 2
    return lv


class Out:
    """a dense output tensor [*shape] inside a NaN-filled flat buffer with 64 spare floats on each side"""

    def __init__(self, *shape):
        self.n = math.prod(shape)
        self.flat = _nan(self.n + 128)
        self.t = self.flat[64:64 + self.n].view(*shape)

    def intact(self):
        b = self.flat.view(torch.int32)
        return bool((b[:64] == NAN32).all()) and bool((b[64 + self.n:] == NAN32).all())


def _fmap(gen, frames, N, D):
    return torch.randn(frames, N, D, generator=gen, device=DEV)


def _pairs(B, frames):
    a = torch.arange(B, device=DEV) % (frames - 1)
    even = torch.arange(B, device=DEV) % 2 == 0
    return torch.where(even, a, a + 1).int(), torch.where(even, a + 1, a).int()


# ----------------------------------------------------------------------------------------------- pp_corr_build
def _check_volume(fmap, idx1, idx2, lvl0, h, w, pairs, rows, what):
    D = fmap.shape[-1]
    c = R.corr_build_c(D)
    worst = 0.0
    for p in pairs:
        f1 = fmap[int(idx1[p])][rows]
        ref, A = R.corr64(f1, fmap[int(idx2[p])])
        got = lvl0[p * h * w + rows][:, :, :w].reshape(len(rows), h * w)
        worst = max(worst, R.check(got, ref, c * 2.0 ** -22 * A + R.TINY, f"{what} pair {p}"))
    return worst


@pytest.mark.parametrize("D,h,w,frames,B", [(256, 30, 54, 3, 3), (128, 17, 23, 2, 2), (256, 90, 160, 2, 1)])
def test_corr_build_f64(D, h, w, frames, B):
    """level 0 of random features (N = 1620, 391, 14400: none a multiple of the 64-pixel tile), pairs with idx1 == idx2
    included; the row padding keeps its NaN"""
    from propainter_b200 import ops
    gen = _gen(D + h)
    fmap = _fmap(gen, frames, h * w, D)
    idx1, idx2 = _pairs(B, frames)
    idx2[-1] = idx1[-1]                                  # a frame with itself
    lv = _nan_levels(B, h, w)
    ops.corr_build(fmap, idx1, idx2, lv, h, w)
    N = h * w
    rows = torch.arange(N, device=DEV) if N <= 2000 else torch.cat([torch.arange(0, N, 97, device=DEV),
                                                                      torch.tensor([N - 1], device=DEV)])
    _note("pp_corr_build", _check_volume(fmap, idx1, idx2, lv[0], h, w, range(B), rows, f"corr D={D} {h}x{w}"))
    if w % 4:
        assert bool(lv[0][:, :, w:].isnan().all())


def test_corr_build_bound_rejects_fewer_tf32_terms():
    """operands whose TF32 low parts are all positive and ~2^-12 of the value: the 3xTF32 kernel stays within the bound,
    float64 volumes of a 2xTF32 and a plain-TF32 split lie outside it"""
    from propainter_b200 import ops
    gen = _gen(5)
    for D in (256, 128):
        h, w = 16, 20
        hi, _ = R.tf32_split64(torch.rand(3, h * w, D, generator=gen, device=DEV) + 0.5)
        fmap = (hi * (1 + 2.0 ** -12 * (1 + 0.5 * torch.rand(hi.shape, generator=gen, device=DEV, dtype=torch.float64)))).float()
        idx1, idx2 = _pairs(2, 3)
        lv = _nan_levels(2, h, w)
        ops.corr_build(fmap, idx1, idx2, lv, h, w)
        _note("pp_corr_build", _check_volume(fmap, idx1, idx2, lv[0], h, w, range(2), torch.arange(h * w, device=DEV),
                                             f"crafted D={D}"))
        f1, f2 = fmap[int(idx1[0])], fmap[int(idx2[0])]
        _, A = R.corr64(f1, f2)
        bound = R.corr_build_c(D) * 2.0 ** -22 * A
        got = lv[0][:h * w].reshape(h * w, h * w)
        for terms in (2, 1):
            assert R.rejects(R.corr_split64(f1, f2, terms), got, bound), (D, terms)
        assert not R.rejects(R.corr_split64(f1, f2, 3), got, bound), D


def test_corr_build_beyond_2g_floats():
    """720p (90 x 160 feature grid), 11 pairs: level 0 holds 2.28e9 floats, so the last pair's rows lie beyond 2^31 floats;
    sampled rows of pairs 0 and 10, the last pixel included"""
    from propainter_b200 import ops
    h, w, B, D = 90, 160, 11, 256
    gen = _gen(11)
    fmap = _fmap(gen, 12, h * w, D)
    idx1, idx2 = _pairs(B, 12)
    lv = ops.corr_alloc(B, h, w, DEV)
    assert lv[0].numel() > 2 ** 31
    ops.corr_build(fmap, idx1, idx2, lv, h, w)
    N = h * w
    rows = torch.cat([torch.arange(0, N, 1009, device=DEV), torch.tensor([N - 2, N - 1], device=DEV)])
    _note("pp_corr_build", _check_volume(fmap, idx1, idx2, lv[0], h, w, (0, B - 1), rows, "corr 720p x 11"))
    last = lv[3][B * N - 1]                                             # pooled from the same far rows
    ref = R.pool32(R.pool32(R.pool32(lv[0][B * N - 1][:, :w].cpu().numpy())))
    assert np.array_equal(last[:, :w >> 3].cpu().numpy(), ref)
    del lv
    torch.cuda.empty_cache()


# ----------------------------------------------------------------------------------------------- pyramids
@pytest.mark.parametrize("h,w,B", [(23, 47, 2), (17, 23, 2), (30, 54, 3)])
def test_pool_pyramids_bit_exact(h, w, B):
    """pp_corr_pool_pyramid and pp_corr_fmap_pyramid: every level equals numpy float32 ((a+b)+c)+d then /4 of the
    device's previous level (23 x 47 -> 11 x 23 -> 5 x 11 -> 2 x 5: every level drops a row and a column), lies within
    the pooling bound of the float64 block average, and is not what another summation order gives"""
    from propainter_b200 import ops
    gen = _gen(h * w)
    fmap = _fmap(gen, B + 1, h * w, 256)
    idx1, idx2 = _pairs(B, B + 1)
    lv = _nan_levels(B, h, w)
    ops.corr_build(fmap, idx1, idx2, lv, h, w)
    planes = [p.cpu().numpy() for p in R.planes64(lv, h, w)]
    a64 = torch.from_numpy(planes[0])
    abs64 = a64.abs()
    swapped = False
    for l in range(1, 4):
        prev = planes[l - 1].astype(np.float32)
        want = R.pool32(prev)
        assert np.array_equal(planes[l].astype(np.float32), want), l
        swapped |= not np.array_equal(R.pool32(prev, order=(0, 2, 1, 3)), want)
        a64, abs64 = R.pool64(a64), R.pool64(abs64)
        _note("pp_corr_pool_pyramid", R.check(torch.from_numpy(planes[l]), a64, R.pool_bound(abs64, l), f"pool level {l}"))
        hl, wl = planes[l].shape[1:]
        if wl % 4:
            assert bool(lv[l][:, :, wl:].isnan().all()), l
    assert swapped
    pooled = ops.corr_fmap_pyramid(fmap, h, w)
    prev = fmap.view(B + 1, h, w, 256).permute(0, 3, 1, 2).cpu().numpy()
    f64 = torch.from_numpy(prev).double()
    fabs = f64.abs()
    for l in range(1, 4):
        want = R.pool32(prev)
        got = pooled[l - 1].view(B + 1, h >> l, w >> l, 256).permute(0, 3, 1, 2).cpu().numpy()
        assert np.array_equal(got, want), l
        f64, fabs = R.pool64(f64), R.pool64(fabs)
        _note("pp_corr_fmap_pyramid", R.check(torch.from_numpy(got), f64, R.pool_bound(fabs, l), f"fmap level {l}"))
        prev = got


# ----------------------------------------------------------------------------------------------- all-pairs lookups
def _lookup(levels, coords, radius, tma):
    from propainter_b200 import ops
    B, h, w, _ = coords.shape
    o = Out(B, h, w, 4 * (2 * radius + 1) ** 2)
    ops.corr_lookup_r(levels, coords, radius, o.t, tma=tma)
    assert o.intact()
    return o.t


def _check_lookup(got, levels, coords, far, h, w, radius, tma, pairs, what, wrong=False):
    K2 = (2 * radius + 1) ** 2
    ref, s, v = R.lookup64(R.planes64(levels, h, w, pairs), coords[list(pairs)], grid_sample32=not tma, radius=radius,
                           corners=True)
    g = got[list(pairs)].reshape(-1, 4 * K2)
    bound = R.lookup_bound(s, v)
    _note("pp_corr_lookup" + ("" if tma else "_ldg") + f" r{radius}", R.check(g, ref, bound, what))
    assert bool((got[far] == 0).all()), what
    if wrong:
        P = R.planes64(levels, h, w, pairs)
        c = coords[list(pairs)]
        assert R.rejects(R.lookup64(P, c, not tma, radius, swap_xy=True)[0], g, bound), what
        for k in range(4):
            assert R.rejects(R.lookup64(P, c, not tma, radius, drop_corner=k)[0], g, bound), (what, k)


@pytest.mark.parametrize("radius", [4, 3])
@pytest.mark.parametrize("B,h,w", [(3, 16, 22), (2, 17, 23), (2, 23, 47)])
def test_corr_lookup_f64(radius, B, h, w):
    """TMA and plain-load lookups on a pyramid with NaN row padding (22, 23, 47 and every level below are not multiples
    of 4), centres of every lookup_coords class plus NaN / inf ones"""
    from propainter_b200 import ops
    gen = _gen(B * h + radius)
    fmap = _fmap(gen, B + 1, h * w, 256)
    idx1, idx2 = _pairs(B, B + 1)
    lv = _nan_levels(B, h, w)
    ops.corr_build(fmap, idx1, idx2, lv, h, w)
    coords, far = R.lookup_coords(B, h, w, seed=B + h + radius, nonfinite=True)
    assert not bool(torch.isfinite(coords).all())
    for tma in (True, False):
        got = _lookup(lv, coords, radius, tma)
        _check_lookup(got, lv, coords, far, h, w, radius, tma, range(B), f"lookup r{radius} {B}x{h}x{w} tma={tma}",
                      wrong=True)


@pytest.mark.parametrize("B,h,w,frames", [(158, 30, 54, 80), (2, 90, 160, 2)])
def test_corr_lookup_production_f64(B, h, w, frames):
    """the C2 batch (158 pairs at 30 x 54, basic and small model) and a 720p pair, NaN row padding; float64 taps of the
    first, middle and last pair"""
    from propainter_b200 import ops
    gen = _gen(B)
    fmap = _fmap(gen, frames, h * w, 256)
    idx1, idx2 = _pairs(B, frames)
    lv = _nan_levels(B, h, w)
    ops.corr_build(fmap, idx1, idx2, lv, h, w)
    coords, far = R.lookup_coords(B, h, w, seed=B + 1, nonfinite=True)
    pairs = sorted({0, B // 2, B - 1})
    for radius in (4, 3):
        for tma in (True, False):
            got = _lookup(lv, coords, radius, tma)
            _check_lookup(got, lv, coords, far, h, w, radius, tma, pairs, f"lookup r{radius} {B}x{h}x{w} tma={tma}")
            del got
    del lv
    torch.cuda.empty_cache()


# ----------------------------------------------------------------------------------------------- on-the-fly lookups
def _otf_ref(fmap, idx1, idx2, coords, h, w, D, radius, sel, scale_wrong=False):
    """float64 taps of the query pixels `sel` (flat indices over pairs x pixels) from float64 dot products with the
    float64-pooled features, and the bound: the blend bound, plus the dot product's FFMA error and the fp32 pooling error
    carried through the weights, plus a dropped off-tile corner of weight <= a few ulp of the coordinate"""
    hw = h * w
    pair, pix = sel // hw, sel % hw
    f2 = fmap.double().view(fmap.shape[0], h, w, D).permute(0, 3, 1, 2)
    a2 = f2.abs()
    planes, eplanes = [], []
    scale = 16.0 if scale_wrong else math.sqrt(D)
    for l in range(4):
        if l:
            f2, a2 = R.pool64(f2), R.pool64(a2)
        pl = torch.empty(len(sel), (h >> l) * (w >> l), dtype=torch.float64, device=DEV)
        el = torch.empty_like(pl)
        for p in pair.unique().tolist():                            # per pair: [P_p, D] x [D, hl*wl]
            m = pair == p
            f1 = fmap[int(idx1[p]), pix[m]].double()
            g, ga = f2[int(idx2[p])].flatten(1), a2[int(idx2[p])].flatten(1)
            pl[m] = f1 @ g / scale
            el[m] = (R.otf_dot_c(D) * R.U * (f1.abs() @ g.abs()) + 3 * l * R.U * (f1.abs() @ ga)) / math.sqrt(D)
        planes.append(pl.view(-1, h >> l, w >> l))
        eplanes.append(el.view(-1, h >> l, w >> l))
    c = coords.reshape(-1, 2)[sel]
    ref, s, v = R.lookup64(planes, c, grid_sample32=True, radius=radius, corners=True)
    e, _ = R.lookup64(eplanes, c, grid_sample32=True, radius=radius)
    K2 = (2 * radius + 1) ** 2
    cf = torch.where(torch.isfinite(c), c.double(), 0.0).abs()
    drop = torch.cat([(8 * R.U * (cf.sum(1, keepdim=True) / 2 ** l + 2 * radius + 2)
                       * planes[l].abs().flatten(1).amax(1, keepdim=True)).expand(-1, K2) for l in range(4)], 1)
    return ref, R.lookup_bound(s, v) + e + drop


@pytest.mark.parametrize("D,radius", [(256, 4), (128, 3)])
@pytest.mark.parametrize("B,h,w", [(2, 17, 23), (3, 30, 54), (2, 90, 160)])
def test_corr_lookup_otf_f64(D, radius, B, h, w):
    """on-the-fly lookups against float64 dot products of the features; the D = 128 scale must be 1/sqrt(128), not 1/16"""
    from propainter_b200 import ops
    gen = _gen(D + B * h)
    fmap = _fmap(gen, B + 1, h * w, D)
    idx1, idx2 = _pairs(B, B + 1)
    pooled = ops.corr_fmap_pyramid(fmap, h, w)
    coords, far = R.lookup_coords(B, h, w, seed=D + h, nonfinite=True)
    K2 = (2 * radius + 1) ** 2
    o = Out(B, h, w, 4 * K2)
    ops.corr_lookup_otf_r(fmap, pooled, idx1, idx2, coords, radius, o.t)
    assert o.intact()
    n = B * h * w
    sel = torch.arange(n, device=DEV) if n <= 4000 else torch.cat([torch.arange(0, n, 7, device=DEV),
                                                                     torch.tensor([n - 1], device=DEV)])
    ref, bound = _otf_ref(fmap, idx1, idx2, coords, h, w, D, radius, sel)
    got = o.t.reshape(-1, 4 * K2)[sel]
    _note(f"pp_corr_lookup_otf D={D} r{radius}", R.check(got, ref, bound, f"otf D={D} {B}x{h}x{w}"))
    assert bool((o.t[far] == 0).all())
    if D == 128:
        assert R.rejects(_otf_ref(fmap, idx1, idx2, coords, h, w, D, radius, sel, scale_wrong=True)[0], got, bound)


def test_corr_lookup_otf_4k_f64():
    """one 4K pair (270 x 480 feature grid, N = 129,600) of the basic model, 600 sampled pixels (the last included)"""
    from propainter_b200 import ops
    h, w, D = 270, 480, 256
    gen = _gen(4)
    fmap = _fmap(gen, 2, h * w, D)
    idx1 = torch.tensor([0], device=DEV, dtype=torch.int32)
    idx2 = torch.tensor([1], device=DEV, dtype=torch.int32)
    pooled = ops.corr_fmap_pyramid(fmap, h, w)
    coords, _ = R.lookup_coords(1, h, w, seed=44, nonfinite=True)
    out = ops.corr_lookup_otf(fmap, pooled, idx1, idx2, coords)
    sel = torch.cat([torch.randint(0, h * w, (599,), generator=gen, device=DEV), torch.tensor([h * w - 1], device=DEV)])
    ref, bound = _otf_ref(fmap, idx1, idx2, coords, h, w, D, 4, sel)
    _note("pp_corr_lookup_otf D=256 r4", R.check(out.reshape(-1, 324)[sel], ref, bound, "otf 4K"))


# ----------------------------------------------------------------------------------------------- convex upsampling
@pytest.mark.parametrize("n,h,w,ld,amp", [(2, 7, 9, 576, 8.0), (1, 30, 54, 640, 1600.0), (3, 5, 3, 576, 1600.0)])
def test_convex_upsample_f64(n, h, w, ld, amp):
    """float64 softmax and blend; mask rows `ld` wide (a channel slice of a wider map when ld > 576); logits up to
    +-amp/4 (+-400: fp32 expf overflows without the max subtraction), 3 x 5 grids where every pixel is a border pixel"""
    from propainter_b200 import ops
    gen = _gen(n * h * w)
    u = torch.rand(n, h, w, ld, generator=gen, device=DEV)
    mask = torch.where(u < 0.1, (u * 20 - 1) * amp, torch.randn(n, h, w, ld, generator=gen, device=DEV) * 4)
    mask_view = mask[..., :576]
    flow = torch.randn(n, h, w, 2, generator=gen, device=DEV) * 5
    got = ops.convex_upsample(mask_view, flow.contiguous(), 0.25)
    ref, bound = R.convex64(mask_view, flow)
    _note("pp_convex_upsample", R.check(got, ref, bound, f"convex {n}x{h}x{w} amp {amp}"))
    if amp > 400:
        assert R.rejects(R.convex64(mask_view, flow, no_max32=True)[0], got, bound)


# ----------------------------------------------------------------------------------------------- instance norm
def _inorm(x, relu=False, res=None, post_relu=False, inplace=False):
    from propainter_b200 import ops
    n, HW, C = x.shape
    xin = x.clone().view(n, HW, 1, C)
    out = ops.instance_norm(xin, relu=relu, res=None if res is None else res.view(n, HW, 1, C), post_relu=post_relu,
                            out=xin if inplace else None)
    if inplace:
        assert out.data_ptr() == xin.data_ptr()
    return out.view(n, HW, C)


@pytest.mark.parametrize("ratio", [0, 3, 10, 30, 100, 1000])
def test_instance_norm_mean_ratio_f64(ratio):
    """|mean| / std swept at the fnet conv1 map of a 4-frame 240 x 432 clip (HW = 120 x 216, C = 64), with 4 constant
    non-zero channels (exactly 0 out); the error must not grow as (|mean| / std)^2"""
    gen = _gen(ratio + 1)
    x = R.inorm_input(gen, 4, 120 * 216, 64, ratio, DEV, const_channels=4)
    got = _inorm(x)
    ref, bound = R.inorm_ref(x)
    _note("pp_instance_norm", R.check(got, ref, bound, f"inorm ratio {ratio}"))
    assert bool((got[:, :, :4] == 0).all())


@pytest.mark.parametrize("C", [8, 16, 24, 32, 64, 96, 128])
@pytest.mark.parametrize("HW", [7, 13, 1001, 60 * 108])
def test_instance_norm_shapes_f64(C, HW):
    """C = 24 and 96 leave threads idle (R = 256 / (C/4) rows per block); HW < 16 has one split, 1001 a ragged last
    chunk; every relu / res / post_relu combination, in place; the bound rejects an unbiased variance and eps added
    outside the square root"""
    gen = _gen(C * HW)
    n = 3
    x = R.inorm_input(gen, n, HW, C, 5.0, DEV, const_channels=1)
    res = torch.randn(n, HW, C, generator=gen, device=DEV)
    for relu, use_res, post in ((False, False, False), (True, False, False), (True, True, True), (False, True, False),
                                (False, False, True)):
        r = res if use_res else None
        got = _inorm(x, relu, r, post, inplace=True)
        ref, bound = R.inorm_ref(x, r, relu, post)
        _note("pp_instance_norm", R.check(got, ref, bound, f"inorm C={C} HW={HW} {relu, use_res, post}"))
    got = _inorm(x)
    _, bound = R.inorm_ref(x)
    small = R.inorm_input(gen, n, HW, C, 0.0, DEV) * 0.01
    got_small = _inorm(small)
    _, bound_small = R.inorm_ref(small)
    if HW > 1:
        assert R.rejects(R.inorm_ref(x, unbiased=True)[0], got, bound)
    assert R.rejects(R.inorm_ref(small, eps_outside=True)[0], got_small, bound_small)


def _raft(small, seed):
    from propainter_b200.RAFT.raft import RAFT
    args = types.SimpleNamespace(small=small, mixed_precision=False, alternate_corr=False)
    return RAFT(args, seed=seed).to(DEV)


def test_instance_norm_real_fnet_inputs_f64(monkeypatch):
    """every instance norm of the seeded basic and small encoders (fnet and cnet) on the synthetic C2 clip (80 frames of
    240 x 432), each call's exact fp32 input against float64; logs the largest |mean| / std per norm"""
    from propainter_b200 import ops, synth
    real = ops.instance_norm
    stats = []

    def rec(x_pm, relu=False, res=None, post_relu=False, eps=1e-5, out=None):
        n, h, w, C = x_pm.shape
        x = x_pm.reshape(n, h * w, C).clone()
        r = None if res is None else res.reshape(n, h * w, C).clone()
        y = real(x_pm, relu=relu, res=res, post_relu=post_relu, eps=eps, out=out)
        ref, bound = R.inorm_ref(x, r, relu, post_relu, eps)
        worst = R.check(y.reshape(n, h * w, C), ref, bound, f"fnet norm {len(stats)} {tuple(x_pm.shape)}")
        stats.append((tuple(x_pm.shape), R.ratio_max(x), worst))
        return y

    monkeypatch.setattr(ops, "instance_norm", rec)
    u8, _, _ = synth.make_clip(80, 240, 432, mask="ellipse", seed=0)
    frames = (torch.from_numpy(u8).permute(0, 3, 1, 2).float() / 255 * 2 - 1).to(DEV)
    for small in (False, True):
        stats.clear()
        _raft(small, seed=0).encode_frames(frames)
        torch.cuda.synchronize()
        assert stats
        for i, (shape, ratio, worst) in enumerate(stats):
            print(f"  {'small' if small else 'basic'} norm {i} {shape}: max |mean|/std {ratio:.3g}, err/E {worst:.3g}")
            _note("pp_instance_norm", worst)


# ----------------------------------------------------------------------------------------------- production coverage
LOOKUP_GRIDS = {(30, 54), (90, 160)}             # test_corr_lookup_production_f64, test_corr_lookup_otf_f64


def _record(monkeypatch):
    """signatures of every call of the entry points above from RAFT_bi's RAFT (basic and small, all-pairs and on-the-fly
    plans) on a C2-sized and a 720p clip, and from encode_frames"""
    from propainter_b200 import ops
    seen = collections.defaultdict(set)

    def wrap(name, sig):
        real = getattr(ops, name)

        def rec(*a, **k):
            seen[name].add(sig(*a, **k))
            return real(*a, **k)
        monkeypatch.setattr(ops, name, rec)

    wrap("corr_build", lambda fmap, idx1, idx2, levels, h, w: (fmap.shape[-1], h, w))
    wrap("corr_lookup", lambda levels, coords, out=None, tma=True: (4, coords.shape[1], coords.shape[2], bool(tma),
                                                                      None if out is None else out.dtype))
    wrap("corr_lookup_r", lambda levels, coords, radius, out=None, tma=True: (radius, coords.shape[1], coords.shape[2],
                                                                               bool(tma), None))
    wrap("corr_fmap_pyramid", lambda fmap, h, w: (fmap.shape[-1], h, w))
    wrap("corr_lookup_otf", lambda fmap, pooled, idx1, idx2, coords, out=None: (fmap.shape[-1], 4, coords.shape[1],
                                                                                 coords.shape[2]))
    wrap("corr_lookup_otf_r", lambda fmap, pooled, idx1, idx2, coords, radius, out=None: (fmap.shape[-1], radius,
                                                                                           coords.shape[1], coords.shape[2]))
    wrap("convex_upsample", lambda mask_pm, flow_lr, mask_scale=0.25: (mask_pm.stride(-2), float(mask_scale)))
    wrap("instance_norm", lambda x_pm, relu=False, res=None, post_relu=False, eps=1e-5, out=None:
         (x_pm.shape[-1], bool(relu), res is not None, bool(post_relu), out is x_pm, float(eps)))
    gen = torch.Generator().manual_seed(0)
    for small in (False, True):
        net = _raft(small, seed=1)
        for alternate in (False, True):
            net.args.alternate_corr = alternate
            for T, H, W in ((3, 240, 432), (2, 720, 1280)):
                fr = (torch.rand(T, 3, H, W, generator=gen) * 2 - 1).to(DEV)
                net._flows_bidirectional(fr, 2, net.corr_plan(H, W, DEV))
    torch.cuda.synchronize()
    return seen


def test_cases_cover_production_signatures(monkeypatch):
    seen = _record(monkeypatch)
    torch.cuda.empty_cache()
    print("[signatures] " + "; ".join(f"{k}: {sorted(v, key=str)}" for k, v in sorted(seen.items())))
    assert seen["corr_build"] and seen["instance_norm"] and seen["convex_upsample"]
    assert seen["corr_lookup_otf"] | seen["corr_lookup_otf_r"]
    assert {D for D, h, w in seen["corr_build"]} <= {256, 128}            # both in test_corr_build_f64 / crafted
    assert {(h, w) for _, h, w in seen["corr_build"]} <= LOOKUP_GRIDS
    # fp16 lookups (the half-precision refinement) are test_gpu_half_kernels_f64's; fp32 ones are covered here
    for r, h, w, tma, dt in seen["corr_lookup"] | seen["corr_lookup_r"]:
        assert dt in (None, torch.float32, torch.float16) and (h, w) in LOOKUP_GRIDS and r in (3, 4), (r, h, w)
    for D, r, h, w in seen["corr_lookup_otf"] | seen["corr_lookup_otf_r"]:
        assert (D, r) in {(256, 4), (128, 3)} and (h, w) in LOOKUP_GRIDS, (D, r, h, w)
    assert {D for D, h, w in seen["corr_fmap_pyramid"]} <= {256, 128}
    assert seen["convex_upsample"] <= {(576, 0.25), (640, 0.25)}, seen["convex_upsample"]
    combos = {(False, False, False), (True, False, False), (True, True, True), (False, True, False), (False, False, True)}
    for C, relu, res, post, inplace, eps in seen["instance_norm"]:
        assert C in (8, 16, 24, 32, 64, 96, 128) and (relu, res, post) in combos and eps == 1e-5, (C, relu, res, post)


def test_zz_worst_ratios():
    """the worst err/E per kernel over this module's tests (printed with -s)"""
    print("[worst err/E] " + "; ".join(f"{k}: {v:.3g}" for k, v in sorted(WORST.items())))
    assert all(v <= 1.0 for v in WORST.values())
