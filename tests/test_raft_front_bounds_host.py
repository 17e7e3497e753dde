"""The float64 references and bounds of raft_front_ref applied to the host build of the same per-element rules
(tests/hostsim: pp_elem.cuh compiled for the CPU, no FMA contraction): the pyramid pooling, the all-pairs tap rule at
radius 4 and 3, the on-the-fly tile rule, convex upsampling and the instance-norm statistics, so the bound logic and the
wrong-reference checks run without a GPU.  The device kernels get the same checks in test_gpu_raft_front_f64.py."""
import ctypes
import math

import numpy as np
import pytest
import torch

from tests import raft_front_ref as R


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _pyramid(hostsim, planes0, h, w):
    """levels [P][h>>l][roundup4(w>>l)] from level-0 planes [P, h, w] through hs_corr_pool, padding NaN"""
    P = planes0.shape[0]
    lv, hl, wl = [], h, w
    for l in range(4):
        ld = hostsim.hs_corr_ld(wl)
        a = np.full((P, hl, ld), np.nan, np.float32)
        if l == 0:
            a[:, :, :w] = planes0
        else:
            prev = lv[-1]
            hostsim.hs_corr_pool(_p(prev), _p(a), ctypes.c_long(P), prev.shape[1], prev.shape[2], hl, wl, ld)
        lv.append(a)
        hl, wl = hl // 2, wl // 2
    return lv


@pytest.mark.parametrize("h,w", [(23, 47), (16, 22)])
def test_pool_host_bit_exact_and_bounded(hostsim, h, w):
    rng = np.random.default_rng(h)
    planes0 = (rng.standard_normal((6, h, w)) * 3).astype(np.float32)
    lv = _pyramid(hostsim, planes0, h, w)
    a64 = torch.from_numpy(planes0).double()
    abs64 = a64.abs()
    for l in range(1, 4):
        hl, wl = lv[l].shape[1], w >> l
        prev = lv[l - 1][:, :, :w >> (l - 1)]
        assert np.array_equal(lv[l][:, :, :wl], R.pool32(prev)), l
        assert not np.array_equal(R.pool32(prev, order=(0, 2, 1, 3)), R.pool32(prev))
        a64, abs64 = R.pool64(a64), R.pool64(abs64)
        R.check(torch.from_numpy(lv[l][:, :, :wl]), a64, R.pool_bound(abs64, l), f"host pool {l}")
        assert np.isnan(lv[l][:, :, wl:]).all()


@pytest.mark.parametrize("radius", [4, 3])
def test_lookup_host_within_bound(hostsim, radius):
    """hs_corr_lookup_r on NaN-padded levels, every centre class and NaN / inf centres: finite, within the blend bound of
    float64 taps at grid_sample's fp32 coordinates; x/y swapped and dropped corners are rejected"""
    B, h, w = 2, 17, 23
    rng = np.random.default_rng(radius)
    planes0 = rng.standard_normal((B * h * w, h, w)).astype(np.float32)
    lv = _pyramid(hostsim, planes0, h, w)
    coords, far = R.lookup_coords(B, h, w, seed=radius, device="cpu", nonfinite=True)
    c = coords.numpy().reshape(-1, 2).copy()
    K2 = (2 * radius + 1) ** 2
    out = np.empty((B * h * w, 4 * K2), np.float32)
    hostsim.hs_corr_lookup_r(_p(lv[0]), _p(lv[1]), _p(lv[2]), _p(lv[3]), radius, _p(c), _p(out), ctypes.c_long(B * h * w), h, w)
    pl = [torch.from_numpy(a[:, :, :w >> l]).double() for l, a in enumerate(lv)]
    ref, s, v = R.lookup64(pl, coords, grid_sample32=True, radius=radius, corners=True)
    got = torch.from_numpy(out)
    bound = R.lookup_bound(s, v)
    R.check(got, ref, bound, f"host lookup r{radius}")
    assert (got[far.reshape(-1)] == 0).all()
    assert R.rejects(R.lookup64(pl, coords, True, radius, swap_xy=True)[0], got, bound)
    for k in range(4):
        assert R.rejects(R.lookup64(pl, coords, True, radius, drop_corner=k)[0], got, bound), k


@pytest.mark.parametrize("radius", [4, 3])
def test_tile_rule_host_within_bound(hostsim, radius):
    """hs_corr_tap_tile_r: the window of a level sampled from the T x T tile at pp_corr_tile_origin_r (zeros outside the
    level) equals the float64 taps of the whole plane within the blend bound plus an off-tile corner of a few ulp of
    the coordinate; centres of every class, NaN and inf included"""
    hl0, wl0 = 30, 54
    T, K = 2 * radius + 2, 2 * radius + 1
    rng = np.random.default_rng(10 + radius)
    coords, _ = R.lookup_coords(1, hl0, wl0, seed=radius, device="cpu", nonfinite=True)
    c = coords.reshape(-1, 2)[::5]
    for lvl in range(4):
        hl, wl = hl0 >> lvl, wl0 >> lvl
        plane = rng.standard_normal((hl, wl)).astype(np.float32)
        got = np.empty((len(c), K * K), np.float32)
        org = np.empty(2, np.int32)
        for i, (cx, cy) in enumerate(c.numpy()):
            tile = np.zeros((T, T), np.float32)
            hostsim.hs_corr_tap_tile_r(_p(tile), radius, hl, wl, ctypes.c_float(cx), ctypes.c_float(cy), lvl, _p(got[i]),
                                       _p(org))
            tx0, ty0 = int(org[0]), int(org[1])
            for j in range(T):
                for k in range(T):
                    if 0 <= ty0 + j < hl and 0 <= tx0 + k < wl:
                        tile[j, k] = plane[ty0 + j, tx0 + k]
            hostsim.hs_corr_tap_tile_r(_p(tile), radius, hl, wl, ctypes.c_float(cx), ctypes.c_float(cy), lvl, _p(got[i]),
                                       _p(org))
        planes = [torch.zeros(len(c), hl0 >> l, wl0 >> l, dtype=torch.float64) for l in range(4)]
        planes[lvl][:] = torch.from_numpy(plane).double()
        ref, s, v = R.lookup64(planes, c, grid_sample32=True, radius=radius, corners=True)
        sl = slice(lvl * K * K, (lvl + 1) * K * K)
        cf = torch.where(torch.isfinite(c), c.double(), 0.0).abs().sum(1, keepdim=True)
        drop = 8 * R.U * (cf / 2 ** lvl + 2 * radius + 2) * float(np.abs(plane).max())
        g = torch.from_numpy(got)
        bound = R.lookup_bound(s[:, sl], v[:, sl]) + drop
        R.check(g, ref[:, sl], bound, f"host tile r{radius} level {lvl}")
        assert R.rejects(R.lookup64(planes, c, True, radius, swap_xy=True)[0][:, sl], g, bound)


@pytest.mark.parametrize("h,w,amp", [(5, 3, 1600.0), (7, 9, 8.0)])
def test_convex_host_within_bound(hostsim, h, w, amp):
    rng = np.random.default_rng(h)
    n = 2
    u = rng.random((n, h, w, 576))
    mask = np.where(u < 0.1, (u * 20 - 1) * amp, rng.standard_normal((n, h, w, 576)) * 4).astype(np.float32)
    flow = (rng.standard_normal((n, h, w, 2)) * 5).astype(np.float32)
    out = np.empty((n, 2, 8 * h, 8 * w), np.float32)
    hostsim.hs_convex_upsample(_p(mask), 576, ctypes.c_float(0.25), _p(flow), _p(out), n, h, w)
    ref, bound = R.convex64(torch.from_numpy(mask), torch.from_numpy(flow))
    got = torch.from_numpy(out)
    R.check(got, ref, bound, f"host convex {h}x{w}")
    if amp > 400:
        assert R.rejects(R.convex64(torch.from_numpy(mask), torch.from_numpy(flow), no_max32=True)[0], got, bound)


def _old_inorm(x, eps=1e-5):
    """the statistics this kernel used to take: per-thread fp32 sums of x and x^2, E[x^2] - mean^2 (numpy float32 sums
    over R = 16 row-threads of each split, folded in double)"""
    n, HW, C = x.shape
    S = max(1, min(64, (592 + n - 1) // n, (HW + 15) // 16))
    chunk = -(-HW // S)
    su = np.zeros((n, C)); sq = np.zeros((n, C))
    for s in range(S):
        blk = x[:, s * chunk:min(HW, (s + 1) * chunk)]
        for r in range(16):
            a = np.zeros((n, C), np.float32); b = np.zeros((n, C), np.float32)
            for row in blk[:, r::16].transpose(1, 0, 2):
                a += row; b += row * row
            su += a; sq += b
    mean = su / HW
    var = np.maximum(sq / HW - mean * mean, 0)
    return ((x - mean[:, None].astype(np.float32)) * (1 / np.sqrt(var + eps)).astype(np.float32)[:, None])


def _hs_inorm(hostsim, x, res=None, relu=False, post_relu=False):
    n, HW, C = x.shape
    out = np.empty_like(x)
    hostsim.hs_instance_norm(_p(x), _p(res) if res is not None else None, _p(out), n, ctypes.c_long(HW), C, ctypes.c_float(1e-5),
                             int(relu), int(post_relu))
    return out


@pytest.mark.parametrize("ratio", [0, 3, 30, 1000])
def test_instance_norm_host_within_bound(hostsim, ratio):
    """hs_instance_norm (pp_inorm_acc / pp_inorm_fold / pp_inorm_out in the kernel's split) within the bound at
    |mean| / std up to 1000, constant channels exactly 0, every relu / res / post_relu combination; the old fp32
    E[x^2] - mean^2 statistics (from |mean| / std = 30 at this 4000-pixel map), an unbiased variance and eps outside the square root are rejected"""
    gen = torch.Generator().manual_seed(ratio)
    n, HW, C = 2, 4000, 64
    x = R.inorm_input(gen, n, HW, C, ratio, "cpu", const_channels=2)
    xn = x.numpy()
    res = torch.randn(n, HW, C, generator=gen)
    for relu, use_res, post in ((False, False, False), (True, False, False), (True, True, True)):
        r = res if use_res else None
        got = torch.from_numpy(_hs_inorm(hostsim, xn, r.numpy() if use_res else None, relu, post))
        ref, bound = R.inorm_ref(x, r, relu, post)
        R.check(got, ref, bound, f"host inorm ratio {ratio} {relu, use_res, post}")
        assert (got[:, :, :2] == 0).all() if not use_res else True
    got = torch.from_numpy(_hs_inorm(hostsim, xn))
    _, bound = R.inorm_ref(x)
    assert R.rejects(R.inorm_ref(x, unbiased=True)[0], got, bound)
    small = (x - x.mean(1, keepdim=True)) * 0.01
    _, bsmall = R.inorm_ref(small)
    assert R.rejects(R.inorm_ref(small, eps_outside=True)[0], torch.from_numpy(_hs_inorm(hostsim, small.numpy())), bsmall)
    if ratio >= 30:
        ref, _ = R.inorm_ref(x)
        assert R.rejects(ref, torch.from_numpy(_old_inorm(xn)), bound)


def test_instance_norm_host_small_maps(hostsim):
    """HW < 16 (one split) and C with idle threads (24, 96) on the host build"""
    gen = torch.Generator().manual_seed(7)
    for HW, C in ((7, 24), (13, 96), (1, 8), (1001, 128)):
        x = R.inorm_input(gen, 3, HW, C, 10.0, "cpu", const_channels=1)
        got = torch.from_numpy(_hs_inorm(hostsim, x.numpy(), relu=True))
        ref, bound = R.inorm_ref(x, relu=True)
        R.check(got, ref, bound, f"host inorm HW={HW} C={C}")
        assert math.isfinite(float(got.abs().max()))
