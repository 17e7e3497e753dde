"""The float64 references, error bounds and margin rules of scan_gather_ref applied to the host build of the same
per-element rules (tests/hostsim: pp_elem.cuh compiled for the CPU, no FMA contraction), so the bound logic, the margin
classification and the crafted ties run without a GPU.  The host build stores the columns unrounded, so the TF32 checks
of the columns are device-only (test_gpu_scan_gather_f64.py)."""
import ctypes

import numpy as np
import torch

from tests import scan_gather_ref as R


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _smooth(rng, n, h, w, amp):
    import torch.nn.functional as F
    z = torch.from_numpy(rng.standard_normal((n, 2, h // 4 + 2, w // 4 + 2)).astype(np.float32)) * amp
    return F.interpolate(z, size=(h, w), mode="bilinear", align_corners=False).permute(0, 2, 3, 1).contiguous().numpy()


def test_warp_coord32():
    """the numpy float32 restatement of pp_warp_coord: an integer flow on a grid of 2^k + 1 pixels lands on integers (the
    crafted exact cases rely on it), and a 1-pixel axis always samples position 0"""
    for size in (1, 2, 17, 54, 108):
        base = np.arange(size, dtype=np.float32)
        c = R.warp_coord32(base, np.float32(3.0), size)
        if size in (2, 17):
            assert (c == base + 3).all()
        assert np.isfinite(c).all()
    assert (R.warp_coord32(np.arange(5, dtype=np.float32), np.float32(0.7), 1) == 0).all()      # 1-pixel axis: always 0


def test_fb_ties_are_exact_and_strict():
    for fx, fy in ((3, -2), (2, -1), (-2, 1), (0, 0)):
        ties = R.fb_ties(fx, fy, 6)
        assert len(ties) >= 3, (fx, fy)
        for bx, by in ties:
            v, tie = R.fb_valid32(fx, fy, bx, by)
            assert tie and not v                                    # lhs == thr: the strict `<` says invalid
            # float64 of the same quantity sits inside the band, the margin does not decide it
            t = lambda a: torch.tensor([float(a)], dtype=torch.float64)     # noqa: E731
            _, dec = R.fb_margin(t(fx), t(fy), t(bx), t(by), t(0.0), t(0.0))
            assert not dec.item()


def test_tf32_helpers():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(10000, generator=g, dtype=torch.float64) * 7
    i = x.float().view(torch.int32)
    ref = ((i + 0x1000) & ~0x1FFF).view(torch.float32).double()
    assert torch.equal(R.tf32_rna(x.float().double()), ref)
    mid = ((i & ~0x1FFF) | 0x1000).view(torch.float32).double()                 # ties: away from zero
    assert torch.equal(R.tf32_rna(mid), mid + torch.sign(mid) * 0.5 * R.tf32_ulp(mid))
    st = {}
    R.check_tf32(R.tf32_rna(x).float(), x, torch.full_like(x, 1e-12), st)
    assert st["n"] > 9000 and abs(st["sum"] / st["n"]) < 0.02
    trunc = (x.float().view(torch.int32) & ~0x1FFF).view(torch.float32)
    try:
        R.check_tf32(trunc, x, torch.full_like(x, 1e-12), {})
        raise RuntimeError("truncated TF32 values passed")
    except AssertionError:
        pass


def test_deform_cols_host_within_bound(hostsim):
    """hs_deform_cols (pp_deform_tap + pp_deform_weights + pp_deform_sample1) against deform_cols_ref, per element, on a
    ragged map with offsets across every border and on 1-pixel-wide and -high maps; wrong references are rejected."""
    rng = np.random.default_rng(1)
    for (H, W, Cin, use_flow, mr) in ((7, 11, 128, True, 5.0), (1, 9, 128, False, 3.0), (6, 1, 256, True, 5.0)):
        x = rng.standard_normal((H, W, Cin)).astype(np.float32)
        o = (rng.standard_normal((H * W, 432)) * 1.5).astype(np.float32)
        flow = (rng.standard_normal((H * W, 2)) * 2).astype(np.float32) if use_flow else None
        cols = np.empty((H * W, 9 * Cin), np.float32)
        hostsim.hs_deform_cols(_p(x), Cin, _p(o), 432, _p(flow) if flow is not None else None, ctypes.c_float(mr), _p(cols), H, W, Cin)
        got = torch.from_numpy(cols).view(1, H * W, 9, Cin)
        x64 = torch.from_numpy(x).double()[None]
        o32 = torch.from_numpy(o).view(1, H, W, 432)
        fl = torch.from_numpy(flow).view(1, H, W, 2) if flow is not None else None
        worst = 0.0
        for k in range(9):
            ref, E = R.deform_cols_ref(x64, o32, fl, mr, k)
            worst = max(worst, R.check_bound(got[:, :, k], ref, E, f"hs_deform_cols {H}x{W} tap {k}"))
        assert worst > 0
        if H > 1 and W > 1:
            for fault in ("swap", "noflip", "corner", "group", "shift") if use_flow else ("swap", "corner", "group", "shift"):
                bad = any(R.bound_rejects(got[:, :, k], R.deform_cols_ref(x64, o32, fl, mr, k, fault)[0],
                                          R.deform_cols_ref(x64, o32, fl, mr, k)[1]) for k in range(9))
                assert bad, fault


def _tie_case(h, w, fx, fy, rng):
    ties = R.fb_ties(fx, fy, 6)
    fprop = np.empty((h, w, 2), np.float32)
    fprop[..., 0], fprop[..., 1] = fx, fy
    fcheck = (rng.standard_normal((h, w, 2)) * 0.3 - np.array([fx, fy])).astype(np.float32)
    sel = rng.random((h, w)) < 0.7
    tv = np.array(ties, np.float32)[rng.integers(0, len(ties), (h, w))]
    fcheck[sel] = tv[sel]
    return fprop, fcheck


def test_prop_cond_host_by_margin(hostsim):
    rng = np.random.default_rng(2)
    for (h, w, C, kind) in ((30, 54, 64, "rand"), (1, 13, 32, "rand"), (9, 17, 32, "tie")):
        if kind == "tie":
            fprop, fcheck = _tie_case(h, w, 3, -2, rng)
        else:
            fprop = _smooth(rng, 1, h, w, 3.0)[0]
            fcheck = (-fprop + 0.5 * rng.standard_normal((h, w, 2))).astype(np.float32)
        cur = rng.standard_normal((h, w, C)).astype(np.float32)
        prop = rng.standard_normal((h, w, C)).astype(np.float32)
        m = (rng.random((h, w, 2)) > 0.5).astype(np.float32)
        ldc, ldb = 2 * C + 8, 2 * C + 4
        cond = np.full((h, w, ldc), np.nan, np.float32)
        bb = np.full((h, w, ldb), np.nan, np.float32)
        hostsim.hs_prop_cond(_p(cur), C, _p(prop), C, _p(fprop), _p(fcheck), _p(m), _p(cond), ldc, _p(bb), ldb, h, w, C, 0)
        assert (cond[..., :C] == cur).all() and (cond[..., 2 * C:2 * C + 2] == fprop).all()
        assert np.isnan(bb[..., C:2 * C]).all() and (bb[..., 2 * C + 2:] == 0).all()
        ix, iy = R.warp_positions(fprop[None])
        ref, E = R.warp_sample(torch.from_numpy(prop).double()[None], ix, iy)
        got = torch.from_numpy(cond[..., C:2 * C].copy()).view(1, h * w, C)
        R.check_bound(got, ref, E, "hs_prop_cond warped")
        if h > 1 and w > 1 and kind == "rand":        # integral positions or a 1-pixel axis: no lower-right corner to drop
            assert R.bound_rejects(got, R.warp_sample(torch.from_numpy(prop).double()[None], ix, iy, "corner")[0], E)
        b, e = R.warp_sample(torch.from_numpy(fcheck).double()[None], ix, iy)
        f = torch.from_numpy(fprop).double().view(1, -1, 2)
        valid, decided = R.fb_margin(f[..., 0], f[..., 1], b[..., 0], b[..., 1], e[..., 0], e[..., 1])
        gv = torch.from_numpy(cond[..., 2 * C + 2].copy()).view(1, -1)
        # integral positions: exact check-flow samples, so pp_fb_valid's own fp32 arithmetic decides (exact ties included)
        v32, tie = R.fb_valid32(fprop[..., 0].reshape(1, -1), fprop[..., 1].reshape(1, -1), b[..., 0].float().numpy(),
                                b[..., 1].float().numpy())
        it = torch.from_numpy((ix == np.rint(ix)) & (iy == np.rint(iy)))
        valid, decided = torch.where(it, torch.from_numpy(v32), valid), decided | it
        assert torch.equal(gv.bool()[decided], valid[decided])
        assert (~decided).float().mean() < 1e-3
        if kind == "tie":
            assert int((torch.from_numpy(tie) & it).sum()) >= 10


def test_img_prop_scan_host_stepwise(hostsim):
    """hs_img_prop_scan with t = 2: out[0] is the backward step from frame 1, out[1] the forward step from out[0]; each
    checked by margin (bilinear and nearest), with masks of exactly 0.1f and exact fb ties on a power-of-two grid."""
    rng = np.random.default_rng(3)
    for (H, W, kind) in ((40, 56, "rand"), (9, 17, "exact")):
        frames = (rng.random((2, 3, H, W)) * 2 - 1).astype(np.float32)
        masks = np.zeros((2, 1, H, W), np.float32)
        masks[..., H // 4:3 * H // 4, W // 4:3 * W // 4] = 1
        masks[rng.random(masks.shape) < 0.08] = R.F_TENTH
        if kind == "exact":
            ff = rng.integers(-2, 3, (1, 2, H, W)).astype(np.float32) + 0.5 * (rng.random((1, 2, H, W)) < 0.3)
            fb = (-ff + rng.standard_normal(ff.shape) * 0.4).astype(np.float32)
            ff = ff.astype(np.float32)
        else:
            ff = _smooth(rng, 1, H, W, 4.0).transpose(0, 3, 1, 2).copy()
            fb = (-ff + 0.3 * _smooth(rng, 1, H, W, 4.0).transpose(0, 3, 1, 2)).astype(np.float32)
        masked = (frames * (1 - masks)).astype(np.float32)
        for nearest in (1, 0):
            of = np.empty_like(masked)
            om = np.empty_like(masks)
            hostsim.hs_img_prop_scan(_p(masked), _p(ff), _p(fb), _p(masks), _p(of), _p(om), 2, H, W, nearest)
            steps = ((masked[0], masks[0, 0], masked[1], masks[1, 0], ff[0], fb[0], of[0], om[0, 0]),
                     (masked[1], masks[1, 0], of[0], om[0, 0], fb[0], ff[0], of[1], om[1, 0]))
            for s in steps:
                assert _host_step_bad(*s, nearest) == 0
            if not nearest:
                assert _host_step_bad(*steps[0], nearest, "swap") > 0


def _host_step_bad(cur, mc, prev, mprev, fprop, fcheck, got_f, got_m, nearest, fault=None):
    """the device test's step check on CPU tensors (one pixel fails: no combination of open decisions matches)"""
    H, W = mc.shape
    fpm = np.ascontiguousarray(fprop.transpose(1, 2, 0))[None]
    ix, iy = R.warp_positions(fpm, fault)
    b, e = R.warp_sample(torch.from_numpy(np.ascontiguousarray(fcheck.transpose(1, 2, 0))).double()[None], ix, iy)
    f = torch.from_numpy(fpm).double().view(1, -1, 2)
    valid, vdec = R.fb_margin(f[..., 0], f[..., 1], b[..., 0], b[..., 1], e[..., 0], e[..., 1])
    integral = (ix == np.rint(ix)) & (iy == np.rint(iy))
    v32, _ = R.fb_valid32(fpm[..., 0].reshape(1, -1), fpm[..., 1].reshape(1, -1), b[..., 0].float().numpy(), b[..., 1].float().numpy())
    it = torch.from_numpy(integral)
    valid, vdec = torch.where(it, torch.from_numpy(v32), valid)[0], (vdec | it)[0]
    sm, em = R.warp_sample(torch.from_numpy(mprev).double().view(1, H, W, 1), ix, iy)
    mw, mdec = R.threshold_margin(sm[0, :, 0], em[0, :, 0])
    mdec = mdec | it[0]
    p64 = torch.from_numpy(np.ascontiguousarray(prev.transpose(1, 2, 0))).double()[None]
    if nearest:
        wv, ew = R.nearest_sample(p64, ix, iy)[0], None
    else:
        s, e2 = R.warp_sample(p64, ix, iy)
        wv, ew = s[0], e2[0]
    c64 = torch.from_numpy(cur.reshape(3, -1).T.copy()).double()
    g64 = torch.from_numpy(got_f.reshape(3, -1).T.copy()).double()
    mc64 = torch.from_numpy(mc.reshape(-1).copy()).double()
    gm = torch.from_numpy(got_m.reshape(-1).copy())
    ok = torch.zeros_like(gm, dtype=torch.bool)
    for v_c in (False, True):
        for w_c in (False, True):
            allowed = torch.where(vdec, valid == v_c, torch.ones_like(vdec)) & torch.where(mdec, mw == w_c, torch.ones_like(mdec))
            moved = v_c and not w_c
            use = (mc64 > R.F_TENTH) & moved
            m2 = (mc64 > R.F_TENTH) & (not moved)
            fr = torch.where(use[:, None], (g64 - wv).abs() <= (ew if ew is not None else 0), g64 == c64).all(1)
            ok |= allowed & fr & (gm == m2.float())
    return int((~ok).sum())
