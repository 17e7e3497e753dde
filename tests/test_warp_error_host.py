"""CPU tests of the temporal warping error (E_warp, Lai et al. ECCV 2018; occlusion test of Ruder et al. GCPR 2016):
oracle/ewarp_ref.py on hand-computed cases, the host build of the per-pixel rules of pp_elem.cuh against the oracle on
random inputs, evaluate_propainter's aggregation with stand-in ops, and the argument refusals.  The kernels run on the
GPU in test_gpu_warp_error.py.

Equality criterion for occlusion maps: equal wherever both tests lie more than ewarp_ref.MARGIN * (1 + rhs) from their
thresholds (float64); inside that margin a float32 evaluation may decide either way.  Warping error: per pair,
|E_t - oracle| <= 1e-5 * oracle + 1e-9, with the oracle evaluated on the implementation's own occlusion map."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import ewarp_ref

HERE = os.path.dirname(os.path.abspath(__file__))
FP = ctypes.POINTER(ctypes.c_float)
U8P = ctypes.POINTER(ctypes.c_uint8)
DP = ctypes.POINTER(ctypes.c_double)
FLOW_KINDS = ("smooth", "large", "integer")


# ---------------------------------------------------------------- seeded inputs (shared with the GPU tests)
def _upsample(lo, H, W):
    t = torch.nn.functional.interpolate(torch.from_numpy(lo), size=(H, W), mode="bilinear", align_corners=False)
    return t.numpy().astype(np.float32)


def flow_case(kind, N, H, W, seed):
    """(fw, bw) float32 [N,2,H,W].  smooth: a smooth field of a few px and bw = -fw, so the forward-backward test passes
    where the field varies slowly and fails where it does not; large: displacements of up to ~200 px, most of them off
    the frame, with an unrelated bw; integer: piecewise-constant integer displacements (a = b = 0) with bw = -fw."""
    rng = np.random.default_rng(seed)
    if kind == "smooth":
        fw = _upsample(rng.standard_normal((N, 2, 2, 3)).astype(np.float32) * 3, H, W)
        bw = -fw + (rng.standard_normal(fw.shape) * 0.3).astype(np.float32)
    elif kind == "large":
        fw = _upsample(rng.standard_normal((N, 2, 3, 4)).astype(np.float32) * 120, H, W)
        bw = _upsample(rng.standard_normal((N, 2, 3, 4)).astype(np.float32) * 120, H, W)
    elif kind == "integer":
        lo = rng.integers(-4, 5, (N, 2, H // 8 + 1, W // 8 + 1)).astype(np.float32)
        fw = np.repeat(np.repeat(lo, 8, 2), 8, 3)[..., :H, :W]
        bw = -fw
    else:
        raise ValueError(kind)
    return np.ascontiguousarray(fw, np.float32), np.ascontiguousarray(bw, np.float32)


def texture(T, H, W, seed):
    """uint8 [T,H,W,3]: a smooth random texture plus noise, independent per frame"""
    rng = np.random.default_rng(seed)
    lo = rng.uniform(0, 255, (T, 3, H // 6 + 2, W // 6 + 2)).astype(np.float32)
    img = _upsample(lo, H, W) + rng.normal(0, 8, (T, 3, H, W)).astype(np.float32)
    return np.ascontiguousarray(np.clip(img, 0, 255).astype(np.uint8).transpose(0, 2, 3, 1))


def translation_clip(T, H, W, shifts, seed):
    """frames of one texture, frame t+1 = frame t moved by the integer shift (dx, dy) of pair t (frame t+1 at x + d shows
    frame t at x), and the exact flows: fw_t = d, bw_t = -d.  -> (frames uint8 [T,H,W,3], fw, bw [T-1,2,H,W])"""
    pad = max(max(abs(dx), abs(dy)) for dx, dy in shifts) * T
    big = texture(1, H + 2 * pad, W + 2 * pad, seed)[0]
    frames, ox, oy = [], 0, 0
    offs = [(0, 0)]
    for dx, dy in shifts:
        ox, oy = ox + dx, oy + dy
        offs.append((ox, oy))
    for ox, oy in offs:                        # frame(x) = big(x - offset): content moves by +offset
        frames.append(big[pad - oy:pad - oy + H, pad - ox:pad - ox + W])
    fw = np.zeros((T - 1, 2, H, W), np.float32)
    for t, (dx, dy) in enumerate(shifts):
        fw[t, 0], fw[t, 1] = dx, dy
    return np.ascontiguousarray(np.stack(frames)), fw, -fw


# ---------------------------------------------------------------- host build of the rules
@pytest.fixture(scope="module")
def hs(tmp_path_factory):
    lib = os.path.join(str(tmp_path_factory.mktemp("hostsim_ewarp")), "libhostsim_ewarp.so")
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", lib,
                           os.path.join(HERE, "hostsim", "hostsim_ewarp.cpp")])
    return ctypes.CDLL(lib)


def _c(a, dtype, ptr):
    a = np.ascontiguousarray(a, dtype)
    return a, a.ctypes.data_as(ptr)


def hs_occlusion(hs, fw, bw):
    (fw, pf), (bw, pb) = _c(fw, np.float32, FP), _c(bw, np.float32, FP)
    N, _, H, W = fw.shape
    occ = np.empty((N, H, W), np.uint8)
    hs.hs_flow_occlusion(pf, pb, occ.ctypes.data_as(U8P), N, H, W)
    return occ


def hs_sums(hs, frames, fw, occ):
    (fr, pr), (fw, pf), (occ, po) = _c(frames, np.uint8, U8P), _c(fw, np.float32, FP), _c(occ, np.uint8, U8P)
    T, H, W, _ = fr.shape
    out = np.empty((T - 1, 2), np.float64)
    hs.hs_warp_error(pr, pf, po, out.ctypes.data_as(DP), T, H, W)
    return out


def hs_sample(hs, plane, flow):
    (plane, pp), (flow, pf) = _c(plane, np.float32, FP), _c(flow, np.float32, FP)
    H, W = plane.shape
    out = np.empty((H, W), np.float32)
    hs.hs_clamp_sample(pp, pf, out.ctypes.data_as(FP), H, W)
    return out


def check_occlusion(got, fw, bw):
    """-> number of pixels inside the margin; asserts equality outside it"""
    ref, und = ewarp_ref.flow_occlusion(fw, bw), ewarp_ref.undecided(fw, bw)
    bad = (got != ref) & ~und
    assert not bad.any(), f"{int(bad.sum())} decided pixels differ, first at {np.argwhere(bad)[0]}"
    return int(und.sum())


def check_warp_error(e, ref):
    e, ref = np.asarray(e, np.float64), np.asarray(ref, np.float64)
    assert np.all(np.abs(e - ref) <= 1e-5 * ref + 1e-9), (e, ref)


# ---------------------------------------------------------------- the oracle on hand-computed cases
def test_oracle_zero_flow_identical_frames():
    fr = np.repeat(texture(1, 12, 17, 0), 3, 0)
    fw = np.zeros((2, 2, 12, 17), np.float32)
    assert not ewarp_ref.flow_occlusion(fw, fw).any()
    assert np.array_equal(ewarp_ref.warp_error(fr, fw, fw), [0.0, 0.0])


def test_oracle_translation_passes_the_forward_backward_check():
    fr, fw, bw = translation_clip(3, 20, 24, [(3, -2), (-1, 4)], seed=1)
    for F, B in zip(fw, bw):
        l1, r1, l2, r2 = ewarp_ref.occlusion_sides(F, B)
        assert (l1 == 0).all() and (l1 <= r1).all() and (l2 == 0).all()
    assert not ewarp_ref.flow_occlusion(fw, bw).any()
    # frame t+1 sampled at x + d is frame t wherever x + d stays inside the frame
    R = fr.astype(np.float64).transpose(0, 3, 1, 2)
    for t, (dx, dy) in enumerate([(3, -2), (-1, 4)]):
        w = ewarp_ref.sample(R[t + 1], fw[t])
        ys = slice(max(0, -dy), 20 - max(0, dy))
        xs = slice(max(0, -dx), 24 - max(0, dx))
        assert np.array_equal(w[:, ys, xs], R[t][:, ys, xs])
        assert not np.array_equal(w, R[t])                      # the clamped border differs


def test_oracle_far_outside_samples_the_border_pixel():
    img = np.arange(1, 1 + 3 * 5 * 7, dtype=np.float64).reshape(3, 5, 7)
    for (fx, fy), (yy, xx) in (((1000.25, -1000.5), (0, 6)), ((-5e4, 3e4), (4, 0)), ((2e3, 2e3), (4, 6))):
        f = np.empty((2, 5, 7), np.float32)
        f[0], f[1] = fx, fy
        s = ewarp_ref.sample(img, f)
        assert np.allclose(s, img[:, yy, xx][:, None, None], rtol=0, atol=1e-12)
        assert (s != 0).all()


def test_oracle_motion_boundary_fires_in_column_k_only():
    H, W, k = 9, 12, 5
    F = np.zeros((2, H, W), np.float32)
    F[0, :, k + 1:] = 3.0                                       # a vertical step between columns k and k + 1
    _, _, l2, r2 = ewarp_ref.occlusion_sides(F, -F)
    fires = l2 > r2
    assert fires[:, k].all() and fires.sum() == H
    F[1, :, -1] = 2.0                                           # a step into the last column
    _, _, l2, r2 = ewarp_ref.occlusion_sides(F, -F)
    assert (l2 > r2)[:, W - 2].all() and not (l2 > r2)[:, W - 1].any()


def test_oracle_all_occluded_pair_scores_zero():
    fr = texture(3, 10, 14, 2)
    fw = np.zeros((2, 2, 10, 14), np.float32)
    occ = np.zeros((2, 10, 14), np.uint8)
    occ[0] = 1
    sums = ewarp_ref.warp_error_sums(fr, fw, occ)
    assert sums[0, 1] == 0 and sums[1, 1] == 10 * 14
    e = ewarp_ref.warp_error(fr, fw, occ=occ)
    assert e[0] == 0.0 and e[1] > 0
    assert ewarp_ref.ewarp(fr, fw, occ=occ) == e.mean()


# ---------------------------------------------------------------- the host build against the oracle
@pytest.mark.parametrize("kind", FLOW_KINDS)
def test_hostsim_occlusion_matches_oracle(hs, kind):
    fw, bw = flow_case(kind, 3, 37, 53, seed=FLOW_KINDS.index(kind))
    occ = hs_occlusion(hs, fw, bw)
    n = check_occlusion(occ, fw, bw)
    print(f"{kind}: {int(occ.sum())} of {occ.size} occluded, {n} inside the margin")
    assert 0 < occ.sum() < occ.size or kind == "large"


@pytest.mark.parametrize("kind", FLOW_KINDS)
def test_hostsim_sample_matches_oracle(hs, kind):
    fw, _ = flow_case(kind, 1, 29, 41, seed=10 + FLOW_KINDS.index(kind))
    plane = np.random.default_rng(3).standard_normal((29, 41)).astype(np.float32) * 50
    got = hs_sample(hs, plane, fw[0])
    ref = ewarp_ref.sample(plane[None], fw[0])[0]
    assert np.abs(got - ref).max() <= 2e-6 * np.abs(plane).max()
    if kind == "integer":
        assert np.array_equal(got, ref)                         # a = b = 0: one tap, exact


@pytest.mark.parametrize("kind", FLOW_KINDS)
def test_hostsim_warp_error_matches_oracle(hs, kind):
    fw, bw = flow_case(kind, 4, 31, 47, seed=20 + FLOW_KINDS.index(kind))
    fr = texture(5, 31, 47, seed=5)
    occ = hs_occlusion(hs, fw, bw)
    sums = hs_sums(hs, fr, fw, occ)
    ref = ewarp_ref.warp_error_sums(fr, fw, occ)
    assert np.array_equal(sums[:, 1], ref[:, 1])
    check_warp_error(ewarp_ref.per_pair(sums), ewarp_ref.per_pair(ref))


def test_hostsim_translation_clip(hs):
    shifts = [(2, 0), (0, -3), (-1, 1)]
    fr, fw, bw = translation_clip(4, 24, 32, shifts, seed=7)
    occ = hs_occlusion(hs, fw, bw)
    assert not occ.any()
    sums = hs_sums(hs, fr, fw, occ)
    check_warp_error(ewarp_ref.per_pair(sums), ewarp_ref.warp_error(fr, fw, bw))
    inner = np.ones((3, 24, 32), np.uint8)
    inner[:, 4:-4, 4:-4] = 0                                    # keep only the interior
    assert (hs_sums(hs, fr, fw, inner)[:, 0] == 0).all()


# ---------------------------------------------------------------- evaluate_propainter with stand-in ops
def test_evaluate_propainter_aggregates_warp_error(hs, monkeypatch):
    """per video: the mean over its pairs (evaluate.warp_error on the host build of the kernel); over the dataset: the
    mean over videos, not frame-weighted; the script's lines unchanged"""
    from propainter_b200 import evaluate, ops

    def sums_standin(frames_u8, fw, occ=None, bw=None):
        fw, bw = fw.reshape(-1, *fw.shape[-3:]).float().numpy(), bw.reshape(-1, *bw.shape[-3:]).float().numpy()
        return torch.from_numpy(hs_sums(hs, frames_u8.numpy(), fw, hs_occlusion(hs, fw, bw)))

    def video_standin(pipe, fr, mk, fl, task, nl, rs, ri, i3d, cfg, warp_error=False):
        T = fr.shape[0]
        out = {"frames": T, "seconds": 0.01 * T, "seconds_per_frame": 0.01, "comp": fr.float()}
        ps = [20.0 + t for t in range(T)]
        out.update(psnr_per_frame=ps, ssim_per_frame=[0.5] * T, psnr=sum(ps) / T, ssim=0.5)
        if warp_error:
            out.update(evaluate.warp_error(out["comp"].to(torch.uint8), fl))
        return out

    monkeypatch.setattr(ops, "warp_error_sums", sums_standin)
    monkeypatch.setattr(evaluate, "prepare_test_video", lambda fr, mk, size, fl, dev: (torch.from_numpy(fr), mk, fl))
    monkeypatch.setattr(evaluate, "evaluate_video", video_standin)

    class Pipe:
        device = torch.device("cpu")
    videos, want = [], []
    for i, (T, kind) in enumerate(((6, "smooth"), (3, "integer"), (9, "smooth"))):
        fr = texture(T, 24, 40, seed=30 + i)
        fw, bw = flow_case(kind, T - 1, 24, 40, seed=40 + i)
        videos.append((f"v{i}", fr, None, (torch.from_numpy(fw), torch.from_numpy(bw).half())))
        bw16 = bw.astype(np.float16).astype(np.float32)
        want.append(ewarp_ref.warp_error(fr, fw, occ=hs_occlusion(hs, fw, bw16)))
    logged = []
    plain = evaluate.evaluate_propainter(Pipe(), videos, size=(40, 24))
    res = evaluate.evaluate_propainter(Pipe(), videos, size=(40, 24), warp_error=True, log=logged.append)
    for r, w in zip(res["videos"], want):
        check_warp_error(r["ewarp_per_pair"], w)
        assert abs(r["ewarp"] - w.mean()) <= 1e-5 * w.mean() + 1e-9
        assert 0 <= r["occluded_fraction"] <= 1
    per_video = [w.mean() for w in want]
    frame_weighted = sum(w.sum() for w in want) / sum(len(w) for w in want)
    assert abs(res["summary"]["ewarp"] - np.mean(per_video)) <= 1e-5 * np.mean(per_video)
    assert abs(np.mean(per_video) - frame_weighted) > 1e-3 * frame_weighted     # the two averages really differ here
    assert res["ewarp_line"] == f'Average Warping Error = {res["summary"]["ewarp"]:.6f}'
    assert res["line"] == plain["line"] and [r["line"] for r in res["videos"]] == [r["line"] for r in plain["videos"]]
    assert logged == [r["line"] for r in plain["videos"]] + [plain["line"], res["ewarp_line"]]
    assert "ewarp" not in plain["summary"] and "ewarp_line" not in plain and "ewarp" not in plain["videos"][0]


# ---------------------------------------------------------------- refusals
def test_warp_error_ops_refuse_bad_arguments():
    from propainter_b200 import ops
    z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt)
    fr = z(3, 8, 8, 3, dt=torch.uint8)
    with pytest.raises(ValueError):                             # CPU tensors: there is no CPU path
        ops.flow_occlusion(z(2, 2, 8, 8), z(2, 2, 8, 8))
    with pytest.raises(ValueError):
        ops.warp_error(fr, z(2, 2, 8, 8), bw=z(2, 2, 8, 8))
    with pytest.raises(ValueError):
        ops.flow_occlusion(z(2, 2, 8, 8), z(3, 2, 8, 8))
    with pytest.raises(ValueError):
        ops.flow_occlusion(z(2, 2, 8, 8, dt=torch.float64), z(2, 2, 8, 8, dt=torch.float64))
    for shape in ((2, 3, 8, 8), (2, 8, 8), (2, 1, 2, 8, 8), (0, 2, 8, 8)):
        with pytest.raises(ValueError):
            ops.flow_occlusion(z(*shape), z(*shape))
    with pytest.raises(ValueError):                             # T < 2
        ops.warp_error(z(1, 8, 8, 3, dt=torch.uint8), z(0, 2, 8, 8), bw=z(0, 2, 8, 8))
    with pytest.raises(ValueError):                             # frames and flows disagree
        ops.warp_error(fr, z(2, 2, 8, 9), bw=z(2, 2, 8, 9))
    with pytest.raises(ValueError):
        ops.warp_error(fr, z(3, 2, 8, 8), bw=z(3, 2, 8, 8))
    with pytest.raises(ValueError):                             # forward and backward disagree
        ops.warp_error(fr, z(2, 2, 8, 8), bw=z(1, 2, 2, 8, 8))
    with pytest.raises(ValueError):
        ops.warp_error(z(3, 8, 8, 3), z(2, 2, 8, 8), bw=z(2, 2, 8, 8))
    with pytest.raises(ValueError):                             # neither the map nor the backward flows
        ops.warp_error(fr, z(2, 2, 8, 8))
    with pytest.raises(ValueError):
        ops.warp_error(fr, z(2, 2, 8, 8), occ=z(2, 8, 8))
    with pytest.raises(ValueError):
        ops.warp_error(fr, z(2, 2, 8, 8), occ=z(3, 8, 8, dt=torch.uint8))


def test_warp_error_abi_refuses_bad_shapes():
    import __graft_entry__ as g
    g.build()
    from propainter_b200 import _lib
    L = _lib.lib()
    assert L.pp_warp_error_workspace_bytes(80, 240, 432) == 79 * 405 * 2 * 8
    assert L.pp_warp_error_workspace_bytes(30, 1080, 1920) == 29 * 1024 * 2 * 8
    assert L.pp_warp_error_workspace_bytes(1, 240, 432) == 0
    dummy = ctypes.c_void_p(16)                                  # never dereferenced: every call below returns first
    assert L.pp_warp_error(dummy, dummy, dummy, None, dummy, 1, 8, 8, dummy, 1 << 20, None) == -1
    assert L.pp_warp_error(dummy, dummy, dummy, None, dummy, 3, 0, 8, dummy, 1 << 20, None) == -1
    assert L.pp_warp_error(dummy, dummy, None, None, dummy, 3, 8, 8, dummy, 1 << 20, None) == -1
    assert L.pp_warp_error(dummy, dummy, dummy, None, dummy, 3, 8, 8, dummy, 16, None) == -3
    assert L.pp_flow_occlusion(dummy, dummy, dummy, 0, 8, 8, None) == -1
