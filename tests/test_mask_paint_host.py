"""CPU tests of the tracking preview (BaseTracker.track's painter loop, tools/painter.py mask_painter): the oracle
(oracle/painter_ref.py) against the reference's own output in tests/golden/painter_cases.npz (made by
tests/golden/make_golden_painter.py), the chamfer-table rule against cv2.distanceTransform, the host build of the
pp_paint_* rules of pp_elem.cuh (tests/hostsim/hostsim_paint.cpp) against the oracle over a dense random sweep, and the
refusals of ops.mask_paint_u8.  The kernels run on the GPU in test_gpu_mask_paint.py."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import painter_ref
from propainter_b200 import ops

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from cutie_inputs import CLIP, make_clip  # noqa: E402

FIXTURE = os.path.join(HERE, "golden", "painter_cases.npz")
U8P, FP = ctypes.POINTER(ctypes.c_uint8), ctypes.POINTER(ctypes.c_float)


@pytest.fixture(scope="module")
def hs(tmp_path_factory):
    lib = str(tmp_path_factory.mktemp("hostsim_paint") / "libhostsim_paint.so")
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", lib,
                           os.path.join(HERE, "hostsim", "hostsim_paint.cpp")])
    h = ctypes.CDLL(lib)
    h.hs_paint_chamfer.restype = ctypes.c_float
    h.hs_paint_chamfer.argtypes = [ctypes.c_int, ctypes.c_int]
    h.hs_paint_dist.argtypes = [U8P, ctypes.c_int, ctypes.c_int, ctypes.c_int, FP]
    h.hs_paint_contour.restype = ctypes.c_int
    h.hs_paint_contour.argtypes = [ctypes.c_float, ctypes.c_float]
    h.hs_paint_fill.restype = ctypes.c_uint8
    h.hs_paint_fill.argtypes = [ctypes.c_uint8, ctypes.c_uint8, ctypes.c_double, ctypes.c_double]
    h.hs_mask_paint_u8.argtypes = [U8P, U8P, U8P, ctypes.c_int, ctypes.c_double, ctypes.c_double, U8P, ctypes.c_int,
                                   ctypes.c_int, ctypes.c_int, FP]
    return h


@pytest.fixture(scope="module")
def golden():
    return np.load(FIXTURE)


def fixture_cases(g):
    """[(name, frames [T,H,W,3], labels [T,H,W], painted)] of the synthetic cases and the BaseTracker frames"""
    out = [(str(n), g[f"case{i}_frames"], g[f"case{i}_labels"], g[f"case{i}_painted"]) for i, n in enumerate(g["case_names"])]
    frames, _ = make_clip(CLIP["T"], CLIP["H"], CLIP["W"], CLIP["seed"])
    out.append(("base_tracker", frames[g["tracker_t"]], g["tracker_labels"], g["tracker_painted"]))
    return out


def show_labels(g):
    """the show_mask case as a label map: mask i of the selection -> id i + 1"""
    lab = np.zeros(g["show_frame"].shape[:2], np.uint8)
    for i in g["show_selected"]:
        lab[g["show_masks"][i] != 0] = i + 1
    return lab


def host_paint(hs, frames, labels, palette, alpha=0.7):
    frames, labels = np.ascontiguousarray(frames, np.uint8), np.ascontiguousarray(labels, np.uint8)
    palette = np.ascontiguousarray(palette, np.uint8)
    T, H, W = labels.shape
    out = np.empty_like(frames)
    maxima = np.empty((T, 256), np.float32)
    hs.hs_mask_paint_u8(frames.ctypes.data_as(U8P), labels.ctypes.data_as(U8P), palette.ctypes.data_as(U8P), len(palette),
                        alpha, 1 - alpha, out.ctypes.data_as(U8P), T, H, W, maxima.ctypes.data_as(FP))
    return out, maxima


def random_clip(rng, T, H, W, kind, max_id=20):
    frames = rng.integers(0, 256, (T, H, W, 3), dtype=np.uint8)
    if kind == "noise":
        labels = rng.integers(0, 4, (T, H, W))
    elif kind == "sparse":
        labels = (rng.random((T, H, W)) < 0.1) * rng.integers(1, max_id + 1, (T, H, W))
    elif kind == "blobs":
        labels = np.zeros((T, H, W), np.int64)
        yy, xx = np.mgrid[0:H, 0:W]
        for t in range(T):
            for _ in range(rng.integers(0, 6)):
                cy, cx, r = rng.uniform(-3, H + 3), rng.uniform(-3, W + 3), rng.uniform(0.5, max(H, W) / 2)
                labels[t][(yy - cy) ** 2 + (xx - cx) ** 2 <= r * r] = rng.integers(1, max_id + 1)
    elif kind == "dense":
        labels = rng.integers(0, max_id + 1, (T, H, W))
    else:                                                         # one id filling whole frames, or nothing
        labels = np.broadcast_to(rng.integers(0, 3, (T, 1, 1)), (T, H, W))
    return frames, np.ascontiguousarray(labels, np.uint8)


def test_oracle_equals_fixture(golden):
    """the oracle paints every fixture case (synthetic, BaseTracker.track's frames, show_mask) byte for byte as the
    reference did"""
    pal = golden["palette"]
    for name, frames, labels, painted in fixture_cases(golden):
        assert np.array_equal(painter_ref.paint_clip(frames, labels, pal), painted), name
    shown = painter_ref.paint_frame(golden["show_frame"], show_labels(golden), pal)
    assert np.array_equal(shown, golden["show_painted"])


def test_fixture_covers_the_contract(golden):
    """the fixture holds what the contract's corner cases need: ids up to 20, maxima below 3 including the exact-0.5
    ones (a + a, b + b), whole-frame and empty frames, BaseTracker frames with both objects"""
    a, b = painter_ref.A, painter_ref.B
    maxima, ids = set(), set()
    for _, _, labels, _ in fixture_cases(golden):
        for lab in labels:
            ids |= set(np.unique(lab).tolist())
            maxima |= {np.float32(m) for m in painter_ref.object_maxima(lab).values()}
    assert {0, 1, 2, 3, 20} <= ids
    assert {np.float32(a + a), np.float32(b + b), np.float32(3)} <= maxima
    assert all({1, 2} <= set(np.unique(lab).tolist()) for lab in golden["tracker_labels"])


def test_chamfer_table_equals_cv2_distance_transform():
    """min(cv2.distanceTransform(DIST_L2, 3), 3) equals the chamfer-table rule on random, rectangle, all-0 and all-1
    masks, and the oracle's painting with either transform is the same"""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(11)
    n = 0
    for trial in range(200):
        H, W = rng.integers(1, 50, 2)
        kind = trial % 4
        if kind == 0:
            m = (rng.random((H, W)) < rng.uniform(0.02, 0.98)).astype(np.uint8)
        elif kind == 1:
            m = np.zeros((H, W), np.uint8)
            y0, x0 = rng.integers(0, H), rng.integers(0, W)
            m[y0:y0 + rng.integers(1, H + 1), x0:x0 + rng.integers(1, W + 1)] = 1
        else:
            m = np.full((H, W), kind - 2, np.uint8)
        want = np.minimum(cv2.distanceTransform(m, cv2.DIST_L2, 3), np.float32(3))
        assert np.array_equal(painter_ref.clipped_dt_table(m), want), (trial, H, W)
        n += m.size
    frames, labels = random_clip(rng, 3, 31, 45, "noise")
    pal = ops.paint_palette()
    assert np.array_equal(painter_ref.paint_clip(frames, labels, pal, cv2=True), painter_ref.paint_clip(frames, labels, pal))
    assert n > 50000


def test_rules_chamfer_contour_fill(hs):
    """the element rules: the path-sum table in float32, the contour test with its two float32 roundings at every
    (v, M) pair the table allows (v / M exactly 0.5 is not a contour), the float64 fill over all 256 x 256 values"""
    a, b = painter_ref.A, painter_ref.B
    for dy in range(-4, 5):
        for dx in range(-4, 5):
            want = painter_ref.CHAMFER.get((max(abs(dy), abs(dx)), min(abs(dy), abs(dx))), np.float32(3))
            assert np.float32(hs.hs_paint_chamfer(dy, dx)) == want, (dy, dx)
    vals = sorted(set(painter_ref.CHAMFER.values()) | {np.float32(3)})
    for v in vals:
        for M in vals:
            if M >= v:
                want = (np.float32(1) - np.float32(v) / np.float32(M)) > np.float32(0.5)
                assert bool(hs.hs_paint_contour(v, M)) == bool(want), (v, M)
    assert not hs.hs_paint_contour(b, b + b) and not hs.hs_paint_contour(a, a + a) and hs.hs_paint_contour(b, 3.0)
    img = np.arange(256).repeat(256).astype(np.uint8)
    col = np.tile(np.arange(256), 256).astype(np.uint8)
    for alpha in (0.7, 0.5, 0.35):
        want = (img * (1 - alpha) + col.astype(np.int64) * alpha).astype(np.uint8)
        got = np.array([hs.hs_paint_fill(int(i), int(c), alpha, 1 - alpha) for i, c in zip(img, col)], np.uint8)
        assert np.array_equal(got, want), alpha


def test_hostsim_distance_equals_oracle(hs):
    rng = np.random.default_rng(5)
    for trial in range(60):
        H, W = rng.integers(1, 30, 2)
        lab = rng.integers(0, 3, (H, W)).astype(np.uint8) if trial % 2 else (rng.random((H, W)) < 0.5).astype(np.uint8) * 2
        for k in (1, 2):
            got = np.empty((H, W), np.float32)
            hs.hs_paint_dist(np.ascontiguousarray(lab).ctypes.data_as(U8P), H, W, k, got.ctypes.data_as(FP))
            assert np.array_equal(got, painter_ref.object_v((lab == k).astype(np.uint8))), (trial, k)


def test_hostsim_equals_fixture(hs, golden):
    for name, frames, labels, painted in fixture_cases(golden):
        assert np.array_equal(host_paint(hs, frames, labels, golden["palette"])[0], painted), name


@pytest.mark.parametrize("kind", ["noise", "sparse", "blobs", "dense", "full"])
def test_hostsim_equals_oracle_sweep(hs, kind):
    """random clips from 1 x 1 to 40 x 40 pixels, ids up to 20 (and up to 255 with the default palette), several
    alphas: bytes and the per-(frame, id) maxima equal the oracle's"""
    rng = np.random.default_rng(len(kind) * 977 + ord(kind[0]))
    demo = np.load(FIXTURE)["palette"]
    for trial in range(40):
        T, H, W = rng.integers(1, 4), rng.integers(1, 41), rng.integers(1, 41)
        wide = trial % 5 == 4
        frames, labels = random_clip(rng, T, H, W, kind, 255 if wide else 20)
        pal = ops.paint_palette() if wide else demo
        alpha = (0.7, 0.5, 1.0, 0.0, 0.3)[trial % 5]
        got, maxima = host_paint(hs, frames, labels, pal, alpha)
        assert np.array_equal(got, painter_ref.paint_clip(frames, labels, pal, alpha)), (trial, T, H, W, alpha)
        for t in range(T):
            for k, m in painter_ref.object_maxima(labels[t]).items():
                assert maxima[t, k] == np.float32(m), (trial, t, k)


def test_default_palette():
    """257 distinct rows: black, white (the demo's contour colour), then the VOC colormap from colour 1 on"""
    p = ops.paint_palette()
    assert p.shape == (257, 3) and p.dtype == np.uint8 and len({tuple(r) for r in p.tolist()}) == 257
    assert p[0].tolist() == [0, 0, 0] and p[1].tolist() == [255, 255, 255]
    assert p[2:6].tolist() == [[128, 0, 0], [0, 128, 0], [128, 128, 0], [0, 0, 128]]


def test_mask_paint_refusals():
    """ValueError for CPU tensors, other dtypes or shapes, a palette that is not uint8 [N,3], mask_alpha outside [0, 1]
    and a present id without its palette row"""
    fr, lab = torch.zeros(2, 8, 9, 3, dtype=torch.uint8), torch.zeros(2, 8, 9, dtype=torch.uint8)
    with pytest.raises(ValueError, match="CUDA"):
        ops.mask_paint_u8(fr, lab)
    bad = [(fr.float(), lab), (fr[..., :2], lab), (fr[0], lab[0]), (fr[:0], lab[:0]), (fr, lab.int()), (fr, lab[:, :7]),
           (fr, lab[0]), (fr.numpy(), lab)]
    for f, l in bad:
        with pytest.raises(ValueError):
            ops.mask_paint_u8(f, l)
    for pal in (np.zeros((5, 3), np.float32), np.zeros((5, 4), np.uint8), np.zeros(15, np.uint8), np.zeros((1, 3), np.uint8)):
        with pytest.raises(ValueError, match="palette"):
            ops.mask_paint_u8(fr, lab, pal)
    for alpha in (-0.1, 1.5, float("nan")):
        with pytest.raises(ValueError, match="mask_alpha"):
            ops.mask_paint_u8(fr, lab, mask_alpha=alpha)
    lab[1, 3, 4] = 4                                           # id 4 needs row 5
    with pytest.raises(ValueError, match="row 5"):
        ops.mask_paint_u8(fr, lab, np.zeros((5, 3), np.uint8))
    with pytest.raises(ValueError, match="CUDA"):
        ops.mask_paint_u8(fr, lab, np.zeros((6, 3), np.uint8))
