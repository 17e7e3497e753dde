"""CPU tests of video outpainting: the canvas geometry against the reference's expressions, the host build of the two
per-element rules (canvas + masks, green preview) against oracle/outpaint_ref.py bit for bit, and the oracle against the
outpainting fixtures produced by the reference's own code (tests/golden/make_golden_outpaint.py).  The kernels and the
pipeline run on the GPU in test_gpu_outpaint.py."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import ops_ref, outpaint_ref, pipeline_ref
from propainter_b200 import synth
from propainter_b200.inference_propainter import outpaint_geometry
from tests.test_oracle_golden import compare_stages, seeded_state_dicts

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
U8P = ctypes.POINTER(ctypes.c_uint8)
FP = ctypes.POINTER(ctypes.c_float)

# (T, h, w, scale_h, scale_w) -> offsets: 0 / 16 (rim); 16 (rim) / 4; odd margins 19 -> 9 and 37 -> 18 (rim);
# h = 7 inside a rim of 4 at offset 12 (empty inner row range); h = 8 = 2 * rim (empty); offset 9 <= 10 (no rim) / 0
GEOMETRIES = [(2, 128, 128, 1.0, 1.3), (2, 128, 128, 1.25, 1.1), (3, 125, 131, 1.2, 1.3), (1, 7, 9, 5.0, 5.0),
              (1, 8, 8, 4.0, 4.0), (2, 6, 40, 4.0, 1.0)]
GOLDEN = {"outpaint_8x128x128_s1.0x1.3_it6": (1.0, 1.3), "outpaint_8x128x128_s1.25x1.1_it6": (1.25, 1.1)}


@pytest.fixture(scope="module")
def hs(tmp_path_factory):
    lib = os.path.join(str(tmp_path_factory.mktemp("hostsim_outpaint")), "libhostsim_outpaint.so")
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", lib,
                           os.path.join(HERE, "hostsim", "hostsim_outpaint.cpp")])
    return ctypes.CDLL(lib)


def reference_expressions(h, w, sh, sw):
    """inference_propainter.py:124-128, :142-143 as written there"""
    imgH_extr, imgW_extr = int(sh * h), int(sw * w)
    imgH_extr, imgW_extr = imgH_extr - imgH_extr % 8, imgW_extr - imgW_extr % 8
    H_start, W_start = int((imgH_extr - h) / 2), int((imgW_extr - w) / 2)
    return (imgH_extr, imgW_extr), (H_start, W_start), (4 if H_start > 10 else 0, 4 if W_start > 10 else 0)


def test_geometry_matches_reference_expressions():
    n = 0
    for h in (8, 64, 128, 135, 240, 360, 432, 480, 720, 1080, 1920):
        for s in (1.0, 1.05, 1.1, 1.2, 1.25, 1.3, 1.4, 1.5, 1.7, 2.0, 3.0):
            if int(s * h) // 8 * 8 < h:
                continue
            for w, sw in ((432, 1.2), (h, s)):
                got = outpaint_geometry(h, w, s, sw)
                assert got == reference_expressions(h, w, s, sw) == outpaint_ref.geometry(h, w, s, sw), (h, w, s, sw)
                n += 1
    assert n > 150
    # Python doubles, not fp32: 1.4 * 360 = 503.99999999999994
    assert outpaint_geometry(360, 640, 1.4, 1.0)[0] == (496, 640)
    assert int(np.float32(1.4) * np.float32(360)) // 8 * 8 == 504
    assert outpaint_geometry(720, 1280, 1.4, 1.0)[0] == (1000, 1280)
    assert outpaint_geometry(240, 432, 1.0, 1.2) == ((240, 512), (0, 40), (0, 4))          # the script's defaults on C2
    assert outpaint_geometry(1080, 1920, 2.0, 2.0) == ((2160, 3840), (540, 960), (4, 4))


@pytest.mark.parametrize("h,w,sh,sw", [(240, 432, 0.9, 1.2), (240, 432, 1.0, 0.5), (130, 432, 1.0, 1.2),
                                       (240, 431, 1.2, 1.0), (240, 432, float("nan"), 1.2), (240, 432, 1.0, float("inf")),
                                       (240, 432, -1.0, 1.2)])
def test_geometry_refuses_canvas_smaller_than_source(h, w, sh, sw):
    with pytest.raises(ValueError):
        outpaint_geometry(h, w, sh, sw)


def _hs_extrapolate(hs, u8, geo):
    (H, W), (top, left), (rh, rw) = geo
    T, h, w, _ = u8.shape
    src = np.ascontiguousarray(u8)
    canvas = np.empty((T, H, W, 3), np.uint8)
    fm, md = np.empty((T, 1, H, W), np.float32), np.empty((T, 1, H, W), np.float32)
    hs.hs_extrapolate_u8(src.ctypes.data_as(U8P), canvas.ctypes.data_as(U8P), fm.ctypes.data_as(FP), md.ctypes.data_as(FP),
                         T, h, w, H, W, top, left, rh, rw)
    return canvas, fm, md


@pytest.mark.parametrize("T,h,w,sh,sw", GEOMETRIES)
def test_hostsim_extrapolate_matches_oracle(hs, T, h, w, sh, sw):
    rng = np.random.default_rng(h * 1000 + w)
    u8 = rng.integers(0, 256, (T, h, w, 3), dtype=np.uint8)
    geo = outpaint_geometry(h, w, sh, sw)
    canvas, fm, md = _hs_extrapolate(hs, u8, geo)
    ref_c, ref_fm, ref_md, size = outpaint_ref.extrapolate(u8, sh, sw)
    assert size == (geo[0][1], geo[0][0])
    assert np.array_equal(canvas, ref_c)
    assert np.array_equal(fm, ref_fm[0].numpy()) and np.array_equal(md, ref_md[0].numpy())
    (H, W), (top, left), (rh, rw) = geo
    assert (md == 0).sum() == T * h * w                                     # the source rectangle, exactly
    if h <= 2 * rh or w <= 2 * rw:
        assert (fm == 1).all()                                              # the rim swallows the source
    else:
        assert (fm == 0).sum() == T * (h - 2 * rh) * (w - 2 * rw)


def test_hostsim_mask_overlay_exhaustive(hs):
    """every uint8 value in every channel, mask 0 and 1, against numpy's float64 expression"""
    v = np.arange(256, dtype=np.uint8).reshape(16, 16)
    frames = np.ascontiguousarray(np.stack([np.stack([v, v, v], -1)] * 2))            # [2,16,16,3]
    masks = np.zeros((2, 1, 16, 16), np.float32)
    masks[1] = 1.0
    out = np.empty_like(frames)
    hs.hs_mask_overlay_u8(frames.ctypes.data_as(U8P), masks.ctypes.data_as(FP), out.ctypes.data_as(U8P), 2, 16, 16)
    ref = outpaint_ref.mask_overlay(frames, masks)
    assert np.array_equal(out, ref)
    assert np.array_equal(out[0], frames[0])                                 # mask 0: the frame itself
    img = np.arange(256, dtype=np.float64)
    for c, g in enumerate((0.0, 255.0, 0.0)):                                # mask 1: (0.4*img + 0.6*green) truncated
        assert np.array_equal(out[1, ..., c].ravel(), ((1 - 0.6) * img + 0.6 * g).astype(np.uint8))


@pytest.mark.parametrize("name", list(GOLDEN))
def test_oracle_reproduces_outpaint_golden(name):
    g = np.load(os.path.join(GOLD, name + ".npz"))
    sh, sw = GOLDEN[name]
    assert tuple(g["scale"]) == (sh, sw)
    u8, _, _ = synth.make_clip(8, 128, 128, seed=0)
    canvas, fm, md, size = outpaint_ref.extrapolate(u8, sh, sw)
    assert size == tuple(g["size"])
    H, W = canvas.shape[1:3]
    assert np.array_equal(np.unpackbits(g["flow_mask0"])[:H * W].reshape(H, W), fm[0, 0, 0].numpy().astype(np.uint8))
    assert np.array_equal(np.unpackbits(g["mask_dilated0"])[:H * W].reshape(H, W), md[0, 0, 0].numpy().astype(np.uint8))
    comp, st = pipeline_ref.run_pipeline(seeded_state_dicts(), canvas, fm, md, raft_iter=6, return_stages=True)
    res = compare_stages(g, st, {"gt": 1e-5, "pred": 1e-5})
    assert res["upd_m_mismatch"] == 0.0
    d = np.abs(comp.astype(int) - g["comp"].astype(int))
    assert d.max() <= 1 and (d > 0).mean() < 1e-4 and ops_ref.psnr_u8(comp, g["comp"]) > 85.0


def test_outpaint_ops_refuse_cpu_tensors():
    from propainter_b200 import ops
    from propainter_b200.inference_propainter import prepare_outpainting
    u8 = torch.zeros(1, 16, 16, 3, dtype=torch.uint8)
    with pytest.raises(RuntimeError):
        ops.extrapolate_u8(u8, outpaint_geometry(16, 16, 1.0, 1.5))
    with pytest.raises(RuntimeError):
        ops.mask_overlay_u8(u8, torch.zeros(1, 1, 16, 16))
    with pytest.raises(RuntimeError):
        prepare_outpainting(u8, 1.0, 1.5, device="cpu")
