"""GPU tests of video outpainting: k_extrapolate_u8 and k_mask_overlay_u8 bit-exact against oracle/outpaint_ref.py, and
ProPainterPipeline.outpaint against the oracle pipeline (fp32 library math) and against the fixtures the reference's own
code produced (shipping defaults)."""
import os

import numpy as np
import pytest
import torch

from oracle import ops_ref, outpaint_ref, pipeline_ref
from tests.test_outpaint_host import GEOMETRIES, GOLDEN

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(autouse=True)
def _exact_library_math(request):
    """fp32 library convs / GEMMs, except for tests marked `shipping` (the defaults bench.py runs)"""
    from propainter_b200 import config
    if "shipping" in request.keywords:
        yield
        return
    a, b, c = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32, config.LINEAR_TF32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    config.LINEAR_TF32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32, config.LINEAR_TF32 = a, b, c


def sds_of(pipe):
    return {k: {n: v.detach().cpu() for n, v in sd.items()} for k, sd in pipe.state_dicts().items()}


# the host-test geometries, plus T = 1, T = 17 and a source whose sides are not multiples of 8
@pytest.mark.parametrize("T,h,w,sh,sw", GEOMETRIES + [(1, 128, 128, 1.0, 1.3), (17, 64, 96, 1.25, 1.2), (3, 141, 203, 1.3, 1.2)])
def test_extrapolate_bit_exact(T, h, w, sh, sw):
    from propainter_b200 import ops
    from propainter_b200.inference_propainter import outpaint_geometry
    u8 = np.random.default_rng(T * 7 + h).integers(0, 256, (T, h, w, 3), dtype=np.uint8)
    canvas, fm, md = ops.extrapolate_u8(torch.from_numpy(u8).to(DEV), outpaint_geometry(h, w, sh, sw))
    ref_c, ref_fm, ref_md, _ = outpaint_ref.extrapolate(u8, sh, sw)
    assert np.array_equal(canvas.cpu().numpy(), ref_c)
    assert torch.equal(fm.cpu(), ref_fm[0]) and torch.equal(md.cpu(), ref_md[0])


def test_extrapolate_1080p_to_4k():
    """1920x1080 at scale 2.0: a 3840x2160 canvas (8.3 M pixels per frame), through prepare_outpainting"""
    from propainter_b200.inference_propainter import prepare_outpainting
    u8 = np.random.default_rng(4).integers(0, 256, (2, 1080, 1920, 3), dtype=np.uint8)
    canvas, fm, md, size = prepare_outpainting(torch.from_numpy(u8), 2.0, 2.0)
    ref_c, ref_fm, ref_md, ref_size = outpaint_ref.extrapolate(u8, 2.0, 2.0)
    assert size == ref_size == (3840, 2160)
    assert canvas.shape == (2, 2160, 3840, 3) and fm.shape == md.shape == (1, 2, 1, 2160, 3840)
    assert np.array_equal(canvas.cpu().numpy(), ref_c)
    assert torch.equal(fm.cpu(), ref_fm) and torch.equal(md.cpu(), ref_md)


def test_mask_overlay_bit_exact():
    """k_mask_overlay_u8 against numpy's float64 expression: every uint8 value with mask 0 and 1, then random frames with
    the masks of both modes (outpainting border, dilated inpainting ellipse)"""
    from propainter_b200 import ops, synth
    from propainter_b200.inference_propainter import ProPainterPipeline, prepare_outpainting
    v = np.arange(256, dtype=np.uint8).reshape(16, 16)
    frames = np.ascontiguousarray(np.stack([np.stack([v, v, v], -1)] * 2))
    masks = torch.zeros(2, 1, 16, 16)
    masks[1] = 1.0
    got = ops.mask_overlay_u8(torch.from_numpy(frames).to(DEV), masks.to(DEV)).cpu().numpy()
    assert np.array_equal(got, outpaint_ref.mask_overlay(frames, masks.numpy()))
    rng = np.random.default_rng(9)
    src = rng.integers(0, 256, (5, 120, 200, 3), dtype=np.uint8)
    canvas, _, md_out, _ = prepare_outpainting(torch.from_numpy(src), 1.2, 1.3)
    _, _, md_in = synth.make_clip(5, 120, 200, mask="ellipse", seed=2)
    md_in = ops.mask_dilate((md_in[0, :, 0] > 0).to(torch.uint8).to(DEV), 4).unsqueeze(0)
    pipe = ProPainterPipeline(device=DEV)
    for fr, md in ((canvas, md_out), (torch.from_numpy(src).to(DEV), md_in)):
        fr = torch.from_numpy(rng.integers(0, 256, tuple(fr.shape), dtype=np.uint8)).to(DEV)
        got = pipe.masked_preview(fr, md).cpu().numpy()
        assert 0 < md.mean().item() < 1
        assert np.array_equal(got, outpaint_ref.mask_overlay(fr.cpu().numpy(), md.cpu().numpy()))


def test_outpaint_matches_oracle_fp32():
    """outpaint (fp32 library math) against the oracle pipeline run on the oracle's canvas and masks"""
    from propainter_b200 import synth
    from propainter_b200.inference_propainter import InferenceConfig, ProPainterPipeline
    u8, _, _ = synth.make_clip(8, 128, 128, seed=0)
    pipe = ProPainterPipeline(device=DEV)
    comp = pipe.outpaint(torch.from_numpy(u8), 1.25, 1.1, InferenceConfig(raft_iter=6)).cpu().numpy()
    canvas, fm, md, _ = outpaint_ref.extrapolate(u8, 1.25, 1.1)
    ref = pipeline_ref.run_pipeline(sds_of(pipe), canvas, fm, md, raft_iter=6)
    psnr = ops_ref.psnr_u8(comp, ref)
    print(f"outpaint (1.25, 1.1) fp32 vs oracle: PSNR {psnr:.2f} dB, max diff {np.abs(comp.astype(int) - ref.astype(int)).max()}")
    assert comp.shape == (8, 160, 136, 3) and psnr >= 60.0           # measured 76.6 dB, max diff 1 level


@pytest.mark.shipping
@pytest.mark.parametrize("name", list(GOLDEN))
def test_outpaint_shipping_vs_golden(name):
    """Shipping defaults against the reference's outpainting output: PSNR, replay, and the source rectangle kept exactly"""
    from propainter_b200 import synth
    from propainter_b200.inference_propainter import InferenceConfig, ProPainterPipeline, outpaint_geometry
    g = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))
    sh, sw = GOLDEN[name]
    u8, _, _ = synth.make_clip(8, 128, 128, seed=0)
    pipe = ProPainterPipeline(device=DEV)
    cfg = InferenceConfig(raft_iter=6)
    a = pipe.outpaint(torch.from_numpy(u8), sh, sw, cfg).cpu().numpy()
    b = pipe.outpaint(torch.from_numpy(u8), sh, sw, cfg).cpu().numpy()      # second call replays the captured graphs
    assert np.array_equal(a, b)
    psnr = ops_ref.psnr_u8(a, g["comp"])
    print(f"{name}: shipping defaults vs reference golden: PSNR {psnr:.2f} dB, "
          f"max diff {np.abs(a.astype(int) - g['comp'].astype(int)).max()}")
    assert psnr >= 58.0                                              # measured 69.2 / 68.4 dB, max diff 1 level
    _, (top, left), _ = outpaint_geometry(128, 128, sh, sw)
    assert np.array_equal(a[:, top:top + 128, left:left + 128], u8)


@pytest.mark.shipping
def test_outpaint_c2_default_scale():
    """The C2 source (80 x 240 x 432) at the script's default scale (1.0, 1.2): a 240 x 512 canvas, finite stages"""
    from propainter_b200 import synth
    from propainter_b200.inference_propainter import ProPainterPipeline
    u8, _, _ = synth.make_clip(80, 240, 432, mask="ellipse", seed=0)
    pipe = ProPainterPipeline(device=DEV)
    comp, st = pipe.outpaint(torch.from_numpy(u8), return_stages=True)
    assert comp.shape == (80, 240, 512, 3) and comp.dtype == torch.uint8
    for k in ("gt_flows", "pred_flows"):
        assert all(torch.isfinite(f).all() for f in st[k]), k
    assert torch.isfinite(st["updated_frames"]).all()
    assert torch.equal(comp[:, :, 40:472].cpu(), torch.from_numpy(u8))
