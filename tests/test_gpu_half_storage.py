"""Half-precision clip storage (InferenceConfig.half_storage) on the GPU.

With the option on, the four clip-resident stage outputs are rounded once to fp16 (R1 RAFT flows, R2 completed flows, R3
updated frames / masks, R4 encoder features) and every consumer widens them to fp32.  So the result is reproducible
exactly: the kernels that read fp16 equal their fp32 instantiations on the upcast inputs, and the whole pipeline equals
the fp32 stage methods with `.half().float()` applied at R1-R4.  Precision against the fp32 pipeline and the reference
golden, the memory saved and the option's surfaces are checked as well.
"""
import contextlib
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import ops_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
F16 = torch.float16
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@contextlib.contextmanager
def _pinned(graphs=None):
    """plan choices fixed identically for the runs a test compares (no cuDNN search, no plan timing)"""
    from propainter_b200 import config
    prev = (config.AUTOTUNE, config.CUDNN_BENCHMARK, config.UMMA_CONV, config.CUDA_GRAPHS)
    config.AUTOTUNE, config.CUDNN_BENCHMARK, config.UMMA_CONV = False, False, True
    if graphs is not None:
        config.CUDA_GRAPHS = graphs
    try:
        yield
    finally:
        config.AUTOTUNE, config.CUDNN_BENCHMARK, config.UMMA_CONV, config.CUDA_GRAPHS = prev


def _smooth_flow(gen, n, H, W, amp=4.0):
    z = torch.randn(n, 2, H // 8 + 2, W // 8 + 2, generator=gen) * amp
    return F.interpolate(z, size=(H, W), mode="bicubic", align_corners=False)


def _in_nan(x, pad=1):
    """x placed in the middle of a NaN-filled buffer with `pad` extra frames on either side -> (view, buffer)"""
    buf = torch.full((x.shape[0] + 2 * pad,) + tuple(x.shape[1:]), float("nan"), device=DEV, dtype=x.dtype)
    buf[pad:pad + x.shape[0]] = x
    return buf[pad:pad + x.shape[0]], buf


# ---------------------------------------------------------------- kernel level, bit for bit
@pytest.mark.parametrize("T,H,W,lo,hi,nearest", [(8, 128, 128, 0, 8, 1), (8, 128, 128, 0, 8, 0), (80, 240, 432, 0, 80, 1),
                                                 (30, 240, 432, 10, 20, 1), (23, 128, 128, 0, 13, 1), (1, 64, 64, 0, 1, 1)])
def test_scan_u8h_equals_fp32_scan_rounded(T, H, W, lo, hi, nearest):
    """pp_img_prop_scan_u8h = rn16 of (u8_to_frames, masked, the fp32 scan on the upcast flows, the compose) for the kept
    frames; operands in NaN-filled wider buffers, nothing outside the written frames changes, updated masks in {0, 1}"""
    from propainter_b200 import ops
    gen = torch.Generator().manual_seed(T + H)
    u8 = torch.randint(0, 256, (T, H, W, 3), dtype=torch.uint8, generator=gen).to(DEV)
    masks = torch.zeros(T, 1, H, W)
    masks[..., H // 4:3 * H // 4, W // 5:3 * W // 4] = 1
    masks[::3, :, :5, :7] = 1
    masks = masks.to(DEV)
    if T > 1:
        ff = _smooth_flow(gen, T - 1, H, W)
        fb = -ff + 0.3 * _smooth_flow(gen, T - 1, H, W)
    else:
        ff = fb = torch.zeros(0, 2, H, W)
    ff16, fb16 = ff.half().to(DEV), fb.half().to(DEV)

    frames = ops.u8_to_frames(u8)
    prop, um = ops.img_prop_scan((frames * (1 - masks)).contiguous(), ff16.float().contiguous(), fb16.float().contiguous(), masks,
                                 bool(nearest))
    ref_f = (frames * (1 - masks) + prop * masks)[lo:hi].half()
    ref_m = um[lo:hi].half()

    ffv, _ = _in_nan(ff16)
    fbv, _ = _in_nan(fb16)
    mv, _ = _in_nan(masks)
    of, ofb = _in_nan(torch.full((hi - lo, 3, H, W), float("nan"), device=DEV, dtype=F16))
    om, omb = _in_nan(torch.full((hi - lo, 1, H, W), float("nan"), device=DEV, dtype=F16))
    ops.img_prop_scan_u8h(u8, mv, ffv, fbv, of, om, lo, hi, bool(nearest))
    torch.cuda.synchronize()
    assert torch.equal(of.view(torch.int16), ref_f.view(torch.int16))
    assert torch.equal(om.view(torch.int16), ref_m.view(torch.int16))
    assert set(om.unique().tolist()) <= {0.0, 1.0}
    for b in (ofb, omb):
        assert bool(b[0].isnan().all()) and bool(b[-1].isnan().all())


@pytest.mark.parametrize("lt,t,H,W", [(10, 18, 240, 432), (6, 6, 128, 128), (1, 3, 64, 64)])
def test_gen_prep_f16_equals_fp32(lt, t, H, W):
    from propainter_b200 import ops
    gen = torch.Generator().manual_seed(lt)
    ff = _smooth_flow(gen, max(lt - 1, 1), H, W)[:lt - 1].half().to(DEV)
    fb = _smooth_flow(gen, max(lt - 1, 1), H, W)[:lt - 1].half().to(DEV)
    mi = (torch.rand(t, 1, H, W, generator=gen) > 0.6).float().to(DEV)
    mu = (torch.rand(t, 1, H, W, generator=gen) > 0.8).float().to(DEV)
    ffv, ffb = _in_nan(ff)
    fbv, _ = _in_nan(fb)
    got = ops.gen_prep(ffv, fbv, mi, mu, lt)
    ref = ops.gen_prep(ff.float().contiguous(), fb.float().contiguous(), mi, mu, lt)
    for a, b in zip(got, ref):
        assert torch.equal(a, b)
    assert bool(ffb[0].isnan().all())


# ---------------------------------------------------------------- pipeline level, bit for bit
def _emulate(pipe, u8, fm, md, cfg):
    """the fp32 stage methods with .half().float() at R1-R4"""
    from propainter_b200 import ops
    r = lambda pair: tuple(x.half().float() for x in pair)
    ori = u8.to(DEV)
    frames = ops.u8_to_frames(ori).unsqueeze(0)
    gt = r(pipe.compute_flows(frames, cfg))
    pred = r(pipe.complete_flows(gt, fm, cfg))
    upd_f, upd_m = r(pipe.propagate_images(frames, md, pred, cfg))
    enc = pipe.model.encode
    pipe.model.encode = lambda *a, **k: enc(*a, **k).half().float()
    try:
        comp = pipe.generate(upd_f, md, upd_m, pred, ori, cfg)
    finally:
        del pipe.model.encode
    return comp, {"gt_flows": gt, "pred_flows": pred, "updated_frames": upd_f, "updated_masks": upd_m}


@pytest.mark.parametrize("T,H,W,kw", [(8, 128, 128, dict(raft_iter=4)),
                                      (48, 128, 128, dict(raft_iter=2, subvideo_length=16, raft_clip_frames=12))])
def test_pipeline_equals_stage_boundary_emulation(T, H, W, kw):
    from propainter_b200 import synth
    from propainter_b200.inference_propainter import InferenceConfig, ProPainterPipeline
    u8, fm, md = synth.make_clip(T, H, W, mask="ellipse", seed=0)
    fm, md = fm.to(DEV), md.to(DEV)
    pipe = ProPainterPipeline(device=DEV)
    with _pinned():
        comp, st = pipe(torch.from_numpy(u8), fm, md, InferenceConfig(half_storage=True, **kw), return_stages=True)
        ref, rst = _emulate(pipe, torch.from_numpy(u8), fm, md, InferenceConfig(**kw))
    for k in ("gt_flows", "pred_flows"):
        for a, b in zip(st[k], rst[k]):
            assert a.dtype == F16 and a.shape == b.shape and torch.equal(a.float(), b), k
    for k in ("updated_frames", "updated_masks"):
        assert st[k].dtype == F16 and torch.equal(st[k].float(), rst[k]), k
    d = (comp.int() - ref.int()).abs()
    print(f"{T}x{H}x{W}: half storage vs emulation: {int((d > 0).sum())} bytes differ")
    assert torch.equal(comp, ref)


# ---------------------------------------------------------------- precision
def _hole_psnr(a, b, md):
    hole = md[0, :, 0].cpu().numpy() > 0
    return ops_ref.psnr_u8(a[hole], b[hole])


def test_precision_c1_against_fp32():
    from propainter_b200 import synth
    from propainter_b200.inference_propainter import InferenceConfig, ProPainterPipeline
    u8, fm, md = synth.make_clip(8, 128, 128, mask="square", seed=0)
    pipe = ProPainterPipeline(device=DEV)
    a = pipe(torch.from_numpy(u8), fm, md, InferenceConfig(half_storage=True)).cpu().numpy()
    b = pipe(torch.from_numpy(u8), fm, md, InferenceConfig()).cpu().numpy()
    p = _hole_psnr(a, b, md)
    print(f"C1 half storage vs fp32: hole PSNR {p:.2f} dB, max |diff| {np.abs(a.astype(int) - b.astype(int)).max()}")
    assert np.array_equal(a[md[0, :, 0].numpy() == 0], u8[md[0, :, 0].numpy() == 0])
    assert p >= 40.0


def test_precision_c2_against_reference_golden():
    from propainter_b200 import synth
    from propainter_b200.inference_propainter import InferenceConfig, ProPainterPipeline
    g = np.load(os.path.join(GOLD, "c2_80x240x432_ellipse_it20.npz"))
    u8, fm, md = synth.make_clip(80, 240, 432, mask="ellipse", seed=0)
    hole = md[0, :, 0].numpy() > 0
    ref = u8.copy()
    ref[hole] = g["comp_holes"]
    pipe = ProPainterPipeline(device=DEV)
    a = pipe(torch.from_numpy(u8), fm, md, InferenceConfig(half_storage=True)).cpu().numpy()
    b = pipe(torch.from_numpy(u8), fm, md, InferenceConfig()).cpu().numpy()
    ph, pf = ops_ref.psnr_u8(a[hole], ref[hole]), ops_ref.psnr_u8(b[hole], ref[hole])
    print(f"C2 vs reference golden, holes: half storage {ph:.2f} dB, fp32 storage {pf:.2f} dB; "
          f"half vs fp32 {ops_ref.psnr_u8(a[hole], b[hole]):.2f} dB")
    assert ph >= 40.0


# ---------------------------------------------------------------- memory
def _growth(pipe, u8, fm, md, cfg):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    comp = pipe(u8, fm, md, cfg)
    torch.cuda.synchronize()
    grow = torch.cuda.max_memory_allocated() - base
    del comp
    return grow


def test_memory_growth():
    """The clip-resident bytes per frame, as the slope of the peak growth between two clip lengths whose stage workspaces
    are equal (the largest flow-completion sub-video is 50 flows and the largest propagation sub-video 60 frames at both),
    must drop to <= 0.6 of fp32 storage's.  One call's peak also holds those workspaces, which half storage leaves as
    they are: at 160 frames with the default sub-videos they are most of it (measured ratio 0.94), so the test
    compares slopes and only asks one call's peak not to grow."""
    from propainter_b200 import synth
    from propainter_b200.inference_propainter import InferenceConfig, ProPainterPipeline
    u8, fm, md = synth.make_clip(200, 240, 432, mask="ellipse", seed=0)
    u8, fm, md = torch.from_numpy(u8).to(DEV), fm.to(DEV), md.to(DEV)
    pipe = ProPainterPipeline(device=DEV)
    kw = dict(raft_iter=2, raft_clip_frames=12, subvideo_length=40)
    peaks = {}
    with _pinned(graphs=False):
        for T in (120, 200):
            args = (u8[:T].contiguous(), fm[:, :T].contiguous(), md[:, :T].contiguous())
            if T == 120:
                _growth(pipe, *args, InferenceConfig(**kw))                      # lazy weight packing
            peaks[T] = {h: _growth(pipe, *args, InferenceConfig(half_storage=h, **kw)) for h in (False, True)}
            del args
    slope = {h: (peaks[200][h] - peaks[120][h]) / 80 for h in (False, True)}
    px = 240 * 432
    print("240 x 432, peak growth MiB: " + ", ".join(f"{T} frames fp32 {p[False] / 2**20:.0f} half {p[True] / 2**20:.0f} "
                                                     f"(ratio {p[True] / p[False]:.3f})" for T, p in peaks.items()) +
          f"; slope fp32 {slope[False] / px:.1f} B/px/frame, half {slope[True] / px:.1f}, ratio {slope[True] / slope[False]:.3f}")
    assert slope[True] <= 0.6 * slope[False]
    assert all(p[True] <= p[False] for p in peaks.values())


# ---------------------------------------------------------------- surfaces
def test_flows_match_call_stages():
    from propainter_b200 import synth
    from propainter_b200.inference_propainter import InferenceConfig, ProPainterPipeline
    u8, fm, md = synth.make_clip(12, 128, 128, mask="ellipse", seed=1)
    pipe = ProPainterPipeline(device=DEV)
    cfg = InferenceConfig(raft_iter=3, half_storage=True, raft_clip_frames=5, subvideo_length=6)
    with _pinned():
        gt, pred = pipe.flows(torch.from_numpy(u8), fm, cfg)
        _, st = pipe(torch.from_numpy(u8), fm, md, cfg, return_stages=True)
    for a, b in zip(gt + pred, st["gt_flows"] + st["pred_flows"]):
        assert a.dtype == F16 and torch.equal(a, b)


def test_outpaint_and_inpainter_half_storage():
    from propainter_b200 import synth
    from propainter_b200.inference_propainter import InferenceConfig, ProPainterPipeline
    from propainter_b200.inpainter import ProInpainter
    u8, _, _ = synth.make_clip(8, 128, 128, seed=0)
    pipe = ProPainterPipeline(device=DEV)
    a = pipe.outpaint(torch.from_numpy(u8), 1.25, 1.1, InferenceConfig(raft_iter=6, half_storage=True)).cpu().numpy()
    b = pipe.outpaint(torch.from_numpy(u8), 1.25, 1.1, InferenceConfig(raft_iter=6)).cpu().numpy()
    p_out = ops_ref.psnr_u8(a, b)
    inp = ProInpainter(device=DEV)
    _, _, md = synth.make_clip(8, 128, 128, mask="ellipse", seed=0)
    masks = list(md[0, :, 0].numpy().astype(np.uint8))
    ha = np.stack(inp.inpaint(list(u8), masks, raft_iter=4, half_storage=True))
    hb = np.stack(inp.inpaint(list(u8), masks, raft_iter=4))
    p_inp = ops_ref.psnr_u8(ha, hb)
    print(f"outpaint half vs fp32 storage: PSNR {p_out:.2f} dB; ProInpainter.inpaint: PSNR {p_inp:.2f} dB")
    assert a.shape == b.shape and p_out >= 40.0 and p_inp >= 40.0


def test_sharded_runner_rejects_half_storage():
    from propainter_b200.dist import ShardedProPainter
    from propainter_b200.inference_propainter import InferenceConfig
    u8 = torch.zeros(4, 16, 16, 3, dtype=torch.uint8)
    m = torch.zeros(1, 4, 1, 16, 16)
    with pytest.raises(ValueError, match="half_storage"):
        object.__new__(ShardedProPainter)(u8, m, m, InferenceConfig(half_storage=True))
