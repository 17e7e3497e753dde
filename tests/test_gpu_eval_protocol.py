"""GPU tests of the evaluation script's video-completion protocol: pp_composite_blend_f32 and pp_resize_flow_linear_cv bit
for bit against the script's numpy compositing and cv2.resize + rescale (through the oracle's emulation, which
test_eval_protocol_host.py pins to cv2), prepare_test_video against the script's own TestDataset outputs, and
evaluate_video against the fixture made by the unmodified scripts/evaluate_propainter.py::main_worker
(tests/golden/make_golden_eval_protocol.py) with the same seeded weights."""
import os

import numpy as np
import pytest
import torch

from oracle import eval_protocol_ref as epr
from tests.eval_protocol_inputs import digest, video_inputs
from tests.test_eval_protocol_host import RESIZE_CASES, script_blend

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "eval_protocol_2v_128x224.npz")


@pytest.fixture(autouse=True)
def _exact_library_math():
    """fp32 library convs / GEMMs, as the fixture's CPU run"""
    from propainter_b200 import config
    a, b, c = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32, config.LINEAR_TF32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    config.LINEAR_TF32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32, config.LINEAR_TF32 = a, b, c


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLD))


def test_composite_blend_f32_bit_exact():
    from propainter_b200 import ops
    rng = np.random.default_rng(5)
    T, H, W = 9, 40, 56
    ori = rng.integers(0, 256, (T, H, W, 3), dtype=np.uint8)
    masks = (rng.random((T, 1, H, W)) < 0.5).astype(np.float32)
    masks[0], masks[1] = 0, 1
    visits = [(0, [0, 1, 2, 3, 4]), (1, [2, 3, 4, 5, 6, 7]), (2, [4, 5, 6, 7, 8]), (3, [7, 8])]
    preds = {}
    for w, nb in visits:
        p = rng.uniform(-1, 1, (len(nb), 3, H, W)).astype(np.float32)
        edge = (rng.integers(0, 256, p.shape) / 255.0 * 2 - 1).astype(np.float32)
        sel = rng.random(p.shape) < 0.5
        p[sel] = np.nextafter(edge, rng.choice([-2, 2], p.shape).astype(np.float32))[sel]
        preds[w] = p
    ref = script_blend(preds, masks, ori, visits)
    comp = torch.zeros(T, H, W, 3, device=DEV)
    seen = [False] * T
    m, o = torch.from_numpy(masks).to(DEV), torch.from_numpy(ori).to(DEV)
    for w, nb in visits:
        ops.composite_blend_f32(torch.from_numpy(preds[w]).to(DEV), m, o, comp, nb, [not seen[i] for i in nb])
        for i in nb:
            seen[i] = True
    got = comp.cpu().numpy()
    for t in range(T):
        assert np.array_equal(got[t], ref[t].astype(np.float32)), t
    assert (got * 4 % 2 == 1).any()


@pytest.mark.parametrize("src,size", RESIZE_CASES, ids=[f"{s[0]}x{s[1]}-{d[1]}x{d[0]}" for s, d in RESIZE_CASES])
def test_resize_flow_bit_exact(src, size):
    from propainter_b200 import ops
    H, W = src
    f = (np.random.default_rng(H * W).standard_normal((3, 2, H, W)) * 20).astype(np.float32)
    got = ops.resize_flow(torch.from_numpy(f).to(DEV), size).cpu().numpy()
    assert np.array_equal(got, epr.resize_flow(f, size))
    try:
        import cv2
    except ImportError:
        return
    for n in range(len(f)):
        r = cv2.resize(np.ascontiguousarray(f[n].transpose(1, 2, 0)), size, interpolation=cv2.INTER_LINEAR)
        r[:, :, 0] *= size[0] / W
        r[:, :, 1] *= size[1] / H
        assert np.array_equal(got[n], r.transpose(2, 0, 1))


def test_prepare_test_video_matches_dataset(gold):
    from propainter_b200.evaluate import prepare_test_video
    size = tuple(int(s) for s in gold["size"])
    for vi, name in enumerate(gold["names"]):
        fr, mk, fl = video_inputs(int(gold["lengths"][vi]), str(gold["masks_kind"][vi]), int(gold["seeds"][vi]))
        f, m, flows = prepare_test_video(fr, mk, size, fl)
        assert f.dtype == torch.uint8 and m.shape == (1, len(fr), 1, size[1], size[0])
        assert digest(f.cpu().numpy()) == str(gold[f"{name}_sha_frames"])
        assert digest(m.cpu().numpy()) == str(gold[f"{name}_sha_masks"])
        assert digest(np.stack([x.cpu().numpy() for x in flows])) == str(gold[f"{name}_sha_flows"])


def psnr_holes(a, b, hole):
    d = (a[hole].astype(np.float64) - b[hole].astype(np.float64)) ** 2
    return 20 * np.log10(255.0 / np.sqrt(d.mean()))


def test_evaluate_propainter_against_script(gold):
    """The script's run of the fixture's two videos (24 and 17 frames, 144x240 evaluated at 224x128, loaded flows) against
    evaluate_propainter with the same seeded weights.  The composited video inside the holes: >= 60 dB against the
    script's (measured on an H100 80GB HBM3: 72.95 dB for bear, 71.43 dB for swing), well above the 40 dB the
    full-pipeline golden tests hold at this clip size.  Outside the holes it is the input, bit for bit.  Per-frame PSNR /
    SSIM follow from that: both are taken over the whole frame, of which the holes are a part, so a >= 60 dB hole
    difference moves a ~20 dB frame PSNR by under 0.005 dB and SSIM by under 1e-4 (measured: 0.0005 dB, 2.1e-5); the final
    line's PSNR / SSIM agree to their printed digits, VFID within 2 % (measured: equal to its 3 printed digits)."""
    from propainter_b200.evaluate import evaluate_propainter, evaluate_video, prepare_test_video
    from propainter_b200.inference_propainter import ProPainterPipeline
    from propainter_b200.model.i3d import InceptionI3d
    pipe = ProPainterPipeline(device=DEV)
    i3d = InceptionI3d(400, in_channels=3, final_endpoint='Logits', seed=int(gold["i3d_seed"])).to(DEV).eval()
    size = tuple(int(s) for s in gold["size"])
    videos = []
    for vi, name in enumerate(gold["names"]):
        fr, mk, fl = video_inputs(int(gold["lengths"][vi]), str(gold["masks_kind"][vi]), int(gold["seeds"][vi]))
        videos.append((str(name), fr, mk, fl))
        f, m, flows = prepare_test_video(fr, mk, size, fl)
        r = evaluate_video(pipe, f, m, flows, i3d=i3d)
        comp = r["comp"].cpu().numpy().astype(np.float64)
        hole = m[0, :, 0].cpu().numpy() > 0
        ref = f.cpu().numpy().astype(np.float64)
        assert np.array_equal(comp[~hole], ref[~hole])
        ref[hole] = gold[f"{name}_comp4_holes"] / 4.0
        p = psnr_holes(comp, ref, hole)
        dp = np.abs(np.array(r["psnr_per_frame"]) - gold[f"{name}_psnr"]).max()
        ds = np.abs(np.array(r["ssim_per_frame"]) - gold[f"{name}_ssim"]).max()
        print(f"{name}: PSNR in the holes vs the script {p:.2f} dB; per-frame |dPSNR| max {dp:.4f} dB, |dSSIM| max {ds:.2e}")
        assert p >= 60.0, p
        assert dp < 0.005 and ds < 1e-4
        frac = comp[hole] % 1
        assert (frac != 0).any() and set(np.unique(frac * 4)) <= {0.0, 1.0, 2.0, 3.0}   # blended, untruncated
        assert r["i3d"][0].shape == (1024,)
    res = evaluate_propainter(pipe, videos, size=size, i3d=i3d)
    s = res["summary"]
    ref_line = str(gold["summary"]).strip().split("\n")[-1]
    ref_psnr, ref_ssim, ref_vfid = (float(x) for x in ref_line.split("VFID: ")[1].split(" |")[0].split("/"))
    print(res["line"], "| script:", ref_line)
    assert abs(s["psnr"] - ref_psnr) <= 0.005 + 0.005 and abs(s["ssim"] - ref_ssim) <= 5e-5 + 1e-4
    assert abs(s["vfid"] - ref_vfid) <= 0.02 * ref_vfid + 5e-4
    assert [r["name"] for r in res["videos"]] == list(gold["names"]) and res["line"].startswith("Finish evaluation...")


def test_evaluate_video_raft_chunks_match_compute_flows():
    """flows=None runs RAFT in the script's 60-frame chunks (one-frame overlap): the flows evaluate_video computes are
    those of pipe.compute_flows(..., raft_clip_frames=60), bit for bit, over a clip that crosses the chunk boundary, and
    the video from them matches the one from those flows fed in as loaded flows up to the run-to-run spread of stages
    3-4.  That spread: two runs on identical inputs differ in a few values by up to one level (measured on an H100: 9-18
    of the 3.2 M values of this clip, eager and graphed alike), while RAFT and flow completion repeat bit for bit."""
    from propainter_b200 import config, ops, synth
    from propainter_b200.evaluate import evaluate_video
    from propainter_b200.inference_propainter import InferenceConfig, ProPainterPipeline
    prev = (config.AUTOTUNE, config.CUDNN_BENCHMARK, config.UMMA_CONV)
    config.AUTOTUNE, config.CUDNN_BENCHMARK, config.UMMA_CONV = False, False, True
    try:
        pipe = ProPainterPipeline(device=DEV)
        u8, fm, _ = synth.make_clip(66, 128, 128, mask="ellipse", seed=3)
        fr = torch.from_numpy(u8).to(DEV)
        mk = ops.mask_dilate((fm[0, :, 0] > 0).to(torch.uint8).to(DEV), 4).unsqueeze(0)
        seen = []
        compute = pipe.compute_flows
        pipe.compute_flows = lambda frames, cfg: seen.append((cfg.raft_clip_frames, compute(frames, cfg))) or seen[-1][1]
        a = evaluate_video(pipe, fr, mk, None, raft_iter=2)
        del pipe.compute_flows
        flows = pipe.compute_flows(ops.u8_to_frames(fr).unsqueeze(0), InferenceConfig(raft_iter=2, raft_clip_frames=60))
        b = evaluate_video(pipe, fr, mk, (flows[0][0], flows[1][0]), raft_iter=2)
    finally:
        config.AUTOTUNE, config.CUDNN_BENCHMARK, config.UMMA_CONV = prev
    assert len(seen) == 1 and seen[0][0] == 60
    assert torch.equal(seen[0][1][0], flows[0]) and torch.equal(seen[0][1][1], flows[1])
    diff = (a["comp"] - b["comp"]).abs()
    assert diff.max().item() <= 1.0 and (diff > 0).sum().item() <= 100
