"""GPU tests of scripts/compute_flow.py's port: pp_u8_to_frames_resized bit for bit against the host rule and ATen's CPU
resize, compute_flow_video against the flows the unmodified script wrote (tests/golden/make_golden_compute_flow.py) under
the RAFT bars of test_gpu_modules.py / test_gpu_half_operands.py, and compute_flow_video chained into
evaluate_flow_completion against the unmodified evaluate_flow_completion.py --load_flow run on the script's flows.  The
fixture keeps every 4th pixel of the flows in each direction; the comparisons are made there."""
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.compute_flow_inputs import VIDEOS, video_inputs
from tests.test_compute_flow_host import EXACT_SIZES, aten_frames, gold, hostsim_frames, hs, random_frames  # noqa: F401

pytestmark = pytest.mark.gpu
DEV = "cuda"


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


@pytest.fixture(scope="module")
def pipe():
    from propainter_b200.inference_propainter import ProPainterPipeline
    return ProPainterPipeline(device=DEV)


def size_hw(gold):
    return int(gold["size"][1]), int(gold["size"][0])


@pytest.mark.parametrize("T,H0,W0,h,w", EXACT_SIZES, ids=[f"{c[0]}x{c[1]}x{c[2]}-{c[3]}x{c[4]}" for c in EXACT_SIZES])
def test_kernel_bit_exact(hs, T, H0, W0, h, w):
    from propainter_b200 import ops
    u8 = random_frames(T, H0, W0, H0 * W0 + h)
    got = ops.u8_to_frames_resized(u8.to(DEV), (w, h)).cpu()
    assert torch.equal(got, hostsim_frames(hs, u8, h, w))
    assert torch.equal(got, aten_frames(u8, h, w))
    # the script's own placement: ToTensor on the host, then the resize, *2 and -1 on the device
    img = u8.permute(0, 3, 1, 2).contiguous().float().div(255).to(DEV)
    ref = F.interpolate(img, size=(h, w), mode='bilinear', align_corners=False) * 2 - 1
    n = (got != ref.cpu()).sum().item()
    print(f"{T}x{H0}x{W0} -> {h}x{w}: {n} of {got.numel()} values differ from ATen's CUDA resize "
          f"(max {(got - ref.cpu()).abs().max().item():.2e})")


def test_kernel_small_outputs_and_identity(hs):
    from propainter_b200 import ops
    for T, H0, W0, h, w in [(2, 101, 77, 24, 40), (2, 5, 3, 17, 19), (1, 1, 1, 7, 9)]:
        u8 = random_frames(T, H0, W0, w)
        assert torch.equal(ops.u8_to_frames_resized(u8.to(DEV), (w, h)).cpu(), hostsim_frames(hs, u8, h, w))
    u8 = random_frames(3, 37, 53, 1).to(DEV)
    assert torch.equal(ops.u8_to_frames_resized(u8, (53, 37)), ops.u8_to_frames(u8))


def test_kernel_refuses_cpu_and_bad_shapes():
    from propainter_b200 import ops
    with pytest.raises(RuntimeError):
        ops.u8_to_frames_resized(torch.zeros(2, 8, 8, 3, dtype=torch.uint8), (16, 16))
    u8 = torch.zeros(2, 8, 8, 3, dtype=torch.uint8, device=DEV)
    for bad, size in ((u8.float(), (16, 16)), (u8[..., :1], (16, 16)), (u8[0], (16, 16)), (u8, (0, 16)), (u8, (16, -1))):
        with pytest.raises(ValueError):
            ops.u8_to_frames_resized(bad, size)
    with pytest.raises(RuntimeError):
        ops.u8_to_frames_resized(u8[:, ::2], (16, 16))                       # not contiguous


def flow_errors(got, ref):
    rel = float(np.abs(got - ref).max() / np.abs(ref).max())
    epe = float(np.sqrt(((got.astype(np.float64) - ref) ** 2).sum(1)).mean())
    return rel, epe


def check_script_flows(pipe, gold, bar):
    from propainter_b200.evaluate import compute_flow_video
    h, w = size_hw(gold)
    out = {}
    for name, T, mask, seed, native in VIDEOS:
        u8, _ = video_inputs(T, mask, seed, native)
        fw, bw = compute_flow_video(pipe, u8, (w, h), int(gold["raft_iter"]))
        assert fw.dtype == torch.float16 and fw.shape == (T - 1, 2, h, w) and bw.shape == fw.shape
        for got, key in ((fw, "flow_f"), (bw, "flow_b")):
            ref = gold[f"{name}_{key}_sub4"].astype(np.float32)
            rel, epe = flow_errors(got[..., ::4, ::4].float().cpu().numpy(), ref)
            print(f"{name} {key}: rel {rel:.2e} EPE {epe:.4f} px")
            assert rel <= bar and epe <= 0.05, (name, key, rel, epe)
        out[name] = (fw, bw)
    return out


def test_compute_flow_video_matches_script(pipe, gold):
    """fp32 library math: RAFT's bar of test_gpu_modules.py, 2e-3 of the flow scale and <= 0.05 px EPE"""
    check_script_flows(pipe, gold, 2e-3)


@pytest.mark.shipping
def test_compute_flow_video_matches_script_shipping(pipe, gold):
    """the shipping precision (TF32 library convs, fp16-operand refinement): the half-operand bar, 5e-3 and 0.05 px"""
    check_script_flows(pipe, gold, 5e-3)


def test_compute_flow_video_repeats(pipe, gold):
    from propainter_b200.evaluate import compute_flow_video
    name, T, mask, seed, native = VIDEOS[0]
    u8, _ = video_inputs(T, mask, seed, native)
    h, w = size_hw(gold)
    a = compute_flow_video(pipe, torch.from_numpy(u8), (w, h), 4)
    b = compute_flow_video(pipe, torch.from_numpy(u8).to(DEV), (w, h), 4)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_compute_flow_then_flow_completion(pipe, gold):
    """the script chain: compute_flow_video's fp16 flows loaded by evaluate_flow_completion, against the unmodified
    evaluate_flow_completion.py --load_flow run on the .flo files compute_flow.py wrote.  The completed flows within 1e-2
    of their scale (the flow-completion bar of test_gpu_modules.py) on the fixture's every-4th-pixel subsample; each
    per-video EPE within what the two bars imply (an EPE moves by at most max |pred - pred_ref| + max |flow - flow_ref|,
    i.e. 1e-2 of the completed-flow scale + 2e-3 of the flow scale); the records equal evaluate_flow_video's on the same
    prepared inputs; the script's text up to its numbers."""
    from propainter_b200.evaluate import evaluate_flow_completion, evaluate_flow_video, prepare_test_video
    flows = check_script_flows(pipe, gold, 2e-3)
    size = (int(gold["size"][0]), int(gold["size"][1]))
    videos = []
    for name, T, mask, seed, native in VIDEOS:
        _, mk = video_inputs(T, mask, seed, native)
        videos.append((name, mk, flows[name]))
    lines = []
    res = evaluate_flow_completion(pipe, videos, size, log=lines.append)
    ref_lines = str(gold["summary"]).strip().split("\n")
    assert lines == [r["line"] for r in res["videos"]] + [res["line"]] and len(lines) == len(ref_lines)
    pattern = re.compile(r"\[ *\d+/\d+\] Name: .{25} \| EPE: \d+\.\d{4} \| Time: \d+\.\d{4}$")
    for i, (r, (name, T, mask, seed, native)) in enumerate(zip(res["videos"], VIDEOS)):
        assert pattern.match(r["line"]) and r["line"].split(" | EPE")[0] == ref_lines[i].split(" | EPE")[0]
        _, mk, fl = prepare_test_video(None, videos[i][1], size, flows[name], DEV)
        one = evaluate_flow_video(pipe, mk, fl)
        assert (one["epe_forward"], one["epe_backward"]) == (r["epe_forward"], r["epe_backward"])
        bound = 0.0
        for d, p in zip("fb", one["pred_flows"]):
            ref_pred = gold[f"{name}_pred_{d}_sub4"].astype(np.float32)
            got = p[0, ..., ::4, ::4].cpu().numpy()
            e = float(np.abs(got - ref_pred).max() / np.abs(ref_pred).max())
            scale_flow = float(np.abs(gold[f"{name}_flow_{d}_sub4"].astype(np.float32)).max())
            bound = max(bound, 1e-2 * float(np.abs(ref_pred).max()) + 2e-3 * scale_flow)
            print(f"{name} completed {d}: rel {e:.2e}")
            assert e < 1e-2, (name, d, e)
        ref_epe = gold[f"{name}_epe"]
        print(f"{name}: EPE {r['epe_forward']:.5f} {r['epe_backward']:.5f} (script {ref_epe[0]:.5f} {ref_epe[1]:.5f}, "
              f"bound {bound:.3f})")
        assert abs(r["epe_forward"] - ref_epe[0]) <= bound and abs(r["epe_backward"] - ref_epe[1]) <= bound
    assert res["line"].startswith("Finish evaluation... Average Frame EPE: ") and " | | Time: " in res["line"]
    assert res["summary"]["videos"] == len(VIDEOS)
    with pytest.raises(ValueError):
        evaluate_flow_completion(pipe, [("bear", np.zeros((8, 200, 240), np.uint8), None)])
