"""GPU tests of the temporal warping error (k_flow_occlusion / k_warp_error) against oracle/ewarp_ref.py under the
criteria of test_warp_error_host.py: occlusion maps equal outside the float64 margin, E_t within 1e-5 relative of the
oracle evaluated on the kernel's own map, the same bits on every run; and evaluate_video(..., warp_error=True) on the
evaluation-protocol fixture."""
import os

import numpy as np
import pytest
import torch

from oracle import ewarp_ref
from tests.test_warp_error_host import FLOW_KINDS, check_occlusion, check_warp_error, flow_case, texture, translation_clip

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "eval_protocol_2v_128x224.npz")


@pytest.fixture(autouse=True)
def _exact_library_math():
    """fp32 library convs / GEMMs, as test_gpu_eval_protocol.py runs the protocol"""
    from propainter_b200 import config
    a, b, c = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32, config.LINEAR_TF32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    config.LINEAR_TF32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32, config.LINEAR_TF32 = a, b, c


def dev(*arrays):
    return [torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a in arrays]


def check_clip(frames, fw, bw, label):
    """the kernels on one clip against the oracle; -> (E_t, occlusion map)"""
    from propainter_b200 import ops
    fr, f, b = dev(frames, fw, bw)
    occ = ops.flow_occlusion(f, b)
    n = check_occlusion(occ.cpu().numpy(), fw, bw)
    e = ops.warp_error(fr, f, occ=occ)
    ref = ewarp_ref.warp_error(frames, fw, occ=occ.cpu().numpy())
    check_warp_error(e.cpu().numpy(), ref)
    fused = ops.warp_error_sums(fr, f, bw=b)                     # the map computed in the same pass: the same bits
    assert torch.equal(fused, ops.warp_error_sums(fr, f, occ=occ))
    print(f"{label}: {int(occ.sum())} of {occ.numel()} occluded, {n} inside the margin; E_t {e.cpu().numpy()}")
    return e, occ


@pytest.mark.parametrize("kind", FLOW_KINDS)
@pytest.mark.parametrize("T,H,W", [(4, 37, 53), (3, 128, 224), (2, 1, 67), (3, 61, 1)])
def test_kernels_match_oracle(kind, T, H, W):
    """smooth fields, displacements far off the frame and integer displacements (a = b = 0); sides that are not
    multiples of the block size, single rows and columns"""
    fw, bw = flow_case(kind, T - 1, H, W, seed=100 * T + H + W + FLOW_KINDS.index(kind))
    check_clip(texture(T, H, W, seed=H * W), fw, bw, f"{kind} {T}x{H}x{W}")


def test_repeat_calls_are_bit_identical():
    from propainter_b200 import ops
    fw, bw = flow_case("smooth", 9, 240, 432, seed=3)
    fr, f, b = dev(texture(10, 240, 432, seed=4), fw, bw)
    runs = [ops.warp_error_sums(fr, f, bw=b) for _ in range(3)] + [ops.warp_error_sums(fr, f, occ=ops.flow_occlusion(f, b))]
    assert all(torch.equal(runs[0], r) for r in runs[1:])
    assert torch.equal(ops.flow_occlusion(f, b), ops.flow_occlusion(f, b))


def test_translation_clip():
    """integer translations of one texture with their exact flows: nothing occluded, zero error wherever the warp stays
    inside the frame, and the total equals the oracle"""
    from propainter_b200 import ops
    shifts = [(3, 0), (0, -2), (-4, 5), (1, 1), (-2, -3)]
    frames, fw, bw = translation_clip(6, 96, 160, shifts, seed=9)
    e, occ = check_clip(frames, fw, bw, "translation")
    assert not occ.any()
    interior = torch.ones_like(occ)
    interior[:, 8:-8, 8:-8] = 0                                 # occluded = everything but the interior
    fr, f = dev(frames, fw)
    s = ops.warp_error_sums(fr, f, occ=interior).cpu().numpy()
    assert (s[:, 0] == 0).all() and (s[:, 1] == 80 * 144).all()
    assert (e.cpu().numpy() > 0).all()                           # the clamped border does differ
    assert abs(e.mean().item() - ewarp_ref.ewarp(frames, fw, bw)) <= 1e-5 * e.mean().item()


def test_fp16_and_batched_flows():
    """fp16 flows (the .flo content) equal their .float(); [1,N,2,H,W] equals [N,2,H,W]"""
    from propainter_b200 import ops
    fw, bw = flow_case("smooth", 5, 64, 96, seed=11)
    fr, f, b = dev(texture(6, 64, 96, seed=12), fw, bw)
    f16, b16 = f.half(), b.half()
    occ = ops.flow_occlusion(f16, b16)
    assert torch.equal(occ, ops.flow_occlusion(f16.float(), b16.float()))
    assert torch.equal(occ, ops.flow_occlusion(f16[None], b16[None]))
    e = ops.warp_error_sums(fr, f16, bw=b16)
    assert torch.equal(e, ops.warp_error_sums(fr, f16.float(), bw=b16.float()))
    assert torch.equal(e, ops.warp_error_sums(fr, f16[None], bw=b16[None]))
    assert torch.equal(ops.warp_error(fr, f, bw=b), ops.warp_error(fr, f[None], occ=ops.flow_occlusion(f[None], b[None])))


def test_full_hd_clip():
    """4 frames of 1920 x 1080, the size of profiles/warp_error_time.py's second clip"""
    fw, bw = flow_case("smooth", 3, 1080, 1920, seed=13)
    fw, bw = fw * 8, bw * 8
    e, occ = check_clip(texture(4, 1080, 1920, seed=14), fw, bw, "1920x1080")
    assert 0 < occ.float().mean().item() < 0.9


def test_evaluate_video_warp_error_on_protocol_fixture():
    """one video of the eval-protocol fixture prepared at (224, 128) with its loaded flows: the warping-error keys equal
    the oracle on the returned comp truncated to uint8 and those flows; the existing keys are all there, PSNR / SSIM
    within test_gpu_eval_protocol.py's tolerances of the script's.  The synthetic flows are independent noise fields,
    so most pixels are occluded: this checks the plumbing (test_translation_clip checks the non-occluded path)."""
    from propainter_b200 import ops
    from propainter_b200.evaluate import evaluate_video, prepare_test_video, warp_error
    from propainter_b200.inference_propainter import ProPainterPipeline
    from tests.eval_protocol_inputs import video_inputs
    gold = dict(np.load(GOLD))
    size = tuple(int(s) for s in gold["size"])
    name = str(gold["names"][0])
    fr, mk, fl = video_inputs(int(gold["lengths"][0]), str(gold["masks_kind"][0]), int(gold["seeds"][0]))
    f, m, flows = prepare_test_video(fr, mk, size, fl)
    pipe = ProPainterPipeline(device=DEV)
    r = evaluate_video(pipe, f, m, flows, warp_error=True)
    for key in ("frames", "seconds", "seconds_per_frame", "comp", "psnr_per_frame", "ssim_per_frame", "psnr", "ssim"):
        assert key in r, key
    dp = np.abs(np.array(r["psnr_per_frame"]) - gold[f"{name}_psnr"]).max()
    ds = np.abs(np.array(r["ssim_per_frame"]) - gold[f"{name}_ssim"]).max()
    assert dp < 0.005 and ds < 1e-4, (dp, ds)
    comp = r["comp"].to(torch.uint8)
    fw, bw = (x.cpu().numpy() for x in flows)
    occ = ops.flow_occlusion(*flows).cpu().numpy()
    n = check_occlusion(occ, fw, bw)
    ref = ewarp_ref.warp_error(comp.cpu().numpy(), fw, occ=occ)
    check_warp_error(r["ewarp_per_pair"], ref)
    assert len(r["ewarp_per_pair"]) == len(f) - 1
    assert abs(r["ewarp"] - ref.mean()) <= 1e-5 * ref.mean() + 1e-9
    assert abs(r["occluded_fraction"] - occ.mean()) < 1e-12
    assert warp_error(comp, flows) == {k: r[k] for k in ("ewarp", "ewarp_per_pair", "occluded_fraction")}
    print(f"{name}: E_warp {r['ewarp']:.6f} (oracle {ref.mean():.6f}), occluded {r['occluded_fraction']:.3f}, "
          f"{n} pixels inside the margin; |dPSNR| {dp:.4f} dB, |dSSIM| {ds:.2e}")
