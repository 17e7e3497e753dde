"""GPU tests of the flow colour coding (k_flow_maxrad / k_flow_to_image_u8) against the reference's own output
(tests/golden/flowviz_c1.npz) and oracle/flowviz_ref.py under the equality criterion of test_flowviz_host.py, and of
the flow-completion evaluation: ProPainterPipeline.flows, evaluate_flow_clip and flow_preview."""
import os

import numpy as np
import pytest
import torch

from oracle import flowviz_ref
from tests.test_flowviz_host import FIXTURE_CASES, fixture_case

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "flowviz_c1.npz")


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


def rel_err(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-12))


def device_image(flows, normalize, clip=None, bgr=False):
    from propainter_b200 import ops
    return ops.flow_to_image_u8(torch.from_numpy(np.ascontiguousarray(flows)).to(DEV), normalize, clip, bgr).cpu().numpy()


@pytest.mark.parametrize("case", FIXTURE_CASES, ids=[c[0] for c in FIXTURE_CASES])
def test_kernels_match_reference_fixture(case):
    g = np.load(GOLD)
    flows, ref, normalize, clip, bgr = fixture_case(g, case)
    got = device_image(flows, normalize, clip, bgr)
    n_ref = flowviz_ref.check_equal(got, flows, normalize, clip, bgr, ref=ref)
    n_oracle = flowviz_ref.check_equal(got, flows, normalize, clip, bgr)
    print(f"{case[0]}: {n_ref} pixels differ from the reference, {n_oracle} from the oracle (all on rounding boundaries)")


def _field(rng, N, H, W, scales):
    f = rng.standard_normal((N, 2, H, W)).astype(np.float32)
    return (f * np.asarray(scales, np.float32)[:, None, None, None]).astype(np.float32)


@pytest.mark.parametrize("N,H,W", [(1, 64, 64), (17, 37, 53), (3, 1, 129), (5, 130, 7)])
@pytest.mark.parametrize("normalize,clip,bgr", [("frame", None, False), ("clip", None, True), ("frame", 2.0, True),
                                                ("clip", 1.5, False)])
def test_kernels_match_oracle_shapes(N, H, W, normalize, clip, bgr):
    """N = 1 and 17, sides that are not multiples of 8, and frames whose maxima differ by up to 300x (per-clip
    normalisation must use the batch maximum, per-frame each frame's own)"""
    rng = np.random.default_rng(N * 1000 + H + W)
    flows = _field(rng, N, H, W, np.geomspace(0.1, 30.0, N) if N > 1 else [4.0])
    got = device_image(flows, normalize, clip, bgr)
    flowviz_ref.check_equal(got, flows, normalize, clip, bgr)
    if N > 1 and clip is None:
        other = flowviz_ref.flow_to_image(flows, "clip" if normalize == "frame" else "frame", None, bgr)
        assert (got != other).any()                     # the two normalisations really differ on these clips


def test_single_frame_input_and_replay():
    from propainter_b200 import ops
    rng = np.random.default_rng(3)
    flows = torch.from_numpy(_field(rng, 4, 40, 56, [1, 5, 0.5, 9])).to(DEV)
    for normalize in ("frame", "clip"):
        a = ops.flow_to_image_u8(flows, normalize)
        b = ops.flow_to_image_u8(flows, normalize)
        assert a.shape == (4, 40, 56, 3) and a.dtype == torch.uint8 and torch.equal(a, b)
        one = ops.flow_to_image_u8(flows[2], normalize)
        assert one.shape == (40, 56, 3)
        assert torch.equal(one, ops.flow_to_image_u8(flows[2:3], normalize)[0])


def test_kernels_4k_frame():
    """one 3840 x 2160 frame: 8.3 M pixels, 25 MB of output"""
    rng = np.random.default_rng(8)
    lo = torch.from_numpy(rng.standard_normal((1, 2, 17, 30)).astype(np.float32) * 40)
    flows = torch.nn.functional.interpolate(lo, size=(2160, 3840), mode="bilinear", align_corners=False).contiguous().numpy()
    for normalize in ("frame", "clip"):
        got = device_image(flows, normalize)
        n = flowviz_ref.check_equal(got, flows, normalize)
        print(f"4K {normalize}: {n} of {2160 * 3840} pixels differ from the oracle (all on rounding boundaries)")


def test_ops_refuse_cpu_fp16_and_wrong_shapes():
    from propainter_b200 import ops
    with pytest.raises(RuntimeError):
        ops.flow_to_image_u8(torch.zeros(2, 2, 8, 8))
    with pytest.raises(ValueError):
        ops.flow_to_image_u8(torch.zeros(2, 2, 8, 8, dtype=torch.float16, device=DEV))
    for shape in ((2, 3, 8, 8), (3, 8, 8), (8, 8), (1, 1, 2, 8, 8)):
        with pytest.raises(ValueError):
            ops.flow_to_image_u8(torch.zeros(shape, device=DEV))
    with pytest.raises(RuntimeError):
        ops.flow_to_image_u8(torch.zeros(0, 2, 8, 8, device=DEV))


def c1_inputs():
    from propainter_b200 import synth
    u8, fm, md = synth.make_clip(8, 128, 128, mask="square", seed=0)
    return u8, fm, md


def test_flows_bitwise_equal_to_call_stages():
    from propainter_b200.inference_propainter import InferenceConfig, ProPainterPipeline
    u8, fm, md = c1_inputs()
    pipe = ProPainterPipeline(device=DEV)
    cfg = InferenceConfig(raft_iter=6)
    _, st = pipe(torch.from_numpy(u8), fm, md, cfg, return_stages=True)
    gt, pred = pipe.flows(torch.from_numpy(u8), fm, cfg)
    for a, b in zip(gt + pred, st["gt_flows"] + st["pred_flows"]):
        assert a.shape == (1, 7, 2, 128, 128) and torch.equal(a, b)


def test_evaluate_flow_clip_matches_reference():
    """C1 with make_golden's weights: the completed flows against the reference's whole-clip flow completion (the bar of
    the flow-completion module test, 1e-2 relative) and the script's EPE numbers to 1e-3 relative"""
    from propainter_b200 import ops
    from propainter_b200.evaluate import evaluate_flow_clip, flow_epe_summary
    from propainter_b200.inference_propainter import InferenceConfig, ProPainterPipeline
    g = np.load(GOLD)
    u8, fm, _ = c1_inputs()
    masks_u8 = (fm[0, :, 0] > 0).to(torch.uint8).numpy()
    dil = ops.mask_dilate(torch.from_numpy(masks_u8 * 255).to(DEV), 4).cpu().numpy().astype(np.uint8)
    assert np.array_equal(dil.ravel(), np.unpackbits(g["masks"])[:dil.size])          # cv2.dilate's masks, exactly
    pipe = ProPainterPipeline(device=DEV)
    res = evaluate_flow_clip(pipe, u8, masks_u8, cfg=InferenceConfig(raft_iter=int(g["raft_iter"])))
    e = [rel_err(res["pred_flows"][i][..., ::4, ::4].cpu().numpy(), g[k]) for i, k in enumerate(("pred_f", "pred_b"))]
    ef, eb = g["epe"]
    print(f"completed flows rel {e[0]:.2e} {e[1]:.2e}; EPE {res['epe_forward']:.6f} {res['epe_backward']:.6f} "
          f"(reference {ef:.6f} {eb:.6f}); stage 2 {res['seconds']:.4f} s")
    assert e[0] < 1e-2 and e[1] < 1e-2
    assert abs(res["epe_forward"] - ef) <= 1e-3 * ef and abs(res["epe_backward"] - eb) <= 1e-3 * eb
    assert res["frames"] == 8 and res["seconds"] > 0 and abs(res["epe"] - (ef + eb) / 2) <= 1e-3 * (ef + eb) / 2
    assert abs(flow_epe_summary([res])["epe"] - res["epe"]) < 1e-12


def test_evaluate_flow_clip_with_reference_flows():
    from propainter_b200.evaluate import evaluate_flow_clip
    from propainter_b200.inference_propainter import InferenceConfig, ProPainterPipeline
    u8, fm, _ = c1_inputs()
    gen = torch.Generator().manual_seed(1)
    ref = tuple(torch.randn(7, 2, 128, 128, generator=gen) * 3 for _ in range(2))
    pipe = ProPainterPipeline(device=DEV)
    res = evaluate_flow_clip(pipe, u8, (fm[0, :, 0] > 0).numpy(), reference_flows=ref, cfg=InferenceConfig(raft_iter=4))
    for r, p, key in zip(ref, res["pred_flows"], ("epe_forward", "epe_backward")):
        d = r.numpy().astype(np.float64)[None] - p.cpu().numpy().astype(np.float64)
        want = np.sqrt((d ** 2).sum(axis=2)).mean()                           # core/metrics.py calculate_epe, float64
        assert abs(res[key] - want) <= 1e-6 * want, (key, res[key], want)


@pytest.mark.shipping
def test_flow_preview_c2():
    from propainter_b200 import ops, synth
    from propainter_b200.inference_propainter import ProPainterPipeline
    u8, fm, _ = synth.make_clip(80, 240, 432, mask="ellipse", seed=0)
    pipe = ProPainterPipeline(device=DEV)
    _, pred = pipe.flows(torch.from_numpy(u8), fm)
    for normalize in ("frame", "clip"):
        vid = pipe.flow_preview(pred[0], normalize)
        assert vid.shape == (79, 240, 432, 3) and vid.dtype == torch.uint8
        assert torch.equal(vid, ops.flow_to_image_u8(pred[0][0], normalize))
    flows = pred[1][0, :3].cpu().numpy()
    flowviz_ref.check_equal(pipe.flow_preview(pred[1], "frame", bgr=True)[:3].cpu().numpy(), flows, "frame", None, True)
