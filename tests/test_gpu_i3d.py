"""GPU tests of the I3D feature network behind VFID: the three new kernels bit-exact (input packing, max pooling) or
float64-accurate (mean) against the reference's own torch ops, extract_features against the fp32 oracle at every
endpoint and against the reference fixture, a C2-sized batch, and the VFID path through evaluate_clip."""
import functools
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import i3d_ref
from tests.test_i3d_host import FIXTURE, POOLS, fixture_clip, seeded_state_dict, subsample

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(autouse=True)
def _exact_library_math(request):
    """fp32 library convs, except for tests marked `shipping` (the default precision switches)"""
    if "shipping" in request.keywords:
        yield
        return
    a = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = a


def scale_err(a, b):
    """max |a - b| over the output scale max |b|"""
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def bits_equal(a, b):
    """bitwise equality, NaNs compared by position"""
    a, b = a.cpu(), b.cpu()
    return torch.equal(a.isnan(), b.isnan()) and torch.equal(torch.nan_to_num(a).view(torch.int32), torch.nan_to_num(b).view(torch.int32))


@functools.lru_cache(maxsize=None)
def model(seed):
    from propainter_b200.model.i3d import InceptionI3d
    net = InceptionI3d(400, in_channels=3, final_endpoint='Logits')
    net.load_state_dict(seeded_state_dict(seed), strict=True)
    return net.to(DEV)


def padded_ref(x_ncdhw):
    """F.pad of Conv3d_1a_7x7 on an NCDHW video, then pixel-major with the zero 4th channel"""
    x = i3d_ref.same_pad(x_ncdhw, (7, 7, 7), (2, 2, 2)).permute(0, 2, 3, 4, 1)
    return torch.cat([x, torch.zeros_like(x[..., :1])], -1).contiguous()


@pytest.mark.parametrize("B,T,H,W", [(1, 9, 72, 100), (2, 16, 64, 64), (2, 5, 7, 12), (1, 1, 1, 1)])
def test_i3d_input_bit_exact(B, T, H, W):
    from propainter_b200 import ops
    rng = np.random.default_rng(T * H * W)
    u8 = torch.from_numpy(rng.integers(0, 256, (B, T, H, W, 3), dtype=np.uint8))
    ref = padded_ref(u8.permute(0, 4, 1, 2, 3).float().div(255))       # to_tensors on the host, as the reference runs it
    got = ops.i3d_input(u8.to(DEV))
    assert got.shape == ref.shape and bits_equal(got, ref)
    x = torch.randn(B, 3, T, H, W, generator=torch.Generator().manual_seed(B + T))
    got = ops.i3d_input(x.to(DEV))
    assert bits_equal(got, padded_ref(x))


@pytest.mark.parametrize("kernel,stride", POOLS)
@pytest.mark.parametrize("B,T,H,W,C", [(2, 5, 9, 13, 16), (1, 4, 8, 6, 8), (1, 3, 5, 7, 64), (2, 2, 2, 2, 4)])
def test_maxpool3d_same_bit_exact_into_channel_slice(kernel, stride, B, T, H, W, C):
    from propainter_b200 import ops
    gen = torch.Generator().manual_seed(B * 1000 + T * 100 + H * 10 + W)
    x = torch.randn(B, C, T, H, W, generator=gen) - 0.5                  # mostly negative: padded zeros win often
    x.view(-1)[3::11] = -0.0
    x.view(-1)[::37] = float("nan")
    x = x.to(DEV)
    ref = F.max_pool3d(i3d_ref.same_pad(x, kernel, stride), kernel, stride)           # the reference's own ops
    pm = x.permute(0, 2, 3, 4, 1).contiguous()
    buf = torch.full((B,) + tuple(ref.shape[2:]) + (C + 8,), 123.0, device=DEV)
    ops.maxpool3d_same(pm, kernel, stride, out=buf[..., 4:4 + C])
    got = buf[..., 4:4 + C].permute(0, 4, 1, 2, 3)
    assert bits_equal(got, ref)
    assert torch.isnan(got).any()
    assert (buf[..., :4] == 123.0).all() and (buf[..., 4 + C:] == 123.0).all()


@pytest.mark.parametrize("B,T,H,W,C", [(2, 10, 8, 14, 1024), (1, 3, 5, 7, 832), (3, 1, 1, 1, 40)])
def test_mean_thw_matches_float64(B, T, H, W, C):
    from propainter_b200 import ops
    x = (torch.rand(B, T, H, W, C, generator=torch.Generator().manual_seed(C)) * 4).to(DEV)
    got = ops.mean_thw(x)
    ref = x.double().mean((1, 2, 3))
    assert got.shape == (B, C) and got.dtype == torch.float32
    assert float(((got.double() - ref).abs() / ref.abs()).max()) < 1e-6
    assert torch.equal(ops.mean_thw(x), got)                           # fixed-order reduction: same bits every run


def _oracle_maps(sd_dev, x):
    """the fp32 oracle's features and every endpoint map (library convs in fp32 whatever the switches)"""
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        return i3d_ref.extract_features(sd_dev, x, return_maps=True)
    finally:
        torch.backends.cudnn.allow_tf32 = prev


def _check_against_oracle(tol):
    g = np.load(FIXTURE)
    seed = int(g["seed"])
    net = model(seed)
    sd = {k: v.to(DEV) for k, v in seeded_state_dict(seed).items()}
    for tag in g["clips"]:
        x = i3d_ref.video_from_u8(fixture_clip(g, tag)).to(DEV)
        feats, maps = _oracle_maps(sd, x)
        errs = {}
        for name in i3d_ref.ENDPOINTS:
            got = net.extract_features(x, name)
            assert got.shape == maps[name].shape, name
            errs[name] = scale_err(got, maps[name])
        got = net.extract_features(x)
        errs["Logits"] = scale_err(got, feats)
        errs["fixture"] = scale_err(got, g[f"{tag}_features"])
        for name, steps in zip(g["maps"], g["steps"]):
            errs[f"fixture {name}"] = scale_err(subsample(net.extract_features(x, str(name)), steps), g[f"{tag}_{name}"])
        # the uint8 entry point (conversion fused into the input kernel) gives the same features
        errs["u8"] = scale_err(net.features_u8(torch.from_numpy(fixture_clip(g, tag))[None].to(DEV)), feats)
        print(f"{tag}: " + ", ".join(f"{k} {v:.2e}" for k, v in errs.items()))
        bad = {k: v for k, v in errs.items() if not v <= tol}
        assert not bad, (tag, bad)


def test_extract_features_matches_oracle_fp32():
    _check_against_oracle(1e-4)


@pytest.mark.shipping
def test_extract_features_matches_oracle_tf32():
    assert torch.backends.cudnn.allow_tf32
    _check_against_oracle(1e-2)


def test_predictions_and_unknown_endpoints_return_mixed_5c():
    """the reference's loop never breaks for a name it has not built: the whole network runs, the map is returned"""
    net = model(3)
    x = torch.rand(1, 3, 8, 64, 64, generator=torch.Generator().manual_seed(0)).to(DEV)
    m = net.extract_features(x, 'Mixed_5c')
    assert m.shape == (1, 1024, 1, 2, 2)                                # T 8 -> 4 -> 2 -> 1, H, W 64 -> ... -> 2
    assert torch.equal(net.extract_features(x, 'Predictions'), m)
    assert torch.equal(net.extract_features(x.transpose(1, 2).contiguous().transpose(1, 2)), net.extract_features(x))
    with pytest.raises(RuntimeError):
        net.extract_features(x.double())


def test_c2_batch_of_two():
    from propainter_b200 import synth
    from propainter_b200.evaluate import i3d_activations
    net = model(5)
    real, _, _ = synth.make_clip(80, 240, 432, mask="ellipse", seed=0)
    fake, _, _ = synth.make_clip(80, 240, 432, mask="ellipse", seed=1)
    both = torch.from_numpy(np.stack([real, fake])).to(DEV)
    a = i3d_activations(net, both)
    assert a.shape == (2, 1024) and a.dtype == np.float32 and np.isfinite(a).all()
    b = i3d_activations(net, both)
    assert np.array_equal(a, b), "replay differs"
    single = np.stack([i3d_activations(net, real), i3d_activations(net, fake)])
    err = scale_err(a, single)
    print(f"B=2 vs 2 x B=1: {err:.2e} of the output scale" + (" (bit-identical)" if np.array_equal(a, single) else ""))
    assert err <= 1e-5


def test_evaluate_clip_vfid():
    from propainter_b200 import synth
    from propainter_b200.evaluate import evaluate_clip, fid_from_activations, i3d_activations, video_completion_summary
    from propainter_b200.inference_propainter import InferenceConfig, ProPainterPipeline
    net = model(5)
    pipe = ProPainterPipeline(device=DEV)
    results = []
    for seed in range(3):
        u8, fm, _ = synth.make_clip(10, 128, 128, mask="ellipse", seed=seed)
        res = evaluate_clip(pipe, u8, (fm[0, :, 0] > 0).numpy(), cfg=InferenceConfig(raft_iter=4),
                            i3d_activations=functools.partial(i3d_activations, net))
        real, fake = res["i3d"]
        assert real.shape == fake.shape == (1024,) and real.dtype == fake.dtype == np.float32
        assert np.isfinite(real).all() and np.isfinite(fake).all() and not np.array_equal(real, fake)
        results.append(res)
    s = video_completion_summary(results)
    print("summary:", {k: v for k, v in s.items()})
    assert np.isfinite(s["vfid"]) and s["videos"] == 3
    real = np.stack([r["i3d"][0] for r in results])
    cov = np.cov(real, rowvar=False)
    self_fid = fid_from_activations(real, real)
    print(f"VFID of a set against itself: {self_fid:.3e} (trace sum {2 * np.trace(cov):.3e})")
    assert abs(self_fid) <= 1e-5 * 2 * np.trace(cov)
