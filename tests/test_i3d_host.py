"""CPU tests of the I3D feature network behind VFID: the oracle against the reference fixture
(tests/golden/make_golden_i3d.py), the state_dict schema against the reference manifest, the drop-in's constructor and
loading rules, video_completion_summary against a direct restatement of the evaluate script's accumulation, and the host
build of the 'same'-padding and max-pooling rules against the oracle and ATen.  The kernels and the network run on the
GPU in test_gpu_i3d.py."""
import ctypes
import json
import os
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import i3d_ref
from propainter_b200 import schemas
from propainter_b200._params import ParamNet

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
FIXTURE = os.path.join(GOLD, "i3d_clips.npz")
FP = ctypes.POINTER(ctypes.c_float)


def rel_err(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(np.asarray(b)).max(), 1e-12))


def seeded_state_dict(seed):
    """the fixture's weights: the schema's seeded init (Kaiming-normal convs, randomised BN), rebuilt from the seed"""
    return ParamNet(schemas.i3d_schema(), seed=seed).state_dict()


def fixture_clip(g, tag):
    T, H, W, seed = (int(v) for v in g[f"{tag}_shape"])
    return np.random.default_rng(seed).integers(0, 256, (T, H, W, 3), dtype=np.uint8)


def subsample(m, steps):
    c, s = (int(v) for v in steps)
    return m[:, ::c, :, ::s, ::s]


@pytest.fixture(scope="module")
def hs(tmp_path_factory):
    lib = str(tmp_path_factory.mktemp("hostsim_i3d") / "libhostsim_i3d.so")
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", lib,
                           os.path.join(HERE, "hostsim", "hostsim_i3d.cpp")])
    return ctypes.CDLL(lib)


def test_oracle_reproduces_reference_fixture():
    g = np.load(FIXTURE)
    sd = seeded_state_dict(int(g["seed"]))
    torch.set_num_threads(max(torch.get_num_threads(), 4))
    for tag in g["clips"]:
        x = i3d_ref.video_from_u8(fixture_clip(g, tag))
        feats, maps = i3d_ref.extract_features(sd, x, return_maps=True)
        e = rel_err(feats.numpy(), g[f"{tag}_features"])
        assert feats.shape == (1, 1024) and e < 1e-5, (tag, e)
        for name, steps in zip(g["maps"], g["steps"]):
            m = maps[str(name)]
            assert tuple(m.shape) == tuple(g[f"{tag}_{name}_shape"]), (tag, name)
            e = rel_err(subsample(m, steps).numpy(), g[f"{tag}_{name}"])
            assert e < 1e-5, (tag, name, e)


def test_fixture_signal_is_strong():
    """Kaiming-normal weights keep the features O(1); with nn.Conv3d's default init they fade to ~1e-5"""
    g = np.load(FIXTURE)
    for tag in g["clips"]:
        f = g[f"{tag}_features"]
        assert 0.1 < np.abs(f).mean() < 100, (tag, np.abs(f).mean())


def test_schema_matches_reference_manifest():
    man = json.load(open(os.path.join(GOLD, "state_dict_manifest_i3d.json")))["i3d"]
    sd = ParamNet(schemas.i3d_schema(), seed=0).state_dict()
    assert {k: [list(v.shape), str(v.dtype).replace("torch.", "")] for k, v in sd.items()} == man
    assert list(sd) == list(man)
    assert len(sd) == 344 and sum(v.numel() for v in sd.values()) == 12711881


def _reference_format_state_dict(seed=7):
    man = json.load(open(os.path.join(GOLD, "state_dict_manifest_i3d.json")))["i3d"]
    gen = torch.Generator().manual_seed(seed)
    return {k: (torch.full(shape, 3, dtype=torch.int64) if dt == "int64" else torch.randn(shape, generator=gen))
            for k, (shape, dt) in man.items()}


def test_drop_in_loads_reference_state_dict_strict():
    from propainter_b200.model.i3d import InceptionI3d
    sd = _reference_format_state_dict()
    assert "Mixed_5c.b3b.bn.num_batches_tracked" in sd and "logits.conv3d.bias" in sd
    net = InceptionI3d(400, in_channels=3, final_endpoint='Logits')
    net.load_state_dict(sd, strict=True)
    assert torch.equal(net.P["Mixed_4e.b2b.conv3d.weight"], sd["Mixed_4e.b2b.conv3d.weight"])
    assert int(net.P["Conv3d_1a_7x7.bn.num_batches_tracked"]) == 3
    # checkpoints written before BatchNorm had num_batches_tracked load too, as into BatchNorm3d
    old = {k: v for k, v in sd.items() if not k.endswith("num_batches_tracked")}
    net.load_state_dict(old, strict=True)
    assert int(net.P["Conv3d_1a_7x7.bn.num_batches_tracked"]) == 0
    with pytest.raises(RuntimeError):
        net.load_state_dict({k: v for k, v in sd.items() if k != "Mixed_3b.b0.bn.running_var"}, strict=True)


def test_drop_in_constructor_and_unsupported_paths():
    from propainter_b200.model.i3d import InceptionI3d
    with pytest.raises(ValueError):
        InceptionI3d(400, in_channels=3, final_endpoint='Mixed_4f')
    with pytest.raises(ValueError):
        InceptionI3d(final_endpoint='NoSuchEndpoint')
    net = InceptionI3d()
    x = torch.rand(1, 3, 8, 64, 64)
    with pytest.raises(NotImplementedError):
        net(x)
    with pytest.raises(RuntimeError):                   # CPU input: there is no CPU path
        net.extract_features(x)
    with pytest.raises(ValueError):
        net.extract_features(torch.rand(1, 8, 3, 64, 64))


def test_ops_wrappers_raise_on_cpu_tensors():
    from propainter_b200 import ops
    with pytest.raises(RuntimeError):
        ops.i3d_input(torch.zeros(1, 4, 16, 16, 3, dtype=torch.uint8))
    with pytest.raises(RuntimeError):
        ops.i3d_input(torch.zeros(1, 3, 4, 16, 16))
    with pytest.raises(RuntimeError):
        ops.maxpool3d_same(torch.zeros(1, 4, 8, 8, 16), (3, 3, 3), (2, 2, 2))
    with pytest.raises(RuntimeError):
        ops.mean_thw(torch.zeros(2, 2, 3, 3, 1024))


def test_video_completion_summary_matches_script_accumulation():
    """scripts/evaluate_propainter.py:186-251 restated: per-frame lists appended across videos, python sums, calculate_vfid
    (mean, np.cov(rowvar=False), Frechet distance), time_all of seconds per frame"""
    from scipy import linalg

    from propainter_b200.evaluate import video_completion_summary
    rng = np.random.default_rng(0)
    results, frames = [], (5, 3, 7)
    for i, T in enumerate(frames):
        ps = list(rng.uniform(20, 40, T))
        if i == 1:
            ps[1] = float("inf")                        # an identical frame
        results.append({"psnr_per_frame": ps, "ssim_per_frame": list(rng.uniform(0.8, 1.0, T)), "seconds": float(rng.uniform(1, 2)),
                        "i3d": (rng.standard_normal(1024).astype(np.float32), rng.standard_normal(1024).astype(np.float32))})
    total_frame_psnr, total_frame_ssim, time_all, real, fake = [], [], [], [], []
    for r in results:
        for p, s in zip(r["psnr_per_frame"], r["ssim_per_frame"]):
            total_frame_psnr.append(p)
            total_frame_ssim.append(s)
        real.append(r["i3d"][0])
        fake.append(r["i3d"][1])
        time_all.append(r["seconds"] * 1.0 / len(r["psnr_per_frame"]))
    m1, m2 = np.mean(real, axis=0), np.mean(fake, axis=0)
    s1, s2 = np.cov(real, rowvar=False), np.cov(fake, rowvar=False)
    covmean = linalg.sqrtm(s1.dot(s2))
    covmean = covmean.real if np.iscomplexobj(covmean) else covmean
    vfid = (m1 - m2).dot(m1 - m2) + np.trace(s1) + np.trace(s2) - 2 * np.trace(covmean)
    got = video_completion_summary(results)
    assert got["psnr"] == sum(total_frame_psnr) / len(total_frame_psnr) == float("inf")
    assert got["ssim"] == sum(total_frame_ssim) / len(total_frame_ssim)
    assert got["seconds_per_frame"] == sum(time_all) / len(time_all)
    assert got["videos"] == 3
    assert abs(got["vfid"] - vfid) <= 1e-9 * abs(vfid), (got["vfid"], vfid)
    finite = [dict(r, psnr_per_frame=[min(p, 99.0) for p in r["psnr_per_frame"]]) for r in results]
    assert np.isfinite(video_completion_summary(finite)["psnr"])


def test_hostsim_same_pad_matches_oracle(hs):
    for k in (1, 2, 3, 7):
        for s in (1, 2):
            for n in range(1, 65):
                p = i3d_ref.compute_pad(k, s, n)
                assert hs.hs_same_pad(k, s, n) == p, (k, s, n)
                assert hs.hs_same_out(k, s, n) == (n + p - k) // s + 1 == -(-n // s), (k, s, n)


POOLS = [((1, 3, 3), (1, 2, 2)), ((3, 3, 3), (2, 2, 2)), ((2, 2, 2), (2, 2, 2)), ((3, 3, 3), (1, 1, 1))]


@pytest.mark.parametrize("kernel,stride", POOLS)
@pytest.mark.parametrize("T,H,W", [(5, 9, 13), (4, 8, 6), (1, 1, 2)])
def test_hostsim_maxpool_bit_exact_with_aten(hs, kernel, stride, T, H, W):
    gen = torch.Generator().manual_seed(T * 100 + H * 10 + W)
    x = torch.randn(T, H, W, generator=gen) - 0.5
    x.view(-1)[1::7] = -0.0
    x[0, 0, -1] = float("nan")
    ref = i3d_ref.maxpool_same(x[None, None], kernel, stride)[0, 0]
    out = torch.empty(ref.shape)
    hs.hs_maxpool3d_same(ctypes.cast(x.data_ptr(), FP), ctypes.cast(out.data_ptr(), FP), T, H, W, *kernel, *stride)
    assert torch.equal(out.isnan(), ref.isnan())
    assert torch.equal(torch.nan_to_num(out).view(torch.int32), torch.nan_to_num(ref).view(torch.int32))
    assert torch.isnan(out).any()
