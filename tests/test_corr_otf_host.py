"""CPU tests of the on-the-fly RAFT correlation plan (AlternateCorrBlock): the oracle restatement against the all-pairs
oracle, the host build of the kernel's tile rule against both, the plan rule and its batching, and the RAFT plumbing
with the plan forced.  The kernels themselves are checked on the GPU in test_gpu_corr_otf.py."""
import ctypes
import types

import pytest
import torch

from oracle import alt_corr_ref, ops_ref
from tests import ops_emulation_otf

# odd sizes: floor pooling drops a row and / or a column.  Level 3 needs >= 2 rows and columns (h, w >= 16): with one,
# bilinear_sampler's 2*x/(W-1) divides by zero and the reference's windows are NaN.
SHAPES = [(19, 27), (17, 23), (16, 22), (31, 45)]


@pytest.fixture(scope="module")
def hostsim_otf(tmp_path_factory):
    return ops_emulation_otf.build_hostsim(str(tmp_path_factory.mktemp("hostsim_otf")))


def rel_err(a, b):
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-12)


def _case(h, w, seed, B=4):
    """random fmaps of 3 frames, the 4 pairs of test_corr_build_pool_lookup, centres up to +-500 px outside the frame"""
    gen = torch.Generator().manual_seed(seed)
    fm = torch.randn(3, 256, h, w, generator=gen)
    idx1, idx2 = [0, 1, 1, 2], [1, 0, 2, 1]
    ys, xs = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    coords = torch.stack([xs, ys], 0).float()[None].repeat(B, 1, 1, 1) + torch.randn(B, 2, h, w, generator=gen) * 6
    coords[0, :, :2] += 500.0
    coords[1, :, :2] -= 500.0
    coords[2, 0, -1] += 1e4
    return fm, idx1, idx2, coords


@pytest.mark.parametrize("h,w", SHAPES)
def test_alt_oracle_matches_all_pairs_oracle(h, w):
    fm, idx1, idx2, coords = _case(h, w, 0)
    ref = ops_ref.corr_lookup(ops_ref.corr_pyramid(fm[idx1], fm[idx2]), coords)
    got = alt_corr_ref.corr_lookup_alt(fm[idx1], fm[idx2], coords)
    assert got.shape == ref.shape == (4, 324, h, w)
    assert rel_err(got, ref) < 1e-5, rel_err(got, ref)
    assert (got[0, :, :2] == 0).all() and (got[1, :, :2] == 0).all()


@pytest.mark.parametrize("h,w", SHAPES)
def test_hostsim_tile_rule_matches_oracles(hostsim_otf, h, w):
    fm, idx1, idx2, coords = _case(h, w, 1)
    fmap = fm.permute(0, 2, 3, 1).reshape(3, h * w, 256).contiguous()
    pooled = ops_emulation_otf.fmap_pyramid(hostsim_otf, fmap, h, w)
    for l, p in enumerate(pooled, 1):                                  # floor sizes of avg_pool2d(2, stride=2)
        ref = alt_corr_ref.fmap_pyramid(fm)[l]
        assert ref.shape[-2:] == (h >> l, w >> l)
        assert torch.allclose(p.view(3, h >> l, w >> l, 256).permute(0, 3, 1, 2), ref, atol=1e-6)
    got = ops_emulation_otf.lookup_otf(hostsim_otf, fmap, pooled, torch.tensor(idx1), torch.tensor(idx2),
                                       coords.permute(0, 2, 3, 1)).permute(0, 3, 1, 2)
    alt = alt_corr_ref.corr_lookup_alt(fm[idx1], fm[idx2], coords)
    allp = ops_ref.corr_lookup(ops_ref.corr_pyramid(fm[idx1], fm[idx2]), coords)
    assert rel_err(got, alt) < 1e-5 and rel_err(got, allp) < 1e-5, (rel_err(got, alt), rel_err(got, allp))
    assert (got[0, :, :2] == 0).all() and (got[1, :, :2] == 0).all()


def test_plan_rule():
    from propainter_b200.RAFT.raft import ALL_PAIRS, ON_THE_FLY, corr_plan
    gb80 = 80 * 2 ** 30
    for H, W in ((128, 128), (240, 432), (720, 1280), (1080, 1920), (1440, 2560)):    # C1-C5 and 2560x1440
        assert corr_plan(H, W, total_bytes=gb80) == ALL_PAIRS, (H, W)
        assert corr_plan(H, W, alternate=True, total_bytes=gb80) == ON_THE_FLY
    for H, W in ((2160, 3840), (2160, 4096), (4320, 7680)):
        assert corr_plan(H, W, total_bytes=gb80) == ON_THE_FLY, (H, W)
    assert corr_plan(2160, 3840) == ALL_PAIRS                       # no device limit (CPU tensors): size never forces it


def test_on_the_fly_batch_length():
    from propainter_b200.inference_propainter import auto_clip_frames, raft_clip_len
    from propainter_b200.RAFT.raft import ALL_PAIRS, ON_THE_FLY, OTF_BYTES_PER_PAIR_PX
    for T, H, W in ((8, 2160, 3840), (300, 2160, 3840), (300, 720, 1280), (80, 240, 432), (1000, 4320, 7680)):
        clip = auto_clip_frames(T, H, W, ON_THE_FLY)
        per_pair = OTF_BYTES_PER_PAIR_PX * H * W
        assert clip >= raft_clip_len(W)                             # never below the reference's clip length
        if clip > raft_clip_len(W):
            assert clip <= T and 2 * (clip - 1) * per_pair <= 8e9   # the call's pairs fit the 8 GB budget ...
            assert clip == T or 2 * clip * per_pair > 8e9           # ... and one more frame would not
    assert auto_clip_frames(8, 2160, 3840, ON_THE_FLY) == 2
    # the all-pairs plan keeps its pyramid estimate
    for T, H, W in ((80, 240, 432), (300, 720, 1280), (1000, 1080, 1920)):
        n = (H // 8) * (W // 8)
        assert auto_clip_frames(T, H, W, ALL_PAIRS) == max(raft_clip_len(W), min(T, int(8e9 // (5.4 * n * n)) // 2 + 1))


def test_raft_plumbing_on_the_fly(monkeypatch, hostsim, hostsim_otf):
    from oracle import pipeline_ref
    from propainter_b200 import synth
    from propainter_b200.model.modules.flow_comp_raft import RAFT_bi
    ops_emulation_otf.install(monkeypatch, hostsim, hostsim_otf)
    calls = {"otf": 0}
    from propainter_b200 import ops
    lk = ops.corr_lookup_otf
    monkeypatch.setattr(ops, "corr_lookup_otf", lambda *a, **k: (calls.__setitem__("otf", calls["otf"] + 1), lk(*a, **k))[1])
    monkeypatch.setattr(ops, "corr_build", lambda *a, **k: pytest.fail("all-pairs volume built under alternate_corr"))
    net = RAFT_bi(None, "cpu", seed=1)
    net.fix_raft.args = types.SimpleNamespace(alternate_corr=True)
    u8, _, _ = synth.make_clip(3, 128, 144, seed=3)
    frames = pipeline_ref.to_float_frames(u8)
    fw, bw = net(frames, iters=3)
    sd = net.fix_raft.state_dict()
    rf, rb = alt_corr_ref.raft_bi_alt(sd, frames, 3)
    assert rel_err(fw, rf) < 1e-4 and rel_err(bw, rb) < 1e-4, (rel_err(fw, rf), rel_err(bw, rb))
    lo, up = net.fix_raft(frames[0, :2], frames[0, 1:3], iters=2, test_mode=True)
    rlo, rup = alt_corr_ref.raft_forward_alt(sd, frames[0, :2], frames[0, 1:3], 2, return_lowres=True)
    assert rel_err(up, rup) < 1e-4 and rel_err(lo, rlo) < 1e-4
    assert calls["otf"] == 3 + 2
