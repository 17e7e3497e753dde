"""GPU parity of the on-the-fly RAFT correlation plan (AlternateCorrBlock): the two kernels against the oracles and
the all-pairs kernels, and RAFT with the plan forced or chosen by size.  Library convs / GEMMs run in fp32 so the
differences are those of our kernels."""
import types

import pytest
import torch

from oracle import alt_corr_ref, ops_ref, pipeline_ref, raft_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(autouse=True)
def _exact_library_math():
    from propainter_b200 import config
    a, b, c = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32, config.LINEAR_TF32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    config.LINEAR_TF32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32, config.LINEAR_TF32 = a, b, c


def rel_err(a, b):
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-12)


def cpu_sd(m):
    return {k: v.detach().cpu() for k, v in m.state_dict().items()}


@pytest.mark.parametrize("h,w", [(16, 22), (30, 54), (17, 23)])
def test_corr_lookup_otf_small(h, w):
    from propainter_b200 import ops
    gen = torch.Generator().manual_seed(2)
    F_, D = 3, 256
    fm = torch.randn(F_, D, h, w, generator=gen)
    idx1, idx2 = [0, 1, 1, 2], [1, 0, 2, 1]
    i1, i2 = torch.tensor(idx1, dtype=torch.int32, device=DEV), torch.tensor(idx2, dtype=torch.int32, device=DEV)
    fmap = fm.permute(0, 2, 3, 1).reshape(F_, h * w, D).contiguous().to(DEV)
    pooled = ops.corr_fmap_pyramid(fmap, h, w)
    for l, p in enumerate(pooled, 1):
        ref = alt_corr_ref.fmap_pyramid(fm)[l]
        assert torch.allclose(p.cpu().view(F_, h >> l, w >> l, D).permute(0, 3, 1, 2), ref, atol=1e-6)
    B = len(idx1)
    ys, xs = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    coords = torch.stack([xs, ys], 0).float()[None].repeat(B, 1, 1, 1) + torch.randn(B, 2, h, w, generator=gen) * 6
    cpm = coords.permute(0, 2, 3, 1).contiguous().to(DEV)
    got = ops.corr_lookup_otf(fmap, pooled, i1, i2, cpm)
    ref = ops_ref.corr_lookup(ops_ref.corr_pyramid(fm[idx1], fm[idx2]), coords)
    assert torch.allclose(got.cpu().permute(0, 3, 1, 2), ref, atol=1e-4, rtol=1e-4), (got.cpu().permute(0, 3, 1, 2) - ref).abs().max()
    levels = ops.corr_alloc(B, h, w, DEV)
    ops.corr_build(fmap, i1, i2, levels, h, w)
    allp = ops.corr_lookup(levels, cpm)
    assert torch.allclose(got, allp, atol=1e-4, rtol=1e-4), (got - allp).abs().max()
    far = cpm.clone()
    far[0, :2] += 500.0                      # centres far outside the image -> all-zero windows, no out-of-bounds reads
    far[1, :2] -= 500.0
    far[2, 0, 0] = float("inf")
    far[3, 0, 0] = float("nan")
    z = ops.corr_lookup_otf(fmap, pooled, i1, i2, far)
    assert (z[0, :2] == 0).all() and (z[1, :2] == 0).all() and (z[2, 0, 0] == 0).all() and (z[3, 0, 0] == 0).all()
    assert torch.equal(z[:, 2:], got[:, 2:])


def test_corr_lookup_otf_4k_pair():
    """One 3840x2160 pair (270x480 feature grid): a seeded subset of 4,096 query pixels against the oracle in fp32 on
    the GPU (the all-pairs oracle would need a 67 GB volume)."""
    from propainter_b200 import ops
    h, w, D = 270, 480, 256
    g = torch.Generator(device=DEV).manual_seed(5)
    fmap = torch.randn(2, h * w, D, device=DEV, generator=g)
    ys, xs = torch.meshgrid(torch.arange(h, device=DEV), torch.arange(w, device=DEV), indexing="ij")
    coords = (torch.stack([xs, ys], -1).float()[None] + torch.randn(1, h, w, 2, device=DEV, generator=g) * 20).contiguous()
    i1, i2 = torch.tensor([0], dtype=torch.int32, device=DEV), torch.tensor([1], dtype=torch.int32, device=DEV)
    pooled = ops.corr_fmap_pyramid(fmap, h, w)
    got = ops.corr_lookup_otf(fmap, pooled, i1, i2, coords)
    sel = torch.randperm(h * w, generator=torch.Generator().manual_seed(6))[:4096].to(DEV)
    f2 = fmap[1].view(h, w, D).permute(2, 0, 1)[None]
    ref = alt_corr_ref.corr_lookup_alt_points(fmap[0][sel].t()[None], f2, coords.view(1, h * w, 2)[:, sel])
    sub = got.view(h * w, 324)[sel][None]
    assert torch.isfinite(got).all()
    # relative to the output scale: at centres up to x = 480 the grid_sample coordinate round trip alone moves a tap by
    # a few ulp of 480 (~1e-4 px), which on uncorrelated random features changes values by up to ~2e-4 absolute
    assert rel_err(sub, ref) < 1e-4, rel_err(sub, ref)


def _raft_pair(iters_list, T, H, W, oracle_dev):
    from propainter_b200 import synth
    from propainter_b200.model.modules.flow_comp_raft import RAFT_bi
    from propainter_b200.RAFT.raft import ALL_PAIRS, ON_THE_FLY
    net = RAFT_bi(None, DEV, seed=1)
    u8, _, _ = synth.make_clip(T, H, W, seed=3)
    frames = pipeline_ref.to_float_frames(u8)
    sd = {k: v.to(oracle_dev) for k, v in cpu_sd(net.fix_raft).items()}
    for iters in iters_list:
        net.fix_raft.args = None
        assert net.fix_raft.corr_plan(H, W, DEV) == ALL_PAIRS
        af, ab = net(frames.to(DEV), iters=iters)
        net.fix_raft.args = types.SimpleNamespace(alternate_corr=True)
        assert net.fix_raft.corr_plan(H, W, DEV) == ON_THE_FLY
        fw, bw = net(frames.to(DEV), iters=iters)
        rf, rb = alt_corr_ref.raft_bi_alt(sd, frames.to(oracle_dev), iters)
        rf, rb = rf.to(DEV), rb.to(DEV)
        for got, ref, what in ((fw, rf, "otf vs oracle fw"), (bw, rb, "otf vs oracle bw"), (fw, af, "otf vs all-pairs fw"),
                               (bw, ab, "otf vs all-pairs bw")):
            e = rel_err(got, ref)
            epe = ((got - ref) ** 2).sum(2).sqrt().mean().item()
            print(f"{H}x{W} iters={iters} {what}: rel {e:.2e} EPE {epe:.5f}px")
            assert e < 1e-4 and epe < 0.01, (what, e, epe)
        if oracle_dev == DEV:                                  # the all-pairs run against its own oracle at this size too
            pf, pb = raft_ref.raft_bi(sd, frames.to(DEV), iters)
            assert rel_err(af, pf) < 1e-4 and rel_err(ab, pb) < 1e-4
    keys = [k[0] for k in net.fix_raft.graphs.entries]
    assert ("raft_bi", iters_list[-1], ON_THE_FLY) in keys or not keys     # the plan is part of the graph key
    return net, frames


def test_raft_bi_forced_on_the_fly():
    net, frames = _raft_pair((2, 12), 4, 128, 144, "cpu")
    # generic two-image entry point with the plan forced
    lo, up = net.fix_raft(frames[0, :2].to(DEV), frames[0, 1:3].to(DEV), iters=2, test_mode=True)
    rlo, rup = alt_corr_ref.raft_forward_alt(cpu_sd(net.fix_raft), frames[0, :2], frames[0, 1:3], 2, return_lowres=True)
    assert rel_err(up.cpu(), rup) < 1e-4 and rel_err(lo.cpu(), rlo) < 1e-4


def test_raft_bi_720p_both_plans():
    _raft_pair((12,), 3, 720, 1280, DEV)


def test_raft_bi_4k_selects_on_the_fly():
    """3840x2160 needs 181 GB for the smallest all-pairs call: the size alone selects the on-the-fly plan."""
    from propainter_b200 import synth
    from propainter_b200.model.modules.flow_comp_raft import RAFT_bi
    from propainter_b200.RAFT.raft import ON_THE_FLY
    net = RAFT_bi(None, DEV, seed=1)
    assert net.fix_raft.corr_plan(2160, 3840, DEV) == ON_THE_FLY
    u8, _, _ = synth.make_clip(3, 2160, 3840, seed=3)
    frames = pipeline_ref.to_float_frames(u8).to(DEV)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fw, bw = net(frames, iters=20)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    fw2, bw2 = net(frames, iters=20)
    print(f"4K RAFT_bi, 3 frames, 20 iters: peak {peak / 1e9:.2f} GB above the inputs, |flow|max {fw.abs().max().item():.2f}")
    assert fw.shape == (1, 2, 2, 2160, 3840) and torch.isfinite(fw).all() and torch.isfinite(bw).all()
    assert torch.equal(fw, fw2) and torch.equal(bw, bw2)
    assert peak < 16e9, peak                                 # measured ~8 GB: 4 pairs, 3 frames encoded
