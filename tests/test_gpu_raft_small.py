"""GPU parity of RAFT-small (RAFT(args.small=True)): the radius-3 lookups (TMA, plain, on the fly), upflow8, the motion
packing and the gate kernels at C = 96, the model against the reference fixture and the oracle on both correlation plans,
and a pipeline whose RAFT_bi holds a small RAFT.  Library convs / GEMMs run in fp32 so the differences are those of our
kernels."""
import os
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import alt_corr_ref, ops_ref, pipeline_ref, raft_small_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


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


def epe(a, b):
    return ((a - b) ** 2).sum(-3).sqrt().mean().item()


def small_args(alternate=False):
    return types.SimpleNamespace(small=True, mixed_precision=False, alternate_corr=alternate)


# 128 px minimum (16 x 16), widths that are not multiples of 4 at some level, one 1920x1080 pair
LOOKUP_SHAPES = [(16, 16, 3), (17, 23, 3), (30, 54, 2), (135, 240, 1)]


@pytest.mark.parametrize("h,w,B", LOOKUP_SHAPES)
def test_radius3_lookups_match_oracle(h, w, B):
    from propainter_b200 import ops
    gen = torch.Generator(device=DEV).manual_seed(h * w)
    D = 128
    fm = torch.randn(B + 1, D, h, w, device=DEV, generator=gen)
    idx1, idx2 = list(range(B)), list(range(1, B + 1))
    ys, xs = torch.meshgrid(torch.arange(h, device=DEV), torch.arange(w, device=DEV), indexing="ij")
    coords = torch.stack([xs, ys], 0).float()[None].repeat(B, 1, 1, 1) + torch.randn(B, 2, h, w, device=DEV, generator=gen) * 5
    coords[0, :, :2] += 400.0                                       # outside every level: zeros padding
    coords[-1, :, -1] -= 400.0
    cpm = coords.permute(0, 2, 3, 1).contiguous()
    fmap = fm.permute(0, 2, 3, 1).reshape(B + 1, h * w, D).contiguous()
    i1, i2 = torch.tensor(idx1, dtype=torch.int32, device=DEV), torch.tensor(idx2, dtype=torch.int32, device=DEV)
    levels = ops.corr_alloc(B, h, w, DEV)
    ops.corr_build(fmap, i1, i2, levels, h, w)
    pooled = ops.corr_fmap_pyramid(fmap, h, w)
    tma = ops.corr_lookup_r(levels, cpm, 3)
    ldg = ops.corr_lookup_r(levels, cpm, 3, tma=False)
    otf = ops.corr_lookup_otf_r(fmap, pooled, i1, i2, cpm, 3)
    assert tma.shape == (B, h, w, 196)
    if h * w <= 2000:
        ref = ops_ref.corr_lookup(ops_ref.corr_pyramid(fm[idx1], fm[idx2]), coords, radius=3).permute(0, 2, 3, 1)
    else:                                      # 1080p: the alternate oracle over a seeded subset (no 4 GB fp64 volume)
        sel = torch.randperm(h * w, generator=torch.Generator().manual_seed(1))[:2048].to(DEV)
        ref = alt_corr_ref.corr_lookup_alt_points(fmap[0][sel].t()[None], fm[1:2], cpm.view(1, h * w, 2)[:, sel], radius=3)
        tma, ldg, otf = [t.view(1, h * w, 196)[:, sel] for t in (tma, ldg, otf)]
    # Bar: 1e-5 of the output scale.  The oracle evaluates grid_sample's normalise / un-normalise round trip with other
    # roundings than the kernels' rule (the TMA kernel drops it, corr_lookup_tma.cu), and the all-pairs volume comes from
    # a different GEMM; at centres up to x = 54 that moves values by up to 2.4e-5 absolute on these N(0, 1) correlations.
    # At 1920x1080 (centres up to x = 240, against the alternate oracle's pooled features) the bar is the basic model's
    # 1e-4 of the output scale (test_gpu_corr_otf.py), for the same reason.
    bar = 1e-5 if h * w <= 2000 else 1e-4
    for got, what in ((tma, "tma"), (ldg, "ldg"), (otf, "otf")):
        assert rel_err(got, ref) < bar, (what, rel_err(got, ref), (got - ref).abs().max().item())
    assert rel_err(otf, ldg) < bar and rel_err(otf, tma) < bar
    if h * w <= 2000:
        assert (tma[0, :2] == 0).all() and (otf[0, :2] == 0).all()


def test_radius_and_dim_refusals():
    from propainter_b200 import _lib, ops
    L = _lib.lib()
    h, w, B = 16, 16, 1
    levels = ops.corr_alloc(B, h, w, DEV)
    arr = ops._level_array(levels)
    coords = torch.zeros(B, h, w, 2, device=DEV)
    out = torch.empty(B, h, w, 324, device=DEV)
    for r in (0, 2, 5):
        assert L.pp_corr_lookup_r(arr, r, coords.data_ptr(), out.data_ptr(), B, h, w, None) == -1
        assert L.pp_corr_lookup_ldg_r(arr, r, coords.data_ptr(), out.data_ptr(), B, h, w, None) == -1
    i = torch.zeros(1, dtype=torch.int32, device=DEV)
    for D, r in ((64, 3), (192, 3), (256, 3), (128, 4), (128, 2), (512, 4)):
        fmap = torch.zeros(2, h * w, D, device=DEV)
        pooled = ops.corr_fmap_pyramid(fmap, h, w)
        pa = (ops.ctypes.c_void_p * 3)(*[p.data_ptr() for p in pooled])
        assert L.pp_corr_lookup_otf_r(fmap.data_ptr(), pa, D, r, i.data_ptr(), i.data_ptr(), 1, coords.data_ptr(), out.data_ptr(),
                                      h, w, None) == -1, (D, r)
    with pytest.raises(RuntimeError):
        ops.upflow8(torch.zeros(1, 4, 4, 2))                         # CPU tensors are refused


@pytest.mark.parametrize("n,h,w", [(1, 16, 16), (3, 17, 23), (2, 30, 54), (2, 45, 80), (1, 135, 240)])
def test_upflow8_bit_exact_with_aten_cpu(n, h, w):
    from propainter_b200 import ops
    flow = torch.randn(n, 2, h, w, generator=torch.Generator().manual_seed(h + w)) * 9
    ref = 8 * F.interpolate(flow, size=(8 * h, 8 * w), mode="bilinear", align_corners=True)
    got = ops.upflow8(flow.permute(0, 2, 3, 1).contiguous().to(DEV)).cpu()
    assert torch.equal(got, ref), ((got != ref).sum().item(), (got - ref).abs().max().item())


def test_pack_motion_n_and_gates_at_c96():
    from propainter_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(3)
    B, h, w, C = 2, 13, 19, 96
    mot = torch.randn(B, h, w, 80, device=DEV, generator=g)
    bias = torch.randn(80, device=DEV, generator=g)
    flow = torch.randn(B, h, w, 2, device=DEV, generator=g)
    HX = torch.full((B, h, w, 180), 7.0, device=DEV)
    RX = torch.full((B, h, w, 180), 7.0, device=DEV)
    ops.raft_pack_motion_n(mot, flow, HX[..., 96:], RX[..., 96:], 80, bias=bias)
    exp = torch.cat([torch.relu(mot + bias), flow, torch.zeros(B, h, w, 2, device=DEV)], -1)
    assert torch.equal(HX[..., 96:], exp) and torch.equal(RX[..., 96:], exp)
    assert (HX[..., :96] == 7).all()                                  # the state slice is untouched
    net = torch.randn(B, h, w, C, device=DEV, generator=g)
    HX[..., :96] = net
    zr, pre = torch.randn(B, h, w, 2 * C, device=DEV, generator=g), torch.randn(B, h, w, 2 * C, device=DEV, generator=g)
    z = torch.empty(B, h, w, C, device=DEV)
    ops.gru_gate(zr, None, HX[..., :96], z, RX[..., :96], pre=pre)
    s = zr + pre
    assert torch.allclose(z, torch.sigmoid(s[..., :C]), atol=1e-6)
    assert torch.allclose(RX[..., :96], net * torch.sigmoid(s[..., C:]), atol=1e-6)
    q, preq = torch.randn(B, h, w, C, device=DEV, generator=g), torch.randn(B, h, w, C, device=DEV, generator=g)
    netc = torch.empty(B, h, w, C, device=DEV)
    ops.gru_update(q, None, z, HX[..., :96], net_copy=netc, pre=preq)
    ref = (1 - z) * net + z * torch.tanh(q + preq)
    assert torch.allclose(HX[..., :96], ref, atol=1e-6) and torch.equal(netc, HX[..., :96])


def _fixture_net():
    from propainter_b200 import schemas
    from propainter_b200._params import ParamNet
    from propainter_b200.RAFT.raft import RAFT
    g = np.load(os.path.join(GOLD, "raft_small_c1_8x128x128.npz"))
    sd = ParamNet(getattr(schemas, str(g["schema"]))(), seed=int(g["seed"])).state_dict()
    net = RAFT(small_args())
    net.load_state_dict(sd, strict=True)
    return g, sd, net.to(DEV)


def _c1_frames():
    from propainter_b200 import synth
    u8, _, _ = synth.make_clip(8, 128, 128, mask="square", seed=0)
    return pipeline_ref.to_float_frames(u8)[0]


def test_small_raft_matches_fixture_and_oracle():
    """forward (with and without flow_init) and flows_bidirectional against the reference fixture and the oracle, on the
    all-pairs plan and with the on-the-fly plan forced; graph replay bit-identical to eager."""
    from propainter_b200.RAFT.raft import ALL_PAIRS, ON_THE_FLY
    g, sd, net = _fixture_net()
    fr = _c1_frames()
    a, b = fr[:-1].to(DEV), fr[1:].to(DEV)
    for it in (6, 20):
        lr, up = net(a, b, iters=it)
        for got, key in ((lr, f"lowres_fw_it{it}"), (up[..., ::4, ::4], f"up_fw_it{it}")):
            ref = torch.from_numpy(g[key]).to(DEV)
            assert rel_err(got, ref) < 2e-3 and epe(got, ref) < 0.05, (key, rel_err(got, ref), epe(got, ref))
        fw, bw = net.flows_bidirectional(fr.to(DEV), iters=it)
        for got, key in ((fw, f"up_fw_it{it}"), (bw, f"up_bw_it{it}")):
            ref = torch.from_numpy(g[key]).to(DEV)
            assert rel_err(got[..., ::4, ::4], ref) < 2e-3 and epe(got[..., ::4, ::4], ref) < 0.05, key
        eager = net._flows_bidirectional(fr.to(DEV), it, ALL_PAIRS)
        again = net.flows_bidirectional(fr.to(DEV), iters=it)                  # graph replay
        assert torch.equal(again[0], fw) and torch.equal(again[1], bw)
        assert rel_err(eager[0], fw) == 0.0 and rel_err(eager[1], bw) == 0.0, "graph replay differs from eager"
    # flow_init, against the oracle
    init = lr.detach() * 0.5
    lr2, up2 = net(a, b, iters=6, flow_init=init)
    rlr, rup = raft_small_ref.raft_forward({k: v.to(DEV) for k, v in sd.items()}, a, b, 6, flow_init=init, return_lowres=True)
    assert rel_err(up2, rup) < 2e-3 and epe(up2, rup) < 0.05
    # the on-the-fly plan, forced as for the basic model, against the oracle's alternate restatement
    net.args.alternate_corr = True
    assert net.corr_plan(128, 128, DEV) == ON_THE_FLY
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    for it in (6, 20):
        fw, bw = net.flows_bidirectional(fr.to(DEV), iters=it)
        rf, rb = raft_small_ref.raft_bi(sdd, fr[None].to(DEV), it, alternate=True)
        for got, ref in ((fw, rf[0]), (bw, rb[0])):
            assert rel_err(got, ref) < 2e-3 and epe(got, ref) < 0.05, (it, rel_err(got, ref), epe(got, ref))
        lr, up = net(a, b, iters=it)
        rlr, rup = raft_small_ref.raft_forward(sdd, a, b, it, alternate=True, return_lowres=True)
        assert rel_err(up, rup) < 2e-3 and epe(up, rup) < 0.05
    lr2, up2 = net(a, b, iters=6, flow_init=init)
    rlr, rup = raft_small_ref.raft_forward(sdd, a, b, 6, flow_init=init, alternate=True, return_lowres=True)
    assert rel_err(up2, rup) < 2e-3 and epe(up2, rup) < 0.05
    net.args.alternate_corr = False
    with pytest.raises(NotImplementedError):
        net(a, b, iters=2, test_mode=False)


def test_pipeline_with_small_raft(monkeypatch):
    """ProPainterPipeline(fix_raft=RAFT_bi holding a small RAFT) on a C2-sized clip: finite stages, __call__ / flows
    consistent, and PSNR >= 40 dB against the oracle pipeline run with the small oracle RAFT."""
    from propainter_b200 import synth
    from propainter_b200.inference_propainter import InferenceConfig, ProPainterPipeline
    from propainter_b200.model.modules.flow_comp_raft import RAFT_bi
    from propainter_b200.RAFT.raft import RAFT
    bi = RAFT_bi(None, DEV, seed=1)
    bi.fix_raft = RAFT(small_args(), seed=4).to(DEV)
    pipe = ProPainterPipeline(fix_raft=bi, device=DEV)
    u8, fm, md = synth.make_clip(20, 240, 432, mask="ellipse", seed=0)
    cfg = InferenceConfig(raft_iter=20)
    comp, st = pipe(torch.from_numpy(u8), fm, md, cfg, return_stages=True)
    for k in ("gt_flows", "pred_flows"):
        for t in st[k]:
            assert torch.isfinite(t).all(), k
    gt, pred = pipe.flows(torch.from_numpy(u8), fm, cfg)
    for x, y in zip(gt + pred, st["gt_flows"] + st["pred_flows"]):
        assert torch.equal(x, y)
    sds = {k: {n: v.detach().cpu() for n, v in sd.items()} for k, sd in pipe.state_dicts().items()}
    monkeypatch.setattr(pipeline_ref.raft_ref, "raft_bi", raft_small_ref.raft_bi)
    ref = pipeline_ref.run_pipeline(sds, u8, fm, md, raft_iter=cfg.raft_iter)
    psnr = ops_ref.psnr_u8(comp.cpu().numpy(), ref)
    print(f"small-RAFT pipeline vs oracle: {psnr:.2f} dB")
    assert psnr >= 40.0, psnr
