"""CPU tests of RAFT-small (RAFT(args.small=True)): the state_dict schema against the reference manifest, the oracle
against the reference fixture (tests/golden/make_golden_raft_small.py), and the host build of the new per-element rules
(upflow8, radius-3 taps) against ATen and the oracle.  The kernels and the model run on the GPU in
test_gpu_raft_small.py."""
import ctypes
import json
import os
import subprocess
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import alt_corr_ref, ops_ref, raft_small_ref
from propainter_b200 import schemas, synth
from propainter_b200._params import ParamNet

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
FP = ctypes.POINTER(ctypes.c_float)
IP = ctypes.POINTER(ctypes.c_int)


def fp(t):
    assert t.dtype == torch.float32 and t.is_contiguous()
    return ctypes.cast(t.data_ptr(), FP)


def ip(t):
    assert t.dtype == torch.int32 and t.is_contiguous()
    return ctypes.cast(t.data_ptr(), IP)


def rel_err(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(np.asarray(b)).max(), 1e-12))


@pytest.fixture(scope="module")
def hs(tmp_path_factory):
    lib = str(tmp_path_factory.mktemp("hostsim_raft_small") / "libhostsim_raft_small.so")
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", lib,
                           os.path.join(HERE, "hostsim", "hostsim_raft_small.cpp")])
    return ctypes.CDLL(lib)


def test_small_schema_matches_reference_manifest():
    man = json.load(open(os.path.join(GOLD, "state_dict_manifest_raft_small.json")))["raft_small"]
    sd = ParamNet(schemas.raft_small_schema(), seed=0).state_dict()
    assert {k: [list(v.shape), str(v.dtype).replace("torch.", "")] for k, v in sd.items()} == man
    assert list(sd) == list(man)
    assert len(sd) == 106 and sum(v.numel() for v in sd.values()) == 990162
    assert not any("norm" in k for k in sd) and "fnet.layer2.0.downsample.0.weight" in sd


def test_small_raft_loads_reference_shaped_state_dict_strict():
    from propainter_b200.RAFT.raft import RAFT
    man = json.load(open(os.path.join(GOLD, "state_dict_manifest_raft_small.json")))["raft_small"]
    gen = torch.Generator().manual_seed(7)
    sd = {k: torch.randn(shape, generator=gen) for k, (shape, _) in man.items()}
    args = types.SimpleNamespace(small=True, mixed_precision=False, alternate_corr=False)
    net = RAFT(args)
    net.load_state_dict(sd, strict=True)
    assert (args.corr_levels, args.corr_radius) == (4, 3)          # set on args like raft.py:32-33
    assert (net.hidden_dim, net.context_dim) == (96, 64)
    assert torch.equal(net.P["update_block.gru.convq.weight"], sd["update_block.gru.convq.weight"])
    with pytest.raises(RuntimeError):
        RAFT(types.SimpleNamespace(small=False)).load_state_dict(sd, strict=True)
    net.half()                                                     # storage fp16, the forward code sees fp32
    assert net.fnet.conv1.weight.dtype == torch.float16 and net.P["fnet.conv1.weight"].dtype == torch.float32


def _c1_pairs():
    u8, _, _ = synth.make_clip(8, 128, 128, mask="square", seed=0)
    fr = torch.from_numpy(u8).permute(0, 3, 1, 2).contiguous().float().div(255) * 2 - 1
    return fr[:-1], fr[1:]


def test_oracle_reproduces_reference_fixture():
    g = np.load(os.path.join(GOLD, "raft_small_c1_8x128x128.npz"))
    sd = ParamNet(getattr(schemas, str(g["schema"]))(), seed=int(g["seed"])).state_dict()
    a, b = _c1_pairs()
    for it in g["iters"]:
        for tag, (x, y) in (("fw", (a, b)), ("bw", (b, a))):
            lr, up = raft_small_ref.raft_forward(sd, x, y, int(it), return_lowres=True)
            e_lr, e_up = rel_err(lr, g[f"lowres_{tag}_it{it}"]), rel_err(up[..., ::4, ::4], g[f"up_{tag}_it{it}"])
            assert e_lr < 1e-5 and e_up < 1e-5, (tag, it, e_lr, e_up)
    n = g["lookup_it0_fw"].shape[0]
    look = raft_small_ref.lookup_iter0(sd, a[:n], b[:n])
    assert look.shape == (n, 196, 16, 16)
    assert rel_err(look, g["lookup_it0_fw"]) < 1e-5
    # the alternate rule at radius 3 gives the same lookup
    assert rel_err(raft_small_ref.lookup_iter0(sd, a[:n], b[:n], alternate=True), g["lookup_it0_fw"]) < 1e-5


# RAFT's feature grids start at 16 x 16 (128 px frames); odd and even sides, n > 1
UPFLOW8_SHAPES = [(1, 16, 16), (3, 16, 16), (3, 17, 23), (2, 30, 54), (2, 45, 80), (1, 64, 21)]


@pytest.mark.parametrize("n,h,w", UPFLOW8_SHAPES)
def test_hostsim_upflow8_bit_exact_with_aten(hs, n, h, w):
    gen = torch.Generator().manual_seed(h * 100 + w)
    flow = torch.randn(n, 2, h, w, generator=gen) * 7
    ref = 8 * F.interpolate(flow, size=(8 * h, 8 * w), mode="bilinear", align_corners=True)
    assert torch.equal(ref, raft_small_ref.upflow8(flow))
    out = torch.empty(n, 2, 8 * h, 8 * w)
    flow_pm = flow.permute(0, 2, 3, 1).contiguous()                 # kept alive across the call (ctypes holds no reference)
    hs.hs_upflow8(fp(flow_pm), fp(out), n, h, w)
    assert torch.equal(out, ref), (out - ref).abs().max()


def _coords(gen, B, h, w, amp=5.0):
    ys, xs = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    c = torch.stack([xs, ys], 0).float()[None].repeat(B, 1, 1, 1) + torch.randn(B, 2, h, w, generator=gen) * amp
    c[0, :, :2] += 300.0                                            # far outside the level: zeros padding
    c[-1, :, -1] -= 300.0
    return c


@pytest.mark.parametrize("h,w", [(16, 16), (17, 23), (19, 26)])
def test_hostsim_radius3_tap_rules_match_oracle(hs, h, w):
    gen = torch.Generator().manual_seed(h + w)
    D, B = 128, 3
    fm = torch.randn(3, D, h, w, generator=gen)
    idx1, idx2 = [0, 1, 2], [1, 2, 0]
    coords = _coords(gen, B, h, w)
    ref = ops_ref.corr_lookup(ops_ref.corr_pyramid(fm[idx1], fm[idx2]), coords, radius=3)
    assert ref.shape == (B, 196, h, w)
    assert rel_err(alt_corr_ref.corr_lookup_alt(fm[idx1], fm[idx2], coords, radius=3), ref) < 1e-5
    cpm = coords.permute(0, 2, 3, 1).contiguous()
    # all-pairs: the oracle's pyramid stored in the kernel's row-padded planes
    pyr, lv = ops_ref.corr_pyramid(fm[idx1], fm[idx2]), []
    for p in pyr:
        hl, wl = p.shape[-2:]
        q = torch.zeros(p.shape[0], hl, (wl + 3) & ~3)
        q[..., :wl] = p[:, 0]
        lv.append(q.contiguous())
    out = torch.empty(B, h, w, 196)
    hs.hs_corr_lookup_r3(*[fp(q) for q in lv], fp(cpm), fp(out), ctypes.c_long(B * h * w), h, w)
    got = out.permute(0, 3, 1, 2)
    assert (got - ref).abs().max() < 1e-5 and (got[0, :, :2] == 0).all()
    # on the fly: pixel-major feature levels, dot products at lookup time, / sqrt(128)
    fl = [f.permute(0, 2, 3, 1).reshape(3, -1, D).contiguous() for f in alt_corr_ref.fmap_pyramid(fm)]
    out2 = torch.empty(B, h, w, 196)
    i1, i2 = torch.tensor(idx1, dtype=torch.int32), torch.tensor(idx2, dtype=torch.int32)
    hs.hs_corr_lookup_otf_r3(*[fp(f) for f in fl], D, ip(i1), ip(i2), ctypes.c_long(B), fp(cpm), fp(out2), h, w)
    got2 = out2.permute(0, 3, 1, 2)
    assert (got2 - ref).abs().max() < 1e-5 and (got2[0, :, :2] == 0).all()
