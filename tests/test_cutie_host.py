"""CPU tests of the Cutie mask tracker: the state_dict schema against the reference manifest, the drop-in's loading rules,
the tracking schedule (memory frames, sensory updates, FIFO evictions) against the reference run recorded in
tests/golden/cutie_track.npz, MaskMapper's id handling, the driver's refusals of options outside the demo's config, and
the host build of the fused readout's top-k / tie / merge rules (tests/hostsim/hostsim_cutie.cpp) against the oracle.
The kernels and the network run on the GPU in test_gpu_cutie.py."""
import ctypes
import json
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import cutie_ref
from propainter_b200 import schemas
from propainter_b200._params import ParamNet
from propainter_b200.model.cutie import CUTIE
from propainter_b200.tracker import DEMO_CONFIG, MaskMapper, MaskTracker, Schedule

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
FIXTURE = os.path.join(GOLD, "cutie_track.npz")


@pytest.fixture(scope="module")
def hs(tmp_path_factory):
    lib = str(tmp_path_factory.mktemp("hostsim_cutie") / "libhostsim_cutie.so")
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", lib,
                           os.path.join(HERE, "hostsim", "hostsim_cutie.cpp")])
    h = ctypes.CDLL(lib)
    h.hs_topk_select.restype = ctypes.c_int
    h.hs_topk_select.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    h.hs_similarity.restype = ctypes.c_float
    h.hs_similarity.argtypes = [ctypes.c_float, ctypes.c_float]
    h.hs_ring_row.restype = ctypes.c_long
    h.hs_ring_row.argtypes = [ctypes.c_int] * 4
    return h


def select(hs, sim, k, splits=8, tt=16):
    sim = np.ascontiguousarray(sim, np.float32)
    out = np.zeros(max(k, 1), np.int32)
    keff = hs.hs_topk_select(sim.ctypes.data, sim.size, k, splits, tt, out.ctypes.data)
    return out[:keff]


def test_schema_matches_reference_manifest():
    man = json.load(open(os.path.join(GOLD, "state_dict_manifest_cutie.json")))["cutie"]
    sd = ParamNet(schemas.cutie_schema(), seed=0).state_dict()
    assert list(sd) == list(man)
    assert {k: [list(v.shape), str(v.dtype).replace("torch.", "")] for k, v in sd.items()} == man


def test_reference_key_set_loads_strict():
    """a state_dict with exactly the reference's keys and shapes loads strict=True; the inv_freq buffers are the
    reference's PositionalEncoding values"""
    man = json.load(open(os.path.join(GOLD, "state_dict_manifest_cutie.json")))["cutie"]
    sd = {k: torch.zeros(s, dtype=getattr(torch, d)) for k, (s, d) in man.items()}
    net = CUTIE(seed=1)
    net.load_state_dict(sd, strict=True)
    d = 128
    want = 1.0 / (128 ** (torch.arange(0, d, 2).float() / d))
    assert torch.equal(CUTIE(seed=0).P["object_transformer.spatial_pe.inv_freq"], want)


def test_load_weights_converts_single_object_checkpoint():
    """CUTIE.load_weights (cutie.py:202-247): 4-channel mask_encoder.conv1 and 257-channel sensory_compress gain a channel
    (zeros with init_as_zero_if_needed); unknown keys are ignored, missing ones kept"""
    src = ParamNet(schemas.cutie_schema(), seed=3).state_dict()
    src["mask_encoder.conv1.weight"] = src["mask_encoder.conv1.weight"][:, :4].clone()
    src["pixel_fuser.sensory_compress.weight"] = src["pixel_fuser.sensory_compress.weight"][:, :257].clone()
    src["not.a.key"] = torch.zeros(1)
    del src["aux_computer.sensory_aux.projection.bias"]
    net = CUTIE(seed=5)
    before = net.P["aux_computer.sensory_aux.projection.bias"].clone()
    net.load_weights(src, init_as_zero_if_needed=True)
    w = net.P["mask_encoder.conv1.weight"]
    assert w.shape == (64, 5, 7, 7) and torch.equal(w[:, :4], src["mask_encoder.conv1.weight"]) and not w[:, 4].any()
    assert net.P["pixel_fuser.sensory_compress.weight"].shape == (256, 258)[:1] + (258, 1, 1)
    assert torch.equal(net.P["aux_computer.sensory_aux.projection.bias"], before)


def test_schedule_matches_reference_run():
    """memory frames, segmentation, sensory updates and the frames held in working memory (FIFO evictions) of a 32-frame
    run, frame by frame, against the reference InferenceCore's"""
    g = np.load(FIXTURE)
    c = DEMO_CONFIG
    s = Schedule(c["mem_every"], c["stagger_updates"], c["max_mem_frames"] - 1)
    for t, (mem, seg, upd, n) in enumerate(g["track_schedule"]):
        is_mem, need_seg, update = s.begin(has_mask=(t == 0))
        if is_mem:
            s.add()
        assert (is_mem, need_seg, update and need_seg, s.n_frames) == (bool(mem), bool(seg), bool(upd), int(n)), t
        want = [int(f) for f in g["track_mem_frames"][t] if f >= 0]
        assert s.memory_frames() == want, (t, s.memory_frames(), want)
    assert len(g["track_schedule"]) > 5 * c["mem_every"] and s.head != 0          # the FIFO has evicted


@pytest.mark.parametrize("stagger,want", [(5, {1, 2, 3, 4, 5}), (3, {1, 3, 5}), (2, {1, 5})])
def test_stagger_offsets(stagger, want):
    """InferenceCore.__init__ (inference_core.py:34-40)"""
    assert Schedule(5, stagger, 4).stagger_ti == want


def test_mask_mapper_non_consecutive_ids():
    """template ids {3, 7} become objects 1, 2 and map back to 3, 7; consecutive ids map to themselves"""
    m = np.zeros((4, 5), np.uint8)
    m[0, :2], m[3, 3:] = 3, 7
    mp = MaskMapper()
    _, objects = mp.convert_mask(m)
    assert objects == [1, 2] and not mp.coherent
    mapped = mp.input_lut()[m]
    assert set(np.unique(mapped)) == {0, 1, 2}
    assert np.array_equal(mp.output_lut(2)[mapped], m)
    mp2 = MaskMapper()
    m2 = np.where(m == 3, 1, np.where(m == 7, 2, 0)).astype(np.uint8)
    _, objects = mp2.convert_mask(m2)
    assert objects == [1, 2] and mp2.coherent and np.array_equal(mp2.input_lut()[m2], m2)
    assert MaskMapper().convert_mask(np.zeros((3, 3), np.uint8))[1] == []


@pytest.mark.parametrize("opt", [dict(use_long_term=True), dict(flip_aug=True), dict(max_internal_size=480),
                                 dict(chunk_size=1), dict(top_k=40), dict(bogus=1)])
def test_tracker_refuses_options_outside_demo_config(opt):
    with pytest.raises(ValueError):
        MaskTracker(CUTIE(seed=0), "cpu", **opt)


@pytest.mark.parametrize("N,k", [(1000, 30), (31, 30), (30, 30), (17, 30), (1, 30), (300, 1), (257, 32)])
def test_topk_selection_matches_oracle(hs, N, k):
    """distinct similarities: the kernel's split lists + rank merge select the same tokens, in the same order, as a full
    descending sort; k > N keeps all N (the first memory frames of a small frame)"""
    rng = np.random.default_rng(N * 31 + k)
    sim = -rng.exponential(3.0, N).astype(np.float32)
    got = select(hs, sim, k)
    want = cutie_ref.topk_order(torch.from_numpy(sim).view(N, 1), k)[0].numpy()
    assert len(got) == min(k, N) and np.array_equal(got, want)


def test_topk_exact_ties_keep_lower_index(hs):
    """exact ties at and across the k-th place: the lower token index wins, whichever split list it arrives in"""
    N, k = 600, 30
    rng = np.random.default_rng(0)
    sim = np.round(-rng.exponential(2.0, N) - 0.1, 1).astype(np.float32)   # many repeated values, all < 0
    sim[[5, 130, 131, 400, 599]] = 0.0                                   # a tie at the top, across splits and tiles
    got = select(hs, sim, k)
    want = cutie_ref.topk_order(torch.from_numpy(sim).view(N, 1), k)[0].numpy()
    assert np.array_equal(got, want)
    assert list(got[:5]) == [5, 130, 131, 400, 599]
    allsame = np.full(100, -1.5, np.float32)
    assert list(select(hs, allsame, k)) == list(range(30))


def test_topk_skips_nan(hs):
    sim = np.array([-1.0, np.nan, -2.0, -0.5], np.float32)
    assert list(select(hs, sim, 3)) == [3, 0, 2]


def test_similarity_rule_and_ring_rows(hs):
    """(-acc) * shrinkage / 8 in fp32; logical token -> ring row: permanent slot 0, FIFO slots in age order"""
    acc, ms = np.float32(3.7), np.float32(1.9)
    assert hs.hs_similarity(acc, ms) == np.float32(np.float32(-acc * ms) * np.float32(0.125))
    HW = 10
    assert [hs.hs_ring_row(n, HW, 0, 4) for n in (0, 9, 10, 25)] == [0, 9, 10, 25]
    # head 2 of 4 FIFO slots: logical frames 1..4 live in slots 3, 4, 1, 2
    assert [hs.hs_ring_row(f * HW + 1, HW, 2, 4) // HW for f in range(5)] == [0, 3, 4, 1, 2]


def test_oracle_memory_read_matches_dense_reference_formula():
    """the oracle's get_similarity equals the distance form -sum qe (mk - qk)^2 * ms / 8 in float64, and its top-k read
    over all tokens with k = N is the full softmax read"""
    g = torch.Generator().manual_seed(0)
    mk, qk = torch.randn(1, 64, 50, generator=g, dtype=torch.float64), torch.randn(1, 64, 7, generator=g, dtype=torch.float64)
    ms = 1 + torch.rand(1, 1, 50, generator=g, dtype=torch.float64)
    qe = torch.rand(1, 64, 7, generator=g, dtype=torch.float64)
    s = cutie_ref.get_similarity(mk, ms, qk, qe)
    d = -(qe.unsqueeze(2) * (mk.unsqueeze(3) - qk.unsqueeze(2)) ** 2).sum(1) * ms[0, 0].view(1, 50, 1) / 8
    assert torch.allclose(s, d, rtol=1e-12, atol=1e-10)
    v = torch.randn(1, 2, 256, 50, generator=g, dtype=torch.float64)
    full = cutie_ref.readout(cutie_ref.do_softmax(s), v)
    assert torch.allclose(cutie_ref.memory_read(mk, ms, qk, qe, v, 50, torch.float64), full, rtol=1e-10, atol=1e-12)
    sel = torch.arange(50).view(1, 50).expand(7, 50)
    assert torch.allclose(cutie_ref.readout_selected(mk, ms, qk, qe, v, sel)[None], full, rtol=1e-10, atol=1e-12)
