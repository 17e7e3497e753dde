"""CPU tests of scripts/compute_flow.py's port: the host build of the frame-preparation rule (pp_resize_coord /
pp_u8_frame_resized, k_u8_to_frames_resized's per-element code) against ATen's F.interpolate and pp_u8_frame, the oracle's
RAFT against the fixture the unmodified scripts made (tests/golden/make_golden_compute_flow.py), the flow-completion
protocol's text, and the argument checks that need no device.  The kernel and the device runs are tested in
test_gpu_compute_flow.py."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import raft_ref
from propainter_b200 import schemas
from propainter_b200._params import ParamNet
from tests.compute_flow_inputs import GOLD_NAME, VIDEOS, video_inputs

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", GOLD_NAME + ".npz")

# (T, H0, W0, h, w): the sizes the rule was first checked at, odd source sizes, T > 1
EXACT_SIZES = [(1, 720, 1280, 240, 432), (1, 480, 854, 240, 432), (1, 144, 176, 240, 432), (1, 240, 432, 240, 432),
               (1, 200, 240, 128, 160), (1, 96, 120, 128, 160), (3, 37, 53, 128, 160), (3, 97, 131, 128, 160),
               (2, 333, 517, 240, 432), (2, 101, 77, 128, 136), (2, 1080, 1920, 240, 432)]


@pytest.fixture(scope="module")
def hs(tmp_path_factory):
    lib = str(tmp_path_factory.mktemp("hostsim_compute_flow") / "libhostsim_compute_flow.so")
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", lib,
                           os.path.join(HERE, "hostsim", "hostsim_compute_flow.cpp")])
    return ctypes.CDLL(lib)


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLD))


def random_frames(T, H0, W0, seed):
    return torch.from_numpy(np.random.default_rng(seed).integers(0, 256, (T, H0, W0, 3), dtype=np.uint8))


def hostsim_frames(hs, u8, h, w):
    T, H0, W0, _ = u8.shape
    out = torch.empty(T, 3, h, w)
    hs.hs_u8_to_frames_resized(ctypes.c_void_p(u8.data_ptr()), ctypes.c_void_p(out.data_ptr()), T, H0, W0, h, w)
    return out


def aten_frames(u8, h, w):
    """compute_flow.py:67-92 on ATen's CPU kernels: ToTensor (contiguous CHW, / 255), bilinear resize, *2 then -1"""
    img = u8.permute(0, 3, 1, 2).contiguous().float().div(255)
    img = F.interpolate(input=img, size=(h, w), mode='bilinear', align_corners=False)
    img = img * 2
    return img - 1


@pytest.mark.parametrize("T,H0,W0,h,w", EXACT_SIZES, ids=[f"{c[0]}x{c[1]}x{c[2]}-{c[3]}x{c[4]}" for c in EXACT_SIZES])
def test_rule_bit_exact_with_aten_cpu(hs, T, H0, W0, h, w):
    u8 = random_frames(T, H0, W0, H0 * W0 + h)
    assert torch.equal(hostsim_frames(hs, u8, h, w), aten_frames(u8, h, w))


def test_rule_near_aten_at_small_outputs(hs):
    """outputs far below RAFT's sizes go through another ATen code path: a few ulp from the rule (measured <= 3.6e-7)"""
    for T, H0, W0, h, w in [(2, 101, 77, 24, 40), (2, 5, 3, 17, 19), (1, 1, 1, 7, 9), (1, 209, 218, 74, 48)]:
        u8 = random_frames(T, H0, W0, w)
        assert (hostsim_frames(hs, u8, h, w) - aten_frames(u8, h, w)).abs().max().item() <= 2.0 ** -21


def test_rule_at_identity_is_u8_frame(hs):
    u8 = random_frames(2, 37, 53, 3)
    ref = torch.empty(2, 37, 53, 3)
    hs.hs_u8_frame(ctypes.c_void_p(u8.data_ptr()), ctypes.c_void_p(ref.data_ptr()), ctypes.c_long(u8.numel()))
    assert torch.equal(hostsim_frames(hs, u8, 37, 53), ref.permute(0, 3, 1, 2))
    all_values = torch.arange(256, dtype=torch.uint8).reshape(1, 1, 256, 1).expand(1, 1, 256, 3).contiguous()
    want = torch.empty(1, 1, 256, 3)
    hs.hs_u8_frame(ctypes.c_void_p(all_values.data_ptr()), ctypes.c_void_p(want.data_ptr()), ctypes.c_long(768))
    assert torch.equal(hostsim_frames(hs, all_values, 1, 256), want.permute(0, 3, 1, 2))


def fp16_excess(got, ref16):
    """the largest |got - ref| beyond half an fp16 ulp of ref (the rounding flowwrite applied), relative to max |ref|"""
    ref = ref16.astype(np.float32)
    ulp = np.spacing(np.abs(ref16)).astype(np.float32)
    excess = np.maximum(np.abs(got - ref) - 0.5 * ulp, 0)
    return float(excess.max() / np.abs(ref).max())


def test_oracle_reproduces_script_flows(gold):
    """oracle/raft_ref on ATen-resized frames against the .flo contents compute_flow.py wrote: within the `gt` tolerance
    test_oracle_golden.py holds the oracle to (1e-5 of the flow scale), beyond the fp16 rounding of the file, on the
    fixture's every-4th-pixel subsample"""
    sd = ParamNet(schemas.raft_schema(), seed=1).state_dict()
    h, w = int(gold["size"][1]), int(gold["size"][0])
    for name, T, mask, seed, native in VIDEOS:
        u8, _ = video_inputs(T, mask, seed, native)
        frames = aten_frames(torch.from_numpy(u8), h, w)[None]
        with torch.no_grad():
            fw, bw = raft_ref.raft_bi(sd, frames, int(gold["raft_iter"]))
        for got, key in ((fw[0], "flow_f"), (bw[0], "flow_b")):
            e = fp16_excess(got[..., ::4, ::4].numpy(), gold[f"{name}_{key}_sub4"])
            print(f"{name} {key}: {e:.2e}")
            assert e < 1e-5, (name, key, e)


def script_lines(gold):
    return str(gold["summary"]).strip().split("\n")


def test_protocol_lines_from_fixture_numbers(gold):
    from propainter_b200.evaluate import flow_completion_video_line, flow_epe_summary
    lines = script_lines(gold)
    n = len(gold["names"])
    assert len(lines) == n + 1
    recs = []
    for i, name in enumerate(gold["names"]):
        ef, eb = (float(x) for x in gold[f"{name}_epe"])
        avg_time = float(lines[i].rsplit("Time: ", 1)[1])
        epe = float((np.float32(ef) + np.float32(eb)) / 2)
        assert flow_completion_video_line(i, n, str(name), epe, avg_time) == lines[i]
        recs.append({"epe_forward": ef, "epe_backward": eb, "frames": int(gold["lengths"][i]), "seconds": 0.0})
    s = flow_epe_summary(recs)
    t = float(lines[-1].rsplit("Time: ", 1)[1])
    assert f'Finish evaluation... Average Frame EPE: {s["epe"]:.4f} | | Time: {t:.4f}' == lines[-1]


def test_value_errors_without_device():
    from propainter_b200 import ops
    from propainter_b200.evaluate import compute_flow_video, evaluate_flow_completion
    u8 = torch.zeros(3, 64, 64, 3, dtype=torch.uint8)
    for size in ((432, 244), (436, 240), (120, 240), (432, 120), (0, 0)):
        with pytest.raises(ValueError):
            compute_flow_video(None, u8, size)
    for bad in (u8[:1], u8[..., :2], u8.float(), u8[0]):
        with pytest.raises(ValueError):
            compute_flow_video(None, bad, (160, 128))
    for bad in (u8.float(), u8[..., :1], u8[0], u8[:0]):
        with pytest.raises(ValueError):
            ops.u8_to_frames_resized(bad, (32, 32))
    for size in ((0, 32), (32, 0), (-8, 16)):
        with pytest.raises(ValueError):
            ops.u8_to_frames_resized(u8, size)
    masks = np.zeros((3, 64, 64), np.uint8)
    with pytest.raises(ValueError):
        evaluate_flow_completion(None, [("a", masks, (np.zeros((2, 2, 64, 64), np.float32),) * 2), ("b", masks, None)])
