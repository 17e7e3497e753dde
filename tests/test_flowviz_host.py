"""CPU tests of the flow colour coding: oracle/flowviz_ref.py against the fixture produced by the reference's own
flow_to_image functions (tests/golden/make_golden_flowviz.py), the host build of the per-element rules of pp_elem.cuh
against the oracle over a dense sweep, and the argument refusals of the Python layer.  The kernels run on the GPU in
test_gpu_flowviz.py.

Equality criterion: every byte equal, except at pixels whose colour changes when atan2 moves by up to 4 float32 ulps
(numpy's, ATen's and CUDA's atan2 are not correctly rounded); there a byte may differ by one level."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import flowviz_ref

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "flowviz_c1.npz")
U8P = ctypes.POINTER(ctypes.c_uint8)
FP = ctypes.POINTER(ctypes.c_float)

# (fixture key, flow key, normalize, clip_flow key or value, bgr)
FIXTURE_CASES = [("c1_np", "c1_flow", "frame", None, False), ("c1_np_clip_bgr", "c1_flow", "frame", "c1_clip", True),
                 ("c1_pt", "c1_flow", "clip", None, False), ("syn_np", "syn_flow", "frame", None, False),
                 ("syn_np_bgr", "syn_flow", "frame", None, True), ("syn_np_clip", "syn_flow", "frame", 300.0, False),
                 ("syn_pt", "syn_flow", "clip", None, False)]


def fixture_case(g, case):
    key, flow_key, normalize, clip, bgr = case
    clip = float(g[clip]) if isinstance(clip, str) else clip
    return g[flow_key], g[key], normalize, clip, bgr


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


@pytest.fixture(scope="module")
def hs(tmp_path_factory):
    lib = os.path.join(str(tmp_path_factory.mktemp("hostsim_flowviz")), "libhostsim_flowviz.so")
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", lib,
                           os.path.join(HERE, "hostsim", "hostsim_flowviz.cpp")])
    return ctypes.CDLL(lib)


def hs_pixels(hs, u, v, den, variant, bgr=False):
    u, v, den = (np.ascontiguousarray(x, np.float32) for x in (u, v, den))
    out = np.empty(u.shape + (3,), np.uint8)
    hs.hs_flowviz_pixels(u.ctypes.data_as(FP), v.ctypes.data_as(FP), den.ctypes.data_as(FP), out.ctypes.data_as(U8P),
                         ctypes.c_long(u.size), variant, int(bgr))
    return out


def hs_image(hs, flows, normalize, clip_flow=None, bgr=False):
    f = np.ascontiguousarray(flows, np.float32)
    N, _, H, W = f.shape
    out = np.empty((N, H, W, 3), np.uint8)
    hs.hs_flow_to_image_u8(f.ctypes.data_as(FP), out.ctypes.data_as(U8P), N, H, W, 0 if normalize == "frame" else 1,
                           int(clip_flow is not None), ctypes.c_float(clip_flow or 0.0), int(bgr))
    return out


@pytest.mark.parametrize("case", FIXTURE_CASES, ids=[c[0] for c in FIXTURE_CASES])
def test_oracle_reproduces_fixture(gold, case):
    flows, ref, normalize, clip, bgr = fixture_case(gold, case)
    got = flowviz_ref.flow_to_image(flows, normalize, clip, bgr)
    n = flowviz_ref.check_equal(got, flows, normalize, clip, bgr, ref=ref)
    print(f"{case[0]}: {n} pixels differ from the reference, all on a rounding boundary; sensitive set "
          f"{int(flowviz_ref.sensitive(flows, normalize, clip, bgr).sum())} of {ref.size // 3}")


def test_fixture_covers_the_quirks(gold):
    syn = gold["syn_flow"]
    assert (gold["syn_np"][1] == 255).all() and (gold["syn_pt"][1] == 255).all()        # an all-zero frame is white
    rad = np.sqrt(syn[:, 0] ** 2 + syn[:, 1] ** 2)
    den = (rad.reshape(len(syn), -1).max(1) + np.float32(1e-5)).astype(np.float32)
    assert (den[2:] == rad.reshape(len(syn), -1).max(1)[2:]).all()                      # 1e-5 vanishes from 256 px on
    un, vn = syn[:, 0] / den[:, None, None], syn[:, 1] / den[:, None, None]
    over = np.sqrt(un * un + vn * vn) > 1
    assert over[2:].reshape(5, -1).any(1).all() and not over[:2].any()                 # the rad > 1 branch is reached
    g = gold["syn_np"][over]
    assert np.array_equal(g, flowviz_ref.flow_to_image(syn, "frame")[over])
    # torch: the batch maximum (frame 2) normalises above 1; the channel the wheel gives 0 floors to -1 and wraps to 255
    # (numpy's x 0.75 branch keeps it at 0)
    pt, npv = gold["syn_pt"][2][over[2]], gold["syn_np"][2][over[2]]
    assert np.array_equal(pt, flowviz_ref.flow_to_image(syn, "clip")[2][over[2]])
    assert ((pt == 255) & (npv == 0)).any()
    # signed zeros: (+0 or -0, -0) and (+0 or -0, +0) pick wheel ends 0 / 54 -- the first rows of frame 0
    assert (syn[0, 0, 0, :4] == 0).all() and np.array_equal(np.signbit(syn[0, 1, 0, :4]), [False, True, False, True])
    assert np.array_equal(gold["syn_np"][0, 0, :4], flowviz_ref.flow_to_image(syn[:1], "frame")[0, 0, :4])
    assert np.array_equal(gold["syn_np_bgr"], gold["syn_np"][..., ::-1])
    assert not np.array_equal(gold["syn_np_clip"], gold["syn_np"])


def test_colorwheel(hs):
    w = flowviz_ref.colorwheel()
    assert w.shape == (55, 3)
    assert all(hs.hs_colorwheel(k, c) == w[k, c] for k in range(55) for c in range(3))


def _sweep():
    """10^5 angles x radii {0, tiny, 0.5, 1 - ulp, 1, 1 + ulp}, plus both signs of zero on each axis"""
    t = np.linspace(-np.pi, np.pi, 100_000, dtype=np.float64)
    radii = np.array([0.0, 1e-30, 0.5, np.nextafter(np.float32(1), np.float32(0)), 1.0,
                      np.nextafter(np.float32(1), np.float32(2))], np.float32)
    u = (radii[:, None] * np.cos(t)[None]).astype(np.float32).ravel()
    v = (radii[:, None] * np.sin(t)[None]).astype(np.float32).ravel()
    z = [(a, b) for a in (0.0, -0.0) for b in (0.0, -0.0, 1.0, -1.0)] + [(a, b) for a in (1.0, -1.0) for b in (0.0, -0.0)]
    u = np.concatenate([u, np.array([p[0] for p in z], np.float32)])
    v = np.concatenate([v, np.array([p[1] for p in z], np.float32)])
    return u, v


@pytest.mark.parametrize("normalize,bgr", [("frame", False), ("frame", True), ("clip", False), ("clip", True)])
def test_hostsim_rules_dense_sweep(hs, normalize, bgr):
    u, v = _sweep()
    den = np.ones_like(u)                                        # the rule sees the normalised vector itself
    got = hs_pixels(hs, u, v, den, 0 if normalize == "frame" else 1, bgr)
    rule = flowviz_ref.colors_np if normalize == "frame" else flowviz_ref.colors_pt
    ref = rule(u, v, den, bgr)
    bad = np.nonzero((got != ref).any(-1))[0]
    if len(bad):
        sens = np.zeros(len(bad), bool)
        for k in (1, 2, 3, 4):
            for s in (k, -k):
                sens |= (rule(u[bad], v[bad], den[bad], bgr, s) != ref[bad]).any(-1)
        assert sens.all() and np.abs(got[bad].astype(int) - ref[bad].astype(int)).max() <= 1
    print(f"{normalize} bgr={bgr}: {len(bad)} of {len(u)} differ, all on a rounding boundary")
    z = slice(len(u) - 12, None)                                  # signed zeros: bit-exact, no tolerance
    assert np.array_equal(got[z], ref[z])
    assert (got[:100_000] == 255).all()                           # radius 0: white


@pytest.mark.parametrize("normalize,clip,bgr", [("frame", None, False), ("frame", 3.0, True), ("clip", None, True),
                                                ("clip", 2.5, False)])
def test_hostsim_image_matches_oracle(hs, gold, normalize, clip, bgr):
    rng = np.random.default_rng(11)
    flows = np.concatenate([gold["syn_flow"][:, :, :17, :23], rng.standard_normal((3, 2, 17, 23)).astype(np.float32) * 5])
    flowviz_ref.check_equal(hs_image(hs, flows, normalize, clip, bgr), flows, normalize, clip, bgr)


def test_flow_ops_refuse_bad_arguments():
    from propainter_b200 import ops
    with pytest.raises(ValueError):
        ops.flow_to_image_u8(torch.zeros(2, 2, 8, 8, dtype=torch.float16))
    with pytest.raises(ValueError):
        ops.flow_to_image_u8(torch.zeros(2, 2, 8, 8, dtype=torch.float64))
    for shape in ((2, 3, 8, 8), (3, 8, 8), (8, 8), (1, 1, 2, 8, 8)):
        with pytest.raises(ValueError):
            ops.flow_to_image_u8(torch.zeros(shape))
    with pytest.raises(ValueError):
        ops.flow_to_image_u8(torch.zeros(2, 2, 8, 8), normalize="video")
    with pytest.raises(RuntimeError):                            # no CPU path
        ops.flow_to_image_u8(torch.zeros(2, 2, 8, 8))
    with pytest.raises(RuntimeError):
        ops.flow_to_image_u8(torch.zeros(2, 8, 8), normalize="clip")


def test_flow_epe_summary_is_frame_weighted():
    from propainter_b200.evaluate import flow_epe_summary
    rs = [{"frames": 8, "epe_forward": 1.0, "epe_backward": 3.0, "seconds": 0.8},
          {"frames": 3, "epe_forward": 5.0, "epe_backward": 7.0, "seconds": 0.6}]
    # evaluate_flow_completion.py:149-150, 176: each direction's EPE once per flow
    total = [1.0] * 7 + [3.0] * 7 + [5.0] * 2 + [7.0] * 2
    s = flow_epe_summary(rs)
    assert abs(s["epe"] - sum(total) / len(total)) < 1e-12
    assert abs(s["seconds_per_frame"] - (0.8 / 8 * 8 + 0.6 / 3 * 3) / 11) < 1e-12
