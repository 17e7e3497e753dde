"""Argument checks of RAFT's GRU / motion-pack / lookup entry points, called through the C ABI with fake device addresses.

Every one of these kernels moves 4 channels per access (float4 for fp32 rows, 8 bytes for fp16 rows), so an entry point
must refuse a pointer that is off by 2 elements with PP_ERR_ALIGN, and it must do so before it touches CUDA.  On a machine
without a CUDA device that makes the test safe and sharp: a refused call returns PP_ERR_ALIGN, while a call that slipped
past its checks reaches the launch and comes back with a launch error, never with a fault.  For the same reason the test
is skipped where a device is present: there a missing check would launch a kernel on addresses that do not exist.  The
GPU side (tests/test_gpu_half_kernels_f64.py) repeats the refusals with real misaligned views.

An empty call (npix = 0) must return PP_OK without a launch: a zero-block grid is an invalid launch configuration whose
error would stay pending for the next, unrelated kernel.
"""
import ctypes

import pytest
import torch

PP_OK, PP_ERR_SHAPE, PP_ERR_ALIGN = 0, -1, -5
F32, F16 = 4, 2

pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason="fake device addresses are only safe without a CUDA device")


@pytest.fixture(scope="module")
def L():
    import __graft_entry__ as g
    g.build()
    from propainter_b200 import _lib
    return _lib.lib()


def _addr(k):
    """a 256-byte aligned fake device address, distinct per argument slot"""
    return (1 << 40) + (k << 24)


# entry -> (pointer arguments as (name, element bytes), build(ptrs, npix) -> argument tuple); flow is read per element
# and has no alignment requirement beyond its own type
def _gate(f16):
    def build(p, npix, ld=256):
        return (p["zr"], p["bias"], p["pre"], p["net"], ld, p["z"], p["rnet"], ld, npix, 128, None)
    e = F16 if f16 else F32
    return [("zr", e), ("bias", F32), ("pre", F32), ("net", F32), ("z", F32), ("rnet", e)], build


def _update(f16):
    if f16:
        def build(p, npix, ld=256):
            return (p["q"], p["bias"], p["pre"], p["z"], p["net"], ld, p["h_img"], ld, p["net_copy"], npix, 128, None)
        return [("q", F16), ("bias", F32), ("pre", F32), ("z", F32), ("net", F32), ("h_img", F16), ("net_copy", F16)], build

    def build(p, npix, ld=256):
        return (p["q"], p["bias"], p["pre"], p["z"], p["net"], ld, p["net_copy"], npix, 128, None)
    return [("q", F32), ("bias", F32), ("pre", F32), ("z", F32), ("net", F32), ("net_copy", F32)], build


def _pack(f16):
    def build(p, npix, ld=256):
        return (p["mot"], ld, p["bias"], _addr(30) + 4, p["d0"], p["d1"], ld, npix, None)
    e = F16 if f16 else F32
    return [("mot", e), ("bias", F32), ("d0", e), ("d1", e)], build


def _bias_act(x_f16, out_f16):
    def build(p, npix, ld=256):
        return (p["x"], ld, x_f16, p["bias"], p["pre"], ld, p["res"], ld, p["out"], ld, out_f16, npix, 128, 1, 0.0, 0, None)
    return [("x", F16 if x_f16 else F32), ("bias", F32), ("pre", F32), ("res", F32), ("out", F16 if out_f16 else F32)], build


ENTRIES = {
    "pp_gru_gate": _gate(False), "pp_gru_gate_f16": _gate(True),
    "pp_gru_update": _update(False), "pp_gru_update_f16": _update(True),
    "pp_raft_pack_motion": _pack(False), "pp_raft_pack_motion_f16": _pack(True),
    "pp_bias_act_f16[x16,out16]": _bias_act(1, 1), "pp_bias_act_f16[x16,out32]": _bias_act(1, 0),
    "pp_bias_act_f16[x32,out16]": _bias_act(0, 1), "pp_bias_act_f16[x32,out32]": _bias_act(0, 0),
}


def _aligned(ptrs):
    return {name: _addr(k) for k, (name, _) in enumerate(ptrs)}


@pytest.mark.parametrize("entry", sorted(ENTRIES))
def test_misaligned_pointer_is_refused_before_launch(L, entry):
    """each pointer off by 2 elements (8 bytes fp32, 4 bytes fp16) -> PP_ERR_ALIGN; the aligned call is not refused"""
    ptrs, build = ENTRIES[entry]
    fn = getattr(L, entry.split("[")[0])
    base = _aligned(ptrs)
    for name, esize in ptrs:
        p = dict(base)
        p[name] += 2 * esize
        assert fn(*build(p, 1)) == PP_ERR_ALIGN, (entry, name)
    # the same call with every pointer aligned passes the checks and fails only at the launch (no device here)
    assert fn(*build(base, 1)) not in (PP_OK, PP_ERR_ALIGN, PP_ERR_SHAPE), entry


@pytest.mark.parametrize("entry", sorted(ENTRIES))
def test_stride_not_multiple_of_4_is_refused(L, entry):
    ptrs, build = ENTRIES[entry]
    assert getattr(L, entry.split("[")[0])(*build(_aligned(ptrs), 1, ld=258)) == PP_ERR_ALIGN, entry


@pytest.mark.parametrize("entry", sorted(ENTRIES))
def test_empty_input_returns_ok_without_launch(L, entry):
    ptrs, build = ENTRIES[entry]
    assert getattr(L, entry.split("[")[0])(*build(_aligned(ptrs), 0)) == PP_OK, entry


@pytest.mark.parametrize("name", ["pp_corr_lookup", "pp_corr_lookup_ldg", "pp_corr_lookup_f16", "pp_corr_lookup_ldg_f16"])
def test_corr_lookup_shape_checks_and_empty_input(L, name):
    """n_pairs = 0 -> PP_OK before any tensor map is encoded or kernel launched; fp16 rows narrower than the 324 taps and
    feature grids below 16 x 16 are refused"""
    fn = getattr(L, name)
    levels = (ctypes.c_void_p * 4)(*[_addr(k) for k in range(4)])
    f16 = name.endswith("_f16")

    def call(n_pairs, h=30, w=54, ld_out=328):
        extra = (ld_out,) if f16 else ()
        return fn(levels, _addr(5), _addr(6), *extra, n_pairs, h, w, None)
    assert call(0) == PP_OK
    assert call(3, h=15) == PP_ERR_SHAPE and call(3, w=15) == PP_ERR_SHAPE
    if f16:
        assert call(3, ld_out=320) == PP_ERR_SHAPE and call(0, ld_out=323) == PP_ERR_SHAPE
        assert call(3, ld_out=324) not in (PP_OK, PP_ERR_ALIGN, PP_ERR_SHAPE)
