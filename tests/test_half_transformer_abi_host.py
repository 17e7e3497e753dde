"""Argument checks of the transformer's half-operand entry points (pp_ffn_overlap_add_f16, pp_add_layernorm_f16), called
through the C ABI with fake device addresses.

fp16 rows are read 8 halves (16 bytes) at a time per row start, so a pointer off by one fp16 pair or a row stride that is
not a multiple of 8 must come back as PP_ERR_ALIGN before anything touches CUDA, and an empty call must return PP_OK without
a launch.  Skipped where a device is present, for the reason tests/test_half_abi_host.py gives: there a missing check would
launch a kernel on addresses that do not exist.
"""
import pytest
import torch

PP_OK, PP_ERR_SHAPE, PP_ERR_ALIGN = 0, -1, -5

pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason="fake device addresses are only safe without a CUDA device")


@pytest.fixture(scope="module")
def L():
    import __graft_entry__ as g
    g.build()
    from propainter_b200 import _lib
    return _lib.lib()


def _addr(k):
    return (1 << 40) + (k << 24)


def test_ffn_overlap_add_f16_contract(L):
    Y, Z, ws = _addr(1), _addr(2), _addr(3)
    call = lambda y, ldy, z, ldz, frames: L.pp_ffn_overlap_add_f16(y, ldy, z, ldz, frames, 60, 108, 40, ws, 1 << 30, None)
    assert call(Y + 4, 1960, Z, 1960, 2) == PP_ERR_ALIGN
    assert call(Y, 1960, Z + 8, 1960, 2) == PP_ERR_ALIGN
    assert call(Y, 1964, Z, 1964, 2) == PP_ERR_ALIGN
    assert call(Y, 1952, Z, 1960, 2) == PP_ERR_SHAPE
    assert L.pp_ffn_overlap_add_f16(Y, 1960, Z, 1960, 2, 60, 108, 40, ws + 4, 1 << 30, None) == PP_ERR_ALIGN
    assert call(Y, 1960, Z, 1960, 0) == PP_OK


@pytest.mark.parametrize("delta_f16,y_f16", [(0, 1), (1, 0), (1, 1)])
def test_add_layernorm_f16_contract(L, delta_f16, y_f16):
    x, d, g, b, xo, y = (_addr(k) for k in range(1, 7))
    call = lambda x, d, xo, y, rows: L.pp_add_layernorm_f16(x, d, delta_f16, g, b, xo, y, y_f16, rows, 512, 1e-5, None)
    assert call(x, d, xo, y + 8, 10) == PP_ERR_ALIGN
    assert call(x, d + 8, xo, y, 10) == PP_ERR_ALIGN
    assert call(x + 8, d, xo, y, 10) == PP_ERR_ALIGN
    assert call(x, d, None, y, 10) == PP_ERR_SHAPE
    assert call(x, d, xo, y, 0) == PP_OK
    assert call(x, None, None, y, 0) == PP_OK
