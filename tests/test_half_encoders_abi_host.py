"""Argument checks of pp_bias_act_f16_res (the epilogue of RAFT's half-operand context encoder: fp16 x, residual and out),
called through the C ABI with fake device addresses.

fp16 rows are read and written as 8-byte vectors and the bias as 16-byte vectors, so a misaligned row or bias, or a row
stride that is not a multiple of 4, must be refused with PP_ERR_ALIGN, a row stride below C or an unknown activation with
PP_ERR_SHAPE, before anything touches CUDA.  As in tests/test_half_abi_host.py the test is skipped where a device is
present: a missing check would there launch a kernel on addresses that do not exist.
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


def _call(L, x=_addr(0), ld_x=64, bias=_addr(1), res=_addr(2), ld_res=64, out=_addr(3), ld_out=64, n_pix=0, C=64, act=1):
    return L.pp_bias_act_f16_res(x, ld_x, bias, res, ld_res, out, ld_out, n_pix, C, act, 0.0, 1, None)


def test_bias_act_f16_res_accepts_aligned_views(L):
    assert _call(L) == PP_OK
    assert _call(L, res=None) == PP_OK
    assert _call(L, x=_addr(0) + 8, out=_addr(3) + 8, res=_addr(2) + 8, ld_x=68, ld_out=132) == PP_OK


@pytest.mark.parametrize("arg", [dict(x=_addr(0) + 2), dict(out=_addr(3) + 4), dict(res=_addr(2) + 6), dict(bias=_addr(1) + 8),
                                 dict(ld_x=66), dict(ld_out=66), dict(ld_res=70), dict(C=66, ld_x=68, ld_out=68, ld_res=68)])
def test_bias_act_f16_res_refuses_misalignment(L, arg):
    assert _call(L, **arg) == PP_ERR_ALIGN


@pytest.mark.parametrize("arg", [dict(ld_x=60), dict(ld_out=60), dict(ld_res=60), dict(act=5), dict(act=-1)])
def test_bias_act_f16_res_refuses_bad_shapes(L, arg):
    assert _call(L, **arg) == PP_ERR_SHAPE

