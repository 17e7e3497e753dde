"""Argument checks of the fp16 entry points of the propagation scans (pp_conv2d_umma_f16, pp_conv2d_umma_plan_f16,
pp_deform_gather_f16, pp_flow_warp_fbcheck_f16), called through the C ABI with fake device addresses.

fp16 rows feed TMA tensor maps and 8- / 16-byte vector stores, so every fp16 row must start 16-byte aligned with a row stride
of a multiple of 8 halves; a misaligned view must be refused with PP_ERR_ALIGN before anything touches CUDA.  As in
tests/test_half_abi_host.py the test is skipped where a device is present: a missing check would there launch a kernel
on addresses that do not exist.  tests/test_gpu_half_scans.py repeats the refusals with real views.
"""
import ctypes

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
    """a 256-byte aligned fake device address, distinct per argument slot"""
    return (1 << 40) + (k << 24)


def _conv(segC, ld=None, KH=3, Cout=128, H=30, W=54, out=True):
    from propainter_b200._lib import PPConvParams
    p = PPConvParams()
    p.nseg = len(segC)
    for i, C in enumerate(segC):
        p.seg[i].x, p.seg[i].ld, p.seg[i].C = _addr(i), ld if ld is not None else (C + 7) // 8 * 8, C
    p.n, p.H, p.W, p.KH, p.KW, p.Cout = 1, H, W, KH, KH, Cout
    p.w_packed = _addr(8)
    p.bias, p.pre, p.ld_pre, p.res, p.ld_res = _addr(9), _addr(10), Cout, _addr(11), Cout
    p.out, p.ld_out = (_addr(12), Cout) if out else (None, 0)
    p.act, p.slope = 2, 0.1
    return p


def _plan(L, fn, p):
    v = [ctypes.c_int(0) for _ in range(5)]
    rc = getattr(L, fn)(ctypes.byref(p), *[ctypes.byref(x) for x in v])
    return rc, [x.value for x in v]


def test_conv_f16_plan_works_in_64_channel_blocks(L):
    """a 1x1 conv over 256 channels is 8 TF32 blocks (grouped 4 per stage) but 4 fp16 blocks (ungrouped): the two plans
    differ in their rings; the deformable GEMMs (1152 / 2304 columns) group in both"""
    rc32, p32 = _plan(L, "pp_conv2d_umma_plan", _conv([256], KH=1))
    rc16, p16 = _plan(L, "pp_conv2d_umma_plan_f16", _conv([256], KH=1))
    assert rc32 == PP_OK and rc16 == PP_OK and p32[:4] == p16[:4] and p32[4] != p16[4]
    for C in (1152, 2304):
        rc, p = _plan(L, "pp_conv2d_umma_plan_f16", _conv([C], KH=1))
        assert rc == PP_OK and p == _plan(L, "pp_conv2d_umma_plan", _conv([C], KH=1))[1]
    # 3x3 over two 128-channel fp16 states: the same tile and ring as TF32 (the rings are sized in bytes)
    assert _plan(L, "pp_conv2d_umma_plan_f16", _conv([128, 128])) == _plan(L, "pp_conv2d_umma_plan", _conv([128, 128]))


def test_conv_f16_refuses_misaligned_segments(L):
    # ld 132 halves: a multiple of 4 (fine for fp32 rows) but not of 8
    assert _plan(L, "pp_conv2d_umma_plan_f16", _conv([128], ld=132))[0] == PP_ERR_ALIGN
    assert _plan(L, "pp_conv2d_umma_plan", _conv([128], ld=132))[0] == PP_OK
    p = _conv([128, 64])
    p.seg[1].x += 8                                                    # 4 halves off
    assert _plan(L, "pp_conv2d_umma_plan_f16", p)[0] == PP_ERR_ALIGN
    assert L.pp_conv2d_umma_f16(ctypes.byref(p), _addr(13), 128, None) == PP_ERR_ALIGN


def test_conv_f16_out16_checks(L):
    p = _conv([128])
    assert L.pp_conv2d_umma_f16(ctypes.byref(p), _addr(13) + 8, 128, None) == PP_ERR_ALIGN
    assert L.pp_conv2d_umma_f16(ctypes.byref(p), _addr(13), 132, None) == PP_ERR_ALIGN
    q = _conv([128], out=False)
    assert L.pp_conv2d_umma_f16(ctypes.byref(q), None, 0, None) == PP_ERR_SHAPE      # nothing to write
    # fp32 out only, fp16 out16 only, both: past every check, failing only at the launch (no device here)
    for prm, o16 in ((p, None), (q, _addr(13)), (p, _addr(13))):
        assert L.pp_conv2d_umma_f16(ctypes.byref(prm), o16, 128 if o16 else 0, None) not in (PP_OK, PP_ERR_ALIGN, PP_ERR_SHAPE)


def test_deform_gather_f16_checks(L):
    def call(cols, Cin=128, ld_x=128):
        return L.pp_deform_gather_f16(_addr(0), ld_x, None, 0, _addr(1), 432, None, _addr(2), 3.0, cols, 1, 60, 108, Cin, None)
    assert call(_addr(3) + 8) == PP_ERR_ALIGN                          # fp16 columns 8 bytes off
    assert call(_addr(3), ld_x=130) == PP_ERR_ALIGN
    assert call(_addr(3), Cin=192) == PP_ERR_SHAPE
    assert call(_addr(3)) not in (PP_OK, PP_ERR_ALIGN, PP_ERR_SHAPE)


def test_flow_warp_f16_checks(L):
    def call(warped, ld_w=128, ld_f=128):
        return L.pp_flow_warp_fbcheck_f16(_addr(0), ld_f, _addr(1), None, warped, ld_w, None, 0, 1, 60, 108, 128, None)
    assert call(_addr(3) + 8) == PP_ERR_ALIGN
    assert call(_addr(3), ld_w=132) == PP_ERR_ALIGN                    # fp16 rows: ld % 8
    assert call(_addr(3), ld_f=130) == PP_ERR_ALIGN
    assert call(None) == PP_ERR_SHAPE                                  # neither warped nor aux
    assert call(_addr(3)) not in (PP_OK, PP_ERR_ALIGN, PP_ERR_SHAPE)
