"""Half-precision clip storage (InferenceConfig.half_storage) without a device.

- The stage-3 scan on clip storage (pp_img_prop_scan_u8h) compiled for the host by tests/hostsim/hostsim_half.cpp: its
  fp16 outputs must equal the fp32 host scan (hs_img_prop_scan) run on the u8-widened masked frames and the upcast fp16
  flows, composited in the order of ProPainterPipeline.propagate_images and rounded to nearest-even fp16, bit for bit.
- The argument checks of the two new entry points (pp_img_prop_scan_u8h, pp_gen_prep_f16) through the C ABI with fake
  device addresses, in the pattern of tests/test_half_abi_host.py: refused calls return before touching CUDA, an empty call
  returns PP_OK without a launch, and a call that passes its checks fails only at the launch (no device here).
- The option's surfaces that need no device: its default and the sharded runner's refusal.
"""
import ctypes
import os
import subprocess

import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
PP_OK, PP_ERR_SHAPE, PP_ERR_WORKSPACE, PP_ERR_ALIGN = 0, -1, -3, -5
FP = ctypes.POINTER(ctypes.c_float)


@pytest.fixture(scope="module")
def hs(tmp_path_factory):
    lib = str(tmp_path_factory.mktemp("hostsim_half") / "libhostsim_half.so")
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", lib,
                           os.path.join(HERE, "hostsim", "hostsim_half.cpp")])
    h = ctypes.CDLL(lib)
    h.hs_float_to_half.restype, h.hs_float_to_half.argtypes = ctypes.c_uint16, [ctypes.c_float]
    h.hs_half_to_float.restype, h.hs_half_to_float.argtypes = ctypes.c_float, [ctypes.c_uint16]
    return h


def _fp(t):
    assert t.dtype == torch.float32 and t.is_contiguous()
    return ctypes.cast(t.data_ptr(), FP)


def _vp(t):
    assert t.is_contiguous()
    return ctypes.c_void_p(t.data_ptr())


def test_host_fp16_conversions_match_torch(hs):
    """the host build's fp16 rules: widening every binary16 pattern, and round-to-nearest-even on ties, subnormals, the
    overflow edge, infinities and random values, against torch's conversions"""
    bits = torch.arange(0, 1 << 16, dtype=torch.int32).to(torch.int16)
    ref = bits.view(torch.float16).float()
    got = torch.tensor([hs.hs_half_to_float(int(b) & 0xFFFF) for b in bits.tolist()])
    same = (got == ref) | (torch.isnan(got) & torch.isnan(ref))
    assert bool(same.all())
    crafted = [0.0, -0.0, 1.0 + 2 ** -11, 1.0 + 3 * 2 ** -11, 2 ** -25, 3 * 2 ** -25, 2 ** -24 * 1.5, 6.1e-5, 65504.0,
               65519.99, 65520.0, -65520.0, float("inf"), float("-inf"), 1e-8, -1e-8]
    vals = torch.tensor(crafted + (torch.randn(4000, generator=torch.Generator().manual_seed(0)) * 3).tolist())
    ref16 = vals.half().view(torch.int16).to(torch.int32) & 0xFFFF
    got16 = torch.tensor([hs.hs_float_to_half(float(v)) for v in vals.tolist()], dtype=torch.int32)
    assert torch.equal(got16, ref16)


def _smooth_flow(gen, n, H, W, amp=4.0):
    z = torch.randn(n, 2, H // 8 + 2, W // 8 + 2, generator=gen) * amp
    return F.interpolate(z, size=(H, W), mode="bicubic", align_corners=False).contiguous()


def _clip(seed, T, H, W):
    gen = torch.Generator().manual_seed(seed)
    u8 = torch.randint(0, 256, (T, H, W, 3), dtype=torch.uint8, generator=gen)
    if T == 1:
        ff = fb = torch.zeros(0, 2, H, W)
    else:
        ff = _smooth_flow(gen, T - 1, H, W)
        fb = -ff + 0.3 * _smooth_flow(gen, T - 1, H, W)
    masks = torch.zeros(T, 1, H, W)
    masks[..., H // 4:3 * H // 4, W // 5:3 * W // 4] = 1
    masks[::2, :, :3, :5] = 1                                # holes that touch the border on every other frame
    return u8, ff.half().contiguous(), fb.half().contiguous(), masks


@pytest.mark.parametrize("T,H,W,lo,hi", [(6, 40, 56, 0, 6), (9, 24, 32, 3, 7), (7, 24, 32, 0, 4), (5, 16, 24, 2, 5),
                                         (1, 16, 16, 0, 1)])
@pytest.mark.parametrize("nearest", [1, 0])
def test_clip_storage_scan_equals_fp32_scan_rounded(hostsim, hs, T, H, W, lo, hi, nearest):
    """the kept frames [lo, hi) of the clip-storage scan are rn16 of the fp32 path, bit for bit"""
    u8, ff16, fb16, masks = _clip(T * 100 + H, T, H, W)
    frames = torch.empty(T, 3, H, W)
    hostsim.hs_u8_to_frames(ctypes.c_void_p(u8.data_ptr()), _fp(frames), T, H, W)
    masked = (frames * (1 - masks)).contiguous()
    ff, fb = ff16.float().contiguous(), fb16.float().contiguous()
    if T == 1:
        ff = fb = torch.zeros(1)
    prop, um = torch.empty(T, 3, H, W), torch.empty(T, 1, H, W)
    hostsim.hs_img_prop_scan(_fp(masked), _fp(ff), _fp(fb), _fp(masks), _fp(prop), _fp(um), T, H, W, nearest)
    upd = frames * (1 - masks) + prop * masks               # ProPainterPipeline.propagate_images' compose
    ref_f, ref_m = upd[lo:hi].half(), um[lo:hi].half()

    of = torch.full((hi - lo, 3, H, W), 0x7E00, dtype=torch.int16)    # NaN-filled: every element must be written
    om = torch.full((hi - lo, 1, H, W), 0x7E00, dtype=torch.int16)
    hs.hs_img_prop_scan_u8h(_vp(u8), _fp(masks), _vp(ff16), _vp(fb16), _vp(of), _vp(om), T, H, W, lo, hi, nearest)
    assert torch.equal(of, ref_f.view(torch.int16))
    assert torch.equal(om, ref_m.view(torch.int16))
    assert set(om.view(torch.float16).unique().tolist()) <= {0.0, 1.0}
    if T > 1:
        assert 0 < (um[lo:hi] < masks[lo:hi]).float().mean()    # the propagation really fills pixels


# ---------------------------------------------------------------- C ABI argument checks
pytestmark_abi = pytest.mark.skipif(torch.cuda.is_available(), reason="fake device addresses are only safe without a CUDA device")


@pytest.fixture(scope="module")
def L():
    import __graft_entry__ as g
    g.build()
    from propainter_b200 import _lib
    return _lib.lib()


def _addr(k):
    return (1 << 40) + (k << 24)


SCAN_PTRS = ["frames_u8", "masks", "flows_f", "flows_b", "out_frames", "out_masks", "workspace"]


def _scan(L, t=5, H=16, W=24, lo=0, hi=None, ws=None, off=None):
    p = {n: _addr(k) for k, n in enumerate(SCAN_PTRS)}
    for n, d in (off or {}).items():
        p[n] += d
    hi = t if hi is None else hi
    ws = L.pp_img_prop_scan_u8h_workspace_bytes(t, H, W) if ws is None else ws
    return L.pp_img_prop_scan_u8h(*[p[n] for n in SCAN_PTRS], ws, t, H, W, lo, hi, 1, None)


@pytestmark_abi
def test_scan_u8h_argument_checks(L):
    assert L.pp_img_prop_scan_u8h_workspace_bytes(3, 4, 5) == 5 * 4 * 4 * 5 * 4       # (t + 2) frames of 3 + 1 floats
    for name in ("flows_f", "flows_b", "out_frames", "out_masks"):                   # fp16: 2-byte aligned
        assert _scan(L, off={name: 1}) == PP_ERR_ALIGN, name
        assert _scan(L, off={name: 2}) not in (PP_OK, PP_ERR_ALIGN, PP_ERR_SHAPE), name
    for name in ("masks", "workspace"):                                              # fp32: 4-byte aligned
        assert _scan(L, off={name: 2}) == PP_ERR_ALIGN, name
    assert _scan(L, off={"frames_u8": 1}) not in (PP_OK, PP_ERR_ALIGN, PP_ERR_SHAPE)  # bytes: any address
    for kw in (dict(H=1), dict(W=1), dict(t=-1, hi=0), dict(lo=-1), dict(lo=3, hi=2), dict(hi=6), dict(t=0, hi=1)):
        assert _scan(L, **kw) == PP_ERR_SHAPE, kw
    assert _scan(L, off={"flows_f": 1}, lo=3, hi=2) == PP_ERR_SHAPE                    # shapes are checked first
    assert _scan(L, ws=L.pp_img_prop_scan_u8h_workspace_bytes(5, 16, 24) - 4) == PP_ERR_WORKSPACE
    # empty calls: nothing kept -> PP_OK without a launch (also with no workspace at all, and for an empty clip)
    assert _scan(L, lo=2, hi=2) == PP_OK and _scan(L, lo=5, hi=5, ws=0) == PP_OK and _scan(L, t=0, hi=0, ws=0) == PP_OK
    # kept ranges that pass the checks reach the launch
    for lo, hi in ((0, 5), (0, 1), (2, 4), (4, 5)):
        assert _scan(L, lo=lo, hi=hi) not in (PP_OK, PP_ERR_ALIGN, PP_ERR_SHAPE), (lo, hi)


GEN_PTRS = ["flows_f", "flows_b", "masks_in", "masks_upd", "dsf", "dsb", "pmask"]


@pytestmark_abi
def test_gen_prep_f16_argument_checks(L):
    def call(lt=3, H=16, W=24, off=None):
        p = {n: _addr(k) for k, n in enumerate(GEN_PTRS)}
        for n, d in (off or {}).items():
            p[n] += d
        return L.pp_gen_prep_f16(*[p[n] for n in GEN_PTRS], lt, H, W, None)
    for name in ("flows_f", "flows_b"):
        assert call(off={name: 1}) == PP_ERR_ALIGN, name
        assert call(off={name: 2}) not in (PP_OK, PP_ERR_ALIGN, PP_ERR_SHAPE), name
    for name in ("masks_in", "masks_upd", "dsf", "dsb", "pmask"):
        assert call(off={name: 2}) == PP_ERR_ALIGN, name
    for kw in (dict(H=18), dict(W=22), dict(lt=0), dict(H=-4)):
        assert call(**kw) == PP_ERR_SHAPE, kw
    assert call(H=0) == PP_OK and call(W=0) == PP_OK                                 # empty frame: no launch
    assert call() not in (PP_OK, PP_ERR_ALIGN, PP_ERR_SHAPE)


# ---------------------------------------------------------------- surfaces
def test_half_storage_is_off_by_default():
    from propainter_b200.inference_propainter import InferenceConfig
    assert InferenceConfig().half_storage is False
    assert InferenceConfig(fp16=True).half_storage is False          # --fp16 keeps its meaning


def test_sharded_runner_rejects_half_storage():
    from propainter_b200.dist import ShardedProPainter
    from propainter_b200.inference_propainter import InferenceConfig
    runner = object.__new__(ShardedProPainter)                       # the option is refused before any rank state is read
    u8 = torch.zeros(4, 16, 16, 3, dtype=torch.uint8)
    m = torch.zeros(1, 4, 1, 16, 16)
    with pytest.raises(ValueError, match="half_storage"):
        runner(u8, m, m, InferenceConfig(half_storage=True))
