"""Records the C calls propainter_b200.ops makes over a fixed set of cases and writes them to ops_call_trace.json.

A recording stand-in takes the place of the loaded library (_lib._lib): it launches nothing, returns 0 (a fixed size
for the *_workspace_bytes queries) and logs every call with its symbol and arguments as the C side sees them: scalars
converted to their declared types, and each device-call pointer as [input, byte offset] for the case's inputs, "newK"
for the K-th tensor the wrapper allocated itself, "stream" for the launch stream or null, plus the fields of the
parameter structs.  Per case the trace also holds the change of ops.LAUNCHES and the returned tensors' shape, dtype
and strides (or the exception raised).  Pointers of host-side calls (the resampling tables) are only "ptr" / null:
they point at host memory the wrapper frees again.  The wrappers refuse CPU tensors, so the cases need a CUDA device,
but no kernel runs.  tests/test_gpu_ops_trace.py replays the cases on the current tree and compares.

    PYTHONPATH=<tree whose ops is recorded> python tests/golden/make_ops_trace.py
"""
import ctypes
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.append(ROOT)                       # after PYTHONPATH: the package under test may come from another tree
from propainter_b200 import _lib, ops  # noqa: E402

TRACE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ops_call_trace.json")
WS_BYTES = 4096
FAIL_CODE = 7
DEVICE = "cuda"
F32, F16, I32, U8 = torch.float32, torch.float16, torch.int32, torch.uint8
_INTS = (ctypes.c_int, ctypes.c_long, ctypes.c_size_t)


class Inputs:
    """Zero-filled CUDA tensors of one case, by name (views of them resolve to the name and a byte offset).  Each is
    held to the end of the case, so no later tensor of the case can reuse its memory."""

    def __init__(self):
        self.named = []

    def __call__(self, name, *shape, dtype=F32):
        x = torch.zeros(shape, dtype=dtype, device=DEVICE)
        self.named.append((name, x.untyped_storage().data_ptr(), x.untyped_storage().nbytes(), x))
        return x

    def find(self, p):
        for name, base, n, _ in self.named:
            if base <= p < base + max(n, 1):
                return [name, p - base]
        return None


class Recorder:
    """Stands in for the loaded library: logs each call, returns 0 (or FAIL_CODE for the device call `fail_at`)."""

    def __init__(self, inputs, stream, fail_at=None):
        self.inputs, self.stream, self.fail_at = inputs, stream, fail_at
        self.calls, self.new, self.device_calls = [], {}, 0

    def __getattr__(self, symbol):
        if symbol.startswith("__"):
            raise AttributeError(symbol)
        return lambda *args: self._call(symbol, args)

    def _call(self, symbol, args):
        if symbol == "pp_error_string":
            return b"stand-in error"
        types = _lib.SIGNATURES[symbol][1]
        if len(args) != len(types):
            raise TypeError(f"{symbol}: {len(args)} arguments, the signature has {len(types)}")
        device = len(args) > 0 and isinstance(args[-1], ctypes.c_void_p) and args[-1].value == self.stream
        self.calls.append([symbol] + [self._arg(a, ty, device) for a, ty in zip(args, types)])
        if symbol.endswith("_workspace_bytes"):
            return WS_BYTES
        if device:
            self.device_calls += 1
            if self.device_calls - 1 == self.fail_at:
                return FAIL_CODE
        return 0

    def _ptr(self, p, device):
        p = p.value if isinstance(p, ctypes.c_void_p) else p
        if p is None or p == 0:
            return None
        if not device:
            return "ptr"
        if p == self.stream:
            return "stream"
        return self.inputs.find(p) or self.new.setdefault(p, f"new{len(self.new)}")

    def _arg(self, a, ty, device):
        if isinstance(a, ctypes.Array):
            return [self._arg(e, a._type_, device) for e in a]
        if type(a).__name__ == "CArgObject":                      # ctypes.byref(...)
            a = a._obj
        if isinstance(a, ctypes.Structure):
            return {f: self._arg(getattr(a, f), t, device) for f, t in a._fields_}
        if isinstance(a, ctypes._SimpleCData) and not isinstance(a, ctypes.c_void_p):
            ty, a = type(a), a.value
        if ty in _INTS:
            return int(a)
        if ty in (ctypes.c_float, ctypes.c_double):
            return ty(a).value
        return self._ptr(a, device)


def _result(r, inputs):
    if isinstance(r, torch.Tensor):
        return {"shape": list(r.shape), "dtype": str(r.dtype), "stride": list(r.stride()),
                "of": inputs.find(r.data_ptr()) if r.numel() else None}
    if isinstance(r, (tuple, list)):
        return [_result(x, inputs) for x in r]
    return r if r is None or isinstance(r, (int, float)) else repr(r)


def run_case(fn, fail_at=None):
    """One case under the stand-in on a side stream -> (trace entry, Recorder)."""
    saved = _lib._lib
    ops._TABLES.clear()
    ops._PAINT_PALETTE.clear()
    stream = torch.cuda.Stream()
    inputs = Inputs()
    rec = Recorder(inputs, stream.cuda_stream, fail_at)
    _lib._lib = rec
    l0 = ops.LAUNCHES
    try:
        with torch.cuda.stream(stream):
            try:
                out = {"returns": _result(fn(inputs), inputs)}
            except (RuntimeError, ValueError) as e:
                out = {"raises": [type(e).__name__, str(e)]}
        torch.cuda.synchronize()
    finally:
        _lib._lib = saved
    out.update(calls=rec.calls, launches=ops.LAUNCHES - l0)
    return out, rec


# ---------------------------------------------------------------- the cases: every branch of every public wrapper
CASES = {}


def case(fn):
    CASES[fn.__name__] = fn
    return fn


def _levels(t, n=2, h=8, w=8):
    return [t(f"lv{i}", n * h * w, h >> i, ops.corr_ld(w >> i)) for i in range(4)]


def _otf(t, B=2):
    return (t("fmap", 2, 64, 256), [t(f"pool{i}", 2, 64 >> (2 * i), 256) for i in (1, 2, 3)], t("idx1", B, dtype=I32),
            t("idx2", B, dtype=I32), t("coords", B, 8, 8, 2))


@case
def corr_alloc(t):
    return ops.corr_alloc(2, 8, 8, DEVICE)


@case
def corr_build(t):
    return ops.corr_build(t("fmap", 2, 64, 256), t("idx1", 2, dtype=I32), t("idx2", 2, dtype=I32), _levels(t), 8, 8)


@case
def corr_lookup(t):
    return ops.corr_lookup(_levels(t), t("coords", 2, 8, 8, 2))


@case
def corr_lookup_ldg_out(t):
    return ops.corr_lookup(_levels(t), t("coords", 2, 8, 8, 2), t("out", 2, 8, 8, 324), tma=False)


@case
def corr_lookup_f16(t):
    return ops.corr_lookup(_levels(t), t("coords", 2, 8, 8, 2), t("out", 2, 8, 8, 336, dtype=F16))


@case
def corr_lookup_f16_ldg(t):
    return ops.corr_lookup(_levels(t), t("coords", 2, 8, 8, 2), t("out", 2, 8, 8, 328, dtype=F16), tma=False)


@case
def corr_fmap_pyramid(t):
    return ops.corr_fmap_pyramid(t("fmap", 2, 64, 256), 8, 8)


@case
def corr_lookup_otf(t):
    return ops.corr_lookup_otf(*_otf(t))


@case
def corr_lookup_otf_out(t):
    return ops.corr_lookup_otf(*_otf(t), out=t("out", 2, 8, 8, 324))


@case
def corr_lookup_otf_bad_batch(t):
    return ops.corr_lookup_otf(*_otf(t, B=3)[:4], t("coords", 2, 8, 8, 2))


@case
def corr_lookup_r3(t):
    return ops.corr_lookup_r(_levels(t), t("coords", 2, 8, 8, 2), 3)


@case
def corr_lookup_r4_ldg_out(t):
    return ops.corr_lookup_r(_levels(t), t("coords", 2, 8, 8, 2), 4, t("out", 2, 8, 8, 324), tma=False)


@case
def corr_lookup_r3_ldg(t):
    return ops.corr_lookup_r(_levels(t), t("coords", 2, 8, 8, 2), 3, tma=False)


@case
def corr_lookup_otf_r3(t):
    return ops.corr_lookup_otf_r(*_otf(t), 3)


@case
def corr_lookup_otf_r4_out(t):
    return ops.corr_lookup_otf_r(*_otf(t), 4, t("out", 2, 8, 8, 324))


@case
def corr_lookup_otf_r_bad_batch(t):
    return ops.corr_lookup_otf_r(*_otf(t, B=1)[:4], t("coords", 2, 8, 8, 2), 3)


@case
def upflow8(t):
    return ops.upflow8(t("flow", 2, 4, 4, 2))


@case
def convex_upsample(t):
    return ops.convex_upsample(t("mask", 2, 4, 4, 600)[..., :576], t("flow", 2, 4, 4, 2), 0.5)


@case
def img_prop_scan(t):
    return ops.img_prop_scan(t("frames", 3, 3, 8, 8), t("ff", 2, 2, 8, 8), t("fb", 2, 2, 8, 8), t("masks", 3, 1, 8, 8))


@case
def img_prop_scan_bilinear(t):
    return ops.img_prop_scan(t("frames", 3, 3, 8, 8), t("ff", 2, 2, 8, 8), t("fb", 2, 2, 8, 8), t("masks", 3, 1, 8, 8),
                             nearest=False)


def _u8h(t, lo, hi, n):
    return (t("frames", 4, 8, 8, 3, dtype=U8), t("masks", 4, 1, 8, 8), t("ff", 3, 2, 8, 8, dtype=F16), t("fb", 3, 2, 8, 8, dtype=F16),
            t("of", n, 3, 8, 8, dtype=F16), t("om", n, 1, 8, 8, dtype=F16), lo, hi)


@case
def img_prop_scan_u8h(t):
    return ops.img_prop_scan_u8h(*_u8h(t, 0, None, 4))


@case
def img_prop_scan_u8h_band(t):
    return ops.img_prop_scan_u8h(*_u8h(t, 1, 3, 2), nearest=False)


@case
def img_prop_scan_u8h_empty(t):
    return ops.img_prop_scan_u8h(*_u8h(t, 2, 2, 0))


@case
def img_prop_scan_u8h_bad_out(t):
    return ops.img_prop_scan_u8h(*_u8h(t, 0, 2, 3))


@case
def prop_cond(t):
    fe = t("feats", 8, 8, 64)
    return ops.prop_cond(fe[..., :16], fe[..., 16:32], t("fprop", 8, 8, 2), t("fcheck", 8, 8, 2), t("mcur", 8, 8, 2),
                         t("cond", 8, 8, 48)[..., :40], t("bb", 8, 8, 32), False)


@case
def prop_cond_first(t):
    return ops.prop_cond(t("cur", 8, 8, 16), None, t("fprop", 8, 8, 2), t("fcheck", 8, 8, 2), t("mcur", 8, 8, 2), None,
                         t("bb", 8, 8, 32)[..., :20], True)


@case
def deform_align(t):
    return ops.deform_align(t("x", 8, 8, 64), t("o", 8, 8, 440)[..., :432], t("flow", 8, 8, 2), 3.0, t("w", 576, 128),
                            t("bias", 128), t("out", 8, 8, 256)[..., 128:])


@case
def deform_align_no_flow(t):
    return ops.deform_align(t("x", 8, 8, 64), t("o", 8, 8, 432), None, 5, t("w", 576, 128), t("bias", 128), t("out", 8, 8, 128),
                            o_bias=t("ob", 432))


@case
def packing(t):
    w = torch.arange(16 * 40 * 9, dtype=F32, device=DEVICE).reshape(16, 40, 3, 3) * 1e-3
    return (ops.tf32_round(w), ops.pack_conv_weight(w), ops.pack_conv_weight(w, [8, 32]), ops.pack_conv_weight_f16(w),
            ops.pack_deform_weight_umma(w), ops.pack_deform_weight_umma_f16(w), ops.pack_deform_weight(w))


@case
def conv_umma(t):
    return ops.conv_umma([t("x", 2, 8, 8, 8)], t("w", 16, 9 * 32), 3, 3, 16)


@case
def conv_umma_epilogue(t):
    x = t("x", 2, 8, 8, 64)
    return ops.conv_umma([x[..., :8], x[..., 8:48]], t("w", 16, 3 * 32), 1, 1, 16, bias=t("bias", 16), act="leaky", slope=0.1,
                         pre=t("pre", 2, 8, 8, 16), res=t("res", 2, 8, 8, 32)[..., 16:], post_relu=True,
                         out=t("out", 2, 8, 8, 24)[..., :16], round_tf32=True, bn=16, tile_w=8, tile_m=64)


@case
def conv_umma_bad_weight(t):
    return ops.conv_umma([t("x", 2, 8, 8, 8)], t("w", 16, 9 * 64), 3, 3, 16)


@case
def conv_umma_too_many_segs(t):
    return ops.conv_umma([t(f"x{i}", 1, 4, 4, 8) for i in range(5)], t("w", 16, 5 * 32), 1, 1, 16)


@case
def conv_umma_f16(t):
    return ops.conv_umma_f16([t("x", 2, 8, 8, 8, dtype=F16)], t("w", 16, 9 * 64, dtype=F16), 3, 3, 16)


@case
def conv_umma_f16_out32(t):
    return ops.conv_umma_f16([t("x", 2, 8, 8, 8, dtype=F16), t("y", 2, 8, 8, 72, dtype=F16)], t("w", 16, 3 * 64, dtype=F16), 1, 1,
                             16, bias=t("bias", 16), act="relu", pre=t("pre", 2, 8, 8, 16), out=t("out", 2, 8, 8, 16), bn=16)


@case
def conv_umma_f16_both(t):
    return ops.conv_umma_f16([t("x", 2, 8, 8, 16, dtype=F16)[..., :8]], t("w", 16, 64, dtype=F16), 1, 1, 16, res=t("res", 2, 8, 8, 16),
                             act="sigmoid", out=t("out", 2, 8, 8, 16), out16=t("o16", 2, 8, 8, 32, dtype=F16)[..., 16:], tile_w=8)


@case
def conv_umma_f16_bad_out16(t):
    return ops.conv_umma_f16([t("x", 2, 8, 8, 8, dtype=F16)], t("w", 16, 64, dtype=F16), 1, 1, 16, out16=t("o16", 2, 8, 8, 8, dtype=F16))


@case
def conv_plan(t):
    return ops.conv_plan([t("x", 2, 8, 8, 8)], 3, 3, 16, bn=16, out=t("out", 2, 8, 8, 16), bias=t("bias", 16))


@case
def conv_plan_f16_shapes(t):
    return ops.conv_plan([(2, 8, 8, 8), (2, 8, 8, 70)], 3, 3, 16, tile_w=8, half=True)


def _gather(t, n=2):
    return t("x", n, 8, 8, 16), t("o", n, 8, 8, 448)[..., :432]


@case
def deform_gather(t):
    return ops.deform_gather(*_gather(t), t("flow", 2, 8, 8, 2), 3.0)


@case
def deform_gather_x2_f16(t):
    x, o = _gather(t)
    return ops.deform_gather(x, o, None, 2, cols=t("cols", 2, 8, 8, 9 * 32, dtype=F16), o_bias=t("ob", 432), x2=t("x2", 2, 8, 8, 16))


@case
def deform_gather_cols(t):
    return ops.deform_gather(*_gather(t), t("flow", 2, 8, 8, 2), 1.5, cols=t("cols", 2, 8, 8, 9 * 16))


@case
def deform_gather_bad_x2(t):
    x, o = _gather(t)
    return ops.deform_gather(x, o, None, 2, x2=t("x2", 2, 8, 8, 8))


@case
def flow_warp(t):
    return ops.flow_warp_fbcheck(t("feat", 2, 8, 8, 32)[..., :16], t("fprop", 2, 8, 8, 2))


@case
def flow_warp_fbcheck(t):
    return ops.flow_warp_fbcheck(t("feat", 2, 8, 8, 16), t("fprop", 2, 8, 8, 2), t("fcheck", 2, 8, 8, 2), round_tf32=True)


@case
def flow_warp_fbcheck_f16(t):
    return ops.flow_warp_fbcheck(t("feat", 2, 8, 8, 16), t("fprop", 2, 8, 8, 2), t("fcheck", 2, 8, 8, 2),
                                 warped=t("warped", 2, 8, 8, 32, dtype=F16)[..., 16:], aux=t("aux", 2, 8, 8, 8)[..., :4])


@case
def flow_warp_f16_tf32(t):
    return ops.flow_warp_fbcheck(t("feat", 2, 8, 8, 16), t("fprop", 2, 8, 8, 2), warped=t("warped", 2, 8, 8, 16, dtype=F16),
                                 round_tf32=True)


@case
def fbcheck_only(t):
    return ops.flow_warp_fbcheck(None, t("fprop", 2, 8, 8, 2), t("fcheck", 2, 8, 8, 2), want_warp=False)


@case
def gen_prep(t):
    return ops.gen_prep(t("ff", 2, 2, 16, 16), t("fb", 2, 2, 16, 16), t("mi", 3, 1, 16, 16), t("mu", 4, 1, 16, 16), 3)


@case
def gen_prep_f16(t):
    return ops.gen_prep(t("ff", 2, 2, 16, 16, dtype=F16), t("fb", 2, 2, 16, 16, dtype=F16), t("mi", 3, 1, 16, 16),
                        t("mu", 3, 1, 16, 16), 3)


@case
def gen_prep_one_frame(t):
    return ops.gen_prep(t("ff", 0, 2, 16, 16), t("fb", 0, 2, 16, 16), t("mi", 1, 1, 16, 16), t("mu", 1, 1, 16, 16), 1)


@case
def window_mask(t):
    return ops.window_mask(t("pmask", 3, 8, 8, 2), 2, 2, 2, 2)


def _attn(t, dt, T=2, NT=16, C=512):
    return (t("qkv", T, NT, 3 * C, dtype=dt), t("pool", T, 4, 2 * C, dtype=dt), t("ktab", 4, 9, dtype=I32), t("flags", 4, dtype=I32))


@case
def sparse_window_attn(t):
    return ops.sparse_window_attn(*_attn(t, F32), 2, 16, 0, 2)


@case
def sparse_window_attn_mma(t):
    return ops.sparse_window_attn(*_attn(t, F32), 2, 16, 1, 1, impl="mma")


@case
def sparse_window_attn_f16(t):
    return ops.sparse_window_attn(*_attn(t, F16), 2, 16, 0, 1, impl="mma")


@case
def sparse_window_attn_no_keys_out(t):
    return ops.sparse_window_attn(*_attn(t, F32), 2, 16, 2, 2, out=t("out", 2, 16, 1024)[..., :512], WN=20)


@case
def sparse_window_attn_small_c(t):
    return ops.sparse_window_attn(*_attn(t, F16, C=256), 2, 16, 0, 3, C=256)


@case
def ffn_overlap_add(t):
    return ops.ffn_overlap_add(t("Y", 4, 49 * 40), 1, 6, 6)


@case
def ffn_overlap_add_f16(t):
    return ops.ffn_overlap_add(t("Y", 4, 49 * 8, dtype=F16), 1, 6, 6, CH=8)


def _gru(t, dt):
    hx, rx = t("hx", 2, 4, 4, 384, dtype=dt), t("rx", 2, 4, 4, 384, dtype=dt)
    return hx, rx, t("state", 2, 4, 4, 256)[..., :128]


@case
def gru_gate(t):
    hx, rx, _ = _gru(t, F32)
    return ops.gru_gate(t("zr", 2, 4, 4, 256), t("bias", 256), hx[..., :128], t("z", 2, 4, 4, 128), rx[..., :128])


@case
def gru_gate_pre(t):
    hx, rx, _ = _gru(t, F32)
    return ops.gru_gate(t("zr", 2, 4, 4, 256), t("bias", 256), hx[..., :128], t("z", 2, 4, 4, 128), rx[..., 128:256],
                        pre=t("pre", 2, 4, 4, 256))


@case
def gru_gate_f16(t):
    _, rx, state = _gru(t, F16)
    return ops.gru_gate(t("zr", 2, 4, 4, 256, dtype=F16), t("bias", 256), state, t("z", 2, 4, 4, 128), rx[..., :128],
                        pre=t("pre", 2, 4, 4, 256))


@case
def gru_gate_f16_no_pre(t):
    _, rx, state = _gru(t, F16)
    return ops.gru_gate(t("zr", 2, 4, 4, 256, dtype=F16), t("bias", 256), state, t("z", 2, 4, 4, 128), rx[..., :128])


@case
def gru_update(t):
    hx, _, _ = _gru(t, F32)
    return ops.gru_update(t("q", 2, 4, 4, 128), t("bias", 128), t("z", 2, 4, 4, 128), hx[..., :128])


@case
def gru_update_copy_pre(t):
    hx, _, _ = _gru(t, F32)
    return ops.gru_update(t("q", 2, 4, 4, 128), t("bias", 128), t("z", 2, 4, 4, 128), hx[..., 128:256],
                          net_copy=t("copy", 2, 4, 4, 128), pre=t("pre", 2, 4, 4, 128))


@case
def gru_update_f16(t):
    hx, _, state = _gru(t, F16)
    return ops.gru_update(t("q", 2, 4, 4, 128, dtype=F16), t("bias", 128), t("z", 2, 4, 4, 128), state,
                          net_copy=t("copy", 2, 4, 4, 128, dtype=F16), pre=t("pre", 2, 4, 4, 128), h_img=hx[..., :128])


@case
def gru_update_f16_no_img(t):
    _, _, state = _gru(t, F16)
    return ops.gru_update(t("q", 2, 4, 4, 128, dtype=F16), t("bias", 128), t("z", 2, 4, 4, 128), state)


@case
def gru_update_f32_img(t):
    hx, _, state = _gru(t, F16)
    return ops.gru_update(t("q", 2, 4, 4, 128), t("bias", 128), t("z", 2, 4, 4, 128), state, h_img=hx[..., :128])


@case
def raft_pack_motion(t):
    hx, rx, _ = _gru(t, F32)
    return ops.raft_pack_motion(t("mot", 2, 4, 4, 128), t("flow", 2, 4, 4, 2), hx[..., 256:], rx[..., 256:], bias=t("bias", 128))


@case
def raft_pack_motion_f16(t):
    hx, rx, _ = _gru(t, F16)
    return ops.raft_pack_motion(t("mot", 2, 4, 4, 256, dtype=F16)[..., :128], t("flow", 2, 4, 4, 2), hx[..., 256:], rx[..., 256:])


@case
def raft_pack_motion_bad_ld(t):
    hx, _, _ = _gru(t, F32)
    return ops.raft_pack_motion(t("mot", 2, 4, 4, 128), t("flow", 2, 4, 4, 2), hx[..., 256:], t("rx", 2, 4, 4, 128))


@case
def raft_pack_motion_n(t):
    hx, rx, _ = _gru(t, F32)
    return ops.raft_pack_motion_n(t("mot", 2, 4, 4, 96), t("flow", 2, 4, 4, 2), hx[..., 256:340], rx[..., 256:340], 82,
                                  bias=t("bias", 96))


@case
def raft_pack_motion_n_small(t):
    hx, rx, _ = _gru(t, F32)
    return ops.raft_pack_motion_n(t("mot", 2, 4, 4, 96), t("flow", 2, 4, 4, 2), hx[..., 256:336], rx[..., 256:336], 82)


@case
def bias_act_inplace(t):
    return ops.bias_act(t("x", 2, 4, 4, 32)[..., :16], t("bias", 16), "relu")


@case
def bias_act_pre(t):
    return ops.bias_act(t("x", 2, 4, 4, 16), t("bias", 16), "leaky", 0.2, pre=t("pre", 2, 4, 4, 32)[..., 16:],
                        out=t("out", 2, 4, 4, 16))


@case
def bias_act_res(t):
    return ops.bias_act(t("x", 2, 4, 4, 16), None, "tanh", res=t("res", 2, 4, 4, 16), post_relu=True, out=t("out", 2, 4, 4, 16))


@case
def bias_act_f16_in(t):
    return ops.bias_act(t("x", 2, 4, 4, 16, dtype=F16), t("bias", 16), "sigmoid", out=t("out", 2, 4, 4, 16))


@case
def bias_act_f16_out(t):
    return ops.bias_act(t("x", 2, 4, 4, 16), t("bias", 16), "relu", res=t("res", 2, 4, 4, 16), pre=t("pre", 2, 4, 4, 16),
                        out=t("out", 2, 4, 4, 32, dtype=F16)[..., 16:], post_relu=True)


@case
def bias_act_f16_inplace(t):
    return ops.bias_act(t("x", 2, 4, 4, 16, dtype=F16), t("bias", 16))


@case
def bias_act_f16_res(t):
    return ops.bias_act(t("x", 2, 4, 4, 16, dtype=F16), t("bias", 16), "relu", res=t("res", 2, 4, 4, 16, dtype=F16),
                        out=t("out", 2, 4, 4, 16, dtype=F16), post_relu=True)


@case
def bias_act_f16_res_f32_x(t):
    return ops.bias_act(t("x", 2, 4, 4, 16), t("bias", 16), res=t("res", 2, 4, 4, 16, dtype=F16), out=t("out", 2, 4, 4, 16, dtype=F16))


@case
def bias_act_bad_dtype(t):
    return ops.bias_act(t("x", 2, 4, 4, 16, dtype=F16), None, out=t("out", 2, 4, 4, 16, dtype=torch.float64))


@case
def bias_act_shape_mismatch(t):
    return ops.bias_act(t("x", 2, 4, 4, 16), None, out=t("out", 2, 4, 4, 8))


@case
def bias_act_(t):
    return ops.bias_act_(t("x", 2, 4, 4, 16), t("bias", 16), "leaky", 0.1)


@case
def sc_fold(t):
    return ops.sc_fold(t("cols", 8, 49 * 8 + 8, dtype=F16)[:, :49 * 8], t("bmap", 6, 6, 8), 2, 6, 6)


@case
def sc_fold_out(t):
    return ops.sc_fold(t("cols", 4, 49 * 8, dtype=F16), t("bmap", 6, 6, 8), 1, 6, 6, out=t("out", 1, 6, 6, 8, dtype=F16))


@case
def sc_fold_bad(t):
    return ops.sc_fold(t("cols", 5, 49 * 8, dtype=F16), t("bmap", 6, 6, 8), 1, 6, 6)


@case
def pool_depthwise(t):
    return ops.pool_depthwise(t("x", 1, 8, 8, 32)[..., :16], t("w", 4, 16), t("bias", 16), 2, 2)


@case
def pool_depthwise_f16(t):
    return ops.pool_depthwise(t("x", 1, 9, 8, 16, dtype=F16), t("w", 6, 16), t("bias", 16), 3, 2)


@case
def add_layernorm(t):
    return ops.add_layernorm(t("x", 8, 64), t("d", 8, 64), t("g", 64), t("b", 64))


@case
def add_layernorm_first(t):
    return ops.add_layernorm(t("x", 8, 64), None, t("g", 64), t("b", 64), eps=1e-6)


@case
def add_layernorm_f16_delta(t):
    return ops.add_layernorm(t("x", 8, 64), t("d", 8, 64, dtype=F16), t("g", 64), t("b", 64), y_dtype=F16)


@case
def add_layernorm_f16_y(t):
    return ops.add_layernorm(t("x", 8, 64), t("d", 8, 64), t("g", 64), t("b", 64), y_dtype=F16)


@case
def add_layernorm_first_f16_y(t):
    return ops.add_layernorm(t("x", 8, 64), None, t("g", 64), t("b", 64), y_dtype=F16)


@case
def instance_norm(t):
    return ops.instance_norm(t("x", 2, 4, 4, 16))


@case
def instance_norm_res(t):
    return ops.instance_norm(t("x", 2, 4, 4, 16), relu=True, res=t("res", 2, 4, 4, 16), post_relu=True, eps=1e-3,
                             out=t("out", 2, 4, 4, 16))


@case
def upsample2x(t):
    return ops.upsample2x(t("x", 2, 4, 4, 16))


@case
def upsample2x_f16(t):
    return ops.upsample2x(t("x", 2, 4, 4, 16, dtype=F16))


@case
def mask_dilate(t):
    return ops.mask_dilate(t("m", 2, 8, 8, dtype=U8), 3)


@case
def u8_to_frames(t):
    return ops.u8_to_frames(t("f", 2, 8, 8, 3, dtype=U8))


@case
def u8_to_frames_resized(t):
    return ops.u8_to_frames_resized(t("f", 2, 8, 8, 3, dtype=U8), (12, 10))


@case
def u8_to_frames_resized_bad(t):
    return ops.u8_to_frames_resized(t("f", 2, 8, 8, 3, dtype=U8), (0, 10))


def _blend(t, comp_dtype):
    return (t("pred", 2, 3, 8, 8), t("masks", 4, 1, 8, 8), t("ori", 4, 8, 8, 3, dtype=U8), t("comp", 4, 8, 8, 3, dtype=comp_dtype),
            [0, 2], [True, False])


@case
def composite_blend(t):
    return ops.composite_blend(*_blend(t, U8))


@case
def composite_blend_f32(t):
    return ops.composite_blend_f32(*_blend(t, F32))


@case
def composite_blend_f32_bad(t):
    return ops.composite_blend_f32(*_blend(t, U8))


@case
def extrapolate_u8(t):
    return ops.extrapolate_u8(t("f", 2, 8, 8, 3, dtype=U8), ((12, 14), (2, 3), (1, 2)))


@case
def mask_overlay_u8(t):
    return ops.mask_overlay_u8(t("f", 2, 8, 8, 3, dtype=U8), t("m", 1, 2, 1, 8, 8))


@case
def flow_to_image_u8(t):
    return ops.flow_to_image_u8(t("flow", 2, 2, 8, 8))


@case
def flow_to_image_u8_clip(t):
    return ops.flow_to_image_u8(t("flow", 2, 8, 8), "clip", clip_flow=5, bgr=True)


@case
def flow_occlusion(t):
    return ops.flow_occlusion(t("fw", 2, 2, 8, 8), t("bw", 2, 2, 8, 8))


@case
def flow_occlusion_f16(t):
    return ops.flow_occlusion(t("fw", 1, 2, 2, 8, 8, dtype=F16), t("bw", 2, 2, 8, 8, dtype=F16))


@case
def warp_error_sums_occ(t):
    return ops.warp_error_sums(t("f", 3, 8, 8, 3, dtype=U8), t("fw", 2, 2, 8, 8), occ=t("occ", 2, 8, 8, dtype=U8))


@case
def warp_error_sums_bw(t):
    return ops.warp_error_sums(t("f", 3, 8, 8, 3, dtype=U8), t("fw", 2, 2, 8, 8, dtype=F16), bw=t("bw", 1, 2, 2, 8, 8, dtype=F16))


@case
def warp_error(t):
    return ops.warp_error(t("f", 3, 8, 8, 3, dtype=U8), t("fw", 2, 2, 8, 8), bw=t("bw", 2, 2, 8, 8))


@case
def i3d_input_u8(t):
    return ops.i3d_input(t("v", 1, 4, 8, 8, 3, dtype=U8))


@case
def i3d_input_f32(t):
    return ops.i3d_input(t("v", 1, 3, 5, 9, 8))


@case
def maxpool3d_same(t):
    return ops.maxpool3d_same(t("x", 1, 4, 8, 8, 8), (3, 3, 3), (2, 2, 2))


@case
def maxpool3d_same_out(t):
    return ops.maxpool3d_same(t("x", 1, 4, 8, 8, 16)[..., :8], (1, 3, 3), (1, 2, 2), out=t("out", 1, 4, 4, 4, 24)[..., 8:16])


@case
def mean_thw(t):
    return ops.mean_thw(t("x", 2, 2, 4, 4, 16)[..., :8])


@case
def resample_tables(t):
    return [ops.resample_tables(k, 8, 12, DEVICE, h) for k, h in
            (("bicubic", True), ("nearest", True), ("linear_cv", False), ("linear_f32", True))]


@case
def resize_frames_u8(t):
    return ops.resize_frames_u8(t("f", 2, 8, 8, 3, dtype=U8), (12, 10))


@case
def resize_masks_u8(t):
    return ops.resize_masks_u8(t("m", 2, 8, 8, dtype=U8), (12, 10))


@case
def resize_output_u8(t):
    return ops.resize_output_u8(t("f", 2, 8, 8, 3, dtype=U8), (12, 10))


@case
def resize_flow(t):
    return ops.resize_flow(t("flow", 2, 2, 8, 8), (12, 10))


def _cutie(t, nobj=2):
    return (t("key", 3 * 16, 64), t("shrink", 3 * 16), t("value", nobj, 3 * 16, 256), 2, 1, 2, t("qk", 64, 16), t("qe", 64, 16))


@case
def cutie_topk_readout(t):
    return ops.cutie_topk_readout(*_cutie(t), top_k=8)


@case
def cutie_topk_readout_selection(t):
    return ops.cutie_topk_readout(*_cutie(t, 3), top_k=30, num_objects=2, out=t("out", 2, 16, 256), want_selection=True)


@case
def cutie_topk_readout_bad_k(t):
    return ops.cutie_topk_readout(*_cutie(t), top_k=33)


@case
def cutie_frame_in(t):
    return ops.cutie_frame_in(t("f", 10, 12, 3, dtype=U8))


@case
def cutie_labels(t):
    return ops.cutie_labels(t("prob", 3, 16, 16), t("lut", 3, dtype=U8), 10, 12, out=t("out", 10, 12, dtype=U8))


@case
def mask_paint_u8(t):
    return ops.mask_paint_u8(t("f", 2, 8, 8, 3, dtype=U8), t("l", 2, 8, 8, dtype=U8))


@case
def mask_paint_u8_palette(t):
    f = t("f", 2, 8, 8, 3, dtype=U8)
    return ops.mask_paint_u8(f, t("l", 2, 8, 8, dtype=U8), palette=np.zeros((4, 3), np.uint8), mask_alpha=0.5, out=f)


def record():
    return {name: run_case(fn)[0] for name, fn in CASES.items()}


if __name__ == "__main__":
    if not torch.cuda.is_available():
        sys.exit("make_ops_trace: needs a CUDA device (the wrappers refuse CPU tensors; no kernel runs)")
    trace = record()
    with open(TRACE, "w") as f:
        json.dump(trace, f, indent=None, separators=(",", ":"))
        f.write("\n")
    print(f"{len(trace)} cases, {sum(len(c['calls']) for c in trace.values())} calls -> {TRACE}")
