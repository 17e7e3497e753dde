"""Tensor-level wrappers over the C ABI.  Each takes/returns torch CUDA tensors, passes raw pointers +
the current stream, and raises on any non-zero return code.  fp32, except the fp16 operand / result tensors of RAFT's
half-precision refinement convs (corr_lookup, bias_act, gru_gate, gru_update, raft_pack_motion) and of the transformer's
half-operand transformer (sparse_window_attn, pool_depthwise, ffn_overlap_add, add_layernorm); DESIGN.md §4 "Precision".  The
half-precision clip storage (img_prop_scan_u8h, gen_prep) reads and writes fp16 tensors between stages; DESIGN.md §7."""
import collections
import ctypes
import math

import numpy as np
import torch

from . import _lib
from ._lib import PPAttnParams, PPConvParams, PPWindowIds, check

LOG2E = 1.4426950408889634

# number of kernels of libpropainter_b200.so launched so far (bench.py reports the delta as gpu_launches)
LAUNCHES = 0


def _count(n):
    global LAUNCHES
    LAUNCHES += n


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _launch(symbol, *args, launches=1):
    """Call the library's `symbol` with args + the current stream, raise naming it if it fails, and count the
    `launches` kernels it enqueues."""
    global LAUNCHES
    check(getattr(_lib.lib(), symbol)(*args, _stream()), symbol)
    LAUNCHES += launches


def _twin(symbol, t):
    """(symbol, fp32) for the rows of tensor t, or (its fp16 twin symbol_f16, fp16) when t is fp16."""
    return (symbol + "_f16", torch.float16) if t.dtype == torch.float16 else (symbol, torch.float32)


def _p(t, dtype=torch.float32):
    if t is None:
        return None
    if not t.is_cuda:
        raise RuntimeError("propainter_b200 ops need CUDA tensors (there is no CPU path)")
    if t.dtype != dtype:
        raise RuntimeError(f"expected {dtype}, got {t.dtype}")
    return ctypes.c_void_p(t.data_ptr())


def _pd(t, dtype=torch.float32):
    """_p of a tensor that must be contiguous."""
    if t is not None and not t.is_contiguous():
        raise RuntimeError("tensor must be contiguous")
    return _p(t, dtype)


def _pm(t, dtype=torch.float32):
    """pixel-major view [..., C] whose pixels are `ld` elements apart -> (ptr, ld)."""
    if t.stride(-1) != 1:
        raise RuntimeError("channel dim must be unit-stride")
    ld = t.stride(-2)
    exp = ld
    for d in range(t.dim() - 2, -1, -1):
        if t.shape[d] != 1 and t.stride(d) != exp:
            raise RuntimeError("pixel-major view must be dense over its pixels")
        exp *= t.shape[d]
    return _p(t, dtype), ld


def corr_ld(w):
    return (w + 3) & ~3


def corr_alloc(n_pairs, h, w, device):
    """Pyramid buffers [n_pairs*h*w, h>>l, ld_l] (zero-filled once so the row padding is defined)."""
    lv, hl, wl = [], h, w
    for _ in range(4):
        lv.append(torch.zeros(n_pairs * h * w, hl, corr_ld(wl), device=device, dtype=torch.float32))
        hl, wl = hl // 2, wl // 2
    return lv


def _level_array(levels):
    return (ctypes.c_void_p * 4)(*[lv.data_ptr() for lv in levels])


def corr_build(fmap, idx1, idx2, levels, h, w):
    """fmap [frames, h*w, D] pixel-major; idx1/idx2 int32 CUDA [n_pairs]; fills the 4 pyramid levels."""
    n_pairs = idx1.numel()
    _launch("pp_corr_build", _pd(fmap), fmap.shape[-1], _p(idx1, torch.int32), _p(idx2, torch.int32), n_pairs, _p(levels[0]),
            h, w)
    _launch("pp_corr_pool_pyramid", _level_array(levels), n_pairs * h * w, h, w, launches=3)


def corr_lookup(levels, coords, out=None, tma=True):
    """coords [B,h,w,2] -> [B,h,w,324].  tma=False selects the plain-load baseline kernel.  An fp16 `out` [B,h,w,ld >= 324]
    receives the taps rounded to nearest in channels [0, 324) of its rows."""
    return _corr_lookup(levels, coords, None, out, tma)


def corr_lookup_r(levels, coords, radius, out=None, tma=True):
    """corr_lookup with window radius 3 (RAFT-small) or 4: coords [B,h,w,2] -> [B,h,w,4*(2*radius+1)**2]."""
    return _corr_lookup(levels, coords, radius, out, tma)


def _corr_lookup(levels, coords, radius, out, tma):
    """radius None: corr_lookup's fixed-radius entries pp_corr_lookup[_ldg][_f16], else pp_corr_lookup[_ldg]_r."""
    B, h, w, _ = coords.shape
    if out is None:
        out = torch.empty(B, h, w, 4 * (2 * (radius or 4) + 1) ** 2, device=coords.device, dtype=torch.float32)
    sym = "pp_corr_lookup" if tma else "pp_corr_lookup_ldg"
    if radius is None and out.dtype == torch.float16:
        _launch(sym + "_f16", _level_array(levels), _pd(coords), _pd(out, torch.float16), out.shape[-1], B, h, w)
    elif radius is None:
        _launch(sym, _level_array(levels), _pd(coords), _pd(out), B, h, w)
    else:
        _launch(sym + "_r", _level_array(levels), radius, _pd(coords), _pd(out), B, h, w)
    return out


def corr_fmap_pyramid(fmap, h, w):
    """fmap [frames, h*w, D] pixel-major -> levels 1-3 of its per-frame 2x2 average-pooled pyramid, each
    [frames, (h>>l)*(w>>l), D]: the stored half of the on-the-fly correlation (AlternateCorrBlock)."""
    F_, _, D = fmap.shape
    pooled = [torch.empty(F_, (h >> l) * (w >> l), D, device=fmap.device, dtype=torch.float32) for l in (1, 2, 3)]
    _launch("pp_corr_fmap_pyramid", _pd(fmap), D, F_, h, w, (ctypes.c_void_p * 3)(*[p.data_ptr() for p in pooled]), launches=3)
    return pooled


def corr_lookup_otf(fmap, pooled, idx1, idx2, coords, out=None):
    """corr_lookup without the all-pairs volume: pair p correlates frame idx1[p] with idx2[p] (int32 CUDA [n_pairs]) of
    fmap [frames, h*w, 256] and its pooled levels (corr_fmap_pyramid) at lookup time.  coords [B,h,w,2] -> [B,h,w,324]."""
    return _corr_lookup_otf(fmap, pooled, idx1, idx2, coords, None, out)


def corr_lookup_otf_r(fmap, pooled, idx1, idx2, coords, radius, out=None):
    """corr_lookup_otf with (D, radius) = (256, 4) or (128, 3): fmap [frames, h*w, D] -> [B,h,w,4*(2*radius+1)**2]."""
    return _corr_lookup_otf(fmap, pooled, idx1, idx2, coords, radius, out)


def _corr_lookup_otf(fmap, pooled, idx1, idx2, coords, radius, out):
    """radius None: pp_corr_lookup_otf (radius 4), else pp_corr_lookup_otf_r."""
    sym, rad = ("pp_corr_lookup_otf", ()) if radius is None else ("pp_corr_lookup_otf_r", (radius,))
    B, h, w, _ = coords.shape
    if idx1.numel() != B or idx2.numel() != B:
        raise RuntimeError(f"{sym[3:]}: one (idx1, idx2) entry per coords batch row")
    if out is None:
        out = torch.empty(B, h, w, 4 * (2 * (radius or 4) + 1) ** 2, device=coords.device, dtype=torch.float32)
    levels = (ctypes.c_void_p * 3)(*[_pd(p).value for p in pooled])
    _launch(sym, _pd(fmap), levels, fmap.shape[-1], *rad, _p(idx1, torch.int32), _p(idx2, torch.int32), B, _pd(coords), _pd(out),
            h, w)
    return out


def upflow8(flow_lr):
    """RAFT-small's upflow8 (RAFT/utils/utils.py:80-82): flow_lr pixel-major [n,h,w,2] -> planar [n,2,8h,8w], bit-exact
    with 8 * F.interpolate(flow, (8h, 8w), mode="bilinear", align_corners=True) on the CPU."""
    n, h, w, _ = flow_lr.shape
    out = torch.empty(n, 2, 8 * h, 8 * w, device=flow_lr.device, dtype=torch.float32)
    _launch("pp_upflow8", _pd(flow_lr), _p(out), n, h, w)
    return out


def convex_upsample(mask_pm, flow_lr, mask_scale=0.25):
    """mask_pm [n,h,w,576] pixel-major, flow_lr [n,h,w,2] -> planar [n,2,8h,8w]."""
    n, h, w, _ = flow_lr.shape
    mp, ld = _pm(mask_pm)
    out = torch.empty(n, 2, 8 * h, 8 * w, device=flow_lr.device, dtype=torch.float32)
    _launch("pp_convex_upsample", mp, ld, mask_scale, _pd(flow_lr), _p(out), n, h, w)
    return out


def img_prop_scan(frames, flows_f, flows_b, masks, nearest=True):
    """frames [t,3,H,W], flows [t-1,2,H,W], masks [t,1,H,W] (planar) -> (frames_out, masks_out)."""
    t, _, H, W = frames.shape
    ws_bytes = _lib.lib().pp_img_prop_scan_workspace_bytes(t, H, W)
    ws = torch.empty(ws_bytes // 4, device=frames.device, dtype=torch.float32)
    of, om = torch.empty_like(frames), torch.empty_like(masks)
    _launch("pp_img_prop_scan", _pd(frames), _pd(flows_f), _pd(flows_b), _pd(masks), _p(of), _p(om), _p(ws), ws_bytes, t, H, W,
            int(bool(nearest)), launches=2 * (t - 1))
    return of, om


def img_prop_scan_u8h(frames_u8, masks, flows_f, flows_b, out_frames, out_masks, lo=0, hi=None, nearest=True):
    """img_prop_scan on half-precision clip storage, composited: frames_u8 uint8 [t,H,W,3], masks float {0,1} [t,1,H,W],
    fp16 flows [t-1,2,H,W].  Writes frames [lo, hi) of frames * (1 - masks) + prop * masks into fp16 out_frames
    [hi-lo,3,H,W] and of the updated masks into fp16 out_masks [hi-lo,1,H,W] (views of clip buffers); the scan is fp32."""
    t, H, W, _ = frames_u8.shape
    hi = t if hi is None else hi
    if tuple(out_frames.shape) != (hi - lo, 3, H, W) or tuple(out_masks.shape) != (hi - lo, 1, H, W):
        raise RuntimeError(f"img_prop_scan_u8h: outputs for frames [{lo}, {hi}) of a {H}x{W} clip, got "
                           f"{tuple(out_frames.shape)} / {tuple(out_masks.shape)}")
    ws_bytes = _lib.lib().pp_img_prop_scan_u8h_workspace_bytes(t, H, W)
    ws = torch.empty(ws_bytes // 4, device=frames_u8.device, dtype=torch.float32)
    f16 = torch.float16
    _launch("pp_img_prop_scan_u8h", _pd(frames_u8, torch.uint8), _pd(masks), _pd(flows_f, f16), _pd(flows_b, f16),
            _pd(out_frames, f16), _pd(out_masks, f16), _p(ws), ws_bytes, t, H, W, lo, hi, int(bool(nearest)),
            launches=t + hi - (lo > 0) if hi > lo else 0)
    return out_frames, out_masks


def prop_cond(cur, prop, fprop, fcheck, mcur, cond, bb, first):
    """cur/prop [h,w,C] pixel-major views; fprop/fcheck/mcur [h,w,2]; cond [h,w,ldc]; bb [h,w,ldb]."""
    h, w, C = cur.shape
    cp, ldc = _pm(cur)
    pp_, ldp = _pm(prop) if prop is not None else (None, ldc)
    cdp, ldcd = _pm(cond) if cond is not None else (None, 2 * C + 8)
    bp, ldb = _pm(bb)
    _launch("pp_prop_cond", cp, ldc, pp_, ldp, _p(fprop), _p(fcheck), _pd(mcur), cdp, ldcd, bp, ldb, h, w, C, int(bool(first)))


def deform_align(x, o, flow, max_res, w_packed, bias, out, o_bias=None):
    """x [H,W,Cin] view, o [H,W,>=432] view (raw conv_offset.6 output; its bias may be passed as o_bias instead of being
    pre-added), flow [H,W,2]|None, out [H,W,128] view (all pixel-major).  The warp-level mma.sync implementation: kept as
    the measured baseline of deform_gather + conv_umma (config.UMMA_CONV)."""
    H, W, Cin = x.shape
    xp, ldx = _pm(x)
    op, ldo = _pm(o)
    outp, ldout = _pm(out)
    ws_bytes = _lib.lib().pp_deform_align_workspace_bytes(H, W)
    ws = torch.empty(max(ws_bytes // 4, 4), device=x.device, dtype=torch.float32)
    _launch("pp_deform_align", xp, ldx, op, ldo, _p(o_bias), _p(flow), float(max_res), _pd(w_packed), _p(bias), outp, ldout, H, W,
            Cin, out.shape[-1], _p(ws), ws_bytes, launches=3)       # tap pre-pass, GEMM, (split-K reduce)
    return out


def tf32_round(w):
    """fp32 -> nearest TF32 value (ties away from zero, = cvt.rna.tf32.f32), still stored as fp32.  wgmma kind tf32
    ignores the low 13 mantissa bits; rounding once at pack time keeps the products unbiased."""
    i = w.contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)


def _pack_conv_blocks(weight, seg_channels, cb):
    Cout, Cin, KH, KW = weight.shape
    seg_channels = [Cin] if seg_channels is None else list(seg_channels)
    if sum(seg_channels) != Cin:
        raise RuntimeError("pack_conv_weight: segments do not add up to Cin")
    blocks, c0 = [], 0
    for C in seg_channels:
        for b in range(0, C, cb):
            cw = min(cb, C - b)
            blk = weight.new_zeros(Cout, KH, KW, cb)
            blk[..., :cw] = weight[:, c0 + b:c0 + b + cw].permute(0, 2, 3, 1)
            blocks.append(blk.reshape(Cout, KH * KW * cb))
        c0 += C
    return torch.cat(blocks, 1).contiguous()


def pack_conv_weight(weight, seg_channels=None):
    """[Cout,Cin,KH,KW] -> [Cout,K] for pp_conv2d_umma: the input channels are split into the segments `seg_channels`
    (default: one segment), every segment is zero-padded to 32-channel blocks and K runs ((blk*KH + dy)*KW + dx)*32 + c."""
    return tf32_round(_pack_conv_blocks(weight, seg_channels, 32))


def pack_conv_weight_f16(weight, seg_channels=None):
    """pack_conv_weight for pp_conv2d_umma_f16: 64-channel blocks, k = ((blk*KH + dy)*KW + dx)*64 + c, fp16 rounded to nearest
    from the fp32 weight (not from its TF32 image)."""
    return _pack_conv_blocks(weight, seg_channels, 64).to(torch.float16)


def _pm4(t, dtype=torch.float32):
    """[n,H,W,C] pixel-major view (unit channel stride, dense over n*H*W pixels) -> (ptr, ld)."""
    if t.dim() != 4:
        raise RuntimeError("expected [n,H,W,C]")
    return _pm(t, dtype)


def _conv_params(segs, KH, KW, Cout, w_packed=None, bias=None, act="none", slope=0.0, pre=None, res=None, post_relu=False,
                 out=None, round_tf32=False, bn=0, tile_w=0, tile_m=0, half=False):
    """PPConvParams of one pp_conv2d_umma call (see conv_umma; half: of pp_conv2d_umma_f16, fp16 segments and weight in
    64-channel blocks).  A segment may also be given as its shape (n, H, W, C): its pointer is then null and its ld is C
    rounded up to the narrowest row conv_umma accepts (4 floats, 8 halves), which is enough for pp_conv2d_umma_plan."""
    cb, lda, dt = (64, 8, torch.float16) if half else (32, 4, torch.float32)
    if not 1 <= len(segs) <= _lib.PP_CONV_MAX_SEG:
        raise RuntimeError(f"conv_umma: {len(segs)} input segments (1 to {_lib.PP_CONV_MAX_SEG} supported)")
    shapes = [tuple(s.shape) if isinstance(s, torch.Tensor) else tuple(s) for s in segs]
    n, H, W, _ = shapes[0]
    prm = PPConvParams()
    prm.nseg = len(segs)
    kblocks = 0
    for i, (sgm, shp) in enumerate(zip(segs, shapes)):
        if len(shp) != 4 or shp[:3] != (n, H, W):
            raise RuntimeError("conv_umma: segment shape mismatch")
        ptr, ld = _pm4(sgm, dt) if isinstance(sgm, torch.Tensor) else (ctypes.c_void_p(None), (shp[3] + lda - 1) // lda * lda)
        prm.seg[i].x, prm.seg[i].ld, prm.seg[i].C = ptr.value, ld, shp[3]
        kblocks += (shp[3] + cb - 1) // cb
    if w_packed is not None and tuple(w_packed.shape) != (Cout, kblocks * KH * KW * cb):
        raise RuntimeError(f"conv_umma: packed weight {tuple(w_packed.shape)} does not match {(Cout, kblocks * KH * KW * cb)}")
    prm.n, prm.H, prm.W, prm.KH, prm.KW = n, H, W, KH, KW
    prm.w_packed, prm.Cout = _pd(w_packed, dt).value if w_packed is not None else None, Cout
    prm.bias = _p(bias).value if bias is not None else None
    for name, t in (("pre", pre), ("res", res), ("out", out)):
        if t is None:
            setattr(prm, name, None)
            setattr(prm, "ld_" + name, 0)
            continue
        if tuple(t.shape) != (n, H, W, Cout):
            raise RuntimeError(f"conv_umma: {name} shape {tuple(t.shape)} != {(n, H, W, Cout)}")
        ptr, ld = _pm4(t)
        setattr(prm, name, ptr.value)
        setattr(prm, "ld_" + name, ld)
    prm.act, prm.slope, prm.post_relu, prm.round_tf32 = ACT[act], float(slope), int(bool(post_relu)), int(bool(round_tf32))
    prm.bn, prm.tile_w, prm.tile_m = int(bn), int(tile_w), int(tile_m)
    return prm


def conv_umma(segs, w_packed, KH, KW, Cout, bias=None, act="none", slope=0.0, pre=None, res=None, post_relu=False, out=None,
              round_tf32=False, bn=0, tile_w=0, tile_m=0):
    """wgmma implicit-GEMM conv (stride 1, same padding) with fused epilogue.  segs: list of [n,H,W,C_i] pixel-major
    views = the channel-concatenated input; w_packed from pack_conv_weight(weight, [C_i...]); pre / res / out
    [n,H,W,Cout] views (channel slices of wider buffers allowed).  Returns out."""
    if out is None and segs:
        out = segs[0].new_empty(*segs[0].shape[:3], Cout)
    prm = _conv_params(segs, KH, KW, Cout, w_packed, bias, act, slope, pre, res, post_relu, out, round_tf32, bn, tile_w, tile_m)
    _launch("pp_conv2d_umma", ctypes.byref(prm))
    return out


def conv_umma_f16(segs, w_packed, KH, KW, Cout, bias=None, act="none", slope=0.0, pre=None, res=None, post_relu=False, out=None,
                  out16=None, bn=0, tile_w=0, tile_m=0):
    """conv_umma on fp16 operands (pp_conv2d_umma_f16): segs fp16 [n,H,W,C_i] views, w_packed from pack_conv_weight_f16;
    bias / pre / res fp32, fp32 accumulation and epilogue.  Writes the fp32 `out` and / or the fp16 `out16` (rounded to
    nearest once; both from one pass when both are given; neither: a new out16).  Returns out16, else out."""
    if out is None and out16 is None:
        out16 = segs[0].new_empty(*segs[0].shape[:3], Cout)
    prm = _conv_params(segs, KH, KW, Cout, w_packed, bias, act, slope, pre, res, post_relu, out, False, bn, tile_w, tile_m, half=True)
    p16, ld16 = (None, 0)
    if out16 is not None:
        if tuple(out16.shape) != (prm.n, prm.H, prm.W, Cout):
            raise RuntimeError(f"conv_umma_f16: out16 shape {tuple(out16.shape)} != {(prm.n, prm.H, prm.W, Cout)}")
        p16, ld16 = _pm4(out16, torch.float16)
    _launch("pp_conv2d_umma_f16", ctypes.byref(prm), p16, ld16)
    return out16 if out16 is not None else out


ConvPlan = collections.namedtuple("ConvPlan", "tile_h tile_w bn ctas smem_bytes")


def conv_plan(segs, KH, KW, Cout, bn=0, tile_w=0, tile_m=0, out=None, pre=None, res=None, bias=None, half=False):
    """The tile / ring plan conv_umma (half: conv_umma_f16) would launch for these arguments (pp_conv2d_umma_plan[_f16]),
    without launching it: ConvPlan(tile_h, tile_w, bn, ctas, smem_bytes).  segs as in conv_umma, or their shapes
    (n, H, W, C_i).  Raises where conv_umma would refuse the plan."""
    prm = _conv_params(segs, KH, KW, Cout, bias=bias, pre=pre, res=res, out=out, bn=bn, tile_w=tile_w, tile_m=tile_m, half=half)
    vals = [ctypes.c_int(0) for _ in range(5)]
    sym = "pp_conv2d_umma_plan_f16" if half else "pp_conv2d_umma_plan"
    check(getattr(_lib.lib(), sym)(ctypes.byref(prm), *[ctypes.byref(v) for v in vals]), sym)
    return ConvPlan(*[v.value for v in vals])


def deform_gather(x, o, flow, max_res, cols=None, o_bias=None, x2=None):
    """x [n,H,W,Cin] view (or, with x2, the two halves x | x2 of Cin/2 channels each), o [n,H,W,>=432] raw conv_offset
    output, flow [n,H,W,2] | None -> cols [n,H,W,9*Cin] (modulated bilinear samples, k*Cin + c, TF32-rounded; an fp16 `cols`
    receives them rounded to nearest fp16): the A operand of the deformable conv's GEMM."""
    n, H, W, Cin = x.shape
    xp, ldx = _pm4(x)
    x2p, ldx2 = (None, 0)
    if x2 is not None:
        if x2.shape != x.shape:
            raise RuntimeError("deform_gather: x2 must have the shape of x")
        x2p, ldx2 = _pm4(x2)
        Cin *= 2
    op, ldo = _pm4(o)
    if cols is None:
        cols = torch.empty(n, H, W, 9 * Cin, device=x.device, dtype=torch.float32)
    sym, dt = _twin("pp_deform_gather", cols)
    _launch(sym, xp, ldx, x2p, ldx2, op, ldo, _p(o_bias), _pd(flow), float(max_res), _pd(cols, dt), n, H, W, Cin)
    return cols


def flow_warp_fbcheck(feat, fprop, fcheck=None, warped=None, aux=None, want_warp=True, round_tf32=False):
    """flow_warp (bilinear) of pixel-major maps feat [n,h,w,C] by fprop [n,h,w,2] -> warped [n,h,w,C] (views allowed);
    with fcheck also the forward-backward validity: aux [n,h,w,>=3] view receives (fx, fy, valid).  An fp16 `warped` receives
    the samples rounded to nearest fp16 (round_tf32 does not apply).  Returns (warped, aux)."""
    n, h, w = fprop.shape[:3]
    fp_, ldf, wp_, ldw, C = None, 0, None, 0, 0
    f16 = False
    if want_warp:
        C = feat.shape[-1]
        if warped is None:
            warped = torch.empty(n, h, w, C, device=feat.device, dtype=torch.float32)
        f16 = warped.dtype == torch.float16
        fp_, ldf = _pm4(feat)
        wp_, ldw = _pm4(warped, warped.dtype)
    ap, lda = (None, 0)
    if fcheck is not None:
        if aux is None:
            aux = torch.empty(n, h, w, 4, device=fprop.device, dtype=torch.float32)
        ap, lda = _pm4(aux)
    args = (fp_, ldf, _pd(fprop), _pd(fcheck), wp_, ldw, ap, lda, n, h, w, C)
    if f16:
        _launch("pp_flow_warp_fbcheck_f16", *args)
    else:
        _launch("pp_flow_warp_fbcheck", *args, int(bool(round_tf32)))
    return warped, aux


def pack_deform_weight_umma(weight):
    """deform-conv weight [Cout,Cin,3,3] -> [Cout, 9*Cin] with k = tap*Cin + c (the column order of deform_gather), TF32."""
    co, ci = weight.shape[:2]
    return tf32_round(weight.permute(0, 2, 3, 1).reshape(co, 9 * ci).contiguous())


def pack_deform_weight_umma_f16(weight):
    """pack_deform_weight_umma for conv_umma_f16 over fp16 columns: [Cout, 9*Cin], k = tap*Cin + c, rounded to nearest fp16."""
    co, ci = weight.shape[:2]
    return weight.permute(0, 2, 3, 1).reshape(co, 9 * ci).to(torch.float16).contiguous()


def pack_deform_weight(weight):
    """[Cout,Cin,3,3] -> [9*Cin, Cout], row = tap*Cin + c."""
    co, ci = weight.shape[:2]
    return weight.permute(2, 3, 1, 0).reshape(9 * ci, co).contiguous()


def gen_prep(flows_f, flows_b, masks_in, masks_upd, lt):
    """planar flows [lt-1,2,H,W] (fp32, or fp16 clip storage), masks [>=lt,1,H,W] -> dsf, dsb [lt-1,h,w,2], pmask [lt,h,w,2]."""
    H, W = masks_in.shape[-2:]
    h, w = H // 4, W // 4
    dev = masks_in.device
    dsf = torch.empty(max(lt - 1, 1), h, w, 2, device=dev, dtype=torch.float32)
    dsb = torch.empty_like(dsf)
    pmask = torch.empty(lt, h, w, 2, device=dev, dtype=torch.float32)
    sym, dt = _twin("pp_gen_prep", flows_f)                     # fp16: half-precision clip storage, widened in the kernel
    _launch(sym, _pd(flows_f, dt), _pd(flows_b, dt), _pd(masks_in), _pd(masks_upd), _p(dsf), _p(dsb), _p(pmask), lt, H, W)
    return dsf[:lt - 1], dsb[:lt - 1], pmask


def window_mask(pmask, fh, fw, nwh, nww):
    lt, h, w, _ = pmask.shape
    flags = torch.empty(nwh * nww, device=pmask.device, dtype=torch.int32)
    _launch("pp_window_mask", _pd(pmask), lt, h, w, fh, fw, nwh, nww, _p(flags, torch.int32))
    return flags


def sparse_window_attn(qkv, pool_kv, key_tok, flags, t, NT, kf_start, kf_step, out=None, WN=45, C=512, impl="umma"):
    """qkv [t,NT,3C]; pool_kv [t,NP,2C]; key_tok int32 [nwin,NKO]; flags int32 [nwin] -> out [t,NT,C].
    impl: "umma" = wgmma kernel for masked windows (default), "mma" = warp-level mma.sync baseline.  fp16 qkv / pool_kv (the
    half-operand Linear outputs): fp16 out from the fp16 kernels (impl is then ignored: there is one fp16 plan)."""
    dt = qkv.dtype
    if out is None:
        out = torch.empty(t, NT, C, device=qkv.device, dtype=dt)
    prm = PPAttnParams()
    prm.qkv, prm.pool = qkv.data_ptr(), pool_kv.data_ptr()
    prm.key_tok, prm.flags, prm.out = key_tok.data_ptr(), flags.data_ptr(), out.data_ptr()
    prm.ld_qkv, prm.ld_pool, prm.ld_out = qkv.stride(-2), pool_kv.stride(-2), out.stride(-2)
    prm.t, prm.NT, prm.WN, prm.NKO, prm.NP, prm.C = t, NT, WN, key_tok.shape[1], pool_kv.shape[1], C
    prm.kf_start, prm.kf_step = kf_start, kf_step
    prm.nkf = len(range(kf_start, t, kf_step))
    if prm.nkf == 0:
        out.zero_()                 # empty key set: masked windows yield zeros (softmax over an empty dim), see the C entry
    prm.scale_log2 = LOG2E / math.sqrt(128.0)
    for tns, tdt in ((qkv, dt), (pool_kv, dt), (key_tok, torch.int32), (flags, torch.int32)):
        _pd(tns, tdt)                                           # the struct holds raw addresses: check what they point at
    _p(out, dt)
    if dt == torch.float16:
        sym = "pp_sparse_window_attn_f16"
    else:
        sym = "pp_sparse_window_attn" if impl == "umma" else "pp_sparse_window_attn_mma"
    _launch(sym, ctypes.byref(prm), key_tok.shape[0], launches=2)
    return out


def ffn_overlap_add(Y, frames, h, w, CH=40):
    """Y [frames*fh*fw, 49*CH] (tap-major columns) -> gelu(unfold(fold(Y)/norm)) same shape and dtype.  fp16 Y (the
    half-operand fc1 output): fp16 Z, summed in fp32 and rounded once."""
    Z = torch.empty_like(Y)
    ws_bytes = _lib.lib().pp_ffn_overlap_add_workspace_bytes(frames, h, w, CH)
    ws = torch.empty(ws_bytes // 4, device=Y.device, dtype=torch.float32)
    sym, dt = _twin("pp_ffn_overlap_add", Y)
    _launch(sym, _pd(Y, dt), Y.shape[-1], _p(Z, dt), Z.shape[-1], frames, h, w, CH, _p(ws), ws_bytes, launches=2)
    return Z


def gru_gate(zr_pm, bias, net_view, z_out, rnet_view, pre=None):
    """zr_pm [..,2C] raw gate conv output; net_view / rnet_view: C-channel slices of HX / RX; z_out dense [..,C];
    bias [2C] / pre [..,2C] optional addends.  fp16 zr_pm: rnet_view is fp16 too, net_view the fp32 state."""
    C = z_out.shape[-1]
    np_, ldn = _pm(net_view)
    sym, dt = _twin("pp_gru_gate", zr_pm)
    rp, ldr = _pm(rnet_view, dt)
    _launch(sym, _pd(zr_pm, dt), _p(bias), _pd(pre), np_, ldn, _pd(z_out), rp, ldr, z_out.numel() // C, C)


def gru_update(q_pm, bias, z, net_view, net_copy=None, pre=None, h_img=None):
    """h = (1-z)*h + z*tanh(q+bias+pre) in place on the state slice; `net_copy` (dense) also receives h.  fp16 q_pm: the
    state net_view stays fp32, its fp16 image goes to h_img (a C-channel slice of the fp16 HX) and the fp16 net_copy."""
    C = z.shape[-1]
    np_, ldn = _pm(net_view)
    sym, dt = _twin("pp_gru_update", q_pm)
    img = ()                                                    # pp_gru_update_f16's (h_img, ld)
    if dt == torch.float16:
        img = _pm(h_img, dt) if h_img is not None else (None, C)
    elif h_img is not None:
        raise RuntimeError("gru_update: h_img is the fp16 image of the state (fp16 q_pm only)")
    _launch(sym, _pd(q_pm, dt), _p(bias), _pd(pre), _pd(z), np_, ldn, *img, _pd(net_copy, dt), z.numel() // C, C)


def raft_pack_motion(mot_pm, flow_pm, d0_view, d1_view, bias=None):
    """mot_pm [..,128] (channels 126,127 ignored), flow_pm [..,2] -> 128-channel slot views of HX and RX.
    With `bias`, mot_pm is the raw conv output and relu(mot + bias) is applied on the way.  fp16 mot_pm: fp16 HX / RX."""
    sym, dt = _twin("pp_raft_pack_motion", mot_pm)
    mp, ldm = _pm(mot_pm, dt)
    p0, ld0 = _pm(d0_view, dt)
    p1, ld1 = _pm(d1_view, dt)
    if ld0 != ld1:
        raise RuntimeError("HX / RX must share the pixel stride")
    _launch(sym, mp, ldm, _p(bias), _pd(flow_pm), p0, p1, ld0, flow_pm.numel() // 2)


def raft_pack_motion_n(mot_pm, flow_pm, d0_view, d1_view, cmot, bias=None):
    """raft_pack_motion for `cmot` motion channels: channels [0,cmot) of mot_pm (+ bias, ReLU), the 2 flow channels, zeros
    up to roundup4(cmot+2) -> that many channels of the slot views d0_view / d1_view (of HX and RX)."""
    mp, ldm = _pm(mot_pm)
    p0, ld0 = _pm(d0_view)
    p1, ld1 = _pm(d1_view)
    if ld0 != ld1:
        raise RuntimeError("HX / RX must share the pixel stride")
    if mot_pm.shape[-1] < cmot or d0_view.shape[-1] < ((cmot + 5) & ~3) or (bias is not None and bias.numel() < cmot):
        raise RuntimeError("raft_pack_motion_n: channel counts too small for cmot")
    _launch("pp_raft_pack_motion_n", mp, ldm, _p(bias), _pd(flow_pm), p0, p1, ld0, flow_pm.numel() // 2, cmot)


ACT = {"none": 0, "relu": 1, "leaky": 2, "sigmoid": 3, "tanh": 4}


def bias_act(x_pm, bias=None, act="none", slope=0.0, res=None, post_relu=False, out=None, pre=None):
    """out = post(act(x + bias + pre) + res) on pixel-major views [..., C] (unit channel stride, dense over pixels; x / pre /
    res / out may each be a channel slice of a wider buffer).  out=None -> in place on x_pm.  Returns out.  x_pm and out may
    be fp16 (RAFT's half-precision refinement convs); bias / pre and the arithmetic are fp32.  res is fp32, or fp16 with fp16
    x and out (the residual blocks of RAFT's half-operand context encoder)."""
    C = x_pm.shape[-1]
    out = x_pm if out is None else out
    if out.shape != x_pm.shape or (res is not None and res.shape != x_pm.shape) or (pre is not None and pre.shape != x_pm.shape):
        raise RuntimeError("bias_act: shape mismatch")
    f16, f32 = torch.float16, torch.float32
    if res is not None and res.dtype == f16:
        if x_pm.dtype != f16 or out.dtype != f16 or pre is not None:
            raise RuntimeError("bias_act: an fp16 residual needs fp16 x and out and no pre")
        sym, xdt, odt, rdt = "pp_bias_act_f16_res", f16, f16, f16
    elif f16 in (x_pm.dtype, out.dtype):
        if not {x_pm.dtype, out.dtype} <= {f16, f32}:
            raise RuntimeError(f"bias_act: x / out must be fp32 or fp16, got {x_pm.dtype} / {out.dtype}")
        sym, xdt, odt, rdt = "pp_bias_act_f16", x_pm.dtype, out.dtype, f32
    else:
        sym, xdt, odt, rdt = "pp_bias_act" if pre is None else "pp_bias_act_pre", f32, f32, f32
    xp, ldx = _pm(x_pm, xdt)
    op, ldo = _pm(out, odt)
    rp, ldr = _pm(res, rdt) if res is not None else (None, C)
    tail = (x_pm.numel() // C, C, ACT[act], float(slope), int(bool(post_relu)))
    if sym == "pp_bias_act_f16":                                # takes the row types, and pre always
        pp, ldp = _pm(pre) if pre is not None else (None, C)
        _launch(sym, xp, ldx, int(xdt == f16), _p(bias), pp, ldp, rp, ldr, op, ldo, int(odt == f16), *tail)
    else:
        _launch(sym, xp, ldx, _p(bias), *(_pm(pre) if pre is not None else ()), rp, ldr, op, ldo, *tail)
    return out


def bias_act_(x_pm, bias, act="none", slope=0.0):
    """in-place act(x + bias); returns x_pm."""
    return bias_act(x_pm, bias, act, slope)


def sc_fold(cols, bmap, frames, h, w, out=None):
    """SoftComp's fold after its Linear layer: fp16 tap-major columns [frames*fh*fw, 49*C] (column tap*C + c) + the folded
    Linear bias bmap (fp32 pixel-major [h,w,C]) -> fp16 pixel-major [frames,h,w,C] (7x7 / stride 3 / pad 3 overlap-add, fp32
    sums in a fixed order)."""
    C = bmap.shape[-1]
    fh, fw = (h - 1) // 3 + 1, (w - 1) // 3 + 1
    if cols.dim() != 2 or cols.shape[0] != frames * fh * fw or cols.stride(1) != 1 or tuple(bmap.shape) != (h, w, C):
        raise RuntimeError("sc_fold: shape mismatch")
    out = torch.empty(frames, h, w, C, device=cols.device, dtype=torch.float16) if out is None else out
    if tuple(out.shape) != (frames, h, w, C):
        raise RuntimeError("sc_fold: out shape mismatch")
    _launch("pp_sc_fold_f16", _p(cols, torch.float16), cols.stride(0), _pd(bmap), _pd(out, torch.float16), frames, h, w, C)
    return out


def pool_depthwise(x_pm, w_taps, bias, kh, kw):
    """depthwise conv, kernel = stride = (kh,kw): x_pm [n,H,W,C] -> [n,H//kh,W//kw,C]; w_taps [kh*kw, C].  fp16 x_pm (the
    half-operand LayerNorm output): fp16 out, weights / bias / sums fp32."""
    n, H, W, C = x_pm.shape
    sym, dt = _twin("pp_pool_depthwise", x_pm)
    xp, ld = _pm(x_pm, dt)
    out = torch.empty(n, (H - kh) // kh + 1, (W - kw) // kw + 1, C, device=x_pm.device, dtype=dt)
    _launch(sym, xp, ld, _pd(w_taps), _p(bias), _p(out, dt), n, H, W, C, kh, kw)
    return out


def add_layernorm(x, delta, gamma, beta, eps=1e-5, y_dtype=torch.float32):
    """(x + delta, LayerNorm(x + delta)) over the last dim; delta=None -> (x, LayerNorm(x)).  Dense tensors.  x fp32; delta
    fp32 or fp16 (the half-operand fc2 output); y in y_dtype, fp32 or fp16 (the half-operand fc1 operand)."""
    C = x.shape[-1]
    y = torch.empty_like(x, dtype=y_dtype)
    xo = torch.empty_like(x) if delta is not None else None
    dt = delta.dtype if delta is not None else torch.float32
    if torch.float16 in (y_dtype, dt):
        _launch("pp_add_layernorm_f16", _pd(x), _pd(delta, dt), int(dt == torch.float16), _p(gamma), _p(beta), _p(xo),
                _p(y, y_dtype), int(y_dtype == torch.float16), x.numel() // C, C, float(eps))
    else:
        _launch("pp_add_layernorm", _pd(x), _pd(delta), _p(gamma), _p(beta), _p(xo), _p(y), x.numel() // C, C, float(eps))
    return (xo if delta is not None else x), y


def instance_norm(x_pm, relu=False, res=None, post_relu=False, eps=1e-5, out=None):
    """InstanceNorm2d(affine=False) on a dense pixel-major map [n,h,w,C] (+ ReLU, + residual add, + final ReLU)."""
    n, h, w, C = x_pm.shape
    out = torch.empty_like(x_pm) if out is None else out
    nbytes = _lib.lib().pp_instance_norm_workspace_bytes(n, h * w, C)
    ws = torch.empty(max(nbytes // 4, 4), device=x_pm.device, dtype=torch.float32)
    _launch("pp_instance_norm", _pd(x_pm), _pd(res), _pd(out), n, h * w, C, float(eps), int(bool(relu)), int(bool(post_relu)),
            _p(ws), ws.numel() * 4, launches=2)
    return out


def upsample2x(x_pm):
    """pixel-major [n,h,w,C] -> [n,2h,2w,C], bilinear, align_corners=True.  fp16 x_pm (the half-operand decoder): fp16 out,
    blended in fp32."""
    n, h, w, C = x_pm.shape
    out = torch.empty(n, 2 * h, 2 * w, C, device=x_pm.device, dtype=x_pm.dtype)
    sym, dt = _twin("pp_upsample2x_bilinear", x_pm)
    _launch(sym, _pd(x_pm, dt), _p(out, dt), n, h, w, C)
    return out


def mask_dilate(masks_u8, iterations):
    """uint8 [T,H,W] (non-zero = hole) -> float {0,1} [T,1,H,W], dilated `iterations` times with the 3x3 cross."""
    T, H, W = masks_u8.shape
    out = torch.empty(T, 1, H, W, device=masks_u8.device, dtype=torch.float32)
    _launch("pp_mask_dilate", _pd(masks_u8, torch.uint8), _p(out), T, H, W, int(iterations))
    return out


def u8_to_frames(frames_u8):
    """uint8 [T,H,W,3] -> float planar [T,3,H,W] in [-1,1]."""
    T, H, W, _ = frames_u8.shape
    out = torch.empty(T, 3, H, W, device=frames_u8.device, dtype=torch.float32)
    _launch("pp_u8_to_frames", _pd(frames_u8, torch.uint8), _p(out), T, H, W)
    return out


def u8_to_frames_resized(frames_u8, size):
    """scripts/compute_flow.py:67-92: uint8 RGB [T,H0,W0,3] -> float planar [T,3,h,w] in [-1,1], size = (w, h): v / 255,
    torch's bilinear F.interpolate (align_corners=False, no antialias), then *2 - 1.  Bit for bit with that sequence on
    ATen's CPU kernel; at the frames' own size equal to u8_to_frames."""
    if frames_u8.dtype != torch.uint8 or frames_u8.dim() != 4 or frames_u8.shape[-1] != 3 or frames_u8.shape[0] < 1:
        raise ValueError(f"u8_to_frames_resized: expected uint8 frames [T,H,W,3], got {frames_u8.dtype} {tuple(frames_u8.shape)}")
    w, h = (int(s) for s in size)
    T, H0, W0, _ = frames_u8.shape
    if w < 1 or h < 1 or H0 < 1 or W0 < 1:
        raise ValueError(f"u8_to_frames_resized: cannot resize {H0}x{W0} frames to size {tuple(size)}")
    out = torch.empty(T, 3, h, w, device=frames_u8.device, dtype=torch.float32)
    _launch("pp_u8_to_frames_resized", _pd(frames_u8, torch.uint8), _p(out), T, H0, W0, h, w)
    return out


def composite_blend(pred, masks, ori_u8, comp_u8, frame_ids, first_flags):
    """pred [n,3,H,W]; masks [T,1,H,W]; ori/comp uint8 [T,H,W,3] (comp updated in place)."""
    _composite_blend("pp_composite_blend_u8", torch.uint8, pred, masks, ori_u8, comp_u8, frame_ids, first_flags)


def composite_blend_f32(pred, masks, ori_u8, comp_f32, frame_ids, first_flags):
    """The evaluation script's compositing (evaluate_propainter.py:166-179): as composite_blend, but comp is a float32
    clip [T,H,W,3] (updated in place) and a later visit's 1/2-1/2 blend is not truncated."""
    if comp_f32.dtype != torch.float32:
        raise RuntimeError(f"composite_blend_f32: comp must be float32, got {comp_f32.dtype}")
    _composite_blend("pp_composite_blend_f32", torch.float32, pred, masks, ori_u8, comp_f32, frame_ids, first_flags)


def _composite_blend(sym, comp_dtype, pred, masks, ori_u8, comp, frame_ids, first_flags):
    n, _, H, W = pred.shape
    ids = PPWindowIds()
    ids.n = n
    for i, (f, fl) in enumerate(zip(frame_ids, first_flags)):
        ids.frame[i], ids.first[i] = int(f), int(fl)
    _launch(sym, _pd(pred), _pd(masks), _pd(ori_u8, torch.uint8), _pd(comp, comp_dtype), ctypes.byref(ids), H, W)


def extrapolate_u8(frames_u8, geometry):
    """extrapolation (inference_propainter.py:117-156) on the device: uint8 [T,h,w,3] and a geometry
    ((H, W), (top, left), (rim_h, rim_w)) from inference_propainter.outpaint_geometry -> (canvas uint8 [T,H,W,3],
    flow_masks float {0,1} [T,1,H,W], masks_dilated float {0,1} [T,1,H,W])."""
    (H, W), (top, left), (rim_h, rim_w) = geometry
    if frames_u8.dim() != 4 or frames_u8.shape[-1] != 3:
        raise RuntimeError("extrapolate_u8: expected uint8 frames [T,h,w,3]")
    T, h, w, _ = frames_u8.shape
    src = _pd(frames_u8, torch.uint8)
    dev = frames_u8.device
    canvas = torch.empty(T, H, W, 3, dtype=torch.uint8, device=dev)
    fm = torch.empty(T, 1, H, W, dtype=torch.float32, device=dev)
    md = torch.empty_like(fm)
    _launch("pp_extrapolate_u8", src, _p(canvas, torch.uint8), _p(fm), _p(md), T, h, w, H, W, top, left, rim_h, rim_w)
    return canvas, fm, md


def mask_overlay_u8(frames_u8, masks):
    """The green masked-frame preview of inference_propainter.py:250-261: uint8 [T,H,W,3] + float masks with T*H*W
    elements ([T,1,H,W] or the pipeline's [1,T,1,H,W]) -> uint8 [T,H,W,3]."""
    if frames_u8.dim() != 4 or frames_u8.shape[-1] != 3:
        raise RuntimeError("mask_overlay_u8: expected uint8 frames [T,H,W,3]")
    T, H, W, _ = frames_u8.shape
    if masks.numel() != T * H * W or tuple(masks.shape[-2:]) != (H, W):
        raise RuntimeError(f"mask_overlay_u8: masks {tuple(masks.shape)} do not match frames {tuple(frames_u8.shape)}")
    out = torch.empty_like(frames_u8)
    _launch("pp_mask_overlay_u8", _pd(frames_u8, torch.uint8), _pd(masks), _p(out, torch.uint8), T, H, W)
    return out


FLOWVIZ_NORMALIZE = {"frame": 0, "clip": 1}       # PP_FLOWVIZ_FRAME / PP_FLOWVIZ_CLIP


def flow_to_image_u8(flow, normalize="frame", clip_flow=None, bgr=False):
    """Middlebury colour coding of planar float32 flow (N,2,H,W) or (2,H,W) on the device -> uint8 (N,H,W,3) or (H,W,3),
    RGB (BGR with `bgr`).  normalize="frame": RAFT/utils/flow_viz.py::flow_to_image applied to each frame (rad_max per
    frame, numpy >= 2 arithmetic, the rad > 1 branch); "clip": flow_viz_pt.py::flow_to_image (max_norm over the whole
    batch).  clip_flow: np.clip(flow, 0, clip_flow) before the radius, as flow_viz.py:123-124 does.  Bytes equal the
    reference's except where atan2's last-ulp differences move a colour across a rounding boundary (INTEGRATION.md §3).
    ValueError where flow_viz_pt raises (dtype other than float32, other shapes)."""
    if flow.dtype != torch.float32:
        raise ValueError(f"Flow should be of dtype torch.float, got {flow.dtype}.")
    if normalize not in FLOWVIZ_NORMALIZE:
        raise ValueError(f"normalize must be 'frame' or 'clip', got {normalize!r}")
    single = flow.dim() == 3
    f = flow[None] if single else flow
    if f.dim() != 4 or f.shape[1] != 2:
        raise ValueError(f"Input flow should have shape (2, H, W) or (N, 2, H, W), got {tuple(flow.shape)}.")
    f = f.contiguous()
    N, _, H, W = f.shape
    per_frame = int(normalize == "frame")
    maxima = torch.empty(N if per_frame else 1, dtype=torch.float32, device=f.device)
    out = torch.empty(N, H, W, 3, dtype=torch.uint8, device=f.device)
    has_clip, clip = int(clip_flow is not None), ctypes.c_float(0.0 if clip_flow is None else float(clip_flow))
    _launch("pp_flow_maxrad", _p(f), _p(maxima), N, H, W, per_frame, has_clip, clip)
    _launch("pp_flow_to_image_u8", _p(f), _p(maxima), _p(out, torch.uint8), N, H, W, FLOWVIZ_NORMALIZE[normalize], has_clip, clip,
            int(bool(bgr)))
    return out[0] if single else out


# ---------------------------------------------------------------- temporal warping error (E_warp)
def _ewarp_flows(flow, what):
    """[N,2,H,W] or [1,N,2,H,W], fp32 or fp16 -> [N,2,H,W] (shape and dtype checked; the device is checked by _ewarp_dev)"""
    if not isinstance(flow, torch.Tensor):
        raise ValueError(f"{what}: flows must be a torch tensor, got {type(flow).__name__}")
    f = flow[0] if flow.dim() == 5 and flow.shape[0] == 1 else flow
    if f.dim() != 4 or f.shape[1] != 2 or f.dtype not in (torch.float32, torch.float16):
        raise ValueError(f"{what}: expected fp32 / fp16 flows [N,2,H,W] or [1,N,2,H,W], got {flow.dtype} {tuple(flow.shape)}")
    if f.shape[0] < 1 or f.shape[2] < 1 or f.shape[3] < 1:
        raise ValueError(f"{what}: empty flows {tuple(flow.shape)}")
    return f


def _ewarp_dev(what, *tensors):
    """raise ValueError unless every tensor is on the device; fp16 flows are widened here, once"""
    if not all(t.is_cuda for t in tensors if t is not None):
        raise ValueError(f"{what}: inputs must be CUDA tensors (there is no CPU path)")
    return [None if t is None else t.float().contiguous() if t.is_floating_point() else t.contiguous() for t in tensors]


def flow_occlusion(fw, bw):
    """Occlusion maps of Lai et al.'s warping-error evaluation (the test of Ruder et al.): forward flows fw (frame t ->
    t+1) and backward flows bw (t+1 -> t), each [N,2,H,W] or [1,N,2,H,W] in fp32 or fp16 -> uint8 [N,H,W], 1 = occluded
    (forward-backward check or motion boundary; include/propainter_b200.h)."""
    f, b = _ewarp_flows(fw, "flow_occlusion"), _ewarp_flows(bw, "flow_occlusion")
    if f.shape != b.shape:
        raise ValueError(f"flow_occlusion: forward {tuple(fw.shape)} and backward {tuple(bw.shape)} flows differ in shape")
    f, b = _ewarp_dev("flow_occlusion", f, b)
    N, _, H, W = f.shape
    occ = torch.empty(N, H, W, dtype=torch.uint8, device=f.device)
    _launch("pp_flow_occlusion", _p(f), _p(b), _p(occ, torch.uint8), N, H, W)
    return occ


def warp_error_sums(frames_u8, fw, occ=None, bw=None):
    """The kernel's per-pair result: float64 [T-1,2] = (sum over the non-occluded pixels and RGB of the squared
    difference between frame t+1 warped by fw_t and frame t, both / 255; N_t = the number of those pixels).  frames uint8
    [T,H,W,3] on the device, T >= 2; fw as for flow_occlusion with N = T-1.  The occlusion map is `occ` (uint8
    [T-1,H,W], non-zero = occluded) or, without it, computed from `bw` in the same pass.  Fixed-order float64 sums: the
    same bits on every run."""
    if not isinstance(frames_u8, torch.Tensor) or frames_u8.dtype != torch.uint8 or frames_u8.dim() != 4 or frames_u8.shape[-1] != 3:
        raise ValueError(f"warp_error: expected uint8 frames [T,H,W,3], got {getattr(frames_u8, 'dtype', type(frames_u8))} "
                         f"{tuple(getattr(frames_u8, 'shape', ()))}")
    T, H, W, _ = frames_u8.shape
    if T < 2 or H < 1 or W < 1:
        raise ValueError(f"warp_error: needs at least 2 non-empty frames, got {tuple(frames_u8.shape)}")
    f = _ewarp_flows(fw, "warp_error")
    if tuple(f.shape) != (T - 1, 2, H, W):
        raise ValueError(f"warp_error: flows {tuple(fw.shape)} do not match frames {tuple(frames_u8.shape)}")
    b = None
    if occ is not None:
        if not isinstance(occ, torch.Tensor) or occ.dtype != torch.uint8 or tuple(occ.shape) != (T - 1, H, W):
            raise ValueError(f"warp_error: occ must be a uint8 tensor [{T - 1},{H},{W}]")
    elif bw is not None:
        b = _ewarp_flows(bw, "warp_error")
        if b.shape != f.shape:
            raise ValueError(f"warp_error: backward flows {tuple(bw.shape)} do not match forward flows {tuple(fw.shape)}")
    else:
        raise ValueError("warp_error: needs the occlusion map `occ` or the backward flows `bw`")
    fr, f, b, o = _ewarp_dev("warp_error", frames_u8, f, b, occ)
    ws = torch.empty(_lib.lib().pp_warp_error_workspace_bytes(T, H, W), dtype=torch.uint8, device=f.device)
    out = torch.empty(T - 1, 2, dtype=torch.float64, device=f.device)
    _launch("pp_warp_error", _p(fr, torch.uint8), _p(f), _p(b), _p(o, torch.uint8), _p(out, torch.float64), T, H, W,
            _p(ws, torch.uint8), ws.numel(), launches=2)
    return out


def warp_error(frames_u8, fw, occ=None, bw=None):
    """Per-pair temporal warping error E_t of Lai et al. (ECCV 2018), float64 [T-1] on the device: warp_error_sums'
    sum / (3 N_t), 0 where every pixel is occluded.  Frames [0, 1] scale (no x 1e-3)."""
    s = warp_error_sums(frames_u8, fw, occ, bw)
    return torch.where(s[:, 1] > 0, s[:, 0] / (3 * s[:, 1]).clamp(min=1), torch.zeros_like(s[:, 0]))


# ---------------------------------------------------------------- I3D feature network (VFID)
def same_pad(k, s, n):
    """TF 'same' padding of a k-tap, stride-s window over n samples (pp_same_pad, core/metrics.py:196-200,258-262); the front
    gets pad // 2."""
    p = k - (n % s if n % s else s)
    return max(p, 0)


def same_out(k, s, n):
    """output extent of that window (pp_same_out)"""
    return (n + same_pad(k, s, n) - k) // s + 1


def i3d_input(video):
    """Conv3d_1a_7x7's padded operand: uint8 frames [B,T,H,W,3] (value u8 / 255, as to_tensors) or planar float32
    [B,3,T,H,W] (copied) -> float32 [B,T+pt,H+ph,W+pw,4] with the asymmetric 'same' border of a 7-tap stride-2 window
    and a zero 4th channel."""
    if video.dim() != 5:
        raise RuntimeError(f"i3d_input: expected a 5-d video, got {tuple(video.shape)}")
    u8 = video.dtype == torch.uint8
    if u8:
        if video.shape[-1] != 3:
            raise RuntimeError("i3d_input: uint8 frames must be [B,T,H,W,3]")
        B, T, H, W, _ = video.shape
    else:
        if video.shape[1] != 3:
            raise RuntimeError("i3d_input: float video must be [B,3,T,H,W]")
        B, _, T, H, W = video.shape
    src = _pd(video, video.dtype if u8 else torch.float32)
    out = torch.empty(B, T + same_pad(7, 2, T), H + same_pad(7, 2, H), W + same_pad(7, 2, W), 4, device=video.device,
                      dtype=torch.float32)
    _launch("pp_i3d_input", src, int(u8), _p(out), B, T, H, W)
    return out


def maxpool3d_same(x, kernel, stride, out=None):
    """MaxPool3dSamePadding (core/metrics.py:195-218) on a pixel-major map x [B,T,H,W,C] (dense pixels, C a multiple of 4)
    -> out [B,To,Ho,Wo,C] (may be a channel slice of a wider buffer).  Padded taps count as zeros, as after F.pad."""
    B, T, H, W, C = x.shape
    (kt, kh, kw), (st, sh, sw) = kernel, stride
    shape = (B, same_out(kt, st, T), same_out(kh, sh, H), same_out(kw, sw, W), C)
    if out is None:
        out = torch.empty(shape, device=x.device, dtype=torch.float32)
    if tuple(out.shape) != shape:
        raise RuntimeError(f"maxpool3d_same: out {tuple(out.shape)} != {shape}")
    xp, ldx = _pm(x)
    op, ldo = _pm(out)
    _launch("pp_maxpool3d_same", xp, ldx, op, ldo, B, T, H, W, C, kt, kh, kw, st, sh, sw)
    return out


def mean_thw(x):
    """x.mean(4).mean(3).mean(2) of an NCDHW map, on its pixel-major form x [B,T,H,W,C] -> float32 [B,C]: float64
    fixed-order sums, rounded once."""
    B, C = x.shape[0], x.shape[-1]
    xp, ld = _pm(x)
    out = torch.empty(B, C, device=x.device, dtype=torch.float32)
    _launch("pp_mean_thw", xp, ld, _p(out), B, x[0, ..., 0].numel(), C)
    return out


# ---------------------------------------------------------------- resizing around the path (tables on the host, passes on the device)
_TABLES = {}


def resample_tables(kind, in_size, out_size, device=None, horizontal=True):
    """Per-axis tables of the library resamplers the reference calls (see include/propainter_b200.h), as torch tensors
    (on `device` if given).  kind: "bicubic" -> (bounds int32 [out,2], kk int32 [out,ksize]); "nearest" -> idx int32 [out];
    "linear_cv" -> (ofs int32 [out], coef int16 [out,2])."""
    key = (kind, in_size, out_size, str(device), horizontal)
    if key in _TABLES:
        return _TABLES[key]
    L = _lib.lib()
    if kind == "bicubic":
        ks = L.pp_resample_coeffs_bicubic(in_size, out_size, None, None, 0)
        bounds, kk = torch.empty(out_size, 2, dtype=torch.int32), torch.empty(out_size, ks, dtype=torch.int32)
        check(min(0, L.pp_resample_coeffs_bicubic(in_size, out_size, bounds.data_ptr(), kk.data_ptr(), kk.numel())), "pp_resample_coeffs_bicubic")
        res = (bounds, kk)
    elif kind == "nearest":
        idx = torch.empty(out_size, dtype=torch.int32)
        check(L.pp_resample_index_nearest(in_size, out_size, idx.data_ptr()), "pp_resample_index_nearest")
        res = (idx,)
    elif kind == "linear_cv":
        ofs, coef = torch.empty(out_size, dtype=torch.int32), torch.empty(out_size, 2, dtype=torch.int16)
        check(L.pp_resample_coeffs_linear_cv(in_size, out_size, int(bool(horizontal)), ofs.data_ptr(), coef.data_ptr()), "pp_resample_coeffs_linear_cv")
        res = (ofs, coef)
    elif kind == "linear_f32":
        ofs, coef = torch.empty(out_size, dtype=torch.int32), torch.empty(out_size, 2, dtype=torch.float32)
        check(L.pp_resample_coeffs_linear_f32(in_size, out_size, int(bool(horizontal)), ofs.data_ptr(), coef.data_ptr()),
              "pp_resample_coeffs_linear_f32")
        res = (ofs, coef)
    else:
        raise ValueError(kind)
    if device is not None:
        res = tuple(t.to(device) for t in res)
    _TABLES[key] = res
    return res


def resize_frames_u8(frames_u8, size):
    """resize_frames (inference_propainter.py:34-45): uint8 [T,H,W,3] -> [T,Ho,Wo,3], size = (Wo, Ho) like PIL; = PIL.Image.resize(size)."""
    T, H, W, _ = frames_u8.shape
    Wo, Ho = size
    dev = frames_u8.device
    bx, kx = resample_tables("bicubic", W, Wo, dev)
    by, ky = resample_tables("bicubic", H, Ho, dev)
    out = torch.empty(T, Ho, Wo, 3, dtype=torch.uint8, device=dev)
    nws = _lib.lib().pp_resize_u8_bicubic_workspace_bytes(T, H, Wo)
    ws = torch.empty(max(nws, 16), dtype=torch.uint8, device=dev)
    _launch("pp_resize_u8_bicubic", _pd(frames_u8, torch.uint8), _p(out, torch.uint8), T, H, W, Ho, Wo, _p(bx, torch.int32),
            _p(kx, torch.int32), kx.shape[1], _p(by, torch.int32), _p(ky, torch.int32), ky.shape[1], _p(ws, torch.uint8),
            ws.numel(), launches=2)
    return out


def resize_masks_u8(masks_u8, size):
    """mask_img.resize(size, Image.NEAREST) (inference_propainter.py:95-96): uint8 [T,H,W] -> [T,Ho,Wo]."""
    T, H, W = masks_u8.shape
    Wo, Ho = size
    dev = masks_u8.device
    (ix,), (iy,) = resample_tables("nearest", W, Wo, dev), resample_tables("nearest", H, Ho, dev)
    out = torch.empty(T, Ho, Wo, dtype=torch.uint8, device=dev)
    _launch("pp_resize_u8_nearest", _pd(masks_u8, torch.uint8), _p(out, torch.uint8), T, H, W, Ho, Wo, 1, _p(ix, torch.int32),
            _p(iy, torch.int32))
    return out


def resize_output_u8(frames_u8, size):
    """cv2.resize(f, out_size) of the composited frames (inference_propainter.py:469-470): uint8 [T,H,W,3] -> [T,Ho,Wo,3]."""
    T, H, W, _ = frames_u8.shape
    Wo, Ho = size
    dev = frames_u8.device
    xo, xa = resample_tables("linear_cv", W, Wo, dev, True)
    yo, ya = resample_tables("linear_cv", H, Ho, dev, False)
    out = torch.empty(T, Ho, Wo, 3, dtype=torch.uint8, device=dev)
    _launch("pp_resize_u8_bilinear_cv", _pd(frames_u8, torch.uint8), _p(out, torch.uint8), T, H, W, Ho, Wo, _p(xo, torch.int32),
            _p(xa, torch.int16), _p(yo, torch.int32), _p(ya, torch.int16))
    return out


def resize_flow(flows, size):
    """resize_flow (utils/flow_util.py:6-11) as the evaluation dataset applies it to loaded flows (core/dataset.py:213-214):
    cv2.resize(INTER_LINEAR) of float32 flows, then u *= Wo/W and v *= Ho/H in float32.  Planar [N,2,H,W] -> [N,2,Ho,Wo],
    size = (Wo, Ho) like cv2."""
    if flows.dtype != torch.float32 or flows.dim() != 4 or flows.shape[1] != 2:
        raise ValueError(f"resize_flow: expected float32 flows [N,2,H,W], got {flows.dtype} {tuple(flows.shape)}")
    N, _, H, W = flows.shape
    Wo, Ho = (int(s) for s in size)
    if Wo < 1 or Ho < 1:
        raise ValueError(f"resize_flow: bad size {size}")
    dev = flows.device
    xo, xa = resample_tables("linear_f32", W, Wo, dev, True)
    yo, ya = resample_tables("linear_f32", H, Ho, dev, False)
    out = torch.empty(N, 2, Ho, Wo, dtype=torch.float32, device=dev)
    _launch("pp_resize_flow_linear_cv", _pd(flows), _p(out), N, H, W, Ho, Wo, _p(xo, torch.int32), _p(xa), _p(yo, torch.int32),
            _p(ya))
    return out


# ---------------------------------------------------------------- Cutie mask tracker (web-demos/hugging_face/tracker)
CUTIE_TOPK_MAX = 32


def cutie_topk_readout(mem_key, mem_shrink, mem_value, n_frames, fifo_head, fifo_cap, qk, qe, top_k=30, num_objects=None,
                       out=None, want_selection=False):
    """The working-memory read of MemoryManager.read at top_k (memory_manager.py:160-187): similarity, top-k, softmax and
    the value gather in one pass over ring buffers mem_key [slots*HW,64], mem_shrink [slots*HW], mem_value
    [objects,slots*HW,256] (slots = 1 + fifo_cap; pp_cutie_topk_readout in include/propainter_b200.h) for query keys /
    selections qk, qe [64,HW].  Returns out [num_objects,HW,256] (pixel-major), plus (sel_idx [HW,top_k] int32,
    sel_w [HW,top_k]) when want_selection."""
    HW = qk.shape[-1]
    if qk.shape != (64, HW) or qe.shape != (64, HW):
        raise RuntimeError(f"cutie_topk_readout: qk / qe must be [64,HW], got {tuple(qk.shape)} / {tuple(qe.shape)}")
    slots = 1 + fifo_cap
    if mem_key.shape != (slots * HW, 64) or mem_shrink.numel() != slots * HW or mem_value.shape[1:] != (slots * HW, 256):
        raise RuntimeError("cutie_topk_readout: ring buffers do not match 1 + fifo_cap slots of HW tokens")
    if not 1 <= top_k <= CUTIE_TOPK_MAX:
        raise RuntimeError(f"cutie_topk_readout: top_k={top_k} outside [1, {CUTIE_TOPK_MAX}]")
    nobj = mem_value.shape[0] if num_objects is None else num_objects
    if mem_value.stride(2) != 1 or mem_value.stride(1) != 256:
        raise RuntimeError("cutie_topk_readout: mem_value rows must be dense")
    if out is None:
        out = torch.empty(nobj, HW, 256, device=qk.device, dtype=torch.float32)
    sel_idx = sel_w = None
    if want_selection:
        sel_idx = torch.empty(HW, top_k, device=qk.device, dtype=torch.int32)
        sel_w = torch.empty(HW, top_k, device=qk.device, dtype=torch.float32)
    _launch("pp_cutie_topk_readout", _pd(mem_key), _pd(mem_shrink), _p(mem_value), mem_value.stride(0), n_frames, fifo_head,
            fifo_cap, _pd(qk), _pd(qe), HW, nobj, top_k, _pd(out), _p(sel_idx, torch.int32), _p(sel_w))
    return (out, sel_idx, sel_w) if want_selection else out


def cutie_frame_in(frame_u8, out=None):
    """uint8 frame [H,W,3] on the device -> the normalised, zero-padded network input [1,3,Hp,Wp] (multiples of 16)"""
    if frame_u8.dtype != torch.uint8 or frame_u8.dim() != 3 or frame_u8.shape[-1] != 3:
        raise RuntimeError(f"cutie_frame_in: expected uint8 [H,W,3], got {frame_u8.dtype} {tuple(frame_u8.shape)}")
    H, W, _ = frame_u8.shape
    Hp, Wp = -(-H // 16) * 16, -(-W // 16) * 16
    if out is None:
        out = torch.empty(1, 3, Hp, Wp, device=frame_u8.device, dtype=torch.float32)
    _launch("pp_cutie_frame_in", _pd(frame_u8, torch.uint8), _pd(out), H, W)
    return out


def cutie_labels(prob, lut, H, W, out=None):
    """padded probabilities [K,Hp,Wp] -> uint8 labels [H,W]: argmax, unpad, then lut[K] (uint8, on the device)"""
    K = prob.shape[0]
    if prob.shape[1:] != (-(-H // 16) * 16, -(-W // 16) * 16) or lut.numel() != K or lut.dtype != torch.uint8:
        raise RuntimeError(f"cutie_labels: prob {tuple(prob.shape)} / lut {tuple(lut.shape)} do not fit {H}x{W}")
    if out is None:
        out = torch.empty(H, W, device=prob.device, dtype=torch.uint8)
    _launch("pp_cutie_labels", _pd(prob), K, _pd(lut, torch.uint8), _pd(out, torch.uint8), H, W)
    return out


# ---------------------------------------------------------------- tracking preview (tools/painter.py mask_painter)
def paint_palette():
    """The package's default palette for mask_paint_u8: uint8 [257,3], so every uint8 id k has its row k + 1.  Row 0 is
    black and row 1 white (the contour colour, as in the web demo); row k >= 2 is colour k - 1 of the PASCAL VOC label
    colormap (the bits of k - 1 spread over R, G, B from the most significant bit down), so object 1 is (128, 0, 0),
    object 2 (0, 128, 0), object 3 (128, 128, 0).  The demo's own 22-colour table is passed as `palette` where its exact
    colours are wanted."""
    pal = np.zeros((257, 3), np.uint8)
    pal[1] = 255
    for i in range(1, 256):
        c, rgb = i, [0, 0, 0]
        for j in range(8):
            for ch in range(3):
                rgb[ch] |= ((c >> ch) & 1) << (7 - j)
            c >>= 3
        pal[i + 1] = rgb
    return pal


_PAINT_PALETTE = {}                                # device -> paint_palette() there, made on first use


def mask_paint_u8(frames_u8, labels_u8, palette=None, mask_alpha=0.7, out=None):
    """The web demo's tracking preview (BaseTracker.track's painter loop, base_tracker.py:90-95) for a whole clip on the
    device: frames uint8 [T,H,W,3] and label masks uint8 [T,H,W] (0 = background) -> painted uint8 [T,H,W,3].  Each id k
    present in a frame, in ascending order, is filled with palette row k + 1 at mask_alpha and outlined with row 1
    (mask_painter, tools/painter.py:137-157, contour width 3); bytes equal the reference's for the same palette.
    palette: uint8 [N,3] (tensor or array), default paint_palette().  `out` may be frames_u8 itself.  ValueError for CPU
    tensors, other dtypes or shapes, a palette that is not uint8 [N,3] with N >= 2, mask_alpha outside [0, 1], and a
    present id k with k + 1 >= N (where the reference raises IndexError)."""
    for name, t in (("frames_u8", frames_u8), ("labels_u8", labels_u8)):
        if not isinstance(t, torch.Tensor):
            raise ValueError(f"mask_paint_u8: {name} must be a torch tensor, got {type(t).__name__}")
    if frames_u8.dtype != torch.uint8 or frames_u8.dim() != 4 or frames_u8.shape[-1] != 3 or frames_u8.numel() == 0:
        raise ValueError(f"mask_paint_u8: expected uint8 frames [T,H,W,3], got {frames_u8.dtype} {tuple(frames_u8.shape)}")
    T, H, W, _ = frames_u8.shape
    if labels_u8.dtype != torch.uint8 or tuple(labels_u8.shape) != (T, H, W):
        raise ValueError(f"mask_paint_u8: expected uint8 labels [T,H,W] = {(T, H, W)}, got {labels_u8.dtype} "
                         f"{tuple(labels_u8.shape)}")
    pal = _PAINT_PALETTE.get(frames_u8.device) if palette is None else torch.as_tensor(palette)
    if pal is None:
        pal = torch.from_numpy(paint_palette())
    if pal.dtype != torch.uint8 or pal.dim() != 2 or pal.shape[1] != 3 or pal.shape[0] < 2:
        raise ValueError(f"mask_paint_u8: palette must be uint8 [N,3] with N >= 2, got {pal.dtype} {tuple(pal.shape)}")
    alpha = float(mask_alpha)
    if not 0.0 <= alpha <= 1.0:
        raise ValueError(f"mask_paint_u8: mask_alpha must lie in [0, 1], got {mask_alpha}")
    N = pal.shape[0]
    if N < 257:
        top = int(labels_u8.max())
        if top + 1 >= N:
            raise ValueError(f"mask_paint_u8: id {top} needs palette row {top + 1}, the palette has {N} rows")
    if not frames_u8.is_cuda or labels_u8.device != frames_u8.device:
        raise ValueError(f"mask_paint_u8: frames and labels must be on one CUDA device, got {frames_u8.device} / "
                         f"{labels_u8.device} (there is no CPU path)")
    pal = pal.to(frames_u8.device).contiguous()
    if palette is None:
        _PAINT_PALETTE[frames_u8.device] = pal
    if out is None:
        out = torch.empty_like(frames_u8)
    elif not isinstance(out, torch.Tensor) or out.dtype != torch.uint8 or out.shape != frames_u8.shape or out.device != frames_u8.device:
        raise ValueError("mask_paint_u8: out must be a uint8 tensor shaped and placed like frames_u8")
    ws = torch.empty(_lib.lib().pp_mask_paint_workspace_bytes(T, H, W), dtype=torch.uint8, device=frames_u8.device)
    _launch("pp_mask_paint_u8", _pd(frames_u8, torch.uint8), _pd(labels_u8, torch.uint8), _p(pal, torch.uint8), N,
            (ctypes.c_double * 2)(alpha, 1.0 - alpha), _pd(out, torch.uint8), T, H, W, _p(ws, torch.uint8), ws.numel(),
            launches=3)
    return out
