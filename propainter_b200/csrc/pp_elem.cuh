// Per-element device functions (index arithmetic + sampling rules) of the gather-type kernels.
// Each cites the reference line whose semantics it reproduces.  PP_HD: also compiled by tests/hostsim.
#pragma once
#include "pp_common.cuh"

// ------------------------------------------------------------------------------------------------
// Half-precision clip storage (InferenceConfig.half_storage): fp16 tensors between stages, widened exactly to fp32 on
// load, so every rule below computes in fp32 whatever the storage dtype.  The host build has no cuda_fp16.h: there an
// fp16 value is its IEEE binary16 bit pattern.
#if defined(PP_HOSTSIM)
struct pp_half { uint16_t bits; };
PP_HD float pp_widen(pp_half h) {
  const uint32_t s = (uint32_t)(h.bits & 0x8000u) << 16, e = (h.bits >> 10) & 0x1fu, m = h.bits & 0x3ffu;
  if (e == 0) {                                                   // zero / subnormal: m * 2^-24, exact in fp32
    const float v = ldexpf((float)m, -24);
    return s ? -v : v;
  }
  union { uint32_t u; float f; } r;
  r.u = s | (e == 31 ? 0x7f800000u : (e + 112u) << 23) | (m << 13);
  return r.f;
}
#else
typedef __half pp_half;
PP_HD float pp_widen(__half h) { return __half2float(h); }
#endif
PP_HD float pp_widen(float v) { return v; }

// to_tensors()(frames) * 2 - 1 of one uint8 channel value (core/utils.py:130-170, inference_propainter.py:264): the
// frame conversion of pp_u8_to_frames and the in-kernel widening of pp_img_prop_scan_u8h
PP_HD float pp_u8_frame(uint8_t v) { return PP_SUB(PP_MUL(PP_DIV((float)v, 255.0f), 2.0f), 1.0f); }

// ------------------------------------------------------------------------------------------------
// grid_sample coordinate round trip.
// flow_warp (model/modules/flow_loss_utils.py:34-37): g = 2*(p+f)/max(size-1,1) - 1, then ATen's
// align_corners=True un-normalisation ((g+1)/2)*(size-1).  Kept as separate roundings so that
// 'nearest' picks and the 0.1 / occlusion thresholds land where the reference's do.
PP_HD float pp_warp_coord(float base, float flow, int size) {
  float denom = (float)(size - 1 > 1 ? size - 1 : 1);
  float g = PP_SUB(PP_DIV(PP_MUL(2.0f, PP_ADD(base, flow)), denom), 1.0f);
  return PP_MUL(PP_DIV(PP_ADD(g, 1.0f), 2.0f), (float)(size - 1));
}
// RAFT/utils/utils.py:60-62 (bilinear_sampler): g = 2*x/(W-1) - 1 (no max()).
PP_HD float pp_raft_coord(float pos, int size) {
  float g = PP_SUB(PP_DIV(PP_MUL(2.0f, pos), (float)(size - 1)), 1.0f);
  return PP_MUL(PP_DIV(PP_ADD(g, 1.0f), 2.0f), (float)(size - 1));
}

// Bilinear tap set with zeros padding (grid_sample semantics: out-of-range corners weigh 0).
struct PPTaps {
  int x0, y0;          // top-left corner (may be -1 .. size-1)
  float w00, w01, w10, w11;   // (y0,x0) (y0,x1) (y1,x0) (y1,x1), already zeroed for OOB corners
  int any;             // 0 -> nothing in range
};
PP_HD PPTaps pp_taps(float ix, float iy, int H, int W) {
  PPTaps t;
  t.any = 0; t.x0 = 0; t.y0 = 0; t.w00 = t.w01 = t.w10 = t.w11 = 0.f;
  if (!(ix > -1.0f && ix < (float)W && iy > -1.0f && iy < (float)H)) return t;   // also rejects NaN
  float xf = floorf(ix), yf = floorf(iy);
  int x0 = (int)xf, y0 = (int)yf;
  float wx1 = ix - xf, wy1 = iy - yf;
  float wx0 = (xf + 1.0f) - ix, wy0 = (yf + 1.0f) - iy;
  bool xl = x0 >= 0, xh = x0 + 1 <= W - 1, yl = y0 >= 0, yh = y0 + 1 <= H - 1;
  t.x0 = x0; t.y0 = y0; t.any = 1;
  t.w00 = (yl && xl) ? wx0 * wy0 : 0.f;
  t.w01 = (yl && xh) ? wx1 * wy0 : 0.f;
  t.w10 = (yh && xl) ? wx0 * wy1 : 0.f;
  t.w11 = (yh && xh) ? wx1 * wy1 : 0.f;
  return t;
}
// sample one scalar plane [H][ld] (fp32, or fp16 clip storage widened on load) through a tap set (order nw, ne, sw, se
// like ATen)
template <typename T>
PP_HD float pp_tap_plane(const T* p, int ld, const PPTaps& t) {
  if (!t.any) return 0.f;
  float acc = 0.f;
  const T* r0 = p + (long)t.y0 * ld + t.x0;
  const T* r1 = r0 + ld;
  if (t.w00 != 0.f) acc += pp_widen(r0[0]) * t.w00;
  if (t.w01 != 0.f) acc += pp_widen(r0[1]) * t.w01;
  if (t.w10 != 0.f) acc += pp_widen(r1[0]) * t.w10;
  if (t.w11 != 0.f) acc += pp_widen(r1[1]) * t.w11;
  return acc;
}
// nearest (round-half-to-even, zeros padding): returns linear index or -1
PP_HD long pp_nearest_index(float ix, float iy, int H, int W, int ld) {
  float xn = rintf(ix), yn = rintf(iy);
  if (!(xn >= 0.f && xn <= (float)(W - 1) && yn >= 0.f && yn <= (float)(H - 1))) return -1;
  return (long)yn * ld + (long)xn;
}

// ------------------------------------------------------------------------------------------------
// forward-backward consistency (model/propainter.py:22-31): 1 if |fw + bw(warped)|^2 < 0.01(|fw|^2+|bw|^2)+0.5
PP_HD float pp_fb_valid(float fx, float fy, float bx, float by) {
  float dx = PP_ADD(fx, bx), dy = PP_ADD(fy, by);
  float lhs = PP_ADD(PP_MUL(dx, dx), PP_MUL(dy, dy));
  float mag = PP_ADD(PP_ADD(PP_MUL(fx, fx), PP_MUL(fy, fy)), PP_ADD(PP_MUL(bx, bx), PP_MUL(by, by)));
  float thr = PP_ADD(PP_MUL(0.01f, mag), 0.5f);
  return lhs < thr ? 1.0f : 0.0f;
}

// ------------------------------------------------------------------------------------------------
// One step of the non-learnable image propagation scan (model/propainter.py:144-161), one pixel, in value form: cv the
// pixel's current frame (3 channels), mc its current mask; writes the step's frame values to ov and returns its mask.
// prev / mprev / flows planar ([3][H*W], [H*W], [2][H*W]); flows fp32 or fp16.  `nearest` selects :149's mode.
template <typename TF>
PP_HD float pp_imgprop_values(int pix, int H, int W, const float* cv, float mc, const float* prev, const float* mprev,
                              const TF* fprop, const TF* fcheck, float* ov, int nearest) {
  const int HW = H * W;
  int y = pix / W, x = pix - y * W;
  float fx = pp_widen(fprop[pix]), fy = pp_widen(fprop[HW + pix]);
  float ix = pp_warp_coord((float)x, fx, W), iy = pp_warp_coord((float)y, fy, H);
  PPTaps t = pp_taps(ix, iy, H, W);
  float bx = pp_tap_plane(fcheck, W, t), by = pp_tap_plane(fcheck + HW, W, t);
  float valid = pp_fb_valid(fx, fy, bx, by);
  float mw = pp_tap_plane(mprev, W, t) > 0.1f ? 1.0f : 0.0f;            // binary_mask(:156)
  float gate = PP_MUL(PP_MUL(mc, valid), PP_SUB(1.0f, mw));
  float use = gate > 0.1f ? 1.0f : 0.0f;                                 // :158
  long ni = nearest ? pp_nearest_index(ix, iy, H, W, W) : 0;
  for (int c = 0; c < 3; ++c) {
    float wv;
    if (nearest) wv = ni >= 0 ? prev[(long)c * HW + ni] : 0.f;
    else wv = pp_tap_plane(prev + (long)c * HW, W, t);
    ov[c] = PP_ADD(PP_MUL(use, wv), PP_MUL(PP_SUB(1.0f, use), cv[c]));   // :159
  }
  float m2 = PP_MUL(mc, PP_SUB(1.0f, PP_MUL(valid, PP_SUB(1.0f, mw))));  // :161
  return m2 > 0.1f ? 1.0f : 0.0f;
}
// the same step on planar fp32 frames: cur, out [3][H*W]; mcur, mout [H*W]
PP_HD void pp_imgprop_pixel(int pix, int H, int W, const float* cur, const float* mcur, const float* prev,
                            const float* mprev, const float* fprop, const float* fcheck, float* out,
                            float* mout, int nearest) {
  const int HW = H * W;
  const float cv[3] = {cur[pix], cur[HW + pix], cur[2 * HW + pix]};
  float ov[3];
  const float m = pp_imgprop_values(pix, H, W, cv, mcur[pix], prev, mprev, fprop, fcheck, ov, nearest);
  for (int c = 0; c < 3; ++c) out[(long)c * HW + pix] = ov[c];
  mout[pix] = m;
}
// The updated frame of one channel (inference_propainter.py:389-390, :402; ProPainterPipeline.propagate_images):
// frames * (1 - masks) + prop * masks in the torch expression's order, one rounding per operation.
PP_HD float pp_imgprop_compose(float frame, float prop, float m) {
  return PP_ADD(PP_MUL(frame, PP_SUB(1.0f, m)), PP_MUL(prop, m));
}

// ------------------------------------------------------------------------------------------------
// Learnable feature propagation: per-pixel sampling coordinate + validity (propainter.py:146-148).
// flows are pixel-interleaved [h][w][2] (internal layout of the 1/4-res flows).
struct PPCond { float ix, iy, valid, fx, fy; };
PP_HD PPCond pp_cond_pixel(int y, int x, int h, int w, const float* fprop, const float* fcheck) {
  PPCond c;
  long pix = (long)y * w + x;
  c.fx = fprop[2 * pix]; c.fy = fprop[2 * pix + 1];
  c.ix = pp_warp_coord((float)x, c.fx, w); c.iy = pp_warp_coord((float)y, c.fy, h);
  PPTaps t = pp_taps(c.ix, c.iy, h, w);
  float bx = 0.f, by = 0.f;
  if (t.any) {
    const float* r0 = fcheck + 2 * ((long)t.y0 * w + t.x0);
    const float* r1 = r0 + 2 * w;
    if (t.w00 != 0.f) { bx += r0[0] * t.w00; by += r0[1] * t.w00; }
    if (t.w01 != 0.f) { bx += r0[2] * t.w01; by += r0[3] * t.w01; }
    if (t.w10 != 0.f) { bx += r1[0] * t.w10; by += r1[1] * t.w10; }
    if (t.w11 != 0.f) { bx += r1[2] * t.w11; by += r1[3] * t.w11; }
  }
  c.valid = pp_fb_valid(c.fx, c.fy, bx, by);
  return c;
}
// 4 consecutive channels of a pixel-major feature map through a tap set
PP_HD float4 pp_tap_nhwc4(const float* feat, int ld, int w, const PPTaps& t, int c) {
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
  if (!t.any) return a;
  const float* p00 = feat + ((long)t.y0 * w + t.x0) * ld + c;
#define PP_ACC4(ptr, wt)                                                        \
  if ((wt) != 0.f) { const float4 v = *reinterpret_cast<const float4*>(ptr);   \
    a.x += v.x * (wt); a.y += v.y * (wt); a.z += v.z * (wt); a.w += v.w * (wt); }
  PP_ACC4(p00, t.w00)
  PP_ACC4(p00 + ld, t.w01)
  PP_ACC4(p00 + (long)w * ld, t.w10)
  PP_ACC4(p00 + (long)w * ld + ld, t.w11)
#undef PP_ACC4
  return a;
}

// ------------------------------------------------------------------------------------------------
// Modulated deformable 3x3 sampling (torchvision.ops.deform_conv2d semantics, SURVEY.md §8c):
// `o` = the pixel's raw conv_offset output (432 = 16 groups x 27): channels [0,288) are (dy,dx) pairs
// at g*18+2k+{0,1}, channels [288,432) the modulation logits at 288+g*9+k.
// propainter.py:58-65 / recurrent_flow_completion.py:34-40: offset = max_res*tanh(o) (+ flow.flip), mask = sigmoid.
struct PPDTap { float py, px, m; };
PP_HD PPDTap pp_deform_tap(const float* o, const float* flow_xy, float max_res, int g, int k, int y, int x) {
  PPDTap t;
  float oy = max_res * tanhf(o[g * 18 + 2 * k]);
  float ox = max_res * tanhf(o[g * 18 + 2 * k + 1]);
  if (flow_xy) { oy += flow_xy[1]; ox += flow_xy[0]; }
  t.m = 1.0f / (1.0f + expf(-o[288 + g * 9 + k]));
  t.py = (float)(y - 1 + k / 3) + oy;
  t.px = (float)(x - 1 + k % 3) + ox;
  return t;
}
// corner weights of torchvision's bilinear_interpolate folded with the modulation scalar
struct PPDW { int y0, x0; float w00, w01, w10, w11; };
PP_HD PPDW pp_deform_weights(const PPDTap& t, int H, int W) {
  PPDW d;
  d.y0 = d.x0 = 0; d.w00 = d.w01 = d.w10 = d.w11 = 0.f;
  if (!(t.py > -1.0f && t.py < (float)H && t.px > -1.0f && t.px < (float)W)) return d;
  float yf = floorf(t.py), xf = floorf(t.px);
  d.y0 = (int)yf; d.x0 = (int)xf;
  float ly = t.py - yf, lx = t.px - xf, hy = 1.0f - ly, hx = 1.0f - lx;
  bool yl = d.y0 >= 0, yh = d.y0 + 1 <= H - 1, xl = d.x0 >= 0, xh = d.x0 + 1 <= W - 1;
  d.w00 = (yl && xl) ? hy * hx * t.m : 0.f;
  d.w01 = (yl && xh) ? hy * lx * t.m : 0.f;
  d.w10 = (yh && xl) ? ly * hx * t.m : 0.f;
  d.w11 = (yh && xh) ? ly * lx * t.m : 0.f;
  return d;
}
PP_HD float pp_deform_sample1(const float* x, int ld, int W, const PPDW& d, int c) {
  float a = 0.f;
  const float* p = x + ((long)d.y0 * W + d.x0) * ld + c;
  if (d.w00 != 0.f) a += p[0] * d.w00;
  if (d.w01 != 0.f) a += p[ld] * d.w01;
  if (d.w10 != 0.f) a += p[(long)W * ld] * d.w10;
  if (d.w11 != 0.f) a += p[(long)W * ld + ld] * d.w11;
  return a;
}

// ------------------------------------------------------------------------------------------------
// RAFT correlation pyramid.  Level l plane of one source pixel: [h>>l][ld_l], ld_l = roundup4(w>>l)
// so every row starts 16-byte aligned (TMA-able).
PP_HD int pp_corr_ld(int w_l) { return (w_l + 3) & ~3; }
// RAFT/corr.py:25-27: 2x2 average pooling, ATen order ((a+b)+c)+d then /4
PP_HD float pp_pool4(const float* src, int ld, int y, int x) {
  const float* p = src + (long)(2 * y) * ld + 2 * x;
  float s = PP_ADD(PP_ADD(PP_ADD(p[0], p[1]), p[ld]), p[ld + 1]);
  return PP_DIV(s, 4.0f);
}
// RAFT/corr.py:29-50 with radius R (4: the basic model, 3: RAFT-small, raft.py:29-33): output channel
// l*K^2 + a*K + b (K = 2R+1) samples level l at (cx/2^l + (a-R), cy/2^l + (b-R));
// note the first window axis moves x (reference quirk: delta = stack(meshgrid(dy,dx)) added to (x,y)).
template <int R>
PP_HD float pp_corr_tap_r(const float* plane, int Hl, int Wl, int ld, float cx, float cy, int lvl, int a, int b) {
  float s = (float)(1 << lvl);
  float x = PP_ADD(PP_DIV(cx, s), (float)(a - R));
  float y = PP_ADD(PP_DIV(cy, s), (float)(b - R));
  PPTaps t = pp_taps(pp_raft_coord(x, Wl), pp_raft_coord(y, Hl), Hl, Wl);
  return pp_tap_plane(plane, ld, t);
}
PP_HD float pp_corr_tap(const float* plane, int Hl, int Wl, int ld, float cx, float cy, int lvl, int a, int b) {
  return pp_corr_tap_r<4>(plane, Hl, Wl, ld, cx, cy, lvl, a, b);
}
// AlternateCorrBlock (RAFT/corr.py:83-111) without a stored plane: level `lvl` is sampled from a T x T tile of dot
// products (T = 2R+2), tile[j*T + i] = f1 . f2_l[ty0 + j][tx0 + i] / sqrt(D) (zero outside the level), whose origin is
// the floored level centre minus the window radius.  Far-away or non-finite centres get a tile wholly outside the level.
template <int R>
PP_HD int pp_corr_tile_origin_r(float c, int lvl) {
  float v = floorf(PP_DIV(c, (float)(1 << lvl)));
  v = fminf(fmaxf(v, -1.0e6f), 1.0e6f);
  return (int)v - R;
}
PP_HD int pp_corr_tile_origin(float c, int lvl) { return pp_corr_tile_origin_r<4>(c, lvl); }
// Tap (a, b) of level `lvl` from that tile by the rule of pp_corr_tap_r.  The grid_sample coordinate round trip can move
// a corner by one step at an integer boundary; a corner that lands off the tile then weighs 0 or a few ulp and is dropped.
template <int R>
PP_HD float pp_corr_tap_tile_r(const float* tile, int tx0, int ty0, int Hl, int Wl, float cx, float cy, int lvl, int a, int b) {
  constexpr int T = 2 * R + 2;
  float s = (float)(1 << lvl);
  float x = PP_ADD(PP_DIV(cx, s), (float)(a - R));
  float y = PP_ADD(PP_DIV(cy, s), (float)(b - R));
  PPTaps t = pp_taps(pp_raft_coord(x, Wl), pp_raft_coord(y, Hl), Hl, Wl);
  if (!t.any) return 0.f;
  const int i = t.x0 - tx0, j = t.y0 - ty0;
  const bool i0 = i >= 0 && i < T, i1 = i >= -1 && i < T - 1, j0 = j >= 0 && j < T, j1 = j >= -1 && j < T - 1;
  float acc = 0.f;
  if (t.w00 != 0.f && j0 && i0) acc += tile[j * T + i] * t.w00;
  if (t.w01 != 0.f && j0 && i1) acc += tile[j * T + i + 1] * t.w01;
  if (t.w10 != 0.f && j1 && i0) acc += tile[(j + 1) * T + i] * t.w10;
  if (t.w11 != 0.f && j1 && i1) acc += tile[(j + 1) * T + i + 1] * t.w11;
  return acc;
}
PP_HD float pp_corr_tap_tile(const float* tile, int tx0, int ty0, int Hl, int Wl, float cx, float cy, int lvl, int a, int b) {
  return pp_corr_tap_tile_r<4>(tile, tx0, ty0, Hl, Wl, cx, cy, lvl, a, b);
}

// upflow8 (RAFT/utils/utils.py:80-82, RAFT-small's upsampling, raft.py:136-137): 8 * F.interpolate(flow, (8h, 8w),
// bilinear, align_corners=True), restated from ATen's CPU upsample_bilinear2d: scale = float(in-1) / (out-1),
// src = scale * dst, i0 = min(floor(src), in-1), l1 = clamp(src - i0, 0, 1), i1 = i0 + (i0 < in-1), l0 = 1 - l1.
// ATen's x86 build (the AVX2 / AVX-512 copies of the kernel are compiled with FMA) contracts each `t0*w0 + t1*w1` of the
// separable blend into fma(t0, w0, t1*w1): row values fma(v00, lx0, v01*lx1), then fma(row0, ly0, row1*ly1), then * 8.
// The rule does exactly that, with explicit roundings; it equals ATen bit for bit on every grid RAFT produces
// (h, w >= 16; measured with torch 2.11 on x86).  Plain mul-add (no FMA) differs by up to 1 ulp on ~20% of pixels.
struct PPLin { int i0, i1; float l0, l1; };
// the taps and weights of one source coordinate: i0 = min(floor(src), in-1), l1 = clamp(src - i0, 0, 1)
PP_HD PPLin pp_lin_taps(float src, int in) {
  PPLin u;
  u.i0 = (int)floorf(src);
  if (u.i0 > in - 1) u.i0 = in - 1;
  u.l1 = fminf(fmaxf(PP_SUB(src, (float)u.i0), 0.0f), 1.0f);
  u.i1 = u.i0 + (u.i0 < in - 1 ? 1 : 0);
  u.l0 = PP_SUB(1.0f, u.l1);
  return u;
}
PP_HD PPLin pp_upflow8_coord(int dst, int in) {
  const int out = 8 * in;
  const float scale = out > 1 ? PP_DIV((float)(in - 1), (float)(out - 1)) : 0.0f;
  return pp_lin_taps(PP_MUL(scale, (float)dst), in);
}
// ATen's separable blend as its x86 build contracts it (see above)
PP_HD float pp_lin_blend(float v00, float v01, float v10, float v11, const PPLin& uy, const PPLin& ux) {
  const float t0 = PP_FMA(v00, ux.l0, PP_MUL(v01, ux.l1));
  const float t1 = PP_FMA(v10, ux.l0, PP_MUL(v11, ux.l1));
  return PP_FMA(t0, uy.l0, PP_MUL(t1, uy.l1));
}
PP_HD float pp_upflow8_blend(float v00, float v01, float v10, float v11, const PPLin& uy, const PPLin& ux) {
  return PP_MUL(8.0f, pp_lin_blend(v00, v01, v10, v11, uy, ux));
}

// F.interpolate(img, size=(h, w), mode='bilinear', align_corners=False), no antialias (scripts/compute_flow.py:81-89),
// restated from ATen's CPU upsample_bilinear2d the same way: scale = float(in) / out, src = max(scale * (dst + 0.5) - 0.5,
// 0) with the x86 build's FMA contraction (fma(scale, dst + 0.5, -0.5)), then the taps and the blend above.  Equals ATen's
// contiguous NCHW kernel bit for bit on uint8 / 255 frames at every output size RAFT accepts (measured with torch 2.11 on
// x86: down- and up-scaling, odd source sizes, identity); without the FMA in src about 16% of the values of 720x1280 ->
// 240x432 differ.  Small outputs (e.g. 74x48) take another ATen code path that differs from this rule by a few ulp.
// At in == out it picks the source pixel with weight 1 exactly.
PP_HD PPLin pp_resize_coord(int dst, int in, int out) {
  const float scale = PP_DIV((float)in, (float)out);
  return pp_lin_taps(fmaxf(PP_FMA(scale, PP_ADD((float)dst, 0.5f), -0.5f), 0.0f), in);
}
// One value of compute_flow.py:67-92 for one channel: ToTensor's v / 255 at each tap, the resize, then img*2 - 1 as two
// roundings.  At the identity size this is pp_u8_frame.
PP_HD float pp_u8_frame_resized(uint8_t v00, uint8_t v01, uint8_t v10, uint8_t v11, const PPLin& uy, const PPLin& ux) {
  const float b = pp_lin_blend(PP_DIV((float)v00, 255.0f), PP_DIV((float)v01, 255.0f), PP_DIV((float)v10, 255.0f),
                               PP_DIV((float)v11, 255.0f), uy, ux);
  return PP_SUB(PP_MUL(b, 2.0f), 1.0f);
}

// RAFT/raft.py:73-84: convex 8x upsampling of one low-res pixel's (i,j) sub-pixel.
// mask pixel-major [..][576], channel k*64 + i*8 + j; flow_lr pixel-interleaved [h][w][2].
PP_HD float2 pp_convex_up(const float* mask_px, float mask_scale, const float* flow_lr, int h, int w, int y, int x,
                         int i, int j) {
  float lg[9], mx = -INFINITY;
  for (int k = 0; k < 9; ++k) { lg[k] = mask_scale * mask_px[k * 64 + i * 8 + j]; mx = fmaxf(mx, lg[k]); }
  float den = 0.f;
  for (int k = 0; k < 9; ++k) { lg[k] = expf(lg[k] - mx); den += lg[k]; }
  float ox = 0.f, oy = 0.f;
  for (int k = 0; k < 9; ++k) {
    int yy = y + k / 3 - 1, xx = x + k % 3 - 1;
    if (yy < 0 || yy >= h || xx < 0 || xx >= w) continue;
    float p = lg[k] / den;
    const float* f = flow_lr + 2 * ((long)yy * w + xx);
    ox += p * (8.0f * f[0]); oy += p * (8.0f * f[1]);
  }
  float2 r; r.x = ox; r.y = oy;
  return r;
}

// ------------------------------------------------------------------------------------------------
// InstanceNorm statistics (nn.InstanceNorm2d, affine=False; k_inorm_stats / k_inorm_apply of gather_kernels.cu).  Each
// (sample, channel) is shifted by its value at pixel 0, p, and the sums of d = x - p and d^2 are kept in double: d and
// d^2 of fp32 inputs are exact in double, so the variance E[d^2] - E[d]^2 does not cancel the way E[x^2] - mean^2 in
// fp32 does when |mean| >> std, and a constant channel gives d = 0, mean = p exactly and 0 out.
// Splits of the pixel range per sample: ~4 CTAs per SM over the whole batch, >= 16 rows each.
PP_HD int pp_inorm_splits(int n, long HW) {
  int s = (592 + n - 1) / n;
  if (s > 64) s = 64;
  if ((long)s * 16 > HW) s = (int)((HW + 15) / 16);
  return s < 1 ? 1 : s;
}
PP_HD void pp_inorm_acc(double& s, double& q, float x, float p) {
  const double d = (double)x - (double)p;
  s += d;
  q += d * d;
}
struct PPNormStat { float mean, rstd; };
// the sums over all HW pixels -> fp32 mean and 1/sqrt(biased var + eps), each rounded once from double
PP_HD PPNormStat pp_inorm_fold(double s, double q, long HW, float p, float eps) {
  const double md = s / (double)HW;
  double var = q / (double)HW - md * md;
  if (var < 0.0) var = 0.0;
  PPNormStat r;
  r.mean = (float)((double)p + md);
  r.rstd = (float)(1.0 / sqrt(var + (double)eps));
  return r;
}
// one output: (x - mean) * rstd, then the optional ReLU, residual add and ReLU of ResidualBlock (extractor.py:49-57)
PP_HD float pp_inorm_out(float x, const PPNormStat& st, int relu, const float* res, int post_relu) {
  float y = PP_MUL(PP_SUB(x, st.mean), st.rstd);
  if (relu) y = fmaxf(y, 0.f);
  if (res) y = PP_ADD(y, *res);
  if (post_relu) y = fmaxf(y, 0.f);
  return y;
}

// ------------------------------------------------------------------------------------------------
// InpaintGenerator.forward down-sampling (propainter.py:338-342; stencils pinned in SURVEY.md §8c):
// bilinear 1/4 (align_corners=False) == mean of the centre 2x2 of each 4x4 block; then /4.
// The flow plane is fp32 or fp16 clip storage (widened on load).
template <typename T>
PP_HD float pp_flow_ds4(const T* plane, int W, int y, int x) {
  const T* p = plane + (long)(4 * y + 1) * W + 4 * x + 1;
  float top = 0.5f * pp_widen(p[0]) + 0.5f * pp_widen(p[1]);
  float bot = 0.5f * pp_widen(p[W]) + 0.5f * pp_widen(p[W + 1]);
  return PP_DIV(0.5f * top + 0.5f * bot, 4.0f);
}

// ------------------------------------------------------------------------------------------------
// Soft-split geometry (kernel 7, stride 3, pad 3; sparse_transformer.py:19-31,74-101).
// FusionFeedForward's fold -> /normaliser -> unfold on the fc1 activations.  Hidden columns are stored
// tap-major: col = tap*CH + c (the fc1 rows / fc2 columns are permuted once at weight-pack time).
PP_HD float pp_ffn_fold(const float* Y, int ldy, int CH, int fh, int fw, int y, int x, int c) {
  // sum of all (token, tap) contributions that land on feature pixel (y,x), divided by their count
  float s = 0.f; int n = 0;
  for (int ty = (y + 3) / 3, ky; ty >= 0 && (ky = y + 3 - 3 * ty) < 7; --ty) {
    if (ty >= fh) continue;
    for (int tx = (x + 3) / 3, kx; tx >= 0 && (kx = x + 3 - 3 * tx) < 7; --tx) {
      if (tx >= fw) continue;
      s += Y[((long)ty * fw + tx) * ldy + (ky * 7 + kx) * CH + c];
      ++n;
    }
  }
  return s / (float)n;
}
PP_HD float pp_gelu(float v) { return 0.5f * v * (1.0f + erff(v * 0.70710678118654752440f)); }

// ------------------------------------------------------------------------------------------------
// x2 bilinear up-sampling with align_corners=True (ATen upsample_bilinear2d): src = dst*(in-1)/(2in-1)
struct PPUp { int i0, step; float l0, l1; };
PP_HD PPUp pp_up2_coord(int dst, int in) {
  PPUp u;
  const float scale = (float)(in - 1) / (float)(2 * in - 1);
  const float s = scale * (float)dst;
  u.i0 = (int)s;
  u.step = u.i0 < in - 1 ? 1 : 0;
  u.l1 = s - (float)u.i0;
  u.l0 = 1.0f - u.l1;
  return u;
}
PP_HD float pp_up2_blend(float v00, float v01, float v10, float v11, const PPUp& uy, const PPUp& ux) {
  return uy.l0 * (ux.l0 * v00 + ux.l1 * v01) + uy.l1 * (ux.l0 * v10 + ux.l1 * v11);
}

// ------------------------------------------------------------------------------------------------
// Final compositing (inference_propainter.py:437-450): uint8 truncation, masked composite,
// order-dependent 1/2-1/2 running blend (truncating again).
PP_HD uint8_t pp_composite_img(float pred, float mask, uint8_t ori) {
  float v = PP_MUL(PP_DIV(PP_ADD(pred, 1.0f), 2.0f), 255.0f);
  uint8_t p8 = (uint8_t)(int)v;                     // numpy astype(uint8) of a value in [0,255]
  uint8_t bm = (uint8_t)(int)mask;
  return (uint8_t)(p8 * bm + ori * (uint8_t)(1 - bm));
}
PP_HD uint8_t pp_composite(float pred, float mask, uint8_t ori, uint8_t prev, int first) {
  uint8_t img = pp_composite_img(pred, mask, ori);
  if (first) return img;
  float b = PP_ADD(PP_MUL((float)prev, 0.5f), PP_MUL((float)img, 0.5f));
  return (uint8_t)(int)b;
}
// The evaluation script's compositing (scripts/evaluate_propainter.py:166-179): the same uint8 `img`, but a later visit
// blends into a float32 frame and is not truncated again, so a frame seen by k windows holds multiples of 2^-(k-1).
PP_HD float pp_composite_f32(float pred, float mask, uint8_t ori, float prev, int first) {
  float img = (float)pp_composite_img(pred, mask, ori);
  if (first) return img;
  return PP_ADD(PP_MUL(prev, 0.5f), PP_MUL(img, 0.5f));
}

// ------------------------------------------------------------------------------------------------
// Mask preparation (inference_propainter.py:93-107): scipy.ndimage.binary_dilation with the default cross
// structure, `iterations` times == union over the L1 ball of that radius; iterations = 0 -> plain binarisation.
PP_HD float pp_mask_dilate_pixel(const uint8_t* m, int H, int W, int y, int x, int iterations) {
  for (int dy = -iterations; dy <= iterations; ++dy) {
    const int yy = y + dy;
    if (yy < 0 || yy >= H) continue;
    const int r = iterations - (dy < 0 ? -dy : dy);
    for (int dx = -r; dx <= r; ++dx) {
      const int xx = x + dx;
      if (xx >= 0 && xx < W && m[(long)yy * W + xx] != 0) return 1.0f;
    }
  }
  return 0.0f;
}

// ------------------------------------------------------------------------------------------------
// Video outpainting (extrapolation, inference_propainter.py:117-156).  The h x w source sits at (top, left) of the
// zero canvas; canvas pixel (y, x) shows source pixel pp_outpaint_src (-1: border, value 0).
PP_HD long pp_outpaint_src(int y, int x, int top, int left, int h, int w) {
  const int sy = y - top, sx = x - left;
  return (sy >= 0 && sy < h && sx >= 0 && sx < w) ? (long)sy * w + sx : -1;
}
// Mask value of canvas pixel (y, x): 0 inside [top+rim_h, top+h-rim_h) x [left+rim_w, left+w-rim_w), 1 elsewhere
// (:144-151).  rim (4 if offset > 10 else 0) gives the flow mask, rim 0 the dilated mask.  Like the numpy slice, an
// empty range (h <= 2*rim_h) clears nothing.
PP_HD float pp_outpaint_mask(int y, int x, int top, int left, int h, int w, int rim_h, int rim_w) {
  const bool in = y >= top + rim_h && y < top + h - rim_h && x >= left + rim_w && x < left + w - rim_w;
  return in ? 0.0f : 1.0f;
}
// Green preview of the masked region (inference_propainter.py:251-261), one channel c of one pixel, in float64 as numpy
// computes it: fuse = (1-a)*img + a*green, mask*fuse + (1-mask)*img, astype(uint8) truncation; a = 0.6, green = (0,255,0).
PP_HD uint8_t pp_mask_overlay(uint8_t img, float mask, int c) {
  const double a = 0.6, v = (double)img, m = (double)mask;
  const double green = c == 1 ? 255.0 : 0.0;
  const double fuse = PP_DADD(PP_DMUL(PP_DSUB(1.0, a), v), PP_DMUL(a, green));
  const double out = PP_DADD(PP_DMUL(m, fuse), PP_DMUL(PP_DSUB(1.0, m), v));
  return (uint8_t)(int)out;
}

// ------------------------------------------------------------------------------------------------
// Optical-flow colour coding: the Middlebury colour wheel of RAFT/utils/flow_viz.py (numpy, one [H,W,2] frame at a
// time) and RAFT/utils/flow_viz_pt.py (torch, normalised over the whole batch).  Each rule follows the arithmetic the
// reference executes, one rounding per operation.

// make_colorwheel (flow_viz.py:20-67 = flow_viz_pt.py:73-118): entry k in [0, 55), channel c.  The reference's
// floor(255 * i / n) is an exact integer quotient here (a non-integral 255 i / n lies >= 1/15 from an integer).
PP_HD int pp_colorwheel(int k, int c) {
  int r, g, b;
  if (k < 15) { r = 255; g = 255 * k / 15; b = 0; }                              // RY
  else if (k < 21) { r = 255 - 255 * (k - 15) / 6; g = 255; b = 0; }              // YG
  else if (k < 25) { r = 0; g = 255; b = 255 * (k - 21) / 4; }                    // GC
  else if (k < 36) { r = 0; g = 255 - 255 * (k - 25) / 11; b = 255; }             // CB
  else if (k < 49) { r = 255 * (k - 36) / 13; g = 0; b = 255; }                   // BM
  else { r = 255; g = 0; b = 255 - 255 * (k - 49) / 6; }                          // MR
  return c == 0 ? r : (c == 1 ? g : b);
}
// np.clip(flow, 0, clip_flow) (flow_viz.py:124): minimum(maximum(x, 0), c).  A negative component becomes 0, -0.0 stays
// -0.0 (it is not below 0) and NaN passes, as numpy does.
PP_HD float pp_flow_clip(float x, float c) {
  x = x < 0.0f ? 0.0f : x;
  return x > c ? c : x;
}
// float32 sqrt(u^2 + v^2): rad of flow_viz.py:127 / :88, the norm of flow_viz_pt.py:29 / :55
PP_HD float pp_flow_rad(float u, float v) { return PP_SQRT(PP_ADD(PP_MUL(u, u), PP_MUL(v, v))); }
// float32 atan2 rounded once from float64: within half an ulp of the exact angle except for double-rounding ties.
// numpy's and ATen's float32 atan2 are not correctly rounded (up to 3 ulp off in numpy's AVX-512 path), so a pixel
// whose colour sits on a rounding boundary may differ by one level (INTEGRATION.md §3).  Signed zeros follow C99:
// atan2(-0.0, -u) = -pi, atan2(+0.0, -u) = +pi.
PP_HD float pp_atan2f(float y, float x) { return (float)atan2((double)y, (double)x); }
// wheel position of a normalised flow vector: (atan2(-v, -u) / pi + 1) / 2 * 54 in float32 (flow_viz.py:89-90,
// flow_viz_pt.py:56-57; both divide by float32 pi).  k0 is clamped to [0, 54] only for memory safety: a finite input
// gives fk in [0, 54].
struct PPWheelPos { float fk; int k0, k1; };
PP_HD PPWheelPos pp_wheel_pos(float un, float vn) {
  const float a = PP_DIV(pp_atan2f(-vn, -un), 3.14159274101257324f);
  PPWheelPos w;
  w.fk = PP_MUL(PP_DIV(PP_ADD(a, 1.0f), 2.0f), 54.0f);
  const int k0 = (int)floorf(w.fk);
  const int k = k0 < 0 ? 0 : (k0 > 54 ? 54 : k0);
  w.k0 = k;
  w.k1 = k < 54 ? k + 1 : 0;                                                      // k1[k1 == ncols] = 0
  return w;
}
// numpy variant, one pixel: flow_to_image (flow_viz.py:109-132) + flow_uv_to_colors (:70-106) for float32 input under
// numpy >= 2 (NEP 50).  den = rad_max + 1e-5 of the (clipped) frame in float32; u, v already clipped.  float32 through
// fk; f = fk - k0 (float32 - int32) is float64, and so is everything after it: col0/col1, the blend, the rad <= 1
// lerp (float32 rad widened) and the reachable rad > 1 branch (x 0.75), floor(255 col) cast to uint8.
PP_HD void pp_flowviz_np(float u, float v, float den, int bgr, uint8_t* rgb) {
  const float un = PP_DIV(u, den), vn = PP_DIV(v, den);
  const float rad = pp_flow_rad(un, vn);
  const PPWheelPos w = pp_wheel_pos(un, vn);
  const double f = PP_DSUB((double)w.fk, (double)w.k0);
  for (int c = 0; c < 3; ++c) {
    const double col0 = PP_DDIV((double)pp_colorwheel(w.k0, c), 255.0);
    const double col1 = PP_DDIV((double)pp_colorwheel(w.k1, c), 255.0);
    double col = PP_DADD(PP_DMUL(PP_DSUB(1.0, f), col0), PP_DMUL(f, col1));
    col = rad <= 1.0f ? PP_DSUB(1.0, PP_DMUL((double)rad, PP_DSUB(1.0, col))) : PP_DMUL(col, 0.75);
    rgb[bgr ? 2 - c : c] = (uint8_t)(int)floor(PP_DMUL(255.0, col));
  }
}
// torch variant, one pixel: flow_to_image + _normalized_flow_to_image (flow_viz_pt.py:6-70), all float32.  den =
// max_norm + FLT_EPSILON over the whole batch; ATen's CPU kernel divides (no reciprocal).  No rad > 1 branch: when the
// largest vector normalises to just above 1, 1 - norm (1 - col) can fall below 0 and floor gives -1, which the
// float -> uint8 copy wraps to 255 through int32 (x86 ATen); the rule keeps that wrap.
PP_HD void pp_flowviz_pt(float u, float v, float den, int bgr, uint8_t* rgb) {
  const float un = PP_DIV(u, den), vn = PP_DIV(v, den);
  const float norm = pp_flow_rad(un, vn);
  const PPWheelPos w = pp_wheel_pos(un, vn);
  const float f = PP_SUB(w.fk, (float)w.k0);
  for (int c = 0; c < 3; ++c) {
    const float col0 = PP_DIV((float)pp_colorwheel(w.k0, c), 255.0f);
    const float col1 = PP_DIV((float)pp_colorwheel(w.k1, c), 255.0f);
    float col = PP_ADD(PP_MUL(PP_SUB(1.0f, f), col0), PP_MUL(f, col1));
    col = PP_SUB(1.0f, PP_MUL(norm, PP_SUB(1.0f, col)));
    rgb[bgr ? 2 - c : c] = (uint8_t)(int)floorf(PP_MUL(255.0f, col));
  }
}

// ---- tracking preview: BaseTracker.track's painter loop (web-demos/hugging_face/tracker/base_tracker.py:90-95) ----
// mask_painter (tools/painter.py:137-157) at contour_width 3 paints object k over the image in two steps: the fill where
// the label is k, then the contour colour where |clip(fore - back, -3, 3)| / max over the frame, with values above 0.5 set
// to 1, has 1 - that value > 0.5 (vis_add_mask, :106-110).  fore / back are cv2.distanceTransform(DIST_L2, 3) of the
// object and of its complement: a 3x3 chamfer accumulated in float32 with steps a = 0.955 (axial), b = 1.3693 (diagonal).
// Clipped at 3, only six path sums stay below 3, so min(DT, 3) of a pixel is the least of the table below over the
// opposite-class pixels of its 7x7 window (pixels outside the frame never count), or 3 if there are none.

// path sum of the chamfer to offset (dy, dx), in cv2's float32 order; 3 (the clip) for every longer path and for (0, 0)
PP_HD float pp_paint_chamfer(int dy, int dx) {
  dy = dy < 0 ? -dy : dy;
  dx = dx < 0 ? -dx : dx;
  const int p = dy > dx ? dy : dx, q = dy > dx ? dx : dy;
  const float a = 0.955f, b = 1.3693f;
  if (p == 1) return q == 0 ? a : b;
  if (p == 2) return q == 0 ? PP_ADD(a, a) : (q == 1 ? PP_ADD(a, b) : PP_ADD(b, b));
  if (p == 3 && q == 0) return PP_ADD(PP_ADD(a, a), a);
  return 3.0f;
}
// v = |clip(fore - back, -3, 3)| of the pixel at c for object k: min(DT, 3) inside the object against the pixels that are
// not k, outside it against the pixels that are.  c points into a label window (rows ld apart, -1 outside the frame)
// holding the 3 rows / columns around it.
template <typename L>
PP_HD float pp_paint_dist(const L* c, int ld, int k) {
  const bool in = c[0] == k;
  float v = 3.0f;
#pragma unroll
  for (int dy = -3; dy <= 3; ++dy)
#pragma unroll
    for (int dx = -3; dx <= 3; ++dx) {
      const float d = pp_paint_chamfer(dy, dx);
      const int l = c[dy * ld + dx];
      if (d < 3.0f && l >= 0 && (l == k) != in) v = fminf(v, d);
    }
  return v;
}
// the smallest non-zero id above prev among the pixel and the window pixels the table reaches (256 if none).  An id
// that only occurs farther away has v = 3 here and paints nothing at this pixel.
template <typename L>
PP_HD int pp_paint_next_id(const L* c, int ld, int prev) {
  int k = 256;
#pragma unroll
  for (int dy = -3; dy <= 3; ++dy)
#pragma unroll
    for (int dx = -3; dx <= 3; ++dx) {
      const int l = c[dy * ld + dx];
      if ((pp_paint_chamfer(dy, dx) < 3.0f || (dy == 0 && dx == 0)) && l > prev && l < k) k = l;
    }
  return k;
}
// The contour test 1 - v / M > 0.5 with M the maximum of v over the frame (> 0: every pixel has v >= a), in the
// reference's two float32 roundings: it differs from v / M < 0.5 where v / M lies within an ulp of 0.5 (v = b, M = 2b).
PP_HD bool pp_paint_contour(float v, float M) { return PP_SUB(1.0f, PP_DIV(v, M)) > 0.5f; }
// the fill of one channel in float64 as numpy evaluates it: img * (1 - alpha) + color * alpha, truncated to uint8;
// oma = 1 - alpha as the caller computed it (0.30000000000000004 for alpha = 0.7)
PP_HD uint8_t pp_paint_fill(uint8_t img, uint8_t color, double alpha, double oma) {
  return (uint8_t)(int)PP_DADD(PP_DMUL((double)img, oma), PP_DMUL((double)color, alpha));
}
// The ids of a frame whose maximum M can be below 3: M < 3 needs v < 3 at every pixel, pixel (0, 0) included, so they
// are among the ids k with v < 3 at (0, 0) (at most 11 ids reach a corner).  c is (0, 0)'s window; out[] gets them in
// ascending order; returns their count.  Every other present id has M = 3.
template <typename L>
PP_HD int pp_paint_candidates(const L* c, int ld, int* out) {
  int n = 0;
  for (int k = pp_paint_next_id(c, ld, 0); k < 256; k = pp_paint_next_id(c, ld, k))
    if (pp_paint_dist(c, ld, k) < 3.0f) out[n++] = k;
  return n;
}
// One pixel rgb of the loop: each id k of its window in ascending order (the reference skips absent ids; ids of the
// window are present), fill with palette row k + 1 where the pixel is k, then the contour with row 1 where it lies on
// k's contour.  maxima[k]: M of id k in this frame.  Ids with no palette row (k + 1 >= n_colors) are not painted.
template <typename L>
PP_HD void pp_paint_pixel(const L* c, int ld, const float* maxima, const uint8_t* palette, int n_colors, double alpha,
                          double oma, uint8_t* rgb) {
  for (int k = pp_paint_next_id(c, ld, 0); k < 256 && k + 1 < n_colors; k = pp_paint_next_id(c, ld, k)) {
    if (c[0] == k)
      for (int ch = 0; ch < 3; ++ch) rgb[ch] = pp_paint_fill(rgb[ch], palette[(k + 1) * 3 + ch], alpha, oma);
    if (pp_paint_contour(pp_paint_dist(c, ld, k), maxima[k]))
      for (int ch = 0; ch < 3; ++ch) rgb[ch] = palette[3 + ch];
  }
}

// ---- I3D (core/metrics.py:195-569) ----
// TF 'same' padding of a k-tap, stride-s window over n samples: Unit3D.compute_pad / MaxPool3dSamePadding.compute_pad
// (core/metrics.py:196-200,258-262).  The front takes pad / 2, the back the rest, so even pads of 5 split 2 / 3.
PP_HD int pp_same_pad(int k, int s, int n) {
  const int r = n % s;
  const int p = r == 0 ? k - s : k - r;
  return p > 0 ? p : 0;
}
// output extent of that window: ceil(n / s) for every (k, s) I3D uses
PP_HD int pp_same_out(int k, int s, int n) { return (n + pp_same_pad(k, s, n) - k) / s + 1; }
// one tap of ATen's max pooling (max_pool3d_with_indices): a larger value or a NaN replaces the running maximum, so
// the first NaN sticks and, among equal values (+0 / -0), the first tap in (t, y, x) order wins
PP_HD float pp_pool_max(float m, float v) { return (v > m || isnan(v)) ? v : m; }

// ---- temporal warping error (Lai et al., "Learning Blind Video Temporal Consistency", ECCV 2018) ----
// Border-clamped bilinear sample of FlowNet2's Resample2d, the warp of Lai et al.'s evaluation: pixel (x, y) moved by
// (fx, fy) in float32; taps floor and floor + 1 on each axis, each clamped into the frame; weights from the unclamped
// fractions a, b.  Far outside the frame this returns the border pixel (not grid_sample's zeros of pp_taps).  Indices
// are clamped in float, so a huge or NaN coordinate cannot overflow the int conversion.  32-bit pixel indices: one
// frame's H * W * 3 stays below 2^31.
struct PPClampTaps {
  int i00, i01, i10, i11;         // pixel indices y * W + x of (yT, xL) (yT, xR) (yB, xL) (yB, xR)
  float w00, w01, w10, w11;       // (1-a)(1-b), a(1-b), (1-a)b, ab
};
PP_HD PPClampTaps pp_clamp_taps(int x, int y, float fx, float fy, int H, int W) {
  const float xf = PP_ADD((float)x, fx), yf = PP_ADD((float)y, fy);
  const float flx = floorf(xf), fly = floorf(yf);
  const float a = PP_SUB(xf, flx), b = PP_SUB(yf, fly);
  const float wm = (float)(W - 1), hm = (float)(H - 1);
  const int xl = (int)fminf(fmaxf(flx, 0.0f), wm), xr = (int)fminf(fmaxf(PP_ADD(flx, 1.0f), 0.0f), wm);
  const int yt = (int)fminf(fmaxf(fly, 0.0f), hm), yb = (int)fminf(fmaxf(PP_ADD(fly, 1.0f), 0.0f), hm);
  PPClampTaps t;
  t.i00 = yt * W + xl; t.i01 = yt * W + xr; t.i10 = yb * W + xl; t.i11 = yb * W + xr;
  const float ra = PP_SUB(1.0f, a), rb = PP_SUB(1.0f, b);
  t.w00 = PP_MUL(ra, rb); t.w01 = PP_MUL(a, rb); t.w10 = PP_MUL(ra, b); t.w11 = PP_MUL(a, b);
  return t;
}
// a value as the warp reads it: flow components as they are, uint8 frame values as v / 255 in float32
PP_HD float pp_ewarp_load(float v) { return v; }
PP_HD float pp_ewarp_load(uint8_t v) { return PP_DIV((float)v, 255.0f); }
// one channel of a plane whose pixels are `stride` elements apart, sampled through a tap set in Resample2d's order
template <typename T>
PP_HD float pp_clamp_sample(const T* p, int stride, const PPClampTaps& t) {
  float acc = PP_MUL(t.w00, pp_ewarp_load(p[t.i00 * stride]));
  acc = PP_ADD(acc, PP_MUL(t.w01, pp_ewarp_load(p[t.i01 * stride])));
  acc = PP_ADD(acc, PP_MUL(t.w10, pp_ewarp_load(p[t.i10 * stride])));
  return PP_ADD(acc, PP_MUL(t.w11, pp_ewarp_load(p[t.i11 * stride])));
}
// occlusion test 1 of Ruder et al. ("Artistic style transfer for videos", GCPR 2016), forward-backward consistency:
// occluded where |F + w|^2 > 0.01 (|F|^2 + |w|^2) + 0.5, w = B sampled at x + F(x); squared magnitudes, no root
PP_HD int pp_occ_fb(float fx, float fy, float wx, float wy) {
  const float sx = PP_ADD(fx, wx), sy = PP_ADD(fy, wy);
  const float lhs = PP_ADD(PP_MUL(sx, sx), PP_MUL(sy, sy));
  const float mag = PP_ADD(PP_ADD(PP_MUL(fx, fx), PP_MUL(fy, fy)), PP_ADD(PP_MUL(wx, wx), PP_MUL(wy, wy)));
  return lhs > PP_ADD(PP_MUL(0.01f, mag), 0.5f);
}
// occlusion test 2 (motion boundary): du = F(y, x) - F(y, x+1), dv = F(y, x) - F(y+1, x) per component (0 in the last
// column / row); occluded where du_x^2 + dv_x^2 + du_y^2 + dv_y^2 > 0.01 |F|^2 + 0.002
PP_HD int pp_occ_motion(float dux, float dvx, float duy, float dvy, float fx, float fy) {
  const float lhs = PP_ADD(PP_ADD(PP_ADD(PP_MUL(dux, dux), PP_MUL(dvx, dvx)), PP_MUL(duy, duy)), PP_MUL(dvy, dvy));
  return lhs > PP_ADD(PP_MUL(0.01f, PP_ADD(PP_MUL(fx, fx), PP_MUL(fy, fy))), 0.002f);
}
// the occlusion map O_t at pixel p = (x, y) of one pair: F, B planar [2][H][W] (forward t -> t+1, backward t+1 -> t),
// `t` the tap set of x + F(x).  1 = occluded (either test).
PP_HD int pp_flow_occluded(const float* F, const float* B, const PPClampTaps& t, int x, int y, int H, int W) {
  const int HW = H * W, p = y * W + x;
  const float fx = F[p], fy = F[HW + p];
  if (pp_occ_fb(fx, fy, pp_clamp_sample(B, 1, t), pp_clamp_sample(B + HW, 1, t))) return 1;
  const float dux = x + 1 < W ? PP_SUB(fx, F[p + 1]) : 0.0f, duy = x + 1 < W ? PP_SUB(fy, F[HW + p + 1]) : 0.0f;
  const float dvx = y + 1 < H ? PP_SUB(fx, F[p + W]) : 0.0f, dvy = y + 1 < H ? PP_SUB(fy, F[HW + p + W]) : 0.0f;
  return pp_occ_motion(dux, dvx, duy, dvy, fx, fy);
}
// per-pixel squared difference of the warping error: sum over RGB of (S(next / 255, F)(p) - cur(p) / 255)^2, frames
// uint8 pixel-major [H][W][3]
PP_HD float pp_warp_sqdiff(const uint8_t* next, const uint8_t* cur, const PPClampTaps& t, int p) {
  float s = 0.0f;
  for (int c = 0; c < 3; ++c) {
    const float d = PP_SUB(pp_clamp_sample(next + c, 3, t), pp_ewarp_load(cur[p * 3 + c]));
    s = PP_ADD(s, PP_MUL(d, d));
  }
  return s;
}
