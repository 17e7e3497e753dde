// Per-element device functions (index arithmetic + sampling rules) of the gather-type kernels.
// Each cites the reference line whose semantics it reproduces.  PP_HD: also compiled by tests/hostsim.
#pragma once
#include "pp_common.cuh"

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
// sample one scalar plane [H][ld] through a tap set (order nw, ne, sw, se like ATen)
PP_HD float pp_tap_plane(const float* p, int ld, const PPTaps& t) {
  if (!t.any) return 0.f;
  float acc = 0.f;
  const float* r0 = p + (long)t.y0 * ld + t.x0;
  const float* r1 = r0 + ld;
  if (t.w00 != 0.f) acc += r0[0] * t.w00;
  if (t.w01 != 0.f) acc += r0[1] * t.w01;
  if (t.w10 != 0.f) acc += r1[0] * t.w10;
  if (t.w11 != 0.f) acc += r1[1] * t.w11;
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
// One step of the non-learnable image propagation scan (model/propainter.py:144-161), one pixel.
// All tensors planar: frames 3 planes of H*W, masks/flows likewise.  `nearest` selects :149's mode.
PP_HD void pp_imgprop_pixel(int pix, int H, int W, const float* cur, const float* mcur, const float* prev,
                            const float* mprev, const float* fprop, const float* fcheck, float* out,
                            float* mout, int nearest) {
  const int HW = H * W;
  int y = pix / W, x = pix - y * W;
  float fx = fprop[pix], fy = fprop[HW + pix];
  float ix = pp_warp_coord((float)x, fx, W), iy = pp_warp_coord((float)y, fy, H);
  PPTaps t = pp_taps(ix, iy, H, W);
  float bx = pp_tap_plane(fcheck, W, t), by = pp_tap_plane(fcheck + HW, W, t);
  float valid = pp_fb_valid(fx, fy, bx, by);
  float mw = pp_tap_plane(mprev, W, t) > 0.1f ? 1.0f : 0.0f;            // binary_mask(:156)
  float mc = mcur[pix];
  float gate = PP_MUL(PP_MUL(mc, valid), PP_SUB(1.0f, mw));
  float use = gate > 0.1f ? 1.0f : 0.0f;                                 // :158
  long ni = nearest ? pp_nearest_index(ix, iy, H, W, W) : 0;
  for (int c = 0; c < 3; ++c) {
    float wv;
    if (nearest) wv = ni >= 0 ? prev[(long)c * HW + ni] : 0.f;
    else wv = pp_tap_plane(prev + (long)c * HW, W, t);
    float cv = cur[(long)c * HW + pix];
    out[(long)c * HW + pix] = PP_ADD(PP_MUL(use, wv), PP_MUL(PP_SUB(1.0f, use), cv));   // :159
  }
  float m2 = PP_MUL(mc, PP_SUB(1.0f, PP_MUL(valid, PP_SUB(1.0f, mw))));  // :161
  mout[pix] = m2 > 0.1f ? 1.0f : 0.0f;
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
// RAFT/corr.py:29-50: output channel l*81 + a*9 + b samples level l at (cx/2^l + (a-4), cy/2^l + (b-4));
// note the first window axis moves x (reference quirk: delta = stack(meshgrid(dy,dx)) added to (x,y)).
PP_HD float pp_corr_tap(const float* plane, int Hl, int Wl, int ld, float cx, float cy, int lvl, int a, int b) {
  float s = (float)(1 << lvl);
  float x = PP_ADD(PP_DIV(cx, s), (float)(a - 4));
  float y = PP_ADD(PP_DIV(cy, s), (float)(b - 4));
  PPTaps t = pp_taps(pp_raft_coord(x, Wl), pp_raft_coord(y, Hl), Hl, Wl);
  return pp_tap_plane(plane, ld, t);
}
// AlternateCorrBlock (RAFT/corr.py:83-111) without a stored plane: level `lvl` is sampled from a 10x10 tile of dot
// products, tile[j*10 + i] = f1 . f2_l[ty0 + j][tx0 + i] / sqrt(D) (zero outside the level), whose origin is the
// floored level centre minus the window radius.  Far-away or non-finite centres get a tile wholly outside the level.
PP_HD int pp_corr_tile_origin(float c, int lvl) {
  float v = floorf(PP_DIV(c, (float)(1 << lvl)));
  v = fminf(fmaxf(v, -1.0e6f), 1.0e6f);
  return (int)v - 4;
}
// Tap (a, b) of level `lvl` from that tile by the rule of pp_corr_tap.  The grid_sample coordinate round trip can move
// a corner by one step at an integer boundary; a corner that lands off the tile then weighs 0 or a few ulp and is dropped.
PP_HD float pp_corr_tap_tile(const float* tile, int tx0, int ty0, int Hl, int Wl, float cx, float cy, int lvl, int a, int b) {
  float s = (float)(1 << lvl);
  float x = PP_ADD(PP_DIV(cx, s), (float)(a - 4));
  float y = PP_ADD(PP_DIV(cy, s), (float)(b - 4));
  PPTaps t = pp_taps(pp_raft_coord(x, Wl), pp_raft_coord(y, Hl), Hl, Wl);
  if (!t.any) return 0.f;
  const int i = t.x0 - tx0, j = t.y0 - ty0;
  const bool i0 = i >= 0 && i < 10, i1 = i >= -1 && i < 9, j0 = j >= 0 && j < 10, j1 = j >= -1 && j < 9;
  float acc = 0.f;
  if (t.w00 != 0.f && j0 && i0) acc += tile[j * 10 + i] * t.w00;
  if (t.w01 != 0.f && j0 && i1) acc += tile[j * 10 + i + 1] * t.w01;
  if (t.w10 != 0.f && j1 && i0) acc += tile[(j + 1) * 10 + i] * t.w10;
  if (t.w11 != 0.f && j1 && i1) acc += tile[(j + 1) * 10 + i + 1] * t.w11;
  return acc;
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
// InpaintGenerator.forward down-sampling (propainter.py:338-342; stencils pinned in SURVEY.md §8c):
// bilinear 1/4 (align_corners=False) == mean of the centre 2x2 of each 4x4 block; then /4.
PP_HD float pp_flow_ds4(const float* plane, int W, int y, int x) {
  const float* p = plane + (long)(4 * y + 1) * W + 4 * x + 1;
  float top = 0.5f * p[0] + 0.5f * p[1];
  float bot = 0.5f * p[W] + 0.5f * p[W + 1];
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
PP_HD uint8_t pp_composite(float pred, float mask, uint8_t ori, uint8_t prev, int first) {
  float v = PP_MUL(PP_DIV(PP_ADD(pred, 1.0f), 2.0f), 255.0f);
  uint8_t p8 = (uint8_t)(int)v;                     // numpy astype(uint8) of a value in [0,255]
  uint8_t bm = (uint8_t)(int)mask;
  uint8_t img = (uint8_t)(p8 * bm + ori * (uint8_t)(1 - bm));
  if (first) return img;
  float b = PP_ADD(PP_MUL((float)prev, 0.5f), PP_MUL((float)img, 0.5f));
  return (uint8_t)(int)b;
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
