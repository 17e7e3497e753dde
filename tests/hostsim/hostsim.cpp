// TEST HARNESS ONLY (never loaded by the product): compiles the per-element rules of
// propainter_b200/csrc/pp_elem.cuh for the host so the CPU test-suite can check the index arithmetic
// and sampling rules of the gather kernels against the oracle without a GPU.  Loops here play the
// role of the CUDA grid; they mirror the launchers in gather_kernels.cu / mma_kernels.cu.
#define PP_HOSTSIM 1
#include <cstring>
#include <vector>
#include "../../propainter_b200/csrc/pp_elem.cuh"

extern "C" {

void hs_img_prop_scan(const float* frames, const float* ff, const float* fb, const float* masks, float* of, float* om,
                      int t, int H, int W, int nearest) {
  const long HW = (long)H * W;
  std::vector<float> bf((size_t)t * 3 * HW), bm((size_t)t * HW);
  memcpy(&bf[(size_t)(t - 1) * 3 * HW], frames + (long)(t - 1) * 3 * HW, 3 * HW * sizeof(float));
  memcpy(&bm[(size_t)(t - 1) * HW], masks + (long)(t - 1) * HW, HW * sizeof(float));
  for (int i = t - 2; i >= 0; --i)
    for (int p = 0; p < HW; ++p)
      pp_imgprop_pixel(p, H, W, frames + (long)i * 3 * HW, masks + (long)i * HW, &bf[(size_t)(i + 1) * 3 * HW],
                       &bm[(size_t)(i + 1) * HW], ff + (long)i * 2 * HW, fb + (long)i * 2 * HW, &bf[(size_t)i * 3 * HW],
                       &bm[(size_t)i * HW], nearest);
  memcpy(of, bf.data(), 3 * HW * sizeof(float));
  memcpy(om, bm.data(), HW * sizeof(float));
  for (int i = 1; i < t; ++i)
    for (int p = 0; p < HW; ++p)
      pp_imgprop_pixel(p, H, W, &bf[(size_t)i * 3 * HW], &bm[(size_t)i * HW], of + (long)(i - 1) * 3 * HW,
                       om + (long)(i - 1) * HW, fb + (long)(i - 1) * 2 * HW, ff + (long)(i - 1) * 2 * HW,
                       of + (long)i * 3 * HW, om + (long)i * HW, nearest);
}

void hs_prop_cond(const float* cur, int ld_cur, const float* prop, int ld_prop, const float* fprop, const float* fcheck,
                  const float* mcur, float* cond, int ld_cond, float* bb, int ld_bb, int h, int w, int C, int first) {
  for (long pix = 0; pix < (long)h * w; ++pix) {
    int y = (int)(pix / w), x = (int)(pix % w);
    PPCond c = {0, 0, 0, 0, 0};
    PPTaps t = {};
    if (!first) { c = pp_cond_pixel(y, x, h, w, fprop, fcheck); t = pp_taps(c.ix, c.iy, h, w); }
    float* bbp = bb + pix * ld_bb;
    float* cdp = cond ? cond + pix * ld_cond : nullptr;
    for (int ch = 0; ch < C; ch += 4) {
      float4 v = *reinterpret_cast<const float4*>(cur + pix * ld_cur + ch);
      memcpy(bbp + ch, &v, 16);
      if (first) memcpy(bbp + C + ch, &v, 16);
      else {
        memcpy(cdp + ch, &v, 16);
        float4 wv = pp_tap_nhwc4(prop, ld_prop, w, t, ch);
        memcpy(cdp + C + ch, &wv, 16);
      }
    }
    bbp[2 * C] = mcur[2 * pix]; bbp[2 * C + 1] = mcur[2 * pix + 1];
    for (int ch = 2 * C + 2; ch < ld_bb; ++ch) bbp[ch] = 0.f;
    if (!first) {
      cdp[2 * C] = c.fx; cdp[2 * C + 1] = c.fy; cdp[2 * C + 2] = c.valid;
      cdp[2 * C + 3] = mcur[2 * pix]; cdp[2 * C + 4] = mcur[2 * pix + 1];
      for (int ch = 2 * C + 5; ch < ld_cond; ++ch) cdp[ch] = 0.f;
    }
  }
}

int hs_corr_ld(int w) { return pp_corr_ld(w); }

void hs_corr_pool(const float* src, float* dst, long planes, int Hs, int lds, int Hd, int Wd, int ldd) {
  for (long p = 0; p < planes; ++p)
    for (int y = 0; y < Hd; ++y)
      for (int x = 0; x < Wd; ++x)
        dst[p * (long)Hd * ldd + (long)y * ldd + x] = pp_pool4(src + p * (long)Hs * lds, lds, y, x);
}

void hs_corr_lookup(const float* l0, const float* l1, const float* l2, const float* l3, const float* coords, float* out,
                    long npix, int h, int w) {
  const float* lv[4] = {l0, l1, l2, l3};
  for (long pix = 0; pix < npix; ++pix) {
    int hl = h, wl = w;
    for (int l = 0; l < 4; ++l) {
      int ld = pp_corr_ld(wl);
      for (int tap = 0; tap < 81; ++tap)
        out[pix * 324 + l * 81 + tap] =
            pp_corr_tap(lv[l] + pix * (long)hl * ld, hl, wl, ld, coords[2 * pix], coords[2 * pix + 1], l, tap / 9, tap % 9);
      hl >>= 1; wl >>= 1;
    }
  }
}

// k_corr_lookup<R> (radius 3 or 4): levels [npix][h>>l][roundup4(w>>l)], coords [npix][2] -> out [npix][4K^2]
void hs_corr_lookup_r(const float* l0, const float* l1, const float* l2, const float* l3, int radius, const float* coords,
                      float* out, long npix, int h, int w) {
  const float* lv[4] = {l0, l1, l2, l3};
  const int K = 2 * radius + 1;
  for (long pix = 0; pix < npix; ++pix) {
    int hl = h, wl = w;
    for (int l = 0; l < 4; ++l) {
      const int ld = pp_corr_ld(wl);
      const float* pl = lv[l] + pix * (long)hl * ld;
      for (int t = 0; t < K * K; ++t)
        out[pix * 4 * K * K + l * K * K + t] =
            radius == 3 ? pp_corr_tap_r<3>(pl, hl, wl, ld, coords[2 * pix], coords[2 * pix + 1], l, t / K, t % K)
                        : pp_corr_tap_r<4>(pl, hl, wl, ld, coords[2 * pix], coords[2 * pix + 1], l, t / K, t % K);
      hl >>= 1; wl >>= 1;
    }
  }
}

// the on-the-fly tile rule of one level (k_corr_lookup_otf): tile [T*T] (T = 2R+2) at the origin pp_corr_tile_origin_r
// of (cx, cy) -> out [K*K]; origin [2] receives (tx0, ty0)
void hs_corr_tap_tile_r(const float* tile, int radius, int hl, int wl, float cx, float cy, int lvl, float* out, int* origin) {
  const int K = 2 * radius + 1;
  const int tx0 = radius == 3 ? pp_corr_tile_origin_r<3>(cx, lvl) : pp_corr_tile_origin_r<4>(cx, lvl);
  const int ty0 = radius == 3 ? pp_corr_tile_origin_r<3>(cy, lvl) : pp_corr_tile_origin_r<4>(cy, lvl);
  origin[0] = tx0; origin[1] = ty0;
  for (int t = 0; t < K * K; ++t)
    out[t] = radius == 3 ? pp_corr_tap_tile_r<3>(tile, tx0, ty0, hl, wl, cx, cy, lvl, t / K, t % K)
                         : pp_corr_tap_tile_r<4>(tile, tx0, ty0, hl, wl, cx, cy, lvl, t / K, t % K);
}

// pp_instance_norm on x [n][HW][C]: the statistics rules in k_inorm_stats' split of the rows (S chunks, R row-threads
// per chunk, merged in thread order), then pp_inorm_fold and pp_inorm_out; res nullable
void hs_instance_norm(const float* x, const float* res, float* out, int n, long HW, int C, float eps, int relu, int post_relu) {
  const int S = pp_inorm_splits(n, HW), chunk = (int)((HW + S - 1) / S), R = 256 / (C / 4);
  std::vector<PPNormStat> st((size_t)C);
  for (long b = 0; b < n; ++b) {
    const float* xb = x + b * HW * C;
    for (int c = 0; c < C; ++c) {
      double su = 0.0, sq = 0.0;
      for (int s = 0; s < S; ++s) {
        const long r0 = (long)s * chunk, r1 = r0 + chunk < HW ? r0 + chunk : HW;
        double a = 0.0, q = 0.0;
        for (int r = 0; r < R; ++r) {
          double ta = 0.0, tq = 0.0;
          for (long row = r0 + r; row < r1; row += R) pp_inorm_acc(ta, tq, xb[row * C + c], xb[c]);
          a += ta; q += tq;
        }
        su += a; sq += q;
      }
      st[c] = pp_inorm_fold(su, sq, HW, xb[c], eps);
    }
    for (long i = 0; i < HW * C; ++i) {
      const long o = b * HW * C + i;
      out[o] = pp_inorm_out(x[o], st[i % C], relu, res ? res + o : nullptr, post_relu);
    }
  }
}

void hs_convex_upsample(const float* mask, int ld_mask, float scale, const float* flow_lr, float* out, int n, int h, int w) {
  const long H = 8L * h, W = 8L * w;
  for (int b = 0; b < n; ++b)
    for (int y = 0; y < h; ++y)
      for (int x = 0; x < w; ++x)
        for (int s = 0; s < 64; ++s) {
          long px = ((long)b * h + y) * w + x;
          float2 v = pp_convex_up(mask + px * ld_mask, scale, flow_lr + (long)b * h * w * 2, h, w, y, x, s >> 3, s & 7);
          float* ob = out + (long)b * 2 * H * W + (8L * y + (s >> 3)) * W + 8L * x + (s & 7);
          ob[0] = v.x; ob[H * W] = v.y;
        }
}

void hs_flow_ds4(const float* planes, float* out, int n, int H, int W) {   // [n][H][W] -> [n][H/4][W/4]
  for (int i = 0; i < n; ++i)
    for (int y = 0; y < H / 4; ++y)
      for (int x = 0; x < W / 4; ++x) out[((long)i * (H / 4) + y) * (W / 4) + x] = pp_flow_ds4(planes + (long)i * H * W, W, y, x);
}

void hs_deform_cols(const float* x, int ld_x, const float* o, int ld_o, const float* flow, float max_res, float* cols,
                    int H, int W, int Cin) {   // cols [H*W][9*Cin], column = tap*Cin + c
  int cpg = Cin / 16;
  for (long pix = 0; pix < (long)H * W; ++pix) {
    int y = (int)(pix / W), xx = (int)(pix % W);
    for (int k = 0; k < 9; ++k)
      for (int c = 0; c < Cin; ++c) {
        PPDTap t = pp_deform_tap(o + pix * ld_o, flow ? flow + 2 * pix : nullptr, max_res, c / cpg, k, y, xx);
        PPDW d = pp_deform_weights(t, H, W);
        cols[pix * 9 * Cin + (long)k * Cin + c] = pp_deform_sample1(x, ld_x, W, d, c);
      }
  }
}

void hs_ffn_overlap_add(const float* Y, int ldy, float* Z, int ldz, int frames, int h, int w, int CH) {
  int fh = (h - 1) / 3 + 1, fw = (w - 1) / 3 + 1;
  std::vector<float> F((size_t)frames * h * w * CH);
  for (int f = 0; f < frames; ++f)
    for (int y = 0; y < h; ++y)
      for (int x = 0; x < w; ++x)
        for (int c = 0; c < CH; ++c)
          F[(((size_t)f * h + y) * w + x) * CH + c] = pp_ffn_fold(Y + (long)f * fh * fw * ldy, ldy, CH, fh, fw, y, x, c);
  for (long tok = 0; tok < (long)frames * fh * fw; ++tok) {
    int f = (int)(tok / (fh * fw)), tr = (int)(tok % (fh * fw)), ty = tr / fw, tx = tr % fw;
    for (int tap = 0; tap < 49; ++tap)
      for (int c = 0; c < CH; ++c) {
        int y = 3 * ty - 3 + tap / 7, x = 3 * tx - 3 + tap % 7;
        float v = 0.f;
        if (y >= 0 && y < h && x >= 0 && x < w) v = pp_gelu(F[(((size_t)f * h + y) * w + x) * CH + c]);
        Z[tok * ldz + tap * CH + c] = v;
      }
  }
}

void hs_u8_to_frames(const uint8_t* src, float* dst, int T, int H, int W) {
  long HW = (long)H * W;
  for (long f = 0; f < T; ++f)
    for (int c = 0; c < 3; ++c)
      for (long p = 0; p < HW; ++p) {
        float v = (float)src[(f * HW + p) * 3 + c] / 255.0f;
        dst[(f * 3 + c) * HW + p] = v * 2.0f - 1.0f;
      }
}

void hs_composite(const float* pred, const float* masks, const uint8_t* ori, uint8_t* comp, int n, const int* frame,
                  const int* first, int H, int W) {
  long HW = (long)H * W;
  for (int k = 0; k < n; ++k)
    for (long p = 0; p < HW; ++p)
      for (int c = 0; c < 3; ++c) {
        long o = ((long)frame[k] * HW + p) * 3 + c;
        comp[o] = pp_composite(pred[((long)k * 3 + c) * HW + p], masks[(long)frame[k] * HW + p], ori[o], comp[o], first[k]);
      }
}
}

extern "C" void hs_upsample2x(const float* src, float* dst, int n, int h, int w, int C) {
  const int H = 2 * h, W = 2 * w;
  for (int b = 0; b < n; ++b)
    for (int y = 0; y < H; ++y)
      for (int x = 0; x < W; ++x) {
        PPUp uy = pp_up2_coord(y, h), ux = pp_up2_coord(x, w);
        for (int c = 0; c < C; ++c) {
          const float* p = src + (((long)b * h + uy.i0) * w + ux.i0) * C + c;
          dst[(((long)b * H + y) * W + x) * C + c] =
              pp_up2_blend(p[0], p[(long)ux.step * C], p[(long)uy.step * w * C], p[((long)uy.step * w + ux.step) * C], uy, ux);
        }
      }
}

extern "C" void hs_mask_dilate(const uint8_t* src, float* dst, int T, int H, int W, int iterations) {
  for (long f = 0; f < T; ++f)
    for (int y = 0; y < H; ++y)
      for (int x = 0; x < W; ++x) dst[(f * H + y) * W + x] = pp_mask_dilate_pixel(src + f * H * W, H, W, y, x, iterations);
}
