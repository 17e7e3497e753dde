// TEST HARNESS ONLY (never loaded by the product): host build of RAFT-small's per-element rules from pp_elem.cuh --
// upflow8 (k_upflow8 of propainter_b200/csrc/gather_kernels.cu) and the radius-3 all-pairs / on-the-fly tap rules
// (k_corr_lookup<3>, k_corr_lookup_otf<128, 3>) -- so the CPU test-suite can check them against ATen and the oracle.
// Loops play the role of the CUDA grid.
#define PP_HOSTSIM 1
#include <cmath>
#include "../../propainter_b200/csrc/pp_elem.cuh"

extern "C" {

// flow_lr pixel-major [n][h][w][2] -> out planar [n][2][8h][8w]
void hs_upflow8(const float* flow_lr, float* out, int n, int h, int w) {
  const long H = 8L * h, W = 8L * w;
  for (long b = 0; b < n; ++b)
    for (int y = 0; y < H; ++y)
      for (int x = 0; x < W; ++x) {
        const PPLin uy = pp_upflow8_coord(y, h), ux = pp_upflow8_coord(x, w);
        const float* f = flow_lr + b * h * w * 2;
        for (int c = 0; c < 2; ++c)
          out[((b * 2 + c) * H + y) * W + x] =
              pp_upflow8_blend(f[((long)uy.i0 * w + ux.i0) * 2 + c], f[((long)uy.i0 * w + ux.i1) * 2 + c],
                               f[((long)uy.i1 * w + ux.i0) * 2 + c], f[((long)uy.i1 * w + ux.i1) * 2 + c], uy, ux);
      }
}

// all-pairs radius-3 lookup: levels lv[l] = [npix][h>>l][roundup4(w>>l)], coords [npix][2] -> out [npix][196]
void hs_corr_lookup_r3(const float* l0, const float* l1, const float* l2, const float* l3, const float* coords, float* out,
                       long npix, int h, int w) {
  const float* lv[4] = {l0, l1, l2, l3};
  for (long pix = 0; pix < npix; ++pix) {
    int hl = h, wl = w;
    for (int l = 0; l < 4; ++l) {
      const int ld = pp_corr_ld(wl);
      for (int t = 0; t < 49; ++t)
        out[pix * 196 + l * 49 + t] = pp_corr_tap_r<3>(lv[l] + pix * (long)hl * ld, hl, wl, ld, coords[2 * pix], coords[2 * pix + 1],
                                                       l, t / 7, t % 7);
      hl >>= 1; wl >>= 1;
    }
  }
}

// on-the-fly radius-3 lookup (D channels): levels lv[l] = [frames][(h>>l)*(w>>l)][D] -> out [n_pairs*h*w][196]
void hs_corr_lookup_otf_r3(const float* l0, const float* l1, const float* l2, const float* l3, int D, const int* idx1,
                           const int* idx2, long n_pairs, const float* coords, float* out, int h, int w) {
  const float* lv[4] = {l0, l1, l2, l3};
  const long hw = (long)h * w;
  const float sd = std::sqrt((float)D);
  float tile[64];
  for (long pix = 0; pix < n_pairs * hw; ++pix) {
    const long pair = pix / hw, i = pix % hw;
    const float cx = coords[2 * pix], cy = coords[2 * pix + 1];
    const float* f1 = l0 + ((long)idx1[pair] * hw + i) * D;
    for (int l = 0; l < 4; ++l) {
      const int hl = h >> l, wl = w >> l;
      const float* f2 = lv[l] + (long)idx2[pair] * hl * wl * D;
      const int tx0 = pp_corr_tile_origin_r<3>(cx, l), ty0 = pp_corr_tile_origin_r<3>(cy, l);
      for (int pos = 0; pos < 64; ++pos) {
        const int yy = ty0 + pos / 8, xx = tx0 + pos % 8;
        float s = 0.f;
        if (yy >= 0 && yy < hl && xx >= 0 && xx < wl) {
          const float* q = f2 + ((long)yy * wl + xx) * D;
          for (int c = 0; c < D; ++c) s += f1[c] * q[c];
        }
        tile[pos] = s / sd;
      }
      for (int t = 0; t < 49; ++t)
        out[pix * 196 + l * 49 + t] = pp_corr_tap_tile_r<3>(tile, tx0, ty0, hl, wl, cx, cy, l, t / 7, t % 7);
    }
  }
}

}
