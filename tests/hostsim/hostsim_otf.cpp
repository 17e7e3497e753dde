// TEST HARNESS ONLY (never loaded by the product): host build of the on-the-fly RAFT correlation
// (propainter_b200/csrc/corr_otf.cu) from the per-element rules of pp_elem.cuh, so the CPU test-suite can check
// the tile origin and tap rule against the oracle.  Loops play the role of the CUDA grid.
#define PP_HOSTSIM 1
#include <cmath>
#include "../../propainter_b200/csrc/pp_elem.cuh"

extern "C" {

// one 2x2 average-pooling level of a pixel-major feature map [frames][hs*ws][D] -> [frames][(hs/2)*(ws/2)][D]
void hs_fmap_pool(const float* src, float* dst, long frames, int hs, int ws, int D) {
  const int hd = hs / 2, wd = ws / 2;
  for (long f = 0; f < frames; ++f)
    for (int y = 0; y < hd; ++y)
      for (int x = 0; x < wd; ++x)
        for (int c = 0; c < D; ++c) {
          const float* p = src + ((f * hs + 2 * y) * ws + 2 * x) * (long)D + c;
          dst[((f * hd + y) * wd + x) * (long)D + c] = PP_DIV(PP_ADD(PP_ADD(PP_ADD(p[0], p[D]), p[(long)ws * D]), p[(long)ws * D + D]), 4.0f);
        }
}

// levels lv[l] = [frames][(h>>l)*(w>>l)][D]; coords [n_pairs*h*w][2] -> out [n_pairs*h*w][324]
void hs_corr_lookup_otf(const float* l0, const float* l1, const float* l2, const float* l3, int D, const int* idx1,
                        const int* idx2, long n_pairs, const float* coords, float* out, int h, int w) {
  const float* lv[4] = {l0, l1, l2, l3};
  const long hw = (long)h * w;
  const float scale = 1.0f / std::sqrt((float)D);
  float tile[100];
  for (long pix = 0; pix < n_pairs * hw; ++pix) {
    const long pair = pix / hw, i = pix % hw;
    const float cx = coords[2 * pix], cy = coords[2 * pix + 1];
    const float* f1 = l0 + ((long)idx1[pair] * hw + i) * D;
    for (int l = 0; l < 4; ++l) {
      const int hl = h >> l, wl = w >> l;
      const float* f2 = lv[l] + (long)idx2[pair] * hl * wl * D;
      const int tx0 = pp_corr_tile_origin(cx, l), ty0 = pp_corr_tile_origin(cy, l);
      for (int pos = 0; pos < 100; ++pos) {
        const int yy = ty0 + pos / 10, xx = tx0 + pos % 10;
        float s = 0.f;
        if (yy >= 0 && yy < hl && xx >= 0 && xx < wl) {
          const float* q = f2 + ((long)yy * wl + xx) * D;
          for (int c = 0; c < D; ++c) s += f1[c] * q[c];
        }
        tile[pos] = s * scale;
      }
      for (int t = 0; t < 81; ++t) out[pix * 324 + l * 81 + t] = pp_corr_tap_tile(tile, tx0, ty0, hl, wl, cx, cy, l, t / 9, t % 9);
    }
  }
}

}
