// TEST HARNESS ONLY (never loaded by the product): host build of the tracking preview (k_mask_paint_partial,
// k_mask_paint_maxima and k_mask_paint_u8 of propainter_b200/csrc/cutie_kernels.cu) from the per-element rules of
// pp_elem.cuh, so the CPU test-suite can check them against oracle/painter_ref.py.  Loops play the role of the CUDA grid;
// the maxima are taken over whole frames instead of tiles (the maximum does not depend on the grouping).
#define PP_HOSTSIM 1
#include <vector>
#include "../../propainter_b200/csrc/pp_elem.cuh"

// frame labels [H][W] -> window storage [(H+6)][(W+6)] with -1 outside the frame
static std::vector<int> hs_pad(const uint8_t* lab, int H, int W) {
  const int ld = W + 6;
  std::vector<int> s((size_t)(H + 6) * ld, -1);
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) s[(size_t)(y + 3) * ld + x + 3] = lab[(long)y * W + x];
  return s;
}

extern "C" {

// the chamfer path sum of offset (dy, dx)
float hs_paint_chamfer(int dy, int dx) { return pp_paint_chamfer(dy, dx); }

// v of every pixel for object k: labels uint8 [H][W] -> out float [H][W]
void hs_paint_dist(const uint8_t* lab, int H, int W, int k, float* out) {
  const std::vector<int> s = hs_pad(lab, H, W);
  const int ld = W + 6;
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) out[(long)y * W + x] = pp_paint_dist(&s[(size_t)(y + 3) * ld + x + 3], ld, k);
}

int hs_paint_contour(float v, float M) { return pp_paint_contour(v, M); }

uint8_t hs_paint_fill(uint8_t img, uint8_t color, double alpha, double oma) { return pp_paint_fill(img, color, alpha, oma); }

// frames uint8 [T][H][W][3], labels uint8 [T][H][W], palette [n_colors][3] -> out uint8 [T][H][W][3]; maxima float
// [T][256] receives the per-(frame, id) M the painting used
void hs_mask_paint_u8(const uint8_t* frames, const uint8_t* labels, const uint8_t* palette, int n_colors, double alpha,
                      double oma, uint8_t* out, int T, int H, int W, float* maxima) {
  const int ld = W + 6;
  const long HW = (long)H * W;
  for (int f = 0; f < T; ++f) {
    const std::vector<int> s = hs_pad(labels + f * HW, H, W);
    float* M = maxima + (long)f * 256;
    for (int k = 0; k < 256; ++k) M[k] = 3.0f;
    int cand[16];
    const int n = pp_paint_candidates(&s[3 * (size_t)ld + 3], ld, cand);
    for (int j = 0; j < n; ++j) {
      float m = 0.0f;
      for (int y = 0; y < H; ++y)
        for (int x = 0; x < W; ++x) m = fmaxf(m, pp_paint_dist(&s[(size_t)(y + 3) * ld + x + 3], ld, cand[j]));
      M[cand[j]] = m;
    }
    for (long p = 0; p < HW; ++p) {
      const int y = (int)(p / W), x = (int)(p % W);
      uint8_t rgb[3] = {frames[(f * HW + p) * 3], frames[(f * HW + p) * 3 + 1], frames[(f * HW + p) * 3 + 2]};
      pp_paint_pixel(&s[(size_t)(y + 3) * ld + x + 3], ld, M, palette, n_colors, alpha, oma, rgb);
      for (int c = 0; c < 3; ++c) out[(f * HW + p) * 3 + c] = rgb[c];
    }
  }
}

}
