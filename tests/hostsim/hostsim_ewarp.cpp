// TEST HARNESS ONLY (never loaded by the product): host build of the warping-error kernels (k_flow_occlusion /
// k_warp_error of propainter_b200/csrc/gather_kernels.cu) from the per-pixel rules of pp_elem.cuh, so the CPU test-suite
// can check them against oracle/ewarp_ref.py.  Loops play the role of the CUDA grid; the float64 sums run in pixel
// order rather than the kernel's block order.
#define PP_HOSTSIM 1
#include "../../propainter_b200/csrc/pp_elem.cuh"

extern "C" {

// S(plane, flow) at every pixel: plane [H][W], flow planar [2][H][W] -> out [H][W]
void hs_clamp_sample(const float* plane, const float* flow, float* out, int H, int W) {
  const long HW = (long)H * W;
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      const int p = y * W + x;
      out[p] = pp_clamp_sample(plane, 1, pp_clamp_taps(x, y, flow[p], flow[HW + p], H, W));
    }
}

// O_t of every pair: fw, bw [N][2][H][W] -> occ [N][H][W]
void hs_flow_occlusion(const float* fw, const float* bw, uint8_t* occ, int N, int H, int W) {
  const long HW = (long)H * W;
  for (int n = 0; n < N; ++n)
    for (int y = 0; y < H; ++y)
      for (int x = 0; x < W; ++x) {
        const int p = y * W + x;
        const float* F = fw + (long)n * 2 * HW;
        const PPClampTaps t = pp_clamp_taps(x, y, F[p], F[HW + p], H, W);
        occ[n * HW + p] = (uint8_t)pp_flow_occluded(F, bw + (long)n * 2 * HW, t, x, y, H, W);
      }
}

// (sum, N_t) per pair: frames uint8 [T][H][W][3], fw [T-1][2][H][W], occ [T-1][H][W] -> out float64 [T-1][2]
void hs_warp_error(const uint8_t* frames, const float* fw, const uint8_t* occ, double* out, int T, int H, int W) {
  const long HW = (long)H * W;
  for (int n = 0; n < T - 1; ++n) {
    const float* F = fw + (long)n * 2 * HW;
    const uint8_t* cur = frames + (long)n * HW * 3;
    double s = 0.0, c = 0.0;
    for (int y = 0; y < H; ++y)
      for (int x = 0; x < W; ++x) {
        const int p = y * W + x;
        if (occ[n * HW + p]) continue;
        s += (double)pp_warp_sqdiff(cur + HW * 3, cur, pp_clamp_taps(x, y, F[p], F[HW + p], H, W), p);
        c += 1.0;
      }
    out[2 * n] = s;
    out[2 * n + 1] = c;
  }
}

}
