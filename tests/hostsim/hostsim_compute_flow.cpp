// TEST HARNESS ONLY (never loaded by the product): host build of compute_flow.py's frame preparation from pp_elem.cuh --
// k_u8_to_frames_resized of propainter_b200/csrc/resize_kernels.cu -- so the CPU test-suite can check the rule against
// ATen's F.interpolate and pp_u8_frame.  Loops play the role of the CUDA grid.
#define PP_HOSTSIM 1
#include <cmath>
#include "../../propainter_b200/csrc/pp_elem.cuh"

extern "C" {

// uint8 RGB [T][H0][W0][3] -> planar [T][3][h][w]
void hs_u8_to_frames_resized(const uint8_t* src, float* dst, int T, int H0, int W0, int h, int w) {
  const long hw = (long)h * w;
  for (long t = 0; t < T; ++t)
    for (int y = 0; y < h; ++y)
      for (int x = 0; x < w; ++x) {
        const PPLin uy = pp_resize_coord(y, H0, h), ux = pp_resize_coord(x, W0, w);
        const uint8_t* r0 = src + (t * H0 + uy.i0) * W0 * 3;
        const uint8_t* r1 = src + (t * H0 + uy.i1) * W0 * 3;
        for (int c = 0; c < 3; ++c)
          dst[(t * 3 + c) * hw + (long)y * w + x] =
              pp_u8_frame_resized(r0[ux.i0 * 3 + c], r0[ux.i1 * 3 + c], r1[ux.i0 * 3 + c], r1[ux.i1 * 3 + c], uy, ux);
      }
}

// pp_u8_frame of every value: uint8 [n] -> float [n]
void hs_u8_frame(const uint8_t* src, float* dst, long n) {
  for (long i = 0; i < n; ++i) dst[i] = pp_u8_frame(src[i]);
}

}
