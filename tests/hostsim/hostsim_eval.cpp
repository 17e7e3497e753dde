// TEST HARNESS ONLY (never loaded by the product): host build of k_composite_f32 (propainter_b200/csrc/gather_kernels.cu),
// the evaluation protocol's float-valued compositing, from the per-element rule pp_composite_f32 of pp_elem.cuh, so the
// CPU test-suite can check it against the script's numpy loop.  The loops play the role of the CUDA grid.
#define PP_HOSTSIM 1
#include "../../propainter_b200/csrc/pp_elem.cuh"

extern "C" void hs_composite_f32(const float* pred, const float* masks, const uint8_t* ori, float* comp, int n,
                                 const int* frame, const int* first, int H, int W) {
  long HW = (long)H * W;
  for (int k = 0; k < n; ++k)
    for (long p = 0; p < HW; ++p)
      for (int c = 0; c < 3; ++c) {
        long o = ((long)frame[k] * HW + p) * 3 + c;
        comp[o] = pp_composite_f32(pred[((long)k * 3 + c) * HW + p], masks[(long)frame[k] * HW + p], ori[o], comp[o], first[k]);
      }
}
