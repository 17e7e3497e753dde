// TEST HARNESS ONLY (never loaded by the product): host build of the video-outpainting kernels
// (k_extrapolate_u8 / k_mask_overlay_u8 of propainter_b200/csrc/gather_kernels.cu) from the per-element rules of
// pp_elem.cuh, so the CPU test-suite can check them against oracle/outpaint_ref.py.  Loops play the role of the CUDA grid.
#define PP_HOSTSIM 1
#include "../../propainter_b200/csrc/pp_elem.cuh"

extern "C" {

// uint8 [T][h][w][3] -> canvas uint8 [T][H][W][3], flow / dilated masks float [T][1][H][W]
void hs_extrapolate_u8(const uint8_t* src, uint8_t* canvas, float* flow_masks, float* masks_dilated, int T, int h, int w,
                       int H, int W, int top, int left, int rim_h, int rim_w) {
  const long HW = (long)H * W;
  for (long i = 0; i < (long)T * HW; ++i) {
    const long f = i / HW, p = i - f * HW;
    const int y = (int)(p / W), x = (int)(p - (long)y * W);
    const long s = pp_outpaint_src(y, x, top, left, h, w);
    for (int c = 0; c < 3; ++c) canvas[i * 3 + c] = s >= 0 ? src[(f * h * w + s) * 3 + c] : 0;
    flow_masks[i] = pp_outpaint_mask(y, x, top, left, h, w, rim_h, rim_w);
    masks_dilated[i] = pp_outpaint_mask(y, x, top, left, h, w, 0, 0);
  }
}

// uint8 [T][H][W][3] + masks [T][1][H][W] -> preview uint8 [T][H][W][3]
void hs_mask_overlay_u8(const uint8_t* frames, const float* masks, uint8_t* out, int T, int H, int W) {
  for (long i = 0; i < (long)T * H * W * 3; ++i) out[i] = pp_mask_overlay(frames[i], masks[i / 3], (int)(i % 3));
}

}
