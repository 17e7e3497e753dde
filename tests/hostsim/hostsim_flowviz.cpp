// TEST HARNESS ONLY (never loaded by the product): host build of the flow colour-coding kernels (k_flow_maxrad /
// k_flow_to_image_u8 of propainter_b200/csrc/gather_kernels.cu) from the per-element rules of pp_elem.cuh, so the CPU
// test-suite can check them against oracle/flowviz_ref.py.  Loops play the role of the CUDA grid.
#define PP_HOSTSIM 1
#include "../../propainter_b200/csrc/pp_elem.cuh"

extern "C" {

int hs_colorwheel(int k, int c) { return pp_colorwheel(k, c); }

// one pixel per (u[i], v[i], den[i]); variant 0 = numpy (flow_viz.py), 1 = torch (flow_viz_pt.py) -> rgb[i][3]
void hs_flowviz_pixels(const float* u, const float* v, const float* den, uint8_t* rgb, long n, int variant, int bgr) {
  for (long i = 0; i < n; ++i) {
    if (variant == 0) pp_flowviz_np(u[i], v[i], den[i], bgr, rgb + i * 3);
    else pp_flowviz_pt(u[i], v[i], den[i], bgr, rgb + i * 3);
  }
}

// planar flow [N][2][H][W] -> uint8 [N][H][W][3]: the group maxima pass, then the colour pass
void hs_flow_to_image_u8(const float* flow, uint8_t* out, int N, int H, int W, int variant, int has_clip, float clip_flow,
                         int bgr) {
  const long HW = (long)H * W;
  float batch_max = 0.0f;
  float* maxima = new float[N];
  for (int n = 0; n < N; ++n) {
    float m = 0.0f;
    for (long p = 0; p < HW; ++p) {
      float a = flow[(long)n * 2 * HW + p], b = flow[(long)n * 2 * HW + HW + p];
      if (has_clip) { a = pp_flow_clip(a, clip_flow); b = pp_flow_clip(b, clip_flow); }
      m = fmaxf(m, pp_flow_rad(a, b));
    }
    maxima[n] = m;
    batch_max = fmaxf(batch_max, m);
  }
  for (int n = 0; n < N; ++n) {
    const float den = variant == 0 ? maxima[n] + 1e-5f : batch_max + 1.1920928955078125e-07f;
    for (long p = 0; p < HW; ++p) {
      float u = flow[(long)n * 2 * HW + p], v = flow[(long)n * 2 * HW + HW + p];
      if (has_clip) { u = pp_flow_clip(u, clip_flow); v = pp_flow_clip(v, clip_flow); }
      uint8_t* o = out + ((long)n * HW + p) * 3;
      if (variant == 0) pp_flowviz_np(u, v, den, bgr, o);
      else pp_flowviz_pt(u, v, den, bgr, o);
    }
  }
  delete[] maxima;
}

}
