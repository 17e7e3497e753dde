// TEST HARNESS ONLY (never loaded by the product): host build of the I3D rules from pp_elem.cuh -- the 'same' padding
// and output extent of k_i3d_input / k_maxpool3d_same, and ATen's max-pooling tap rule -- so the CPU test-suite can
// check them against the oracle and ATen.
#define PP_HOSTSIM 1
#include <cmath>
#include "../../propainter_b200/csrc/pp_elem.cuh"

extern "C" {

int hs_same_pad(int k, int s, int n) { return pp_same_pad(k, s, n); }
int hs_same_out(int k, int s, int n) { return pp_same_out(k, s, n); }

// k_maxpool3d_same over one channel: x [T][H][W] -> out [To][Ho][Wo]
void hs_maxpool3d_same(const float* x, float* out, int T, int H, int W, int kt, int kh, int kw, int st, int sh, int sw) {
  const int To = pp_same_out(kt, st, T), Ho = pp_same_out(kh, sh, H), Wo = pp_same_out(kw, sw, W);
  const int ft = pp_same_pad(kt, st, T) / 2, fh = pp_same_pad(kh, sh, H) / 2, fw = pp_same_pad(kw, sw, W) / 2;
  for (int to = 0; to < To; ++to)
    for (int yo = 0; yo < Ho; ++yo)
      for (int xo = 0; xo < Wo; ++xo) {
        float m = -INFINITY;
        for (int dt = 0; dt < kt; ++dt)
          for (int dy = 0; dy < kh; ++dy)
            for (int dx = 0; dx < kw; ++dx) {
              const int t = to * st - ft + dt, y = yo * sh - fh + dy, xx = xo * sw - fw + dx;
              const bool in = t >= 0 && t < T && y >= 0 && y < H && xx >= 0 && xx < W;
              m = pp_pool_max(m, in ? x[((long)t * H + y) * W + xx] : 0.0f);
            }
        out[((long)to * Ho + yo) * Wo + xo] = m;
      }
}
}
