// The non-convolution layers of the I3D feature network behind VFID (core/metrics.py:195-569) on sm_90a: input packing
// with Conv3d_1a_7x7's asymmetric 'same' border, MaxPool3dSamePadding, and the final mean over (T, H, W).  Feature
// maps are pixel-major NDHWC [B][T][H][W][ld]; the convolutions stay cuDNN calls and their eval-BN bias + ReLU epilogue
// is pp_bias_act (DESIGN.md §4).
#include "pp_elem.cuh"
#include "../../include/propainter_b200.h"

#define PP_LAUNCH_CHECK() do { if (cudaPeekAtLastError() != cudaSuccess) return PP_ERR_LAUNCH; } while (0)

static inline int pp_blocks(long n, int per) { return (int)((n + per - 1) / per); }

// ================================================================ input packing
// One thread per padded output pixel: 3 channels + a zero 4th (16-byte rows), zero outside the source.  U8: frames
// [B][T][H][W][3], value u8 / 255 rounded once (to_tensors, core/utils.py:169); otherwise planar float [B][3][T][H][W].
template <bool U8>
__global__ void __launch_bounds__(256) k_i3d_input(const void* __restrict__ src, float* __restrict__ dst, int B, int T, int H,
                                                   int W, int Tp, int Hp, int Wp, int ft, int fh, int fw) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)B * Tp * Hp * Wp) return;
  long r = i;
  const int x = (int)(r % Wp); r /= Wp;
  const int y = (int)(r % Hp); r /= Hp;
  const int t = (int)(r % Tp);
  const int b = (int)(r / Tp);
  const int ts = t - ft, ys = y - fh, xs = x - fw;
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (ts >= 0 && ts < T && ys >= 0 && ys < H && xs >= 0 && xs < W) {
    const long plane = (long)T * H * W;
    const long p = ((long)ts * H + ys) * W + xs;
    if (U8) {
      const uint8_t* s = static_cast<const uint8_t*>(src) + ((long)b * plane + p) * 3;
      v.x = PP_DIV((float)s[0], 255.0f);
      v.y = PP_DIV((float)s[1], 255.0f);
      v.z = PP_DIV((float)s[2], 255.0f);
    } else {
      const float* s = static_cast<const float*>(src) + (long)b * 3 * plane + p;
      v.x = s[0];
      v.y = s[plane];
      v.z = s[2 * plane];
    }
  }
  reinterpret_cast<float4*>(dst)[i] = v;
}

// replaces to_tensors (core/utils.py:151-170), the transpose(1, 2) of get_i3d_activations (core/metrics.py:183) and the
// F.pad of Conv3d_1a_7x7's Unit3D.forward (core/metrics.py:264-279)
extern "C" int pp_i3d_input(const void* src, int src_u8, float* dst, int B, int T, int H, int W, cudaStream_t stream) {
  if (B < 1 || T < 1 || H < 1 || W < 1) return PP_ERR_SHAPE;
  if ((uintptr_t)dst & 15) return PP_ERR_ALIGN;
  const int pt = pp_same_pad(7, 2, T), ph = pp_same_pad(7, 2, H), pw = pp_same_pad(7, 2, W);
  const int Tp = T + pt, Hp = H + ph, Wp = W + pw;
  const long n = (long)B * Tp * Hp * Wp;
  if (src_u8)
    k_i3d_input<true><<<pp_blocks(n, 256), 256, 0, stream>>>(src, dst, B, T, H, W, Tp, Hp, Wp, pt / 2, ph / 2, pw / 2);
  else
    k_i3d_input<false><<<pp_blocks(n, 256), 256, 0, stream>>>(src, dst, B, T, H, W, Tp, Hp, Wp, pt / 2, ph / 2, pw / 2);
  PP_LAUNCH_CHECK();
  return PP_OK;
}

// ================================================================ max pooling, TF 'same' border of zeros
// One thread per (output pixel, 4 channels); the channel group is the fastest index, so a warp reads whole rows.
// Out-of-range taps are the zeros F.pad inserts, visited in ATen's (t, y, x) order.
__global__ void __launch_bounds__(256) k_maxpool3d_same(const float* __restrict__ x, int ld_x, float* __restrict__ out,
                                                        int ld_out, int B, int T, int H, int W, int C, int To, int Ho,
                                                        int Wo, int kt, int kh, int kw, int st, int sh, int sw, int ft,
                                                        int fh, int fw) {
  const int c4n = C >> 2;
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)B * To * Ho * Wo * c4n) return;
  const int c = (int)(i % c4n) * 4;
  long r = i / c4n;
  const int xo = (int)(r % Wo); r /= Wo;
  const int yo = (int)(r % Ho); r /= Ho;
  const int to = (int)(r % To);
  const int b = (int)(r / To);
  float m[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
  for (int dt = 0; dt < kt; ++dt) {
    const int t = to * st - ft + dt;
    for (int dy = 0; dy < kh; ++dy) {
      const int y = yo * sh - fh + dy;
      for (int dx = 0; dx < kw; ++dx) {
        const int xx = xo * sw - fw + dx;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (t >= 0 && t < T && y >= 0 && y < H && xx >= 0 && xx < W)
          v = pp_ld4(x + (((long)b * T + t) * H + y) * (long)W * ld_x + (long)xx * ld_x + c);
        m[0] = pp_pool_max(m[0], v.x);
        m[1] = pp_pool_max(m[1], v.y);
        m[2] = pp_pool_max(m[2], v.z);
        m[3] = pp_pool_max(m[3], v.w);
      }
    }
  }
  pp_st4(out + (((long)b * To + to) * Ho + yo) * (long)Wo * ld_out + (long)xo * ld_out + c, make_float4(m[0], m[1], m[2], m[3]));
}

// replaces MaxPool3dSamePadding.forward (core/metrics.py:202-218): F.pad + nn.MaxPool3d
extern "C" int pp_maxpool3d_same(const float* x, int ld_x, float* out, int ld_out, int B, int T, int H, int W, int C, int kt,
                                 int kh, int kw, int st, int sh, int sw, cudaStream_t stream) {
  if (B < 1 || T < 1 || H < 1 || W < 1 || C < 1 || kt < 1 || kh < 1 || kw < 1 || st < 1 || sh < 1 || sw < 1) return PP_ERR_SHAPE;
  if (ld_x < C || ld_out < C) return PP_ERR_SHAPE;
  if (C % 4 || ld_x % 4 || ld_out % 4 || ((uintptr_t)x & 15) || ((uintptr_t)out & 15)) return PP_ERR_ALIGN;
  const int To = pp_same_out(kt, st, T), Ho = pp_same_out(kh, sh, H), Wo = pp_same_out(kw, sw, W);
  const long n = (long)B * To * Ho * Wo * (C / 4);
  k_maxpool3d_same<<<pp_blocks(n, 256), 256, 0, stream>>>(x, ld_x, out, ld_out, B, T, H, W, C, To, Ho, Wo, kt, kh, kw, st, sh, sw,
                                                          pp_same_pad(kt, st, T) / 2, pp_same_pad(kh, sh, H) / 2,
                                                          pp_same_pad(kw, sw, W) / 2);
  PP_LAUNCH_CHECK();
  return PP_OK;
}

// ================================================================ mean over (T, H, W)
// One block per (sample, 32 channels): 8 warps stride over the N pixels in float64, each lane owning one channel (a
// warp reads 128 contiguous bytes per pixel), then warp 0 adds the 8 partial sums in a fixed order and rounds once.
// No atomics: the result is the same on every run.
__global__ void __launch_bounds__(256) k_mean_thw(const float* __restrict__ x, int ld, float* __restrict__ out, long N, int C) {
  __shared__ double part[8][32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int b = blockIdx.y, c = blockIdx.x * 32 + lane;
  double s = 0.0;
  if (c < C)
    for (long p = wid; p < N; p += 8) s = PP_DADD(s, (double)x[((long)b * N + p) * ld + c]);
  part[wid][lane] = s;
  __syncthreads();
  if (wid == 0 && c < C) {
    double t = part[0][lane];
    for (int k = 1; k < 8; ++k) t = PP_DADD(t, part[k][lane]);
    out[(long)b * C + c] = (float)PP_DDIV(t, (double)N);
  }
}

// replaces x.mean(4).mean(3).mean(2) of InceptionI3d.extract_features (core/metrics.py:566-567)
extern "C" int pp_mean_thw(const float* x, int ld, float* out, int B, long N, int C, cudaStream_t stream) {
  if (B < 1 || B > 65535 || N < 1 || C < 1 || ld < C) return PP_ERR_SHAPE;
  k_mean_thw<<<dim3((C + 31) / 32, B), 256, 0, stream>>>(x, ld, out, N, C);
  PP_LAUNCH_CHECK();
  return PP_OK;
}
