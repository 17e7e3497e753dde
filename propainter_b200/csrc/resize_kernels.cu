// Device-side frame / mask resizing around the hot path (SURVEY.md section 8f item 1), bit-compatible with the libraries the
// reference calls on the host:
//   * resize_frames (inference_propainter.py:34-45): PIL.Image.resize(process_size) = Pillow's separable resampler with
//     the BICUBIC filter on 8-bit pixels (third-party dependency, Pillow `src/libImaging/Resample.c`; not vendored in the
//     reference tree).  Restated from its published algorithm: per axis, double-precision windowed coefficients normalised
//     to sum 1, converted to 22-bit fixed point, horizontal pass then vertical pass through an 8-bit intermediate, each
//     output = clip8((2^21 + sum coeff*pixel) >> 22).  The coefficient tables are built on the HOST by
//     pp_resample_coeffs_bicubic (plain C doubles, the same operation order as Pillow; no FMA contraction on the host
//     compiler's baseline x86-64 / aarch64 targets) and handed to the kernels as device arrays.
//   * read_mask's mask_img.resize(size, Image.NEAREST) (:95-96): Pillow's nearest-neighbour affine scaling,
//     source x = (int)(xo), xo starting at scale/2 and accumulated by += scale in double (Geometry.c) -- table on the host.
//   * the output cv2.resize(f, out_size) (:469-470): OpenCV's 8-bit INTER_LINEAR: 11-bit fixed-point coefficients from
//     float fractions, horizontal pass into int, vertical pass ((b0*(S0>>4))>>16 + (b1*(S1>>4))>>16 + 2) >> 2 (resize.cpp).
//   * the evaluation dataset's resize_flow (core/dataset.py:213-214, utils/flow_util.py:6-11): OpenCV's float32
//     INTER_LINEAR (float coefficients, separable, unfused products and sums; exact 2x down-scaling is its INTER_AREA
//     fast path) and the per-component rescale, on planar float32 flows [N][2][H][W].
//   * scripts/compute_flow.py's frame preparation (:67-92): ToTensor, torch F.interpolate(bilinear, align_corners=False)
//     and *2 - 1, fused into one pass from uint8 frames to RAFT's planar fp32 input (pp_resize_coord in pp_elem.cuh).
// The uint8 kernels: uint8 [T][H][W][3] (masks [T][H][W]) in, same layout out; stream-ordered; the caller owns tables + scratch.
#include <math.h>
#include <stdint.h>
#include "pp_common.cuh"
#include "pp_elem.cuh"
#include "../../include/propainter_b200.h"

#define RS_PREC 22

// ---------------------------------------------------------------- host: coefficient tables
static double rs_bicubic(double x) {
  const double a = -0.5;
  if (x < 0.0) x = -x;
  if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
  if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
  return 0.0;
}

// Pillow precompute_coeffs + normalize_coeffs_8bpc for the full-image box.  bounds [out_size*2] = (first source index,
// tap count); kk [out_size*ksize] fixed-point taps.  Returns ksize (taps per output), or < 0 if `kk_capacity` ints do not
// hold out_size*ksize.  Call with kk == NULL to query ksize only.
extern "C" int pp_resample_coeffs_bicubic(int in_size, int out_size, int* bounds, int* kk, long kk_capacity) {
  if (in_size < 1 || out_size < 1) return PP_ERR_SHAPE;
  const float in0 = 0.f, in1 = (float)in_size;
  double filterscale, scale;
  filterscale = scale = (double)(in1 - in0) / out_size;
  if (filterscale < 1.0) filterscale = 1.0;
  const double support = 2.0 * filterscale;
  const int ksize = (int)ceil(support) * 2 + 1;
  if (!kk) return ksize;
  if ((long)out_size * ksize > kk_capacity || !bounds) return PP_ERR_WORKSPACE;
  double* k = (double*)malloc(sizeof(double) * (size_t)ksize);
  if (!k) return PP_ERR_WORKSPACE;
  for (int xx = 0; xx < out_size; ++xx) {
    const double center = in0 + (xx + 0.5) * scale;
    double ww = 0.0;
    const double ss = 1.0 / filterscale;
    int xmin = (int)(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = (int)(center + support + 0.5);
    if (xmax > in_size) xmax = in_size;
    xmax -= xmin;
    int x;
    for (x = 0; x < xmax; ++x) {
      const double w = rs_bicubic((x + xmin - center + 0.5) * ss);
      k[x] = w;
      ww += w;
    }
    for (x = 0; x < xmax; ++x)
      if (ww != 0.0) k[x] /= ww;
    for (; x < ksize; ++x) k[x] = 0;
    for (x = 0; x < ksize; ++x)
      kk[(long)xx * ksize + x] = k[x] < 0 ? (int)(-0.5 + k[x] * (1 << RS_PREC)) : (int)(0.5 + k[x] * (1 << RS_PREC));
    bounds[xx * 2] = xmin;
    bounds[xx * 2 + 1] = xmax;
  }
  free(k);
  return ksize;
}

// Pillow nearest scaling (ImagingScaleAffine for a pure scale): src index of every destination index
extern "C" int pp_resample_index_nearest(int in_size, int out_size, int* idx) {
  if (in_size < 1 || out_size < 1 || !idx) return PP_ERR_SHAPE;
  const double a0 = (double)in_size / out_size;
  double xo = 0.0 + a0 * 0.5;
  for (int x = 0; x < out_size; ++x) {
    int xi = (int)(xo < 0 ? xo - 1 : xo);                  // COORD(): floor towards -inf for negatives, else truncation
    if (xi < 0) xi = 0;
    if (xi >= in_size) xi = in_size - 1;
    idx[x] = xi;
    xo += a0;
  }
  return PP_OK;
}

// OpenCV INTER_LINEAR tables for one axis: ofs[out] = left / top source index, coef[out*2] = 11-bit taps.
// `horizontal`: border taps are reset like resize.cpp does for x (fx = 0 at the clamped ends); the vertical pass keeps its
// fraction and clamps the rows instead.
extern "C" int pp_resample_coeffs_linear_cv(int in_size, int out_size, int horizontal, int* ofs, short* coef) {
  if (in_size < 1 || out_size < 1 || !ofs || !coef) return PP_ERR_SHAPE;
  const double inv_scale = (double)out_size / in_size, scale = 1.0 / inv_scale;
  for (int d = 0; d < out_size; ++d) {
    float f = (float)((d + 0.5) * scale - 0.5);
    int s = (int)floorf(f);
    f -= s;
    if (horizontal) {
      if (s < 0) { f = 0; s = 0; }
      if (s >= in_size - 1) { f = 0; s = in_size - 1; }
    }
    ofs[d] = s;
    const float c0 = (1.f - f) * 2048.f, c1 = f * 2048.f;
    coef[2 * d] = (short)lrintf(c0);                          // saturate_cast<short>(float): round half to even
    coef[2 * d + 1] = (short)lrintf(c1);
  }
  return PP_OK;
}

// OpenCV INTER_LINEAR tables of the float32 path for one axis: ofs[out] = left / top source index, coef[out*2] =
// (1 - f, f) in float.  Same coordinate rule as above; the horizontal border reset likewise.
extern "C" int pp_resample_coeffs_linear_f32(int in_size, int out_size, int horizontal, int* ofs, float* coef) {
  if (in_size < 1 || out_size < 1 || !ofs || !coef) return PP_ERR_SHAPE;
  const double inv_scale = (double)out_size / in_size, scale = 1.0 / inv_scale;
  for (int d = 0; d < out_size; ++d) {
    float f = (float)((d + 0.5) * scale - 0.5);
    int s = (int)floorf(f);
    f -= s;
    if (horizontal) {
      if (s < 0) { f = 0; s = 0; }
      if (s >= in_size - 1) { f = 0; s = in_size - 1; }
    }
    ofs[d] = s;
    coef[2 * d] = 1.f - f;
    coef[2 * d + 1] = f;
  }
  return PP_OK;
}

// ---------------------------------------------------------------- device
__device__ __forceinline__ uint8_t rs_clip8(int v) {
  v >>= RS_PREC;
  return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// horizontal: src [rows][Win][3] -> dst [rows][Wout][3]
__global__ void __launch_bounds__(256) k_resample_h(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, long rows, int Win, int Wout,
                                                    const int* __restrict__ bounds, const int* __restrict__ kk, int ksize) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * Wout) return;
  const long r = i / Wout; const int xx = (int)(i - r * Wout);
  const int xmin = bounds[2 * xx], n = bounds[2 * xx + 1];
  const int* k = kk + (long)xx * ksize;
  const uint8_t* p = src + (r * Win + xmin) * 3;
  int s0 = 1 << (RS_PREC - 1), s1 = s0, s2 = s0;
  for (int x = 0; x < n; ++x) { const int w = k[x]; s0 += p[3 * x] * w; s1 += p[3 * x + 1] * w; s2 += p[3 * x + 2] * w; }
  uint8_t* o = dst + i * 3;
  o[0] = rs_clip8(s0); o[1] = rs_clip8(s1); o[2] = rs_clip8(s2);
}
// vertical: src [T][Hin][W][3] -> dst [T][Hout][W][3]
__global__ void __launch_bounds__(256) k_resample_v(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int T, int Hin, int Hout, int W,
                                                    const int* __restrict__ bounds, const int* __restrict__ kk, int ksize) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;           // over T*Hout*W*3 bytes
  const long row_bytes = (long)W * 3;
  if (i >= (long)T * Hout * row_bytes) return;
  const long tr = i / row_bytes; const long b = i - tr * row_bytes;
  const int t = (int)(tr / Hout), yy = (int)(tr - (long)t * Hout);
  const int ymin = bounds[2 * yy], n = bounds[2 * yy + 1];
  const int* k = kk + (long)yy * ksize;
  const uint8_t* p = src + ((long)t * Hin + ymin) * row_bytes + b;
  int s = 1 << (RS_PREC - 1);
  for (int y = 0; y < n; ++y) s += p[(long)y * row_bytes] * k[y];
  dst[i] = rs_clip8(s);
}

extern "C" size_t pp_resize_u8_bicubic_workspace_bytes(int T, int H, int Wo) { return (size_t)T * H * Wo * 3; }
// resize_frames (inference_propainter.py:34-45) on the device.  Tables from pp_resample_coeffs_bicubic, copied to the device
// by the caller.  H == Ho or W == Wo skips that pass (Pillow does the same).
extern "C" int pp_resize_u8_bicubic(const uint8_t* src, uint8_t* dst, int T, int H, int W, int Ho, int Wo, const int* bounds_x,
                                    const int* kk_x, int ksize_x, const int* bounds_y, const int* kk_y, int ksize_y, void* workspace,
                                    size_t ws_bytes, cudaStream_t stream) {
  if (T < 1 || H < 1 || W < 1 || Ho < 1 || Wo < 1) return PP_ERR_SHAPE;
  const bool need_h = Wo != W, need_v = Ho != H;
  if (!need_h && !need_v) return cudaMemcpyAsync(dst, src, (size_t)T * H * W * 3, cudaMemcpyDeviceToDevice, stream) == cudaSuccess ? PP_OK : PP_ERR_LAUNCH;
  const uint8_t* mid = src;
  if (need_h) {
    uint8_t* hdst = need_v ? (uint8_t*)workspace : dst;
    if (need_v && ws_bytes < pp_resize_u8_bicubic_workspace_bytes(T, H, Wo)) return PP_ERR_WORKSPACE;
    const long n = (long)T * H * Wo;
    k_resample_h<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(src, hdst, (long)T * H, W, Wo, bounds_x, kk_x, ksize_x);
    mid = hdst;
  }
  if (need_v) {
    const long n = (long)T * Ho * Wo * 3;
    k_resample_v<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(mid, dst, T, H, Ho, Wo, bounds_y, kk_y, ksize_y);
  }
  return cudaPeekAtLastError() == cudaSuccess ? PP_OK : PP_ERR_LAUNCH;
}

__global__ void __launch_bounds__(256) k_resize_nearest(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int T, int H, int W, int Ho, int Wo,
                                                        int C, const int* __restrict__ ix, const int* __restrict__ iy) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)T * Ho * Wo) return;
  const int x = (int)(i % Wo); const long r = i / Wo; const int y = (int)(r % Ho); const int t = (int)(r / Ho);
  const uint8_t* p = src + (((long)t * H + iy[y]) * W + ix[x]) * C;
  for (int c = 0; c < C; ++c) dst[i * C + c] = p[c];
}
// mask_img.resize(size, Image.NEAREST) (inference_propainter.py:95-96); C = 1 (masks) or 3
extern "C" int pp_resize_u8_nearest(const uint8_t* src, uint8_t* dst, int T, int H, int W, int Ho, int Wo, int C, const int* idx_x,
                                    const int* idx_y, cudaStream_t stream) {
  if (T < 1 || H < 1 || W < 1 || Ho < 1 || Wo < 1 || C < 1 || C > 4) return PP_ERR_SHAPE;
  const long n = (long)T * Ho * Wo;
  k_resize_nearest<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(src, dst, T, H, W, Ho, Wo, C, idx_x, idx_y);
  return cudaPeekAtLastError() == cudaSuccess ? PP_OK : PP_ERR_LAUNCH;
}

__global__ void __launch_bounds__(256) k_resize_linear_cv(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int T, int H, int W, int Ho,
    int Wo, const int* __restrict__ xofs, const short* __restrict__ alpha, const int* __restrict__ yofs, const short* __restrict__ beta) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)T * Ho * Wo) return;
  const int x = (int)(i % Wo); const long r = i / Wo; const int y = (int)(r % Ho); const int t = (int)(r / Ho);
  const int sx = xofs[x], a0 = alpha[2 * x], a1 = alpha[2 * x + 1];
  const int sx1 = sx + 1 < W ? sx + 1 : sx;                              // a1 == 0 whenever sx is the last column
  int sy0 = yofs[y], sy1 = sy0 + 1;
  sy0 = sy0 < 0 ? 0 : (sy0 > H - 1 ? H - 1 : sy0);
  sy1 = sy1 < 0 ? 0 : (sy1 > H - 1 ? H - 1 : sy1);
  const int b0 = beta[2 * y], b1 = beta[2 * y + 1];
  const uint8_t* r0 = src + ((long)t * H + sy0) * W * 3;
  const uint8_t* r1 = src + ((long)t * H + sy1) * W * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int S0 = r0[sx * 3 + c] * a0 + r0[sx1 * 3 + c] * a1;
    const int S1 = r1[sx * 3 + c] * a0 + r1[sx1 * 3 + c] * a1;
    dst[i * 3 + c] = (uint8_t)((((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2);
  }
}
// cv2.resize(f, out_size) of the composited frames (inference_propainter.py:469-470), 8-bit INTER_LINEAR; tables from
// pp_resample_coeffs_linear_cv.  Exact 2x down-scaling takes OpenCV's area path instead and is rejected here.
extern "C" int pp_resize_u8_bilinear_cv(const uint8_t* src, uint8_t* dst, int T, int H, int W, int Ho, int Wo, const int* xofs,
                                        const short* alpha, const int* yofs, const short* beta, cudaStream_t stream) {
  if (T < 1 || H < 1 || W < 1 || Ho < 1 || Wo < 1) return PP_ERR_SHAPE;
  if (W == 2 * Wo && H == 2 * Ho) return PP_ERR_SHAPE;
  const long n = (long)T * Ho * Wo;
  k_resize_linear_cv<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(src, dst, T, H, W, Ho, Wo, xofs, alpha, yofs, beta);
  return cudaPeekAtLastError() == cudaSuccess ? PP_OK : PP_ERR_LAUNCH;
}

// One output value of resize_flow (utils/flow_util.py:6-11) per thread, planar [N][2][H][W] -> [N][2][Ho][Wo].  Every
// product and sum is rounded on its own (OpenCV's float kernels are not contracted to FMA on its x86 builds), then the
// component's in-place `*= new / old` with the ratio already rounded to float32 (numpy's weak Python scalar).
__device__ __forceinline__ float rs_row_linear(const float* __restrict__ row, int W, int sx, float a0, float a1) {
  return sx + 1 < W ? PP_ADD(PP_MUL(row[sx], a0), PP_MUL(row[sx + 1], a1)) : PP_MUL(row[sx], a0);   // right border: a0 = 1
}
__global__ void __launch_bounds__(256) k_resize_flow_linear(const float* __restrict__ src, float* __restrict__ dst, int N, int H,
    int W, int Ho, int Wo, const int* __restrict__ xofs, const float* __restrict__ alpha, const int* __restrict__ yofs,
    const float* __restrict__ beta, float scale_u, float scale_v) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)N * 2 * Ho * Wo) return;
  const int x = (int)(i % Wo); const long r = i / Wo; const int y = (int)(r % Ho); const long plane = r / Ho;
  const float* s = src + plane * H * W;
  const int sx = xofs[x];
  const float a0 = alpha[2 * x], a1 = alpha[2 * x + 1];
  int sy0 = yofs[y], sy1 = sy0 + 1;
  sy0 = sy0 < 0 ? 0 : (sy0 > H - 1 ? H - 1 : sy0);                    // rows clamp, their weights stay (resize.cpp)
  sy1 = sy1 < 0 ? 0 : (sy1 > H - 1 ? H - 1 : sy1);
  const float r0 = rs_row_linear(s + (long)sy0 * W, W, sx, a0, a1), r1 = rs_row_linear(s + (long)sy1 * W, W, sx, a0, a1);
  const float v = PP_ADD(PP_MUL(r0, beta[2 * y]), PP_MUL(r1, beta[2 * y + 1]));
  dst[i] = PP_MUL(v, (plane & 1) ? scale_v : scale_u);
}
// exact 2x down-scaling on both axes: OpenCV's INTER_AREA fast path, ((a + b) + c) + d over the 2x2 block, times 0.25
__global__ void __launch_bounds__(256) k_resize_flow_area2(const float* __restrict__ src, float* __restrict__ dst, int N, int H,
    int W, int Ho, int Wo, float scale_u, float scale_v) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)N * 2 * Ho * Wo) return;
  const int x = (int)(i % Wo); const long r = i / Wo; const int y = (int)(r % Ho); const long plane = r / Ho;
  const float* p = src + (plane * H + 2L * y) * W + 2L * x;
  const float sum = PP_ADD(PP_ADD(PP_ADD(p[0], p[1]), p[W]), p[W + 1]);
  dst[i] = PP_MUL(PP_MUL(sum, 0.25f), (plane & 1) ? scale_v : scale_u);
}
extern "C" int pp_resize_flow_linear_cv(const float* src, float* dst, int N, int H, int W, int Ho, int Wo, const int* xofs,
                                        const float* alpha, const int* yofs, const float* beta, cudaStream_t stream) {
  if (N < 1 || H < 1 || W < 1 || Ho < 1 || Wo < 1) return PP_ERR_SHAPE;
  const long n = (long)N * 2 * Ho * Wo;
  const float su = (float)((double)Wo / W), sv = (float)((double)Ho / H);
  if (Ho == H && Wo == W)                                                // cv2.resize copies; the ratios are 1
    return cudaMemcpyAsync(dst, src, (size_t)n * sizeof(float), cudaMemcpyDeviceToDevice, stream) == cudaSuccess ? PP_OK : PP_ERR_LAUNCH;
  if (W == 2 * Wo && H == 2 * Ho)
    k_resize_flow_area2<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(src, dst, N, H, W, Ho, Wo, su, sv);
  else if (!xofs || !alpha || !yofs || !beta)
    return PP_ERR_SHAPE;
  else
    k_resize_flow_linear<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(src, dst, N, H, W, Ho, Wo, xofs, alpha, yofs, beta, su, sv);
  return cudaPeekAtLastError() == cudaSuccess ? PP_OK : PP_ERR_LAUNCH;
}

// scripts/compute_flow.py:67-92 on the device: uint8 RGB [T][H0][W0][3] -> planar fp32 [T][3][h][w] in [-1,1], the rule of
// pp_resize_coord / pp_u8_frame_resized.  One thread per output pixel, all three channels (the taps of a pixel share rows).
__global__ void __launch_bounds__(256) k_u8_to_frames_resized(const uint8_t* __restrict__ src, float* __restrict__ dst, int T, int H0,
                                                              int W0, int h, int w) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const long hw = (long)h * w;
  if (i >= (long)T * hw) return;
  const int x = (int)(i % w); const long r = i / w; const int y = (int)(r % h); const long t = r / h;
  const PPLin uy = pp_resize_coord(y, H0, h), ux = pp_resize_coord(x, W0, w);
  const uint8_t* f = src + t * H0 * W0 * 3;
  const uint8_t* r0 = f + (long)uy.i0 * W0 * 3;
  const uint8_t* r1 = f + (long)uy.i1 * W0 * 3;
  const int x0 = ux.i0 * 3, x1 = ux.i1 * 3;
  float* o = dst + t * 3 * hw + (long)y * w + x;
#pragma unroll
  for (int c = 0; c < 3; ++c) o[c * hw] = pp_u8_frame_resized(r0[x0 + c], r0[x1 + c], r1[x0 + c], r1[x1 + c], uy, ux);
}
extern "C" int pp_u8_to_frames_resized(const uint8_t* src, float* dst, int T, int H0, int W0, int h, int w, cudaStream_t stream) {
  if (T < 1 || H0 < 1 || W0 < 1 || h < 1 || w < 1) return PP_ERR_SHAPE;
  const long n = (long)T * h * w;
  k_u8_to_frames_resized<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(src, dst, T, H0, W0, h, w);
  return cudaPeekAtLastError() == cudaSuccess ? PP_OK : PP_ERR_LAUNCH;
}
