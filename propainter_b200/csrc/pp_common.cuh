// Common definitions for the propainter_b200 sm_90a kernels.
//
// Layout conventions (DESIGN.md §3):
//   * "planar"  : [n][c][H][W]   -- tensors that cross the reference API boundary (frames, flows, masks)
//   * "pixel-major" (NHWC) : [n][H][W][ld] with ld >= C -- every internal feature map; kernels take the
//     pixel stride `ld` explicitly so they can read / write channel slices of wider concat buffers.
//
// Element functions (per output element, no inter-thread cooperation) are PP_HD so that
// tests/hostsim can compile the very same index arithmetic for the CPU test-suite.  The product
// never runs them on the host.
#pragma once
#include <stdint.h>
#include <math.h>

#if defined(PP_HOSTSIM)
#define PP_HD static inline
struct float4 { float x, y, z, w; };
struct float2 { float x, y; };
static inline float4 make_float4(float a, float b, float c, float d) { float4 r = {a, b, c, d}; return r; }
#else
#include <cuda_runtime.h>
#define PP_HD __host__ __device__ __forceinline__
#endif

// error codes of the C ABI (include/propainter_b200.h)
#define PP_OK 0
#define PP_ERR_SHAPE (-1)
#define PP_ERR_DTYPE (-2)
#define PP_ERR_WORKSPACE (-3)
#define PP_ERR_LAUNCH (-4)
#define PP_ERR_ALIGN (-5)

// Unfused fp32 arithmetic for the discontinuous paths (nearest rounding, thresholds): nvcc would
// otherwise contract a*b+c into FMA and move results across rounding boundaries relative to ATen.
#if defined(__CUDA_ARCH__)
#define PP_MUL(a, b) __fmul_rn((a), (b))
#define PP_ADD(a, b) __fadd_rn((a), (b))
#define PP_SUB(a, b) __fsub_rn((a), (b))
#define PP_DIV(a, b) __fdiv_rn((a), (b))
#else
#define PP_MUL(a, b) ((a) * (b))
#define PP_ADD(a, b) ((a) + (b))
#define PP_SUB(a, b) ((a) - (b))
#define PP_DIV(a, b) ((a) / (b))
#endif
// the same for double, where a rule restates a float64 numpy expression bit for bit
#if defined(__CUDA_ARCH__)
#define PP_DMUL(a, b) __dmul_rn((a), (b))
#define PP_DADD(a, b) __dadd_rn((a), (b))
#define PP_DSUB(a, b) __dsub_rn((a), (b))
#else
#define PP_DMUL(a, b) ((a) * (b))
#define PP_DADD(a, b) ((a) + (b))
#define PP_DSUB(a, b) ((a) - (b))
#endif
// correctly rounded square root and float64 division (the flow colour rules)
#if defined(__CUDA_ARCH__)
#define PP_SQRT(a) __fsqrt_rn(a)
#define PP_DDIV(a, b) __ddiv_rn((a), (b))
#else
#define PP_SQRT(a) sqrtf(a)
#define PP_DDIV(a, b) ((a) / (b))
#endif

// one fused multiply-add, rounded once (where the restated library kernel is compiled with FMA contraction)
#if defined(__CUDA_ARCH__)
#define PP_FMA(a, b, c) __fmaf_rn((a), (b), (c))
#else
#define PP_FMA(a, b, c) fmaf((a), (b), (c))
#endif

#if !defined(PP_HOSTSIM)
// SM count of the current device, queried once (132 if none answers)
static inline int pp_num_sms() {
  static int n = 0;
  int dev = 0;
  if (n < 1 && (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n < 1)) {
    cudaGetLastError();
    n = 132;
  }
  return n;
}
#define PP_NUM_SMS pp_num_sms()

// fp32 or fp16 pixel-major rows for the elementwise kernels around the half-operand library convs (DESIGN.md §4
// "Precision"): 4 consecutive channels in as float4 (fp16 rows: 8-byte aligned), out rounded to nearest.
#include <cuda_fp16.h>
__device__ __forceinline__ float4 pp_ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float4 pp_ld4(const __half* p) {
  const uint2 u = *reinterpret_cast<const uint2*>(p);
  const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
  return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ void pp_st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ void pp_st4(__half* p, float4 v) {
  const __half2 a = __floats2half2_rn(v.x, v.y), b = __floats2half2_rn(v.z, v.w);
  uint2 u;
  u.x = *reinterpret_cast<const uint32_t*>(&a);
  u.y = *reinterpret_cast<const uint32_t*>(&b);
  *reinterpret_cast<uint2*>(p) = u;
}
__device__ __forceinline__ void pp_st1(float* p, float v) { *p = v; }
__device__ __forceinline__ void pp_st1(__half* p, float v) { *p = __float2half_rn(v); }
#endif
