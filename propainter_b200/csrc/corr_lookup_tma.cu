// RAFT correlation lookup, TMA-staged (sm_90a).
//
// One warp per source pixel.  For each of the 4 pyramid levels the warp's elected lane issues one
// cp.async.bulk.tensor (TMA, 3-D tiled: x, y, plane) that lands the 16x10 neighbourhood of the lookup
// centre in shared memory (radius 3: 12x8; the box's innermost coordinate is rounded down to a multiple of 4 floats: a
// tiled TMA load whose first element is not 16-byte aligned faults with "illegal instruction" -- measured
// with profiles/probes/tma_probe.cu); out-of-range rows / columns are zero-filled by the TMA unit, which *is*
// grid_sample's zeros padding, so the inner loop has no bounds logic on loads.  The 81 (radius 3: 49) taps of a level
// are then bilinear blends of shared-memory values and are written as one contiguous 324-float (196-float) run.
// Replaces CorrBlock.__call__ (RAFT/corr.py:29-50) + bilinear_sampler (RAFT/utils/utils.py:57-71).
#include <cuda.h>
#include "pp_elem.cuh"
#include "../../include/propainter_b200.h"

#define LK_WARPS 8

// Staging geometry of window radius R (4: the basic model, 3: RAFT-small).  K = 2R+1 taps per axis; taps b = 0..K-1
// read rows b and b+1, so the box has K+1 rows, and K+1 columns + up to 3 because the box must start 16-byte aligned.
template <int R> struct LkGeom;
template <> struct LkGeom<4> {
  static constexpr int BOX = 10, BOXW = 16;
  static constexpr int LVL_FLOATS = 192;    // 640 B box + pad: level l's box starts 768 B (+0 banks) after level l-1's
};
template <> struct LkGeom<3> {
  static constexpr int BOX = 8, BOXW = 12;
  static constexpr int LVL_FLOATS = 96;     // 384 B box: every level's box starts 128-byte aligned
};

__device__ __forceinline__ uint32_t lk_smem(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

template <int R>
__device__ __forceinline__ int lk_base(float c, float inv) {
  float v = floorf(c * inv);
  v = fminf(fmaxf(v, -1.0e6f), 1.0e6f);
  return (int)v - R;
}

// TO = __half: the taps are blended in fp32 and rounded to nearest once, into rows of ld_out >= 4K^2 halves (the operand
// of the half-precision convc1); TO = float: ld_out = 4K^2.
template <int R, typename TO>
__global__ void __launch_bounds__(LK_WARPS * 32) k_corr_lookup_tma(const __grid_constant__ CUtensorMap tm0,
    const __grid_constant__ CUtensorMap tm1, const __grid_constant__ CUtensorMap tm2,
    const __grid_constant__ CUtensorMap tm3, const float* __restrict__ coords, TO* __restrict__ out, int ld_out, long npix,
    int h, int w) {
  constexpr int K = 2 * R + 1, NCH = 4 * K * K;
  constexpr int LK_BOX = LkGeom<R>::BOX, LK_BOXW = LkGeom<R>::BOXW, LK_LVL_FLOATS = LkGeom<R>::LVL_FLOATS;
  constexpr int LPP = 32 / K, NPASS = (4 + LPP - 1) / LPP;     // levels per pass of the warp, passes
  __shared__ __align__(128) float patch[LK_WARPS][4][LK_LVL_FLOATS];
  __shared__ __align__(8) unsigned long long bar[LK_WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long pix = (long)blockIdx.x * LK_WARPS + warp;
  if (pix >= npix) return;
  const float cx = coords[2 * pix], cy = coords[2 * pix + 1];
  const uint32_t bar_a = lk_smem(&bar[warp]);
  int bx[4], by[4];
#pragma unroll
  for (int l = 0; l < 4; ++l) { bx[l] = lk_base<R>(cx, 1.0f / (float)(1 << l)) & ~3; by[l] = lk_base<R>(cy, 1.0f / (float)(1 << l)); }
  if (lane == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar_a));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_a), "r"(4 * LK_BOX * LK_BOXW * 4) : "memory");
    const CUtensorMap* tms[4] = {&tm0, &tm1, &tm2, &tm3};
#pragma unroll
    for (int l = 0; l < 4; ++l)
      asm volatile(
          "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
          ::"r"(lk_smem(&patch[warp][l][0])), "l"(tms[l]), "r"(bx[l]), "r"(by[l]), "r"((int)pix), "r"(bar_a) : "memory");
  }
  __syncwarp();
  {                                       // wait for the 4 boxes (phase 0), bounded spin
    uint32_t done = 0;
    for (int spin = 0; spin < (1 << 22) && !done; ++spin)
      asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0; selp.u32 %0, 1, 0, p; }"
                   : "=r"(done) : "r"(bar_a) : "memory");
    if (!done) __trap();
  }
  TO* o = out + pix * ld_out;
  // Register-blocked along y: a lane owns one (level, x-tap a) column and slides down the K+1 staged rows, so each
  // shared-memory value is read once per column pair (2(K+1) loads for K taps instead of 4K) and the K results of a lane
  // are K consecutive output floats (index l*K^2 + a*K + b).  A pass covers LPP levels: R = 4 takes levels 0-2 (27
  // lanes), then level 3 (9 lanes); R = 3 takes all 4 levels (28 lanes) in one pass.
  // All taps of a level share the fractional part of the centre (integer tap offsets): corners outside the image read
  // the zeros TMA filled in.  (The reference sends every tap through grid_sample's normalise / un-normalise round trip,
  // RAFT/utils/utils.py:60-65, which only adds ~1e-6 px of rounding noise -- dropped, well inside the 1e-4 tolerance.)
#pragma unroll
  for (int pass = 0; pass < NPASS; ++pass) {
    const int nl = 4 - pass * LPP < LPP ? 4 - pass * LPP : LPP;                 // levels of this pass
    const int l = nl == 1 ? pass * LPP : pass * LPP + lane / K, a = nl == 1 ? lane : lane - K * (lane / K);
    const bool act = lane < nl * K;
    if (act) {
      const float inv = 1.0f / (float)(1 << l);
      const float xl = cx * inv, yl = cy * inv;
      const bool sane = fabsf(xl) < 1.0e6f && fabsf(yl) < 1.0e6f;
      const float wx1 = sane ? xl - floorf(xl) : 0.f, wy1 = sane ? yl - floorf(yl) : 0.f;
      const float wx0 = sane ? 1.0f - wx1 : 0.f, wy0 = sane ? 1.0f - wy1 : 0.f;
      int bxl = bx[0];
      if (l == 1) bxl = bx[1]; else if (l == 2) bxl = bx[2]; else if (l == 3) bxl = bx[3];
      const float* q = &patch[warp][l][0] + (lk_base<R>(cx, inv) - bxl) + a;   // row 0 of this lane's column pair
      float top = wx0 * q[0] + wx1 * q[1];
      TO* ol = o + l * (K * K) + a * K;
#pragma unroll
      for (int b = 0; b < K; ++b) {
        q += LK_BOXW;
        const float bot = wx0 * q[0] + wx1 * q[1];
        pp_st1(ol + b, wy0 * top + wy1 * bot);
        top = bot;
      }
    }
  }
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled lk_encoder() {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess ||
      qres != cudaDriverEntryPointSuccess)
    return nullptr;
  return (PFN_encodeTiled)fn;
}

template <int R, typename TO>
static int corr_lookup_tma(const float* const* levels, const float* coords, TO* out, int ld_out, long n_pairs, int h, int w,
                           cudaStream_t stream) {
  if ((h >> 3) < 2 || (w >> 3) < 2) return PP_ERR_SHAPE;
  if (n_pairs <= 0) return PP_OK;          // nothing to look up: no tensor maps, no zero-block launch
  const long npix = n_pairs * h * w;
  if (npix > 0x7fffffffL) return PP_ERR_SHAPE;
  PFN_encodeTiled enc = lk_encoder();
  if (!enc) return PP_ERR_LAUNCH;
  CUtensorMap tm[4];
  int hl = h, wl = w;
  for (int l = 0; l < 4; ++l) {
    // x extent wl, not the row stride ld: columns wl..ld-1 are row padding, which the TMA unit must zero-fill like any
    // other column outside the level (a tap's right corner at x = wl weighs wx1, and the padding is never written)
    const int ld = pp_corr_ld(wl);
    cuuint64_t dims[3] = {(cuuint64_t)wl, (cuuint64_t)hl, (cuuint64_t)npix};
    cuuint64_t strides[2] = {(cuuint64_t)ld * 4, (cuuint64_t)hl * ld * 4};
    cuuint32_t box[3] = {LkGeom<R>::BOXW, LkGeom<R>::BOX, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    if (((uintptr_t)levels[l] & 15) != 0) return PP_ERR_ALIGN;
    CUresult r = enc(&tm[l], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, (void*)levels[l], dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return PP_ERR_LAUNCH;
    hl >>= 1; wl >>= 1;
  }
  k_corr_lookup_tma<R, TO><<<(int)((npix + LK_WARPS - 1) / LK_WARPS), LK_WARPS * 32, 0, stream>>>(tm[0], tm[1], tm[2], tm[3],
                                                                                                  coords, out, ld_out, npix, h, w);
  if (cudaPeekAtLastError() != cudaSuccess) return PP_ERR_LAUNCH;
  return PP_OK;
}

extern "C" int pp_corr_lookup(const float* const* levels, const float* coords, float* out, long n_pairs, int h, int w,
                              cudaStream_t stream) {
  return corr_lookup_tma<4>(levels, coords, out, 324, n_pairs, h, w, stream);
}

extern "C" int pp_corr_lookup_f16(const float* const* levels, const float* coords, void* out, int ld_out, long n_pairs, int h,
                                  int w, cudaStream_t stream) {
  if (ld_out < 324) return PP_ERR_SHAPE;
  return corr_lookup_tma<4>(levels, coords, (__half*)out, ld_out, n_pairs, h, w, stream);
}

extern "C" int pp_corr_lookup_r(const float* const* levels, int radius, const float* coords, float* out, long n_pairs, int h,
                                int w, cudaStream_t stream) {
  if (radius == 4) return corr_lookup_tma<4>(levels, coords, out, 324, n_pairs, h, w, stream);
  if (radius == 3) return corr_lookup_tma<3>(levels, coords, out, 196, n_pairs, h, w, stream);
  return PP_ERR_SHAPE;
}
