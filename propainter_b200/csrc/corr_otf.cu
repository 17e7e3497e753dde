// RAFT correlation lookup without the all-pairs volume (AlternateCorrBlock, RAFT/corr.py:83-111), sm_90a.
//
// The all-pairs plan stores 4 pooled correlation levels per pair, ~5.4 N^2 bytes (N = h*w feature pixels): 91 GB per
// pair at 3840x2160.  This plan stores the feature pyramid instead and forms the 9x9 window dot products at lookup time.
//
// Pyramid (k_fmap_pool): the reference pools the correlation volume (corr.py:25-27).  Average pooling is linear,
// avgpool_y(f1 . f2) = f1 . avgpool(f2), so pooling fmap2 gives the same levels up to rounding.  Levels 1-3 are pooled
// per frame, not per pair: [frames][(h>>l)*(w>>l)][D], floor sizes like avg_pool2d(2, stride=2), the 2x2 sum in
// pp_pool4's order.  Both flow directions read the same levels; they add ~N*D*4/3 floats per frame.
//
// Lookup (k_corr_lookup_otf, written for D = 256 / radius 4; RAFT-small's D = 128 / radius 3 instance keeps 4 channels
// per lane and an 8x8 tile, see the kernel): one warp per query pixel (pair p, pixel i).  The 81 taps of a level share one
// fractional offset, so the warp computes the 10x10 integer-position dot products f1_i . f2_l[ty0+j][tx0+i] once, in
// fp32 FFMA, keeps them in shared memory and applies pp_corr_tap_tile (the sampling rule of the all-pairs path) to that
// tile.  The result differs from the all-pairs lookup only in the rounding of the dot products.  Lane k holds channels
// [4k, 4k+4) and [128+4k, 128+4k+4) of f1 in registers; for each of the 25 positions of a batch it loads the same
// channels of f2 (two coalesced 512-byte warp loads), and a 31-shuffle butterfly leaves position k's full sum on lane
// k.  Positions outside the level are skipped (zeros padding) on a warp-uniform branch, so a centre anywhere -- also far
// outside the image or non-finite -- reads nothing out of bounds and gives an all-zero window.  Offsets are 64-bit.
//
// Bound, per query pixel and refinement iteration: 4 levels x 100 dot products x D=256 = 204,800 FLOP, and 400 KB of
// f2 read through L1.  Every 512-byte warp load feeds 4 FFMA per lane, so the kernel is L1-throughput bound (4 L1
// wavefronts per 4 warp FFMA instructions): its ceiling is about a quarter of the FP32 peak.  Neighbouring query
// pixels of a CTA share most of their windows under smooth flow, so L2 / HBM traffic is a fraction of the L1 bytes.
#include "pp_elem.cuh"
#include "../../include/propainter_b200.h"

#define OTF_WARPS 8

__global__ void k_fmap_pool(const float* __restrict__ src, float* __restrict__ dst, long n4, int hs, int ws, int hd, int wd,
                            int D) {
  const int d4 = D >> 2;
  for (long e = (long)blockIdx.x * blockDim.x + threadIdx.x; e < n4; e += (long)gridDim.x * blockDim.x) {
    const int c = (int)(e % d4) * 4;
    long r = e / d4;
    const int x = (int)(r % wd);
    r /= wd;
    const int y = (int)(r % hd);
    const long f = r / hd;
    const float* p = src + ((f * hs + 2 * y) * ws + 2 * x) * (long)D + c;
    const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + D);
    const float4 cc = *reinterpret_cast<const float4*>(p + (long)ws * D), d = *reinterpret_cast<const float4*>(p + (long)ws * D + D);
    float4 o;
    o.x = PP_DIV(PP_ADD(PP_ADD(PP_ADD(a.x, b.x), cc.x), d.x), 4.0f);
    o.y = PP_DIV(PP_ADD(PP_ADD(PP_ADD(a.y, b.y), cc.y), d.y), 4.0f);
    o.z = PP_DIV(PP_ADD(PP_ADD(PP_ADD(a.z, b.z), cc.z), d.z), 4.0f);
    o.w = PP_DIV(PP_ADD(PP_ADD(PP_ADD(a.w, b.w), cc.w), d.w), 4.0f);
    *reinterpret_cast<float4*>(dst + ((f * hd + y) * wd + x) * (long)D + c) = o;
  }
}

// channels [4*lane, 4*lane+4) (and [128+4*lane, ...) for D = 256) of f2 at q dotted with the same channels of f1
template <int D>
__device__ __forceinline__ float otf_dot(const float4& a0, const float4& a1, const float* q, int lane) {
  const float4 b0 = __ldg(reinterpret_cast<const float4*>(q) + lane);
  float s = a0.x * b0.x;
  s = fmaf(a0.y, b0.y, s); s = fmaf(a0.z, b0.z, s); s = fmaf(a0.w, b0.w, s);
  if constexpr (D == 256) {
    const float4 b1 = __ldg(reinterpret_cast<const float4*>(q + 128) + lane);
    s = fmaf(a1.x, b1.x, s); s = fmaf(a1.y, b1.y, s); s = fmaf(a1.z, b1.z, s); s = fmaf(a1.w, b1.w, s);
  }
  return s;
}

template <int K>
__device__ __forceinline__ void otf_rs_step(float (&v)[32], int lane) {
  const bool up = (lane & K) != 0;
#pragma unroll
  for (int j = 0; j < K; ++j) {
    const float send = up ? v[j] : v[j + K];
    const float keep = up ? v[j + K] : v[j];
    v[j] = keep + __shfl_xor_sync(0xffffffffu, send, K);
  }
}

// (D, R) = (256, 4): the basic model; (128, 3): RAFT-small (raft.py:29-33, fnet output_dim=128).  The tile is T x T,
// T = 2R+2 (10x10 / 8x8), reduced in batches of BATCH <= 32 positions (4 x 25 / 2 x 32).
template <int D, int R>
__global__ void __launch_bounds__(OTF_WARPS * 32) k_corr_lookup_otf(const float* __restrict__ fmap, const float* __restrict__ pool1,
    const float* __restrict__ pool2, const float* __restrict__ pool3, const int* __restrict__ idx1, const int* __restrict__ idx2,
    const float* __restrict__ coords, float* __restrict__ out, long npix, int h, int w) {
  static_assert(D == 128 || D == 256, "lanes hold 4 or 8 channels");
  constexpr int K = 2 * R + 1, T = 2 * R + 2, NPOS = T * T, NB = (NPOS + 31) / 32, BATCH = NPOS / NB, NCH = 4 * K * K;
  static_assert(NB * BATCH == NPOS, "batches must tile the window");
  __shared__ float tile[OTF_WARPS][NPOS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long pix = (long)blockIdx.x * OTF_WARPS + warp;
  if (pix >= npix) return;                                    // whole warps only: npix is counted in warps
  const long hw = (long)h * w;
  const long pair = pix / hw, i = pix - pair * hw;
  const float cx = coords[2 * pix], cy = coords[2 * pix + 1];
  const float* f1 = fmap + ((long)idx1[pair] * hw + i) * D;
  const float4 a0 = __ldg(reinterpret_cast<const float4*>(f1) + lane);
  float4 a1 = make_float4(0.f, 0.f, 0.f, 0.f);
  if constexpr (D == 256) a1 = __ldg(reinterpret_cast<const float4*>(f1 + 128) + lane);
  const long f2i = idx2[pair];
  float* o = out + pix * NCH;
  float* tl = tile[warp];
#pragma unroll 1
  for (int l = 0; l < 4; ++l) {
    const int hl = h >> l, wl = w >> l;
    const float* f2 = (l == 0 ? fmap : l == 1 ? pool1 : l == 2 ? pool2 : pool3) + f2i * hl * wl * D;
    const int tx0 = pp_corr_tile_origin_r<R>(cx, l), ty0 = pp_corr_tile_origin_r<R>(cy, l);
#pragma unroll 1
    for (int bt = 0; bt < NB; ++bt) {
      float v[32];
#pragma unroll
      for (int k = 0; k < 32; ++k) v[k] = 0.f;
#pragma unroll
      for (int k = 0; k < BATCH; ++k) {
        const int pos = bt * BATCH + k;
        const int yy = ty0 + pos / T, xx = tx0 + pos % T;
        if (yy >= 0 && yy < hl && xx >= 0 && xx < wl)          // warp-uniform
          v[k] = otf_dot<D>(a0, a1, f2 + ((long)yy * wl + xx) * D, lane);
      }
      // reduce-scatter: after the step of width k a lane keeps the k partial sums of its half of the positions
      otf_rs_step<16>(v, lane); otf_rs_step<8>(v, lane); otf_rs_step<4>(v, lane); otf_rs_step<2>(v, lane);
      otf_rs_step<1>(v, lane);
      if (lane < BATCH) {
        if constexpr (D == 256) tl[bt * BATCH + lane] = v[0] * (1.0f / 16.0f);      // / sqrt(D), exact for D = 256
        else tl[bt * BATCH + lane] = __fdiv_rn(v[0], __fsqrt_rn((float)D));       // / torch.sqrt(tensor(D).float())
      }
    }
    __syncwarp();
    for (int t = lane; t < K * K; t += 32) o[l * (K * K) + t] = pp_corr_tap_tile_r<R>(tl, tx0, ty0, hl, wl, cx, cy, l, t / K, t % K);
    __syncwarp();
  }
}

extern "C" int pp_corr_fmap_pyramid(const float* fmap, int D, int frames, int h, int w, float* const* pooled, cudaStream_t stream) {
  if (D <= 0 || (D & 3) || frames <= 0 || (h >> 3) < 1 || (w >> 3) < 1) return PP_ERR_SHAPE;
  if (((uintptr_t)fmap & 15) != 0) return PP_ERR_ALIGN;
  const float* src = fmap;
  int hs = h, ws = w;
  for (int l = 0; l < 3; ++l) {
    if (((uintptr_t)pooled[l] & 15) != 0) return PP_ERR_ALIGN;
    const int hd = hs >> 1, wd = ws >> 1;
    const long n4 = (long)frames * hd * wd * (D >> 2);
    const long blocks = (n4 + 255) / 256;
    k_fmap_pool<<<(int)(blocks < 65536L * 16 ? blocks : 65536L * 16), 256, 0, stream>>>(src, pooled[l], n4, hs, ws, hd, wd, D);
    if (cudaPeekAtLastError() != cudaSuccess) return PP_ERR_LAUNCH;
    src = pooled[l]; hs = hd; ws = wd;
  }
  return PP_OK;
}

template <int D, int R>
static int corr_lookup_otf(const float* fmap, const float* const* pooled, const int* idx1, const int* idx2, int n_pairs,
                           const float* coords, float* out, int h, int w, cudaStream_t stream) {
  if (n_pairs <= 0 || (h >> 3) < 2 || (w >> 3) < 2) return PP_ERR_SHAPE;
  if (((uintptr_t)fmap & 15) || ((uintptr_t)pooled[0] & 15) || ((uintptr_t)pooled[1] & 15) || ((uintptr_t)pooled[2] & 15))
    return PP_ERR_ALIGN;
  const long npix = (long)n_pairs * h * w;
  const long blocks = (npix + OTF_WARPS - 1) / OTF_WARPS;
  if (blocks > 0x7fffffffL) return PP_ERR_SHAPE;
  k_corr_lookup_otf<D, R><<<(unsigned)blocks, OTF_WARPS * 32, 0, stream>>>(fmap, pooled[0], pooled[1], pooled[2], idx1, idx2,
                                                                          coords, out, npix, h, w);
  if (cudaPeekAtLastError() != cudaSuccess) return PP_ERR_LAUNCH;
  return PP_OK;
}

extern "C" int pp_corr_lookup_otf(const float* fmap, const float* const* pooled, int D, const int* idx1, const int* idx2, int n_pairs,
                                  const float* coords, float* out, int h, int w, cudaStream_t stream) {
  if (D != 256) return PP_ERR_SHAPE;
  return corr_lookup_otf<256, 4>(fmap, pooled, idx1, idx2, n_pairs, coords, out, h, w, stream);
}

extern "C" int pp_corr_lookup_otf_r(const float* fmap, const float* const* pooled, int D, int radius, const int* idx1,
                                    const int* idx2, int n_pairs, const float* coords, float* out, int h, int w,
                                    cudaStream_t stream) {
  if (D == 256 && radius == 4) return corr_lookup_otf<256, 4>(fmap, pooled, idx1, idx2, n_pairs, coords, out, h, w, stream);
  if (D == 128 && radius == 3) return corr_lookup_otf<128, 3>(fmap, pooled, idx1, idx2, n_pairs, coords, out, h, w, stream);
  return PP_ERR_SHAPE;
}
