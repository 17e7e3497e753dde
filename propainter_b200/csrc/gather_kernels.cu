// HBM/L2-bound gather, stencil and elementwise kernels of the ProPainter hot path (sm_90a).
// One thread (or one warp) per output element; the per-element rules live in pp_elem.cuh.
#include <stdlib.h>
#include <type_traits>
#include "pp_elem.cuh"
#include "pp_mma.cuh"
#include "../../include/propainter_b200.h"

#define PP_LAUNCH_CHECK() do { if (cudaPeekAtLastError() != cudaSuccess) return PP_ERR_LAUNCH; } while (0)

static inline int pp_blocks(long n, int per) { return (int)((n + per - 1) / per); }

// ================================================================ image propagation scan
__global__ void __launch_bounds__(256) k_imgprop_step(int H, int W, const float* __restrict__ cur,
    const float* __restrict__ mcur, const float* __restrict__ prev, const float* __restrict__ mprev,
    const float* __restrict__ fprop, const float* __restrict__ fcheck, float* __restrict__ out,
    float* __restrict__ mout, int nearest) {
  int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix < H * W) pp_imgprop_pixel(pix, H, W, cur, mcur, prev, mprev, fprop, fcheck, out, mout, nearest);
}

extern "C" size_t pp_img_prop_scan_workspace_bytes(int t, int H, int W) {
  return (size_t)t * 4 * H * W * sizeof(float);
}

// replaces InpaintGenerator.img_propagation (model/propainter.py:315-317 -> :104-190, learnable=False)
extern "C" int pp_img_prop_scan(const float* frames, const float* flows_f, const float* flows_b,
                                const float* masks, float* out_frames, float* out_masks, void* workspace,
                                size_t ws_bytes, int t, int H, int W, int nearest, cudaStream_t stream) {
  if (t < 1 || H < 2 || W < 2) return PP_ERR_SHAPE;
  if (ws_bytes < pp_img_prop_scan_workspace_bytes(t, H, W)) return PP_ERR_WORKSPACE;
  const long HW = (long)H * W;
  float* bf = (float*)workspace;             // backward-scan frames [t][3][HW]
  float* bm = bf + (long)t * 3 * HW;         // backward-scan masks  [t][HW]
  const int blocks = pp_blocks(HW, 256);
  // backward scan: t-1 -> 0, propagates along the forward flows
  cudaMemcpyAsync(bf + (long)(t - 1) * 3 * HW, frames + (long)(t - 1) * 3 * HW, 3 * HW * sizeof(float),
                  cudaMemcpyDeviceToDevice, stream);
  cudaMemcpyAsync(bm + (long)(t - 1) * HW, masks + (long)(t - 1) * HW, HW * sizeof(float),
                  cudaMemcpyDeviceToDevice, stream);
  for (int i = t - 2; i >= 0; --i)
    k_imgprop_step<<<blocks, 256, 0, stream>>>(H, W, frames + (long)i * 3 * HW, masks + (long)i * HW,
        bf + (long)(i + 1) * 3 * HW, bm + (long)(i + 1) * HW, flows_f + (long)i * 2 * HW,
        flows_b + (long)i * 2 * HW, bf + (long)i * 3 * HW, bm + (long)i * HW, nearest);
  // forward scan: consumes the backward scan's frames and masks (:138-139)
  cudaMemcpyAsync(out_frames, bf, 3 * HW * sizeof(float), cudaMemcpyDeviceToDevice, stream);
  cudaMemcpyAsync(out_masks, bm, HW * sizeof(float), cudaMemcpyDeviceToDevice, stream);
  for (int i = 1; i < t; ++i)
    k_imgprop_step<<<blocks, 256, 0, stream>>>(H, W, bf + (long)i * 3 * HW, bm + (long)i * HW,
        out_frames + (long)(i - 1) * 3 * HW, out_masks + (long)(i - 1) * HW, flows_b + (long)(i - 1) * 2 * HW,
        flows_f + (long)(i - 1) * 2 * HW, out_frames + (long)i * 3 * HW, out_masks + (long)i * HW, nearest);
  PP_LAUNCH_CHECK();
  return PP_OK;
}

// ---- the same scan on half-precision clip storage (InferenceConfig.half_storage)
// One step, one pixel.  The current frame is the masked uint8 frame, frames * (1 - masks) widened here (cur == nullptr: a
// backward step), or the backward scan's fp32 result (cur: a forward step).  prev == nullptr: the first frame of a
// direction, copied through (:141-143).  out16 != nullptr: the frame is in the kept range, and the step's epilogue stores
// the composited frame and the updated mask, each rounded once to fp16.  The recurrent state (out, mout) stays fp32.
__global__ void __launch_bounds__(256) k_imgprop_step_u8h(int H, int W, const uint8_t* __restrict__ u8,
    const float* __restrict__ md, const float* __restrict__ cur, const float* __restrict__ mcur,
    const float* __restrict__ prev, const float* __restrict__ mprev, const __half* __restrict__ fprop,
    const __half* __restrict__ fcheck, float* __restrict__ out, float* __restrict__ mout, __half* __restrict__ out16,
    __half* __restrict__ mout16, int nearest) {
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  const int HW = H * W;
  if (pix >= HW) return;
  const float m = md[pix];
  float fr[3], cv[3], ov[3];
  for (int c = 0; c < 3; ++c) {
    fr[c] = pp_u8_frame(u8[3 * (long)pix + c]);
    cv[c] = cur ? cur[(long)c * HW + pix] : PP_MUL(fr[c], PP_SUB(1.0f, m));   // frames * (1 - masks_dilated)
  }
  float mo = mcur ? mcur[pix] : m;
  if (prev) mo = pp_imgprop_values(pix, H, W, cv, mo, prev, mprev, fprop, fcheck, ov, nearest);
  else for (int c = 0; c < 3; ++c) ov[c] = cv[c];
  if (out) {
    for (int c = 0; c < 3; ++c) out[(long)c * HW + pix] = ov[c];
    mout[pix] = mo;
  }
  if (out16) {
    for (int c = 0; c < 3; ++c) out16[(long)c * HW + pix] = __float2half_rn(pp_imgprop_compose(fr[c], ov[c], m));
    mout16[pix] = __float2half_rn(mo);
  }
}

extern "C" size_t pp_img_prop_scan_u8h_workspace_bytes(int t, int H, int W) {
  return ((size_t)t + 2) * 4 * H * W * sizeof(float);
}

// pp_img_prop_scan on clip storage, composited (model/propainter.py:315-317; inference_propainter.py:372, 389-390, 402):
// see include/propainter_b200.h
extern "C" int pp_img_prop_scan_u8h(const uint8_t* frames_u8, const float* masks, const void* flows_f, const void* flows_b,
                                    void* out_frames, void* out_masks, void* workspace, size_t ws_bytes, int t, int H, int W,
                                    int lo, int hi, int nearest, cudaStream_t stream) {
  if (t < 0 || H < 2 || W < 2 || lo < 0 || lo > hi || hi > t) return PP_ERR_SHAPE;
  if (((uintptr_t)flows_f | (uintptr_t)flows_b | (uintptr_t)out_frames | (uintptr_t)out_masks) & 1) return PP_ERR_ALIGN;
  if (((uintptr_t)masks | (uintptr_t)workspace) & 3) return PP_ERR_ALIGN;
  if (lo == hi) return PP_OK;                                // nothing kept: no launch
  if (ws_bytes < pp_img_prop_scan_u8h_workspace_bytes(t, H, W)) return PP_ERR_WORKSPACE;
  const long HW = (long)H * W;
  const __half* ff = (const __half*)flows_f;
  const __half* fb = (const __half*)flows_b;
  __half* of = (__half*)out_frames;
  __half* om = (__half*)out_masks;
  float* bf = (float*)workspace;             // backward-scan frames [t][3][HW]
  float* bm = bf + (long)t * 3 * HW;         // backward-scan masks  [t][HW]
  float* rf = bm + (long)t * HW;             // forward-scan state, a two-frame ring: frames [2][3][HW]
  float* rm = rf + 2 * 3 * HW;               //                                       masks  [2][HW]
  const int blocks = pp_blocks(HW, 256);
#define PP_U8(i) (frames_u8 + (long)(i) * 3 * HW)
#define PP_MD(i) (masks + (long)(i) * HW)
  // backward scan: t-1 -> 0, propagates along the forward flows
  k_imgprop_step_u8h<<<blocks, 256, 0, stream>>>(H, W, PP_U8(t - 1), PP_MD(t - 1), nullptr, nullptr, nullptr, nullptr,
      nullptr, nullptr, bf + (long)(t - 1) * 3 * HW, bm + (long)(t - 1) * HW, nullptr, nullptr, nearest);
  for (int i = t - 2; i >= 0; --i)
    k_imgprop_step_u8h<<<blocks, 256, 0, stream>>>(H, W, PP_U8(i), PP_MD(i), nullptr, nullptr,
        bf + (long)(i + 1) * 3 * HW, bm + (long)(i + 1) * HW, ff + (long)i * 2 * HW, fb + (long)i * 2 * HW,
        bf + (long)i * 3 * HW, bm + (long)i * HW, nullptr, nullptr, nearest);
  // forward scan: consumes the backward scan's frames and masks (:138-139); frame 0 is the backward result itself
  if (lo == 0)
    k_imgprop_step_u8h<<<blocks, 256, 0, stream>>>(H, W, PP_U8(0), PP_MD(0), bf, bm, nullptr, nullptr, nullptr, nullptr,
        nullptr, nullptr, of, om, nearest);
  for (int i = 1; i < hi; ++i) {
    const float* pf = i == 1 ? bf : rf + (long)((i - 1) & 1) * 3 * HW;
    const float* pm = i == 1 ? bm : rm + (long)((i - 1) & 1) * HW;
    const bool keep = i >= lo;
    k_imgprop_step_u8h<<<blocks, 256, 0, stream>>>(H, W, PP_U8(i), PP_MD(i), bf + (long)i * 3 * HW, bm + (long)i * HW,
        pf, pm, fb + (long)(i - 1) * 2 * HW, ff + (long)(i - 1) * 2 * HW, rf + (long)(i & 1) * 3 * HW, rm + (long)(i & 1) * HW,
        keep ? of + (long)(i - lo) * 3 * HW : nullptr, keep ? om + (long)(i - lo) * HW : nullptr, nearest);
  }
#undef PP_U8
#undef PP_MD
  PP_LAUNCH_CHECK();
  return PP_OK;
}

// ================================================================ learnable propagation: cond assembly
// One warp per pixel: lane 0 evaluates the sampling coordinate + fb-consistency and broadcasts it by
// shuffle; the 32 lanes then gather the 4 bilinear corners as float4 channel vectors (coalesced 512 B
// per corner for C=128) and write the concat buffers the offset-net / backbone convs consume.
__global__ void __launch_bounds__(256) k_prop_cond(int h, int w, int C, const float* __restrict__ cur, int ld_cur,
    const float* __restrict__ prop, int ld_prop, const float* __restrict__ fprop,
    const float* __restrict__ fcheck, const float* __restrict__ mcur, float* __restrict__ cond, int ld_cond,
    float* __restrict__ bb, int ld_bb, int first) {
  const int lane = threadIdx.x & 31;
  const long pix = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (pix >= (long)h * w) return;
  const int y = (int)(pix / w), x = (int)(pix - (long)y * w);
  float ix = 0.f, iy = 0.f, valid = 0.f, fx = 0.f, fy = 0.f;
  if (!first) {
    if (lane == 0) {
      PPCond c = pp_cond_pixel(y, x, h, w, fprop, fcheck);
      ix = c.ix; iy = c.iy; valid = c.valid; fx = c.fx; fy = c.fy;
    }
    ix = __shfl_sync(0xffffffffu, ix, 0); iy = __shfl_sync(0xffffffffu, iy, 0);
    valid = __shfl_sync(0xffffffffu, valid, 0);
    fx = __shfl_sync(0xffffffffu, fx, 0); fy = __shfl_sync(0xffffffffu, fy, 0);
  }
  const PPTaps t = first ? PPTaps() : pp_taps(ix, iy, h, w);
  const float* curp = cur + pix * ld_cur;
  float* bbp = bb + pix * ld_bb;
  float* cdp = first ? nullptr : cond + pix * ld_cond;
  for (int c = lane * 4; c < C; c += 128) {
    const float4 v = *reinterpret_cast<const float4*>(curp + c);
    *reinterpret_cast<float4*>(bbp + c) = v;
    if (first) {
      *reinterpret_cast<float4*>(bbp + C + c) = v;          // feat_prop = feat_current (:141-143)
    } else {
      *reinterpret_cast<float4*>(cdp + c) = v;
      *reinterpret_cast<float4*>(cdp + C + c) = pp_tap_nhwc4(prop, ld_prop, w, t, c);
    }
  }
  if (lane == 0) {
    const float m0 = mcur[2 * pix], m1 = mcur[2 * pix + 1];
    bbp[2 * C] = m0; bbp[2 * C + 1] = m1;
    for (int c = 2 * C + 2; c < ld_bb; ++c) bbp[c] = 0.f;
    if (!first) {
      cdp[2 * C] = fx; cdp[2 * C + 1] = fy; cdp[2 * C + 2] = valid; cdp[2 * C + 3] = m0; cdp[2 * C + 4] = m1;
      for (int c = 2 * C + 5; c < ld_cond; ++c) cdp[c] = 0.f;
    }
  }
}

// replaces the flow_warp + fbConsistencyCheck + torch.cat prologue of one step of
// BidirectionalPropagation(learnable=True) (model/propainter.py:144-166)
extern "C" int pp_prop_cond(const float* cur, int ld_cur, const float* prop, int ld_prop, const float* fprop,
                            const float* fcheck, const float* mcur, float* cond, int ld_cond, float* bb, int ld_bb,
                            int h, int w, int C, int first, cudaStream_t stream) {
  if (C % 4 || ld_cur % 4 || ld_prop % 4 || ld_cond % 4 || ld_bb % 4) return PP_ERR_ALIGN;
  if (ld_bb < 2 * C + 2 || (!first && ld_cond < 2 * C + 5)) return PP_ERR_SHAPE;
  const long n = (long)h * w;
  k_prop_cond<<<pp_blocks(n, 8), 256, 0, stream>>>(h, w, C, cur, ld_cur, prop, ld_prop, fprop, fcheck, mcur, cond,
                                                    ld_cond, bb, ld_bb, first);
  PP_LAUNCH_CHECK();
  return PP_OK;
}

// flow_warp + fbConsistencyCheck as a standalone op (SURVEY.md section 8b "flow_warp_fbcheck"), batched over n maps.
// One warp per pixel; every lane derives the sampling position itself from the pixel's flow (two broadcast loads) instead
// of waiting for lane 0 + shuffles, then gathers the 4 bilinear corners as float4 channel vectors (coalesced 512 B per
// corner for C = 128).  `aux` (optional) receives (fx, fy, valid): the step-independent condition channels of
// DeformableAlignment's offset net, so their share of conv_offset.0 can be convolved once per scan.  TW = __half: `warped`
// is stored rounded to nearest fp16 (the operand of the fp16 scan convs); the sampling stays fp32.
template <typename TW>
__global__ void __launch_bounds__(256) k_flow_warp(long npix, int h, int w, int C, const float* __restrict__ feat, int ld_f,
    const float* __restrict__ fprop, const float* __restrict__ fcheck, TW* __restrict__ warped, int ld_w,
    float* __restrict__ aux, int ld_a, int round_tf32) {
  asm volatile("griddepcontrol.launch_dependents;");              // programmatic dependent launch (see conv_umma.cu)
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const int lane = threadIdx.x & 31;
  const long pix = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (pix >= npix) return;
  const long HW = (long)h * w, img = pix / HW, pim = pix - img * HW;
  const int y = (int)(pim / w), x = (int)(pim - (long)y * w);
  const float* fp = fprop + img * HW * 2;
  const float fx = fp[2 * pim], fy = fp[2 * pim + 1];
  const float ix = pp_warp_coord((float)x, fx, w), iy = pp_warp_coord((float)y, fy, h);
  const PPTaps t = pp_taps(ix, iy, h, w);
  if (warped) {
    const float* f = feat + img * HW * ld_f;
    TW* o = warped + pix * ld_w;
    for (int c = lane * 4; c < C; c += 128) {
      float4 v = pp_tap_nhwc4(f, ld_f, w, t, c);
      if constexpr (std::is_same<TW, __half>::value) {
        const __half2 lo = __floats2half2_rn(v.x, v.y), hi = __floats2half2_rn(v.z, v.w);
        uint2 u;
        u.x = *reinterpret_cast<const uint32_t*>(&lo); u.y = *reinterpret_cast<const uint32_t*>(&hi);
        *reinterpret_cast<uint2*>(o + c) = u;
      } else {
        if (round_tf32) {
          v.x = __uint_as_float(pp_tf32(v.x)); v.y = __uint_as_float(pp_tf32(v.y));
          v.z = __uint_as_float(pp_tf32(v.z)); v.w = __uint_as_float(pp_tf32(v.w));
        }
        *reinterpret_cast<float4*>(o + c) = v;
      }
    }
  }
  if (aux && lane == 0) {
    const PPCond c = pp_cond_pixel(y, x, h, w, fp, fcheck + img * HW * 2);
    float* a = aux + pix * ld_a;
    a[0] = c.fx; a[1] = c.fy; a[2] = c.valid;
  }
}

template <typename TW>
static int fw_run(const float* feat, int ld_f, const float* fprop, const float* fcheck, TW* warped, int ld_w, float* aux, int ld_a,
                  int n, int h, int w, int C, int round_tf32, cudaStream_t stream) {
  const int lda = sizeof(TW) == 2 ? 8 : 4;                       // fp16 rows: 16-byte row strides (a conv operand)
  if (n < 1 || h < 1 || w < 1 || (!warped && !aux)) return PP_ERR_SHAPE;
  if (warped && (!feat || C % 4 || ld_f % 4 || ld_w % lda || ((uintptr_t)feat & 15) || ((uintptr_t)warped & 15))) return PP_ERR_ALIGN;
  if (aux && (!fcheck || ld_a < 3)) return PP_ERR_SHAPE;
  const long npix = (long)n * h * w;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)pp_blocks(npix, 8)); cfg.blockDim = dim3(256); cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  const char* env = getenv("PP_PDL");
  cfg.attrs = attr; cfg.numAttrs = (env && env[0] == '0') ? 0 : 1;
  if (cudaLaunchKernelEx(&cfg, k_flow_warp<TW>, npix, h, w, C, feat, ld_f, fprop, fcheck, warped, ld_w, aux, ld_a, round_tf32) != cudaSuccess)
    return PP_ERR_LAUNCH;
  PP_LAUNCH_CHECK();
  return PP_OK;
}

// flow_warp (model/modules/flow_loss_utils.py:6-45, bilinear / zeros / align_corners=True) of pixel-major maps and
// fbConsistencyCheck (model/propainter.py:22-31); see include/propainter_b200.h
extern "C" int pp_flow_warp_fbcheck(const float* feat, int ld_f, const float* fprop, const float* fcheck, float* warped, int ld_w,
                                    float* aux, int ld_a, int n, int h, int w, int C, int round_tf32, cudaStream_t stream) {
  return fw_run(feat, ld_f, fprop, fcheck, warped, ld_w, aux, ld_a, n, h, w, C, round_tf32, stream);
}

extern "C" int pp_flow_warp_fbcheck_f16(const float* feat, int ld_f, const float* fprop, const float* fcheck, void* warped, int ld_w,
                                        float* aux, int ld_a, int n, int h, int w, int C, cudaStream_t stream) {
  return fw_run(feat, ld_f, fprop, fcheck, static_cast<__half*>(warped), ld_w, aux, ld_a, n, h, w, C, 0, stream);
}

// ================================================================ RAFT correlation pyramid + lookup
__global__ void __launch_bounds__(256) k_corr_pool(const float* __restrict__ src, float* __restrict__ dst, long planes,
                                                   int Hs, int lds, int Hd, int Wd, int ldd) {
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  long per = (long)Hd * Wd;
  if (i >= planes * per) return;
  long p = i / per; int r = (int)(i - p * per); int y = r / Wd, x = r - y * Wd;
  dst[p * (long)Hd * ldd + (long)y * ldd + x] = pp_pool4(src + p * (long)Hs * lds, lds, y, x);
}

// RAFT/corr.py:25-27: levels 1..3 from level 0 (level 0 is written by pp_corr_build)
extern "C" int pp_corr_pool_pyramid(float* const* levels, long planes, int h, int w, cudaStream_t stream) {
  int hs = h, ws = w;
  for (int l = 1; l < 4; ++l) {
    int hd = hs / 2, wd = ws / 2;
    if (hd < 2 || wd < 2) return PP_ERR_SHAPE;        // the reference divides by (size-1): NaN below 2
    long n = planes * hd * wd;
    k_corr_pool<<<pp_blocks(n, 256), 256, 0, stream>>>(levels[l - 1], levels[l], planes, hs, pp_corr_ld(ws), hd, wd,
                                                        pp_corr_ld(wd));
    hs = hd; ws = wd;
  }
  PP_LAUNCH_CHECK();
  return PP_OK;
}

struct PPLevels { const float* p[4]; };

// One warp per source pixel: 4 levels x K^2 taps (K = 2R+1: 81 for radius 4, 49 for radius 3); each lane walks taps
// lane, lane+32, ... so that the 4K^2 results of a pixel are written as one contiguous run (pixel-major output feeds
// the 1x1 motion-encoder conv directly).  The per-pixel planes (<= 6.7 KB + 1.7 + 0.4 + 0.1) stay in L1.
template <int R, typename TO>
__global__ void __launch_bounds__(256) k_corr_lookup(PPLevels lv, const float* __restrict__ coords,
                                                     TO* __restrict__ out, int ld_out, long npix, int h, int w) {
  constexpr int K = 2 * R + 1;
  const int lane = threadIdx.x & 31;
  const long pix = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (pix >= npix) return;
  const float cx = coords[2 * pix], cy = coords[2 * pix + 1];
  TO* o = out + pix * ld_out;
  int hl = h, wl = w;
#pragma unroll
  for (int l = 0; l < 4; ++l) {
    const int ld = pp_corr_ld(wl);
    const float* plane = lv.p[l] + pix * (long)hl * ld;
    for (int tap = lane; tap < K * K; tap += 32)
      pp_st1(o + l * (K * K) + tap, pp_corr_tap_r<R>(plane, hl, wl, ld, cx, cy, l, tap / K, tap % K));
    hl >>= 1; wl >>= 1;
  }
}

template <int R, typename TO>
static int corr_lookup_ldg(const float* const* levels, const float* coords, TO* out, int ld_out, long n_pairs, int h, int w,
                           cudaStream_t stream) {
  if ((h >> 3) < 2 || (w >> 3) < 2) return PP_ERR_SHAPE;
  if (n_pairs <= 0) return PP_OK;          // a zero-block grid would leave a launch error behind for the next kernel
  PPLevels lv;
  for (int l = 0; l < 4; ++l) lv.p[l] = levels[l];
  const long npix = n_pairs * h * w;
  k_corr_lookup<R, TO><<<pp_blocks(npix, 8), 256, 0, stream>>>(lv, coords, out, ld_out, npix, h, w);
  PP_LAUNCH_CHECK();
  return PP_OK;
}

// Plain-load variant of the lookup (kept as the measured baseline of the TMA-staged kernel in
// corr_lookup_tma.cu; same contract as pp_corr_lookup)
extern "C" int pp_corr_lookup_ldg(const float* const* levels, const float* coords, float* out, long n_pairs, int h,
                              int w, cudaStream_t stream) {
  return corr_lookup_ldg<4>(levels, coords, out, 324, n_pairs, h, w, stream);
}
// fp16 output rows of ld_out >= 324 halves (pp_corr_lookup_f16's contract)
extern "C" int pp_corr_lookup_ldg_f16(const float* const* levels, const float* coords, void* out, int ld_out, long n_pairs, int h,
                                      int w, cudaStream_t stream) {
  if (ld_out < 324) return PP_ERR_SHAPE;
  return corr_lookup_ldg<4>(levels, coords, (__half*)out, ld_out, n_pairs, h, w, stream);
}
// the same with window radius 3 or 4 (pp_corr_lookup_r's contract)
extern "C" int pp_corr_lookup_ldg_r(const float* const* levels, int radius, const float* coords, float* out, long n_pairs,
                                    int h, int w, cudaStream_t stream) {
  if (radius == 4) return corr_lookup_ldg<4>(levels, coords, out, 324, n_pairs, h, w, stream);
  if (radius == 3) return corr_lookup_ldg<3>(levels, coords, out, 196, n_pairs, h, w, stream);
  return PP_ERR_SHAPE;
}

__global__ void __launch_bounds__(256) k_convex_up(const float* __restrict__ mask, int ld_mask, float mask_scale,
    const float* __restrict__ flow_lr, float* __restrict__ out, int n, int h, int w) {
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;        // over n*h*w*64, sub-pixel fastest
  long total = (long)n * h * w * 64;
  if (i >= total) return;
  int sub = (int)(i & 63); long px = i >> 6;
  int b = (int)(px / ((long)h * w)); int r = (int)(px - (long)b * h * w); int y = r / w, x = r - y * w;
  int si = sub >> 3, sj = sub & 7;
  float2 v = pp_convex_up(mask + px * ld_mask, mask_scale, flow_lr + (long)b * h * w * 2, h, w, y, x, si, sj);
  const long H = 8L * h, W = 8L * w;
  float* ob = out + (long)b * 2 * H * W + (8L * y + si) * W + 8L * x + sj;
  ob[0] = v.x; ob[H * W] = v.y;
}

// replaces RAFT.upsample_flow (RAFT/raft.py:73-84); mask_scale folds update.py:135's 0.25
extern "C" int pp_convex_upsample(const float* mask, int ld_mask, float mask_scale, const float* flow_lr, float* out,
                                  int n, int h, int w, cudaStream_t stream) {
  if (ld_mask < 576) return PP_ERR_SHAPE;
  long total = (long)n * h * w * 64;
  k_convex_up<<<pp_blocks(total, 256), 256, 0, stream>>>(mask, ld_mask, mask_scale, flow_lr, out, n, h, w);
  PP_LAUNCH_CHECK();
  return PP_OK;
}

// ================================================================ generator input preparation
template <typename TF>
__global__ void __launch_bounds__(256) k_gen_prep(const TF* __restrict__ flows_f, const TF* __restrict__ flows_b,
    const float* __restrict__ masks_in, const float* __restrict__ masks_upd, float* __restrict__ dsf,
    float* __restrict__ dsb, float* __restrict__ pmask, int lt, int H, int W) {
  const int h = H / 4, w = W / 4;
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  long per = (long)h * w;
  if (i >= (long)lt * per) return;
  int f = (int)(i / per); int r = (int)(i - (long)f * per); int y = r / w, x = r - y * w;
  const long HW = (long)H * W;
  if (f < lt - 1) {
    const TF* pf = flows_f + (long)f * 2 * HW; const TF* pb = flows_b + (long)f * 2 * HW;
    dsf[2 * i] = pp_flow_ds4(pf, W, y, x); dsf[2 * i + 1] = pp_flow_ds4(pf + HW, W, y, x);
    dsb[2 * i] = pp_flow_ds4(pb, W, y, x); dsb[2 * i + 1] = pp_flow_ds4(pb + HW, W, y, x);
  }
  pmask[2 * i] = masks_in[(long)f * HW + (long)(4 * y) * W + 4 * x];          // 'nearest' 1/4: element [4i,4j]
  pmask[2 * i + 1] = masks_upd[(long)f * HW + (long)(4 * y) * W + 4 * x];
}

// replaces the F.interpolate block of InpaintGenerator.forward (model/propainter.py:338-342, :352)
extern "C" int pp_gen_prep(const float* flows_f, const float* flows_b, const float* masks_in, const float* masks_upd,
                           float* dsf, float* dsb, float* pmask, int lt, int H, int W, cudaStream_t stream) {
  if (H % 4 || W % 4 || lt < 1) return PP_ERR_SHAPE;
  long n = (long)lt * (H / 4) * (W / 4);
  k_gen_prep<float><<<pp_blocks(n, 256), 256, 0, stream>>>(flows_f, flows_b, masks_in, masks_upd, dsf, dsb, pmask, lt, H, W);
  PP_LAUNCH_CHECK();
  return PP_OK;
}
// the same on fp16 clip-storage flows (2-byte aligned), widened on load
extern "C" int pp_gen_prep_f16(const void* flows_f, const void* flows_b, const float* masks_in, const float* masks_upd,
                               float* dsf, float* dsb, float* pmask, int lt, int H, int W, cudaStream_t stream) {
  if (H < 0 || W < 0 || H % 4 || W % 4 || lt < 1) return PP_ERR_SHAPE;
  if (((uintptr_t)flows_f | (uintptr_t)flows_b) & 1) return PP_ERR_ALIGN;
  if (((uintptr_t)masks_in | (uintptr_t)masks_upd | (uintptr_t)dsf | (uintptr_t)dsb | (uintptr_t)pmask) & 3) return PP_ERR_ALIGN;
  const long n = (long)lt * (H / 4) * (W / 4);
  if (n == 0) return PP_OK;                                  // an empty frame: no launch
  k_gen_prep<__half><<<pp_blocks(n, 256), 256, 0, stream>>>((const __half*)flows_f, (const __half*)flows_b, masks_in, masks_upd,
                                                            dsf, dsb, pmask, lt, H, W);
  PP_LAUNCH_CHECK();
  return PP_OK;
}

// window flag = any(local frame) any(token in window) any(7x7/s3/p3 patch pixel) of the 1/4-res input mask
__global__ void __launch_bounds__(128) k_window_mask(const float* __restrict__ pmask, int lt, int h, int w, int fh,
                                                     int fw, int nww, int* __restrict__ flags) {
  const int win = blockIdx.x;
  const int wy = win / nww, wx = win - wy * nww;
  int hit = 0;
  const int per = 5 * 9 * 49;
  for (int i = threadIdx.x; i < lt * per; i += blockDim.x) {
    int f = i / per, r = i - f * per;
    int tok = r / 49, tap = r - tok * 49;
    int ty = wy * 5 + tok / 9, tx = wx * 9 + tok % 9;
    if (ty >= fh || tx >= fw) continue;                    // zero padding of the token grid (:168-170)
    int y = 3 * ty - 3 + tap / 7, x = 3 * tx - 3 + tap % 7;
    if (y < 0 || y >= h || x < 0 || x >= w) continue;
    if (pmask[2 * ((long)f * h * w + (long)y * w + x)] > 0.f) hit = 1;
  }
  hit = __syncthreads_or(hit);
  if (threadIdx.x == 0) flags[win] = hit;
}

// replaces max_pool (propainter.py:349-350) + SparseWindowAttention's window max-pool/sum (:224-229)
extern "C" int pp_window_mask(const float* pmask, int lt, int h, int w, int fh, int fw, int nwh, int nww, int* flags,
                              cudaStream_t stream) {
  k_window_mask<<<nwh * nww, 128, 0, stream>>>(pmask, lt, h, w, fh, fw, nww, flags);
  PP_LAUNCH_CHECK();
  return PP_OK;
}

// ================================================================ fusion feed-forward overlap-add
// fold (+ /count + GELU, applied once per feature pixel instead of once per (token, tap)) ...
// T = __half (the transformer's half-operand Linear layers): fc1's fp16 output in, fc2's fp16 operand out; the fold sums in
// fp32 in the same order and the workspace F stays fp32, so the result is the fp32 kernel's on the widened rows, rounded once.
template <typename T>
__global__ void __launch_bounds__(256) k_ffn_fold_gelu(const T* __restrict__ Y, int ldy, int CH, int fh, int fw, int h,
                                                       int w, float* __restrict__ F) {
  const int c4n = CH >> 2;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;       // over h*w*(CH/4) of frame blockIdx.y
  if (i >= h * w * c4n) return;
  const int c = (i % c4n) * 4, px = i / c4n, y = px / w, x = px - y * w;
  const T* Yf = Y + (long)blockIdx.y * fh * fw * ldy;
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  int n = 0;
  for (int ty = (y + 3) / 3, ky; ty >= 0 && (ky = y + 3 - 3 * ty) < 7; --ty) {
    if (ty >= fh) continue;
    for (int tx = (x + 3) / 3, kx; tx >= 0 && (kx = x + 3 - 3 * tx) < 7; --tx) {
      if (tx >= fw) continue;
      const float4 v = pp_ld4(Yf + (long)(ty * fw + tx) * ldy + (ky * 7 + kx) * CH + c);
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
      ++n;
    }
  }
  const float d = (float)n;
  float4 o;
  o.x = pp_gelu(s.x / d); o.y = pp_gelu(s.y / d); o.z = pp_gelu(s.z / d); o.w = pp_gelu(s.w / d);
  *reinterpret_cast<float4*>(F + ((long)blockIdx.y * h * w + px) * CH + c) = o;
}
// ... then unfold is a pure gather-copy (out-of-image taps read as gelu(0) = 0)
template <typename T>
__global__ void __launch_bounds__(256) k_ffn_unfold(const float* __restrict__ F, int CH, int fh, int fw, int h, int w,
                                                    T* __restrict__ Z, int ldz) {
  const int c4n = CH >> 2;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;       // over fh*fw*49*(CH/4) of frame blockIdx.y
  if (i >= fh * fw * 49 * c4n) return;
  const int c = (i % c4n) * 4, r = i / c4n, tap = r % 49, tok = r / 49, ty = tok / fw, tx = tok - ty * fw;
  const int y = 3 * ty - 3 + tap / 7, x = 3 * tx - 3 + tap % 7;
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (y >= 0 && y < h && x >= 0 && x < w)
    v = *reinterpret_cast<const float4*>(F + (((long)blockIdx.y * h + y) * w + x) * CH + c);
  pp_st4(Z + ((long)blockIdx.y * fh * fw + tok) * ldz + tap * CH + c, v);
}

extern "C" size_t pp_ffn_overlap_add_workspace_bytes(int frames, int h, int w, int CH) {
  return (size_t)frames * h * w * CH * sizeof(float);
}
template <typename T>
static int pp_ffn_launch(const T* Y, int ldy, T* Z, int ldz, int frames, int h, int w, int CH, void* workspace, size_t ws_bytes,
                         cudaStream_t stream) {
  const int fh = (h - 1) / 3 + 1, fw = (w - 1) / 3 + 1;
  if (ws_bytes < pp_ffn_overlap_add_workspace_bytes(frames, h, w, CH)) return PP_ERR_WORKSPACE;
  float* F = (float*)workspace;
  const long n1 = (long)h * w * (CH / 4), n2 = (long)fh * fw * 49 * (CH / 4);
  if (n2 > 0x7fffffffL) return PP_ERR_SHAPE;
  k_ffn_fold_gelu<T><<<dim3(pp_blocks(n1, 256), frames), 256, 0, stream>>>(Y, ldy, CH, fh, fw, h, w, F);
  k_ffn_unfold<T><<<dim3(pp_blocks(n2, 256), frames), 256, 0, stream>>>(F, CH, fh, fw, h, w, Z, ldz);
  PP_LAUNCH_CHECK();
  return PP_OK;
}
// replaces fold -> /normalizer -> unfold -> GELU of FusionFeedForward.forward
// (model/modules/sparse_transformer.py:81-100).  Y,Z: [frames*fh*fw][ld], columns tap-major (tap*CH+c).
extern "C" int pp_ffn_overlap_add(const float* Y, int ldy, float* Z, int ldz, int frames, int h, int w, int CH,
                                  void* workspace, size_t ws_bytes, cudaStream_t stream) {
  if (ldy < 49 * CH || ldz < 49 * CH || frames < 1 || frames > 65535) return PP_ERR_SHAPE;
  if (CH % 4 || ldy % 4 || ldz % 4) return PP_ERR_ALIGN;
  return pp_ffn_launch(Y, ldy, Z, ldz, frames, h, w, CH, workspace, ws_bytes, stream);
}
// the same on fp16 rows of Y and Z (16-byte aligned, ld % 8 == 0); frames = 0 returns PP_OK without a launch
extern "C" int pp_ffn_overlap_add_f16(const void* Y, int ldy, void* Z, int ldz, int frames, int h, int w, int CH,
                                      void* workspace, size_t ws_bytes, cudaStream_t stream) {
  if (ldy < 49 * CH || ldz < 49 * CH || frames < 0 || frames > 65535) return PP_ERR_SHAPE;
  if (CH % 4 || ldy % 8 || ldz % 8 || ((uintptr_t)Y & 15) || ((uintptr_t)Z & 15) || ((uintptr_t)workspace & 15)) return PP_ERR_ALIGN;
  if (frames == 0 || h <= 0 || w <= 0) return PP_OK;
  return pp_ffn_launch((const __half*)Y, ldy, (__half*)Z, ldz, frames, h, w, CH, workspace, ws_bytes, stream);
}

// ================================================================ SoftComp fold
// SoftComp's Linear(512 -> 6272) + fold(7x7, stride 3, pad 3) (model/modules/sparse_transformer.py:49-61) as a GEMM into
// tap-major columns (tap*C + c) followed by this overlap-add: out[f,y,x,c] = sum over the tokens whose 7x7 patch covers
// (y,x) of cols[token][tap*C + c], in a fixed order (ty, tx descending), plus bmap[y,x,c], the fold of the Linear bias.
// T = __half: fp16 columns in, fp16 out (sc.bias_conv's operand); the sum is fp32 and rounded once.  No atomics, so the
// result is the same on every run.
template <typename T>
__global__ void __launch_bounds__(256) k_sc_fold(const T* __restrict__ cols, long ldc, const float* __restrict__ bmap, int C,
                                                 int fh, int fw, int h, int w, T* __restrict__ out) {
  const int c4n = C >> 2;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;       // over h*w*(C/4) of frame blockIdx.y
  if (i >= h * w * c4n) return;
  const int c = (i % c4n) * 4, px = i / c4n, y = px / w, x = px - y * w;
  const T* cf = cols + (long)blockIdx.y * fh * fw * ldc;
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int ty = (y + 3) / 3, ky; ty >= 0 && (ky = y + 3 - 3 * ty) < 7; --ty) {
    if (ty >= fh) continue;
    for (int tx = (x + 3) / 3, kx; tx >= 0 && (kx = x + 3 - 3 * tx) < 7; --tx) {
      if (tx >= fw) continue;
      const float4 v = pp_ld4(cf + (long)(ty * fw + tx) * ldc + (ky * 7 + kx) * C + c);
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
  }
  const float4 b = *reinterpret_cast<const float4*>(bmap + (long)px * C + c);
  pp_st4(out + ((long)blockIdx.y * h * w + px) * C + c, make_float4(s.x + b.x, s.y + b.y, s.z + b.z, s.w + b.w));
}
// cols: fp16 [frames*fh*fw][ldc], fh = (h-1)/3+1, fw = (w-1)/3+1; bmap fp32 [h][w][C]; out fp16 [frames][h][w][C].
// frames = 0 returns PP_OK without a launch.
extern "C" int pp_sc_fold_f16(const void* cols, long ldc, const float* bmap, void* out, int frames, int h, int w, int C,
                              cudaStream_t stream) {
  if (frames < 0 || frames > 65535 || h < 1 || w < 1 || C < 4 || ldc < 49L * C || (long)h * w * C > 0x7fffffffL) return PP_ERR_SHAPE;
  if (C % 4 || ldc % 4 || ((uintptr_t)cols & 7) || ((uintptr_t)out & 7) || ((uintptr_t)bmap & 15)) return PP_ERR_ALIGN;
  if (frames == 0) return PP_OK;
  k_sc_fold<__half><<<dim3(pp_blocks((long)h * w * (C / 4), 256), frames), 256, 0, stream>>>(
      (const __half*)cols, ldc, bmap, C, (h - 1) / 3 + 1, (w - 1) / 3 + 1, h, w, (__half*)out);
  PP_LAUNCH_CHECK();
  return PP_OK;
}

// ================================================================ conv epilogue + x2 upsampling
// out = post(act(x + bias[c]) + res) on pixel-major tensors with explicit pixel strides: one pass instead of cuDNN's
// separate bias add_ kernel, the activation kernel, the residual add and (with a strided `out`) the torch.cat that
// would place the result into a concat buffer.  act: 0 none, 1 relu, 2 leaky(slope), 3 sigmoid, 4 tanh; bias / res may
// be NULL; post_relu applies a final ReLU (residual blocks).  out may alias x.  TX / TO: fp32 or fp16 rows of x / out
// (the half-operand convs of RAFT's refinement loop); bias, pre, res and the arithmetic stay fp32.
template <typename TX, typename TO>
__global__ void __launch_bounds__(256) k_bias_act(const TX* x, int ld_x, const float* __restrict__ bias, const float* res,
                                                  int ld_res, TO* out, int ld_out, long n_pix, int C, int act, float slope,
                                                  int post_relu, const float* __restrict__ pre = nullptr, int ld_pre = 0) {
  const int c4n = C >> 2;
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pix * c4n) return;
  const long pix = i / c4n; const int c = (int)(i - pix * c4n) * 4;
  const float4 v = pp_ld4(x + pix * ld_x + c);
  float r[4] = {v.x, v.y, v.z, v.w};
  if (bias != nullptr) {
    const float4 b = *reinterpret_cast<const float4*>(bias + c);
    r[0] += b.x; r[1] += b.y; r[2] += b.z; r[3] += b.w;
  }
  if (pre != nullptr) {                           // per-pixel pre-activation addend: a conv share computed ahead of the scan
    const float4 b = *reinterpret_cast<const float4*>(pre + pix * ld_pre + c);
    r[0] += b.x; r[1] += b.y; r[2] += b.z; r[3] += b.w;
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    float t = r[k];
    if (act == 1) t = fmaxf(t, 0.f);
    else if (act == 2) t = t > 0.f ? t : t * slope;
    else if (act == 3) t = 1.0f / (1.0f + expf(-t));
    else if (act == 4) t = tanhf(t);
    r[k] = t;
  }
  if (res != nullptr) {
    const float4 q = *reinterpret_cast<const float4*>(res + pix * ld_res + c);
    r[0] += q.x; r[1] += q.y; r[2] += q.z; r[3] += q.w;
  }
  if (post_relu) {
#pragma unroll
    for (int k = 0; k < 4; ++k) r[k] = fmaxf(r[k], 0.f);
  }
  pp_st4(out + pix * ld_out + c, make_float4(r[0], r[1], r[2], r[3]));
}
// replaces the bias add of F.conv2d, the following ReLU / LeakyReLU / sigmoid / tanh call, the residual `x + y`
// (+ ReLU) of the encoder blocks / propagation backbones, and the torch.cat into a concat buffer
extern "C" int pp_bias_act(const float* x, int ld_x, const float* bias, const float* res, int ld_res, float* out, int ld_out,
                           long n_pix, int C, int act, float slope, int post_relu, cudaStream_t stream) {
  if (C % 4 || ld_x % 4 || ld_out % 4 || (res && ld_res % 4)) return PP_ERR_ALIGN;
  if (((uintptr_t)x & 15) || ((uintptr_t)out & 15) || ((uintptr_t)bias & 15) || ((uintptr_t)res & 15)) return PP_ERR_ALIGN;
  if (ld_x < C || ld_out < C || (res && ld_res < C) || act < 0 || act > 4) return PP_ERR_SHAPE;
  if (n_pix <= 0) return PP_OK;
  k_bias_act<float, float><<<pp_blocks(n_pix * (C / 4), 256), 256, 0, stream>>>(x, ld_x, bias, res, ld_res, out, ld_out, n_pix, C,
                                                                              act, slope, post_relu);
  PP_LAUNCH_CHECK();
  return PP_OK;
}

// pp_bias_act with a per-pixel pre-activation addend: out = post(act(x + bias + pre) + res).  conv(cat[a, b]) =
// conv_a(a) + conv_b(b): the share of a recurrent step's conv that only sees step-independent inputs (current frame, flow,
// masks) is convolved once per scan for all frames and enters here (model/propainter.py:151,171,
// model/recurrent_flow_completion.py:96-106).
extern "C" int pp_bias_act_pre(const float* x, int ld_x, const float* bias, const float* pre, int ld_pre, const float* res,
                               int ld_res, float* out, int ld_out, long n_pix, int C, int act, float slope, int post_relu,
                               cudaStream_t stream) {
  if (pre == nullptr) return pp_bias_act(x, ld_x, bias, res, ld_res, out, ld_out, n_pix, C, act, slope, post_relu, stream);
  if (C % 4 || ld_x % 4 || ld_out % 4 || ld_pre % 4 || (res && ld_res % 4)) return PP_ERR_ALIGN;
  if (((uintptr_t)x & 15) || ((uintptr_t)out & 15) || ((uintptr_t)bias & 15) || ((uintptr_t)res & 15) || ((uintptr_t)pre & 15))
    return PP_ERR_ALIGN;
  if (ld_x < C || ld_out < C || ld_pre < C || (res && ld_res < C) || act < 0 || act > 4) return PP_ERR_SHAPE;
  if (n_pix <= 0) return PP_OK;
  k_bias_act<float, float><<<pp_blocks(n_pix * (C / 4), 256), 256, 0, stream>>>(x, ld_x, bias, res, ld_res, out, ld_out, n_pix, C,
                                                                              act, slope, post_relu, pre, ld_pre);
  PP_LAUNCH_CHECK();
  return PP_OK;
}

// pp_bias_act_pre with fp16 x (x_f16) and / or fp16 out (out_f16); fp16 rows 8-byte aligned, fp32 ones 16-byte.
extern "C" int pp_bias_act_f16(const void* x, int ld_x, int x_f16, const float* bias, const float* pre, int ld_pre, const float* res,
                               int ld_res, void* out, int ld_out, int out_f16, long n_pix, int C, int act, float slope, int post_relu,
                               cudaStream_t stream) {
  if (C % 4 || ld_x % 4 || ld_out % 4 || (pre && ld_pre % 4) || (res && ld_res % 4)) return PP_ERR_ALIGN;
  if (((uintptr_t)x & (x_f16 ? 7 : 15)) || ((uintptr_t)out & (out_f16 ? 7 : 15)) || ((uintptr_t)bias & 15) || ((uintptr_t)res & 15) ||
      ((uintptr_t)pre & 15))
    return PP_ERR_ALIGN;
  if (ld_x < C || ld_out < C || (pre && ld_pre < C) || (res && ld_res < C) || act < 0 || act > 4) return PP_ERR_SHAPE;
  if (n_pix <= 0) return PP_OK;
  const int nb = pp_blocks(n_pix * (C / 4), 256);
  if (x_f16 && out_f16)
    k_bias_act<__half, __half><<<nb, 256, 0, stream>>>((const __half*)x, ld_x, bias, res, ld_res, (__half*)out, ld_out, n_pix, C, act,
                                                       slope, post_relu, pre, ld_pre);
  else if (x_f16)
    k_bias_act<__half, float><<<nb, 256, 0, stream>>>((const __half*)x, ld_x, bias, res, ld_res, (float*)out, ld_out, n_pix, C, act,
                                                      slope, post_relu, pre, ld_pre);
  else if (out_f16)
    k_bias_act<float, __half><<<nb, 256, 0, stream>>>((const float*)x, ld_x, bias, res, ld_res, (__half*)out, ld_out, n_pix, C, act,
                                                      slope, post_relu, pre, ld_pre);
  else
    k_bias_act<float, float><<<nb, 256, 0, stream>>>((const float*)x, ld_x, bias, res, ld_res, (float*)out, ld_out, n_pix, C, act,
                                                     slope, post_relu, pre, ld_pre);
  PP_LAUNCH_CHECK();
  return PP_OK;
}

// ================================================================ InstanceNorm (RAFT feature encoder)
// RAFT/extractor.py:18-21,125 (nn.InstanceNorm2d, affine=False, eps 1e-5) on channels-last maps [n][HW][C]:
// per (sample, channel) biased mean / variance over HW.  Pass 1 writes per-chunk partial sums of the pivot-shifted values
// in double (pp_inorm_acc) and the pivots; pass 2 folds them (pp_inorm_fold) and applies (x-mean)*rstd, the ReLU that
// always follows, and optionally the block's residual add + ReLU.  3 passes over the map (2 reads, 1 write) instead of
// F.instance_norm's NHWC->NCHW copy, batch_norm and copy back.  The pivots are copied to the workspace so that pass 2 may
// overwrite pixel 0 in place.
__global__ void __launch_bounds__(256) k_inorm_stats(const float* __restrict__ x, long HW, int C, int chunk, int S,
                                                     double* __restrict__ part, float* __restrict__ pivot) {
  __shared__ double sh[8][256];
  const int c4n = C >> 2, R = 256 / c4n;
  const int q = threadIdx.x % c4n, r = threadIdx.x / c4n;
  const long n = blockIdx.y; const int s = blockIdx.x;
  const long r0 = (long)s * chunk; const long r1 = r0 + chunk < HW ? r0 + chunk : HW;
  const float4 p = *reinterpret_cast<const float4*>(x + n * HW * C + 4 * q);
  double a[4] = {0.0, 0.0, 0.0, 0.0}, b[4] = {0.0, 0.0, 0.0, 0.0};
  if (r < R)
    for (long row = r0 + r; row < r1; row += R) {
      const float4 v = *reinterpret_cast<const float4*>(x + (n * HW + row) * C + 4 * q);
      pp_inorm_acc(a[0], b[0], v.x, p.x); pp_inorm_acc(a[1], b[1], v.y, p.y);
      pp_inorm_acc(a[2], b[2], v.z, p.z); pp_inorm_acc(a[3], b[3], v.w, p.w);
    }
#pragma unroll
  for (int e = 0; e < 4; ++e) { sh[e][threadIdx.x] = a[e]; sh[4 + e][threadIdx.x] = b[e]; }
  __syncthreads();
  if (r == 0) {
    for (int j = 1; j < R; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) { a[e] += sh[e][j * c4n + q]; b[e] += sh[4 + e][j * c4n + q]; }
    double* dst = part + ((n * S + s) * 2) * C + 4 * q;
#pragma unroll
    for (int e = 0; e < 4; ++e) { dst[e] = a[e]; dst[C + e] = b[e]; }
    if (s == 0) *reinterpret_cast<float4*>(pivot + n * C + 4 * q) = p;
  }
}
__global__ void __launch_bounds__(256) k_inorm_apply(const float* x, const double* __restrict__ part, const float* __restrict__ pivot,
                                                     int S, const float* res, float* out, long HW, int C, int chunk, float eps,
                                                     int relu, int post_relu) {
  __shared__ PPNormStat s_st[512];
  const long n = blockIdx.y; const int s = blockIdx.x;
  for (int c = threadIdx.x; c < C; c += 256) {
    double su = 0.0, sq = 0.0;
    for (int j = 0; j < S; ++j) {
      su += part[((n * S + j) * 2) * C + c];
      sq += part[((n * S + j) * 2 + 1) * C + c];
    }
    s_st[c] = pp_inorm_fold(su, sq, HW, pivot[n * C + c], eps);
  }
  __syncthreads();
  const int c4n = C >> 2, R = 256 / c4n;
  const int q = threadIdx.x % c4n, r = threadIdx.x / c4n;
  if (r >= R) return;
  const long r0 = (long)s * chunk; const long r1 = r0 + chunk < HW ? r0 + chunk : HW;
  for (long row = r0 + r; row < r1; row += R) {
    const long off = (n * HW + row) * C + 4 * q;
    const float4 v = *reinterpret_cast<const float4*>(x + off);
    const float4 t = res ? *reinterpret_cast<const float4*>(res + off) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float vx[4] = {v.x, v.y, v.z, v.w}, tx[4] = {t.x, t.y, t.z, t.w};
    float y[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) y[e] = pp_inorm_out(vx[e], s_st[4 * q + e], relu, res ? &tx[e] : nullptr, post_relu);
    *reinterpret_cast<float4*>(out + off) = make_float4(y[0], y[1], y[2], y[3]);
  }
}
// workspace: n*S*2*C double partial sums, then n*C float pivots
extern "C" size_t pp_instance_norm_workspace_bytes(int n, long HW, int C) {
  return (size_t)n * pp_inorm_splits(n, HW) * 2 * C * sizeof(double) + (size_t)n * C * sizeof(float);
}
// replaces F.instance_norm (+ F.relu, + the residual `relu(x + y)` of ResidualBlock.forward extractor.py:49-57)
extern "C" int pp_instance_norm(const float* x, const float* res, float* out, int n, long HW, int C, float eps, int relu,
                                int post_relu, void* workspace, size_t ws_bytes, cudaStream_t stream) {
  if (C % 4 || ((uintptr_t)x & 15) || ((uintptr_t)out & 15) || ((uintptr_t)res & 15) || ((uintptr_t)workspace & 15)) return PP_ERR_ALIGN;
  if (C < 4 || C > 512 || n < 1 || n > 65535 || HW < 1) return PP_ERR_SHAPE;
  if (ws_bytes < pp_instance_norm_workspace_bytes(n, HW, C)) return PP_ERR_WORKSPACE;
  const int S = pp_inorm_splits(n, HW);
  const int chunk = (int)((HW + S - 1) / S);
  double* part = (double*)workspace;
  float* pivot = (float*)(part + (size_t)n * S * 2 * C);
  k_inorm_stats<<<dim3(S, n), 256, 0, stream>>>(x, HW, C, chunk, S, part, pivot);
  k_inorm_apply<<<dim3(S, n), 256, 0, stream>>>(x, part, pivot, S, res, out, HW, C, chunk, eps, relu, post_relu);
  PP_LAUNCH_CHECK();
  return PP_OK;
}

// T = __half (the generator's half-operand decoder): fp16 rows in and out, the blend in fp32, the result rounded once; each
// thread takes 8 channels (16-byte loads and stores) instead of 4.
template <typename T>
__global__ void __launch_bounds__(256) k_upsample2x(const T* __restrict__ src, T* __restrict__ dst, int n, int h, int w, int C) {
  constexpr int V = 16 / sizeof(T);                            // channels per thread
  const int cvn = C >> (V == 4 ? 2 : 3), H = 2 * h, W = 2 * w;
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;  // over n*H*W*(C/V)
  if (i >= (long)n * H * W * cvn) return;
  const int c = (int)(i % cvn) * V; const long px = i / cvn;
  const int b = (int)(px / ((long)H * W)); const int r = (int)(px - (long)b * H * W); const int y = r / W, x = r - y * W;
  const PPUp uy = pp_up2_coord(y, h), ux = pp_up2_coord(x, w);
  const T* p = src + (((long)b * h + uy.i0) * w + ux.i0) * C + c;
#pragma unroll
  for (int k = 0; k < V; k += 4) {
    const float4 v00 = pp_ld4(p + k), v01 = pp_ld4(p + (long)ux.step * C + k);
    const float4 v10 = pp_ld4(p + (long)uy.step * w * C + k);
    const float4 v11 = pp_ld4(p + ((long)uy.step * w + ux.step) * C + k);
    float4 o;
    o.x = pp_up2_blend(v00.x, v01.x, v10.x, v11.x, uy, ux); o.y = pp_up2_blend(v00.y, v01.y, v10.y, v11.y, uy, ux);
    o.z = pp_up2_blend(v00.z, v01.z, v10.z, v11.z, uy, ux); o.w = pp_up2_blend(v00.w, v01.w, v10.w, v11.w, uy, ux);
    pp_st4(dst + i * V + k, o);
  }
}
// replaces F.interpolate(scale_factor=2, mode='bilinear', align_corners=True) of `deconv`
// (model/propainter.py:248-253, model/recurrent_flow_completion.py:141-146); pixel-major in/out
extern "C" int pp_upsample2x_bilinear(const float* src, float* dst, int n, int h, int w, int C, cudaStream_t stream) {
  if (C % 4) return PP_ERR_ALIGN;
  if (h < 2 || w < 2) return PP_ERR_SHAPE;
  const long total = (long)n * 4 * h * w * (C / 4);
  k_upsample2x<float><<<pp_blocks(total, 256), 256, 0, stream>>>(src, dst, n, h, w, C);
  PP_LAUNCH_CHECK();
  return PP_OK;
}
// the same on fp16 rows (16-byte aligned, C % 8 == 0); n = 0 returns PP_OK without a launch
extern "C" int pp_upsample2x_bilinear_f16(const void* src, void* dst, int n, int h, int w, int C, cudaStream_t stream) {
  if (C % 8 || ((uintptr_t)src & 15) || ((uintptr_t)dst & 15)) return PP_ERR_ALIGN;
  if (n < 0 || h < 2 || w < 2) return PP_ERR_SHAPE;
  if (n == 0) return PP_OK;
  const long total = (long)n * 4 * h * w * (C / 8);
  k_upsample2x<__half><<<pp_blocks(total, 256), 256, 0, stream>>>((const __half*)src, (__half*)dst, n, h, w, C);
  PP_LAUNCH_CHECK();
  return PP_OK;
}

// ================================================================ RAFT SepConvGRU elementwise fusion
// RAFT/update.py:45-60.  The recurrent state lives in two persistent pixel-major buffers
//   HX = [net | inp | motion | flow]   (input of the z/r gate conv)
//   RX = [r*net | inp | motion | flow] (input of the candidate conv)
// so no torch.cat is needed inside the 20-iteration loop.
// T = __half (half-operand gate convs): zr / q are the fp16 conv outputs and r*h goes into an fp16 RX; the state `net`,
// z, bias and pre stay fp32, and gru_update writes the fp16 image of the new state into HX (h_img).
template <typename T>
__global__ void __launch_bounds__(256) k_gru_gate(const T* __restrict__ zr, const float* __restrict__ bias,
    const float* __restrict__ pre, const float* __restrict__ net, int ld_net, float* __restrict__ z, T* __restrict__ rnet,
    int ld_r, long npix, int C) {
  const int c4n = C >> 2;
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npix * c4n) return;
  const long pix = i / c4n; const int c = (int)(i - pix * c4n) * 4;
  float4 zv = pp_ld4(zr + pix * 2 * C + c), rv = pp_ld4(zr + pix * 2 * C + C + c);
  float4 bz = make_float4(0.f, 0.f, 0.f, 0.f), br = bz;
  if (bias != nullptr) { bz = *reinterpret_cast<const float4*>(bias + c); br = *reinterpret_cast<const float4*>(bias + C + c); }
  if (pre != nullptr) {           // iteration-invariant part of the gate convs (context features), precomputed per pixel
    const float4 pz = *reinterpret_cast<const float4*>(pre + pix * 2 * C + c), pr = *reinterpret_cast<const float4*>(pre + pix * 2 * C + C + c);
    zv.x += pz.x; zv.y += pz.y; zv.z += pz.z; zv.w += pz.w; rv.x += pr.x; rv.y += pr.y; rv.z += pr.z; rv.w += pr.w;
  }
  const float4 h = *reinterpret_cast<const float4*>(net + pix * ld_net + c);
  float4 zo, ro;
  zo.x = 1.0f / (1.0f + expf(-(zv.x + bz.x))); zo.y = 1.0f / (1.0f + expf(-(zv.y + bz.y)));
  zo.z = 1.0f / (1.0f + expf(-(zv.z + bz.z))); zo.w = 1.0f / (1.0f + expf(-(zv.w + bz.w)));
  ro.x = h.x / (1.0f + expf(-(rv.x + br.x))); ro.y = h.y / (1.0f + expf(-(rv.y + br.y)));
  ro.z = h.z / (1.0f + expf(-(rv.z + br.z))); ro.w = h.w / (1.0f + expf(-(rv.w + br.w)));
  *reinterpret_cast<float4*>(z + pix * C + c) = zo;
  pp_st4(rnet + pix * ld_r + c, ro);
}
template <typename T>
__global__ void __launch_bounds__(256) k_gru_update(const T* __restrict__ q, const float* __restrict__ bias,
    const float* __restrict__ pre, const float* __restrict__ z, float* __restrict__ net, int ld_net, T* __restrict__ h_img,
    int ld_img, T* __restrict__ net_copy, long npix, int C) {
  const int c4n = C >> 2;
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npix * c4n) return;
  const long pix = i / c4n; const int c = (int)(i - pix * c4n) * 4;
  float4 qv = pp_ld4(q + pix * C + c), b = make_float4(0.f, 0.f, 0.f, 0.f);
  if (bias != nullptr) b = *reinterpret_cast<const float4*>(bias + c);
  if (pre != nullptr) {
    const float4 pq = *reinterpret_cast<const float4*>(pre + pix * C + c);
    qv.x += pq.x; qv.y += pq.y; qv.z += pq.z; qv.w += pq.w;
  }
  const float4 zv = *reinterpret_cast<const float4*>(z + pix * C + c);
  float4 h = *reinterpret_cast<float4*>(net + pix * ld_net + c);
  h.x = (1.0f - zv.x) * h.x + zv.x * tanhf(qv.x + b.x); h.y = (1.0f - zv.y) * h.y + zv.y * tanhf(qv.y + b.y);
  h.z = (1.0f - zv.z) * h.z + zv.z * tanhf(qv.z + b.z); h.w = (1.0f - zv.w) * h.w + zv.w * tanhf(qv.w + b.w);
  *reinterpret_cast<float4*>(net + pix * ld_net + c) = h;
  if (h_img != nullptr) pp_st4(h_img + pix * ld_img + c, h);
  if (net_copy != nullptr) pp_st4(net_copy + pix * C + c, h);                    // dense copy for the flow / mask heads
}
// z = sigmoid(conv_z), r*h (update.py:47-49 / :54-56): zr = raw output of the fused z|r conv [npix][2C]
extern "C" int pp_gru_gate(const float* zr, const float* bias, const float* pre, const float* net, int ld_net, float* z,
                           float* rnet, int ld_r, long npix, int C, cudaStream_t stream) {
  if (C % 4 || ld_net % 4 || ld_r % 4 || ((uintptr_t)zr & 15) || ((uintptr_t)net & 15) || ((uintptr_t)z & 15) ||
      ((uintptr_t)rnet & 15) || ((uintptr_t)pre & 15) || ((uintptr_t)bias & 15))
    return PP_ERR_ALIGN;
  if (npix <= 0) return PP_OK;
  k_gru_gate<float><<<pp_blocks(npix * (C / 4), 256), 256, 0, stream>>>(zr, bias, pre, net, ld_net, z, rnet, ld_r, npix, C);
  PP_LAUNCH_CHECK();
  return PP_OK;
}
// the same with the fp16 gate conv output `zr` and an fp16 rnet slice (8-byte aligned rows); net, z, bias, pre fp32
extern "C" int pp_gru_gate_f16(const void* zr, const float* bias, const float* pre, const float* net, int ld_net, float* z,
                               void* rnet, int ld_r, long npix, int C, cudaStream_t stream) {
  if (C % 4 || ld_net % 4 || ld_r % 4 || ((uintptr_t)zr & 7) || ((uintptr_t)rnet & 7) || ((uintptr_t)net & 15) ||
      ((uintptr_t)z & 15) || ((uintptr_t)pre & 15) || ((uintptr_t)bias & 15))
    return PP_ERR_ALIGN;
  if (npix <= 0) return PP_OK;
  k_gru_gate<__half><<<pp_blocks(npix * (C / 4), 256), 256, 0, stream>>>((const __half*)zr, bias, pre, net, ld_net, z, (__half*)rnet,
                                                                        ld_r, npix, C);
  PP_LAUNCH_CHECK();
  return PP_OK;
}
// h = (1-z)*h + z*tanh(conv_q) in place (update.py:50-51 / :57-58); net_copy (nullable) also receives h densely
extern "C" int pp_gru_update(const float* q, const float* bias, const float* pre, const float* z, float* net, int ld_net,
                             float* net_copy, long npix, int C, cudaStream_t stream) {
  if (C % 4 || ld_net % 4 || ((uintptr_t)q & 15) || ((uintptr_t)z & 15) || ((uintptr_t)net & 15) || ((uintptr_t)net_copy & 15) ||
      ((uintptr_t)pre & 15) || ((uintptr_t)bias & 15))
    return PP_ERR_ALIGN;
  if (npix <= 0) return PP_OK;
  k_gru_update<float><<<pp_blocks(npix * (C / 4), 256), 256, 0, stream>>>(q, bias, pre, z, net, ld_net, nullptr, 0, net_copy, npix, C);
  PP_LAUNCH_CHECK();
  return PP_OK;
}
// the same with the fp16 candidate conv output `q`: the fp32 state `net` is updated in place and its fp16 image is written
// to h_img (ld_img; the state slice of HX, nullable) and net_copy (dense, nullable)
extern "C" int pp_gru_update_f16(const void* q, const float* bias, const float* pre, const float* z, float* net, int ld_net,
                                 void* h_img, int ld_img, void* net_copy, long npix, int C, cudaStream_t stream) {
  if (C % 4 || ld_net % 4 || ld_img % 4 || ((uintptr_t)q & 7) || ((uintptr_t)h_img & 7) || ((uintptr_t)net_copy & 7) ||
      ((uintptr_t)net & 15) || ((uintptr_t)z & 15) || ((uintptr_t)pre & 15) || ((uintptr_t)bias & 15))
    return PP_ERR_ALIGN;
  if (npix <= 0) return PP_OK;
  k_gru_update<__half><<<pp_blocks(npix * (C / 4), 256), 256, 0, stream>>>((const __half*)q, bias, pre, z, net, ld_net, (__half*)h_img,
                                                                          ld_img, (__half*)net_copy, npix, C);
  PP_LAUNCH_CHECK();
  return PP_OK;
}
// motion features [out(126) | flow(2)] (update.py:95-97) written into the same channel slot of two buffers
template <typename T>
__global__ void __launch_bounds__(256) k_raft_pack_motion(const T* __restrict__ mot, int ld_mot, const float* __restrict__ bias,
    const float* __restrict__ flow, T* __restrict__ d0, T* __restrict__ d1, int ld, long npix) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;   // 32 float4 per pixel (128 channels)
  if (i >= npix * 32) return;
  const long pix = i >> 5; const int c = (int)(i & 31) * 4;
  float4 v = pp_ld4(mot + pix * ld_mot + c);
  if (bias != nullptr) {                                        // raw conv output: bias + ReLU of update.py:96 applied here
    const float4 b = *reinterpret_cast<const float4*>(bias + c);
    v.x = fmaxf(v.x + b.x, 0.f); v.y = fmaxf(v.y + b.y, 0.f); v.z = fmaxf(v.z + b.z, 0.f); v.w = fmaxf(v.w + b.w, 0.f);
  }
  if (c == 124) { v.z = flow[2 * pix]; v.w = flow[2 * pix + 1]; }
  pp_st4(d0 + pix * ld + c, v);
  pp_st4(d1 + pix * ld + c, v);
}
extern "C" int pp_raft_pack_motion(const float* mot, int ld_mot, const float* bias, const float* flow, float* d0, float* d1,
                                   int ld, long npix, cudaStream_t stream) {
  if (ld % 4 || ld_mot % 4 || ((uintptr_t)mot & 15) || ((uintptr_t)d0 & 15) || ((uintptr_t)d1 & 15) || ((uintptr_t)bias & 15))
    return PP_ERR_ALIGN;
  if (npix <= 0) return PP_OK;
  k_raft_pack_motion<float><<<pp_blocks(npix * 32, 256), 256, 0, stream>>>(mot, ld_mot, bias, flow, d0, d1, ld, npix);
  PP_LAUNCH_CHECK();
  return PP_OK;
}
// the same from the fp16 motion conv output into fp16 HX / RX slots (8-byte aligned rows); bias and flow fp32
extern "C" int pp_raft_pack_motion_f16(const void* mot, int ld_mot, const float* bias, const float* flow, void* d0, void* d1, int ld,
                                       long npix, cudaStream_t stream) {
  if (ld % 4 || ld_mot % 4 || ((uintptr_t)mot & 7) || ((uintptr_t)d0 & 7) || ((uintptr_t)d1 & 7) || ((uintptr_t)bias & 15))
    return PP_ERR_ALIGN;
  if (npix <= 0) return PP_OK;
  k_raft_pack_motion<__half><<<pp_blocks(npix * 32, 256), 256, 0, stream>>>((const __half*)mot, ld_mot, bias, flow, (__half*)d0,
                                                                            (__half*)d1, ld, npix);
  PP_LAUNCH_CHECK();
  return PP_OK;
}

// the same for a motion conv of any width (RAFT-small: SmallMotionEncoder.conv, 80 channels, update.py:62-77): channels
// [0,cmot) of `mot` (+ bias, ReLU) and the 2 flow channels fill [0, cmot+2) of the slot, zeros its pad up to
// roundup4(cmot+2).  Scalar reads: `mot` / `bias` need only cmot channels.
__global__ void __launch_bounds__(256) k_raft_pack_motion_n(const float* __restrict__ mot, int ld_mot, const float* __restrict__ bias,
    const float* __restrict__ flow, float* __restrict__ d0, float* __restrict__ d1, int ld, long npix, int cmot) {
  const int s4 = (cmot + 5) >> 2;                                 // float4 per slot row
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npix * s4) return;
  const long pix = i / s4; const int c = (int)(i - pix * s4) * 4;
  float v[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int e = c + k;
    float x = 0.f;
    if (e < cmot) {
      x = mot[pix * ld_mot + e];
      if (bias != nullptr) x = fmaxf(x + bias[e], 0.f);
    } else if (e < cmot + 2) {
      x = flow[2 * pix + (e - cmot)];
    }
    v[k] = x;
  }
  const float4 o = make_float4(v[0], v[1], v[2], v[3]);
  *reinterpret_cast<float4*>(d0 + pix * ld + c) = o;
  *reinterpret_cast<float4*>(d1 + pix * ld + c) = o;
}
extern "C" int pp_raft_pack_motion_n(const float* mot, int ld_mot, const float* bias, const float* flow, float* d0, float* d1,
                                     int ld, long npix, int cmot, cudaStream_t stream) {
  if (cmot < 1 || ld_mot < cmot || ld < ((cmot + 5) & ~3) || npix < 0) return PP_ERR_SHAPE;
  if (ld % 4 || ((uintptr_t)d0 & 15) || ((uintptr_t)d1 & 15)) return PP_ERR_ALIGN;
  if (npix == 0) return PP_OK;
  k_raft_pack_motion_n<<<pp_blocks(npix * ((cmot + 5) >> 2), 256), 256, 0, stream>>>(mot, ld_mot, bias, flow, d0, d1, ld, npix, cmot);
  PP_LAUNCH_CHECK();
  return PP_OK;
}

// upflow8 of RAFT-small (raft.py:136-137, RAFT/utils/utils.py:80-82): one thread per output pixel, both flow channels.
// flow_lr pixel-major [n][h][w][2] -> out planar [n][2][8h][8w], the rule of pp_upflow8_coord / pp_upflow8_blend.
__global__ void __launch_bounds__(256) k_upflow8(const float* __restrict__ flow_lr, float* __restrict__ out, int n, int h, int w) {
  const long H = 8L * h, W = 8L * w;
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;     // over n*H*W
  if (i >= (long)n * H * W) return;
  const long b = i / (H * W), r = i - b * H * W;
  const int y = (int)(r / W), x = (int)(r - (long)y * W);
  const PPLin uy = pp_upflow8_coord(y, h), ux = pp_upflow8_coord(x, w);
  const float2* f = reinterpret_cast<const float2*>(flow_lr) + b * h * w;
  const float2 v00 = f[(long)uy.i0 * w + ux.i0], v01 = f[(long)uy.i0 * w + ux.i1];
  const float2 v10 = f[(long)uy.i1 * w + ux.i0], v11 = f[(long)uy.i1 * w + ux.i1];
  float* o = out + b * 2 * H * W + r;
  o[0] = pp_upflow8_blend(v00.x, v01.x, v10.x, v11.x, uy, ux);
  o[H * W] = pp_upflow8_blend(v00.y, v01.y, v10.y, v11.y, uy, ux);
}
extern "C" int pp_upflow8(const float* flow_lr, float* out, int n, int h, int w, cudaStream_t stream) {
  if (n < 1 || h < 1 || w < 1) return PP_ERR_SHAPE;
  if ((uintptr_t)flow_lr & 7) return PP_ERR_ALIGN;
  if ((long)n * 64 * h * w / 256 >= 0x7fffffffL) return PP_ERR_SHAPE;
  k_upflow8<<<pp_blocks((long)n * 64 * h * w, 256), 256, 0, stream>>>(flow_lr, out, n, h, w);
  PP_LAUNCH_CHECK();
  return PP_OK;
}

// ================================================================ transformer glue
// pool_layer of SparseWindowAttention (sparse_transformer.py:131-133,203-206): depthwise Conv2d with kernel = stride =
// pool_size, no padding, on the pixel-major token grid.  x [n][H][W][C] (pixel stride ld_x), w tap-major [kh*kw][C].
// T = __half: the fp16 LayerNorm output in, fp16 pooled tokens out (the operand of the pooled K/V Linear); weights, bias and
// the fma chain stay fp32, rounded once on the store.
template <typename T>
__global__ void __launch_bounds__(256) k_pool_depthwise(const T* __restrict__ x, int ld_x, const float* __restrict__ w,
    const float* __restrict__ bias, T* __restrict__ out, int n, int H, int W, int C, int kh, int kw, int ph, int pw) {
  const int c4n = C >> 2;
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)n * ph * pw * c4n) return;
  const int c = (int)(i % c4n) * 4; long r = i / c4n;
  const int px = (int)(r % pw); r /= pw; const int py = (int)(r % ph); const int f = (int)(r / ph);
  float4 acc = *reinterpret_cast<const float4*>(bias + c);
  for (int a = 0; a < kh; ++a)
    for (int b = 0; b < kw; ++b) {
      const float4 v = pp_ld4(x + (((long)f * H + (py * kh + a)) * W + (px * kw + b)) * ld_x + c);
      const float4 k = *reinterpret_cast<const float4*>(w + (long)(a * kw + b) * C + c);
      acc.x = fmaf(v.x, k.x, acc.x); acc.y = fmaf(v.y, k.y, acc.y); acc.z = fmaf(v.z, k.z, acc.z); acc.w = fmaf(v.w, k.w, acc.w);
    }
  pp_st4(out + i * 4, acc);
}
extern "C" int pp_pool_depthwise(const float* x, int ld_x, const float* w_taps, const float* bias, float* out, int n, int H, int W,
                                 int C, int kh, int kw, cudaStream_t stream) {
  if (C % 4 || ld_x % 4 || ((uintptr_t)x & 15) || ((uintptr_t)w_taps & 15) || ((uintptr_t)bias & 15) || ((uintptr_t)out & 15))
    return PP_ERR_ALIGN;
  if (kh < 1 || kw < 1 || H < kh || W < kw || n < 1 || ld_x < C) return PP_ERR_SHAPE;
  const int ph = (H - kh) / kh + 1, pw = (W - kw) / kw + 1;
  const long total = (long)n * ph * pw * (C / 4);
  k_pool_depthwise<float><<<pp_blocks(total, 256), 256, 0, stream>>>(x, ld_x, w_taps, bias, out, n, H, W, C, kh, kw, ph, pw);
  PP_LAUNCH_CHECK();
  return PP_OK;
}
// the same on fp16 x and out (16-byte aligned, C % 8 == 0, ld_x % 8 == 0); n = 0 returns PP_OK without a launch
extern "C" int pp_pool_depthwise_f16(const void* x, int ld_x, const float* w_taps, const float* bias, void* out, int n, int H, int W,
                                     int C, int kh, int kw, cudaStream_t stream) {
  if (C % 8 || ld_x % 8 || ((uintptr_t)x & 15) || ((uintptr_t)w_taps & 15) || ((uintptr_t)bias & 15) || ((uintptr_t)out & 15))
    return PP_ERR_ALIGN;
  if (kh < 1 || kw < 1 || n < 0 || ld_x < C) return PP_ERR_SHAPE;
  if (n == 0) return PP_OK;
  if (H < kh || W < kw) return PP_ERR_SHAPE;
  const int ph = (H - kh) / kh + 1, pw = (W - kw) / kw + 1;
  const long total = (long)n * ph * pw * (C / 4);
  k_pool_depthwise<__half><<<pp_blocks(total, 256), 256, 0, stream>>>((const __half*)x, ld_x, w_taps, bias, (__half*)out, n, H, W, C,
                                                                     kh, kw, ph, pw);
  PP_LAUNCH_CHECK();
  return PP_OK;
}

// residual add + LayerNorm of TemporalSparseTransformer.forward (sparse_transformer.py:322-334): x_out = x + delta,
// y = LN(x_out)*gamma + beta in one pass (one warp per token row, statistics two-pass in registers).  delta == NULL:
// plain LayerNorm (x_out not written).
// TD / TY = __half: fp16 delta (fc2's fp16 output) and / or fp16 y (the operand of the next half-operand Linear layers); the
// residual stream x / x_out, the statistics and the arithmetic stay fp32, y is rounded once on the store.
template <int NV, typename TD, typename TY>
__global__ void __launch_bounds__(256) k_add_layernorm(const float* __restrict__ x, const TD* __restrict__ delta,
    const float* __restrict__ gamma, const float* __restrict__ beta, float* __restrict__ x_out, TY* __restrict__ y, long rows,
    float eps) {
  constexpr int C = NV * 128;
  const long row = (long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  float4 v[NV];
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const long off = row * C + (k * 32 + lane) * 4;
    v[k] = *reinterpret_cast<const float4*>(x + off);
    if (delta != nullptr) {
      const float4 d = pp_ld4(delta + off);
      v[k].x += d.x; v[k].y += d.y; v[k].z += d.z; v[k].w += d.w;
      *reinterpret_cast<float4*>(x_out + off) = v[k];
    }
    s += (v[k].x + v[k].y) + (v[k].z + v[k].w);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s * (1.0f / C);
  float q = 0.f;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const float a = v[k].x - mean, b = v[k].y - mean, c = v[k].z - mean, d = v[k].w - mean;
    q += (a * a + b * b) + (c * c + d * d);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = 1.0f / sqrtf(q * (1.0f / C) + eps);
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int ci = (k * 32 + lane) * 4;
    const float4 g = *reinterpret_cast<const float4*>(gamma + ci), b = *reinterpret_cast<const float4*>(beta + ci);
    float4 o;
    o.x = (v[k].x - mean) * rstd * g.x + b.x; o.y = (v[k].y - mean) * rstd * g.y + b.y;
    o.z = (v[k].z - mean) * rstd * g.z + b.z; o.w = (v[k].w - mean) * rstd * g.w + b.w;
    pp_st4(y + row * C + ci, o);
  }
}
template <typename TD, typename TY>
static int pp_add_layernorm_launch(const float* x, const TD* delta, const float* gamma, const float* beta, float* x_out, TY* y,
                                   long rows, int C, float eps, cudaStream_t stream) {
  const unsigned grid = (unsigned)((rows + 7) / 8);
  switch (C) {
    case 128: k_add_layernorm<1, TD, TY><<<grid, 256, 0, stream>>>(x, delta, gamma, beta, x_out, y, rows, eps); break;
    case 256: k_add_layernorm<2, TD, TY><<<grid, 256, 0, stream>>>(x, delta, gamma, beta, x_out, y, rows, eps); break;
    case 512: k_add_layernorm<4, TD, TY><<<grid, 256, 0, stream>>>(x, delta, gamma, beta, x_out, y, rows, eps); break;
    case 1024: k_add_layernorm<8, TD, TY><<<grid, 256, 0, stream>>>(x, delta, gamma, beta, x_out, y, rows, eps); break;
    default: return PP_ERR_SHAPE;
  }
  PP_LAUNCH_CHECK();
  return PP_OK;
}
// the same with fp16 (delta_f16 != 0) or fp32 delta and fp16 (y_f16 != 0) or fp32 y; x / x_out stay fp32
extern "C" int pp_add_layernorm_f16(const float* x, const void* delta, int delta_f16, const float* gamma, const float* beta,
                                    float* x_out, void* y, int y_f16, long rows, int C, float eps, cudaStream_t stream) {
  if (((uintptr_t)x & 15) || ((uintptr_t)delta & 15) || ((uintptr_t)gamma & 15) || ((uintptr_t)beta & 15) ||
      ((uintptr_t)x_out & 15) || ((uintptr_t)y & 15)) return PP_ERR_ALIGN;
  if (rows < 0 || (delta != nullptr && x_out == nullptr)) return PP_ERR_SHAPE;
  if (rows == 0) return PP_OK;
  if (delta_f16 && y_f16) return pp_add_layernorm_launch(x, (const __half*)delta, gamma, beta, x_out, (__half*)y, rows, C, eps, stream);
  if (delta_f16) return pp_add_layernorm_launch(x, (const __half*)delta, gamma, beta, x_out, (float*)y, rows, C, eps, stream);
  if (y_f16) return pp_add_layernorm_launch(x, (const float*)delta, gamma, beta, x_out, (__half*)y, rows, C, eps, stream);
  return pp_add_layernorm_launch(x, (const float*)delta, gamma, beta, x_out, (float*)y, rows, C, eps, stream);
}
extern "C" int pp_add_layernorm(const float* x, const float* delta, const float* gamma, const float* beta, float* x_out, float* y,
                                long rows, int C, float eps, cudaStream_t stream) {
  return pp_add_layernorm_f16(x, delta, 0, gamma, beta, x_out, y, 0, rows, C, eps, stream);
}

// ================================================================ mask preparation
__global__ void __launch_bounds__(256) k_mask_dilate(const uint8_t* __restrict__ src, float* __restrict__ dst, int T, int H,
                                                     int W, int iterations) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const long HW = (long)H * W;
  if (i >= (long)T * HW) return;
  const long f = i / HW; const int r = (int)(i - f * HW); const int y = r / W, x = r - y * W;
  dst[i] = pp_mask_dilate_pixel(src + f * HW, H, W, y, x, iterations);
}
// replaces the per-frame scipy.ndimage.binary_dilation + to_tensors of read_mask (inference_propainter.py:93-107, :265-266)
extern "C" int pp_mask_dilate(const uint8_t* src, float* dst, int T, int H, int W, int iterations, cudaStream_t stream) {
  if (iterations < 0 || iterations > 64) return PP_ERR_SHAPE;
  k_mask_dilate<<<pp_blocks((long)T * H * W, 256), 256, 0, stream>>>(src, dst, T, H, W, iterations);
  PP_LAUNCH_CHECK();
  return PP_OK;
}

// ================================================================ frame conversion + compositing
__global__ void __launch_bounds__(256) k_u8_to_frames(const uint8_t* __restrict__ src, float* __restrict__ dst, int T,
                                                      int H, int W) {
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;      // over T*3*H*W (planar output order)
  long HW = (long)H * W;
  if (i >= (long)T * 3 * HW) return;
  long f = i / (3 * HW); long r = i - f * 3 * HW; int c = (int)(r / HW); long p = r - (long)c * HW;
  dst[i] = pp_u8_frame(src[(f * HW + p) * 3 + c]);
}
// replaces to_tensors()(frames)*2-1 (core/utils.py:130-170, inference_propainter.py:264)
extern "C" int pp_u8_to_frames(const uint8_t* src, float* dst, int T, int H, int W, cudaStream_t stream) {
  long n = (long)T * 3 * H * W;
  k_u8_to_frames<<<pp_blocks(n, 256), 256, 0, stream>>>(src, dst, T, H, W);
  PP_LAUNCH_CHECK();
  return PP_OK;
}

__global__ void __launch_bounds__(256) k_composite(const float* __restrict__ pred, const float* __restrict__ masks,
    const uint8_t* __restrict__ ori, uint8_t* __restrict__ comp, PPWindowIds ids, int H, int W) {
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;      // over n*H*W*3 (HWC order of the uint8 output)
  long HW = (long)H * W;
  if (i >= (long)ids.n * HW * 3) return;
  int k = (int)(i / (HW * 3)); long r = i - (long)k * HW * 3; long p = r / 3; int c = (int)(r - p * 3);
  int idx = ids.frame[k];
  long o = ((long)idx * HW + p) * 3 + c;
  comp[o] = pp_composite(pred[((long)k * 3 + c) * HW + p], masks[(long)idx * HW + p], ori[o], comp[o], ids.first[k]);
}
// replaces the numpy compositing / blending of inference_propainter.py:437-450 (no device->host sync)
extern "C" int pp_composite_blend_u8(const float* pred, const float* masks, const uint8_t* ori, uint8_t* comp,
                                     const PPWindowIds* ids, int H, int W, cudaStream_t stream) {
  if (ids->n < 1 || ids->n > PP_MAX_WINDOW) return PP_ERR_SHAPE;
  long n = (long)ids->n * H * W * 3;
  k_composite<<<pp_blocks(n, 256), 256, 0, stream>>>(pred, masks, ori, comp, *ids, H, W);
  PP_LAUNCH_CHECK();
  return PP_OK;
}

__global__ void __launch_bounds__(256) k_composite_f32(const float* __restrict__ pred, const float* __restrict__ masks,
    const uint8_t* __restrict__ ori, float* __restrict__ comp, PPWindowIds ids, int H, int W) {
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;      // over n*H*W*3 (HWC order of the float32 clip buffer)
  long HW = (long)H * W;
  if (i >= (long)ids.n * HW * 3) return;
  int k = (int)(i / (HW * 3)); long r = i - (long)k * HW * 3; long p = r / 3; int c = (int)(r - p * 3);
  int idx = ids.frame[k];
  long o = ((long)idx * HW + p) * 3 + c;
  comp[o] = pp_composite_f32(pred[((long)k * 3 + c) * HW + p], masks[(long)idx * HW + p], ori[o], comp[o], ids.first[k]);
}
// the float-valued compositing / blending of scripts/evaluate_propainter.py:166-179 (the evaluation protocol)
extern "C" int pp_composite_blend_f32(const float* pred, const float* masks, const uint8_t* ori, float* comp,
                                      const PPWindowIds* ids, int H, int W, cudaStream_t stream) {
  if (ids->n < 1 || ids->n > PP_MAX_WINDOW) return PP_ERR_SHAPE;
  long n = (long)ids->n * H * W * 3;
  k_composite_f32<<<pp_blocks(n, 256), 256, 0, stream>>>(pred, masks, ori, comp, *ids, H, W);
  PP_LAUNCH_CHECK();
  return PP_OK;
}

// ================================================================ video outpainting + masked preview
// One thread per canvas pixel: its 3 canvas bytes and its value in both masks.  64-bit offsets (a 3840x2160 canvas
// holds 8.3 M pixels per frame).
__global__ void __launch_bounds__(256) k_extrapolate_u8(const uint8_t* __restrict__ src, uint8_t* __restrict__ canvas,
    float* __restrict__ flow_masks, float* __restrict__ masks_dilated, int T, int h, int w, int H, int W, int top,
    int left, int rim_h, int rim_w) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;  // over T*H*W
  const long HW = (long)H * W;
  if (i >= (long)T * HW) return;
  const long f = i / HW; const long p = i - f * HW; const int y = (int)(p / W), x = (int)(p - (long)y * W);
  const long s = pp_outpaint_src(y, x, top, left, h, w);
  uint8_t r = 0, g = 0, b = 0;
  if (s >= 0) {
    const uint8_t* sp = src + (f * h * w + s) * 3;
    r = sp[0]; g = sp[1]; b = sp[2];
  }
  uint8_t* cp = canvas + i * 3;
  cp[0] = r; cp[1] = g; cp[2] = b;
  flow_masks[i] = pp_outpaint_mask(y, x, top, left, h, w, rim_h, rim_w);
  masks_dilated[i] = pp_outpaint_mask(y, x, top, left, h, w, 0, 0);
}
// replaces extrapolation (inference_propainter.py:117-156) + to_tensors of its masks (:265-266): uint8 frames
// [T][h][w][3] -> zero-bordered canvas [T][H][W][3] and float {0,1} flow / dilated masks [T][1][H][W]
extern "C" int pp_extrapolate_u8(const uint8_t* src, uint8_t* canvas, float* flow_masks, float* masks_dilated, int T, int h,
                                 int w, int H, int W, int top, int left, int rim_h, int rim_w, cudaStream_t stream) {
  if (T < 1 || h < 1 || w < 1 || top < 0 || left < 0 || rim_h < 0 || rim_w < 0) return PP_ERR_SHAPE;
  if ((long)top + h > H || (long)left + w > W) return PP_ERR_SHAPE;
  const long n = (long)T * H * W;
  k_extrapolate_u8<<<pp_blocks(n, 256), 256, 0, stream>>>(src, canvas, flow_masks, masks_dilated, T, h, w, H, W, top, left,
                                                          rim_h, rim_w);
  PP_LAUNCH_CHECK();
  return PP_OK;
}

__global__ void __launch_bounds__(256) k_mask_overlay_u8(const uint8_t* __restrict__ frames, const float* __restrict__ masks,
                                                         uint8_t* __restrict__ out, int T, int H, int W) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;  // over T*H*W*3 (HWC order of the uint8 frames)
  const long HW = (long)H * W;
  if (i >= (long)T * HW * 3) return;
  const long p = i / 3; const int c = (int)(i - p * 3);
  out[i] = pp_mask_overlay(frames[i], masks[p], c);
}
// replaces the masked_frame_for_save loop of inference_propainter.py:250-261 (green overlay, alpha 0.6): frames uint8
// [T][H][W][3] + masks [T][1][H][W] -> preview uint8 [T][H][W][3]
extern "C" int pp_mask_overlay_u8(const uint8_t* frames, const float* masks, uint8_t* out, int T, int H, int W,
                                  cudaStream_t stream) {
  if (T < 1 || H < 1 || W < 1) return PP_ERR_SHAPE;
  const long n = (long)T * H * W * 3;
  k_mask_overlay_u8<<<pp_blocks(n, 256), 256, 0, stream>>>(frames, masks, out, T, H, W);
  PP_LAUNCH_CHECK();
  return PP_OK;
}

// ================================================================ optical-flow colour coding
// Planar flow [N][2][H][W] float32 -> uint8 [N][H][W][3].  Two HBM-bound passes: the group maxima of the (clipped)
// radius (8 B read per pixel), then one thread per pixel (8 B read, 3 B written).  64-bit offsets: a 4K clip's output
// passes 2^31 bytes.
__global__ void __launch_bounds__(256) k_flow_maxrad(const float* __restrict__ flow, float* __restrict__ maxima, long HW,
                                                     int per_frame, int has_clip, float clip_flow) {
  const int n = blockIdx.y;
  const float* u = flow + (long)n * 2 * HW;
  const float* v = u + HW;
  float m = 0.0f;
  for (long p = (long)blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += (long)gridDim.x * blockDim.x) {
    float a = __ldg(u + p), b = __ldg(v + p);
    if (has_clip) { a = pp_flow_clip(a, clip_flow); b = pp_flow_clip(b, clip_flow); }
    m = fmaxf(m, pp_flow_rad(a, b));
  }
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  __shared__ float red[8];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < 8; ++i) m = fmaxf(m, red[i]);
    // a non-negative float orders like its bit pattern, so the integer max is the float max, in any order
    atomicMax((int*)(maxima + (per_frame ? n : 0)), __float_as_int(m));
  }
}
// the per-frame rad_max of flow_viz.py:127-128 (per_frame = 1, maxima[N]) or the batch max_norm of flow_viz_pt.py:29
// (per_frame = 0, maxima[1]); clears the maxima on the stream first
extern "C" int pp_flow_maxrad(const float* flow, float* maxima, int N, int H, int W, int per_frame, int has_clip,
                              float clip_flow, cudaStream_t stream) {
  if (N < 1 || N > 65535 || H < 1 || W < 1) return PP_ERR_SHAPE;
  const long HW = (long)H * W;
  if (cudaMemsetAsync(maxima, 0, (per_frame ? N : 1) * sizeof(float), stream) != cudaSuccess) return PP_ERR_LAUNCH;
  const int bx = pp_blocks(HW, 256 * 8) < 512 ? pp_blocks(HW, 256 * 8) : 512;
  k_flow_maxrad<<<dim3(bx, N), 256, 0, stream>>>(flow, maxima, HW, per_frame, has_clip, clip_flow);
  PP_LAUNCH_CHECK();
  return PP_OK;
}

__global__ void __launch_bounds__(256) k_flow_to_image_u8(const float* __restrict__ flow, const float* __restrict__ maxima,
                                                          uint8_t* __restrict__ out, int N, long HW, int variant,
                                                          int has_clip, float clip_flow, int bgr) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;  // over N*H*W
  if (i >= (long)N * HW) return;
  const long n = i / HW, p = i - n * HW;
  float u = __ldg(flow + n * 2 * HW + p), v = __ldg(flow + n * 2 * HW + HW + p);
  if (has_clip) { u = pp_flow_clip(u, clip_flow); v = pp_flow_clip(v, clip_flow); }
  uint8_t rgb[3];
  if (variant == PP_FLOWVIZ_FRAME) pp_flowviz_np(u, v, PP_ADD(__ldg(maxima + n), 1e-5f), bgr, rgb);
  else pp_flowviz_pt(u, v, PP_ADD(__ldg(maxima), 1.1920928955078125e-07f), bgr, rgb);
  uint8_t* o = out + i * 3;
  o[0] = rgb[0]; o[1] = rgb[1]; o[2] = rgb[2];
}
// replaces RAFT/utils/flow_viz.py::flow_to_image per frame (PP_FLOWVIZ_FRAME, maxima[N] from pp_flow_maxrad) and
// flow_viz_pt.py::flow_to_image over the batch (PP_FLOWVIZ_CLIP, maxima[1]), written pixel-major
extern "C" int pp_flow_to_image_u8(const float* flow, const float* maxima, uint8_t* out, int N, int H, int W, int variant,
                                   int has_clip, float clip_flow, int bgr, cudaStream_t stream) {
  if (N < 1 || H < 1 || W < 1) return PP_ERR_SHAPE;
  if (variant != PP_FLOWVIZ_FRAME && variant != PP_FLOWVIZ_CLIP) return PP_ERR_SHAPE;
  const long HW = (long)H * W, n = (long)N * HW;
  k_flow_to_image_u8<<<pp_blocks(n, 256), 256, 0, stream>>>(flow, maxima, out, N, HW, variant, has_clip, clip_flow, bgr != 0);
  PP_LAUNCH_CHECK();
  return PP_OK;
}
