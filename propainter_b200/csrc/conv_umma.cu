// Implicit-GEMM stride-1 "same" convolution on the warpgroup tensor-core instructions (wgmma, TMA, mbarrier), sm_90a.
//
// Replaces the cuDNN convolutions of the two recurrent propagation scans -- the offset nets and backbones of
// BidirectionalPropagation (model/propainter.py:42-50,86-96,121-175; model/recurrent_flow_completion.py:17-29,60-116) --
// and, as a 1x1 conv over the sampled columns, the GEMM of torchvision.ops.deform_conv2d (model/propainter.py:67-69,
// model/recurrent_flow_completion.py:42-44), together with everything that followed each of them as separate launches:
// bias add, LeakyReLU / ReLU / sigmoid / tanh, residual add, final ReLU, placement into a channel slice of a concat
// buffer, and the torch.cat that built the conv input (inputs are given as up to 4 channel segments).
//
//   out[p][n] = post( act( sum_{seg,c,dy,dx} W[n][seg,c,dy,dx] * x_seg[p + (dy,dx)][c]  + bias[n] + pre[p][n] ) + res[p][n] )
//
// One CTA = one M-pixel tile (BH x BW pixels of one map, M = BH*BW = 128 or 64) x BN output channels.
//   * A operand: no im2col.  For every 32-channel block TMA lands KW shifted copies of the (BH+KH-1) x BW halo box
//     (4-D tiled tensor map, SWIZZLE_128B; out-of-range rows/columns/channels are zero-filled by the TMA unit = the conv's
//     zero padding and the channel padding to a multiple of 32).  A box is [(BH+KH-1)*BW rows][128 B] = exactly the K-major
//     SWIZZLE_128B layout wgmma wants, and tap row dy is the same box read from row dy*BW on: a shared-memory descriptor
//     whose start address moves by dy*BW*128 B (a multiple of the 1 KB swizzle atom), so one copy feeds KH taps.
//   * B operand: packed weights [Cout][K], K index = ((blk*KH + dy)*KW + dx)*32 + c, loaded as [BN x 32] K-major boxes.
//   * D: fp32 registers of the consumer warpgroups (warpgroup w: pixels 64w .. 64w+63 of the tile, m64nBNk8 per k-step);
//     TF32 products (weights are pre-rounded to TF32 at pack time; activations written by this kernel are optionally rounded
//     on store so the next conv's operands are round-to-nearest TF32 too).
//   * fp16 instance (F16 = true, pp_conv2d_umma_f16): fp16 operands, m64nNk16 f32.f16.f16, fp32 accumulation.  A 128-byte
//     SW128 row holds 64 halves, so a "block" is 64 channels and every k-step / box / slot has the byte size of the TF32
//     instance: the pipeline is the same with half as many blocks.  The epilogue arithmetic is fp32 (bias / pre / res read as
//     fp32); it writes an fp32 `out`, an fp16 `out16` rounded to nearest once, or both from the same registers.
// Warp roles: warps 0-7 two consumer warpgroups (wgmma issue + epilogue; the second idles on 64-pixel tiles), warp 8 TMA
// producer.  Two rings: A (one slot per 32-channel block) and B (one slot per (block, dy) = KW taps), mbarrier full/empty
// pairs; a consumer releases a slot once the wgmma group that read it has retired.  Descriptor encodings: pp_umma.cuh.
#include <cuda.h>
#include <stdlib.h>
#include <type_traits>
#include "pp_elem.cuh"
#include "pp_mma.cuh"
#include "pp_umma.cuh"
#include "../../include/propainter_b200.h"

#define CV_THREADS 288
#define CV_MAX_A_SLOTS 6
#define CV_MAX_B_SLOTS 8
#define CV_SMEM_BUDGET (216 * 1024)

struct alignas(64) CVParams {
  CUtensorMap tmA[PP_CONV_MAX_SEG];
  CUtensorMap tmB;
  int seg_blocks[PP_CONV_MAX_SEG];   // pipeline blocks per segment (kgroup: groups of KW 32-channel blocks)
  int seg_kblocks[PP_CONV_MAX_SEG];  // real 32-channel blocks per segment (= K extent of the segment / 32 per tap)
  int nseg, nblk, kreal;      // nblk pipeline blocks; kreal real 32-channel blocks
  int n, H, W, KH, KW, BH, BW, BN, M;    // M = BH*BW = 128 or 64 (pixels per CTA, one m64 warpgroup tile per 64)
  int kgroup;                 // 1x1 convs: the `KW` loop walks `KW` consecutive 32-channel blocks (one pipeline stage = KW blocks)
  int tiles_x, tiles_y;
  int na, nb;                 // ring depths
  int ring_bytes;             // A ring + B ring
  int a_copy_bytes;           // (BH+KH-1)*BW*128
  int Cout;
  const float* bias; const float* pre; const float* res; float* out;
  int ld_pre, ld_res, ld_out;
  int act, post_relu, round_tf32;
  float slope;
  __half* out16; int ld_out16;        // fp16 instance only
};

__device__ __forceinline__ void cv_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void cv_tma4(uint32_t dst, const CUtensorMap* tm, int c, int x, int y, int n, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
               ::"r"(dst), "l"(tm), "r"(c), "r"(x), "r"(y), "r"(n), "r"(bar) : "memory");
}
__device__ __forceinline__ void cv_tma2(uint32_t dst, const CUtensorMap* tm, int k, int n, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
               ::"r"(dst), "l"(tm), "r"(k), "r"(n), "r"(bar) : "memory");
}
template <int BN, bool F16>
__device__ __forceinline__ void cv_mma(float (&d)[BN / 2], uint64_t a, uint64_t b, int scale_d) {
  if constexpr (F16) {
    if constexpr (BN == 32) wg_mma_ss_n32_f16(d, a, b, scale_d);
    else if constexpr (BN == 64) wg_mma_ss_n64_f16(d, a, b, scale_d);
    else wg_mma_ss_n128_f16(d, a, b, scale_d);
  } else {
    if constexpr (BN == 32) wg_mma_ss_n32(d, a, b, scale_d);
    else if constexpr (BN == 64) wg_mma_ss_n64(d, a, b, scale_d);
    else wg_mma_ss_n128(d, a, b, scale_d);
  }
}

template <int BN, bool F16>
__global__ void __launch_bounds__(CV_THREADS, 1) k_conv_umma(const __grid_constant__ CVParams p) {
  constexpr int CB = F16 ? 64 : 32;                               // channels per 128-byte block
  extern __shared__ __align__(1024) uint8_t cv_raw[];
  uint8_t* base = cv_raw + ((1024u - (ua_smem(cv_raw) & 1023u)) & 1023u);
  const int a_slot_bytes = p.KW * p.a_copy_bytes;
  const int b_tap_bytes = BN * 128, b_slot_bytes = p.KW * b_tap_bytes;
  uint8_t* sA = base;
  uint8_t* sB = sA + p.na * a_slot_bytes;
  uint8_t* tail = base + p.ring_bytes;
  // barriers: [0,na) a_full  [8,8+na) a_empty  [16,16+nb) b_full  [24,24+nb) b_empty
  unsigned long long* bars = reinterpret_cast<unsigned long long*>(tail);
  const uint32_t b0 = ua_smem(bars);
  auto bar = [&](int i) { return b0 + 8u * (uint32_t)i; };
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int tile = blockIdx.x, n0 = blockIdx.y * BN;
  const int tpi = p.tiles_x * p.tiles_y;
  const int img = tile / tpi, trem = tile - img * tpi;
  const int y0 = (trem / p.tiles_x) * p.BH, x0 = (trem % p.tiles_x) * p.BW;
  const int nwg = p.M >> 6;                                       // consumer warpgroups with pixels to compute

  if (tid == 0) {
    for (int i = 0; i < p.na; ++i) { ua_bar_init(bar(i), 1); ua_bar_init(bar(8 + i), 4 * nwg); }
    for (int i = 0; i < p.nb; ++i) { ua_bar_init(bar(16 + i), 1); ua_bar_init(bar(24 + i), 4 * nwg); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  // Programmatic dependent launch: everything above (barrier init, parameter / descriptor fetch) touches no global memory
  // and overlaps the tail of the previous kernel in the stream; the next kernel may start its own prologue now.  Global
  // reads and writes below wait for the previous grid to have completed and flushed.
  asm volatile("griddepcontrol.launch_dependents;");
  asm volatile("griddepcontrol.wait;" ::: "memory");

  if (warp == 8) {
    // ================================================= TMA producer: all 32 lanes stay converged, one elected lane issues
    int seg = 0, cb = 0, kbase = 0;                                  // kbase: first real k-block of the current segment
    for (int blk = 0; blk < p.nblk; ++blk) {
      const int sa = blk % p.na;
      ua_bar_wait(bar(8 + sa), ((blk / p.na) & 1) ^ 1);
      if (ua_elect()) {
        cv_expect_tx(bar(sa), (uint32_t)a_slot_bytes);
        for (int dx = 0; dx < p.KW; ++dx)
          if (p.kgroup)
            cv_tma4(ua_smem(sA + sa * a_slot_bytes + dx * p.a_copy_bytes), &p.tmA[seg], (cb * p.KW + dx) * CB, x0, y0, img, bar(sa));
          else
            cv_tma4(ua_smem(sA + sa * a_slot_bytes + dx * p.a_copy_bytes), &p.tmA[seg], cb * CB, x0 + dx - p.KW / 2,
                    y0 - p.KH / 2, img, bar(sa));
      }
      __syncwarp();
      for (int dy = 0; dy < p.KH; ++dy) {
        const int ib = blk * p.KH + dy, sb = ib % p.nb;
        ua_bar_wait(bar(24 + sb), ((ib / p.nb) & 1) ^ 1);
        if (ua_elect()) {
          cv_expect_tx(bar(16 + sb), (uint32_t)b_slot_bytes);
          for (int dx = 0; dx < p.KW; ++dx)
            cv_tma2(ua_smem(sB + sb * b_slot_bytes + dx * b_tap_bytes), &p.tmB,
                    (p.kgroup ? kbase + cb * p.KW + dx : ib * p.KW + dx) * CB, n0, bar(16 + sb));
        }
        __syncwarp();
      }
      if (++cb == p.seg_blocks[seg]) { cb = 0; kbase += p.seg_kblocks[seg]; ++seg; }
    }
    return;
  }
  const int wg = warp >> 2;
  if (wg >= nwg) return;                                          // 64-pixel tiles: the second warpgroup has no rows
  // ================================================= consumer warpgroup: wgmma issue, then the epilogue from registers
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  // Each (block, dy) step is one wgmma group.  With two or more slots in both rings a slot is released one group late
  // (wait_group 1), so the next group's wgmmas are issued before the previous ones retire; a one-slot ring is released at
  // once (the producer could otherwise not fill the slot the next group waits for).
  const bool defer = p.na >= 2 && p.nb >= 2;
  int prev_sa = -1, prev_sb = -1;
  const uint32_t row_off = (uint32_t)wg * 64 * 128;               // this warpgroup's 64 pixel rows inside every A copy
  for (int blk = 0; blk < p.nblk; ++blk) {
    const int sa = blk % p.na;
    ua_bar_wait(bar(sa), (blk / p.na) & 1);
    const uint64_t a_desc0 = ua_desc(ua_smem(sA + sa * a_slot_bytes) + row_off);
    for (int dy = 0; dy < p.KH; ++dy) {
      const int ib = blk * p.KH + dy, sb = ib % p.nb;
      ua_bar_wait(bar(16 + sb), (ib / p.nb) & 1);
      const uint64_t b_desc0 = ua_desc(ua_smem(sB + sb * b_slot_bytes));
      // descriptors advance in their 16-byte address field: +2 per 32-byte k-step (8 floats / 16 halves), + tap / row offsets >> 4
      uint64_t ad = a_desc0 + (uint64_t)((dy * p.BW * 128) >> 4), bd = b_desc0;
      wg_fence();
      for (int dx = 0; dx < p.KW; ++dx) {
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) cv_mma<BN, F16>(acc, ad + 2 * ks, bd + 2 * ks, 1);
        ad += (uint64_t)(p.a_copy_bytes >> 4); bd += (uint64_t)(b_tap_bytes >> 4);
      }
      wg_commit();
      const int last_a = dy == p.KH - 1 ? sa : -1;
      if (defer) {
        wg_wait<1>();
        if (prev_sb >= 0 && lane == 0) {
          ua_bar_arrive(bar(24 + prev_sb));
          if (prev_sa >= 0) ua_bar_arrive(bar(8 + prev_sa));
        }
        prev_sb = sb; prev_sa = last_a;
      } else {
        wg_wait<0>();
        if (lane == 0) {
          ua_bar_arrive(bar(24 + sb));
          if (last_a >= 0) ua_bar_arrive(bar(8 + last_a));
        }
      }
    }
  }
  wg_wait<0>();
  wg_pin(acc);

  // ================================================= epilogue straight from the accumulator registers: each thread owns
  // two pixel rows x (2 adjacent channels per 8-channel group); a warp's float2 accesses cover whole 32-byte sectors.
  const int g = lane >> 2, t = lane & 3;
  const float* __restrict__ bias = p.bias;
  const int post_relu = p.post_relu, round_tf32 = p.round_tf32;
  const float slope = p.slope;
  const float* prow[2]; const float* rrow[2]; float* orow[2]; __half* hrow[2];
  bool ok[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = wg * 64 + (warp & 3) * 16 + g + 8 * h;
    const int y = y0 + r / p.BW, x = x0 + r % p.BW;
    ok[h] = y < p.H && x < p.W;
    const long pix = ok[h] ? ((long)img * p.H + y) * p.W + x : 0;
    if constexpr (F16) {
      orow[h] = p.out ? p.out + pix * p.ld_out + n0 + 2 * t : nullptr;
      hrow[h] = p.out16 ? p.out16 + pix * p.ld_out16 + n0 + 2 * t : nullptr;
    } else {
      orow[h] = p.out + pix * p.ld_out + n0 + 2 * t;
    }
    prow[h] = p.pre ? p.pre + pix * p.ld_pre + n0 + 2 * t : nullptr;
    rrow[h] = p.res ? p.res + pix * p.ld_res + n0 + 2 * t : nullptr;
  }
  // the activation is selected once (warp-uniform branch), not per element: with the switch inside the element loop the
  // exp / tanh paths would be inlined once per element
  auto finish = [&](auto actf) {
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int n = n0 + 8 * j + 2 * t;
      if (n >= p.Cout) continue;                                  // Cout % 4 == 0: n < Cout implies n + 1 < Cout
      const float2 bv = bias ? __ldg(reinterpret_cast<const float2*>(bias + n)) : make_float2(0.f, 0.f);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (!ok[h]) continue;
        const float2 pv = prow[h] ? *reinterpret_cast<const float2*>(prow[h] + 8 * j) : make_float2(0.f, 0.f);
        const float2 rv = rrow[h] ? *reinterpret_cast<const float2*>(rrow[h] + 8 * j) : make_float2(0.f, 0.f);
        float2 a;
        a.x = actf(acc[4 * j + 2 * h] + (bv.x + pv.x)) + rv.x;
        a.y = actf(acc[4 * j + 2 * h + 1] + (bv.y + pv.y)) + rv.y;
        if (post_relu) { a.x = fmaxf(a.x, 0.f); a.y = fmaxf(a.y, 0.f); }
        if constexpr (F16) {
          if (orow[h]) *reinterpret_cast<float2*>(orow[h] + 8 * j) = a;
          if (hrow[h]) *reinterpret_cast<__half2*>(hrow[h] + 8 * j) = __float22half2_rn(a);
        } else {
          if (round_tf32) { a.x = __uint_as_float(pp_tf32(a.x)); a.y = __uint_as_float(pp_tf32(a.y)); }
          *reinterpret_cast<float2*>(orow[h] + 8 * j) = a;
        }
      }
    }
  };
  const int act = p.act;
  if (act == 0) finish([](float v) { return v; });
  else if (act == 1) finish([](float v) { return fmaxf(v, 0.f); });
  else if (act == 2) finish([slope](float v) { return v > 0.f ? v : v * slope; });
  else if (act == 3) finish([](float v) { return 1.0f / (1.0f + expf(-v)); });
  else finish([](float v) { return tanhf(v); });
}

// launch with the programmatic-stream-serialization attribute (PDL); PP_PDL=0 in the environment falls back to plain launches
static bool cv_pdl_enabled() {
  static int on = -1;
  if (on < 0) { const char* e = getenv("PP_PDL"); on = (e && e[0] == '0') ? 0 : 1; }
  return on != 0;
}
template <typename... KArgs, typename... Args>
static cudaError_t cv_launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = cv_pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

typedef CUresult (*PFN_cvEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                      const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                      CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_cvEncodeTiled cv_encoder() {
  static PFN_cvEncodeTiled cached = nullptr;      // idempotent lookup (same pointer every time): benign if raced
  if (cached) return cached;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess ||
      qres != cudaDriverEntryPointSuccess)
    return nullptr;
  cached = (PFN_cvEncodeTiled)fn;
  return cached;
}

// tile / ring plan shared by the launcher and pp_conv2d_umma_plan (so callers and tests can see what will run).  f16: blocks of
// 64 channels (128 B of halves); the boxes, slots and per-k-step costs are those of the TF32 instance.
static int cv_plan(const PPConvParams* q, CVParams* p, int* smem_bytes, bool f16) {
  const int cb = f16 ? 64 : 32, lda = f16 ? 8 : 4;               // channels per block; ld granule of a 16-byte row stride
  if (q->nseg < 1 || q->nseg > PP_CONV_MAX_SEG || q->n < 1 || q->H < 1 || q->W < 1) return PP_ERR_SHAPE;
  if (q->KH < 1 || q->KW < 1 || q->KH > 7 || q->KW > 7 || !(q->KH & 1) || !(q->KW & 1)) return PP_ERR_SHAPE;
  if (q->Cout < 4 || q->Cout % 4) return PP_ERR_SHAPE;
  int nblk = 0, kblocks = 0;
  for (int s = 0; s < q->nseg; ++s) {
    if (q->seg[s].C < 1) return PP_ERR_SHAPE;
    if (q->seg[s].ld % lda || ((uintptr_t)q->seg[s].x & 15)) return PP_ERR_ALIGN;
    p->seg_kblocks[s] = (q->seg[s].C + cb - 1) / cb;
    kblocks += p->seg_kblocks[s];
  }
  // 1x1 convs (plain GEMMs over the channels): a pipeline stage of one 128-byte block holds only 4 wgmmas per warpgroup,
  // less work than the fixed cost of a stage (two barrier round trips, a wgmma group commit and wait).  Group 4 consecutive
  // blocks per stage (the tap loop walks channels instead of x-shifts).
  const int kv = (q->KH == 1 && q->KW == 1 && kblocks >= 8) ? 4 : 0;
  p->kgroup = kv ? 1 : 0;
  for (int s = 0; s < q->nseg; ++s) {
    p->seg_blocks[s] = kv ? (p->seg_kblocks[s] + kv - 1) / kv : p->seg_kblocks[s];
    nblk += p->seg_blocks[s];
  }
  if (q->ld_out % 4 || ((uintptr_t)q->out & 15) || ((uintptr_t)q->w_packed & 15)) return PP_ERR_ALIGN;
  if (q->bias && ((uintptr_t)q->bias & 15)) return PP_ERR_ALIGN;
  if (q->pre && (q->ld_pre % 4 || ((uintptr_t)q->pre & 15))) return PP_ERR_ALIGN;
  if (q->res && (q->ld_res % 4 || ((uintptr_t)q->res & 15))) return PP_ERR_ALIGN;
  p->nseg = q->nseg; p->nblk = nblk;
  p->n = q->n; p->H = q->H; p->W = q->W; p->KH = q->KH; p->KW = kv ? kv : q->KW;
  p->kreal = kblocks;
  // tile shape: (M/8) x 8 or (M/16) x 16 pixels, whichever wastes fewer padded pixels (ties: 8 columns)
  int bw = q->tile_w;
  if (bw != 8 && bw != 16) {
    const int mm = q->tile_m == 64 ? 64 : 128;
    const long a8 = (long)((q->W + 7) / 8) * ((q->H + mm / 8 - 1) / (mm / 8)), a16 = (long)((q->W + 15) / 16) * ((q->H + mm / 16 - 1) / (mm / 16));
    bw = a16 < a8 ? 16 : 8;
  }
  const int M = q->tile_m == 64 ? 64 : 128;                      // pixels per CTA = 64 per consumer warpgroup
  p->M = M;
  p->BW = bw; p->BH = M / bw;
  p->tiles_x = (q->W + p->BW - 1) / p->BW; p->tiles_y = (q->H + p->BH - 1) / p->BH;
  const long tiles = (long)p->tiles_x * p->tiles_y * q->n;
  if (tiles > 0x7fffffffL) return PP_ERR_SHAPE;
  // N tile.  Model of one k-step of 8 channels for the CTA's two warpgroups (m64nNk8 each, both operands in shared memory):
  // the tensor cores need ~N cycles (1024 TF32 FMA per cycle per SM) and shared memory delivers the 2 x 2 KB A slices plus
  // 2 x N x 32 B of B at 128 B per cycle, ~32 + N/2 cycles; the larger bounds the step.  An fp16 k-step (m64nNk16, 16
  // channels in the same 32 bytes) costs the same: twice the FMAs at twice the rate (2048 per cycle), the same bytes.  One CTA runs per SM (shared
  // memory), CTAs beyond one per SM run as further waves.  Pick the N that minimises waves x step cost; ties go to the
  // larger tile (fewer re-reads of A from L2).
  int bn = q->bn;
  if (bn != 32 && bn != 64 && bn != 128) {
    long best = -1;
    for (int cand = 128; cand >= 32; cand >>= 1) {
      const long ctas = tiles * ((q->Cout + cand - 1) / cand), waves = (ctas + PP_NUM_SMS - 1) / PP_NUM_SMS;
      const long cost = waves * (cand > 32 + cand / 2 ? cand : 32 + cand / 2);
      if (best < 0 || cost < best) { best = cost; bn = cand; }
    }
  }
  p->BN = bn;
  p->a_copy_bytes = (p->BH + p->KH - 1) * p->BW * 128;
  const int a_slot = p->KW * p->a_copy_bytes, b_slot = p->KW * bn * 128;
  int na = (q->KH * q->KW == 1 && !p->kgroup) ? 4 : 2;
  if (na > nblk) na = nblk;
  if (na * a_slot + b_slot > CV_SMEM_BUDGET) na = 1;
  if (na * a_slot + b_slot > CV_SMEM_BUDGET) return PP_ERR_SHAPE;
  int nb = (CV_SMEM_BUDGET - na * a_slot) / b_slot;
  if (nb > CV_MAX_B_SLOTS) nb = CV_MAX_B_SLOTS;
  if (nb > nblk * q->KH) nb = nblk * q->KH;
  // spend what is left on more A slots (1x1 convs: deeper prefetch of the only large operand)
  while (na < CV_MAX_A_SLOTS && na < nblk && (na + 1) * a_slot + nb * b_slot <= CV_SMEM_BUDGET) ++na;
  p->na = na; p->nb = nb;
  p->ring_bytes = na * a_slot + nb * b_slot;
  *smem_bytes = p->ring_bytes + 512 + 1024;
  p->Cout = q->Cout;
  p->bias = q->bias; p->pre = q->pre; p->res = q->res; p->out = q->out;
  p->ld_pre = q->ld_pre; p->ld_res = q->ld_res; p->ld_out = q->ld_out;
  p->act = q->act; p->post_relu = q->post_relu; p->round_tf32 = q->round_tf32; p->slope = q->slope;
  p->out16 = nullptr; p->ld_out16 = 0;
  return PP_OK;
}

static int cv_plan_report(const PPConvParams* q, bool f16, int* tile_h, int* tile_w, int* bn, int* ctas, int* smem_bytes) {
  CVParams p;
  int smem = 0;
  const int rc = cv_plan(q, &p, &smem, f16);
  if (rc != PP_OK) return rc;
  if (tile_h) *tile_h = p.BH;
  if (tile_w) *tile_w = p.BW;
  if (bn) *bn = p.BN;
  if (ctas) *ctas = p.tiles_x * p.tiles_y * p.n * ((p.Cout + p.BN - 1) / p.BN);
  if (smem_bytes) *smem_bytes = smem;
  return PP_OK;
}

extern "C" int pp_conv2d_umma_plan(const PPConvParams* q, int* tile_h, int* tile_w, int* bn, int* ctas, int* smem_bytes) {
  return cv_plan_report(q, false, tile_h, tile_w, bn, ctas, smem_bytes);
}

extern "C" int pp_conv2d_umma_plan_f16(const PPConvParams* q, int* tile_h, int* tile_w, int* bn, int* ctas, int* smem_bytes) {
  return cv_plan_report(q, true, tile_h, tile_w, bn, ctas, smem_bytes);
}

static int cv_run(const PPConvParams* q, __half* out16, int ld_out16, bool f16, cudaStream_t stream) {
  CVParams p;
  int smem = 0;
  int rc = cv_plan(q, &p, &smem, f16);
  if (rc != PP_OK) return rc;
  if (f16) {
    if (!q->out && !out16) return PP_ERR_SHAPE;
    if (out16 && (ld_out16 % 8 || ((uintptr_t)out16 & 15))) return PP_ERR_ALIGN;
    p.out16 = out16; p.ld_out16 = ld_out16;
  } else if (!q->out) {
    return PP_ERR_SHAPE;
  }
  const int cb = f16 ? 64 : 32, esz = f16 ? 2 : 4;
  const CUtensorMapDataType dt = f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  PFN_cvEncodeTiled enc = cv_encoder();
  if (!enc) return PP_ERR_LAUNCH;
  for (int s = 0; s < q->nseg; ++s) {
    const cuuint64_t ld = (cuuint64_t)q->seg[s].ld;
    cuuint64_t dims[4] = {(cuuint64_t)q->seg[s].C, (cuuint64_t)q->W, (cuuint64_t)q->H, (cuuint64_t)q->n};
    cuuint64_t strides[3] = {ld * esz, ld * esz * (cuuint64_t)q->W, ld * esz * (cuuint64_t)q->W * (cuuint64_t)q->H};
    cuuint32_t box[4] = {(cuuint32_t)cb, (cuuint32_t)p.BW, (cuuint32_t)(p.BH + p.KH - 1), 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    if (enc(&p.tmA[s], dt, 4, (void*)q->seg[s].x, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return PP_ERR_LAUNCH;
  }
  {
    const cuuint64_t ktot = (cuuint64_t)p.kreal * q->KH * q->KW * cb;
    cuuint64_t dims[2] = {ktot, (cuuint64_t)q->Cout};
    cuuint64_t strides[1] = {ktot * esz};
    cuuint32_t box[2] = {(cuuint32_t)cb, (cuuint32_t)p.BN};
    cuuint32_t estr[2] = {1, 1};
    if (enc(&p.tmB, dt, 2, (void*)q->w_packed, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return PP_ERR_LAUNCH;
  }
  void (*kernel)(const CVParams) = f16 ? (p.BN == 32 ? k_conv_umma<32, true> : p.BN == 64 ? k_conv_umma<64, true> : k_conv_umma<128, true>)
                                        : (p.BN == 32 ? k_conv_umma<32, false> : p.BN == 64 ? k_conv_umma<64, false> : k_conv_umma<128, false>);
  if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, CV_SMEM_BUDGET + 2048) != cudaSuccess)
    return PP_ERR_LAUNCH;
  dim3 grid((unsigned)(p.tiles_x * p.tiles_y * p.n), (unsigned)((p.Cout + p.BN - 1) / p.BN));
  if (cv_launch(kernel, grid, dim3(CV_THREADS), (size_t)smem, stream, p) != cudaSuccess) return PP_ERR_LAUNCH;
  return cudaPeekAtLastError() == cudaSuccess ? PP_OK : PP_ERR_LAUNCH;
}

extern "C" int pp_conv2d_umma(const PPConvParams* q, cudaStream_t stream) { return cv_run(q, nullptr, 0, false, stream); }

extern "C" int pp_conv2d_umma_f16(const PPConvParams* q, void* out16, int ld_out16, cudaStream_t stream) {
  return cv_run(q, static_cast<__half*>(out16), ld_out16, true, stream);
}

// ================================================================ deformable sampling -> columns
// First half of torchvision.ops.deform_conv2d (3x3, stride 1, pad 1, 16 offset groups) as called from
// DeformableAlignment.forward / SecondOrderDeformableAlignment.forward (model/propainter.py:57-69,
// model/recurrent_flow_completion.py:31-44): decode the raw conv_offset output (max_res*tanh offsets (+ flow.flip),
// sigmoid modulation), sample x bilinearly at the 9 x 16 positions of every pixel and write the modulated samples as
// columns cols[p][k*Cin + c] (rounded to TF32: they are the A operand of the GEMM that follows = pp_conv2d_umma with a
// 1x1 kernel over `cols`; the fp16 instance rounds them to nearest fp16 instead, for pp_conv2d_umma_f16).  One warp per pixel: lane <-> (group, half of the group's channels), so per tap a warp reads
// 16 positions x 4 corners x 32/64 B and writes one contiguous Cin*4-byte run.
template <int CPL, typename TC>   // channels per lane: 4 (Cin = 128) or 8 (Cin = 256); column type float (TF32) or __half
__global__ void __launch_bounds__(256) k_deform_gather(const float* __restrict__ x, int ld_x, const float* __restrict__ x2, int ld_x2,
    const float* __restrict__ o, int ld_o,
    const float* __restrict__ obias, const float* __restrict__ flow, float max_res, TC* __restrict__ cols, long npix, int H, int W) {
  // One warp per pixel, lane <-> (offset group g, half of the group's channels).  The 27 offset-net outputs of (pixel, g)
  // are fetched up front, then the 9 taps run in batches of 3 with all 12 (24) corner loads of a batch in flight before
  // the first one is used: the kernel is latency-bound (two dependent memory round trips per tap), so what matters is
  // how many independent loads each warp keeps outstanding.
  asm volatile("griddepcontrol.launch_dependents;");
  asm volatile("griddepcontrol.wait;" ::: "memory");               // inputs come from the previous kernel in the stream (PDL)
  const long pix = (long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (pix >= npix) return;
  const int lane = threadIdx.x & 31, g = lane >> 1, half = lane & 1;
  const long HW = (long)H * W, img = pix / HW, pim = pix - img * HW;
  const int y = (int)(pim / W), xx = (int)(pim - (long)y * W);
  const float* op = o + pix * ld_o;
  float2 off[9]; float ml[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) { off[k] = *reinterpret_cast<const float2*>(op + g * 18 + 2 * k); ml[k] = op[288 + g * 9 + k]; }
  float fy = 0.f, fx = 0.f;
  if (flow) { fx = flow[2 * pix]; fy = flow[2 * pix + 1]; }
  if (obias) {
#pragma unroll
    for (int k = 0; k < 9; ++k) { off[k].x += obias[g * 18 + 2 * k]; off[k].y += obias[g * 18 + 2 * k + 1]; ml[k] += obias[288 + g * 9 + k]; }
  }
  constexpr int CIN = CPL * 32, NV = CPL / 4;
  const int c = g * (2 * CPL) + half * CPL;
  // x2 != NULL: the input channels are split over two maps of CIN/2 channels each (offset groups 0-7 | 8-15): the two
  // previous states of the second-order scan live in different slots of the history buffer (no torch.cat)
  const bool second = x2 != nullptr && c >= CIN / 2;
  if (second) { x = x2; ld_x = ld_x2; }
  const int cs = second ? c - CIN / 2 : c;
  const float* xi = x + img * HW * ld_x;
  TC* dst = cols + pix * (9L * CIN) + c;
#pragma unroll
  for (int kb = 0; kb < 9; kb += 3) {
    float wts[3][4];
    float4 v[3][4][NV];
#pragma unroll
    for (int u = 0; u < 3; ++u) {
      const int k = kb + u;
      PPDTap t;
      t.py = (float)(y - 1 + k / 3) + (max_res * tanhf(off[k].x) + fy);      // same association as pp_deform_tap (pp_elem.cuh)
      t.px = (float)(xx - 1 + k % 3) + (max_res * tanhf(off[k].y) + fx);
      t.m = 1.0f / (1.0f + expf(-ml[k]));
      const PPDW d = pp_deform_weights(t, H, W);
      wts[u][0] = d.w00; wts[u][1] = d.w01; wts[u][2] = d.w10; wts[u][3] = d.w11;
      const float* p00 = xi + ((long)d.y0 * W + d.x0) * ld_x + cs;
      const float* q[4] = {p00, p00 + ld_x, p00 + (long)W * ld_x, p00 + (long)W * ld_x + ld_x};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float* a = wts[u][j] != 0.f ? q[j] : xi + cs;                // never dereference an out-of-image corner
#pragma unroll
        for (int i = 0; i < NV; ++i) v[u][j][i] = *reinterpret_cast<const float4*>(a + 4 * i);
      }
    }
#pragma unroll
    for (int u = 0; u < 3; ++u) {
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float w = wts[u][j];
          acc.x += v[u][j][i].x * w; acc.y += v[u][j][i].y * w; acc.z += v[u][j][i].z * w; acc.w += v[u][j][i].w * w;
        }
        if constexpr (std::is_same<TC, __half>::value) {
          const __half2 lo = __floats2half2_rn(acc.x, acc.y), hi = __floats2half2_rn(acc.z, acc.w);
          uint2 v;
          v.x = *reinterpret_cast<const uint32_t*>(&lo); v.y = *reinterpret_cast<const uint32_t*>(&hi);
          *reinterpret_cast<uint2*>(dst + (long)(kb + u) * CIN + 4 * i) = v;
        } else {
          *reinterpret_cast<float4*>(dst + (long)(kb + u) * CIN + 4 * i) =
              make_float4(__uint_as_float(pp_tf32(acc.x)), __uint_as_float(pp_tf32(acc.y)), __uint_as_float(pp_tf32(acc.z)), __uint_as_float(pp_tf32(acc.w)));
        }
      }
    }
  }
}

template <typename TC>
static int dg_run(const float* x, int ld_x, const float* x2, int ld_x2, const float* o, int ld_o, const float* o_bias, const float* flow,
                  float max_res, TC* cols, int n, int H, int W, int Cin, cudaStream_t stream) {
  if ((Cin != 128 && Cin != 256) || n < 1 || H < 1 || W < 1) return PP_ERR_SHAPE;
  if (ld_x % 4 || ld_o < 432 || ((uintptr_t)x & 15) || ((uintptr_t)cols & 15)) return PP_ERR_ALIGN;
  if (x2 && (ld_x2 % 4 || ((uintptr_t)x2 & 15))) return PP_ERR_ALIGN;
  if (ld_o % 2 || ((uintptr_t)o & 7)) return PP_ERR_ALIGN;           // (dy,dx) pairs are fetched as float2
  const long npix = (long)n * H * W;
  const long blocks = (npix + 7) / 8;
  if (blocks > 0x7fffffffL) return PP_ERR_SHAPE;
  cudaError_t e;
  if (Cin == 128) e = cv_launch(k_deform_gather<4, TC>, dim3((unsigned)blocks), dim3(256), 0, stream, x, ld_x, x2, ld_x2, o, ld_o, o_bias, flow, max_res, cols, npix, H, W);
  else e = cv_launch(k_deform_gather<8, TC>, dim3((unsigned)blocks), dim3(256), 0, stream, x, ld_x, x2, ld_x2, o, ld_o, o_bias, flow, max_res, cols, npix, H, W);
  if (e != cudaSuccess) return PP_ERR_LAUNCH;
  return cudaPeekAtLastError() == cudaSuccess ? PP_OK : PP_ERR_LAUNCH;
}

extern "C" int pp_deform_gather(const float* x, int ld_x, const float* x2, int ld_x2, const float* o, int ld_o, const float* o_bias,
                                const float* flow, float max_res, float* cols, int n, int H, int W, int Cin, cudaStream_t stream) {
  return dg_run(x, ld_x, x2, ld_x2, o, ld_o, o_bias, flow, max_res, cols, n, H, W, Cin, stream);
}

extern "C" int pp_deform_gather_f16(const float* x, int ld_x, const float* x2, int ld_x2, const float* o, int ld_o, const float* o_bias,
                                    const float* flow, float max_res, void* cols, int n, int H, int W, int Cin, cudaStream_t stream) {
  return dg_run(x, ld_x, x2, ld_x2, o, ld_o, o_bias, flow, max_res, static_cast<__half*>(cols), n, H, W, Cin, stream);
}
