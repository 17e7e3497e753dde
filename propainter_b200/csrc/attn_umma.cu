// Mask-guided sparse window attention on the warpgroup tensor-core instructions (wgmma), sm_90a.
//
// Replaces SparseWindowAttention.forward (model/modules/sparse_transformer.py:177-275) for *masked*
// windows: 128 query rows x 128 head dims per CTA, keys streamed in tiles of 64 (own + rolled tokens by
// table lookup, pooled tokens), flash-style online softmax.  Unmasked windows (45x45 per frame) stay on
// the small mma.sync kernel in mma_kernels.cu.
//
// S = Q K^T (wgmma m64n64k8 tf32, Q and K tiles K-major SWIZZLE_128B in smem), online softmax in registers, O += P V
// (m64n128k8, P from registers, V transposed into a K-major tile by the producers: TF32 wgmma operands are K-major).
// Warps 0-7: two consumer warpgroups (64 query rows each); warps 8-11: K/V producers.  Two stages, mbarrier pairs.
// P's accumulator fragment holds keys 2t, 2t+1 of each k8 step, the A fragment expects keys t, t+4: inside every group
// of 8 keys V^T column t holds key 2t and column t+4 key 2t+1, which is the same sum.
#include "pp_elem.cuh"
#include "pp_mma.cuh"
#include "pp_umma.cuh"
#include "../../include/propainter_b200.h"

#define UA_BM 128
#define UA_BN 64
#define UA_THREADS 384                             // 2 consumer warpgroups + 1 producer warpgroup
#define UA_Q_BYTES (UA_BM * 128 * 4)               // 64 KB: 4 k-blocks of [128 rows x 128 B]
#define UA_K_BYTES (UA_BN * 128 * 4)               // 32 KB: 4 k-blocks of [64 rows x 128 B]
#define UA_V_BYTES (128 * UA_BN * 4)               // 32 KB: 2 k-blocks of [128 rows x 128 B]  (V^T: rows = head dim)
#define UA_STAGE_BYTES (UA_K_BYTES + UA_V_BYTES)
#define UA_STAGES 2
#define UA_TAIL_BYTES 3072                         // barriers, token table (<= 224 ints at +256), key row pointers (+1152)
#define UA_SMEM_BYTES (UA_Q_BYTES + UA_STAGES * UA_STAGE_BYTES + UA_TAIL_BYTES + 1024)
static_assert(UA_SMEM_BYTES <= 227 * 1024, "the stages do not fit the 227 KB of shared memory");

// column of key `kk` (0..63) in the V^T tile: the renaming described above, inside each group of 8 keys
__device__ __forceinline__ int ua_vcol(int kk) { return (kk & ~7) | ((kk & 1) << 2) | ((kk >> 1) & 3); }

__global__ void __launch_bounds__(UA_THREADS, 1) k_sparse_attn_umma(PPAttnParams p) {
  extern __shared__ __align__(1024) uint8_t ua_raw[];
  const int win = blockIdx.z, head = blockIdx.y;
  if (p.flags[win] == 0) return;
  // SWIZZLE_128B tiles need 1 KB alignment; the pad is applied as an offset so the pointer stays in the shared window
  uint8_t* base = ua_raw + ((1024u - (ua_smem(ua_raw) & 1023u)) & 1023u);
  uint8_t* sQ = base;
  uint8_t* stages = base + UA_Q_BYTES;
  uint8_t* tail = stages + UA_STAGES * UA_STAGE_BYTES;
  // barriers: 0,1 kv_full[2]  2,3 kv_empty[2]
  unsigned long long* bars = reinterpret_cast<unsigned long long*>(tail);
  int* stab = reinterpret_cast<int*>(tail + 256);                      // this window's token table, staged once
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int* ktab = p.key_tok + (long)win * p.NKO;
  const int hoff = head * 128;
  const int q0 = blockIdx.x * UA_BM;
  const int nq = min(UA_BM, p.t * p.WN - q0);
  const int keys_per_frame = p.NKO + p.NP;
  const int nkeys = p.nkf * keys_per_frame;
  const int ntiles = (nkeys + UA_BN - 1) / UA_BN;
  const uint32_t b0 = ua_smem(&bars[0]);
  auto bar = [&](int i) { return b0 + 8u * (uint32_t)i; };

  if (tid == 0) {
    for (int i = 0; i < UA_STAGES; ++i) { ua_bar_init(bar(i), 128); ua_bar_init(bar(2 + i), 8); }   // full: producer threads; empty: consumer warps
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = tid; i < p.NKO; i += UA_THREADS) stab[i] = ktab[i];
  __syncthreads();

  if (warp >= 8) {
    // ================================================= producers: K tile (cp.async) + V^T tile (transposing stores)
    const int ptid = tid - 256;
    for (int j = 0; j < ntiles; ++j) {
      const int s = j % UA_STAGES, use = j / UA_STAGES;
      ua_bar_wait(bar(2 + s), (use & 1) ^ 1);                            // stage free (passes immediately on first use)
      uint8_t* sK = stages + s * UA_STAGE_BYTES;
      uint8_t* sV = sK + UA_K_BYTES;
      // row pointers of the tile's 64 keys (K part; V follows at +C in token rows and pooled rows alike)
      const float** kp = reinterpret_cast<const float**>(tail + 1152) + s * UA_BN;        // per stage
      if (ptid < UA_BN) {
        const int jk = j * UA_BN + ptid;
        const float* src = nullptr;
        if (jk < nkeys) {
          const int kfi = jk / keys_per_frame, slot = jk - kfi * keys_per_frame, fr = p.kf_start + kfi * p.kf_step;
          src = slot < p.NKO ? p.qkv + ((long)fr * p.NT + stab[slot]) * p.ld_qkv + p.C + hoff
                             : p.pool + ((long)fr * p.NP + (slot - p.NKO)) * p.ld_pool + hoff;
        }
        kp[ptid] = src;
      }
      asm volatile("bar.sync 1, 128;" ::: "memory");                     // producer warpgroup only
      // K rows: a warp copies whole 512-byte rows (lane <-> 16-byte chunk) straight into the swizzled tile
#pragma unroll 4
      for (int i = 0; i < 16; ++i) {
        const int kk = (ptid >> 5) + 4 * i, c4 = ptid & 31;
        const float* src = kp[kk];
        uint8_t* dk = sK + ua_off(kk, c4 * 4, UA_BN);
        if (src) pp_cp_async16(dk, src + c4 * 4);
        else *reinterpret_cast<float4*>(dk) = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      pp_cp_async_commit();
      // V^T: thread <-> (key, half of the head dims).  For a fixed head dim the 32 lanes of a warp (32 keys) store one whole
      // 128-byte row of the swizzled tile: no bank conflicts.  The row's other 16-byte pieces are read by the following
      // loads of the same lane, so the strided global loads hit L1 after the first.
      {
        const int key = ptid & 63, half = ptid >> 6, col = ua_vcol(key);
        const float* vr = kp[key];
#pragma unroll 2
        for (int i0 = 0; i0 < 16; i0 += 8) {
          float4 v[8];
#pragma unroll
          for (int i = 0; i < 8; ++i)
            v[i] = vr ? __ldg(reinterpret_cast<const float4*>(vr + p.C + half * 64 + 4 * (i0 + i))) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int d = half * 64 + 4 * (i0 + i);
            *reinterpret_cast<uint32_t*>(sV + ua_off(d + 0, col, 128)) = pp_tf32(v[i].x);
            *reinterpret_cast<uint32_t*>(sV + ua_off(d + 1, col, 128)) = pp_tf32(v[i].y);
            *reinterpret_cast<uint32_t*>(sV + ua_off(d + 2, col, 128)) = pp_tf32(v[i].z);
            *reinterpret_cast<uint32_t*>(sV + ua_off(d + 3, col, 128)) = pp_tf32(v[i].w);
          }
        }
      }
      pp_cp_async_wait<0>();
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic-proxy writes -> visible to wgmma
      ua_bar_arrive(bar(s));
    }
    return;
  }

  // ================================================= consumer warpgroup wg: query rows 64wg .. 64wg+63 of the tile
  const int wg = warp >> 2, g = lane >> 2, t = lane & 3;
  {   // Q rows of this warpgroup -> shared memory (thread <-> row), pre-scaled into the log2 domain, rounded to TF32
    const int row = wg * 64 + (tid & 63), c_half = (tid >> 6) & 1;
    const float* qrow = nullptr;
    if (row < nq) { const int qi = q0 + row, fr = qi / p.WN; qrow = p.qkv + ((long)fr * p.NT + stab[qi - fr * p.WN]) * p.ld_qkv + hoff; }
#pragma unroll 4
    for (int c = c_half * 64; c < c_half * 64 + 64; c += 4) {
      const float4 v = qrow ? *reinterpret_cast<const float4*>(qrow + c) : make_float4(0.f, 0.f, 0.f, 0.f);
      // round-to-nearest TF32 here: the tensor core would otherwise truncate the fp32 mantissa
      *reinterpret_cast<uint4*>(sQ + ua_off(row, c, UA_BM)) =
          make_uint4(pp_tf32(v.x * p.scale_log2), pp_tf32(v.y * p.scale_log2), pp_tf32(v.z * p.scale_log2), pp_tf32(v.w * p.scale_log2));
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    if (wg == 0) asm volatile("bar.sync 2, 128;" ::: "memory");
    else asm volatile("bar.sync 3, 128;" ::: "memory");
  }
  const uint64_t qd = ua_desc(ua_smem(sQ) + (uint32_t)wg * 64 * 128);
  float o[64], sacc[32];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;             // rows g and g + 8 of this warp's 16
  for (int j = 0; j < ntiles; ++j) {
    const int s = j % UA_STAGES;
    ua_bar_wait(bar(s), (j / UA_STAGES) & 1);
    const uint32_t kaddr = ua_smem(stages + s * UA_STAGE_BYTES);
    const uint64_t kd = ua_desc(kaddr), vd = ua_desc(kaddr + UA_K_BYTES);
    // ---- S = Q K^T: 128 head dims = 4 k-blocks x 4 k-steps of 8
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < 16; ++ks)
      wg_mma_ss_n64(sacc, qd + (uint64_t)(((ks >> 2) * (UA_BM * 128) + (ks & 3) * 32) >> 4),
                    kd + (uint64_t)(((ks >> 2) * (UA_BN * 128) + (ks & 3) * 32) >> 4), ks > 0);
    wg_commit();
    wg_wait<0>();
    wg_pin(sacc);
    const int kbase = j * UA_BN;
    if (kbase + UA_BN > nkeys) {                                        // ragged last tile: mask the missing keys
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const int k0 = kbase + 8 * c + 2 * t;
        if (k0 >= nkeys) { sacc[4 * c] = -INFINITY; sacc[4 * c + 2] = -INFINITY; }
        if (k0 + 1 >= nkeys) { sacc[4 * c + 1] = -INFINITY; sacc[4 * c + 3] = -INFINITY; }
      }
    }
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      mx0 = fmaxf(mx0, fmaxf(sacc[4 * c], sacc[4 * c + 1]));
      mx1 = fmaxf(mx1, fmaxf(sacc[4 * c + 2], sacc[4 * c + 3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
    const float al0 = exp2f(m0 - mn0), al1 = exp2f(m1 - mn1);           // m = -inf on the first tile -> alpha = 0
    m0 = mn0; m1 = mn1;
    float rs0 = 0.f, rs1 = 0.f;
    uint32_t pa[8][4];
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const float e0 = exp2f(sacc[4 * c] - mn0), e1 = exp2f(sacc[4 * c + 1] - mn0);
      const float e2 = exp2f(sacc[4 * c + 2] - mn1), e3 = exp2f(sacc[4 * c + 3] - mn1);
      rs0 += e0 + e1; rs1 += e2 + e3;
      // A fragment of k-step c: (row g, key 2t) (row g+8, key 2t) (row g, key 2t+1) (row g+8, key 2t+1)
      pa[c][0] = pp_tf32(e0); pa[c][1] = pp_tf32(e2); pa[c][2] = pp_tf32(e1); pa[c][3] = pp_tf32(e3);
    }
    l0 = l0 * al0 + rs0; l1 = l1 * al1 + rs1;
#pragma unroll
    for (int c = 0; c < 16; ++c) { o[4 * c] *= al0; o[4 * c + 1] *= al0; o[4 * c + 2] *= al1; o[4 * c + 3] *= al1; }
    // ---- O += P V: 64 keys = 2 k-blocks x 4 k-steps of 8
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < 8; ++ks)
      wg_mma_rs_n128(o, pa[ks], vd + (uint64_t)(((ks >> 2) * (128 * 128) + (ks & 3) * 32) >> 4), 1);
    wg_commit();
    wg_wait<0>();
    wg_pin(o);
    if (lane == 0) ua_bar_arrive(bar(2 + s));                           // this warp is done with the stage
  }
  // ---- epilogue: O / l -> global
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
  const int ra = wg * 64 + (warp & 3) * 16 + g, rb = ra + 8;
  float* oa = nullptr; float* ob = nullptr;
  if (ra < nq) { const int qi = q0 + ra, fr = qi / p.WN; oa = p.out + ((long)fr * p.NT + stab[qi - fr * p.WN]) * p.ld_out + hoff; }
  if (rb < nq) { const int qi = q0 + rb, fr = qi / p.WN; ob = p.out + ((long)fr * p.NT + stab[qi - fr * p.WN]) * p.ld_out + hoff; }
#pragma unroll
  for (int c = 0; c < 16; ++c) {
    const int n = 8 * c + 2 * t;
    if (oa) *reinterpret_cast<float2*>(oa + n) = make_float2(o[4 * c] * inv0, o[4 * c + 1] * inv0);
    if (ob) *reinterpret_cast<float2*>(ob + n) = make_float2(o[4 * c + 2] * inv1, o[4 * c + 3] * inv1);
  }
}

// masked windows on wgmma; called by pp_sparse_window_attn (mma_kernels.cu)
int pp_launch_sparse_attn_umma(const PPAttnParams& p, int n_windows, cudaStream_t stream) {
  if (p.NKO > 224) return PP_ERR_SHAPE;
  if (cudaFuncSetAttribute(k_sparse_attn_umma, cudaFuncAttributeMaxDynamicSharedMemorySize, UA_SMEM_BYTES) != cudaSuccess)
    return PP_ERR_LAUNCH;
  dim3 grid((p.t * p.WN + UA_BM - 1) / UA_BM, p.C / 128, n_windows);
  k_sparse_attn_umma<<<grid, UA_THREADS, UA_SMEM_BYTES, stream>>>(p);
  return cudaPeekAtLastError() == cudaSuccess ? PP_OK : PP_ERR_LAUNCH;
}

// ================================================================ fp16 operands (config.HALF_OPERANDS)
// Same tiling and pipeline on m64nNk16 f32.f16.f16: qkv / pool rows are fp16, the output is fp16 (rounded once).  K and V
// tiles are the same plain row copies (cp.async, no transposing producers): K is read K-major, V through the B-transpose bit
// as an MN-major operand.  P goes from the S accumulator straight into A fragments (keys 2t, 2t+1 / 2t+8, 2t+9 of each k16
// step are exactly the accumulator's columns of two adjacent n8 blocks).  Softmax statistics and O stay fp32.
#define UH_BN 64
#define UH_Q_BYTES (UA_BM * 128 * 2)               // 32 KB: 2 k-blocks of [128 rows x 128 B]
#define UH_K_BYTES (UH_BN * 128 * 2)               // 16 KB: 2 k-blocks of [64 keys x 128 B]
#define UH_V_BYTES (UH_BN * 128 * 2)               // 16 KB: 2 blocks of 64 head dims, [64 keys x 128 B] each (MN-major)
#define UH_STAGE_BYTES (UH_K_BYTES + UH_V_BYTES)
#define UH_STAGES 3
#define UH_TAIL_BYTES 4096                         // barriers, token table (<= 224 ints at +256), key row pointers (+1152)
#define UH_SMEM_BYTES (UH_Q_BYTES + UH_STAGES * UH_STAGE_BYTES + UH_TAIL_BYTES + 1024)
static_assert(1152 + UH_STAGES * UH_BN * 8 <= UH_TAIL_BYTES, "key row pointers overflow the tail");

__device__ __forceinline__ uint32_t uh_pack(float a, float b) {
  const __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}

__global__ void __launch_bounds__(UA_THREADS, 1) k_sparse_attn_umma_f16(PPAttnParams p) {
  extern __shared__ __align__(1024) uint8_t ua_raw[];
  const int win = blockIdx.z, head = blockIdx.y;
  if (p.flags[win] == 0) return;
  uint8_t* base = ua_raw + ((1024u - (ua_smem(ua_raw) & 1023u)) & 1023u);
  uint8_t* sQ = base;
  uint8_t* stages = base + UH_Q_BYTES;
  uint8_t* tail = stages + UH_STAGES * UH_STAGE_BYTES;
  unsigned long long* bars = reinterpret_cast<unsigned long long*>(tail);   // full[S], empty[S]
  int* stab = reinterpret_cast<int*>(tail + 256);
  const __half* qkv = reinterpret_cast<const __half*>(p.qkv);
  const __half* pool = reinterpret_cast<const __half*>(p.pool);
  __half* out = reinterpret_cast<__half*>(p.out);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int* ktab = p.key_tok + (long)win * p.NKO;
  const int hoff = head * 128;
  const int q0 = blockIdx.x * UA_BM;
  const int nq = min(UA_BM, p.t * p.WN - q0);
  const int keys_per_frame = p.NKO + p.NP;
  const int nkeys = p.nkf * keys_per_frame;
  const int ntiles = (nkeys + UH_BN - 1) / UH_BN;
  const uint32_t b0 = ua_smem(&bars[0]);
  auto bar = [&](int i) { return b0 + 8u * (uint32_t)i; };

  if (tid == 0) {
    for (int i = 0; i < UH_STAGES; ++i) { ua_bar_init(bar(i), 128); ua_bar_init(bar(UH_STAGES + i), 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = tid; i < p.NKO; i += UA_THREADS) stab[i] = ktab[i];
  __syncthreads();

  if (warp >= 8) {
    // ================================================= producers: K and V rows of the tile, both plain 16-byte copies
    const int ptid = tid - 256;
    for (int j = 0; j < ntiles; ++j) {
      const int s = j % UH_STAGES, use = j / UH_STAGES;
      ua_bar_wait(bar(UH_STAGES + s), (use & 1) ^ 1);
      uint8_t* sK = stages + s * UH_STAGE_BYTES;
      uint8_t* sV = sK + UH_K_BYTES;
      const __half** kp = reinterpret_cast<const __half**>(tail + 1152) + s * UH_BN;
      if (ptid < UH_BN) {
        const int jk = j * UH_BN + ptid;
        const __half* src = nullptr;
        if (jk < nkeys) {
          const int kfi = jk / keys_per_frame, slot = jk - kfi * keys_per_frame, fr = p.kf_start + kfi * p.kf_step;
          src = slot < p.NKO ? qkv + ((long)fr * p.NT + stab[slot]) * p.ld_qkv + p.C + hoff
                             : pool + ((long)fr * p.NP + (slot - p.NKO)) * p.ld_pool + hoff;
        }
        kp[ptid] = src;
      }
      asm volatile("bar.sync 1, 128;" ::: "memory");
      // a key row is 256 bytes of K and 256 of V: 16 chunks each; chunk c8 holds head dims 8*c8 .. 8*c8+7 (4 half pairs)
#pragma unroll 4
      for (int i = 0; i < 8; ++i) {
        const int kk = (ptid >> 4) + 8 * i, c8 = ptid & 15;
        const __half* src = kp[kk];
        const uint32_t off = ua_off(kk, c8 * 4, UH_BN);
        if (src) {
          pp_cp_async16(sK + off, src + c8 * 8);
          pp_cp_async16(sV + off, src + p.C + c8 * 8);
        } else {
          *reinterpret_cast<uint4*>(sK + off) = make_uint4(0u, 0u, 0u, 0u);
          *reinterpret_cast<uint4*>(sV + off) = make_uint4(0u, 0u, 0u, 0u);
        }
      }
      pp_cp_async_commit();
      pp_cp_async_wait<0>();
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      ua_bar_arrive(bar(s));
    }
    return;
  }

  const int wg = warp >> 2, g = lane >> 2, t = lane & 3;
  {   // Q rows -> shared memory, scaled into the log2 domain in fp32 and rounded to fp16 once
    const int row = wg * 64 + (tid & 63), c_half = (tid >> 6) & 1;
    const __half* qrow = nullptr;
    if (row < nq) { const int qi = q0 + row, fr = qi / p.WN; qrow = qkv + ((long)fr * p.NT + stab[qi - fr * p.WN]) * p.ld_qkv + hoff; }
#pragma unroll 4
    for (int c = c_half * 64; c < c_half * 64 + 64; c += 8) {
      uint4 u = make_uint4(0u, 0u, 0u, 0u);
      if (qrow) {
        const float4 a = pp_ld4(qrow + c), b = pp_ld4(qrow + c + 4);
        const float sc = p.scale_log2;
        u = make_uint4(uh_pack(a.x * sc, a.y * sc), uh_pack(a.z * sc, a.w * sc), uh_pack(b.x * sc, b.y * sc), uh_pack(b.z * sc, b.w * sc));
      }
      *reinterpret_cast<uint4*>(sQ + ua_off(row, c / 2, UA_BM)) = u;
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    if (wg == 0) asm volatile("bar.sync 2, 128;" ::: "memory");
    else asm volatile("bar.sync 3, 128;" ::: "memory");
  }
  const uint64_t qd = ua_desc(ua_smem(sQ) + (uint32_t)wg * 64 * 128);
  float o[64], sacc[32];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  for (int j = 0; j < ntiles; ++j) {
    const int s = j % UH_STAGES;
    ua_bar_wait(bar(s), (j / UH_STAGES) & 1);
    const uint32_t kaddr = ua_smem(stages + s * UH_STAGE_BYTES);
    const uint64_t kd = ua_desc(kaddr), vd = ua_desc_mn(kaddr + UH_K_BYTES, UH_BN * 128);
    // ---- S = Q K^T: 128 head dims = 2 k-blocks x 4 k-steps of 16
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < 8; ++ks)
      wg_mma_ss_n64_f16(sacc, qd + (uint64_t)(((ks >> 2) * (UA_BM * 128) + (ks & 3) * 32) >> 4),
                        kd + (uint64_t)(((ks >> 2) * (UH_BN * 128) + (ks & 3) * 32) >> 4), ks > 0);
    wg_commit();
    wg_wait<0>();
    wg_pin(sacc);
    const int kbase = j * UH_BN;
    if (kbase + UH_BN > nkeys) {
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const int k0 = kbase + 8 * c + 2 * t;
        if (k0 >= nkeys) { sacc[4 * c] = -INFINITY; sacc[4 * c + 2] = -INFINITY; }
        if (k0 + 1 >= nkeys) { sacc[4 * c + 1] = -INFINITY; sacc[4 * c + 3] = -INFINITY; }
      }
    }
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      mx0 = fmaxf(mx0, fmaxf(sacc[4 * c], sacc[4 * c + 1]));
      mx1 = fmaxf(mx1, fmaxf(sacc[4 * c + 2], sacc[4 * c + 3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
    const float al0 = exp2f(m0 - mn0), al1 = exp2f(m1 - mn1);
    m0 = mn0; m1 = mn1;
    float rs0 = 0.f, rs1 = 0.f;
    float e[32];
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      e[4 * c] = exp2f(sacc[4 * c] - mn0); e[4 * c + 1] = exp2f(sacc[4 * c + 1] - mn0);
      e[4 * c + 2] = exp2f(sacc[4 * c + 2] - mn1); e[4 * c + 3] = exp2f(sacc[4 * c + 3] - mn1);
      rs0 += e[4 * c] + e[4 * c + 1]; rs1 += e[4 * c + 2] + e[4 * c + 3];
    }
    uint32_t pa[4][4];
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {                    // keys 16ks + {2t, 2t+1} = n8 block 2ks, + {8+2t, 9+2t} = block 2ks+1
      pa[ks][0] = uh_pack(e[8 * ks], e[8 * ks + 1]);
      pa[ks][1] = uh_pack(e[8 * ks + 2], e[8 * ks + 3]);
      pa[ks][2] = uh_pack(e[8 * ks + 4], e[8 * ks + 5]);
      pa[ks][3] = uh_pack(e[8 * ks + 6], e[8 * ks + 7]);
    }
    l0 = l0 * al0 + rs0; l1 = l1 * al1 + rs1;
#pragma unroll
    for (int c = 0; c < 16; ++c) { o[4 * c] *= al0; o[4 * c + 1] *= al0; o[4 * c + 2] *= al1; o[4 * c + 3] *= al1; }
    // ---- O += P V: 64 keys = 4 k-steps of 16 = 2 swizzle atoms of 8 keys each
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) wg_mma_rs_n128_f16_tb(o, pa[ks], vd + (uint64_t)((ks * 2048) >> 4), 1);
    wg_commit();
    wg_wait<0>();
    wg_pin(o);
    if (lane == 0) ua_bar_arrive(bar(UH_STAGES + s));
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
  const int ra = wg * 64 + (warp & 3) * 16 + g, rb = ra + 8;
  __half* oa = nullptr; __half* ob = nullptr;
  if (ra < nq) { const int qi = q0 + ra, fr = qi / p.WN; oa = out + ((long)fr * p.NT + stab[qi - fr * p.WN]) * p.ld_out + hoff; }
  if (rb < nq) { const int qi = q0 + rb, fr = qi / p.WN; ob = out + ((long)fr * p.NT + stab[qi - fr * p.WN]) * p.ld_out + hoff; }
#pragma unroll
  for (int c = 0; c < 16; ++c) {
    const int n = 8 * c + 2 * t;
    if (oa) *reinterpret_cast<uint32_t*>(oa + n) = uh_pack(o[4 * c] * inv0, o[4 * c + 1] * inv0);
    if (ob) *reinterpret_cast<uint32_t*>(ob + n) = uh_pack(o[4 * c + 2] * inv1, o[4 * c + 3] * inv1);
  }
}

int pp_launch_sparse_attn_umma_f16(const PPAttnParams& p, int n_windows, cudaStream_t stream) {
  if (p.NKO > 224) return PP_ERR_SHAPE;
  if (cudaFuncSetAttribute(k_sparse_attn_umma_f16, cudaFuncAttributeMaxDynamicSharedMemorySize, UH_SMEM_BYTES) != cudaSuccess)
    return PP_ERR_LAUNCH;
  dim3 grid((p.t * p.WN + UA_BM - 1) / UA_BM, p.C / 128, n_windows);
  k_sparse_attn_umma_f16<<<grid, UA_THREADS, UH_SMEM_BYTES, stream>>>(p);
  return cudaPeekAtLastError() == cudaSuccess ? PP_OK : PP_ERR_LAUNCH;
}
