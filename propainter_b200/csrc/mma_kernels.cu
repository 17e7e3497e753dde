// Tensor-core kernels of the ProPainter hot path, first generation: warp-level TF32 mma.sync tiles.
//   * pp_corr_build        RAFT all-pairs correlation (3xTF32 split => fp32-accurate), level-0 writer
//   * pp_deform_align      modulated deformable 3x3 alignment: offset prep + bilinear gather + GEMM fused
//   * pp_sparse_window_attn mask-guided sparse window attention, flash-style, K/V gathered arithmetically
//   * pp_sparse_window_attn_f16 the same on fp16 operands (unmasked windows here on m16n8k16, masked ones in attn_umma.cu)
#include "pp_elem.cuh"
#include "pp_mma.cuh"
#include "../../include/propainter_b200.h"

#define PP_LAUNCH_CHECK() do { if (cudaPeekAtLastError() != cudaSuccess) return PP_ERR_LAUNCH; } while (0)

// ================================================================ RAFT correlation volume (level 0)
// C[i][j] = <f1[i,:], f2[j,:]> / sqrt(D)  (RAFT/corr.py:52-60).  fmaps pixel-major [frame][h*w][D].
// 64x64x32 tiles, 4 warps (2x2) of 32x32; fp32 accuracy kept with the 3xTF32 split
// (a_hi*b_hi + a_lo*b_hi + a_hi*b_lo) because the reference computes this matmul in full fp32.
__global__ void __launch_bounds__(128) k_corr_build(const float* __restrict__ fmap, int D, const int* __restrict__ idx1,
    const int* __restrict__ idx2, float* __restrict__ lvl0, int h, int w, int ld0, float scale) {
  __shared__ __align__(16) float As[64][36];
  __shared__ __align__(16) float Bs[64][36];
  const int N = h * w;
  const int pair = blockIdx.z, i0 = blockIdx.y * 64, j0 = blockIdx.x * 64;
  const float* A = fmap + (long)idx1[pair] * N * D;
  const float* B = fmap + (long)idx2[pair] * N * D;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int wm = warp >> 1, wn = warp & 1;
  float acc[2][4][4];
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[a][b][c] = 0.f;

  for (int k0 = 0; k0 < D; k0 += 32) {
    __syncthreads();
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      int idx = tid + 128 * r, row = idx >> 3, c4 = idx & 7;
      int ia = min(i0 + row, N - 1), jb = min(j0 + row, N - 1);
      pp_cp_async16(&As[row][c4 * 4], A + (long)ia * D + k0 + c4 * 4);
      pp_cp_async16(&Bs[row][c4 * 4], B + (long)jb * D + k0 + c4 * 4);
    }
    pp_cp_async_commit();
    pp_cp_async_wait<0>();
    __syncthreads();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      uint32_t ah[2][4], al[2][4], bh[4][2], bl[4][2];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        const int r0 = wm * 32 + mt * 16 + g;
        float v[4] = {As[r0][ks * 8 + t], As[r0 + 8][ks * 8 + t], As[r0][ks * 8 + t + 4], As[r0 + 8][ks * 8 + t + 4]};
#pragma unroll
        for (int q = 0; q < 4; ++q) { ah[mt][q] = pp_tf32(v[q]); al[mt][q] = pp_tf32(v[q] - __uint_as_float(ah[mt][q])); }
      }
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        const int c0 = wn * 32 + nt * 8 + g;
        float v[2] = {Bs[c0][ks * 8 + t], Bs[c0][ks * 8 + t + 4]};
#pragma unroll
        for (int q = 0; q < 2; ++q) { bh[nt][q] = pp_tf32(v[q]); bl[nt][q] = pp_tf32(v[q] - __uint_as_float(bh[nt][q])); }
      }
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          pp_mma_tf32(acc[mt][nt], al[mt], bh[nt]);
          pp_mma_tf32(acc[mt][nt], ah[mt], bl[nt]);
          pp_mma_tf32(acc[mt][nt], ah[mt], bh[nt]);
        }
    }
  }
  const long plane = (long)h * ld0;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        int i = i0 + wm * 32 + mt * 16 + g + ((q & 2) ? 8 : 0);
        int j = j0 + wn * 32 + nt * 8 + 2 * t + (q & 1);
        if (i < N && j < N) {
          int y2 = j / w, x2 = j - y2 * w;
          lvl0[((long)pair * N + i) * plane + (long)y2 * ld0 + x2] = acc[mt][nt][q] * scale;
        }
      }
}

// replaces CorrBlock.corr (RAFT/corr.py:52-60); pooled levels come from pp_corr_pool_pyramid
extern "C" int pp_corr_build(const float* fmap, int D, const int* idx1, const int* idx2, int n_pairs, float* lvl0,
                             int h, int w, cudaStream_t stream) {
  if (D % 32 || n_pairs < 1) return PP_ERR_SHAPE;
  const int N = h * w;
  dim3 grid((N + 63) / 64, (N + 63) / 64, n_pairs);
  k_corr_build<<<grid, 128, 0, stream>>>(fmap, D, idx1, idx2, lvl0, h, w, pp_corr_ld(w), 1.0f / sqrtf((float)D));
  PP_LAUNCH_CHECK();
  return PP_OK;
}

// ================================================================ deformable alignment
// out[p][n] = bias[n] + sum_{k<9,c<Cin} Wp[k*Cin+c][n] * sample(x, p, k, c)            (TF32 MMA)
// CTA = 32 pixels x 128 outputs, 4 warps (2 along M x 2 along N).  Each K-step stages the modulated
// bilinear samples of (tap k, 32 channels) for the 32 pixels into shared memory -- the im2col matrix
// torchvision materialises in HBM never exists -- and the matching 32x128 weight slab via cp.async.
// Two-stage software pipeline: while the tensor cores work on stage i, the weight slab of stage i+1 is
// in flight (cp.async) and the gather's global loads for stage i+1 are already issued into registers.
// Fragment loads are vectorised by renaming indices the MMA is indifferent to: inside each 8-wide
// k-step logical k=t / t+4 live at physical 2t / 2t+1 (one LDS.64 for A, adjacent rows for B), and
// the 8 n-tiles of a warp are interleaved (physical column 32q+4g+j <-> tile 4q+j, n=g) so that one
// LDS.128 of B feeds four MMAs and the epilogue stores float4.
#define DA_LDA 40
#define DA_LDB 132

// pre-pass: decode the offset-net output once per (pixel, tap, group) -> (py, px, modulation), so the GEMM kernel's
// inner loop has no transcendental math and reads its sampling positions as one aligned 16-byte load.
// propainter.py:58-65 / recurrent_flow_completion.py:34-40; `obias` = bias of conv_offset.6 (folded in here).
__global__ void __launch_bounds__(256) k_deform_taps(const float* __restrict__ o, int ld_o, const float* __restrict__ obias,
    const float* __restrict__ flow, float max_res, float4* __restrict__ taps, int H, int W) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;      // (pix*9 + k)*16 + g
  if (i >= (long)H * W * 144) return;
  const int g = (int)(i & 15); const long r = i >> 4; const int k = (int)(r % 9); const long pix = r / 9;
  const int y = (int)(pix / W), x = (int)(pix - (long)y * W);
  const float* op = o + pix * ld_o;
  float oy = op[g * 18 + 2 * k], ox = op[g * 18 + 2 * k + 1], ml = op[288 + g * 9 + k];
  if (obias) { oy += obias[g * 18 + 2 * k]; ox += obias[g * 18 + 2 * k + 1]; ml += obias[288 + g * 9 + k]; }
  oy = max_res * tanhf(oy); ox = max_res * tanhf(ox);
  if (flow) { oy += flow[2 * pix + 1]; ox += flow[2 * pix]; }
  taps[i] = make_float4((float)(y - 1 + k / 3) + oy, (float)(x - 1 + k % 3) + ox, 1.0f / (1.0f + expf(-ml)), 0.f);
}

struct DARaw { float4 u[4], v[4]; float w[4]; };
// issue the 8 corner loads of (tap position tp, 8 channels from c); corners with zero weight read a safe address
__device__ __forceinline__ void da_issue(const float* __restrict__ x, int ld_x, const float4 tp, int H, int W, int c, bool valid,
                                         DARaw& r) {
  PPDTap t; t.py = tp.x; t.px = tp.y; t.m = valid ? tp.z : 0.f;
  const PPDW d = pp_deform_weights(t, H, W);
  r.w[0] = d.w00; r.w[1] = d.w01; r.w[2] = d.w10; r.w[3] = d.w11;
  const float* p = x + ((long)d.y0 * W + d.x0) * ld_x + c;
  const float* q[4] = {p, p + ld_x, p + (long)W * ld_x, p + (long)W * ld_x + ld_x};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float* a = r.w[j] != 0.f ? q[j] : x + c;                // never dereference an out-of-image corner
    r.u[j] = *reinterpret_cast<const float4*>(a);
    r.v[j] = *reinterpret_cast<const float4*>(a + 4);
  }
}
__device__ __forceinline__ void da_combine(const DARaw& r, float4& s0, float4& s1) {
  s0 = make_float4(0.f, 0.f, 0.f, 0.f); s1 = s0;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float w = r.w[j];
    s0.x += r.u[j].x * w; s0.y += r.u[j].y * w; s0.z += r.u[j].z * w; s0.w += r.u[j].w * w;
    s1.x += r.v[j].x * w; s1.y += r.v[j].y * w; s1.z += r.v[j].z * w; s1.w += r.v[j].w * w;
  }
}

#define DA_NAME k_deform_align
#define DA_EXTRA_PARAMS
#define DA_NPIX ((long)H * W)
#define DA_REBASE
#include "deform_align_body.inc"
#undef DA_NAME
#undef DA_EXTRA_PARAMS
#undef DA_NPIX
#undef DA_REBASE
__global__ void __launch_bounds__(256) k_deform_reduce(const float* __restrict__ part, const float* __restrict__ bias,
                                                       float* __restrict__ out, int ld_out, long npix, int splits) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;     // over npix*32 float4
  if (i >= npix * 32) return;
  const long pix = i >> 5; const int n = (int)(i & 31) * 4;
  float4 s = *reinterpret_cast<const float4*>(bias + n);
  for (int k = 0; k < splits; ++k) {                                // fixed order: deterministic
    const float4 v = *reinterpret_cast<const float4*>(part + ((long)k * npix + pix) * 128 + n);
    s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
  }
  *reinterpret_cast<float4*>(out + pix * ld_out + n) = s;
}

// split-K factor: the kernel is latency-bound, so what matters is (waves of resident CTAs) x (K-steps per CTA + prologue).
// 4 CTAs fit per SM (126 registers x 128 threads, 44 KB shared memory); ties go to the smaller factor (less reduce traffic).
static int da_splits(long npix, int nit) {
  const long ctas = (npix + 31) / 32, slots = 4L * PP_NUM_SMS;
  int best = 1; long best_cost = -1;
  for (int s = 1; s <= 9; ++s) {
    const long waves = (ctas * s + slots - 1) / slots, steps = (nit + s - 1) / s;
    const long cost = waves * (steps + 2) * 16 + (s > 1 ? s : 0);
    if (best_cost < 0 || cost < best_cost) { best = s; best_cost = cost; }
  }
  return best;
}
extern "C" size_t pp_deform_align_workspace_bytes(int H, int W) {
  const long npix = (long)H * W;
  const int s = da_splits(npix, 36) > da_splits(npix, 72) ? da_splits(npix, 36) : da_splits(npix, 72);
  return (size_t)npix * 144 * sizeof(float4) + (s > 1 ? (size_t)s * npix * 128 * sizeof(float) : 0);   // tap records + split-K partials
}

// replaces DeformableAlignment.forward / SecondOrderDeformableAlignment.forward after the offset-net
// convs (model/propainter.py:57-69, model/recurrent_flow_completion.py:31-44 -> torchvision deform_conv2d).
// `o` is the raw output of conv_offset.6; pass its bias as `o_bias` if it has not been added yet (else NULL).
extern "C" int pp_deform_align(const float* x, int ld_x, const float* o, int ld_o, const float* o_bias, const float* flow,
                               float max_res, const float* w_packed, const float* bias, float* out, int ld_out, int H, int W,
                               int Cin, int Cout, void* workspace, size_t ws_bytes, cudaStream_t stream) {
  if (Cout != 128 || Cin % 32 || (Cin / 16) % 8) return PP_ERR_SHAPE;
  if (ld_x % 4 || ld_out % 4 || ld_o < 432 || ((uintptr_t)out & 15) || ((uintptr_t)bias & 15) || ((uintptr_t)x & 15)) return PP_ERR_ALIGN;
  const long npix = (long)H * W;
  const int splits = da_splits(npix, 9 * (Cin / 32));
  if (ws_bytes < pp_deform_align_workspace_bytes(H, W) || ((uintptr_t)workspace & 15)) return PP_ERR_WORKSPACE;
  float4* taps = (float4*)workspace;
  float* part = (float*)(taps + npix * 144);
  k_deform_taps<<<(int)((npix * 144 + 255) / 256), 256, 0, stream>>>(o, ld_o, o_bias, flow, max_res, taps, H, W);
  dim3 grid((unsigned)((npix + 31) / 32), splits);
  k_deform_align<<<grid, 128, 0, stream>>>(x, ld_x, taps, w_packed, bias, out, ld_out, H, W, Cin, part);
  if (splits > 1)
    k_deform_reduce<<<(int)((npix * 32 + 255) / 256), 256, 0, stream>>>(part, bias, out, ld_out, npix, splits);
  PP_LAUNCH_CHECK();
  return PP_OK;
}

// ================================================================ sparse window attention
// sparse_transformer.py:158-281.  One CTA = NWARPS*16 query rows of one (window, head); flash-style online
// softmax over key tiles of 64.  Keys of a masked window, per key frame: 45 own + 148 rolled (token
// table) + pooled tokens; unmasked windows attend per frame to their own 45 tokens.  Nothing is
// materialised: K/V rows (512 B per head) are gathered with cp.async straight from the QKV buffer into
// a two-stage shared-memory ring, so the gather of tile i+1 overlaps the MMAs of tile i.
// Fragment loads are 128-bit: for QK^T the 16 dims of two k-steps are renamed so a lane's float4 of K
// (and of Q) covers (k=t, k=t+4) of both steps; for PV the 16 head-dim tiles are interleaved (physical
// column 32q+4g+j <-> tile 4q+j, n=g) and P's C-fragment is reused as the A-fragment (keys 2t, 2t+1).
#define AT_LDK 144
#define AT_LDV 132
#define AT_LDQ 136                       // query staging stride: 128 x 136 floats fit inside one stage
#define AT_STAGE (64 * AT_LDK + 64 * AT_LDV)
template <bool MASKED, int NWARPS>
__global__ void __launch_bounds__(NWARPS * 32) k_sparse_attn(PPAttnParams p) {
  extern __shared__ __align__(16) float smem[];
  constexpr int ROWS = NWARPS * 16, NT_ = NWARPS * 32;
  const int win = blockIdx.z, head = blockIdx.y;
  if (MASKED != (p.flags[win] != 0)) return;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int* ktab = p.key_tok + (long)win * p.NKO;
  const int hoff = head * 128;
  const int q0 = MASKED ? blockIdx.x * ROWS : blockIdx.x * p.WN;
  const int nq = MASKED ? min(ROWS, p.t * p.WN - q0) : p.WN;
  const int keys_per_frame = p.NKO + p.NP;
  const int nkeys = MASKED ? p.nkf * keys_per_frame : p.WN;
  const int ntiles = (nkeys + 63) / 64;

  auto Kst = [&](int st) { return smem + st * AT_STAGE; };
  auto Vst = [&](int st) { return smem + st * AT_STAGE + 64 * AT_LDK; };
  auto gather = [&](int tile, int st) {
    float* Ks = Kst(st); float* Vs = Vst(st);
    for (int idx = tid; idx < 64 * 32; idx += NT_) {
      const int key = idx >> 5, c4 = idx & 31, j = tile * 64 + key;
      if (j < nkeys) {
        const float* src;
        if (MASKED) {
          const int kfi = j / keys_per_frame, slot = j - kfi * keys_per_frame;
          const int fr = p.kf_start + kfi * p.kf_step;
          if (slot < p.NKO) src = p.qkv + ((long)fr * p.NT + ktab[slot]) * p.ld_qkv + p.C + hoff;
          else src = p.pool + ((long)fr * p.NP + (slot - p.NKO)) * p.ld_pool + hoff;          // pool rows: K at 0, V at C
        } else {
          src = p.qkv + ((long)blockIdx.x * p.NT + ktab[j]) * p.ld_qkv + p.C + hoff;
        }
        pp_cp_async16(Ks + key * AT_LDK + c4 * 4, src + c4 * 4);
        pp_cp_async16(Vs + key * AT_LDV + c4 * 4, src + p.C + c4 * 4);
      } else {
        const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
        *reinterpret_cast<float4*>(Ks + key * AT_LDK + c4 * 4) = z;
        *reinterpret_cast<float4*>(Vs + key * AT_LDV + c4 * 4) = z;
      }
    }
    pp_cp_async_commit();
  };

  // ---- stage the query tile through stage 1 (free until the second key tile), scaled into the log2 domain
  static_assert(ROWS * AT_LDQ <= AT_STAGE, "query tile must fit in one stage");
  // masked: Q is staged through stage 1 (free until the 2nd key tile); unmasked windows have a single key tile and
  // run with ONE stage of shared memory (3 CTAs/SM instead of 1): Q goes through stage 0 before the gather.
  float* Qs = MASKED ? Kst(1) : Kst(0);
  for (int idx = tid; idx < ROWS * 32; idx += NT_) {
    const int row = idx >> 5, c4 = idx & 31;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (row < nq) {
      const int qi = q0 + row, fr = qi / p.WN, tok = ktab[qi - fr * p.WN];
      v = *reinterpret_cast<const float4*>(p.qkv + ((long)fr * p.NT + tok) * p.ld_qkv + hoff + c4 * 4);
    }
    v.x *= p.scale_log2; v.y *= p.scale_log2; v.z *= p.scale_log2; v.w *= p.scale_log2;
    *reinterpret_cast<float4*>(Qs + row * AT_LDQ + c4 * 4) = v;
  }
  if (MASKED) gather(0, 0);
  __syncthreads();
  uint32_t qa[16][4];
  {
    const float* r0 = Qs + (warp * 16 + g) * AT_LDQ;
    const float* r1 = r0 + 8 * AT_LDQ;
#pragma unroll
    for (int j = 0; j < 8; ++j) {                                         // dims 16j .. 16j+15 = k-steps 2j, 2j+1
      const float4 lo = *reinterpret_cast<const float4*>(r0 + 16 * j + 4 * t);
      const float4 hi = *reinterpret_cast<const float4*>(r1 + 16 * j + 4 * t);
      qa[2 * j][0] = pp_tf32(lo.x); qa[2 * j][1] = pp_tf32(hi.x); qa[2 * j][2] = pp_tf32(lo.y); qa[2 * j][3] = pp_tf32(hi.y);
      qa[2 * j + 1][0] = pp_tf32(lo.z); qa[2 * j + 1][1] = pp_tf32(hi.z); qa[2 * j + 1][2] = pp_tf32(lo.w); qa[2 * j + 1][3] = pp_tf32(hi.w);
    }
  }
  if (!MASKED) { __syncthreads(); gather(0, 0); }          // every warp has its Q fragments; stage 0 may be overwritten
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  float oacc[16][4];
#pragma unroll
  for (int a = 0; a < 16; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) oacc[a][b] = 0.f;

  for (int tile = 0; tile < ntiles; ++tile) {
    const int cur = tile & 1;
    pp_cp_async_wait<0>();
    __syncthreads();                          // tile landed; every warp is done with the other stage (and with Qs)
    if (tile + 1 < ntiles) gather(tile + 1, cur ^ 1);
    const float* Ks = Kst(cur); const float* Vs = Vst(cur);
    const int kt0 = tile * 64;

    // ---- S = Q K^T (already scaled, log2 domain)
    float s[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
      const float* kr = Ks + (nt * 8 + g) * AT_LDK + 4 * t;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 kv = *reinterpret_cast<const float4*>(kr + 16 * j);
        uint32_t b[2];
        b[0] = pp_tf32(kv.x); b[1] = pp_tf32(kv.y); pp_mma_tf32(s[nt], qa[2 * j], b);
        b[0] = pp_tf32(kv.z); b[1] = pp_tf32(kv.w); pp_mma_tf32(s[nt], qa[2 * j + 1], b);
      }
    }
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const int j = kt0 + nt * 8 + 2 * t;
      if (j >= nkeys) { s[nt][0] = -INFINITY; s[nt][2] = -INFINITY; }
      if (j + 1 >= nkeys) { s[nt][1] = -INFINITY; s[nt][3] = -INFINITY; }
      mx0 = fmaxf(mx0, fmaxf(s[nt][0], s[nt][1]));
      mx1 = fmaxf(mx1, fmaxf(s[nt][2], s[nt][3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
    const float al0 = exp2f(m0 - mn0), al1 = exp2f(m1 - mn1);
    m0 = mn0; m1 = mn1;
    float rs0 = 0.f, rs1 = 0.f;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      s[nt][0] = exp2f(s[nt][0] - mn0); s[nt][1] = exp2f(s[nt][1] - mn0);
      s[nt][2] = exp2f(s[nt][2] - mn1); s[nt][3] = exp2f(s[nt][3] - mn1);
      rs0 += s[nt][0] + s[nt][1]; rs1 += s[nt][2] + s[nt][3];
    }
    l0 = l0 * al0 + rs0; l1 = l1 * al1 + rs1;
#pragma unroll
    for (int nt = 0; nt < 16; ++nt) { oacc[nt][0] *= al0; oacc[nt][1] *= al0; oacc[nt][2] *= al1; oacc[nt][3] *= al1; }

    // ---- O += P V
#pragma unroll
    for (int kg = 0; kg < 8; ++kg) {
      const uint32_t a[4] = {pp_tf32(s[kg][0]), pp_tf32(s[kg][2]), pp_tf32(s[kg][1]), pp_tf32(s[kg][3])};
      const float* v0 = Vs + (kg * 8 + 2 * t) * AT_LDV + 4 * g;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float4 x0 = *reinterpret_cast<const float4*>(v0 + 32 * q);
        const float4 x1 = *reinterpret_cast<const float4*>(v0 + AT_LDV + 32 * q);
        uint32_t b[2];
        b[0] = pp_tf32(x0.x); b[1] = pp_tf32(x1.x); pp_mma_tf32(oacc[4 * q + 0], a, b);
        b[0] = pp_tf32(x0.y); b[1] = pp_tf32(x1.y); pp_mma_tf32(oacc[4 * q + 1], a, b);
        b[0] = pp_tf32(x0.z); b[1] = pp_tf32(x1.z); pp_mma_tf32(oacc[4 * q + 2], a, b);
        b[0] = pp_tf32(x0.w); b[1] = pp_tf32(x1.w); pp_mma_tf32(oacc[4 * q + 3], a, b);
      }
    }
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
  const int ra = warp * 16 + g, rb = ra + 8;
  float* oa = nullptr; float* ob = nullptr;
  if (ra < nq) { int qi = q0 + ra, fr = qi / p.WN; oa = p.out + ((long)fr * p.NT + ktab[qi - fr * p.WN]) * p.ld_out + hoff; }
  if (rb < nq) { int qi = q0 + rb, fr = qi / p.WN; ob = p.out + ((long)fr * p.NT + ktab[qi - fr * p.WN]) * p.ld_out + hoff; }
  // tile 4q+j, C-fragment column 2t+c  <->  head-dim column 32q + 4(2t+c) + j
#pragma unroll
  for (int q = 0; q < 4; ++q)
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const int n = 32 * q + 4 * (2 * t + c);
      if (oa) *reinterpret_cast<float4*>(oa + n) = make_float4(oacc[4 * q][c] * inv0, oacc[4 * q + 1][c] * inv0, oacc[4 * q + 2][c] * inv0, oacc[4 * q + 3][c] * inv0);
      if (ob) *reinterpret_cast<float4*>(ob + n) = make_float4(oacc[4 * q][c + 2] * inv1, oacc[4 * q + 1][c + 2] * inv1, oacc[4 * q + 2][c + 2] * inv1, oacc[4 * q + 3][c + 2] * inv1);
    }
}

// ---------------------------------------------------------------------------------------------------------------
// AT_UNMASKED_LOOP = 1 (default since round 2; 0 = one CTA per frame): unmasked windows with one CTA walking several frames of its
// (window, head).  The one-frame CTAs above are a serial load -> compute -> store chain;
// here the K/V rows of frame f+1 arrive by cp.async in the other
// stage while frame f is computed, stages hold 48 instead of 64 key rows (2 CTAs/SM with both stages), and the Q
// fragments come straight from global memory.  Same fragment maps and summation order as k_sparse_attn<false,4>, so
// the results are bit-identical.
#ifndef AT_UNMASKED_LOOP
#define AT_UNMASKED_LOOP 1
#endif
#define AU_KEYS 48
#define AU_STAGE (AU_KEYS * AT_LDK + AU_KEYS * AT_LDV)
__global__ void __launch_bounds__(128, 2) k_attn_unmasked_frames(PPAttnParams p, int fpc) {
  extern __shared__ __align__(16) float smem[];
  const int win = blockIdx.z, head = blockIdx.y;
  if (p.flags[win] != 0) return;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int* ktab = p.key_tok + (long)win * p.NKO;
  const int hoff = head * 128, WN = p.WN;
  const int f0 = blockIdx.x * fpc, f1 = min(p.t, f0 + fpc);
  if (f0 >= f1) return;
  auto Kst = [&](int st) { return smem + st * AU_STAGE; };
  auto Vst = [&](int st) { return smem + st * AU_STAGE + AU_KEYS * AT_LDK; };
  auto gather = [&](int f, int st) {
    float* Ks = Kst(st); float* Vs = Vst(st);
    for (int idx = tid; idx < WN * 32; idx += 128) {
      const int key = idx >> 5, c4 = idx & 31;
      const float* src = p.qkv + ((long)f * p.NT + ktab[key]) * p.ld_qkv + p.C + hoff;
      pp_cp_async16(Ks + key * AT_LDK + c4 * 4, src + c4 * 4);
      pp_cp_async16(Vs + key * AT_LDV + c4 * 4, src + p.C + c4 * 4);
    }
    pp_cp_async_commit();
  };
  // pad key rows [WN, 48) of both stages: zero once (their P is 0, but 0 * stale-NaN would poison the accumulators)
  for (int idx = tid; idx < 2 * (AU_KEYS - WN) * 32; idx += 128) {
    const int st = idx / ((AU_KEYS - WN) * 32), r = idx - st * (AU_KEYS - WN) * 32, key = WN + (r >> 5), c4 = r & 31;
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    *reinterpret_cast<float4*>(Kst(st) + key * AT_LDK + c4 * 4) = z;
    *reinterpret_cast<float4*>(Vst(st) + key * AT_LDV + c4 * 4) = z;
  }
  gather(f0, 0);
  const int ra = warp * 16 + g, rb = ra + 8;
  const int ta = ra < WN ? ktab[ra] : -1, tb = rb < WN ? ktab[rb] : -1;
  for (int f = f0; f < f1; ++f) {
    const int cur = (f - f0) & 1;
    // ---- Q fragments of frame f straight from global (rows ra / rb of this warp), scaled into the log2 domain
    uint32_t qa[16][4];
    {
      const float* r0 = p.qkv + ((long)f * p.NT + (ta >= 0 ? ta : 0)) * p.ld_qkv + hoff;
      const float* r1 = p.qkv + ((long)f * p.NT + (tb >= 0 ? tb : 0)) * p.ld_qkv + hoff;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float4 lo = make_float4(0.f, 0.f, 0.f, 0.f), hi = lo;
        if (ta >= 0) lo = *reinterpret_cast<const float4*>(r0 + 16 * j + 4 * t);
        if (tb >= 0) hi = *reinterpret_cast<const float4*>(r1 + 16 * j + 4 * t);
        lo.x *= p.scale_log2; lo.y *= p.scale_log2; lo.z *= p.scale_log2; lo.w *= p.scale_log2;
        hi.x *= p.scale_log2; hi.y *= p.scale_log2; hi.z *= p.scale_log2; hi.w *= p.scale_log2;
        qa[2 * j][0] = pp_tf32(lo.x); qa[2 * j][1] = pp_tf32(hi.x); qa[2 * j][2] = pp_tf32(lo.y); qa[2 * j][3] = pp_tf32(hi.y);
        qa[2 * j + 1][0] = pp_tf32(lo.z); qa[2 * j + 1][1] = pp_tf32(hi.z); qa[2 * j + 1][2] = pp_tf32(lo.w); qa[2 * j + 1][3] = pp_tf32(hi.w);
      }
    }
    pp_cp_async_wait<0>();
    __syncthreads();                          // frame f landed; every warp is done with the other stage
    if (f + 1 < f1) gather(f + 1, cur ^ 1);
    if (warp * 16 >= WN) continue;            // this warp's 16 query rows are all padding (no barrier below this point)
    const float* Ks = Kst(cur); const float* Vs = Vst(cur);
    // ---- S = Q K^T, 6 n-tiles of 8 keys
    float s[6][4];
#pragma unroll
    for (int nt = 0; nt < 6; ++nt) {
      s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
      const float* kr = Ks + (nt * 8 + g) * AT_LDK + 4 * t;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 kv = *reinterpret_cast<const float4*>(kr + 16 * j);
        uint32_t b[2];
        b[0] = pp_tf32(kv.x); b[1] = pp_tf32(kv.y); pp_mma_tf32(s[nt], qa[2 * j], b);
        b[0] = pp_tf32(kv.z); b[1] = pp_tf32(kv.w); pp_mma_tf32(s[nt], qa[2 * j + 1], b);
      }
    }
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < 6; ++nt) {
      const int j = nt * 8 + 2 * t;
      if (j >= WN) { s[nt][0] = -INFINITY; s[nt][2] = -INFINITY; }
      if (j + 1 >= WN) { s[nt][1] = -INFINITY; s[nt][3] = -INFINITY; }
      mx0 = fmaxf(mx0, fmaxf(s[nt][0], s[nt][1]));
      mx1 = fmaxf(mx1, fmaxf(s[nt][2], s[nt][3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    float l0 = 0.f, l1 = 0.f;
#pragma unroll
    for (int nt = 0; nt < 6; ++nt) {
      s[nt][0] = exp2f(s[nt][0] - mx0); s[nt][1] = exp2f(s[nt][1] - mx0);
      s[nt][2] = exp2f(s[nt][2] - mx1); s[nt][3] = exp2f(s[nt][3] - mx1);
      l0 += s[nt][0] + s[nt][1]; l1 += s[nt][2] + s[nt][3];
    }
    // ---- O = P V
    float oacc[16][4];
#pragma unroll
    for (int a = 0; a < 16; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b) oacc[a][b] = 0.f;
#pragma unroll
    for (int kg = 0; kg < 6; ++kg) {
      const uint32_t a[4] = {pp_tf32(s[kg][0]), pp_tf32(s[kg][2]), pp_tf32(s[kg][1]), pp_tf32(s[kg][3])};
      const float* v0 = Vs + (kg * 8 + 2 * t) * AT_LDV + 4 * g;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float4 x0 = *reinterpret_cast<const float4*>(v0 + 32 * q);
        const float4 x1 = *reinterpret_cast<const float4*>(v0 + AT_LDV + 32 * q);
        uint32_t b[2];
        b[0] = pp_tf32(x0.x); b[1] = pp_tf32(x1.x); pp_mma_tf32(oacc[4 * q + 0], a, b);
        b[0] = pp_tf32(x0.y); b[1] = pp_tf32(x1.y); pp_mma_tf32(oacc[4 * q + 1], a, b);
        b[0] = pp_tf32(x0.z); b[1] = pp_tf32(x1.z); pp_mma_tf32(oacc[4 * q + 2], a, b);
        b[0] = pp_tf32(x0.w); b[1] = pp_tf32(x1.w); pp_mma_tf32(oacc[4 * q + 3], a, b);
      }
    }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
    float* oa = ta >= 0 ? p.out + ((long)f * p.NT + ta) * p.ld_out + hoff : nullptr;
    float* ob = tb >= 0 ? p.out + ((long)f * p.NT + tb) * p.ld_out + hoff : nullptr;
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int n = 32 * q + 4 * (2 * t + c);
        if (oa) *reinterpret_cast<float4*>(oa + n) = make_float4(oacc[4 * q][c] * inv0, oacc[4 * q + 1][c] * inv0, oacc[4 * q + 2][c] * inv0, oacc[4 * q + 3][c] * inv0);
        if (ob) *reinterpret_cast<float4*>(ob + n) = make_float4(oacc[4 * q][c + 2] * inv1, oacc[4 * q + 1][c + 2] * inv1, oacc[4 * q + 2][c + 2] * inv1, oacc[4 * q + 3][c + 2] * inv1);
      }
  }
}

// fp16 operands (config.HALF_OPERANDS): the unmasked-window kernel above on mma.sync m16n8k16 f32.f16.f16.  fp16 qkv rows in,
// fp16 out (rounded once); Q scaled into the log2 domain in fp32 and rounded once; P's accumulator fragment is the A fragment
// of the P V step as it stands, V fragments come transposed out of row-major key rows by ldmatrix.trans.
#define AH_LD 136                                 // halves per staged key row: 272 bytes, conflict-free ldmatrix / 32-bit loads
#define AH_STAGE (2 * AU_KEYS * AH_LD)
__device__ __forceinline__ uint32_t ah_pack(float a, float b) {
  const __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}
__global__ void __launch_bounds__(128, 2) k_attn_unmasked_frames_f16(PPAttnParams p, int fpc) {
  extern __shared__ __align__(16) __half hsm[];
  const int win = blockIdx.z, head = blockIdx.y;
  if (p.flags[win] != 0) return;
  const __half* qkv = reinterpret_cast<const __half*>(p.qkv);
  __half* out = reinterpret_cast<__half*>(p.out);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int* ktab = p.key_tok + (long)win * p.NKO;
  const int hoff = head * 128, WN = p.WN;
  const int f0 = blockIdx.x * fpc, f1 = min(p.t, f0 + fpc);
  if (f0 >= f1) return;
  auto Kst = [&](int st) { return hsm + st * AH_STAGE; };
  auto Vst = [&](int st) { return hsm + st * AH_STAGE + AU_KEYS * AH_LD; };
  auto gather = [&](int f, int st) {
    __half* Ks = Kst(st); __half* Vs = Vst(st);
    for (int idx = tid; idx < WN * 16; idx += 128) {
      const int key = idx >> 4, c8 = idx & 15;
      const __half* src = qkv + ((long)f * p.NT + ktab[key]) * p.ld_qkv + p.C + hoff;
      pp_cp_async16(Ks + key * AH_LD + c8 * 8, src + c8 * 8);
      pp_cp_async16(Vs + key * AH_LD + c8 * 8, src + p.C + c8 * 8);
    }
    pp_cp_async_commit();
  };
  // pad key rows [WN, 48) of both stages: zero once (their P is 0, but 0 * stale-NaN would poison the accumulators)
  for (int idx = tid; idx < 2 * (AU_KEYS - WN) * 16; idx += 128) {
    const int st = idx / ((AU_KEYS - WN) * 16), r = idx - st * (AU_KEYS - WN) * 16, key = WN + (r >> 4), c8 = r & 15;
    *reinterpret_cast<uint4*>(Kst(st) + key * AH_LD + c8 * 8) = make_uint4(0u, 0u, 0u, 0u);
    *reinterpret_cast<uint4*>(Vst(st) + key * AH_LD + c8 * 8) = make_uint4(0u, 0u, 0u, 0u);
  }
  gather(f0, 0);
  const int ra = warp * 16 + g, rb = ra + 8;
  const int ta = ra < WN ? ktab[ra] : -1, tb = rb < WN ? ktab[rb] : -1;
  for (int f = f0; f < f1; ++f) {
    const int cur = (f - f0) & 1;
    uint32_t qa[8][4];
    {
      const __half* r0 = qkv + ((long)f * p.NT + (ta >= 0 ? ta : 0)) * p.ld_qkv + hoff;
      const __half* r1 = qkv + ((long)f * p.NT + (tb >= 0 ? tb : 0)) * p.ld_qkv + hoff;
      const float sc = p.scale_log2;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int d = 16 * j + 8 * h + 2 * t;
          float2 lo = make_float2(0.f, 0.f), hi = lo;
          if (ta >= 0) lo = __half22float2(*reinterpret_cast<const __half2*>(r0 + d));
          if (tb >= 0) hi = __half22float2(*reinterpret_cast<const __half2*>(r1 + d));
          qa[j][2 * h] = ah_pack(lo.x * sc, lo.y * sc);
          qa[j][2 * h + 1] = ah_pack(hi.x * sc, hi.y * sc);
        }
      }
    }
    pp_cp_async_wait<0>();
    __syncthreads();
    if (f + 1 < f1) gather(f + 1, cur ^ 1);
    if (warp * 16 >= WN) continue;
    const __half* Ks = Kst(cur); const __half* Vs = Vst(cur);
    float s[6][4];
#pragma unroll
    for (int nt = 0; nt < 6; ++nt) {
      s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
      const __half* kr = Ks + (nt * 8 + g) * AH_LD + 2 * t;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const uint32_t b[2] = {*reinterpret_cast<const uint32_t*>(kr + 16 * j), *reinterpret_cast<const uint32_t*>(kr + 16 * j + 8)};
        pp_mma_f16(s[nt], qa[j], b);
      }
    }
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < 6; ++nt) {
      const int j = nt * 8 + 2 * t;
      if (j >= WN) { s[nt][0] = -INFINITY; s[nt][2] = -INFINITY; }
      if (j + 1 >= WN) { s[nt][1] = -INFINITY; s[nt][3] = -INFINITY; }
      mx0 = fmaxf(mx0, fmaxf(s[nt][0], s[nt][1]));
      mx1 = fmaxf(mx1, fmaxf(s[nt][2], s[nt][3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    float l0 = 0.f, l1 = 0.f;
#pragma unroll
    for (int nt = 0; nt < 6; ++nt) {
      s[nt][0] = exp2f(s[nt][0] - mx0); s[nt][1] = exp2f(s[nt][1] - mx0);
      s[nt][2] = exp2f(s[nt][2] - mx1); s[nt][3] = exp2f(s[nt][3] - mx1);
      l0 += s[nt][0] + s[nt][1]; l1 += s[nt][2] + s[nt][3];
    }
    float oacc[16][4];
#pragma unroll
    for (int a = 0; a < 16; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b) oacc[a][b] = 0.f;
#pragma unroll
    for (int kk = 0; kk < 3; ++kk) {                       // 16 keys per step: n8 blocks 2kk (keys 2t..) and 2kk+1 (keys 8+2t..)
      const uint32_t a[4] = {ah_pack(s[2 * kk][0], s[2 * kk][1]), ah_pack(s[2 * kk][2], s[2 * kk][3]),
                             ah_pack(s[2 * kk + 1][0], s[2 * kk + 1][1]), ah_pack(s[2 * kk + 1][2], s[2 * kk + 1][3])};
      const __half* vrow = Vs + (16 * kk + ((lane >> 3) & 1) * 8 + (lane & 7)) * AH_LD + (lane >> 4) * 8;
#pragma unroll
      for (int np = 0; np < 8; ++np) {                     // head dims 16np .. 16np+15 = n8 tiles 2np, 2np+1
        uint32_t r[4];
        pp_ldmatrix_x4_trans(r, vrow + 16 * np);
        const uint32_t b0[2] = {r[0], r[1]}, b1[2] = {r[2], r[3]};
        pp_mma_f16(oacc[2 * np], a, b0);
        pp_mma_f16(oacc[2 * np + 1], a, b1);
      }
    }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
    __half* oa = ta >= 0 ? out + ((long)f * p.NT + ta) * p.ld_out + hoff : nullptr;
    __half* ob = tb >= 0 ? out + ((long)f * p.NT + tb) * p.ld_out + hoff : nullptr;
#pragma unroll
    for (int nt = 0; nt < 16; ++nt) {
      const int n = 8 * nt + 2 * t;
      if (oa) *reinterpret_cast<uint32_t*>(oa + n) = ah_pack(oacc[nt][0] * inv0, oacc[nt][1] * inv0);
      if (ob) *reinterpret_cast<uint32_t*>(ob + n) = ah_pack(oacc[nt][2] * inv1, oacc[nt][3] * inv1);
    }
  }
}

int pp_launch_sparse_attn_umma(const PPAttnParams& p, int n_windows, cudaStream_t stream);   // attn_umma.cu
int pp_launch_sparse_attn_umma_f16(const PPAttnParams& p, int n_windows, cudaStream_t stream);

static int pp_attn_check(const PPAttnParams& p) {
  if (p.C != 512 || p.WN > 64 || p.WN < 1 || p.ld_qkv % 4 || p.ld_pool % 4 || p.ld_out % 4 || p.nkf < 0) return PP_ERR_SHAPE;
  if (((uintptr_t)p.qkv & 15) || ((uintptr_t)p.pool & 15) || ((uintptr_t)p.out & 15)) return PP_ERR_ALIGN;
  return PP_OK;
}
static int pp_attn_unmasked(const PPAttnParams& p, int n_windows, cudaStream_t stream) {
#if AT_UNMASKED_LOOP
  if (p.WN <= AU_KEYS && p.WN >= 1) {
    const int smem2 = 2 * AU_STAGE * (int)sizeof(float);
    if (cudaFuncSetAttribute(k_attn_unmasked_frames, cudaFuncAttributeMaxDynamicSharedMemorySize, smem2) != cudaSuccess)
      return PP_ERR_LAUNCH;
    int fpc = (p.t * (p.C / 128) * n_windows + 2 * PP_NUM_SMS - 1) / (2 * PP_NUM_SMS);         // ~one wave of 2 CTAs/SM over all (frame, head, window) units
    fpc = fpc < 1 ? 1 : (fpc > 8 ? 8 : fpc);
    dim3 gl((p.t + fpc - 1) / fpc, p.C / 128, n_windows);
    k_attn_unmasked_frames<<<gl, 128, smem2, stream>>>(p, fpc);
    PP_LAUNCH_CHECK();
    return PP_OK;
  }
#endif
  const int smem1 = AT_STAGE * (int)sizeof(float);
  if (cudaFuncSetAttribute(k_sparse_attn<false, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem1) != cudaSuccess)
    return PP_ERR_LAUNCH;
  dim3 gu(p.t, p.C / 128, n_windows);
  k_sparse_attn<false, 4><<<gu, 128, smem1, stream>>>(p);
  PP_LAUNCH_CHECK();
  return PP_OK;
}

// replaces SparseWindowAttention.forward between the q/k/v Linear layers and `proj`
// (model/modules/sparse_transformer.py:177-275).  Masked windows: wgmma kernel (attn_umma.cu);
// unmasked windows (45x45 per frame): warp-level mma.sync kernel above.
extern "C" int pp_sparse_window_attn(const PPAttnParams* prm, int n_windows, cudaStream_t stream) {
  const PPAttnParams& p = *prm;
  int rc = pp_attn_check(p);
  if (rc != PP_OK) return rc;
  // nkf == 0 (t = 1 on an odd layer: T_ind is empty, sparse_transformer.py:339): masked windows attend to an empty key set,
  // for which the reference's softmax-then-matmul yields zeros -- the caller pre-zeroes `out` and only the unmasked windows run
  if (p.nkf > 0) {
    rc = pp_launch_sparse_attn_umma(p, n_windows, stream);
    if (rc != PP_OK) return rc;
  }
  return pp_attn_unmasked(p, n_windows, stream);
}

// same contract, masked windows on the warp-level mma.sync kernel (baseline of the wgmma kernel)
extern "C" int pp_sparse_window_attn_mma(const PPAttnParams* prm, int n_windows, cudaStream_t stream) {
  const PPAttnParams& p = *prm;
  int rc = pp_attn_check(p);
  if (rc != PP_OK) return rc;
  if (p.nkf <= 0) return pp_attn_unmasked(p, n_windows, stream);     // see pp_sparse_window_attn
  const int smem = 2 * AT_STAGE * (int)sizeof(float);
  if (cudaFuncSetAttribute(k_sparse_attn<true, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess)
    return PP_ERR_LAUNCH;
  dim3 gm((p.t * p.WN + 127) / 128, p.C / 128, n_windows);
  k_sparse_attn<true, 8><<<gm, 256, smem, stream>>>(p);
  PP_LAUNCH_CHECK();
  return pp_attn_unmasked(p, n_windows, stream);
}

// fp16 qkv / pool_kv in, fp16 out: masked windows on the f16 wgmma kernel (attn_umma.cu), unmasked windows on the f16 mma.sync
// kernel above.  Rows 16-byte aligned with ld % 8 == 0 (else PP_ERR_ALIGN); t = 0 or no window returns PP_OK without a launch.
extern "C" int pp_sparse_window_attn_f16(const PPAttnParams* prm, int n_windows, cudaStream_t stream) {
  const PPAttnParams& p = *prm;
  if (p.C != 512 || p.WN > AU_KEYS || p.WN < 1 || p.nkf < 0 || p.t < 0 || n_windows < 0) return PP_ERR_SHAPE;
  if (p.ld_qkv % 8 || p.ld_pool % 8 || p.ld_out % 8 || ((uintptr_t)p.qkv & 15) || ((uintptr_t)p.pool & 15) || ((uintptr_t)p.out & 15))
    return PP_ERR_ALIGN;
  if (p.t == 0 || n_windows == 0) return PP_OK;
  if (p.nkf > 0) {                                         // nkf == 0: see pp_sparse_window_attn (the caller pre-zeroes `out`)
    const int rc = pp_launch_sparse_attn_umma_f16(p, n_windows, stream);
    if (rc != PP_OK) return rc;
  }
  const int smem = 2 * AH_STAGE * (int)sizeof(__half);
  if (cudaFuncSetAttribute(k_attn_unmasked_frames_f16, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess)
    return PP_ERR_LAUNCH;
  int fpc = (p.t * (p.C / 128) * n_windows + 2 * PP_NUM_SMS - 1) / (2 * PP_NUM_SMS);
  fpc = fpc < 1 ? 1 : (fpc > 8 ? 8 : fpc);
  dim3 gl((p.t + fpc - 1) / fpc, p.C / 128, n_windows);
  k_attn_unmasked_frames_f16<<<gl, 128, smem, stream>>>(p, fpc);
  PP_LAUNCH_CHECK();
  return PP_OK;
}
