// The web demo's Cutie mask tracker on sm_90a (web-demos/hugging_face/tracker): the fused top-k memory readout of the
// working memory, and the frame / label passes at the two ends of a tracking step.  The networks' convolutions stay
// cuDNN calls (propainter_b200/model/cutie.py).  And the tracking preview: the painted frames BaseTracker.track returns.
#include <limits.h>
#include "pp_elem.cuh"
#include "pp_topk.cuh"
#include "../../include/propainter_b200.h"

#define PP_LAUNCH_CHECK() do { if (cudaPeekAtLastError() != cudaSuccess) return PP_ERR_LAUNCH; } while (0)

static inline int pp_blocks(long n, int per) { return (int)((n + per - 1) / per); }

// ================================================================ fused top-k readout
// One block per RO_TQ query columns.  Phase 1: RO_S splits of RO_TQ threads each scan the memory in tiles of
// RO_S * RO_TT tokens (split s takes tokens [s * RO_TT, (s + 1) * RO_TT) of every tile), computing each similarity in
// fp32 on the CUDA cores from the exact form -sum_c qe_c (mk_c - qk_c)^2 and keeping a running top-k per thread.
// Phase 2: the RO_S lists of a column are merged by rank (pp_topk_rank), the softmax runs over the k survivors.
// Phase 3: each warp gathers the selected value rows of every object, 256 channels per query, into pixel-major out.
#define RO_TQ 16
#define RO_S 8
#define RO_TT 16
#define RO_TILE (RO_S * RO_TT)
#define RO_CK 64
#define RO_CV 256
#define RO_THREADS (RO_TQ * RO_S)
#define RO_MK_LD (RO_CK + 4)                      // rows stay 16-byte aligned for the float4 reads

struct RoSmemScan {
  __align__(16) float mk[RO_TILE * RO_MK_LD];
  float ms[RO_TILE];
};
struct RoSmemMerge {
  float cv[RO_TQ * RO_S * PP_TOPK_MAX];
  int ci[RO_TQ * RO_S * PP_TOPK_MAX];
};

__global__ void __launch_bounds__(RO_THREADS) k_cutie_topk_readout(
    const float* __restrict__ mem_key, const float* __restrict__ mem_shrink, const float* __restrict__ mem_value,
    long value_obj_stride, int N, int frame_tokens, int fifo_head, int fifo_cap, const float* __restrict__ qk,
    const float* __restrict__ qe, int HW, int num_objects, int top_k, float* __restrict__ out, int* __restrict__ sel_idx,
    float* __restrict__ sel_w) {
  __shared__ union { RoSmemScan scan; RoSmemMerge merge; } sm;
  __shared__ float q_k[RO_CK * RO_TQ], q_e[RO_CK * RO_TQ];
  __shared__ float s_v[RO_TQ * PP_TOPK_MAX];
  __shared__ int s_i[RO_TQ * PP_TOPK_MAX];

  const int t = threadIdx.x, q = t % RO_TQ, s = t / RO_TQ;
  const int q0 = blockIdx.x * RO_TQ;
  const int keff = top_k < N ? top_k : N;                  // fewer than k memory tokens: keep them all
  for (int i = t; i < RO_CK * RO_TQ; i += RO_THREADS) {
    const int c = i / RO_TQ, qq = i % RO_TQ;
    const bool in = q0 + qq < HW;
    q_k[i] = in ? qk[(long)c * HW + q0 + qq] : 0.f;
    q_e[i] = in ? qe[(long)c * HW + q0 + qq] : 0.f;
  }

  float val[PP_TOPK_MAX];
  int idx[PP_TOPK_MAX];
  int cnt = 0, worst = 0;
  for (int n0 = 0; n0 < N; n0 += RO_TILE) {
    __syncthreads();
    for (int i = t; i < RO_TILE * RO_CK / 4; i += RO_THREADS) {
      const int r = i / (RO_CK / 4), c = (i % (RO_CK / 4)) * 4, n = n0 + r;
      const float4 v = n < N ? *reinterpret_cast<const float4*>(mem_key + pp_ring_row(n, frame_tokens, fifo_head, fifo_cap) * RO_CK + c)
                             : make_float4(0.f, 0.f, 0.f, 0.f);
      *reinterpret_cast<float4*>(sm.scan.mk + r * RO_MK_LD + c) = v;
    }
    if (t < RO_TILE) {
      const int n = n0 + t;
      sm.scan.ms[t] = n < N ? mem_shrink[pp_ring_row(n, frame_tokens, fifo_head, fifo_cap)] : 0.f;
    }
    __syncthreads();
    float acc[RO_TT];
#pragma unroll
    for (int j = 0; j < RO_TT; ++j) acc[j] = 0.f;
    // four channels per step: one float4 of each memory key (the two splits of a warp read two rows: no conflict)
    const float* mk = sm.scan.mk + s * RO_TT * RO_MK_LD;
    for (int c = 0; c < RO_CK; c += 4) {
      float kq[4], eq[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        kq[i] = q_k[(c + i) * RO_TQ + q];
        eq[i] = q_e[(c + i) * RO_TQ + q];
      }
#pragma unroll
      for (int j = 0; j < RO_TT; ++j) {
        const float4 m = *reinterpret_cast<const float4*>(mk + j * RO_MK_LD + c);
        float d = m.x - kq[0];
        acc[j] = fmaf(eq[0] * d, d, acc[j]);
        d = m.y - kq[1];
        acc[j] = fmaf(eq[1] * d, d, acc[j]);
        d = m.z - kq[2];
        acc[j] = fmaf(eq[2] * d, d, acc[j]);
        d = m.w - kq[3];
        acc[j] = fmaf(eq[3] * d, d, acc[j]);
      }
    }
    if (q0 + q < HW) {
#pragma unroll
      for (int j = 0; j < RO_TT; ++j) {
        const int n = n0 + s * RO_TT + j;
        if (n < N) pp_topk_push(val, idx, cnt, worst, keff, pp_cutie_similarity(acc[j], sm.scan.ms[s * RO_TT + j]), n);
      }
    }
  }
  __syncthreads();                                         // the scan tiles become the merge lists
  {
    float* cv = sm.merge.cv + (q * RO_S + s) * PP_TOPK_MAX;
    int* ci = sm.merge.ci + (q * RO_S + s) * PP_TOPK_MAX;
    for (int j = 0; j < PP_TOPK_MAX; ++j) {
      cv[j] = j < cnt ? val[j] : 0.f;
      ci[j] = j < cnt ? idx[j] : -1;
    }
  }
  __syncthreads();
  for (int e = t; e < RO_TQ * RO_S * PP_TOPK_MAX; e += RO_THREADS) {
    const int qq = e / (RO_S * PP_TOPK_MAX), c = e % (RO_S * PP_TOPK_MAX);
    const float* cv = sm.merge.cv + qq * RO_S * PP_TOPK_MAX;
    const int* ci = sm.merge.ci + qq * RO_S * PP_TOPK_MAX;
    if (ci[c] < 0) continue;
    const int r = pp_topk_rank(cv, ci, RO_S * PP_TOPK_MAX, c);
    if (r < keff) {
      s_v[qq * PP_TOPK_MAX + r] = cv[c];
      s_i[qq * PP_TOPK_MAX + r] = ci[c];
    }
  }
  __syncthreads();
  if (t < RO_TQ) {
    // softmax over the survivors, shifted by their maximum (the reference exponentiates the raw values)
    float* v = s_v + t * PP_TOPK_MAX;
    const int* ix = s_i + t * PP_TOPK_MAX;
    int kq = q0 + t < HW ? keff : 0;
    if (kq > 0 && !(v[0] == v[0])) kq = 0;                  // every similarity of the column was NaN
    const float m = kq > 0 ? v[0] : 0.f;
    float sum = 0.f;
    for (int j = 0; j < kq; ++j) {
      v[j] = expf(v[j] - m);
      sum += v[j];
    }
    for (int j = 0; j < kq; ++j) v[j] = v[j] / sum;
    if (q0 + t < HW && sel_idx != nullptr) {
      for (int j = 0; j < top_k; ++j) {
        sel_idx[(long)(q0 + t) * top_k + j] = j < kq ? ix[j] : -1;
        sel_w[(long)(q0 + t) * top_k + j] = j < kq ? v[j] : 0.f;
      }
    }
    if (kq == 0)
      for (int j = 0; j < keff; ++j) v[j] = 0.f;
  }
  __syncthreads();
  const int warp = t / 32, lane = t % 32;
  for (int qq = warp; qq < RO_TQ; qq += RO_THREADS / 32) {
    const int qg = q0 + qq;
    if (qg >= HW) continue;
    for (int o = 0; o < num_objects; ++o) {
      const float* vo = mem_value + (long)o * value_obj_stride;
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
      for (int j = 0; j < keff; ++j) {
        const float w = s_v[qq * PP_TOPK_MAX + j];
        const int n = s_i[qq * PP_TOPK_MAX + j];
        if (n < 0) continue;
        const float* row = vo + pp_ring_row(n, frame_tokens, fifo_head, fifo_cap) * RO_CV;
        const float4 x = *reinterpret_cast<const float4*>(row + lane * 4);
        const float4 y = *reinterpret_cast<const float4*>(row + 128 + lane * 4);
        a.x = fmaf(w, x.x, a.x); a.y = fmaf(w, x.y, a.y); a.z = fmaf(w, x.z, a.z); a.w = fmaf(w, x.w, a.w);
        b.x = fmaf(w, y.x, b.x); b.y = fmaf(w, y.y, b.y); b.z = fmaf(w, y.z, b.z); b.w = fmaf(w, y.w, b.w);
      }
      float* po = out + ((long)o * HW + qg) * RO_CV;
      *reinterpret_cast<float4*>(po + lane * 4) = a;
      *reinterpret_cast<float4*>(po + 128 + lane * 4) = b;
    }
  }
}

// replaces get_similarity + do_softmax(top_k) + the dense bmm of MemoryManager.read / _readout
// (tracker/inference/memory_manager.py:160-187,68-79; tracker/model/utils/memory_utils.py:6-73)
extern "C" int pp_cutie_topk_readout(const float* mem_key, const float* mem_shrink, const float* mem_value, long value_obj_stride,
                                     int n_frames, int fifo_head, int fifo_cap, const float* qk, const float* qe, int HW,
                                     int num_objects, int top_k, float* out, int* sel_idx, float* sel_w, cudaStream_t stream) {
  if (HW < 1 || n_frames < 1 || fifo_cap < 0 || n_frames > 1 + fifo_cap || num_objects < 0 || top_k < 1 ||
      top_k > PP_TOPK_MAX || fifo_head < 0 || (fifo_cap > 0 && fifo_head >= fifo_cap))
    return PP_ERR_SHAPE;
  if ((long)n_frames * HW > INT_MAX / 2) return PP_ERR_SHAPE;
  if (((uintptr_t)mem_key & 15) || ((uintptr_t)mem_value & 15) || ((uintptr_t)out & 15) || (value_obj_stride & 3))
    return PP_ERR_ALIGN;
  if ((sel_idx == nullptr) != (sel_w == nullptr)) return PP_ERR_SHAPE;
  k_cutie_topk_readout<<<pp_blocks(HW, RO_TQ), RO_THREADS, 0, stream>>>(
      mem_key, mem_shrink, mem_value, value_obj_stride, n_frames * HW, HW, fifo_head, fifo_cap > 0 ? fifo_cap : 1, qk, qe, HW,
      num_objects, top_k, out, sel_idx, sel_w);
  PP_LAUNCH_CHECK();
  return PP_OK;
}

// ================================================================ frame in
// image_to_torch (/ 255, base_tracker.py:46-51), pad_divide_by(image, 16) (tensor_utils.py:6-21, zeros) and the
// normalisation of encode_image (cutie.py:59-62), in that order: the padding is normalised too.
__global__ void __launch_bounds__(256) k_cutie_frame_in(const uint8_t* __restrict__ frame, float* __restrict__ out, int H, int W,
                                                        int Hp, int Wp, int top, int left) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)Hp * Wp) return;
  const int x = (int)(i % Wp), y = (int)(i / Wp);
  const int ys = y - top, xs = x - left;
  const bool in = ys >= 0 && ys < H && xs >= 0 && xs < W;
  const float mean[3] = {0.485f, 0.456f, 0.406f}, std_[3] = {0.229f, 0.224f, 0.225f};
  for (int c = 0; c < 3; ++c) {
    const float v = in ? PP_DIV((float)frame[((long)ys * W + xs) * 3 + c], 255.0f) : 0.0f;
    out[(long)c * Hp * Wp + i] = PP_DIV(PP_SUB(v, mean[c]), std_[c]);
  }
}

extern "C" int pp_cutie_frame_in(const uint8_t* frame, float* out, int H, int W, cudaStream_t stream) {
  if (H < 1 || W < 1) return PP_ERR_SHAPE;
  const int Hp = (H + 15) / 16 * 16, Wp = (W + 15) / 16 * 16;
  const long n = (long)Hp * Wp;
  k_cutie_frame_in<<<pp_blocks(n, 256), 256, 0, stream>>>(frame, out, H, W, Hp, Wp, (Hp - H) / 2, (Wp - W) / 2);
  PP_LAUNCH_CHECK();
  return PP_OK;
}

// ================================================================ labels out
// torch.argmax over the probability channels (first maximum; NaN counts as the maximum, as in ATen), unpad
// (tensor_utils.py:24-42) and MaskMapper's remapping back to the user's ids (base_tracker.py:82-87): lut[channel].
__global__ void __launch_bounds__(256) k_cutie_labels(const float* __restrict__ prob, int K, int Hp, int Wp, int top, int left,
                                                      const uint8_t* __restrict__ lut, uint8_t* __restrict__ out, int H, int W) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)H * W) return;
  const int x = (int)(i % W), y = (int)(i / W);
  const long p = (long)(y + top) * Wp + x + left, plane = (long)Hp * Wp;
  float best = prob[p];
  int arg = 0;
  for (int k = 1; k < K && best == best; ++k) {
    const float v = prob[k * plane + p];
    if (v > best || !(v == v)) {
      best = v;
      arg = k;
    }
  }
  out[i] = lut[arg];
}

extern "C" int pp_cutie_labels(const float* prob, int K, const uint8_t* lut, uint8_t* out, int H, int W, cudaStream_t stream) {
  if (K < 1 || K > 256 || H < 1 || W < 1) return PP_ERR_SHAPE;
  const int Hp = (H + 15) / 16 * 16, Wp = (W + 15) / 16 * 16;
  const long n = (long)H * W;
  k_cutie_labels<<<pp_blocks(n, 256), 256, 0, stream>>>(prob, K, Hp, Wp, (Hp - H) / 2, (Wp - W) / 2, lut, out, H, W);
  PP_LAUNCH_CHECK();
  return PP_OK;
}

// ================================================================ tracking preview
// BaseTracker.track's painter loop (base_tracker.py:90-95) over a whole clip, from the rules of pp_elem.cuh.  Pass 1
// finds the per-(frame, object) maxima M: k_mask_paint_partial takes, per 32 x 32 tile, the maximum of v for each id of
// pp_paint_candidates (none in most frames: then the block returns at once), k_mask_paint_maxima reduces the tiles and
// sets M = 3 for every other id.  Pass 2 (k_mask_paint_u8) paints each pixel from its 7x7 label window.  Each block
// stages its tile's labels with a 3-pixel halo in shared memory, -1 outside the frame.  Maxima in a fixed tree, no
// atomics: the same bits on every run.
#define MP_TILE 32
#define MP_ROWS 8                                  // 32 x 8 threads, 4 rows of the tile each
#define MP_THREADS (MP_TILE * MP_ROWS)
#define MP_LD (MP_TILE + 6)
#define MP_CANDS 16                                // >= the 11 ids that can reach pixel (0, 0)

static inline long mp_tiles(int H, int W) { return (long)((H + MP_TILE - 1) / MP_TILE) * ((W + MP_TILE - 1) / MP_TILE); }

__device__ void mp_stage(const uint8_t* __restrict__ lab, int H, int W, int y0, int x0, int* s) {
  for (int i = threadIdx.y * MP_TILE + threadIdx.x; i < MP_LD * MP_LD; i += MP_THREADS) {
    const int y = y0 - 3 + i / MP_LD, x = x0 - 3 + i % MP_LD;
    s[i] = (y >= 0 && y < H && x >= 0 && x < W) ? lab[(long)y * W + x] : -1;
  }
}

// pp_paint_candidates of one frame's pixel (0, 0), read from global memory by one thread
__device__ int mp_candidates(const uint8_t* __restrict__ lab, int H, int W, int* out) {
  int w[49];
#pragma unroll
  for (int i = 0; i < 49; ++i) {
    const int y = i / 7 - 3, x = i % 7 - 3;
    w[i] = (y >= 0 && y < H && x >= 0 && x < W) ? lab[(long)y * W + x] : -1;
  }
  return pp_paint_candidates(w + 24, 7, out);
}

// maximum over the block's threads, result valid in thread 0; red holds MP_THREADS / 32 floats
__device__ float mp_block_max(float v, float* red) {
  const int t = threadIdx.y * MP_TILE + threadIdx.x;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  if ((t & 31) == 0) red[t >> 5] = v;
  __syncthreads();
  if (t == 0)
    for (int i = 1; i < MP_THREADS / 32; ++i) v = fmaxf(v, red[i]);
  __syncthreads();
  return v;
}

__global__ void __launch_bounds__(MP_THREADS) k_mask_paint_partial(const uint8_t* __restrict__ labels, int H, int W, int tiles_x,
                                                                   long ntiles, float* __restrict__ partial) {
  __shared__ int s_lab[MP_LD * MP_LD];
  __shared__ int s_cand[MP_CANDS], s_n;
  __shared__ float s_red[MP_THREADS / 32];
  const int f = blockIdx.y, t = threadIdx.y * MP_TILE + threadIdx.x;
  const uint8_t* lab = labels + (long)f * H * W;
  if (t == 0) s_n = mp_candidates(lab, H, W, s_cand);
  __syncthreads();
  const int n = s_n;
  if (n == 0) return;
  const int y0 = (blockIdx.x / tiles_x) * MP_TILE, x0 = (blockIdx.x % tiles_x) * MP_TILE;
  mp_stage(lab, H, W, y0, x0, s_lab);
  __syncthreads();
  for (int j = 0; j < n; ++j) {
    float m = 0.0f;
    if (x0 + (int)threadIdx.x < W)
      for (int r = threadIdx.y; r < MP_TILE && y0 + r < H; r += MP_ROWS)
        m = fmaxf(m, pp_paint_dist(s_lab + (r + 3) * MP_LD + threadIdx.x + 3, MP_LD, s_cand[j]));
    m = mp_block_max(m, s_red);
    if (t == 0) partial[((long)f * ntiles + blockIdx.x) * MP_CANDS + j] = m;
  }
}

__global__ void __launch_bounds__(MP_THREADS) k_mask_paint_maxima(const uint8_t* __restrict__ labels, int H, int W, long ntiles,
                                                                  const float* __restrict__ partial, float* __restrict__ maxima) {
  __shared__ int s_cand[MP_CANDS], s_n;
  __shared__ float s_red[MP_THREADS / 32];
  const int f = blockIdx.x, t = threadIdx.y * MP_TILE + threadIdx.x;
  if (t == 0) s_n = mp_candidates(labels + (long)f * H * W, H, W, s_cand);
  maxima[(long)f * 256 + t] = 3.0f;
  __syncthreads();
  for (int j = 0; j < s_n; ++j) {
    float m = 0.0f;
    for (long i = t; i < ntiles; i += MP_THREADS) m = fmaxf(m, partial[((long)f * ntiles + i) * MP_CANDS + j]);
    m = mp_block_max(m, s_red);
    if (t == 0) maxima[(long)f * 256 + s_cand[j]] = m;
  }
}

// frames and out may be the same buffer: each thread reads a pixel before it writes it, and no other thread touches it
__global__ void __launch_bounds__(MP_THREADS) k_mask_paint_u8(const uint8_t* frames, const uint8_t* __restrict__ labels,
                                                              const uint8_t* __restrict__ palette, int n_colors, double alpha,
                                                              double oma, const float* __restrict__ maxima, uint8_t* out, int H,
                                                              int W, int tiles_x) {
  __shared__ int s_lab[MP_LD * MP_LD];
  __shared__ float s_max[256];
  __shared__ uint8_t s_pal[257 * 3];
  const int f = blockIdx.y, t = threadIdx.y * MP_TILE + threadIdx.x;
  const long HW = (long)H * W;
  const int y0 = (blockIdx.x / tiles_x) * MP_TILE, x0 = (blockIdx.x % tiles_x) * MP_TILE;
  mp_stage(labels + f * HW, H, W, y0, x0, s_lab);
  s_max[t] = maxima[(long)f * 256 + t];
  for (int i = t; i < n_colors * 3; i += MP_THREADS) s_pal[i] = palette[i];
  __syncthreads();
  const int x = x0 + threadIdx.x;
  if (x >= W) return;
  for (int r = threadIdx.y; r < MP_TILE && y0 + r < H; r += MP_ROWS) {
    const long p = (f * HW + (long)(y0 + r) * W + x) * 3;
    uint8_t rgb[3] = {frames[p], frames[p + 1], frames[p + 2]};
    const int* c = s_lab + (r + 3) * MP_LD + threadIdx.x + 3;
    int w[49];                                     // the window in registers (only the reached entries are read)
#pragma unroll
    for (int i = 0; i < 49; ++i) w[i] = c[(i / 7 - 3) * MP_LD + i % 7 - 3];
    pp_paint_pixel(w + 24, 7, s_max, s_pal, n_colors, alpha, oma, rgb);
    out[p] = rgb[0];
    out[p + 1] = rgb[1];
    out[p + 2] = rgb[2];
  }
}

extern "C" size_t pp_mask_paint_workspace_bytes(int T, int H, int W) {
  if (T < 1 || H < 1 || W < 1) return 0;
  return (size_t)T * 256 * sizeof(float) + (size_t)T * mp_tiles(H, W) * MP_CANDS * sizeof(float);
}

extern "C" int pp_mask_paint_u8(const uint8_t* frames, const uint8_t* labels, const uint8_t* palette, int n_colors,
                                const double* alpha, uint8_t* out, int T, int H, int W, void* workspace, size_t workspace_bytes,
                                cudaStream_t stream) {
  if (T < 1 || T > 65535 || H < 1 || W < 1 || n_colors < 2 || alpha == nullptr) return PP_ERR_SHAPE;
  const long ntiles = mp_tiles(H, W);
  if (ntiles > INT_MAX) return PP_ERR_SHAPE;
  if (workspace == nullptr || workspace_bytes < pp_mask_paint_workspace_bytes(T, H, W)) return PP_ERR_WORKSPACE;
  if ((uintptr_t)workspace & 3) return PP_ERR_ALIGN;
  float* maxima = static_cast<float*>(workspace);
  float* partial = maxima + (size_t)T * 256;
  const int tiles_x = (W + MP_TILE - 1) / MP_TILE;
  const dim3 block(MP_TILE, MP_ROWS), grid((unsigned)ntiles, T);
  k_mask_paint_partial<<<grid, block, 0, stream>>>(labels, H, W, tiles_x, ntiles, partial);
  PP_LAUNCH_CHECK();
  k_mask_paint_maxima<<<T, block, 0, stream>>>(labels, H, W, ntiles, partial, maxima);
  PP_LAUNCH_CHECK();
  k_mask_paint_u8<<<grid, block, 0, stream>>>(frames, labels, palette, n_colors < 257 ? n_colors : 257, alpha[0], alpha[1],
                                              maxima, out, H, W, tiles_x);
  PP_LAUNCH_CHECK();
  return PP_OK;
}
