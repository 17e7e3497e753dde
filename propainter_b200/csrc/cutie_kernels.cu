// The web demo's Cutie mask tracker on sm_90a (web-demos/hugging_face/tracker): the fused top-k memory readout of the
// working memory, and the frame / label passes at the two ends of a tracking step.  The networks' convolutions stay
// cuDNN calls (propainter_b200/model/cutie.py).
#include <limits.h>
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
