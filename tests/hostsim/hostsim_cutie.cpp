// TEST HARNESS ONLY (never loaded by the product): host build of the Cutie readout's element rules from pp_topk.cuh --
// the running top-k with its tie order, the rank merge of the per-split lists and the ring-buffer row of a memory token
// -- so the CPU test-suite can check them against the oracle's selection rule.
#define PP_HOSTSIM 1
#include <cmath>
#include "../../propainter_b200/csrc/pp_topk.cuh"

extern "C" {

// the kernel's selection for one query column: `splits` lists, split s taking tokens [s*tt, (s+1)*tt) of every tile of
// splits*tt tokens, each a running top-k (keff = min(k, N)); then the rank merge.  sim [N] -> out_idx [keff] in rank
// order; returns keff.
int hs_topk_select(const float* sim, int N, int k, int splits, int tt, int* out_idx) {
  const int keff = k < N ? k : N;
  float cv[64 * PP_TOPK_MAX];
  int ci[64 * PP_TOPK_MAX];
  for (int s = 0; s < splits; ++s) {
    float val[PP_TOPK_MAX];
    int idx[PP_TOPK_MAX];
    int cnt = 0, worst = 0;
    for (int n0 = 0; n0 < N; n0 += splits * tt)
      for (int j = 0; j < tt; ++j) {
        const int n = n0 + s * tt + j;
        if (n < N) pp_topk_push(val, idx, cnt, worst, keff, sim[n], n);
      }
    for (int j = 0; j < PP_TOPK_MAX; ++j) {
      cv[s * PP_TOPK_MAX + j] = j < cnt ? val[j] : 0.f;
      ci[s * PP_TOPK_MAX + j] = j < cnt ? idx[j] : -1;
    }
  }
  for (int j = 0; j < keff; ++j) out_idx[j] = -1;
  for (int c = 0; c < splits * PP_TOPK_MAX; ++c) {
    if (ci[c] < 0) continue;
    const int r = pp_topk_rank(cv, ci, splits * PP_TOPK_MAX, c);
    if (r < keff) out_idx[r] = ci[c];
  }
  return keff;
}

float hs_similarity(float acc, float shrinkage) { return pp_cutie_similarity(acc, shrinkage); }
long hs_ring_row(int n, int frame_tokens, int fifo_head, int fifo_cap) { return pp_ring_row(n, frame_tokens, fifo_head, fifo_cap); }
}
