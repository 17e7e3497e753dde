// Per-element rules of the Cutie memory readout (pp_cutie_topk_readout): the running top-k of one query column and the
// order that breaks ties.  PP_HD: also compiled by tests/hostsim/hostsim_cutie.cpp.
//
// do_softmax(similarity, top_k) (tracker/model/utils/memory_utils.py:45-73) keeps the k largest similarities of each
// query column with torch.topk, whose choice among equal values is unspecified.  Here the order is total: (s, n) ranks
// above (v, m) when s > v, or s == v and n < m, so of equal similarities the earlier memory token (lower logical index:
// the permanent frame first, then the FIFO frames oldest first) is kept.  NaN similarities never enter a list.
#pragma once
#include "pp_common.cuh"

#define PP_TOPK_MAX 32

PP_HD bool pp_topk_beats(float s, int n, float v, int m) { return s > v || (s == v && n < m); }

// position of the lowest-ranked entry of a full list
PP_HD int pp_topk_worst(const float* val, const int* idx, int k) {
  int w = 0;
  for (int i = 1; i < k; ++i)
    if (pp_topk_beats(val[w], idx[w], val[i], idx[i])) w = i;
  return w;
}

// offer (s, n) to the unordered list val/idx of capacity k holding cnt entries; `worst` is the lowest-ranked position
// once the list is full.  Candidates arrive in increasing n within one list.
PP_HD void pp_topk_push(float* val, int* idx, int& cnt, int& worst, int k, float s, int n) {
  if (!(s == s)) return;
  if (cnt < k) {
    val[cnt] = s;
    idx[cnt] = n;
    if (++cnt == k) worst = pp_topk_worst(val, idx, k);
    return;
  }
  if (!pp_topk_beats(s, n, val[worst], idx[worst])) return;
  val[worst] = s;
  idx[worst] = n;
  worst = pp_topk_worst(val, idx, k);
}

// rank of candidate c among the `n` candidates (v, i) with i >= 0 (i < 0 marks an empty slot): how many of them beat it.
// The union of per-split top-k lists holds the global top-k, and the rank is its place in the merged list.
PP_HD int pp_topk_rank(const float* v, const int* i, int n, int c) {
  int r = 0;
  for (int d = 0; d < n; ++d)
    if (i[d] >= 0 && pp_topk_beats(v[d], i[d], v[c], i[c])) ++r;
  return r;
}

// the anisotropic-L2 similarity of get_similarity (memory_utils.py:6-42) from its accumulated sum acc = sum_c qe_c *
// (mk_c - qk_c)^2 = a_sq - 2ab + b_sq: (-acc) * shrinkage / sqrt(64), the division by 8 being exact
PP_HD float pp_cutie_similarity(float acc, float shrinkage) { return PP_MUL(PP_MUL(-acc, shrinkage), 0.125f); }

// logical memory token n -> row of the ring buffers: frame 0 is the permanent slot 0; logical frame f >= 1 is FIFO slot
// 1 + (head + f - 1) % fifo_cap, head being the slot of the oldest FIFO frame
PP_HD long pp_ring_row(int n, int frame_tokens, int fifo_head, int fifo_cap) {
  const int f = n / frame_tokens, o = n - f * frame_tokens;
  const int slot = f == 0 ? 0 : 1 + (fifo_head + f - 1) % fifo_cap;
  return (long)slot * frame_tokens + o;
}
