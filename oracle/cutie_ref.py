"""Plain-torch restatement of the Cutie working-memory read (web-demos/hugging_face/tracker/model/utils/memory_utils.py,
tracker/inference/memory_manager.py:160-187), over explicit tensors: the dense reference the fused top-k readout
(ops.cutie_topk_readout) is tested against.  ``dtype`` selects fp32 (the reference's arithmetic) or float64.

Shapes follow the reference: mk [B,64,N], ms [B,1,N], qk / qe [B,64,HW], values [B,objects,256,N]."""
import math

import torch


def get_similarity(mk, ms, qk, qe):
    """memory_utils.py:6-42 (with selection): (-a^2 + 2ab - b^2) * shrinkage / sqrt(CK) -> [B,N,HW]"""
    CK = mk.shape[1]
    mk = mk.flatten(start_dim=2)
    ms = ms.flatten(start_dim=1).unsqueeze(2)
    qk = qk.flatten(start_dim=2)
    qe = qe.flatten(start_dim=2)
    mk = mk.transpose(1, 2)
    a_sq = mk.pow(2) @ qe
    two_ab = 2 * (mk @ (qk * qe))
    b_sq = (qe * qk.pow(2)).sum(1, keepdim=True)
    return (-a_sq + two_ab - b_sq) * ms / math.sqrt(CK)


def do_softmax(similarity, top_k=None):
    """memory_utils.py:45-73 (not inplace, no usage): top-k softmax scattered into a dense [B,N,HW] affinity"""
    if top_k is not None:
        values, indices = torch.topk(similarity, k=top_k, dim=1)
        x_exp = values.exp()
        x_exp = x_exp / torch.sum(x_exp, dim=1, keepdim=True)
        return torch.zeros_like(similarity).scatter_(1, indices, x_exp)
    maxes = torch.max(similarity, dim=1, keepdim=True)[0]
    x_exp = torch.exp(similarity - maxes)
    return x_exp / torch.sum(x_exp, dim=1, keepdim=True)


def readout(affinity, v):
    """MemoryManager._readout (memory_manager.py:68-79): v [B,objects,C,N] @ affinity -> [B,objects,C,HW]"""
    bs, K, C, N = v.shape
    return (v.reshape(bs, K * C, N) @ affinity).view(bs, K, C, -1)


def memory_read(mk, ms, qk, qe, v, top_k=30, dtype=torch.float32):
    """the dense read of MemoryManager.read at top_k (N >= top_k as torch.topk requires)"""
    c = [t.to(dtype) for t in (mk, ms, qk, qe, v)]
    return readout(do_softmax(get_similarity(*c[:4]), top_k), c[4])


def readout_selected(mk, ms, qk, qe, v, sel_idx, dtype=torch.float64):
    """the read over a given selected set sel_idx [HW,k] (int, -1 = unused; batch 1): similarity of the selected tokens,
    softmax over them, weighted sum of their values -> [objects,C,HW].  With sel_idx from the kernel this isolates the
    arithmetic from the selection."""
    mk, ms, qk, qe, v = (t[0].to(dtype) for t in (mk, ms, qk, qe, v))
    HW, k = sel_idx.shape
    valid = sel_idx >= 0
    idx = sel_idx.clamp(min=0).long()
    m = mk[:, idx]                                                   # [64,HW,k]
    s = -(qe.unsqueeze(-1) * (m - qk.unsqueeze(-1)) ** 2).sum(0) * ms[0, idx] / math.sqrt(mk.shape[0])
    s = s.masked_fill(~valid, float("-inf"))
    w = torch.softmax(s, dim=1)                                      # [HW,k]
    return torch.einsum("hk,ochk->och", w, v[:, :, idx])


def topk_order(similarity, top_k):
    """the kernel's selection rule on a [N,HW] similarity (float64 or fp32): per column the min(top_k, N) largest, ties
    to the lower token index, in descending order -> indices [HW,min(top_k,N)]"""
    N, HW = similarity.shape
    k = min(top_k, N)
    # sort by (-value, index): a stable sort of the values in descending order keeps the lower index first among ties
    order = torch.sort(similarity.t(), dim=1, descending=True, stable=True).indices
    return order[:, :k]
