"""Oracle (test infrastructure): the masked sparse window attention at the interface of pp_sparse_window_attn, in float64.

Where generator_ref.window_attention starts from the token map and builds the rolled / pooled key sets with torch.roll
and window partitions (sparse_transformer.py:177-275), this restatement takes exactly what the kernel takes: the q | k | v
projections of every token of the padded grid, the k | v projections of the pooled tokens, the per-window key table
(window_index.window_key_table, or any other table), the window flags and the key-frame range.  So a kernel test can
use tables, window sizes and key frames the model never produces, and still have a plain reference.

  * A masked window (flag != 0) owns the tokens key_tok[w, :WN]; each of its t*WN queries attends, for every frame f of
    range(kf_start, t, kf_step), to the tokens key_tok[w, :] of frame f and then to the pooled tokens of frame f.  With no
    key frame the key set is empty and the window's outputs are zeros (softmax over an empty dim, then the matmul).
  * An unmasked window attends per frame to its own WN tokens of the same frame.
Heads of 128 channels, scale 1/sqrt(128).  Tokens that no window owns are left at zero.
"""
import math

import torch

HEAD_DIM = 128


def _attend(q, k, v):
    """q [..., nq, C], k / v [..., nk, C] -> [..., nq, C], softmax(q k^T / sqrt(128)) v per 128-channel head."""
    C = q.shape[-1]
    nh = C // HEAD_DIM
    sh = lambda z: z.unflatten(-1, (nh, HEAD_DIM)).transpose(-3, -2)           # [..., heads, n, 128]
    a = torch.softmax(sh(q) @ sh(k).transpose(-2, -1) / math.sqrt(HEAD_DIM), dim=-1)
    return (a @ sh(v)).transpose(-3, -2).flatten(-2)


def masked_keys(qkv, pool_kv, tab, kfs):
    """Key and value rows [nkeys, C] of a masked window with token table `tab` over the key frames `kfs`, in the kernel's
    key order: per key frame the table tokens, then the pooled tokens."""
    C = qkv.shape[-1] // 3
    K = torch.cat([torch.cat([qkv[f, tab, C:2 * C], pool_kv[f, :, :C]], 0) for f in kfs], 0)
    V = torch.cat([torch.cat([qkv[f, tab, 2 * C:], pool_kv[f, :, C:]], 0) for f in kfs], 0)
    return K, V


def window_attention_table(qkv, pool_kv, key_tok, flags, t, WN, kf_start, kf_step):
    """qkv [t,NT,3C]; pool_kv [t,NP,2C]; key_tok int [nwin,NKO]; flags [nwin] -> out [t,NT,C] float64."""
    qkv, pool = qkv.double(), pool_kv.double()
    C = qkv.shape[-1] // 3
    q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
    key_tok, flags = key_tok.long(), flags.tolist()
    kfs = list(range(kf_start, t, kf_step))
    out = torch.zeros(t, qkv.shape[1], C, dtype=torch.float64, device=qkv.device)
    for w, flag in enumerate(flags):
        own = key_tok[w, :WN]
        if not flag:
            out[:, own] = _attend(q[:, own], k[:, own], v[:, own])
        elif kfs:
            K, V = masked_keys(qkv, pool, key_tok[w], kfs)
            out[:, own] = _attend(q[:, own].reshape(t * WN, C), K, V).view(t, WN, C)
    return out
