"""oracle/attn_table_ref (the float64 restatement of the sparse window attention at the kernel's interface: q/k/v rows,
pooled k/v rows, key table, flags, key frames) equals generator_ref.window_attention, which builds the same key sets with
torch.roll and window partitions.  CPU, float64: agreement to rounding pins the restatement before the GPU tests use it
as their reference."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import attn_table_ref, generator_ref
from propainter_b200.window_index import padded_grid, window_key_table

C = 512


def _inputs(gen, t, lt, fh, fw, masked_cols):
    sd = {}
    for n in ("query", "key", "value"):
        sd[f"a.{n}.weight"] = torch.randn(C, C, generator=gen, dtype=torch.float64) / math.sqrt(C)
        sd[f"a.{n}.bias"] = torch.randn(C, generator=gen, dtype=torch.float64) * 0.1
    sd["a.proj.weight"] = torch.eye(C, dtype=torch.float64)
    sd["a.proj.bias"] = torch.zeros(C, dtype=torch.float64)
    sd["a.pool_layer.weight"] = torch.randn(C, 1, 4, 4, generator=gen, dtype=torch.float64) / 4
    sd["a.pool_layer.bias"] = torch.randn(C, generator=gen, dtype=torch.float64) * 0.1
    x = torch.randn(1, t, fh, fw, C, generator=gen, dtype=torch.float64)
    mask = torch.zeros(1, lt, fh, fw, 1, dtype=torch.float64)
    if masked_cols is not None:
        mask[:, :, 2:9, masked_cols[0]:masked_cols[1]] = 1
    return sd, x, mask


def _interface(sd, x, mask):
    """The kernel's operands, built as the model builds them: projections of the padded grid, pooled projections,
    key table, window flags."""
    _, t, fh, fw, _ = x.shape
    H2, W2 = padded_grid(fh, fw)
    xp = F.pad(x[0], (0, 0, 0, W2 - fw, 0, H2 - fh))
    wqkv = torch.cat([sd["a.query.weight"], sd["a.key.weight"], sd["a.value.weight"]], 0)
    bqkv = torch.cat([sd["a.query.bias"], sd["a.key.bias"], sd["a.value.bias"]], 0)
    qkv = F.linear(xp, wqkv, bqkv).view(t, H2 * W2, 3 * C)
    pooled = F.conv2d(xp.permute(0, 3, 1, 2), sd["a.pool_layer.weight"], sd["a.pool_layer.bias"], stride=4,
                      groups=C).permute(0, 2, 3, 1).reshape(t, -1, C)
    pool_kv = F.linear(pooled, wqkv[C:], bqkv[C:])
    mp = F.pad(mask[0, ..., 0], (0, W2 - fw, 0, H2 - fh))
    flags = (F.max_pool2d(mp[:, None], (5, 9), (5, 9)).view(mask.shape[1], -1).sum(0) > 0).int()
    return qkv, pool_kv, torch.from_numpy(window_key_table(H2, W2)), flags, (H2, W2)


@pytest.mark.parametrize("t,lt,fh,fw,masked_cols", [(4, 3, 20, 36, (10, 20)), (3, 2, 11, 11, (0, 5)), (1, 1, 11, 20, (3, 12))])
@pytest.mark.parametrize("layer", [0, 1])
def test_table_restatement_matches_window_attention(t, lt, fh, fw, masked_cols, layer):
    gen = torch.Generator().manual_seed(100 * t + fh + layer)
    sd, x, mask = _inputs(gen, t, lt, fh, fw, masked_cols)
    t_ind = torch.arange(layer % 2, t, 2)
    ref = generator_ref.window_attention(sd, "a", x, mask, t_ind)[0]
    qkv, pool_kv, ktab, flags, (H2, W2) = _interface(sd, x, mask)
    assert 0 < int(flags.sum()) < flags.numel()                              # both kinds of window take part
    full = attn_table_ref.window_attention_table(qkv, pool_kv, ktab, flags, t, 45, layer % 2, 2)
    got = full.view(t, H2, W2, C)[:, :fh, :fw]
    assert got.dtype == torch.float64
    err = (got - ref).abs().max().item()
    assert err < 1e-12 * ref.abs().max().item(), err
    masked_tok = ktab[flags.bool(), :45].reshape(-1).long()
    if len(t_ind) == 0:                                   # t = 1 on an odd layer: masked windows have no key frame -> zeros
        assert (full[:, masked_tok] == 0).all() and (full != 0).any()
    else:
        assert (full[:, masked_tok] != 0).all()
