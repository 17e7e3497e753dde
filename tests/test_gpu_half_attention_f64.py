"""The fp16 window-attention kernels (pp_sparse_window_attn_f16: f16 wgmma for masked windows, mma.sync m16n8k16 for unmasked
ones) against a float64 recomputation on the same fp16 inputs.

The TF32 kernels run on the same inputs widened to fp32 and their output is rounded to fp16, the form in which the
half-operand proj Linear would consume it; the fp16 kernels' error must stay within 1.5x of that.  Cases cover ragged query
tiles (t*45 not a multiple of 128), ragged key tiles, an empty key set (nkf = 0), t = 1, all-masked and none-masked flags,
the padded token grid and the C2 window shape.  `out` is a view of a wider NaN-filled buffer: the columns beyond it must stay
untouched.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _ref(qkv, pool, ktab, flags, t, kf_start, kf_step, C=512, WN=45):
    """float64 SparseWindowAttention between q/k/v and proj on the index tables"""
    q, k, v = qkv[..., :C].double(), qkv[..., C:2 * C].double(), qkv[..., 2 * C:].double()
    pk, pv = pool[..., :C].double(), pool[..., C:].double()
    out = torch.zeros(t, qkv.shape[1], C, dtype=torch.float64, device=DEV)
    kf = list(range(kf_start, t, kf_step))
    scale = 1.0 / math.sqrt(128)
    for wi in range(ktab.shape[0]):
        own, allk = ktab[wi, :WN].long(), ktab[wi].long()
        for hd in range(C // 128):
            sl = slice(hd * 128, (hd + 1) * 128)
            qw = q[:, own, sl]                                                   # [t, WN, 128]
            if flags[wi] != 0:
                if not kf:
                    continue
                K = torch.cat([torch.cat([k[f][allk][:, sl], pk[f][:, sl]], 0) for f in kf], 0)
                V = torch.cat([torch.cat([v[f][allk][:, sl], pv[f][:, sl]], 0) for f in kf], 0)
                out[:, own, sl] = torch.softmax(qw @ K.t() * scale, -1) @ V
            else:
                a = torch.softmax(qw @ k[:, own, sl].transpose(1, 2) * scale, -1)
                out[:, own, sl] = a @ v[:, own, sl]
    return out


def _case(H2, W2, t, kf_start, kf_step, flag_rule, seed):
    from propainter_b200.window_index import window_key_table
    gen = torch.Generator(device=DEV).manual_seed(seed)
    ktab = torch.from_numpy(window_key_table(H2, W2)).to(DEV)
    nwin, NT, NP = ktab.shape[0], H2 * W2, (H2 // 4) * (W2 // 4)
    flags = torch.tensor([flag_rule(i) for i in range(nwin)], dtype=torch.int32, device=DEV)
    qkv = (torch.randn(t, NT, 1536, device=DEV, generator=gen) * 1.5).half()
    pool = (torch.randn(t, NP, 1024, device=DEV, generator=gen) * 1.5).half()
    return qkv, pool, ktab, flags


CASES = {   # (padded token grid, t, key frames, flags)
    "c2": ((20, 36), 18, (0, 2), lambda i: int(i % 3 == 0)),
    "c2_odd_layer": ((20, 36), 17, (1, 2), lambda i: int(i % 2 == 0)),
    "padded_grid": ((15, 18), 5, (0, 2), lambda i: int(i % 2 == 1)),
    "all_masked": ((10, 18), 3, (0, 2), lambda i: 1),
    "none_masked": ((10, 18), 7, (0, 2), lambda i: 0),
    "t1": ((10, 18), 1, (0, 2), lambda i: int(i == 0)),
    "nkf0": ((10, 18), 1, (1, 2), lambda i: int(i % 2 == 0)),
}


@pytest.mark.parametrize("name", list(CASES))
def test_attention_f16_vs_float64(name):
    from propainter_b200 import ops
    (H2, W2), t, (ks, kstep), rule = CASES[name]
    qkv, pool, ktab, flags = _case(H2, W2, t, ks, kstep, rule, seed=len(name))
    NT = H2 * W2
    ref = _ref(qkv, pool, ktab, flags, t, ks, kstep)
    buf = torch.full((t, NT, 520), float("nan"), device=DEV, dtype=torch.float16)
    o16 = ops.sparse_window_attn(qkv, pool, ktab, flags, t, NT, ks, kstep, out=buf[..., :512])
    o32 = ops.sparse_window_attn(qkv.float(), pool.float(), ktab, flags, t, NT, ks, kstep).half()
    torch.cuda.synchronize()
    assert torch.isnan(buf[..., 512:]).all()
    scale = ref.abs().max().item()
    e16 = (o16.double() - ref).abs().max().item() / scale
    e32 = (o32.double() - ref).abs().max().item() / scale
    print(f"{name}: |ref|max {scale:.3f}  fp16 kernels {e16:.2e}  TF32 kernels (out rounded to fp16) {e32:.2e}")
    assert bool(torch.isfinite(o16).all())
    assert e16 < 2e-3 and e16 <= 1.5 * e32 + 1e-6


def test_attention_f16_refuses_misaligned():
    from propainter_b200 import ops
    qkv, pool, ktab, flags = _case(10, 18, 2, 0, 2, lambda i: i % 2, seed=0)
    flat = torch.zeros(2 * 180 * 1536 + 8, device=DEV, dtype=torch.float16)
    with pytest.raises(RuntimeError, match="misaligned"):
        ops.sparse_window_attn(flat[2:2 + 2 * 180 * 1536].view(2, 180, 1536), pool, ktab, flags, 2, 180, 0, 2)
