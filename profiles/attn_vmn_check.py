"""Checks + times the wgmma attention kernel of whichever library build PROPAINTER_B200_LIB points at against the
mma.sync kernel (same inputs as ncu_targets.py):  python profiles/attn_vmn_check.py"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from propainter_b200 import _lib, ops  # noqa: E402
from propainter_b200.window_index import window_key_table  # noqa: E402

dev = "cuda"
torch.manual_seed(0)
t, H2, W2, C = 18, 20, 36, 512
qkv = torch.randn(t, H2 * W2, 3 * C, device=dev)
pool = torch.randn(t, 45, 2 * C, device=dev)
ktab = torch.from_numpy(window_key_table(H2, W2)).to(dev)
print("library:", _lib.LIB_PATH)
for nm, masked in (("5of16", [5, 6, 9, 10, 11]), ("16of16", list(range(16)))):
    flags = torch.zeros(16, dtype=torch.int32, device=dev)
    flags[masked] = 1
    a = ops.sparse_window_attn(qkv, pool, ktab, flags, t, H2 * W2, 0, 2, impl="umma")
    b = ops.sparse_window_attn(qkv, pool, ktab, flags, t, H2 * W2, 0, 2, impl="mma")
    torch.cuda.synchronize()
    err = (a - b).abs().max().item() / b.abs().max().item()
    ts = {}
    for impl in ("umma", "mma"):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            ops.sparse_window_attn(qkv, pool, ktab, flags, t, H2 * W2, 0, 2, impl=impl)
        e1.record()
        torch.cuda.synchronize()
        ts[impl] = e0.elapsed_time(e1) * 100
    print(f"{nm}: umma vs mma rel max diff {err:.2e}; umma {ts['umma']:.1f} us, mma {ts['mma']:.1f} us")
