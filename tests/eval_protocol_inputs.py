"""Inputs of the evaluation-protocol fixture (tests/golden/make_golden_eval_protocol.py), regenerated from seeds by the
tests: synth.make_clip frames / masks at the native 144 x 240 and seeded synthetic flows."""
import hashlib

import numpy as np

from propainter_b200 import synth

NATIVE = (144, 240)


def synthetic_flows(T, H, W, seed):
    """(forward, backward) float32 [T-1,2,H,W]: a coarse random field (16 x 16 px cells, up to ~6 px) plus per-pixel
    noise, rounded to fp16 -- what flowread returns for the .flo files flowwrite stores.  Exact arithmetic only, so the
    values are the same on every machine."""
    rng = np.random.default_rng(1000 + seed)
    out = []
    for _ in range(2):
        coarse = rng.integers(-24, 25, (T - 1, 2, H // 16 + 1, W // 16 + 1)).astype(np.float32) * np.float32(0.25)
        f = np.repeat(np.repeat(coarse, 16, 2), 16, 3)[..., :H, :W]
        f = f + rng.integers(-64, 65, f.shape).astype(np.float32) * np.float32(1 / 64)
        out.append(f.astype(np.float16).astype(np.float32))
    return tuple(out)


def video_inputs(T, mask, seed):
    """-> (frames uint8 [T,144,240,3] RGB, masks uint8 [T,144,240] 0 / 255, flows)"""
    u8, fm, _ = synth.make_clip(T, NATIVE[0], NATIVE[1], mask=mask, seed=seed)
    return u8, (fm[0, :, 0].numpy() > 0).astype(np.uint8) * 255, synthetic_flows(T, NATIVE[0], NATIVE[1], seed)


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()
