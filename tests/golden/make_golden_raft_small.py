"""Generates tests/golden/raft_small_c1_8x128x128.npz and tests/golden/state_dict_manifest_raft_small.json (the small
model's state_dict schema, in the format of state_dict_manifest.json) by running the
UNMODIFIED reference RAFT(args.small=True) (imported read-only from /root/reference) in the authoring container.  Not
runnable on the GPU box (no /root/reference there); the committed fixture is what travels.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_raft_small.py

Weights: the seeded synthetic state_dict of the product's ParamNet(raft_small_schema(), seed=SEED), loaded into the
reference module with strict=True.  Frames: C1 (synth.make_clip(8, 128, 128, mask="square", seed=0)) scaled to [-1, 1];
pairs i -> i+1 (forward) and i+1 -> i (backward) on the all-pairs plan (CorrBlock), at 6 and 20 iterations.
Upsampled flows are stored at every 4th pixel (the subsampling of the other golden vectors); the lookup of iteration 0
(196 channels) for the first two forward pairs.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(1, "/root/reference")

from RAFT import RAFT as RefRAFT  # noqa: E402
from RAFT.corr import CorrBlock  # noqa: E402
from RAFT.utils.utils import coords_grid  # noqa: E402

from propainter_b200 import schemas, synth  # noqa: E402
from propainter_b200._params import ParamNet  # noqa: E402

SEED = 4
ITERS = (6, 20)
LOOKUP_PAIRS = 2
GOLD = os.path.dirname(os.path.abspath(__file__))


def c1_frames():
    u8, _, _ = synth.make_clip(8, 128, 128, mask="square", seed=0)
    return torch.from_numpy(u8).permute(0, 3, 1, 2).contiguous().float().div(255) * 2 - 1


@torch.no_grad()
def main():
    torch.set_num_threads(4)
    sd = ParamNet(schemas.raft_small_schema(), seed=SEED).state_dict()
    args = argparse.Namespace(small=True, mixed_precision=False, alternate_corr=False)
    ref = RefRAFT(args).eval()
    ref.load_state_dict(sd, strict=True)
    assert args.corr_radius == 3 and args.corr_levels == 4
    fr = c1_frames()
    a, b = fr[:-1], fr[1:]
    out = {"seed": np.int64(SEED), "schema": np.array("raft_small_schema"), "iters": np.array(ITERS)}
    for it in ITERS:
        for tag, (x, y) in (("fw", (a, b)), ("bw", (b, a))):
            lr, up = ref(x, y, iters=it, test_mode=True)
            out[f"lowres_{tag}_it{it}"] = lr.numpy()
            out[f"up_{tag}_it{it}"] = up[..., ::4, ::4].contiguous().numpy()
    f1, f2 = ref.fnet([a[:LOOKUP_PAIRS], b[:LOOKUP_PAIRS]])
    corr = CorrBlock(f1.float(), f2.float(), radius=args.corr_radius)
    out["lookup_it0_fw"] = corr(coords_grid(LOOKUP_PAIRS, 16, 16)).numpy()
    np.savez_compressed(os.path.join(GOLD, "raft_small_c1_8x128x128.npz"), **out)

    man = {"raft_small": {k: [list(v.shape), str(v.dtype).replace("torch.", "")] for k, v in ref.state_dict().items()}}
    with open(os.path.join(GOLD, "state_dict_manifest_raft_small.json"), "w") as f:
        f.write(json.dumps(man, indent=0))


if __name__ == "__main__":
    main()
