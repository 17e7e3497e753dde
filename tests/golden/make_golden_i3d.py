"""Generates tests/golden/i3d_clips.npz and tests/golden/state_dict_manifest_i3d.json (InceptionI3d's state_dict schema, in
the format of state_dict_manifest.json) by running the UNMODIFIED reference InceptionI3d (core/metrics.py, imported
read-only from /root/reference) in the authoring container.  Not runnable on the GPU box (no /root/reference there); the
committed fixture is what travels.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_i3d.py

core.metrics imports skimage and core.utils at module level (for PSNR / SSIM and to_tensors); I3D needs neither, so both
are replaced by empty stand-ins in sys.modules before the import.

Weights: the seeded synthetic state_dict of the product's ParamNet(i3d_schema(), seed=SEED) -- Kaiming-normal conv weights,
randomised BN statistics and affine parameters (schemas._unit3d) -- loaded into the reference module with strict=True;
the ~51 MB of weights are rebuilt from the seed by the tests.  Inputs: two seeded uint8 clips (CLIPS), 9x72x100 (odd
sizes at several depths: both branches of compute_pad in time and space) and 16x64x64 (all even), converted as
calculate_i3d_activations does (to_tensors, unsqueeze(0), transpose(1, 2)).  Stored per clip: the 1024-d features and the
maps of MAPS, subsampled by (channel step, spatial step) as the other golden vectors are.
"""
import json
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(1, "/root/reference")

_sk = types.ModuleType("skimage")
_sk.measure = types.ModuleType("skimage.measure")
_cu = types.ModuleType("core.utils")
_cu.to_tensors = None
sys.modules.update({"skimage": _sk, "skimage.measure": _sk.measure, "core.utils": _cu})

from core.metrics import InceptionI3d as RefI3d  # noqa: E402

from propainter_b200 import schemas  # noqa: E402
from propainter_b200._params import ParamNet  # noqa: E402

SEED = 11
CLIPS = {"c9x72x100": (9, 72, 100, 1), "c16x64x64": (16, 64, 64, 2)}      # T, H, W, seed
MAPS = {"Conv3d_1a_7x7": (4, 3), "MaxPool3d_2a_3x3": (4, 2), "Mixed_3b": (8, 1), "MaxPool3d_4a_3x3": (4, 1), "Mixed_5c": (2, 1)}
GOLD = os.path.dirname(os.path.abspath(__file__))


def clip_u8(T, H, W, seed):
    return np.random.default_rng(seed).integers(0, 256, (T, H, W, 3), dtype=np.uint8)


def subsample(m, steps):
    c, s = steps
    return m[:, ::c, :, ::s, ::s]


@torch.no_grad()
def main():
    torch.set_num_threads(8)
    sd = ParamNet(schemas.i3d_schema(), seed=SEED).state_dict()
    ref = RefI3d(400, in_channels=3, final_endpoint='Logits').eval()
    ref.load_state_dict(sd, strict=True)
    out = {"seed": np.int64(SEED), "clips": np.array(list(CLIPS)), "maps": np.array(list(MAPS)),
           "steps": np.array(list(MAPS.values()), np.int64)}
    for tag, (T, H, W, seed) in CLIPS.items():
        u8 = clip_u8(T, H, W, seed)
        video = torch.from_numpy(u8).permute(0, 3, 1, 2).contiguous().float().div(255)   # to_tensors: [T,3,H,W]
        x = video.unsqueeze(0).transpose(1, 2)                                            # get_i3d_activations
        out[f"{tag}_shape"] = np.array([T, H, W, seed], np.int64)
        out[f"{tag}_features"] = ref.extract_features(x, 'Logits').numpy()
        for name, steps in MAPS.items():
            m = ref.extract_features(x, name)
            out[f"{tag}_{name}_shape"] = np.array(m.shape, np.int64)
            out[f"{tag}_{name}"] = subsample(m, steps).contiguous().numpy()
        print(tag, "features |max| %.4g mean %.4g" % (np.abs(out[f"{tag}_features"]).max(), out[f"{tag}_features"].mean()))
    np.savez_compressed(os.path.join(GOLD, "i3d_clips.npz"), **out)

    man = {"i3d": {k: [list(v.shape), str(v.dtype).replace("torch.", "")] for k, v in ref.state_dict().items()}}
    with open(os.path.join(GOLD, "state_dict_manifest_i3d.json"), "w") as f:
        f.write(json.dumps(man, indent=0))


if __name__ == "__main__":
    main()
