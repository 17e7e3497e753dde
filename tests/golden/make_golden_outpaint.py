"""Generates the video-outpainting fixtures tests/golden/outpaint_*.npz by running the UNMODIFIED reference code (read-only
from /root/reference) in the authoring container; the committed fixtures are what travels.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_outpaint.py

The front end is the reference's own `extrapolation` (inference_propainter.py:117-156) and its mask conversion
`Stack` + `ToTorchFormatTensor` (core/utils.py:130-170, the to_tensors of inference_propainter.py:265-266).  Neither
module is importable here (the script needs imageio and keeps its logic under __main__, core/utils needs matplotlib),
so those definitions are taken from the source files with `ast` and compiled as they stand.  The four stages are the
reference modules driven by make_golden.reference_pipeline, with make_golden's seeded weights and summary format; each
fixture also stores the first frame's two masks, bit-packed.
"""
import ast
import os
import sys

import numpy as np
import torch
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden  # noqa: E402  (puts the repository and the reference on sys.path)

from propainter_b200 import synth  # noqa: E402

REF = "/root/reference"


def reference_definitions(path, names):
    """the top-level functions / classes `names` of a reference source file, compiled unmodified"""
    tree = ast.parse(open(path).read(), path)
    body = [n for n in tree.body if isinstance(n, (ast.FunctionDef, ast.ClassDef)) and n.name in names]
    assert {n.name for n in body} == set(names), names
    ns = {"np": np, "torch": torch, "Image": Image}
    exec(compile(ast.Module(body=body, type_ignores=[]), path, "exec"), ns)
    return ns


CASES = {
    # canvas 128x160: top 0 (no row rim), left 16 (rim 4)
    "outpaint_8x128x128_s1.0x1.3_it6": dict(T=8, H=128, W=128, scale=(1.0, 1.3), raft_iter=6),
    # canvas 160x136: top 16 (rim 4), left 4 (no column rim)
    "outpaint_8x128x128_s1.25x1.1_it6": dict(T=8, H=128, W=128, scale=(1.25, 1.1), raft_iter=6),
}

if __name__ == "__main__":
    ns = reference_definitions(os.path.join(REF, "inference_propainter.py"), ["extrapolation"])
    ns.update(reference_definitions(os.path.join(REF, "core", "utils.py"), ["Stack", "ToTorchFormatTensor"]))
    to_tensors = lambda imgs: ns["ToTorchFormatTensor"]()(ns["Stack"]()(imgs))
    nets = make_golden.build_reference()
    for name, c in CASES.items():
        u8, _, _ = synth.make_clip(c["T"], c["H"], c["W"], seed=0)
        frames, flow_masks, masks_dilated, size = ns["extrapolation"]([Image.fromarray(f) for f in u8], c["scale"])
        canvas = np.stack([np.array(f).astype(np.uint8) for f in frames])
        fm, md = to_tensors(flow_masks).unsqueeze(0), to_tensors(masks_dilated).unsqueeze(0)
        assert canvas.shape[1:3] == (size[1], size[0])
        comp, st = make_golden.reference_pipeline(nets, canvas, fm, md, raft_iter=c["raft_iter"])
        make_golden.summarize(name, comp, st, HERE, stride=4)
        path = os.path.join(HERE, name + ".npz")
        data = dict(np.load(path))
        data.update(flow_mask0=np.packbits(fm[0, 0, 0].numpy().astype(np.uint8)),
                    mask_dilated0=np.packbits(md[0, 0, 0].numpy().astype(np.uint8)),
                    size=np.array(size), scale=np.array(c["scale"]))
        np.savez_compressed(path, **data)
        print(name, "done", comp.shape, os.path.getsize(path) // 1024, "KiB")
