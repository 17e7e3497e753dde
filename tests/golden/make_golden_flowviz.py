"""Generates tests/golden/flowviz_c1.npz by running the UNMODIFIED reference code (read-only from /root/reference) in the
authoring container; the committed fixture is what travels.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_flowviz.py

Colour coding: the reference's own `flow_to_image` of RAFT/utils/flow_viz.py (numpy) and RAFT/utils/flow_viz_pt.py
(torch, with its module-level `torch.pi` assignment).  RAFT/utils/__init__.py imports more than those files need, so the
definitions are taken from the source files with `ast` and compiled as they stand.  Inputs:
  * two of the full-resolution forward RAFT flows of the C1 clip (8 x 128 x 128, square mask; pairs 0 and 6, whose
    maxima differ), reference RAFT with make_golden's seeded weights and 20 iterations (evaluate_flow_completion.py's
    short-clip branch).  Two flows keep the fixture under 1 MB and still exercise per-frame against per-batch maxima;
  * synthetic fields: signed-zero axes, exact diagonals, an all-zero frame, and frames whose largest vector (256-1000 px)
    normalises to just above 1, so the numpy variant takes its `rad > 1` branch.
Flow completion: the reference RecurrentFlowCompleteNet run once over the whole C1 clip as evaluate_flow_completion.py
:132-133 does (masks binarised and cv2.dilate'd 4x with the 3x3 cross as TestDataset does), a stride-4 subsample of the
completed flows, and the script's two EPE numbers (:143-144) against the RAFT flows of the unmasked frames.
"""
import ast
import os
import sys

import cv2
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden  # noqa: E402  (puts the repository and the reference on sys.path)

from propainter_b200 import synth  # noqa: E402

REF = "/root/reference"
NAME = "flowviz_c1"
C1_PAIRS = (0, 6)


def reference_module(path, names):
    """the top-level functions `names` of a reference source file plus its module-level attribute assignments (the
    `torch.pi = ...` of flow_viz_pt.py), compiled unmodified"""
    tree = ast.parse(open(path).read(), path)
    body = [n for n in tree.body if (isinstance(n, ast.FunctionDef) and n.name in names)
            or (isinstance(n, ast.Assign) and all(isinstance(t, ast.Attribute) for t in n.targets))]
    assert {n.name for n in body if isinstance(n, ast.FunctionDef)} == set(names), names
    ns = {"np": np, "torch": torch}
    exec(compile(ast.Module(body=body, type_ignores=[]), path, "exec"), ns)
    return ns


def big_vector(rng, pt_wrap):
    """a float32 vector of 256-1000 px that normalises (by itself + 1e-5, which float32 drops) to a norm above 1; with
    `pt_wrap` also one whose colour has a zero channel, where flow_viz_pt's floor(255 (1 - norm)) gives -1"""
    while True:
        r, t = rng.uniform(256, 1000), rng.uniform(-np.pi, np.pi)
        u, v = np.float32(r * np.cos(t)), np.float32(r * np.sin(t))
        rad = np.sqrt(u * u + v * v)
        den = rad + np.float32(1e-5)
        un, vn = u / den, v / den
        if np.sqrt(un * un + vn * vn) <= 1:
            continue
        if not pt_wrap:
            return u, v
        fk = (np.arctan2(-vn, -un) / np.float32(np.pi) + np.float32(1)) / np.float32(2) * np.float32(54)
        if int(fk) not in (20, 35):                 # both wheel entries share a zero channel (all but YG->GC, GC->CB)
            return u, v


def synthetic(rng):
    """[7,2,32,48] float32: 0 axes / signed zeros / diagonals, 1 all zero, 2-6 random fields whose largest vector takes
    the rad > 1 branch (frame 2's is the batch maximum and pushes the torch variant's floor to -1 where possible)"""
    N, H, W = 7, 32, 48
    f = np.zeros((N, 2, H, W), np.float32)
    special = [(u, v) for u in (0.0, -0.0) for v in (0.0, -0.0)]
    special += [(s * a, z) for s in (1, -1) for a in (1.0, 7.5) for z in (0.0, -0.0)]
    special += [(z, s * a) for s in (1, -1) for a in (1.0, 7.5) for z in (0.0, -0.0)]
    special += [(su * a, sv * a) for su in (1, -1) for sv in (1, -1) for a in (0.25, 3.0, 12.0)]
    g = rng.standard_normal((2, H, W)).astype(np.float32) * 4
    for i, (u, v) in enumerate(special):
        g[0, i // W, i % W], g[1, i // W, i % W] = u, v
    f[0] = g
    for n in range(2, N):
        u, v = big_vector(rng, pt_wrap=n == 2)
        r = np.hypot(u, v)
        scale = r * (0.99 if n == 2 else 0.5 - 0.05 * n)
        f[n] = rng.uniform(-1, 1, (2, H, W)).astype(np.float32) * np.float32(scale / np.sqrt(2))
        y, x = rng.integers(0, H), rng.integers(0, W)
        f[n, 0, y, x], f[n, 1, y, x] = u, v
    return f


def numpy_variant(ns, flows, **kw):
    return np.stack([ns["flow_to_image"](fl.transpose(1, 2, 0), **kw) for fl in flows])


def torch_variant(ns, flows):
    return ns["flow_to_image"](torch.from_numpy(flows)).permute(0, 2, 3, 1).contiguous().numpy()


if __name__ == "__main__":
    npv = reference_module(os.path.join(REF, "RAFT", "utils", "flow_viz.py"),
                           ["make_colorwheel", "flow_uv_to_colors", "flow_to_image"])
    ptv = reference_module(os.path.join(REF, "RAFT", "utils", "flow_viz_pt.py"),
                           ["flow_to_image", "_normalized_flow_to_image", "_make_colorwheel"])
    raft, rfc, _ = make_golden.build_reference()
    u8, fm, _ = synth.make_clip(8, 128, 128, mask="square", seed=0)
    frames = (torch.from_numpy(u8).permute(0, 3, 1, 2).contiguous().float().div(255) * 2 - 1).unsqueeze(0)
    with torch.no_grad():
        gt = make_golden.raft_bi(raft, frames, 20)
        kernel = cv2.getStructuringElement(cv2.MORPH_CROSS, (3, 3))
        m = [cv2.dilate((fm[0, t, 0].numpy() > 0).astype(np.uint8), kernel, iterations=4) for t in range(fm.shape[1])]
        masks = torch.from_numpy(np.stack(m)).float()[None, :, None]
        pred, _ = rfc.forward_bidirect_flow(gt, masks)
        pred = rfc.combine_flow(gt, pred, masks)
    epe1 = torch.mean(torch.sum((gt[0] - pred[0]) ** 2, dim=2).sqrt())
    epe2 = torch.mean(torch.sum((gt[1] - pred[1]) ** 2, dim=2).sqrt())
    c1 = gt[0][0, list(C1_PAIRS)].contiguous().numpy()                   # [2,2,128,128] float32
    clip_c1 = float(np.float32(np.abs(c1).max() * 0.5))
    syn = synthetic(np.random.default_rng(5))
    out = dict(
        c1_flow=c1, c1_pairs=np.array(C1_PAIRS), c1_clip=np.array(clip_c1),
        c1_np=numpy_variant(npv, c1), c1_np_clip_bgr=numpy_variant(npv, c1, clip_flow=clip_c1, convert_to_bgr=True),
        c1_pt=torch_variant(ptv, c1),
        syn_flow=syn, syn_np=numpy_variant(npv, syn), syn_np_bgr=numpy_variant(npv, syn, convert_to_bgr=True),
        syn_np_clip=numpy_variant(npv, syn, clip_flow=300.0), syn_pt=torch_variant(ptv, syn),
        pred_f=pred[0][..., ::4, ::4].contiguous().numpy(), pred_b=pred[1][..., ::4, ::4].contiguous().numpy(),
        epe=np.array([epe1.item(), epe2.item()]), masks=np.packbits(masks.numpy().astype(np.uint8)), raft_iter=np.array(20))
    path = os.path.join(HERE, NAME + ".npz")
    np.savez_compressed(path, **out)
    print(NAME, "EPE", out["epe"], "clip", clip_c1, "|flow|max", np.abs(c1).max(), os.path.getsize(path) // 1024, "KiB")
