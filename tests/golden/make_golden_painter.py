"""Generates tests/golden/painter_cases.npz by running the UNMODIFIED reference painter (web-demos/hugging_face/tools/
painter.py, and tracker/base_tracker.py for the tracked frames, imported read-only from /root/reference) on the CPU in
the authoring container.  Not runnable on the GPU box (no /root/reference there); the committed fixture is what travels.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_painter.py

Stored:
  * palette: the demo's colour table as the painter indexes it (colormap().astype('uint8'), [86,3])
  * case{i}_frames / _labels / _painted (+ case_names): synthetic uint8 clips [T,H,W,3] and label maps [T,H,W] through
    BaseTracker.track's painter loop (base_tracker.py:90-95, restated in loop() below: ascending ids, absent ids skipped,
    mask_color = id + 1): border-touching, whole-frame, 1-px and line objects, diagonal contacts, adjacent objects whose
    contours overlap, non-consecutive ids up to 20, empty frames, tiny frames where an object's maximum M is below 3
    (among them M = a + a and M = b + b, where v / M is exactly 0.5), random label maps
  * show_*: the template preview of app.py's show_mask (:191-197): three non-overlapping 0/1 masks, the selection
    ["mask_001", "mask_003"] painted with mask_color = mask_number + 2
  * tracker_*: tests/cutie_inputs.CLIP through the unmodified BaseTracker.track (seeded weights, the stand-ins of
    make_golden_cutie.py, whose omegaconf stub gains OmegaConf.create): the labels and painted frames it returns at
    frames tracker_t; the tests regenerate the input frames with cutie_inputs.make_clip
"""
import os
import sys
import tempfile
import types

import numpy as np
import torch

GOLD = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, GOLD)
import make_golden_cutie as mgc  # noqa: E402  (ROOT, tests/ and the reference on sys.path; download stand-ins)

from tools.painter import colormap, mask_painter  # noqa: E402

from cutie_inputs import CLIP, make_clip  # noqa: E402
from oracle import painter_ref  # noqa: E402
from propainter_b200 import schemas  # noqa: E402
from propainter_b200._params import ParamNet  # noqa: E402

TRACKER_T = (0, 9, 31)                  # the template frame, a tracked frame, the last frame


def loop(frame, final_mask):
    """base_tracker.py:90-95, verbatim in effect"""
    num_objs = final_mask.max()
    painted_image = frame
    for obj in range(1, num_objs + 1):
        if np.max(final_mask == obj) == 0:
            continue
        painted_image = mask_painter(painted_image, (final_mask == obj).astype('uint8'), mask_color=obj + 1)
    return painted_image


def rect(lab, y0, y1, x0, x1, k):
    lab[y0:y1, x0:x1] = k
    return lab


def tiny_cases(rng):
    """tiny frames where some object's maximum M is a + a or b + b (v / M exactly 0.5 at v = a or b), and others < 3"""
    a, b = painter_ref.A, painter_ref.B
    want = {np.float32(a + a): 2, np.float32(b + b): 2, np.float32((a + a) + a): 1, np.float32(a + b): 1, np.float32(b): 1}
    out = []
    for _ in range(20000):
        if not any(want.values()):
            break
        H, W = rng.integers(1, 7, 2)
        lab = (rng.integers(0, 3, (H, W)) * (rng.random((H, W)) < 0.7)).astype(np.uint8)
        hit = [m for m in painter_ref.object_maxima(lab).values() if want.get(np.float32(m), 0) > 0]
        if hit:
            want[np.float32(hit[0])] -= 1
            out.append(lab)
    assert not any(want.values()), want
    return out


def cases(rng):
    c = {}
    lab = np.zeros((20, 30), np.uint8)
    rect(lab, 0, 6, 0, 9, 1)                       # the top-left corner
    rect(lab, 8, 20, 24, 30, 2)                    # the right and bottom edges
    rect(lab, 0, 20, 14, 16, 3)                    # top to bottom
    c["border"] = lab
    c["whole_frame"] = np.full((12, 17), 3, np.uint8)
    lab = np.zeros((15, 15), np.uint8)
    lab[7, 7], lab[0, 14], lab[3, 3], lab[4, 4] = 4, 5, 1, 2     # single pixels, a corner, a diagonal contact
    c["one_pixel"] = lab
    lab = np.zeros((24, 24), np.uint8)
    lab[5, 2:20] = 1                               # horizontal, vertical and diagonal 1-px lines
    lab[2:22, 12] = 2
    for i in range(16):
        lab[4 + i, 3 + i] = 6
    c["lines"] = lab
    lab = np.zeros((16, 16), np.uint8)
    for y in range(16):
        for x in range(16):
            if (y // 2 + x // 2) % 2 == 0:
                lab[y, x] = 1 + (y // 4) % 2       # 2x2 blocks touching at corners
    c["diagonal"] = lab
    lab = np.zeros((30, 40), np.uint8)
    rect(lab, 5, 25, 5, 15, 1)
    rect(lab, 5, 25, 15, 25, 2)                    # adjacent: overlapping contours
    rect(lab, 10, 20, 25, 33, 3)
    c["adjacent"] = lab
    lab = np.zeros((40, 50), np.uint8)
    for k, (y, x, r) in zip((2, 7, 13, 20), ((10, 10, 6), (12, 30, 8), (30, 15, 7), (28, 38, 9))):
        yy, xx = np.mgrid[0:40, 0:50]
        lab[(yy - y) ** 2 + (xx - x) ** 2 <= r * r] = k
    c["ids_to_20"] = lab
    c["empty"] = np.zeros((9, 11), np.uint8)
    for i, lab in enumerate(tiny_cases(rng)):
        c[f"tiny_{i}"] = lab
    c["tiny_1x1"] = np.ones((1, 1), np.uint8)
    c["tiny_1x7"] = np.array([[0, 1, 1, 0, 2, 0, 1]], np.uint8)
    c["random_4"] = rng.integers(0, 4, (37, 53)).astype(np.uint8)
    c["random_sparse"] = ((rng.random((41, 29)) < 0.1) * rng.integers(1, 6, (41, 29))).astype(np.uint8)
    out = {name: (lab[None], rng.integers(0, 256, lab.shape + (3,), dtype=np.uint8)[None]) for name, lab in c.items()}
    # one clip of several frames: blobs moving across an odd-sized frame, one frame empty, one with a corner object
    T, H, W = 5, 45, 67
    yy, xx = np.mgrid[0:H, 0:W]
    clip = np.zeros((T, H, W), np.uint8)
    for t in range(T):
        if t == 2:
            continue
        clip[t][(yy - 10 - 5 * t) ** 2 + (xx - 8 - 12 * t) ** 2 <= 64] = 1
        clip[t][(np.abs(yy - 30) <= 6) & (np.abs(xx - 60 + 9 * t) <= 10)] = 4
    clip[4, :3, :3] = 2
    out["clip"] = (clip, rng.integers(0, 256, (T, H, W, 3), dtype=np.uint8))
    return out


def show_mask_case(rng):
    H, W = 48, 64
    masks = np.zeros((3, H, W), np.uint8)
    masks[0, 5:20, 5:25] = 1
    masks[1, 25:40, 10:30] = 1
    masks[2, 10:45, 35:60] = 1
    frame = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    dropdown = ["mask_003", "mask_001"]
    dropdown.sort()                                # app.py:191-197
    select_frame = frame
    for name in dropdown:
        mask_number = int(name.split("_")[1]) - 1
        select_frame = mask_painter(select_frame, masks[mask_number].astype('uint8'), mask_color=mask_number + 2)
    return frame, masks, np.array([int(n.split("_")[1]) - 1 for n in dropdown], np.int64), select_frame


@torch.no_grad()
def tracker_frames():
    mgc._om.OmegaConf = types.SimpleNamespace(create=lambda c: mgc.config())
    from tracker.base_tracker import BaseTracker
    sd = ParamNet(schemas.cutie_schema(), seed=mgc.SEED).state_dict()
    with tempfile.TemporaryDirectory() as d:
        ck = os.path.join(d, "cutie.pth")
        torch.save(sd, ck)
        bt = BaseTracker(ck, "cpu")
    frames, masks = make_clip(CLIP["T"], CLIP["H"], CLIP["W"], CLIP["seed"])
    labels, painted = [], []
    for t in range(max(TRACKER_T) + 1):
        m, _, p = bt.track(frames[t], masks[0] if t == 0 else None)
        if t in TRACKER_T:
            labels.append(m)
            painted.append(p)
            print("tracker frame", t, "ids", np.unique(m).tolist())
    return np.stack(labels), np.stack(painted)


def main():
    torch.set_num_threads(8)
    rng = np.random.default_rng(2024)
    palette = colormap().astype('uint8')
    out = {"palette": palette}
    cs = cases(rng)
    out["case_names"] = np.array(list(cs))
    for i, (name, (labels, frames)) in enumerate(cs.items()):
        painted = np.stack([loop(f, l) for f, l in zip(frames, labels)])
        assert np.array_equal(painted, painter_ref.paint_clip(frames, labels, palette)), name
        out[f"case{i}_frames"], out[f"case{i}_labels"], out[f"case{i}_painted"] = frames, labels, painted
        print(f"case {name}: {labels.shape}, {int((painted != frames).sum())} bytes painted")
    frame, masks, sel, shown = show_mask_case(rng)
    out.update(show_frame=frame, show_masks=masks, show_selected=sel, show_painted=shown)
    labels, painted = tracker_frames()
    out.update(tracker_t=np.array(TRACKER_T, np.int64), tracker_labels=labels, tracker_painted=painted)
    np.savez_compressed(os.path.join(GOLD, "painter_cases.npz"), **out)


if __name__ == "__main__":
    main()
