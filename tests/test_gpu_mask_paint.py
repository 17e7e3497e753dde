"""GPU tests of the tracking preview (k_mask_paint_partial / k_mask_paint_maxima / k_mask_paint_u8, ops.mask_paint_u8):
byte for byte against the reference's painter output in tests/golden/painter_cases.npz (synthetic cases, BaseTracker.track's
own frames, show_mask's template preview), against the host build of the same rules on random clips up to 3840 x 2160
with 20 objects, repeated calls, and the trackers' return_painted / paint_masks entry points."""
import numpy as np
import pytest
import torch

from propainter_b200 import ops
from propainter_b200.inpainter import ProInpainter
from propainter_b200.model.cutie import CUTIE
from propainter_b200.tracker import MaskTracker
from tests.cutie_inputs import make_clip
from tests.test_mask_paint_host import fixture_cases, golden, host_paint, hs, random_clip, show_labels  # noqa: F401

DEV = "cuda:0"

pytestmark = pytest.mark.gpu


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def paint(frames, labels, palette=None, alpha=0.7):
    return ops.mask_paint_u8(dev(frames), dev(labels), palette, alpha).cpu().numpy()


def test_kernel_equals_fixture(golden):
    """every fixture case in one launch per case, BaseTracker.track's three frames in one launch, all equal to the
    reference's bytes; and the same-size cases again stacked into one clip"""
    pal = golden["palette"]
    for name, frames, labels, painted in fixture_cases(golden):
        got = paint(frames, labels, pal)
        assert np.array_equal(got, painted), (name, int((got != painted).sum()))
    tiny = [(f, l, p) for n, f, l, p in fixture_cases(golden) if f.shape[1:3] == (5, 5)]
    assert len(tiny) >= 2
    f, l, p = (np.concatenate(x) for x in zip(*tiny))
    assert np.array_equal(paint(f, l, pal), p)


@pytest.mark.parametrize("T,H,W,kind", [(3, 37, 53, "noise"), (4, 64, 96, "blobs"), (2, 1, 300, "dense"), (2, 300, 1, "sparse"),
                                        (5, 33, 31, "full"), (3, 480, 854, "blobs"), (2, 1080, 1920, "blobs"),
                                        (1, 1080, 1920, "dense"), (1, 2160, 3840, "blobs")])
def test_kernel_equals_host_build(hs, T, H, W, kind):
    """random clips with ids up to 20 (blobs: up to 5 random discs per frame, some crossing the border; dense / noise:
    every pixel near a boundary, so the per-object maxima fall below 3 and pass 1 does its reduction at scale)"""
    rng = np.random.default_rng(T * 7919 + H * 31 + W)
    frames, labels = random_clip(rng, T, H, W, kind, 20)
    pal = ops.paint_palette()
    want, _ = host_paint(hs, frames, labels, pal)
    got = paint(frames, labels, pal)
    assert np.array_equal(got, want), int((got != want).sum())


def test_alpha_and_demo_palette_and_in_place(hs, golden):
    rng = np.random.default_rng(3)
    frames, labels = random_clip(rng, 3, 70, 90, "blobs", 20)
    for alpha in (0.0, 0.35, 1.0):
        assert np.array_equal(paint(frames, labels, golden["palette"], alpha), host_paint(hs, frames, labels, golden["palette"], alpha)[0])
    f, l = dev(frames), dev(labels)
    want = ops.mask_paint_u8(f, l)
    assert ops.mask_paint_u8(f, l, out=f) is f and torch.equal(f, want)
    top = int(labels.max())
    with pytest.raises(ValueError, match=f"row {top + 1}"):
        ops.mask_paint_u8(f, l, golden["palette"][:top + 1])


def test_repeated_calls_identical():
    rng = np.random.default_rng(9)
    frames, labels = random_clip(rng, 4, 480, 854, "dense", 20)
    f, l = dev(frames), dev(labels)
    a = ops.mask_paint_u8(f, l)
    for _ in range(3):
        assert torch.equal(ops.mask_paint_u8(f, l), a)


def test_track_return_painted(golden):
    """track(..., return_painted=True) returns the same labels (and probabilities) as without the flag, bit for bit, and
    painted frames equal to ops.mask_paint_u8 over those labels; ProInpainter.track passes the flags through"""
    frames, masks = make_clip(6, 96, 128, 5, ids=(3, 7))
    tr = MaskTracker(CUTIE(seed=2), DEV)
    lab = tr.track(frames, masks[0])
    lab2, painted = tr.track(frames, masks[0], return_painted=True)
    lab3, probs3, painted3 = tr.track(frames, masks[0], return_probs=True, return_painted=True, palette=golden["palette"])
    _, probs = tr.track(frames, masks[0], return_probs=True)
    assert torch.equal(lab, lab2) and torch.equal(lab, lab3) and torch.equal(probs, probs3)
    assert painted.shape == (6, 96, 128, 3) and painted.dtype == torch.uint8 and painted.is_cuda
    assert torch.equal(painted, ops.mask_paint_u8(dev(frames), lab))
    assert not torch.equal(painted3, painted)
    pi = ProInpainter(device=DEV)
    plab, ppainted = pi.track(frames, masks[0], return_painted=True)
    assert torch.equal(ppainted, ops.mask_paint_u8(dev(frames), plab))


def test_paint_masks_reproduces_show_mask(golden):
    """ProInpainter.paint_masks over the demo's mask list (unselected masks zeroed) equals show_mask's preview"""
    pi = ProInpainter(device=DEV)
    masks = [m if i in set(golden["show_selected"].tolist()) else np.zeros_like(m) for i, m in enumerate(golden["show_masks"])]
    got = pi.paint_masks(golden["show_frame"], masks, golden["palette"])
    assert got.shape == golden["show_frame"].shape and np.array_equal(got.cpu().numpy(), golden["show_painted"])
    assert np.array_equal(paint(golden["show_frame"][None], show_labels(golden)[None], golden["palette"])[0],
                          golden["show_painted"])
