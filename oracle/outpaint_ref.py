"""Oracle (test infrastructure): the video-outpainting front end of the inference driver, restated in plain numpy.

inference_propainter.py:117-156 (extrapolation: canvas size, offset, zero-bordered frames, the flow mask with its
4-px rim and the dilated mask), :265-266 (to_tensors of the masks: 0/255 images -> float {0,1}) and :250-261 (the green
masked-frame preview, float64).  Arrays in, arrays out; no PIL.
"""
import numpy as np
import torch


def geometry(h, w, scale_h, scale_w):
    """:123-128, :142-143 -> ((H, W), (top, left), (rim_h, rim_w)); Python doubles, like the script's argparse floats."""
    H = int(float(scale_h) * h)
    W = int(float(scale_w) * w)
    H -= H % 8
    W -= W % 8
    top = int((H - h) / 2)
    left = int((W - w) / 2)
    return (H, W), (top, left), (4 if top > 10 else 0, 4 if left > 10 else 0)


def masks(geo, h, w):
    """:144-151: (flow_mask, mask_dilated) uint8 {0,1} [H,W] -- one frame; every frame shares them (:153-154)."""
    (H, W), (top, left), (rh, rw) = geo
    flow = np.ones((H, W), np.uint8)
    flow[top + rh:top + h - rh, left + rw:left + w - rw] = 0       # numpy slice: an empty range clears nothing
    dil = np.ones((H, W), np.uint8)
    dil[top:top + h, left:left + w] = 0
    return flow, dil


def canvas(frames_u8, geo):
    """:132-136: uint8 [T,h,w,3] -> uint8 [T,H,W,3], the source at (top, left), zeros elsewhere."""
    (H, W), (top, left), _ = geo
    T, h, w, _ = frames_u8.shape
    out = np.zeros((T, H, W, 3), np.uint8)
    out[:, top:top + h, left:left + w] = frames_u8
    return out


def extrapolate(frames_u8, scale_h=1.0, scale_w=1.2):
    """The whole front end: (canvas uint8 [T,H,W,3], flow_masks, masks_dilated float32 {0,1} [1,T,1,H,W], (W, H))."""
    frames_u8 = np.asarray(frames_u8)
    T, h, w, _ = frames_u8.shape
    geo = geometry(h, w, scale_h, scale_w)
    fm, md = masks(geo, h, w)
    stack = lambda m: torch.from_numpy(np.repeat(m[None, None].astype(np.float32), T, 0)).unsqueeze(0)
    H, W = geo[0]
    return canvas(frames_u8, geo), stack(fm), stack(md), (W, H)


def mask_overlay(frames_u8, masks_f):
    """:250-261: uint8 [T,H,W,3] + masks with T*H*W values -> uint8 [T,H,W,3], in float64 as the script computes it."""
    frames_u8 = np.asarray(frames_u8)
    T, H, W, _ = frames_u8.shape
    m = np.asarray(masks_f, dtype=np.float64).reshape(T, H, W, 1)
    img = frames_u8.astype(np.float64)
    green = np.zeros(3)
    green[1] = 255.0
    alpha = 0.6
    fuse = (1 - alpha) * img + alpha * green
    return (m * fuse + (1 - m) * img).astype(np.uint8)
