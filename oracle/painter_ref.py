"""Oracle (test infrastructure): the web demo's tracking preview restated on the CPU in numpy (+ cv2 for the distance
transform, where it is installed).

BaseTracker.track paints each id k present in a frame, in ascending order, with mask_painter at contour width 3
(web-demos/hugging_face/tracker/base_tracker.py:90-95, tools/painter.py:106-157):
  * v = |clip(fore - back, -3, 3)|, fore / back the float32 cv2.distanceTransform(DIST_L2, 3) of the object mask and of
    its complement: min(DT, 3) to the other class, at every pixel
  * c = v / max(v) in float32; contour where 1 - c > 0.5 in float32 (setting c > 0.5 to 1 first changes nothing there)
  * fill: img * (1 - alpha) + palette[k + 1] * alpha in float64 where the label is k, truncated to uint8; then the
    contour pixels take palette[1]

`clipped_dt` is the distance transform the painter uses: the chamfer-table rule (float32 path sums of cv2's 3x3 mask
below 3, over the 7x7 window) by default, or min(cv2.distanceTransform, 3) with cv2=True.
"""
import numpy as np

A, B = np.float32(0.955), np.float32(1.3693)
THREE = np.float32(3)
# (|dy|, |dx|) with dy >= dx -> the float32 path sum of cv2's chamfer; every other offset sums to more than 3
CHAMFER = {(1, 0): A, (1, 1): B, (2, 0): A + A, (2, 1): A + B, (2, 2): B + B, (3, 0): (A + A) + A}


def chamfer_offsets():
    """[(dy, dx, d)]: every signed offset of the 7x7 window whose path sum d is below 3"""
    out = []
    for (p, q), d in CHAMFER.items():
        for dy, dx in {(p, q), (q, p)}:
            for sy in ((1, -1) if dy else (1,)):
                for sx in ((1, -1) if dx else (1,)):
                    out.append((sy * dy, sx * dx, d))
    return out


def clipped_dt_table(m):
    """min(cv2.distanceTransform(m, DIST_L2, 3), 3) of a 0/1 mask [H,W] from the chamfer table: float32 [H,W]"""
    H, W = m.shape
    out = np.full((H, W), THREE, np.float32)
    zero = m == 0
    for dy, dx, d in chamfer_offsets():
        # out[y, x] takes d where m[y + dy, x + dx] == 0 (inside the frame)
        y0, y1, x0, x1 = max(0, -dy), min(H, H - dy), max(0, -dx), min(W, W - dx)
        if y1 <= y0 or x1 <= x0:
            continue
        hit = np.zeros((H, W), bool)
        hit[y0:y1, x0:x1] = zero[y0 + dy:y1 + dy, x0 + dx:x1 + dx]
        out[hit] = np.minimum(out[hit], d)
    out[zero] = 0
    return out


def clipped_dt_cv2(m):
    import cv2
    return np.minimum(cv2.distanceTransform(np.ascontiguousarray(m, np.uint8), cv2.DIST_L2, 3), THREE)


def object_v(m, cv2=False):
    """v = |clip(fore - back, -3, 3)| of a 0/1 object mask: float32 [H,W]"""
    dt = clipped_dt_cv2 if cv2 else clipped_dt_table
    return np.where(m == 1, dt(m), dt(1 - m)).astype(np.float32)


def paint_object(img, m, color, contour_color, alpha=0.7, cv2=False):
    """mask_painter of one 0/1 object mask over img uint8 [H,W,3] -> a new uint8 [H,W,3]"""
    v = object_v(m, cv2)
    c = v / v.max()
    contour = (np.float32(1) - c) > np.float32(0.5)
    out = img.copy()
    sel = m == 1
    out[sel] = (out[sel] * (1 - alpha) + np.asarray(color, np.int64) * alpha).astype(np.uint8)
    out[contour] = contour_color
    return out


def paint_frame(img, labels, palette, alpha=0.7, cv2=False):
    """the painter loop of BaseTracker.track: uint8 [H,W,3] + labels uint8 [H,W] -> painted uint8 [H,W,3]"""
    out = img
    for k in range(1, int(labels.max()) + 1):
        m = (labels == k).astype(np.uint8)
        if m.any():
            out = paint_object(out, m, palette[k + 1], palette[1], alpha, cv2)
    return out.copy() if out is img else out


def paint_clip(frames, labels, palette, alpha=0.7, cv2=False):
    """paint_frame over a clip [T,H,W,3] / [T,H,W]"""
    return np.stack([paint_frame(f, l, palette, alpha, cv2) for f, l in zip(frames, labels)])


def object_maxima(labels):
    """{k: max v over the frame} for every id present in a frame"""
    return {k: float(object_v((labels == k).astype(np.uint8)).max()) for k in np.unique(labels) if k != 0}
