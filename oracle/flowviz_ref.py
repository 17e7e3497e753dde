"""Oracle (test infrastructure): the two Middlebury flow colour codings of the reference, restated on the CPU.

numpy variant: RAFT/utils/flow_viz.py:70-132 for a float32 [H,W,2] frame under numpy >= 2 (NEP 50): float32 up to fk,
float64 from f = fk - k0 on, the rad > 1 branch.  torch variant: RAFT/utils/flow_viz_pt.py:6-70, float32 throughout,
normalised over the whole batch.  Both take planar flow [N,2,H,W] and return uint8 [N,H,W,3] (RGB, or BGR).

`shift` moves every atan2 result by that many float32 ulps.  atan2 is not correctly rounded in numpy's float32 path,
in ATen or in CUDA, so implementations may disagree in its last ulps; `sensitive` marks the pixels whose colour changes
under a shift of up to +-4 ulps -- the only pixels where two faithful implementations may differ (by one level).
"""
import numpy as np
import torch

NCOLS = 55


def colorwheel():
    """make_colorwheel: float64 [55,3]; segment lengths RY 15, YG 6, GC 4, CB 11, BM 13, MR 6"""
    w = np.zeros((NCOLS, 3))
    ramp = lambda n: np.floor(255 * np.arange(n) / n)
    segs = [(15, (255, "up", 0)), (6, ("down", 255, 0)), (4, (0, 255, "up")), (11, (0, "down", 255)),
            (13, ("up", 0, 255)), (6, (255, 0, "down"))]
    k = 0
    for n, chans in segs:
        for c, val in enumerate(chans):
            w[k:k + n, c] = ramp(n) if val == "up" else 255 - ramp(n) if val == "down" else val
        k += n
    return w


def _shift_ulps(x, k):
    for _ in range(abs(int(k))):
        x = np.nextafter(x, np.float32(np.inf if k > 0 else -np.inf)).astype(np.float32)
    return x


def clip(flow, clip_flow):
    """np.clip(flow, 0, clip_flow) in float32 (flow_viz.py:124)"""
    return flow if clip_flow is None else np.clip(np.asarray(flow, np.float32), 0, clip_flow).astype(np.float32)


def _wheel(un, vn, atan2, shift):
    """float32 fk, int k0 / k1 of normalised components (flow_viz.py:89-93, flow_viz_pt.py:56-60)"""
    a = _shift_ulps(atan2(-vn, -un), shift) / np.float32(np.pi)
    fk = ((a + np.float32(1)) / np.float32(2) * np.float32(NCOLS - 1)).astype(np.float32)
    k0 = np.floor(fk).astype(np.int32)
    k1 = k0 + 1
    k1[k1 == NCOLS] = 0
    return fk, k0, k1


def colors_np(u, v, den, bgr=False, shift=0):
    """numpy variant per pixel: float32 u, v (clipped), float32 den = rad_max + 1e-5 -> uint8 [..., 3]"""
    un, vn = (u / den).astype(np.float32), (v / den).astype(np.float32)
    rad = np.sqrt(un * un + vn * vn).astype(np.float32)
    fk, k0, k1 = _wheel(un, vn, np.arctan2, shift)
    f = fk.astype(np.float64) - k0.astype(np.float64)
    w = colorwheel()
    out = np.zeros(u.shape + (3,), np.uint8)
    inside = rad <= 1
    for i in range(3):
        col = (1 - f) * (w[k0, i] / 255.0) + f * (w[k1, i] / 255.0)
        col = np.where(inside, 1 - rad.astype(np.float64) * (1 - col), col * 0.75)
        out[..., 2 - i if bgr else i] = np.floor(255 * col)
    return out


def colors_pt(u, v, den, bgr=False, shift=0):
    """torch variant per pixel: float32 u, v, float32 den = max_norm + eps -> uint8 [..., 3] (float32 throughout; the
    float -> uint8 copy goes through int32, so floor = -1 wraps to 255)"""
    un, vn = (u / den).astype(np.float32), (v / den).astype(np.float32)
    norm = np.sqrt(un * un + vn * vn).astype(np.float32)
    atan2 = lambda y, x: torch.atan2(torch.from_numpy(np.ascontiguousarray(y)), torch.from_numpy(np.ascontiguousarray(x))).numpy()
    fk, k0, k1 = _wheel(un, vn, atan2, shift)
    f = (fk - k0.astype(np.float32)).astype(np.float32)
    w = colorwheel().astype(np.float32)
    one = np.float32(1)
    out = np.zeros(u.shape + (3,), np.uint8)
    for i in range(3):
        col = (one - f) * (w[k0, i] / np.float32(255)) + f * (w[k1, i] / np.float32(255))
        col = (one - norm * (one - col)).astype(np.float32)
        out[..., 2 - i if bgr else i] = np.floor(np.float32(255) * col).astype(np.int32).astype(np.uint8)
    return out


def denominators(flows, normalize, clip_flow=None):
    """float32 per-frame den [N]: rad_max + 1e-5 per frame ("frame") or max_norm + eps over the batch ("clip")"""
    f = clip(np.asarray(flows, np.float32), clip_flow)
    rad = np.sqrt(f[:, 0] * f[:, 0] + f[:, 1] * f[:, 1]).astype(np.float32)
    if normalize == "frame":
        return (rad.reshape(len(f), -1).max(1) + np.float32(1e-5)).astype(np.float32)
    return np.full(len(f), rad.max() + np.finfo(np.float32).eps, np.float32)


def flow_to_image(flows, normalize="frame", clip_flow=None, bgr=False, shift=0, index=None):
    """planar float32 [N,2,H,W] -> uint8 [N,H,W,3]; with `index` (a tuple of n, y, x arrays) only those pixels, [P,3]"""
    f = clip(np.asarray(flows, np.float32), clip_flow)
    den = denominators(flows, normalize, clip_flow)[:, None, None] * np.ones((1,) + f.shape[2:], np.float32)
    u, v = f[:, 0], f[:, 1]
    if index is not None:
        u, v, den = u[index], v[index], den[index]
    rule = colors_np if normalize == "frame" else colors_pt
    return rule(u, v, den, bgr, shift)


def sensitive(flows, normalize="frame", clip_flow=None, bgr=False, index=None, ulps=4):
    """bool mask of the pixels whose bytes change when atan2 moves by up to +-`ulps` float32 ulps"""
    base = flow_to_image(flows, normalize, clip_flow, bgr, 0, index)
    out = np.zeros(base.shape[:-1], bool)
    for k in range(1, ulps + 1):
        for s in (k, -k):
            out |= (flow_to_image(flows, normalize, clip_flow, bgr, s, index) != base).any(-1)
    return out


def check_equal(got, flows, normalize="frame", clip_flow=None, bgr=False, ref=None):
    """The equality criterion: bytes equal `ref` (default: this restatement) except at sensitive pixels, where they may
    differ by one level.  Returns (number of differing pixels, size of the sensitive set among them)."""
    ref = flow_to_image(flows, normalize, clip_flow, bgr) if ref is None else ref
    got = np.asarray(got)
    assert got.shape == ref.shape and got.dtype == np.uint8, (got.shape, ref.shape)
    d = np.abs(got.astype(int) - ref.astype(int))
    bad = np.nonzero(d.max(-1) > 0)
    if len(bad[0]):
        sens = sensitive(flows, normalize, clip_flow, bgr, index=bad)
        assert sens.all(), f"{int((~sens).sum())} of {len(bad[0])} differing pixels are not on a rounding boundary"
        assert d.max() <= 1, int(d.max())
    return len(bad[0])
