"""Oracle (test infrastructure): the temporal warping error E_warp, restated in float64 numpy.

The metric is the evaluation of Lai et al., "Learning Blind Video Temporal Consistency" (ECCV 2018), with the occlusion
test of Ruder et al., "Artistic style transfer for videos" (GCPR 2016).  The reference does not compute it; this module
restates the published protocol, and agreement with Lai et al.'s own tool has not been checked.

Inputs: frames uint8 [T,H,W,3] (read as value / 255), forward flows fw [T-1,2,H,W] (frame t -> t+1, channel 0 = x) and
backward flows bw [T-1,2,H,W] (frame t+1 -> t).

* S(img, F): FlowNet2 Resample2d's border-clamped bilinear sample of img at x + F(x).  The coordinate x + F(x) is rounded
  to float32, as Resample2d computes it; everything after it is float64.  Taps floor and floor + 1 on each axis, clamped
  into the frame; weights (1-a)(1-b), a(1-b), (1-a)b, ab from the unclamped fractions.
* O_t = 1 where |F + S(B, F)|^2 > 0.01 (|F|^2 + |S(B, F)|^2) + 0.5 (forward-backward check) or
  |du|^2 + |dv|^2 > 0.01 |F|^2 + 0.002 (motion boundary; forward differences of F, 0 in the last column / row).
* E_t = sum over pixels with O_t = 0 and the 3 channels of (S(R_{t+1}, F_t) - R_t)^2 / (3 N_t), 0 when N_t = 0.
* E_warp of a video = mean_t E_t; of a dataset = the mean of the per-video values.

`undecided` marks the pixels where one of the two tests lies within MARGIN * (1 + rhs) of its threshold: there a
float32 implementation may decide either way.
"""
import numpy as np

MARGIN = 1e-5


def _as_flows(f):
    f = np.asarray(f)
    return f.reshape(-1, *f.shape[-3:])


def sample(img, flow):
    """S(img, flow): img [C,H,W] (any real dtype), flow [2,H,W] -> float64 [C,H,W]"""
    img = np.asarray(img, np.float64)
    _, H, W = img.shape
    y, x = np.mgrid[0:H, 0:W]
    xf = (x.astype(np.float32) + np.asarray(flow[0], np.float32)).astype(np.float64)
    yf = (y.astype(np.float32) + np.asarray(flow[1], np.float32)).astype(np.float64)
    flx, fly = np.floor(xf), np.floor(yf)
    a, b = xf - flx, yf - fly
    xl, xr = (np.clip(v, 0, W - 1).astype(np.int64) for v in (flx, flx + 1))
    yt, yb = (np.clip(v, 0, H - 1).astype(np.int64) for v in (fly, fly + 1))
    return ((1 - a) * (1 - b) * img[:, yt, xl] + a * (1 - b) * img[:, yt, xr]
            + (1 - a) * b * img[:, yb, xl] + a * b * img[:, yb, xr])


def occlusion_sides(F, B):
    """the two tests of one pair, F / B [2,H,W]: (lhs1, rhs1, lhs2, rhs2) float64 [H,W]; occluded where lhs > rhs"""
    F = np.asarray(F, np.float64)
    w = sample(B, F)
    lhs1 = ((F + w) ** 2).sum(0)
    rhs1 = 0.01 * ((F ** 2).sum(0) + (w ** 2).sum(0)) + 0.5
    du, dv = np.zeros_like(F), np.zeros_like(F)
    du[:, :, :-1] = F[:, :, :-1] - F[:, :, 1:]
    dv[:, :-1, :] = F[:, :-1, :] - F[:, 1:, :]
    lhs2 = (du ** 2).sum(0) + (dv ** 2).sum(0)
    rhs2 = 0.01 * (F ** 2).sum(0) + 0.002
    return lhs1, rhs1, lhs2, rhs2


def flow_occlusion(fw, bw):
    """O_t of every pair: fw, bw [N,2,H,W] -> uint8 [N,H,W], 1 = occluded"""
    out = []
    for F, B in zip(_as_flows(fw), _as_flows(bw)):
        l1, r1, l2, r2 = occlusion_sides(F, B)
        out.append(((l1 > r1) | (l2 > r2)).astype(np.uint8))
    return np.stack(out)


def undecided(fw, bw, margin=MARGIN):
    """bool [N,H,W]: a test within margin * (1 + rhs) of its threshold"""
    out = []
    for F, B in zip(_as_flows(fw), _as_flows(bw)):
        l1, r1, l2, r2 = occlusion_sides(F, B)
        out.append((np.abs(l1 - r1) <= margin * (1 + r1)) | (np.abs(l2 - r2) <= margin * (1 + r2)))
    return np.stack(out)


def warp_error_sums(frames_u8, fw, occ):
    """(sum of squared differences over the non-occluded pixels and channels, N_t) per pair: float64 [T-1,2]"""
    R = np.asarray(frames_u8, np.float64).transpose(0, 3, 1, 2) / 255.0
    out = []
    for t, (F, O) in enumerate(zip(_as_flows(fw), np.asarray(occ))):
        d = ((sample(R[t + 1], F) - R[t]) ** 2).sum(0)
        keep = O == 0
        out.append((d[keep].sum(), float(keep.sum())))
    return np.array(out, np.float64).reshape(-1, 2)


def per_pair(sums):
    """E_t from warp_error_sums: sum / (3 N_t), 0 where N_t = 0"""
    s, n = sums[:, 0], sums[:, 1]
    return np.where(n > 0, s / np.maximum(3 * n, 1), 0.0)


def warp_error(frames_u8, fw, bw=None, occ=None):
    """E_t of every pair, float64 [T-1]; the occlusion map is computed from fw / bw unless given"""
    occ = flow_occlusion(fw, bw) if occ is None else occ
    return per_pair(warp_error_sums(frames_u8, fw, occ))


def ewarp(frames_u8, fw, bw=None, occ=None):
    """E_warp of one video: the mean of E_t over its T-1 pairs"""
    return float(warp_error(frames_u8, fw, bw, occ).mean())
