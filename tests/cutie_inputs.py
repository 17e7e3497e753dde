"""Seeded inputs of the Cutie tracker fixtures (tests/golden/make_golden_cutie.py) and tests: a textured clip with two
moving objects, one of which leaves the frame, and its first-frame label mask."""
import numpy as np

CLIP = dict(T=32, H=250, W=430, seed=5)          # odd size, not a multiple of 16; > 5 * mem_every frames so the FIFO evicts
PAIR = dict(H=72, W=100, seed=9)                 # the per-function fixture: two frames and a mask (5x7 = 35 >= 30 tokens)


def _texture(rng, H, W, scale):
    """smooth random colour field (bilinear upsampling of a coarse grid)"""
    gh, gw = H // scale + 2, W // scale + 2
    g = rng.uniform(0, 255, (gh, gw, 3))
    ys = np.linspace(0, gh - 1.001, H)
    xs = np.linspace(0, gw - 1.001, W)
    y0, x0 = ys.astype(int), xs.astype(int)
    fy, fx = (ys - y0)[:, None, None], (xs - x0)[None, :, None]
    a = g[y0][:, x0] * (1 - fx) + g[y0][:, x0 + 1] * fx
    b = g[y0 + 1][:, x0] * (1 - fx) + g[y0 + 1][:, x0 + 1] * fx
    return a * (1 - fy) + b * fy


def make_clip(T, H, W, seed, ids=(1, 2)):
    """-> frames uint8 [T,H,W,3], label masks uint8 [T,H,W] (ids[0]: an ellipse drifting down-right; ids[1]: a square
    leaving through the right edge)"""
    rng = np.random.default_rng(seed)
    bg = _texture(rng, H, W, 24)
    tex = [_texture(rng, H, W, 6) * 0.5 + np.array(c) * 0.5 for c in ((230, 40, 40), (40, 60, 230))]
    yy, xx = np.mgrid[0:H, 0:W]
    frames = np.empty((T, H, W, 3), np.uint8)
    masks = np.zeros((T, H, W), np.uint8)
    for t in range(T):
        img = bg.copy()
        cy, cx = 0.35 * H + 1.2 * t, 0.30 * W + 2.0 * t
        e = ((yy - cy) / (0.18 * H)) ** 2 + ((xx - cx) / (0.12 * W)) ** 2 <= 1
        sy, sx, s = int(0.55 * H), int(0.55 * W + 9.0 * t), int(0.22 * H)
        q = (yy >= sy) & (yy < sy + s) & (xx >= sx) & (xx < sx + s)
        img[e] = tex[0][e]
        img[q] = tex[1][q]
        frames[t] = np.clip(img + rng.normal(0, 4, img.shape), 0, 255).astype(np.uint8)
        masks[t][e] = ids[0]
        masks[t][q] = ids[1]
    return frames, masks
