"""Float64 references and per-element error bounds for the gather kernels of the propagation scans (test harness only).

The rules live in propainter_b200/csrc/pp_elem.cuh.  Their references, restated here from the semantics pp_elem.cuh cites:

  * flow_warp (model/modules/flow_loss_utils.py:6-45) samples at g = 2*(p+f)/max(size-1,1) - 1 unnormalised by ATen's
    align_corners=True rule ((g+1)/2)*(size-1).  `warp_coord32` restates that in numpy float32, one rounding per
    operation, as pp_warp_coord does: the sampling position of a flow warp is bit-exact, and so is everything that
    depends on the position alone (the `nearest` pick, the in-image test, the integer corner).
  * The bilinear samples are sums of four weighted corners.  The kernels' sums may be contracted into FMAs, the host
    build's are not, so neither is a bit-exact reference; the samples are compared with float64 evaluated at the exact
    fp32 position, within a per-element bound E (below).
  * The deformable tap position max_res * tanhf(o) + flow + base is not bit-exact either (tanhf is within 2 ulp): it
    carries a position error dp, which enters E through the local slope of the sampled map.
  * Discontinuous decisions (the forward-backward validity and the 0.1 mask binarisations) are compared by margin: the
    float64 quantity, a bound on its fp32 evaluation error, and "undecided" inside that band.

Error bounds (u = 2^-24, first order; see each constant):
  E = dp * G + REL * sum_j |w_j v_j| + TINY
  G = 2 m max|v| over the 4 x 4 pixels around the cell, a Lipschitz bound of the bilinear sample (zeros padding is
      continuous) that also covers a position error moving the sample into a neighbouring cell.
"""
import numpy as np
import torch
import torch.nn.functional as F

U = 2.0 ** -24
# pp_taps + pp_tap_plane / pp_tap_nhwc4: a corner weight wx*wy has three roundings ((xf+1)-ix, (yf+1)-iy, the product),
# the weighted corner one more, and the four-term sum three (with or without FMA): 7u of sum|w v|, plus 1u of slack for
# the second-order terms.
REL_WARP = 8 * U
# pp_deform_weights + pp_deform_sample1 / da_combine / k_deform_gather: hy, hx (1u each), hy*hx (1u), *m (1u), the
# modulation 1/(1+expf(-l)) itself (expf within 2 ulp: 2u, the add and the division: 2u), the weighted corner (1u), the
# four-term sum (3u): 12u, plus 1u of slack.
REL_DEFORM = 13 * U
TINY = 2.0 ** -110
F01 = float(np.float32(0.01))           # the reference's a1 = 0.01 meets fp32 tensors as 0.01f
F_TENTH = float(np.float32(0.1))        # binary_mask's threshold 0.1 (fp32 masks)
TF32_MID = 0x1000


# ------------------------------------------------------------------------------------------------ coordinates
def warp_coord32(base, flow, size):
    """pp_warp_coord in numpy float32, one rounding per operation (exact: it is the reference's own fp32 expression)."""
    f32 = np.float32
    base, flow = np.asarray(base, np.float32), np.asarray(flow, np.float32)
    g = (f32(2.0) * (base + flow)) / f32(max(size - 1, 1)) - f32(1.0)
    return ((g + f32(1.0)) / f32(2.0)) * f32(size - 1)


def warp_positions(flow_xy, fault=None):
    """flow [n,h,w,2] (x, y) fp32 (numpy or torch) -> exact fp32 sampling positions (ix, iy) as numpy [n,h*w].
    fault="swap": dx and dy exchanged (a wrong reference for the bound-rejection checks)."""
    f = flow_xy.detach().cpu().numpy() if isinstance(flow_xy, torch.Tensor) else np.asarray(flow_xy)
    n, h, w, _ = f.shape
    ys, xs = np.meshgrid(np.arange(h, dtype=np.float32), np.arange(w, dtype=np.float32), indexing="ij")
    fx, fy = (f[..., 1], f[..., 0]) if fault == "swap" else (f[..., 0], f[..., 1])
    return warp_coord32(xs, fx, w).reshape(n, h * w), warp_coord32(ys, fy, h).reshape(n, h * w)


# ------------------------------------------------------------------------------------------------ bilinear sampling
def bilinear(src, ix, iy, fault=None):
    """Bilinear sample, zeros padding (grid_sample / torchvision bilinear_interpolate corner rule), in float64.
    src [n,h,w,G,c]; ix, iy float64 [n,P,G] -> (value [n,P,G,c], sum_j |w_j v_j| [n,P,G,c]).
    fault="corner": the lower-right corner dropped; "shift": the map read one pixel to the right."""
    n, h, w, G, c = src.shape
    flat = src.reshape(n, h * w * G, c)
    inside = (ix > -1) & (ix < w) & (iy > -1) & (iy < h)
    x0, y0 = torch.floor(ix), torch.floor(iy)
    lx, ly = ix - x0, iy - y0
    gidx = torch.arange(G, device=src.device).view(1, 1, G)
    val = torch.zeros(ix.shape + (c,), dtype=torch.float64, device=src.device)
    ab = torch.zeros_like(val)
    for dy, dx, wt in ((0, 0, (1 - ly) * (1 - lx)), (0, 1, (1 - ly) * lx), (1, 0, ly * (1 - lx)), (1, 1, ly * lx)):
        if fault == "corner" and dy == 1 and dx == 1:
            continue
        yi, xi = y0 + dy, x0 + dx + (1 if fault == "shift" else 0)
        ok = inside & (yi >= 0) & (yi <= h - 1) & (xi >= 0) & (xi <= w - 1)
        lin = ((yi.clamp(0, h - 1) * w + xi.clamp(0, w - 1)).long() * G + gidx).reshape(n, -1, 1).expand(-1, -1, c)
        v = torch.gather(flat, 1, lin).view(val.shape)
        term = v * torch.where(ok, wt, torch.zeros_like(wt)).unsqueeze(-1)
        val += term
        ab += term.abs()
    return val, ab


def max4(src):
    """src [n,h,w,G,c] -> [n,h+1,w+1,G,c]: entry (y0+1, x0+1) = max |src| over rows y0-1..y0+2, columns x0-1..x0+2."""
    n, h, w, G, c = src.shape
    a = src.abs().reshape(n, h, w, G * c).permute(0, 3, 1, 2)
    m = F.max_pool2d(F.pad(a, (2, 2, 2, 2)), 4, 1)
    return m.permute(0, 2, 3, 1).reshape(n, h + 1, w + 1, G, c)


def gather_cell(m4, ix, iy):
    """m4 from max4, positions [n,P,G] -> [n,P,G,c] at the (clamped) cell of each position."""
    n, hp, wp, G, c = m4.shape
    x0 = torch.floor(ix).clamp(-1, wp - 2) + 1
    y0 = torch.floor(iy).clamp(-1, hp - 2) + 1
    gidx = torch.arange(G, device=m4.device).view(1, 1, G)
    lin = ((y0 * wp + x0).long() * G + gidx).reshape(n, -1, 1).expand(-1, -1, c)
    return torch.gather(m4.reshape(n, hp * wp * G, c), 1, lin).view(ix.shape + (c,))


def warp_sample(feat64, ix, iy, fault=None):
    """flow_warp of pixel-major maps: feat64 [n,h,w,C], exact positions (numpy [n,P]) -> (ref [n,P,C], E [n,P,C])."""
    dev = feat64.device
    tx = torch.from_numpy(np.asarray(ix, np.float64)).to(dev).unsqueeze(-1)
    ty = torch.from_numpy(np.asarray(iy, np.float64)).to(dev).unsqueeze(-1)
    v, ab = bilinear(feat64.unsqueeze(3), tx, ty, fault)
    return v[:, :, 0], REL_WARP * ab[:, :, 0] + TINY


def nearest_sample(img64, ix, iy):
    """grid_sample mode='nearest' (rintf, half to even; zeros padding) of img64 [n,h,w,C] at exact positions [n,P]."""
    n, h, w, C = img64.shape
    dev = img64.device
    xn = torch.from_numpy(np.rint(np.asarray(ix, np.float64))).to(dev)
    yn = torch.from_numpy(np.rint(np.asarray(iy, np.float64))).to(dev)
    ok = (xn >= 0) & (xn <= w - 1) & (yn >= 0) & (yn <= h - 1)
    lin = (yn.clamp(0, h - 1) * w + xn.clamp(0, w - 1)).long().unsqueeze(-1).expand(-1, -1, C)
    v = torch.gather(img64.reshape(n, h * w, C), 1, lin)
    return torch.where(ok.unsqueeze(-1), v, torch.zeros_like(v))


# ------------------------------------------------------------------------------------------------ decisions by margin
def fb_margin(fx, fy, bx, by, ebx, eby):
    """fbConsistencyCheck (model/propainter.py:22-31) as pp_fb_valid evaluates it, in float64 from the exact fp32 flow
    (fx, fy) and the float64 samples (bx, by) of the check flow, whose fp32 evaluation is within (ebx, eby).
    Returns (valid, decided): the float64 decision lhs < thr, and whether |lhs - thr| exceeds twice the first-order bound
    of the fp32 evaluation error of lhs - thr (samples, then one rounding per operation of pp_fb_valid)."""
    dx, dy = fx + bx, fy + by
    lhs = dx * dx + dy * dy
    mag = (fx * fx + fy * fy) + (bx * bx + by * by)
    thr = F01 * mag + 0.5
    ddx = ebx + U * (fx.abs() + bx.abs() + ebx)                    # dx = fl(fx + bx~)
    ddy = eby + U * (fy.abs() + by.abs() + eby)
    dlhs = (2 * dx.abs() + ddx) * ddx + (2 * dy.abs() + ddy) * ddy + 3 * U * (lhs + ddx * ddx + ddy * ddy)
    dmag = (2 * bx.abs() + ebx) * ebx + (2 * by.abs() + eby) * eby + 4 * U * (mag + ebx * ebx + eby * eby)
    dthr = F01 * dmag + 2 * U * thr
    band = 2 * (dlhs + dthr) + TINY
    return lhs < thr, (lhs - thr).abs() > band


def threshold_margin(s, e, thr=F_TENTH):
    """s > thr for a float64 sample s whose fp32 evaluation is within e -> (decision, decided)."""
    return s > thr, (s - thr).abs() > e


def fb_valid32(fx, fy, bx, by):
    """pp_fb_valid in numpy float32, one rounding per operation (exact where bx, by are exact samples)."""
    f32 = np.float32
    fx, fy, bx, by = (np.asarray(a, np.float32) for a in (fx, fy, bx, by))
    dx, dy = fx + bx, fy + by
    lhs = dx * dx + dy * dy
    mag = (fx * fx + fy * fy) + (bx * bx + by * by)
    thr = f32(0.01) * mag + f32(0.5)
    return lhs < thr, lhs == thr


def fb_ties(fx, fy, count, span=300):
    """Check-flow values (bx, by) for which pp_fb_valid's fp32 lhs equals its threshold exactly, for the flow (fx, fy):
    searched on the float32 grid around the circle lhs = thr."""
    f32 = np.float32
    out = []
    for ang in np.linspace(0.1, 6.2, 64):
        # radius of the circle |d| = rho, d = f + b, on which lhs = thr in exact arithmetic: 0.99 rho^2 + 0.02 rho (f.e)
        # - (0.02 |f|^2 + 0.5) = 0
        fe, ff = fx * np.cos(ang) + fy * np.sin(ang), fx * fx + fy * fy
        r = (-0.02 * fe + np.sqrt((0.02 * fe) ** 2 + 4 * 0.99 * (0.02 * ff + 0.5))) / (2 * 0.99)
        bx0, by0 = f32(-fx + r * np.cos(ang)), f32(-fy + r * np.sin(ang))
        bx = bx0 + np.arange(-span, span + 1, dtype=np.float32) * np.spacing(bx0)
        by = by0 + np.arange(-span, span + 1, dtype=np.float32)[:, None] * np.spacing(by0)
        bx, by = np.broadcast_arrays(bx.astype(np.float32), by.astype(np.float32))
        _, tie = fb_valid32(np.full_like(bx, fx), np.full_like(bx, fy), bx, by)
        k = np.argwhere(tie)
        if len(k):
            out.append((float(bx[tuple(k[0])]), float(by[tuple(k[0])])))
        if len(out) >= count:
            break
    return out


# ------------------------------------------------------------------------------------------------ TF32 outputs
def tf32_ulp(a):
    """TF32 ulp (10 explicit mantissa bits) of |a| (float64), 0 where a == 0."""
    _, ex = torch.frexp(a.abs())
    ulp = torch.ldexp(torch.ones_like(a), (ex - 11).to(torch.int64))
    return torch.where(a == 0, torch.zeros_like(a), ulp)


def tf32_rna(a):
    """float64 -> nearest TF32 value, ties away from zero (cvt.rna.tf32.f32)."""
    ulp = tf32_ulp(a)
    q = a.abs() / torch.where(ulp == 0, torch.ones_like(ulp), ulp)
    return torch.sign(a) * torch.floor(q + 0.5) * ulp


def check_tf32(got, ref, E, stats):
    """TF32-rounded fp32 outputs `got` against float64 `ref` within E (before rounding).  Asserts: low 13 bits zero;
    |got - ref| <= ulp/2 + E; got == rna(ref) wherever ref lies further than E from a TF32 midpoint.  Accumulates the
    signed rounding error (in ulp, towards |ref|) of those decided elements into stats for the bias check."""
    assert ((got.view(torch.int32) & 0x1FFF) == 0).all(), "TF32 output has low mantissa bits set"
    g = got.double()
    err = (g - ref).abs()
    lim = 0.5 * tf32_ulp(ref.abs() + E) + E
    bad = err > lim
    assert not bad.any(), f"{int(bad.sum())} TF32 outputs outside ulp/2 + E, worst err/lim {(err / lim).max().item():.3g}"
    ulp = tf32_ulp(ref)
    q = ref.abs() / torch.where(ulp == 0, torch.ones_like(ulp), ulp)
    dist = (q - torch.floor(q) - 0.5).abs() * ulp
    decided = (dist > E) & (ulp > 0)
    exp = tf32_rna(ref)
    wrong = decided & (g != exp)
    assert not wrong.any(), f"{int(wrong.sum())} decided TF32 outputs differ from rna(ref)"
    s = (torch.sign(ref) * (g - ref) / torch.where(ulp == 0, torch.ones_like(ulp), ulp))[decided]
    stats["n"] = stats.get("n", 0) + int(decided.sum())
    stats["total"] = stats.get("total", 0) + g.numel()
    stats["sum"] = stats.get("sum", 0.0) + float(s.sum())
    stats["worst"] = max(stats.get("worst", 0.0), float((err / lim).max()) if err.numel() else 0.0)


def check_bound(got, ref, E, what):
    """|got - ref| <= E everywhere; returns the worst err / E."""
    err = (got.double() - ref).abs()
    r = err / E
    bad = ~(err <= E)
    assert not bad.any(), f"{what}: {int(bad.sum())} elements outside the bound, worst err/E {r.max().item():.3g}"
    return float(r.max()) if r.numel() else 0.0


def bound_rejects(got, ref, E):
    """True when the wrong reference `ref` fails the same element bound (the bound is not vacuous)."""
    return bool(((got.double() - ref).abs() > E).any())


# ------------------------------------------------------------------------------------------------ deformable sampling
def deform_cols_ref(x64, o32, flow32, max_res, k, fault=None):
    """Tap k (0..8) of torchvision.ops.deform_conv2d's modulated columns as DeformableAlignment /
    SecondOrderDeformableAlignment compute them (model/propainter.py:58-69, recurrent_flow_completion.py:34-44):
    offset = max_res * tanh(o) (+ flow.flip), mask = sigmoid, 16 offset groups, channel c in group c // (Cin/16).
    x64 [n,H,W,Cin] float64; o32 [n,H,W,>=432] fp32 with the bias already added in fp32 (as the kernels add it); flow32
    [n,H,W,2] | None.  Returns (ref [n,H*W,Cin], E [n,H*W,Cin]) in float64.
    fault: "swap" (dy/dx exchanged), "noflip" (flow added unflipped), "corner", "shift" (see bilinear), "group" (each
    group sampled at the next group's offsets)."""
    n, H, W, Cin = x64.shape
    dev = x64.device
    G, cpg = 16, Cin // 16
    g = torch.arange(G, device=dev)
    if fault == "group":
        g = (g + 1) % G
    o = o32.reshape(n, H * W, -1).double()
    oy, ox = o[..., g * 18 + 2 * k], o[..., g * 18 + 2 * k + 1]
    if fault == "swap":
        oy, ox = ox, oy
    ml = o[..., 288 + g * 9 + k]
    ty, tx = torch.tanh(oy), torch.tanh(ox)
    ay, ax = max_res * ty, max_res * tx
    by, bx = ay, ax
    if flow32 is not None:
        fl = flow32.reshape(n, H * W, 1, 2).double()
        fy, fx = (fl[..., 0], fl[..., 1]) if fault == "noflip" else (fl[..., 1], fl[..., 0])
        by, bx = ay + fy, ax + fx
    ys, xs = torch.meshgrid(torch.arange(H, device=dev, dtype=torch.float64), torch.arange(W, device=dev, dtype=torch.float64),
                            indexing="ij")
    py = (ys.reshape(1, -1, 1) - 1 + k // 3) + by
    px = (xs.reshape(1, -1, 1) - 1 + k % 3) + bx
    # fp32 position error: tanhf within 2 ulp (2^-22 relative) scaled by max_res, then one rounding of each of
    # max_res * t, (+ flow) and (+ base); doubled for the second-order terms
    dpy = 2 * (max_res * 2.0 ** -22 * ty.abs() + U * (ay.abs() + by.abs() + py.abs())) + TINY
    dpx = 2 * (max_res * 2.0 ** -22 * tx.abs() + U * (ax.abs() + bx.abs() + px.abs())) + TINY
    m = torch.sigmoid(ml).unsqueeze(-1)
    xs5 = x64.reshape(n, H, W, G, cpg)
    v, ab = bilinear(xs5, px, py, "corner" if fault == "corner" else ("shift" if fault == "shift" else None))
    G4 = 2 * gather_cell(max4(xs5), px, py)
    E = (dpy + dpx).unsqueeze(-1) * m * G4 + REL_DEFORM * m * ab + TINY
    return (v * m).reshape(n, H * W, Cin), E.reshape(n, H * W, Cin)


# ------------------------------------------------------------------------------------------------ deformable alignment
def da_splits(npix, nit, sms):
    """mma_kernels.cu's split-K rule for pp_deform_align, restated: 4 CTAs of 32 pixels per SM, cost = waves x (K-steps
    per CTA + 2) x 16 + split count, ties to the smaller factor."""
    ctas, slots = (npix + 31) // 32, 4 * sms
    best, best_cost = 1, None
    for s in range(1, 10):
        waves, steps = (ctas * s + slots - 1) // slots, (nit + s - 1) // s
        cost = waves * (steps + 2) * 16 + (s if s > 1 else 0)
        if best_cost is None or cost < best_cost:
            best, best_cost = s, cost
    return best
