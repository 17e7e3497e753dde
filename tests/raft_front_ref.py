"""TEST HARNESS ONLY: float64 references, error bounds and input generators for RAFT's fp32 front end -- the all-pairs
correlation (pp_corr_build, pp_corr_pool_pyramid), the feature pyramid of the on-the-fly plan (pp_corr_fmap_pyramid), the
lookups (TMA, plain-load and on-the-fly, radius 4 and 3), convex upsampling and the encoder's instance norm.  Shared by
the device tests (test_gpu_raft_front_f64.py), the fp16 lookup tests (test_gpu_half_kernels_f64.py) and the host build of
the same rules (test_raft_front_bounds_host.py).  Every function takes torch tensors on any device.

u = 2^-24 is the unit roundoff of fp32 (round to nearest); each bound below counts the roundings of the kernel's
expression and keeps the count as its constant."""
import math

import numpy as np
import torch

U = 2.0 ** -24
TINY = 2.0 ** -126          # fp32 has no relative accuracy below its smallest normal


# ----------------------------------------------------------------------------------------------- correlation lookups
def grid_sample_coord32(c, lvl, size, radius=4):
    """the plain-load and on-the-fly kernels' sampling coordinate (pp_corr_tap_r): c / 2^lvl + (a - R) for the K = 2R+1
    taps a, through grid_sample's align_corners=True normalise / unnormalise round trip, every step one IEEE fp32
    operation (numpy); c [P] fp32 -> [P, K] float64"""
    f = np.float32
    x = c.cpu().numpy().astype(f)[:, None] / f(2 ** lvl) + np.arange(-radius, radius + 1, dtype=f)[None, :]
    g = (f(2) * x) / f(size - 1) - f(1)
    return torch.from_numpy((((g + f(1)) / f(2)) * f(size - 1)).astype(np.float64)).to(c.device)


def lookup64(planes, coords, grid_sample32=False, radius=4, swap_xy=False, drop_corner=None, corners=False):
    """float64 CorrBlock lookup (oracle/ops_ref.corr_lookup without its final .float()): planes = 4 float64 levels
    [P, hl, wl], coords [..., 2] (x, y) with P pixels -> (taps [P, 4K^2], s [P, 4K^2] = sum of |weight * corner|), K = 2R+1.
    Channel l*K^2 + a*K + b samples (x + a - R, y + b - R) at level l (the reference's window-axis quirk).  The TMA kernel
    samples at these exact coordinates; the plain-load and on-the-fly kernels follow grid_sample's fp32 coordinate round
    trip (grid_sample32=True), which can move a sample by a few fp32 ulps of the coordinate.  Non-finite centres give 0.
    swap_xy / drop_corner (0-3) build the wrong references the bounds must reject.  corners=True also returns
    v [P, 4K^2] = sum of |corner| over the in-range corners (for lookup_bound)."""
    P = planes[0].shape[0]
    K = 2 * radius + 1
    c = coords.reshape(P, 2).double()
    c = torch.where(torch.isfinite(c).all(1, keepdim=True), c, torch.full_like(c, -1e9))
    d = torch.arange(-radius, radius + 1, dtype=torch.float64, device=c.device)
    outs, mags, vs = [], [], []
    for l, pl in enumerate(planes):
        hl, wl = pl.shape[1:]
        if grid_sample32:
            c32 = c.float()
            x = grid_sample_coord32(c32[:, 0], l, wl, radius)[:, :, None].expand(P, K, K)
            y = grid_sample_coord32(c32[:, 1], l, hl, radius)[:, None, :].expand(P, K, K)
        else:
            x = (c[:, 0, None, None] / 2 ** l + d[None, :, None]).expand(P, K, K)
            y = (c[:, 1, None, None] / 2 ** l + d[None, None, :]).expand(P, K, K)
        if swap_xy:
            x, y = x.transpose(1, 2), y.transpose(1, 2)
        x0, y0 = x.floor(), y.floor()
        fx, fy = x - x0, y - y0
        flat = pl.reshape(P, -1)
        o, m, va = 0, 0, 0
        cs = ((0, 0, (1 - fx) * (1 - fy)), (1, 0, fx * (1 - fy)), (0, 1, (1 - fx) * fy), (1, 1, fx * fy))
        for k, (dx, dy, wgt) in enumerate(cs):
            if k == drop_corner:
                continue
            xi, yi = x0 + dx, y0 + dy
            ok = (xi >= 0) & (xi <= wl - 1) & (yi >= 0) & (yi <= hl - 1)
            idx = (yi.clamp(0, hl - 1) * wl + xi.clamp(0, wl - 1)).long().reshape(P, K * K)
            v = torch.where(ok, torch.gather(flat, 1, idx).view(P, K, K), 0.0)
            o = o + wgt * v
            m = m + (wgt * v).abs()
            va = va + v.abs()
        outs.append(o.reshape(P, K * K))
        mags.append(m.reshape(P, K * K))
        vs.append(va.reshape(P, K * K))
    if corners:
        return torch.cat(outs, 1), torch.cat(mags, 1), torch.cat(vs, 1)
    return torch.cat(outs, 1), torch.cat(mags, 1)


def planes64(levels, h, w, pairs=None):
    """the device pyramid (row-padded planes) as float64 [P, hl, wl], optionally only the pixels of `pairs`"""
    out, hl, wl = [], h, w
    for lv in levels:
        v = lv if pairs is None else torch.cat([lv[p * h * w:(p + 1) * h * w] for p in pairs])
        out.append(v[:, :, :wl].double())
        hl, wl = hl // 2, wl // 2
    return out


def lookup_coords(B, h, w, seed, device="cuda", nonfinite=False):
    """per pixel, by index mod 6: uniform +-6 px around the grid, exact integers, half-integers at level (i // 6) % 4,
    the borders (x = w-1, y = h-1, -0.5), centres 500 px outside (all-zero windows), uniform +-20 px.  nonfinite=True
    replaces every 7th of the far centres by one of (nan, x), (x, inf), (-inf, nan), which must give all-zero windows too.
    -> (coords [B, h, w, 2] fp32, zero-window mask [B, h, w])"""
    gen = torch.Generator(device=device).manual_seed(seed)
    ys, xs = torch.meshgrid(torch.arange(h, device=device), torch.arange(w, device=device), indexing="ij")
    base = torch.stack([xs, ys], -1).double()[None].expand(B, h, w, 2).reshape(-1, 2)
    n = base.shape[0]
    i = torch.arange(n, device=device)
    kind, sub = (i % 6)[:, None], (i // 6)
    uni = lambda r: (torch.rand(n, 2, generator=gen, device=device, dtype=torch.float64) * 2 - 1) * r  # noqa: E731
    ints = base + torch.randint(-6, 7, (n, 2), generator=gen, device=device)
    lvl = (2.0 ** (sub % 4)).double()[:, None]
    halves = ((base / lvl).floor() + torch.randint(-3, 4, (n, 2), generator=gen, device=device) + 0.5) * lvl
    bx = torch.stack([torch.tensor([w - 1.0, -0.5, w - 1.0, -0.5], device=device)[sub % 4],
                      torch.tensor([h - 1.0, -0.5, -0.5, h - 1.0], device=device)[(sub // 4) % 4]], 1).double()
    border = torch.where(torch.rand(n, 2, generator=gen, device=device) < 0.75, bx, base + uni(3))
    far = base + torch.where((sub % 2 == 0)[:, None], 500.0, -500.0)
    c = torch.where(kind == 0, base + uni(6), base + uni(20))
    for k, v in ((1, ints), (2, halves), (3, border), (4, far)):
        c = torch.where(kind == k, v, c)
    c = c.float()
    if nonfinite:
        nf = (kind[:, 0] == 4) & ((sub // 2) % 7 == 0)
        j = (sub // 14) % 3
        bad = torch.stack([torch.where(j == 0, math.nan, torch.where(j == 2, -math.inf, c[:, 0].double())),
                           torch.where(j == 1, math.inf, torch.where(j == 2, math.nan, c[:, 1].double()))], 1).float()
        c = torch.where(nf[:, None], bad, c)
    return c.view(B, h, w, 2), (kind == 4).view(B, h, w)


def lookup_bound(s, v):
    """fp32 blend of one tap: the weight products and the 4-corner sum, <= 7 roundings of magnitude <= s (2^-21 s), and
    the fractional weights themselves, which the kernels round to within u of the exact ones (x - floor(x) of a small
    negative x is 1 - |x|, rounded): at most 2u per corner weight, times the sum v of |corner|"""
    return 8 * U * s + 2 * U * v + TINY


# ----------------------------------------------------------------------------------------------- correlation volume
def corr64(f1, f2):
    """float64 f1 . f2 / sqrt(D) of [P, D] x [Q, D] fp32 rows -> (C [P, Q], A = sum_k |f1_k f2_k| / sqrt(D))"""
    D = f1.shape[-1]
    a, b = f1.double(), f2.double()
    return a @ b.T / math.sqrt(D), a.abs() @ b.abs().T / math.sqrt(D)


def corr_build_c(D):
    """constant c of |C - C64| <= c 2^-22 A for the 3xTF32 split of k_corr_build.  a = hi + lo with hi = tf32(a),
    |a - hi| <= 2^-11 |a|, lo = tf32(a - hi) rounded again by <= 2^-22 |a|: per product the dropped lo*lo and the two lo
    roundings make 3 * 2^-22 |a b|.  The fp32 accumulator takes 3 mma per 8-deep k-step, D/8 steps, each within 2 ulp
    (2^-22) of a partial sum <= A; the final * 1/sqrt(D) (rounded scale and product) adds 2^-23 A."""
    return 3 + 3 * D / 8 + 1


def tf32_split64(a):
    """(hi, lo) of k_corr_build's split as float64: hi = tf32(a) (round to nearest, ties away), lo = tf32(a - hi)"""
    def rna(v):
        i = v.float().view(torch.int32)
        return ((i + 0x1000) & ~0x1FFF).view(torch.float32)
    hi = rna(a)
    lo = rna(a.float() - hi)
    return hi.double(), lo.double()


def corr_split64(f1, f2, terms):
    """float64 volume of a TF32 split build with `terms` products: 3 (lo*hi + hi*lo + hi*hi), 2 (hi*lo + hi*hi), 1"""
    D = f1.shape[-1]
    ah, al = tf32_split64(f1)
    bh, bl = tf32_split64(f2)
    c = ah @ bh.T
    if terms >= 2:
        c = c + ah @ bl.T
    if terms >= 3:
        c = c + al @ bh.T
    return c / math.sqrt(D)


# ----------------------------------------------------------------------------------------------- pooling
def pool32(v, order=(0, 1, 2, 3)):
    """pp_pool4 in numpy float32: ((a+b)+c)+d then /4 over 2x2 blocks of the last two axes (floor sizes), a, b the top
    row, c, d the bottom row; `order` permutes (a, b, c, d) for the wrong reference"""
    v = np.asarray(v, dtype=np.float32)
    H, W = v.shape[-2] // 2 * 2, v.shape[-1] // 2 * 2
    q = [v[..., 0:H:2, 0:W:2], v[..., 0:H:2, 1:W:2], v[..., 1:H:2, 0:W:2], v[..., 1:H:2, 1:W:2]]
    q = [q[i] for i in order]
    return (((q[0] + q[1]) + q[2]) + q[3]) / np.float32(4)


def pool64(v):
    """float64 2x2 average pooling of the last two axes (floor sizes)"""
    H, W = v.shape[-2] // 2 * 2, v.shape[-1] // 2 * 2
    v = v[..., :H, :W]
    return (v[..., 0::2, 0::2] + v[..., 0::2, 1::2] + v[..., 1::2, 0::2] + v[..., 1::2, 1::2]) / 4


def pool_bound(absavg, levels):
    """`levels` fp32 poolings of a value whose float64 block average of |.| is absavg: each pooling's 3 adds are within
    3u of the mean of |children| (the /4 is exact), and averaging does not amplify an earlier level's error"""
    return 3 * levels * U * absavg + TINY


# ----------------------------------------------------------------------------------------------- on-the-fly lookup
def otf_dot_c(D):
    """k_corr_lookup_otf's dot product: D/32 products per lane (a product, then FFMAs), a 5-level butterfly, then
    / sqrt(D) (x 1/16 exact for D = 256; correctly rounded sqrt and division for D = 128): error <= c u A"""
    return D // 32 + 5 + (0 if D == 256 else 2)


# ----------------------------------------------------------------------------------------------- convex upsampling
def convex64(mask, flow, scale=0.25, no_max32=False):
    """RAFT.upsample_flow in float64: mask [n, h, w, 576] (channel k*64 + i*8 + j), flow [n, h, w, 2] -> (out planar
    [n, 2, 8h, 8w], bound).  softmax over k of scale * mask, blended with 8 * the 3x3 neighbours' flow (zeros outside).
    The bound counts the fp32 roundings of pp_convex_up: the logit difference (u |d_k|, which expf passes on as a
    relative error), expf (2 ulp), the 9-term denominator, the division, and the 9 products and sums of the blend:
    8 u sum_k p_k |f_k| (32 + |d_k| + sum_j p_j |d_j|).  no_max32=True returns the kernel without the max subtraction
    (fp32 expf overflows to inf) as the wrong reference."""
    n, h, w, _ = mask.shape
    lg = scale * mask.double().view(n, h, w, 9, 8, 8)
    if no_max32:
        e = torch.exp(lg.float()).double()
        p = e / e.sum(3, keepdim=True)
    else:
        p = torch.softmax(lg, 3)
    d = (lg - lg.amax(3, keepdim=True)).abs()
    dbar = (p * d).sum(3, keepdim=True)
    f = torch.nn.functional.pad(flow.double().permute(0, 3, 1, 2), (1, 1, 1, 1))           # [n, 2, h+2, w+2]
    nb = torch.stack([f[:, :, ky:ky + h, kx:kx + w] for ky in range(3) for kx in range(3)], 2)  # [n, 2, 9, h, w]
    nb = nb.permute(0, 3, 4, 2, 1)[:, :, :, :, None, None, :]                                # [n, h, w, 9, 1, 1, 2]
    out = (p[..., None] * 8 * nb).sum(3)                                                      # [n, h, w, 8, 8, 2]
    bnd = 8 * U * (p[..., None] * (8 * nb).abs() * (32 + d + dbar)[..., None]).sum(3) + TINY
    to_planar = lambda t: t.permute(0, 5, 1, 3, 2, 4).reshape(n, 2, 8 * h, 8 * w)          # noqa: E731
    return to_planar(out), to_planar(bnd)


# ----------------------------------------------------------------------------------------------- instance norm
def inorm64(x, eps=1e-5, unbiased=False, eps_outside=False):
    """nn.InstanceNorm2d(affine=False) in float64 over the exact fp32 inputs x [n, HW, C] -> (y, mean, k) with
    y = (x - mean) * k, k = 1 / sqrt(var + eps) per (sample, channel).  unbiased / eps_outside build the wrong references."""
    x = x.double()
    mean = x.mean(1, keepdim=True)
    var = ((x - mean) ** 2).sum(1, keepdim=True) / (x.shape[1] - (1 if unbiased else 0))
    k = 1 / (var.sqrt() + eps) if eps_outside else 1 / (var + eps).sqrt()
    return (x - mean) * k, mean, k


INORM_C1, INORM_C2 = 4, 2


def inorm_bound(y, out, mean, k):
    """E = c1 u (|y| + 1) + c2 u k |mean| + u |out|.  With the statistics exact to double precision, the kernel rounds
    the mean to fp32 (u |mean|, times k in the output), rstd to fp32 (u |y|), x - mean (u |y| + u^2 k |mean|) and the
    product (u |y|): c1 = 4 > 3, c2 = 2 > 1.  The residual add rounds once more (u |out|).  The error of subtracting
    an fp32-rounded mean grows as |mean| / std, never as its square."""
    return INORM_C1 * U * (y.abs() + 1) + INORM_C2 * U * k * mean.abs() + U * out.abs()


def inorm_ref(x, res=None, relu=False, post_relu=False, eps=1e-5, **wrong):
    """float64 pp_instance_norm output and its bound: x [n, HW, C] -> (out, bound)"""
    y, mean, k = inorm64(x, eps, **wrong)
    o = y.clamp_min(0) if relu else y
    if res is not None:
        o = o + res.double()
    if post_relu:
        o = o.clamp_min(0)
    return o, inorm_bound(y, o, mean, k)


def inorm_input(gen, n, HW, C, ratio, device, const_channels=0):
    """x [n, HW, C] fp32 with per-channel std ~ 1 and mean = +-ratio * std (the sign alternating by channel), so
    |mean| / std ~ ratio; the first `const_channels` channels hold one non-zero constant each (0.1 + c / 7)"""
    z = torch.randn(n, HW, C, generator=gen, device=device, dtype=torch.float64)
    sd = torch.exp(torch.rand(n, 1, C, generator=gen, device=device, dtype=torch.float64) - 0.5)
    sign = torch.where(torch.arange(C, device=device) % 2 == 0, 1.0, -1.0).double()
    x = (z * sd + ratio * sd * sign).float()
    for c in range(const_channels):
        x[:, :, c] = 0.1 + c / 7
    return x


def ratio_max(x):
    """largest |mean| / std over the (sample, channel) pairs of x [n, HW, C] (std 0 excluded)"""
    x = x.double()
    m, s = x.mean(1), x.std(1, unbiased=False)
    r = m.abs() / s
    return float(r[s > 0].max()) if bool((s > 0).any()) else 0.0


def check(got, ref, bound, what):
    """|got - ref| <= bound everywhere, got finite; -> worst err / bound"""
    got = got.double()
    assert bool(torch.isfinite(got).all()), f"{what}: {int((~torch.isfinite(got)).sum())} non-finite outputs"
    err = (got - ref).abs()
    r = err / bound
    worst = float(r.max()) if r.numel() else 0.0
    bad = err > bound
    if bool(bad.any()):
        i = torch.nonzero(bad.reshape(-1))[:4, 0]
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} beyond the bound, worst {worst:.3g}x; at "
                             f"{i.tolist()}: got {got.reshape(-1)[i].tolist()} ref {ref.reshape(-1)[i].tolist()}")
    return worst


def rejects(ref_wrong, got, bound):
    """a wrong reference is rejected when the kernel's output lies beyond the bound from it somewhere"""
    d = (got.double() - ref_wrong).abs()
    return bool(((d > bound) | ~torch.isfinite(ref_wrong)).any())
