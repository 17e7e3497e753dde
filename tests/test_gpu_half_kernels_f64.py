"""RAFT's half-precision refinement kernels (config.HALF_OPERANDS, DESIGN.md §4 "Precision") against float64.

Element level, for each fp16 entry point (corr lookup, bias_act, GRU gate / update, motion pack), every case checks:
  (a) the fp16 output equals the fp32 instantiation's output on the upcast inputs rounded by `.half()`, bit for bit (the
      kernels are one template; only the stores differ);
  (b) against a float64 recomputation from the exact input values: fp32 outputs within 2^-20 (|ref| + s) (+ 2^-126, the
      fp32 underflow floor), fp16 outputs within half an fp16 ulp + delta, and equal to rn16(ref) wherever ref lies
      further than delta from a midpoint between fp16 neighbours.  delta = 2^-21 (|ref| + s), where s bounds how the
      element's operands enter the fp32 expression (below).  The fp32 expressions take at most a few roundings and one
      2-ulp expf / tanhf, so their error is below 2^-22 (|ref| + s): delta keeps a factor 2.  A looser 2^-18 would by
      itself exclude more than 1 % of elements (2 delta / ulp16 >= 2^-7);
  (c) the mean signed rounding error, sign(ref) (got - ref) / ulp16(ref) over the outputs the rounding decides, is below
      0.02 in magnitude over >= 10^5 outputs (round-to-nearest: ~0, truncation: -0.5);
  (d) operands and results are channel slices of wider NaN-filled buffers, fp16 ones 8- but not 16-byte aligned, and no
      element outside the written slices changes.
Then pure conversions against numpy bit for bit, the argument checks and empty calls on the device, and one refinement
loop (`_refine_half`) against a float64 emulation that rounds to fp16 exactly where the device path does.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import ops_ref, pipeline_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
F16, F32 = torch.float16, torch.float32
DELTA16 = 2.0 ** -21            # fp16 outputs: delta = DELTA16 (|ref| + s)
REL32 = 2.0 ** -20              # fp32 outputs
TINY32 = 2.0 ** -126            # fp32 has no relative accuracy below its smallest normal (expf overflow -> exactly 0)
C2_NPIX = 158 * 30 * 54         # DESIGN.md §5: the C2 clip's 158 flow pairs on the 30 x 54 feature grid
RAGGED = 611                    # npix * C / 4 leaves a partial last block of 256 threads for every C used here
SLOPE = float(np.float32(0.1))  # the fp32 slope the kernel receives


@pytest.fixture(autouse=True)
def _strict_fp32_library():
    """torch's own convs / matmuls in strict fp32 (the fp16 convs do not use TF32 either way)"""
    a, b = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = a, b


# ----------------------------------------------------------------------------------------------- fp16 arithmetic helpers
def rn16(x):
    """round-to-nearest-even of float64 values to fp16.  numpy converts float64 -> float16 directly; torch on the CPU
    goes through float32 and would round twice."""
    return np.asarray(x, dtype=np.float64).astype(np.float16)


def ulp16(v):
    """fp16 spacing at v: 2^(max(floor(log2|v|), -14) - 10), 2^-24 in the subnormal range"""
    a = np.abs(np.asarray(v, dtype=np.float64))
    e = np.where(a > 0, np.frexp(a)[1] - 1, -14)
    return np.exp2(np.maximum(e, -14) - 10.0)


def mid_dist(v):
    """distance of float64 v to the nearest midpoint between two adjacent fp16 values"""
    v = np.asarray(v, dtype=np.float64)
    r = rn16(v)
    with np.errstate(over="ignore", invalid="ignore"):
        up = np.nextafter(r, np.float16(np.inf)).astype(np.float64)
        dn = np.nextafter(r, np.float16(-np.inf)).astype(np.float64)
        rr = r.astype(np.float64)
        return np.minimum(np.abs(v - (rr + up) / 2), np.abs(v - (rr + dn) / 2))


def rn16_t(t):
    """rn16 of a float64 torch tensor, back on its device as float64"""
    return torch.from_numpy(rn16(t.detach().cpu().numpy()).astype(np.float64)).to(t.device)


def bits(t):
    return t.view(torch.int16 if t.dtype == F16 else torch.int32)


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(bits(a.contiguous()), bits(b.contiguous()))


class Tally:
    """near-midpoint exclusions and the signed rounding error over the fp16 outputs of one test"""

    def __init__(self):
        self.n = self.near = self.nb = 0
        self.bsum = 0.0

    def check(self, what):
        frac, bias = self.near / max(self.n, 1), self.bsum / max(self.nb, 1)
        print(f"{what}: {self.n} fp16 outputs, near-midpoint fraction {frac:.4%}, rounding bias {bias:+.4f} ulp "
              f"over {self.nb} rounded outputs")
        assert frac < 0.01, (what, frac)
        assert self.nb >= 100_000 and abs(bias) < 0.02, (what, self.nb, bias)


def _first(what, why, bad, g, r):
    i = np.flatnonzero(bad)[:4]
    return f"{what}: {int(bad.sum())} of {bad.size} {why}; at {i.tolist()}: got {g[i].tolist()} ref {r[i].tolist()}"


def check_f16(got, ref, s, what, tally=None, chunk=1 << 22):
    """fp16 tensor `got` against the float64 tensor `ref` (same shape) with operand magnitude `s` (broadcastable):
    within half an ulp + delta, rn16(ref) bit for bit away from midpoints.  Prints and returns the near-midpoint fraction
    and the rounding bias of this case; adds both to `tally`."""
    assert got.dtype == F16 and got.shape == ref.shape, (what, got.dtype, got.shape, ref.shape)
    g_all, r_all = got.detach().reshape(-1), ref.reshape(-1)
    s_all = torch.broadcast_to(torch.as_tensor(s, dtype=torch.float64, device=ref.device), ref.shape).reshape(-1)
    n, near, bsum, nb = r_all.numel(), 0, 0.0, 0
    for i in range(0, n, chunk):
        g16 = g_all[i:i + chunk].cpu().numpy()
        r, sv = r_all[i:i + chunk].cpu().numpy(), s_all[i:i + chunk].cpu().numpy()
        g = g16.astype(np.float64)
        d = DELTA16 * (np.abs(r) + sv)
        u = ulp16(r)
        bad = ~(np.abs(g - r) <= 0.5 * u + d)
        assert not bad.any(), _first(what, "beyond half an fp16 ulp + delta", bad, g, r)
        r16 = rn16(r)
        far = mid_dist(r) > d
        neq = far & (g16 != r16)
        assert not neq.any(), _first(what, "not rn16(ref) away from a midpoint", neq, g, r)
        near += int((~far).sum())
        ex = r16.astype(np.float64) != r                 # outputs whose value the rounding decides
        bsum += float(np.sum(np.sign(r[ex]) * (g[ex] - r[ex]) / u[ex]))
        nb += int(ex.sum())
    frac, bias = near / max(n, 1), bsum / max(nb, 1)
    print(f"  {what}: near-midpoint {frac:.4%}, rounding bias {bias:+.4f} ulp ({nb} of {n} rounded)")
    if tally is not None:
        tally.n += n
        tally.near += near
        tally.bsum += bsum
        tally.nb += nb
    return frac, bias


def check_f32(got, ref, s, what):
    assert got.dtype == F32 and got.shape == ref.shape, (what, got.dtype, got.shape, ref.shape)
    err = (got.double() - ref).abs()
    bound = REL32 * (ref.abs() + s) + TINY32
    ok = err <= bound
    assert bool(ok.all()), f"{what}: {int((~ok).sum())} fp32 outputs off, worst {float((err / bound).max()):.3g}x the bar"


# ----------------------------------------------------------------------------------------------- sentinel buffers
SENTINEL = {F16: 0x7E5A, F32: 0x7FC5A5A5}        # NaN payloads


class Slot:
    """`t`: channels [c0, c0 + C) of pixel rows `ld` wide, in a flat buffer whose row 0 starts `off` elements in and which
    is otherwise filled with a NaN sentinel.  off = 4 puts fp16 rows 8 bytes (not 16) and fp32 rows 16 bytes in."""

    def __init__(self, lead, C, dtype, ld=None, c0=0, off=4):
        self.lead, self.C, self.ld, self.c0, self.off = tuple(lead), C, C if ld is None else ld, c0, off
        self.n = math.prod(self.lead)
        self.flat = torch.empty(off + self.n * self.ld + 8, dtype=dtype, device=DEV)
        bits(self.flat).fill_(SENTINEL[dtype])
        self.t = self._rows(self.flat)[..., c0:c0 + C]
        self.snap()

    def _rows(self, flat):
        return flat[self.off:self.off + self.n * self.ld].view(*self.lead, self.ld)

    def set(self, v):
        self.t.copy_(v)
        self.snap()
        return self

    def snap(self):
        self.before = self.flat.clone()

    def intact(self, lo=0, hi=None):
        """every element outside t[..., lo:hi] holds what it held at the last snap()"""
        hi = self.C if hi is None else hi
        m = torch.zeros(self.flat.shape, dtype=torch.bool, device=DEV)
        self._rows(m)[..., self.c0 + lo:self.c0 + hi] = True
        return torch.equal(bits(self.flat)[~m], bits(self.before)[~m])

    def unchanged(self):
        return torch.equal(bits(self.flat), bits(self.before))


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _randn(gen, *shape, scale=1.0):
    return torch.randn(*shape, generator=gen, device=DEV) * scale


def _spiked(gen, shape, scale, spikes=(30.0, 100.0), frac=0.02):
    """normal values with a fraction of +-30 (the sigmoid saturates to exactly 1 in fp32) and +-100 (expf overflows:
    exactly 0)"""
    x = _randn(gen, *shape, scale=scale)
    u = torch.rand(*shape, generator=gen, device=DEV)
    sgn = torch.where(torch.rand(*shape, generator=gen, device=DEV) < 0.5, -1.0, 1.0)
    for k, v in enumerate(spikes):
        x = torch.where((u >= k * frac) & (u < (k + 1) * frac), sgn * v, x)
    return x


def _with_subnormals(gen, shape, scale, frac=0.1):
    """normal values with a fraction in the fp16 subnormal range (|v| < 2^-14)"""
    x = _randn(gen, *shape, scale=scale)
    tiny = (torch.rand(*shape, generator=gen, device=DEV) * 2 - 1) * 2.0 ** -14
    return torch.where(torch.rand(*shape, generator=gen, device=DEV) < frac, tiny, x)


# ----------------------------------------------------------------------------------------------- correlation lookup
def grid_sample_coord32(c, lvl, size):
    """the plain-load kernel's sampling coordinate (pp_corr_tap_r): c / 2^lvl + (a - 4) for the 9 taps a, through
    grid_sample's align_corners=True normalise / unnormalise round trip, every step one IEEE fp32 operation (numpy);
    c [P] fp32 -> [P, 9] float64"""
    f = np.float32
    x = c.cpu().numpy().astype(f)[:, None] / f(2 ** lvl) + np.arange(-4, 5, dtype=f)[None, :]
    g = (f(2) * x) / f(size - 1) - f(1)
    return torch.from_numpy((((g + f(1)) / f(2)) * f(size - 1)).astype(np.float64)).to(c.device)


def lookup64(planes, coords, grid_sample32=False):
    """float64 CorrBlock lookup (oracle/ops_ref.corr_lookup without its final .float()): planes = 4 float64 levels
    [P, hl, wl], coords [..., 2] (x, y) with P pixels -> (taps [P, 324], s [P, 324] = sum of |weight * corner|).  Channel
    l*81 + a*9 + b samples (x + a - 4, y + b - 4) at level l (the reference's window-axis quirk).  The TMA kernel samples
    at these exact coordinates; the plain-load kernel follows grid_sample's fp32 coordinate round trip
    (grid_sample32=True), which can move a sample by a few fp32 ulps of the coordinate."""
    P = planes[0].shape[0]
    c = coords.reshape(P, 2).double()
    d = torch.arange(-4, 5, dtype=torch.float64, device=c.device)
    outs, mags = [], []
    for l, pl in enumerate(planes):
        hl, wl = pl.shape[1:]
        if grid_sample32:
            x = grid_sample_coord32(coords.reshape(P, 2)[:, 0], l, wl)[:, :, None].expand(P, 9, 9)
            y = grid_sample_coord32(coords.reshape(P, 2)[:, 1], l, hl)[:, None, :].expand(P, 9, 9)
        else:
            x = (c[:, 0, None, None] / 2 ** l + d[None, :, None]).expand(P, 9, 9)
            y = (c[:, 1, None, None] / 2 ** l + d[None, None, :]).expand(P, 9, 9)
        x0, y0 = x.floor(), y.floor()
        fx, fy = x - x0, y - y0
        flat = pl.reshape(P, -1)
        o, m = 0, 0
        for dx, dy, wgt in ((0, 0, (1 - fx) * (1 - fy)), (1, 0, fx * (1 - fy)), (0, 1, (1 - fx) * fy), (1, 1, fx * fy)):
            xi, yi = x0 + dx, y0 + dy
            ok = (xi >= 0) & (xi <= wl - 1) & (yi >= 0) & (yi <= hl - 1)
            idx = (yi.clamp(0, hl - 1) * wl + xi.clamp(0, wl - 1)).long().reshape(P, 81)
            v = torch.where(ok, torch.gather(flat, 1, idx).view(P, 9, 9), 0.0)
            o = o + wgt * v
            m = m + (wgt * v).abs()
        outs.append(o.reshape(P, 81))
        mags.append(m.reshape(P, 81))
    return torch.cat(outs, 1), torch.cat(mags, 1)


def planes64(levels, h, w, pairs=None):
    """the device pyramid (row-padded planes) as float64 [P, hl, wl], optionally only the pixels of `pairs`"""
    out, hl, wl = [], h, w
    for lv in levels:
        v = lv if pairs is None else torch.cat([lv[p * h * w:(p + 1) * h * w] for p in pairs])
        out.append(v[:, :, :wl].double())
        hl, wl = hl // 2, wl // 2
    return out


def lookup_coords(B, h, w, seed):
    """per pixel, by index mod 6: uniform +-6 px around the grid, exact integers, half-integers at level (i // 6) % 4,
    the borders (x = w-1, y = h-1, -0.5), centres 500 px outside (all-zero windows), uniform +-20 px"""
    gen = _gen(seed)
    ys, xs = torch.meshgrid(torch.arange(h, device=DEV), torch.arange(w, device=DEV), indexing="ij")
    base = torch.stack([xs, ys], -1).double()[None].expand(B, h, w, 2).reshape(-1, 2)
    n = base.shape[0]
    i = torch.arange(n, device=DEV)
    kind, sub = (i % 6)[:, None], (i // 6)
    uni = lambda r: (torch.rand(n, 2, generator=gen, device=DEV, dtype=torch.float64) * 2 - 1) * r
    ints = base + torch.randint(-6, 7, (n, 2), generator=gen, device=DEV)
    lvl = (2.0 ** (sub % 4)).double()[:, None]
    halves = ((base / lvl).floor() + torch.randint(-3, 4, (n, 2), generator=gen, device=DEV) + 0.5) * lvl
    bx = torch.stack([torch.tensor([w - 1.0, -0.5, w - 1.0, -0.5], device=DEV)[sub % 4],
                      torch.tensor([h - 1.0, -0.5, -0.5, h - 1.0], device=DEV)[(sub // 4) % 4]], 1).double()
    border = torch.where(torch.rand(n, 2, generator=gen, device=DEV) < 0.75, bx, base + uni(3))
    far = base + torch.where((sub % 2 == 0)[:, None], 500.0, -500.0)
    c = torch.where(kind == 0, base + uni(6), base + uni(20))
    for k, v in ((1, ints), (2, halves), (3, border), (4, far)):
        c = torch.where(kind == k, v, c)
    return c.float().view(B, h, w, 2), (kind == 4).view(B, h, w)


def _pyramid(B, h, w, seed, frames=None):
    """the 4-level device pyramid of B pairs of random 256-channel feature maps (consecutive frames, both directions)"""
    from propainter_b200 import ops
    gen = _gen(seed)
    frames = frames or B + 1
    fmap = _randn(gen, frames, h * w, 256)
    a = torch.arange(B, device=DEV) % (frames - 1)
    idx1 = torch.where(torch.arange(B, device=DEV) % 2 == 0, a, a + 1).int()
    idx2 = torch.where(torch.arange(B, device=DEV) % 2 == 0, a + 1, a).int()
    levels = ops.corr_alloc(B, h, w, DEV)
    ops.corr_build(fmap, idx1, idx2, levels, h, w)
    return levels


@pytest.mark.parametrize("shape", [(3, 16, 22), (4, 17, 23)])
def test_corr_lookup_f16(shape):
    """both lookup kernels into fp16 rows of 324 / 328 / 336 halves: float64 taps on the device pyramid, NaN pads kept"""
    from propainter_b200 import ops
    B, h, w = shape
    levels = _pyramid(B, h, w, seed=B)
    coords, far = lookup_coords(B, h, w, seed=10 + B)
    refs = {tma: lookup64(planes64(levels, h, w), coords, grid_sample32=not tma) for tma in (True, False)}
    ref = refs[True][0]
    # the restatement is the oracle's lookup (grid_sample, align_corners=True, zero padding) in float64
    pyr = [p[:, None].float().cpu() for p in planes64(levels, h, w)]
    oracle = ops_ref.corr_lookup(pyr, coords.permute(0, 3, 1, 2).cpu()).permute(0, 2, 3, 1).reshape(-1, 324)
    assert torch.allclose(ref.float().cpu(), oracle, atol=1e-4, rtol=1e-4)
    tally = Tally()
    for tma in (True, False):
        ref, s = refs[tma]
        out32 = ops.corr_lookup(levels, coords, tma=tma)
        for ld in (324, 328, 336):
            o = Slot((B, h, w), ld, F16)
            ops.corr_lookup(levels, coords, o.t, tma=tma)
            got = o.t[..., :324]
            assert same_bits(got, out32.half()), (tma, ld)
            check_f16(got.reshape(-1, 324), ref, s, f"lookup {shape} tma={tma} ld={ld}", tally)
            assert o.intact(0, 324) and bool(o.t[..., 324:].isnan().all()), (tma, ld)
            assert bool((got[far] == 0).all())
    tally.check(f"lookup {shape}")


def test_corr_lookup_f16_production():
    """the C2 batch: 158 pairs at 30 x 54 (2.3 GB of pyramid), both kernels on every pair; float64 taps of pairs 0, 79
    and 157 (the highest pixel indices included)"""
    from propainter_b200 import ops
    B, h, w = 158, 30, 54
    levels = _pyramid(B, h, w, seed=7, frames=80)
    coords, far = lookup_coords(B, h, w, seed=17)
    pairs = (0, 79, 157)
    tally = Tally()
    o = Slot((B, h, w), 328, F16)
    for tma in (True, False):
        ref, s = lookup64(planes64(levels, h, w, pairs), coords[list(pairs)], grid_sample32=not tma)
        bits(o.flat).fill_(SENTINEL[F16])
        o.snap()
        ops.corr_lookup(levels, coords, o.t, tma=tma)
        got = o.t[..., :324]
        out32 = ops.corr_lookup(levels, coords, tma=tma)
        assert same_bits(got, out32.half()), tma
        del out32
        check_f16(got[list(pairs)].reshape(-1, 324), ref, s, f"lookup C2 tma={tma} pairs {pairs}", tally)
        assert o.intact(0, 324) and bool(o.t[..., 324:].isnan().all())
        assert bool((got[far] == 0).all())
    tally.check("lookup C2")
    del levels, o, got
    torch.cuda.empty_cache()


# ----------------------------------------------------------------------------------------------- float64 references
# Each returns (ref, s) with s such that twice the fp32 error bound of the kernel's expression is 2^-21 (|ref| + s):
# an fp32 sum of exact operands is off by at most 2^-24 per partial sum (e), expf / tanhf by 2 ulp, a sigmoid / tanh
# passes an argument error on scaled by its derivative, and a clamp whose input is negative beyond its own error bound
# returns exactly 0 (s = 0 there).
def _sum(*terms):
    """float64 left-to-right sum of the non-None terms (fp32 order of the kernel) and e = sum of |partial sums|"""
    terms = [t.double() for t in terms if t is not None]
    t, e = terms[0], torch.zeros_like(terms[0])
    for a in terms[1:]:
        t = t + a
        e = e + t.abs()
    return t, e


def _relu(y, s):
    return y.clamp_min(0), torch.where(y > -2.0 ** -20 * (y.abs() + s), s, torch.zeros_like(s))


def bias_act_ref(x, bias, pre, res, act, post_relu):
    """post(act(x + bias + pre) + res)"""
    t, e = _sum(x, bias, pre)
    if act == "none":
        y, s = t, e / 4
    elif act == "relu":
        y, s = _relu(t, e / 4)
    elif act == "leaky":
        y = torch.where(t > 0, t, t * SLOPE)
        s = e / 4 + (y.abs() if res is not None else 0)
    elif act == "sigmoid":
        y = torch.sigmoid(t)
        s = y * (1 - y) * e / 4 + (y if res is not None else 0)
    else:
        y = torch.tanh(t)
        s = (1 - y * y) * e / 4 + (y.abs() if res is not None else 0)
    if res is not None:
        y = y + res.double()
    if post_relu:
        y, s = _relu(y, s)
    return y, s


def gate_ref(zr, bias, pre, h):
    """z = sigmoid(zr_z + pre_z + b_z) and r h = h sigmoid(zr_r + pre_r + b_r): (z, s_z, rh, s_rh)"""
    t, e = _sum(zr, pre, None if bias is None else bias.expand_as(zr))
    g = torch.sigmoid(t)
    C = zr.shape[-1] // 2
    z, gr = g[..., :C], g[..., C:]
    rh = h.double() * gr
    return z, z * (1 - z) * e[..., :C] / 4, rh, rh.abs() * (1 - gr) * e[..., C:] / 4


def update_ref(q, bias, pre, z, h):
    """(1 - z) h + z tanh(q + pre + b)"""
    t, e = _sum(q, pre, None if bias is None else bias.expand_as(q))
    th, zz, hh = torch.tanh(t), z.double(), h.double()
    return (1 - zz) * hh + zz * th, hh.abs() / 2 + zz * (1 - th * th) * e / 4 + zz * th.abs() / 2


def pack_ref(mot, bias):
    """relu(mot + b) (mot alone without bias)"""
    if bias is None:
        return mot.double(), torch.zeros_like(mot, dtype=torch.float64)
    t, e = _sum(mot, bias.expand_as(mot))
    return _relu(t, e / 4)


# ----------------------------------------------------------------------------------------------- bias_act
def _bias_act_f16_entry(x, out, bias, act, slope, res, post_relu, pre):
    """pp_bias_act_f16 called directly (ops.bias_act sends fp32 x / out to pp_bias_act)"""
    from propainter_b200 import _lib, ops
    C = x.shape[-1]
    xp, ldx = ops._pm(x, x.dtype)
    op, ldo = ops._pm(out, out.dtype)
    rp, ldr = ops._pm(res) if res is not None else (None, C)
    pp, ldp = ops._pm(pre) if pre is not None else (None, C)
    _lib.check(_lib.lib().pp_bias_act_f16(xp, ldx, int(x.dtype == F16), ops._p(bias), pp, ldp, rp, ldr, op, ldo,
                                          int(out.dtype == F16), x.numel() // C, C, ops.ACT[act], float(slope),
                                          int(post_relu), ops._stream()), "pp_bias_act_f16")
    return out


def _run_bias_act(gen, npix, C, xdt, odt, act, use_bias, use_pre, use_res, post_relu, tally, label, inplace=False,
                  oslot=None):
    """one case: x / out (fp16 or fp32) as slices of sentinel buffers, pre / res fp32 slices; checks (a), (b), (d)"""
    from propainter_b200 import ops
    lead = (npix,)
    xs = Slot(lead, C, xdt, ld=C + 4)
    xs.set(_randn(gen, npix, C, scale=2.0).to(xdt))
    x0 = xs.t.clone()
    bias = _randn(gen, C, scale=0.5) if use_bias else None
    ps = Slot(lead, C, F32, ld=C + 4).set(_randn(gen, npix, C, scale=0.5)) if use_pre else None
    rs = Slot(lead, C, F32, ld=C + 4).set(_randn(gen, npix, C, scale=0.5)) if use_res else None
    pre, res = (None if sl is None else sl.t for sl in (ps, rs))
    os_ = xs if inplace else (oslot or Slot(lead, C, odt, ld=C + 8))
    os_.snap()
    if xdt == F32 and odt == F32:
        _bias_act_f16_entry(xs.t, os_.t, bias, act, SLOPE, res, post_relu, pre)
    else:
        ops.bias_act(xs.t, bias, act, SLOPE, res=res, post_relu=post_relu, out=None if inplace else os_.t, pre=pre)
    got = os_.t
    # (a) the fp32 instantiation on the upcast input
    want = ops.bias_act(x0.float().contiguous(), bias, act, SLOPE, res=res, post_relu=post_relu,
                        out=torch.empty(npix, C, device=DEV), pre=pre)
    assert same_bits(got, want.to(odt)), label
    # (b)
    ref, s = bias_act_ref(x0, bias, pre, res, act, post_relu)
    if odt == F16:
        check_f16(got, ref, s, label, tally)
    else:
        check_f32(got, ref, s, label)
    # (d)
    assert os_.intact(), label
    assert all(sl.unchanged() for sl in (ps, rs, None if inplace else xs) if sl is not None), label


@pytest.mark.parametrize("xdt,odt", [(F16, F16), (F16, F32), (F32, F16), (F32, F32)], ids=["x16-out16", "x16-out32",
                                                                                          "x32-out16", "x32-out32"])
def test_bias_act_f16_entry(xdt, odt):
    """every activation with and without bias / pre / res / post_relu, C in {4, 64, 128, 192, 256}, npix 1 and ragged"""
    gen = _gen(100)
    tally = Tally()
    Cs = (4, 64, 128, 192, 256)
    k = 0
    for act in ("none", "relu", "leaky", "sigmoid", "tanh"):
        for flags in range(16):
            ub, up, ur, pr = (bool(flags >> i & 1) for i in range(4))
            C = Cs[k % len(Cs)]
            k += 1
            _run_bias_act(gen, RAGGED, C, xdt, odt, act, ub, up, ur, pr, tally,
                          f"bias_act {xdt}->{odt} {act} C={C} bias={ub} pre={up} res={ur} post_relu={pr}")
        for C in Cs:
            _run_bias_act(gen, 1, C, xdt, odt, act, True, True, True, False, tally, f"bias_act {act} npix=1 C={C}")
    if xdt == F16 and odt == F16:
        for C in Cs:
            _run_bias_act(gen, RAGGED, C, F16, F16, "tanh", True, True, False, False, tally, f"in place C={C}", inplace=True)
    if odt == F16:
        tally.check(f"bias_act {xdt}->{odt}")


def test_bias_act_f16_refinement_slices():
    """the epilogues of _refine_half at the C2 size (npix = 255960): convc2 / convf2 into the two slices of the fp16 mot_in,
    convf1 fp32 -> fp16 (128 channels), flow_head.conv1 fp16 -> fp32 (256 channels); convc1 at the ragged size"""
    gen = _gen(200)
    tally = Tally()
    n = C2_NPIX
    for lo, C in ((0, 192), (192, 64)):
        o = Slot((n,), C, F16, ld=256, c0=lo)          # the rest of the 256-channel row must keep its sentinel
        _run_bias_act(gen, n, C, F16, F16, "relu", True, False, False, False, tally, f"mot_in[..., {lo}:{lo + C}]", oslot=o)
    _run_bias_act(gen, n, 128, F32, F16, "relu", True, False, False, False, tally, "convf1 fp32 -> fp16")
    _run_bias_act(gen, n, 256, F16, F32, "relu", True, False, False, False, tally, "flow_head.conv1 fp16 -> fp32")
    _run_bias_act(gen, RAGGED, 256, F16, F16, "relu", True, False, False, False, tally, "convc1 fp16 -> fp16")
    tally.check("bias_act refinement slices")
    torch.cuda.empty_cache()


# ----------------------------------------------------------------------------------------------- GRU gate / update
def test_gru_gate_f16():
    """z = sigmoid(zr_z + b + pre) (fp32), r * h -> RX[..., :128] (fp16); pre-activations of +-30 / +-100, fp16-subnormal
    states; npix 1, ragged and the C2 size"""
    from propainter_b200 import ops
    gen = _gen(300)
    C = 128
    tally = Tally()
    for npix in (1, RAGGED, C2_NPIX):
        for use_bias, use_pre in ((True, False), (False, True)):
            lbl = f"gate npix={npix} bias={use_bias} pre={use_pre}"
            zr = Slot((npix,), 2 * C, F16).set(_spiked(gen, (npix, 2 * C), 3.0).half())
            bias = _randn(gen, 2 * C, scale=0.5) if use_bias else None
            pre = Slot((npix,), 2 * C, F32).set(_randn(gen, npix, 2 * C)).t if use_pre else None
            net = Slot((npix,), C, F32, ld=C + 4).set(_with_subnormals(gen, (npix, C), 1.0))
            z = Slot((npix,), C, F32)
            RX = Slot((npix,), C, F16, ld=256)
            ops.gru_gate(zr.t, bias, net.t, z.t, RX.t, pre=pre)
            # (a)
            z32, r32 = torch.empty(npix, C, device=DEV), torch.empty(npix, C, device=DEV)
            ops.gru_gate(zr.t.float(), bias, net.t, z32, r32, pre=pre)
            assert same_bits(z.t, z32) and same_bits(RX.t, r32.half()), lbl
            # (b)
            zref, sz, rh, sr = gate_ref(zr.t, bias, pre, net.t)
            check_f32(z.t, zref, sz, lbl + " z")
            check_f16(RX.t, rh, sr, lbl + " r*h", tally)
            t = _sum(zr.t, pre, None if bias is None else bias.expand_as(zr.t))[0][:, :C]
            assert bool((z.t[t >= 30] == 1).all()) and bool((z.t[t <= -100] == 0).all()), lbl
            # (d)
            assert z.intact() and RX.intact() and zr.unchanged() and net.unchanged(), lbl
    tally.check("gate r*h")


def test_gru_update_f16():
    """h = (1-z) h + z tanh(q + b + pre) in place on a 128-channel slice of a wider fp32 buffer; its fp16 image into
    HX[..., :128] (the motion slot untouched) and a dense net_copy, each also alone; npix 1, ragged and the C2 size"""
    from propainter_b200 import ops
    gen = _gen(400)
    C = 128
    tally = Tally()
    for npix in (1, RAGGED, C2_NPIX):
        for use_bias, use_pre, use_img, use_copy in ((True, False, True, True), (False, True, True, True),
                                                     (False, True, True, False), (True, True, False, True)):
            lbl = f"update npix={npix} bias={use_bias} pre={use_pre} h_img={use_img} net_copy={use_copy}"
            q = Slot((npix,), C, F16).set(_spiked(gen, (npix, C), 2.0).half())
            bias = _randn(gen, C, scale=0.5) if use_bias else None
            pre = Slot((npix,), C, F32).set(_randn(gen, npix, C)).t if use_pre else None
            zv = torch.sigmoid(_spiked(gen, (npix, C), 3.0))
            z = Slot((npix,), C, F32).set(zv)
            net = Slot((npix,), C, F32, ld=256).set(_with_subnormals(gen, (npix, C), 1.0))
            h0 = net.t.clone()
            HX = Slot((npix,), C, F16, ld=256)
            cp = Slot((npix,), C, F16)
            ops.gru_update(q.t, bias, z.t, net.t, net_copy=cp.t if use_copy else None, pre=pre,
                           h_img=HX.t if use_img else None)
            # (a)
            n32, c32 = h0.clone(), torch.empty(npix, C, device=DEV)
            ops.gru_update(q.t.float(), bias, z.t, n32, net_copy=c32, pre=pre)
            assert same_bits(net.t, n32), lbl
            for on, sl in ((use_img, HX), (use_copy, cp)):
                if on:
                    assert same_bits(sl.t, c32.half()) and same_bits(sl.t, net.t.half()), lbl
            # (b)
            ref, s = update_ref(q.t, bias, pre, z.t, h0)
            check_f32(net.t, ref, s, lbl + " net")
            if use_img:
                check_f16(HX.t, ref, s, lbl + " h_img", tally)
            # (d)
            assert net.intact(), lbl
            assert HX.intact() if use_img else HX.unchanged(), lbl
            assert cp.intact() if use_copy else cp.unchanged(), lbl
            assert q.unchanged() and z.unchanged(), lbl
    tally.check("update h_img")


# ----------------------------------------------------------------------------------------------- motion pack
def test_raft_pack_motion_f16():
    """[relu(mot + b)(126) | flow(2)] into the slots [128, 256) of two fp16 256-channel buffers; npix 1, ragged, C2"""
    from propainter_b200 import ops
    gen = _gen(500)
    tally = Tally()
    for npix in (1, RAGGED, C2_NPIX):
        for use_bias in (True, False):
            lbl = f"pack npix={npix} bias={use_bias}"
            mot = Slot((npix,), 128, F16, ld=132).set(_randn(gen, npix, 128, scale=2.0).half())
            bias = _randn(gen, 128, scale=0.5) if use_bias else None
            flow = _randn(gen, npix, 2, scale=8.0)
            d0, d1 = Slot((npix,), 128, F16, ld=256, c0=128), Slot((npix,), 128, F16, ld=256, c0=128)
            ops.raft_pack_motion(mot.t, flow, d0.t, d1.t, bias=bias)
            # (a)
            a0, a1 = torch.empty(npix, 128, device=DEV), torch.empty(npix, 128, device=DEV)
            ops.raft_pack_motion(mot.t.float(), flow, a0, a1, bias=bias)
            assert same_bits(d0.t, a0.half()) and same_bits(d1.t, d0.t), lbl
            # (b)
            ref, s = pack_ref(mot.t[:, :126], None if bias is None else bias[:126])
            check_f16(d0.t[:, :126], ref, s, lbl, tally)
            assert np.array_equal(d0.t[:, 126:].cpu().numpy().view(np.uint16),
                                  rn16(flow.double().cpu().numpy()).view(np.uint16)), lbl
            # (d)
            assert d0.intact() and d1.intact() and mot.unchanged(), lbl
    tally.check("pack")


# ----------------------------------------------------------------------------------------------- rounding contract
def crafted_f32():
    """fp32 values where rounding to fp16 is decided: zeros, the subnormal edge, ties to even both ways, the overflow
    edge, infinities, NaN and random values spread over 2^-30 ... 2^20"""
    t = 2.0 ** -24
    v = [0.0, -0.0, t, -t, np.nextafter(np.float32(t), np.float32(1)), np.nextafter(np.float32(t), np.float32(0)),
         t / 2, 3 * t / 2, 5 * t / 2, 7 * t / 2, 2 ** -14 - t / 2, 2 ** -14 + t / 2,
         np.nextafter(np.float32(t / 2), np.float32(1)), np.nextafter(np.float32(t / 2), np.float32(0))]
    for e in (-14, -3, 0, 5, 15):
        for k in (0, 1, 2, 3, 1022, 1023):
            v.append(2.0 ** e * (1 + k * 2 ** -10 + 2 ** -11))               # ties: even k down, odd k up
    v += [65504.0, 65519.996, 65520.0, 1e6, np.inf, -np.inf, np.nan]
    rs = np.random.default_rng(0)
    r = np.exp2(rs.uniform(-30, 20, 100_000)) * rs.choice([-1.0, 1.0], 100_000)
    v = np.concatenate([np.array(v, dtype=np.float64), -np.array(v, dtype=np.float64), r]).astype(np.float32)
    return v[: len(v) // 4 * 4]


def _same_as_numpy(got16, want32, what):
    g = got16.cpu().numpy().reshape(-1)
    with np.errstate(over="ignore"):                     # 65520 and beyond round to inf, as they should
        w = want32.astype(np.float16)
    nan = np.isnan(w)
    assert np.array_equal(np.isnan(g), nan), what
    bad = g[~nan].view(np.uint16) != w[~nan].view(np.uint16)
    assert not bad.any(), (what, want32[~nan][bad][:8], g[~nan][bad][:8], w[~nan][bad][:8])


def test_fp16_stores_round_like_numpy():
    """pure conversions (bias_act fp32 -> fp16 without bias / act, the motion pack's flow channels) equal np.float16 of
    every crafted fp32 value bit for bit (NaN as NaN)"""
    from propainter_b200 import ops
    v = crafted_f32()
    x = torch.from_numpy(v).to(DEV)
    out = Slot((len(v) // 4,), 4, F16)
    ops.bias_act(x.view(-1, 4), out=out.t)
    _same_as_numpy(out.t, v, "bias_act fp32 -> fp16")
    assert out.intact()
    n = len(v) // 2
    d0, d1 = Slot((n,), 128, F16, ld=256, c0=128), Slot((n,), 128, F16, ld=256, c0=128)
    ops.raft_pack_motion(torch.zeros(n, 128, device=DEV, dtype=F16), x.view(n, 2), d0.t, d1.t)
    _same_as_numpy(d0.t[:, 126:], v, "pack flow channels")
    assert same_bits(d0.t, d1.t) and d0.intact() and d1.intact()


# ----------------------------------------------------------------------------------------------- argument checks, empty calls
def test_misaligned_and_bad_stride_views_are_refused():
    """views 2 halves / 2 floats off their alignment, a row stride that is not a multiple of 4 and fp16 lookup rows
    narrower than 324 raise before any launch and leave every output untouched (tests/test_half_abi_host.py checks the
    same refusals through the C ABI without a device)"""
    from propainter_b200 import ops
    n, C = 37, 128

    def fresh(dtype, c, off=4, ld=None, c0=0):
        return Slot((n,), c, dtype, ld=ld, c0=c0, off=off).set(torch.ones(n, c, device=DEV).to(dtype))

    for f16 in (True, False):
        dt = F16 if f16 else F32
        # gate: zr, net, z, rnet; update: q, z, net, net_copy (and h_img); pack: mot, d0, d1 -- one at a time
        for bad in ("zr", "net", "z", "rnet", "ld"):
            zr, net, z = fresh(dt, 2 * C, off=2 if bad == "zr" else 4), fresh(F32, C, off=2 if bad == "net" else 4), \
                fresh(F32, C, off=2 if bad == "z" else 4)
            rx = fresh(dt, C, off=2 if bad == "rnet" else 4, ld=258 if bad == "ld" else 256)
            with pytest.raises(RuntimeError):
                ops.gru_gate(zr.t, None, net.t, z.t, rx.t)
            assert all(s.unchanged() for s in (zr, net, z, rx)), (f16, bad)
        for bad in ("q", "z", "net", "copy", "img", "ld"):
            if bad == "img" and not f16:
                continue
            q, z = fresh(dt, C, off=2 if bad == "q" else 4), fresh(F32, C, off=2 if bad == "z" else 4)
            net = fresh(F32, C, off=2 if bad == "net" else 4, ld=258 if bad == "ld" else 256)
            cp = fresh(dt, C, off=2 if bad == "copy" else 4)
            img = fresh(F16, C, off=2 if bad == "img" else 4, ld=256) if f16 else None
            with pytest.raises(RuntimeError):
                ops.gru_update(q.t, None, z.t, net.t, net_copy=cp.t, h_img=img.t if f16 else None)
            assert all(s.unchanged() for s in (q, z, net, cp) + ((img,) if f16 else ())), (f16, bad)
        for bad in ("mot", "d0", "d1", "ld"):
            mot = fresh(dt, C, off=2 if bad == "mot" else 4)
            ld = 258 if bad == "ld" else 256
            d0, d1 = fresh(dt, C, off=2 if bad == "d0" else 4, ld=ld), fresh(dt, C, off=2 if bad == "d1" else 4, ld=ld)
            with pytest.raises(RuntimeError):
                ops.raft_pack_motion(mot.t, torch.zeros(n, 2, device=DEV), d0.t, d1.t)
            assert all(s.unchanged() for s in (mot, d0, d1)), (f16, bad)
    for xdt, odt in ((F16, F16), (F16, F32), (F32, F16)):
        for bad in ("x", "out", "pre", "ld"):
            x = fresh(xdt, C, off=2 if bad == "x" else 4, ld=C + (2 if bad == "ld" else 4))
            out, pre = fresh(odt, C, off=2 if bad == "out" else 4), fresh(F32, C, off=2 if bad == "pre" else 4)
            with pytest.raises(RuntimeError):
                ops.bias_act(x.t, None, "relu", out=out.t, pre=pre.t)
            assert all(s.unchanged() for s in (x, out, pre)), (xdt, odt, bad)
    levels = _pyramid(2, 16, 16, seed=3)
    coords = torch.full((2, 16, 16, 2), 4.0, device=DEV)
    for tma in (True, False):
        o = Slot((2, 16, 16), 320, F16)
        with pytest.raises(RuntimeError):
            ops.corr_lookup(levels, coords, o.t, tma=tma)
        assert o.unchanged()


def test_empty_inputs_return_cleanly():
    """npix = 0 everywhere: no launch, and no launch error left behind for the next kernel"""
    from propainter_b200 import ops
    e = lambda c, dt=F32: torch.empty(0, c, device=DEV, dtype=dt)
    levels = _pyramid(2, 16, 16, seed=4)
    for dt in (F16, F32):
        ops.gru_gate(e(256, dt), None, e(128), e(128), e(128, dt))
        ops.gru_update(e(128, dt), None, e(128), e(128), net_copy=e(128, dt), h_img=e(128, dt) if dt == F16 else None)
        ops.raft_pack_motion(e(128, dt), e(2), e(128, dt), e(128, dt))
        ops.bias_act(e(64, dt), None, "relu", out=e(64, F16))
        for tma in (True, False):
            ops.corr_lookup(levels, torch.empty(0, 16, 16, 2, device=DEV), torch.empty(0, 16, 16, 328, device=DEV, dtype=dt)
                            if dt == F16 else None, tma=tma)
    assert torch.arange(5, device=DEV).sum().item() == 10
    torch.cuda.synchronize()


# ----------------------------------------------------------------------------------------------- the refinement loop
class Emulation:
    """_refine_half in float64 in the layout of oracle/raft_ref.update_block, rounding (rnd=True) to fp16 where the device
    path rounds: the lookup output, the fp16 convs' weights and raw outputs, each fp16 epilogue result, HX / RX
    ([h | motion(126) | flow(2)], the gates' `inp` share kept fp32), h_img and netc.  The state, the coordinates, the
    biases and `pre` stay unrounded.  rnd=False: the plain float64 reference of the same dataflow."""

    def __init__(self, sd, rnd):
        self.R = rn16_t if rnd else (lambda t: t)
        u = "update_block."
        self.sd = {k[len(u):]: v.to(DEV, torch.float64) for k, v in sd.items() if k.startswith(u)}
        P = self.sd
        self.w16 = {k: self.R(P[k + ".weight"]) for k in ("encoder.convc1", "encoder.convc2", "encoder.convf2",
                                                          "encoder.conv", "flow_head.conv1")}
        dyn = lambda w: torch.cat([w[:, :128], w[:, 256:]], 1)
        self.gru = {}
        for tag in "12":
            wzr = torch.cat([P[f"gru.convz{tag}.weight"], P[f"gru.convr{tag}.weight"]], 0)
            bzr = torch.cat([P[f"gru.convz{tag}.bias"], P[f"gru.convr{tag}.bias"]], 0)
            wq, bq = P[f"gru.convq{tag}.weight"], P[f"gru.convq{tag}.bias"]
            self.gru[tag] = (self.R(dyn(wzr)), self.R(dyn(wq)), (wzr[:, 128:256], bzr), (wq[:, 128:256], bq))

    def b(self, k):
        return self.sd[k + ".bias"]

    def conv16(self, x, k, pad):
        """an fp16 conv (x already holds fp16 values): rounded weights, raw output rounded"""
        return self.R(F.conv2d(x, self.w16[k], None, padding=pad))

    def ep16(self, x, k):
        return self.R(F.relu(x + self.b(k)[None, :, None, None]))

    def motion(self, corr, flow):
        """lookup output [B,324,h,w] (rounded) and flow -> [motion(126) | flow(2)] as packed into HX / RX"""
        R = self.R
        cor = self.ep16(self.conv16(corr, "encoder.convc1", 0), "encoder.convc1")
        cor = self.ep16(self.conv16(cor, "encoder.convc2", 1), "encoder.convc2")
        flo = R(F.relu(F.conv2d(flow, self.sd["encoder.convf1.weight"], self.b("encoder.convf1"), padding=3)))
        flo = self.ep16(self.conv16(flo, "encoder.convf2", 1), "encoder.convf2")
        mot = self.ep16(self.conv16(torch.cat([cor, flo], 1), "encoder.conv", 1), "encoder.conv")
        return torch.cat([mot, R(flow)], 1)

    def gate(self, zr, pre, h):
        """raw (rounded) gate conv output + pre -> z, rounded r*h"""
        t = zr + pre
        return torch.sigmoid(t[:, :128]), self.R(torch.sigmoid(t[:, 128:]) * h)

    def update(self, q, pre, z, h):
        return (1 - z) * h + z * torch.tanh(q + pre)

    def run(self, planes, c0, net, inp, iters):
        R = self.R
        pre = {}
        for tag, pad in (("1", (0, 2)), ("2", (2, 0))):
            (wz, bz), (wq, bq) = self.gru[tag][2], self.gru[tag][3]
            pre[tag] = (F.conv2d(inp, wz, bz, padding=pad), F.conv2d(inp, wq, bq, padding=pad))
        c1, h = c0.clone(), net.clone()
        B, _, hh, ww = c0.shape
        himg = R(h)
        for _ in range(iters):
            corr = R(lookup64(planes, c1.permute(0, 2, 3, 1))[0]).view(B, hh, ww, 324).permute(0, 3, 1, 2)
            flow = c1 - c0
            x = self.motion(corr, flow)
            for tag, pad in (("1", (0, 2)), ("2", (2, 0))):
                wzr, wq = self.gru[tag][:2]
                z, rh = self.gate(R(F.conv2d(torch.cat([himg, x], 1), wzr, padding=pad)), pre[tag][0], h)
                h = self.update(R(F.conv2d(torch.cat([rh, x], 1), wq, padding=pad)), pre[tag][1], z, h)
                himg = R(h)
            fh = F.relu(self.conv16(himg, "flow_head.conv1", 1) + self.b("flow_head.conv1")[None, :, None, None])
            c1 = c1 + F.conv2d(fh, self.sd["flow_head.conv2.weight"], self.b("flow_head.conv2"), padding=1)
        flow_lr = c1 - c0
        mask = 0.25 * F.conv2d(F.relu(F.conv2d(h, self.sd["mask.0.weight"], self.b("mask.0"), padding=1)),
                               self.sd["mask.2.weight"], self.b("mask.2"))
        return flow_lr, ops_ref.convex_upsample(flow_lr, mask)


def _nchw(t):
    return t.permute(0, 3, 1, 2).double()


def check_conv_stage(got16, x16, w16, pad, what):
    """a cuDNN fp16 conv output (fp32 accumulation, rounded once) against rn16 of the float64 conv of the same fp16 input
    and weights: within one fp16 ulp plus 2^-16 of sum |w x| (the fp32 accumulation) everywhere; prints and bounds the
    fraction that differs from rn16(conv64)"""
    ref = F.conv2d(x16, w16, padding=pad)
    mag = F.conv2d(x16.abs(), w16.abs(), padding=pad)
    g = _nchw(got16).cpu().numpy()
    r, m = ref.cpu().numpy(), mag.cpu().numpy()
    r16 = rn16(r).astype(np.float64)
    bad = ~(np.abs(g - r16) <= ulp16(r) + 2.0 ** -16 * m)
    assert not bad.any(), _first(what, "beyond one fp16 ulp of rn16(conv64)", bad.reshape(-1), g.reshape(-1), r.reshape(-1))
    frac = float((g != r16).mean())
    print(f"  {what}: {frac:.3%} differ from rn16(conv64)")
    assert frac <= 0.10, (what, frac)


def _record(mp, ops, log):
    """wrap the ops of the refinement loop; log (name, inputs cloned at call time, outputs cloned after)"""
    held = {}

    def wrap(name, fn, before, after):
        def w(*a, **kw):
            b = before(a, kw)
            r = fn(*a, **kw)
            log.append((name, b, after(a, kw, r)))
            return r
        mp.setattr(ops, name, w)

    cl = lambda t: None if t is None else t.clone()
    kw_or = lambda a, kw, i, k: kw[k] if k in kw else (a[i] if len(a) > i else None)

    def pack_before(a, kw):
        held["HX"], held["RX"] = a[2]._base, a[3]._base
        return {"mot": cl(a[0]), "flow": cl(a[1]), "bias": kw.get("bias")}
    wrap("corr_build", ops.corr_build, lambda a, kw: {}, lambda a, kw, r: {"levels": a[3]})
    wrap("corr_lookup", ops.corr_lookup, lambda a, kw: {"coords": cl(a[1])}, lambda a, kw, r: {"out": cl(r)})
    wrap("bias_act", ops.bias_act, lambda a, kw: {"x": cl(a[0]), "bias": kw_or(a, kw, 1, "bias"), "act": kw_or(a, kw, 2, "act")},
         lambda a, kw, r: {"out": cl(r)})
    wrap("raft_pack_motion", ops.raft_pack_motion, pack_before, lambda a, kw, r: {"d0": cl(a[2]), "d1": cl(a[3])})
    wrap("gru_gate", ops.gru_gate,
         lambda a, kw: {"zr": cl(a[0]), "net": cl(a[2]), "pre": cl(kw.get("pre")), "HX": cl(held["HX"])},
         lambda a, kw, r: {"z": cl(a[3]), "rnet": cl(a[4])})
    wrap("gru_update", ops.gru_update,
         lambda a, kw: {"q": cl(a[0]), "z": cl(a[2]), "net": cl(a[3]), "pre": cl(kw.get("pre")), "RX": cl(held["RX"])},
         lambda a, kw, r: {"net": cl(a[3]), "h_img": cl(kw.get("h_img")), "net_copy": cl(kw.get("net_copy"))})


def _stage_checks(E, log, h, w):
    """iteration 1, stage by stage: each stage's emulation fed with the recorded device inputs of that stage"""
    lk = [i for i, (n, _, _) in enumerate(log) if n == "corr_lookup"]
    it1 = log[lk[0]:lk[1] if len(lk) > 1 else len(log)]
    levels = next(o["levels"] for n, _, o in log if n == "corr_build")
    tally = Tally()
    _, a, o = it1[0]
    B = a["coords"].shape[0]
    ref, s = lookup64(planes64(levels, h, w), a["coords"])
    check_f16(o["out"][..., :324].reshape(-1, 324), ref, s, "stage lookup", tally)
    assert bool((o["out"][..., 324:] == 0).all()), "the lookup wrote into the zero pad channels of convc1's input"
    corr = _nchw(o["out"][..., :324])
    ba = [(a, o) for n, a, o in it1 if n == "bias_act"][:5]
    pk = next((a, o) for n, a, o in it1 if n == "raft_pack_motion")
    gates = [(a, o) for n, a, o in it1 if n == "gru_gate"]
    upds = [(a, o) for n, a, o in it1 if n == "gru_update"]
    assert len(ba) == 5 and len(gates) == 2 and len(upds) == 2

    def epilogue(i, what):
        a, o = ba[i]
        ref, s = bias_act_ref(a["x"], a["bias"], None, None, "relu", False)
        if o["out"].dtype == F16:
            check_f16(o["out"], ref, s, "stage " + what, tally)
        else:
            check_f32(o["out"], ref, s, "stage " + what)
        return _nchw(o["out"])

    check_conv_stage(ba[0][0]["x"], corr, E.w16["encoder.convc1"], 0, "stage conv convc1")
    cor = epilogue(0, "convc1 epilogue")
    check_conv_stage(ba[1][0]["x"], cor, E.w16["encoder.convc2"], 1, "stage conv convc2")
    cor = epilogue(1, "convc2 epilogue")
    flo = epilogue(2, "convf1 epilogue (fp32 -> fp16)")
    check_conv_stage(ba[3][0]["x"], flo, E.w16["encoder.convf2"], 1, "stage conv convf2")
    flo = epilogue(3, "convf2 epilogue")
    pa, po = pk
    check_conv_stage(pa["mot"][..., :126], torch.cat([cor, flo], 1), E.w16["encoder.conv"], 1, "stage conv motion")
    assert bool((pa["mot"][..., 126:] == 0).all())
    check_f16(po["d0"][..., :126], *pack_ref(pa["mot"][..., :126], pa["bias"][:126]), "stage motion pack", tally)
    assert np.array_equal(po["d0"][..., 126:].cpu().numpy().view(np.uint16),
                          rn16(pa["flow"].double().cpu().numpy()).view(np.uint16)) and same_bits(po["d0"], po["d1"])
    for k, ((ga, go), (ua, uo)) in enumerate(zip(gates, upds)):
        tag, pad = ("1", (0, 2)) if k == 0 else ("2", (2, 0))
        wzr, wq = E.gru[tag][:2]
        check_conv_stage(ga["zr"], _nchw(ga["HX"]), wzr, pad, f"stage conv gate z|r {tag}")
        zref, sz, rh, sr = gate_ref(ga["zr"], None, ga["pre"], ga["net"])
        check_f32(go["z"], zref, sz, f"stage gate z {tag}")
        check_f16(go["rnet"], rh, sr, f"stage gate r*h {tag}", tally)
        check_conv_stage(ua["q"], _nchw(ua["RX"]), wq, pad, f"stage conv candidate {tag}")
        ref, s = update_ref(ua["q"], None, ua["pre"], ua["z"], ua["net"])
        check_f32(uo["net"], ref, s, f"stage update net {tag}")
        check_f16(uo["h_img"], ref, s, f"stage update h_img {tag}", tally)
        assert same_bits(uo["h_img"], uo["net"].half())
    netc = upds[1][1]["net_copy"]
    assert same_bits(netc, upds[1][1]["h_img"])
    check_conv_stage(ba[4][0]["x"], _nchw(netc), E.w16["flow_head.conv1"], 1, "stage conv flow_head.conv1")
    epilogue(4, "flow_head.conv1 epilogue (fp16 -> fp32)")
    print(f"  stage fp16 outputs: {tally.n}, near-midpoint {tally.near / tally.n:.4%}")
    assert tally.near / tally.n < 0.01


def _clip(name):
    from propainter_b200 import synth
    if name == "4x128x144":
        u8, _, _ = synth.make_clip(4, 128, 144, seed=3)
    else:
        u8, _, _ = synth.make_clip(80, 240, 432, mask="ellipse", seed=0)
        u8 = u8[:3]
    return pipeline_ref.to_float_frames(u8)[0].to(DEV)


@pytest.mark.parametrize("clip", ["4x128x144", "3x240x432"])
def test_refine_half_matches_rounding_emulation(clip):
    """_refine_half (cuDNN TF32 off, so its fp32 convs are exact fp32 and fp16 rounding is the only approximation) against
    the float64 emulation with and without the fp16 roundings, both on the device's fp32 correlation pyramid.  e_ref, the
    error against the unrounded dataflow, stays in the fp16 class (<= 5e-3 of the flow scale); e_emu, against the rounding
    emulation, must be at most half of it.  A wiring error (a slot, a pad, the h_img carry, a tensor left fp32 or rounded
    twice) gives a ratio well above 1.

    The ratio cannot approach 0: cuDNN accumulates in fp32 in its own order, so 0.03-1 % of the fp16 conv outputs land one
    ulp from rn16(conv64) (the stage checks print these fractions and pass everywhere else bit for bit).  Such 1-ulp
    differences add in quadrature against the ~0.29-ulp rms rounding error of every element, sqrt(12 p) for a fraction
    p, and grow through the later layers.  Measured on an H100 80GB HBM3 (700 W power limit): 0.29-0.31 on 4x128x144 and
    0.32-0.40 on the C2 frames, for 1 and 3 iterations."""
    from propainter_b200 import ops
    from propainter_b200.model.modules.flow_comp_raft import RAFT_bi
    net = RAFT_bi(None, DEV, seed=1)
    raft = net.fix_raft
    frames = _clip(clip)
    l = frames.shape[0]
    with torch.no_grad():
        fmap, hnet, inp, hw = raft.encode_frames(frames)
    h, w = hw
    a = torch.arange(l - 1, device=DEV, dtype=torch.int32)
    idx1, idx2 = torch.cat([a, a + 1]), torch.cat([a + 1, a])
    sel = idx1.long()
    sd = {k: v.detach().cpu() for k, v in raft.state_dict().items()}
    emu = {rnd: Emulation(sd, rnd) for rnd in (True, False)}
    ys, xs = torch.meshgrid(torch.arange(h, device=DEV), torch.arange(w, device=DEV), indexing="ij")
    c0 = torch.stack([xs, ys], 0).double()[None].repeat(len(sel), 1, 1, 1)
    net64, inp64 = hnet[sel].double(), inp[sel].double()
    for iters in (1, 3):
        log = []
        mp = pytest.MonkeyPatch()
        try:
            _record(mp, ops, log)
            with torch.no_grad():
                flow_lr, up = raft._refine_half(fmap, idx1, idx2, hnet[sel], inp[sel], hw, iters)
            torch.cuda.synchronize()
        finally:
            mp.undo()
        print(f"{clip} iters={iters}")
        if iters == 1:
            _stage_checks(emu[True], log, h, w)
        # the emulation samples the device's own fp32 pyramid: the fp16 roundings are all that differs
        planes = planes64(next(o["levels"] for n, _, o in log if n == "corr_build"), h, w)
        (el, eu), (rl, ru) = (emu[rnd].run(planes, c0, net64, inp64, iters) for rnd in (True, False))
        rel = lambda got, want, ref: float((got.double() - want).abs().max() / ref.abs().max())
        rms = lambda got, want: float((got.double() - want).pow(2).mean().sqrt())
        e_emu = max(rel(flow_lr, el, rl), rel(up, eu, ru))
        e_ref = max(rel(flow_lr, rl, rl), rel(up, ru, ru))
        print(f"  e_emu {e_emu:.3e}  e_ref {e_ref:.3e}  ratio {e_emu / e_ref:.3f}  |flow|max {float(ru.abs().max()):.2f}  "
              f"(flow_lr {rel(flow_lr, el, rl) / rel(flow_lr, rl, rl):.3f}, up {rel(up, eu, ru) / rel(up, ru, ru):.3f}; "
              f"rms ratio flow_lr {rms(flow_lr, el) / rms(flow_lr, rl):.3f}, up {rms(up, eu) / rms(up, ru):.3f})")
        assert e_ref <= 5e-3, e_ref
        assert e_emu <= 0.5 * e_ref, (e_emu, e_ref)
