"""Oracle (test infrastructure): RAFT's AlternateCorrBlock (RAFT/corr.py:83-111) in plain torch fp32, and RAFT run with it.

The math is AlternateCorrBlock's: fmap2 is average-pooled into the pyramid (not the correlation volume), f2 is
bilinearly sampled at every window position of every level (zeros padding, align_corners=True, the sampling rule of
CorrBlock corr.py:29-50 + bilinear_sampler RAFT/utils/utils.py:57-71), dotted with f1 and divided by sqrt(D).

The reference's own alternate path cannot run: its ``alt_cuda_corr`` extension is not vendored, the import failure is
swallowed (corr.py:5-9) and corr.py:106 calls the module object.  Its output layout is therefore CorrBlock's by
definition: channel l*81 + a*9 + b samples level l at (x/2^l + a - 4, y/2^l + b - 4), the first window axis moving x
(the reference quirk noted in ops_ref.corr_lookup).  Pooling is linear, so this equals
``ops_ref.corr_lookup(ops_ref.corr_pyramid(f1, f2), coords)`` up to rounding.
"""
import math

import torch
import torch.nn.functional as F

from . import ops_ref, raft_ref


def fmap_pyramid(f2, levels=4):
    """f2 [B,D,h,w] -> [f2, avg_pool2d(f2, 2), ...] (the pooled fmap2 list of corr.py:89-93)."""
    pyr = [f2]
    for _ in range(levels - 1):
        pyr.append(F.avg_pool2d(pyr[-1], 2, stride=2))
    return pyr


def corr_lookup_alt_points(f1q, f2, cq, radius=4, chunk=2048):
    """Windows of P query points.  f1q [B,D,P] query features, f2 [B,D,h,w], cq [B,P,2] (x,y) level-0 centres ->
    [B,P,4*(2r+1)^2] in CorrBlock's channel order.  Points go through in chunks to bound the sampled-feature buffer."""
    B, D, P = f1q.shape
    r = radius
    d = torch.linspace(-r, r, 2 * r + 1, device=f1q.device)
    delta = torch.stack(torch.meshgrid(d, d, indexing="ij"), dim=-1).view(1, 1, (2 * r + 1) ** 2, 2)   # [a*9+b] = (d[a], d[b])
    pyr = fmap_pyramid(f2)
    out = torch.empty(B, P, len(pyr) * (2 * r + 1) ** 2, device=f1q.device, dtype=f1q.dtype)
    for p0 in range(0, P, chunk):
        f1c, cc = f1q[:, :, p0:p0 + chunk], cq[:, p0:p0 + chunk]
        outs = []
        for i, f in enumerate(pyr):
            H, W = f.shape[-2:]
            pos = cc[:, :, None, :] / 2 ** i + delta                                  # [B,p,81,2]
            g = torch.stack([2 * pos[..., 0] / (W - 1) - 1, 2 * pos[..., 1] / (H - 1) - 1], -1)
            s = F.grid_sample(f, g, align_corners=True)                               # [B,D,p,81]
            outs.append(torch.einsum("bdpk,bdp->bpk", s, f1c) / math.sqrt(D))
        out[:, p0:p0 + chunk] = torch.cat(outs, -1)
    return out


def corr_lookup_alt(f1, f2, coords, radius=4):
    """f1, f2 [B,D,h,w], coords [B,2,h,w] (x,y) -> [B,4*(2r+1)^2,h,w], the layout of ops_ref.corr_lookup."""
    B, D, h, w = f1.shape
    out = corr_lookup_alt_points(f1.reshape(B, D, h * w), f2, coords.reshape(B, 2, h * w).transpose(1, 2), radius)
    return out.transpose(1, 2).reshape(B, -1, h, w).contiguous()


def raft_forward_alt(sd, image1, image2, iters=20, return_lowres=False):
    """raft_ref.raft_forward with the lookup of AlternateCorrBlock (args.alternate_corr, raft.py:106-109)."""
    image1, image2 = image1.contiguous(), image2.contiguous()
    n = image1.shape[0]
    fm = raft_ref.encoder(sd, "fnet", torch.cat([image1, image2], 0), "instance").float()
    f1, f2 = fm[:n], fm[n:]
    cn = raft_ref.encoder(sd, "cnet", image1, "batch")
    net, inp = torch.tanh(cn[:, :128]), torch.relu(cn[:, 128:])
    N, _, H, W = image1.shape
    h, w = H // 8, W // 8
    ys, xs = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    c0 = torch.stack([xs, ys], 0).float()[None].repeat(N, 1, 1, 1).to(image1.device)
    c1 = c0.clone()
    up = None
    for _ in range(iters):
        corr = corr_lookup_alt(f1, f2, c1)
        net, up_mask, d = raft_ref.update_block(sd, net, inp, corr, c1 - c0)
        c1 = c1 + d
        up = ops_ref.convex_upsample(c1 - c0, up_mask)
    if return_lowres:
        return c1 - c0, up
    return up


def raft_bi_alt(sd, frames, iters=20):
    """raft_ref.raft_bi with the alternate lookup.  frames [b,l,3,h,w] -> (fwd, bwd) each [b,l-1,2,h,w]."""
    b, l, c, h, w = frames.shape
    a = frames[:, :-1].reshape(-1, c, h, w)
    bb = frames[:, 1:].reshape(-1, c, h, w)
    fw = raft_forward_alt(sd, a, bb, iters)
    bw = raft_forward_alt(sd, bb, a, iters)
    return fw.view(b, l - 1, 2, h, w), bw.view(b, l - 1, 2, h, w)
