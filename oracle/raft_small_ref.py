"""Oracle (test infrastructure): RAFT-small (RAFT(args.small=True)) flow in functional torch fp32.

Follows RAFT/raft.py:29-33,48-51,87-146, SmallEncoder RAFT/extractor.py:195-267 with BottleneckBlock :60-115,
SmallUpdateBlock RAFT/update.py:16-31 (ConvGRU), :62-77 (SmallMotionEncoder), :99-112, and upflow8
RAFT/utils/utils.py:80-82.  Correlation: CorrBlock (corr.py:13-60) at radius 3, or with ``alternate=True``
AlternateCorrBlock's rule (oracle/alt_corr_ref.py) at radius 3.  The reference's AlternateCorrBlock divides by a
hard-coded 16.0 (corr.py:111), which is 1/sqrt(D) only for the basic model's D = 256; its kernel is not vendored, so the
alternate plan here keeps CorrBlock's /sqrt(D) (D = 128) and both plans compute the same lookup.
``sd`` holds the reference's state_dict (keys without the DataParallel ``module.`` prefix).
"""
import torch
import torch.nn.functional as F

from . import alt_corr_ref, ops_ref

RADIUS = 3
HDIM, CDIM = 96, 64                               # raft.py:30-31


def _cv(sd, k, x, stride=1, pad=0):
    return F.conv2d(x, sd[k + ".weight"], sd[k + ".bias"], stride=stride, padding=pad)


def _norm(x, kind):
    """InstanceNorm2d (no affine, fnet) or nn.Sequential() (norm_fn='none', cnet)."""
    return F.instance_norm(x, eps=1e-5) if kind == "instance" else x


def _bottleneck(sd, p, x, kind, stride):
    """extractor.py:60-115 (BottleneckBlock.forward)."""
    y = F.relu(_norm(_cv(sd, p + ".conv1", x), kind))
    y = F.relu(_norm(_cv(sd, p + ".conv2", y, stride, 1), kind))
    y = F.relu(_norm(_cv(sd, p + ".conv3", y), kind))
    if stride != 1:
        x = _norm(_cv(sd, p + ".downsample.0", x, stride, 0), kind)
    return F.relu(x + y)


def encoder(sd, p, x, kind):
    """extractor.py:244-267 (SmallEncoder.forward, eval)."""
    x = F.relu(_norm(_cv(sd, p + ".conv1", x, 2, 3), kind))
    for li, stride in ((1, 1), (2, 2), (3, 2)):
        x = _bottleneck(sd, f"{p}.layer{li}.0", x, kind, stride)
        x = _bottleneck(sd, f"{p}.layer{li}.1", x, kind, 1)
    return _cv(sd, p + ".conv2", x)


def update_block(sd, net, inp, corr, flow):
    """update.py:99-112: SmallMotionEncoder (:62-77), ConvGRU (:16-31), FlowHead (:6-14); no mask head."""
    u = "update_block."
    cor = F.relu(_cv(sd, u + "encoder.convc1", corr))
    flo = F.relu(_cv(sd, u + "encoder.convf1", flow, 1, 3))
    flo = F.relu(_cv(sd, u + "encoder.convf2", flo, 1, 1))
    mot = F.relu(_cv(sd, u + "encoder.conv", torch.cat([cor, flo], 1), 1, 1))
    x = torch.cat([inp, mot, flow], 1)
    hx = torch.cat([net, x], 1)
    z = torch.sigmoid(_cv(sd, u + "gru.convz", hx, 1, 1))
    r = torch.sigmoid(_cv(sd, u + "gru.convr", hx, 1, 1))
    q = torch.tanh(_cv(sd, u + "gru.convq", torch.cat([r * net, x], 1), 1, 1))
    net = (1 - z) * net + z * q
    dflow = _cv(sd, u + "flow_head.conv2", F.relu(_cv(sd, u + "flow_head.conv1", net, 1, 1)), 1, 1)
    return net, dflow


def upflow8(flow):
    """RAFT/utils/utils.py:80-82."""
    return 8 * F.interpolate(flow, size=(8 * flow.shape[2], 8 * flow.shape[3]), mode="bilinear", align_corners=True)


def features(sd, image1, image2):
    """fnet of both images (fp32) and the split context (raft.py:100-116): (fmap1, fmap2, net, inp)."""
    n = image1.shape[0]
    fm = encoder(sd, "fnet", torch.cat([image1.contiguous(), image2.contiguous()], 0), "instance").float()
    cn = encoder(sd, "cnet", image1.contiguous(), "none")
    return fm[:n], fm[n:], torch.tanh(cn[:, :HDIM]), torch.relu(cn[:, HDIM:])


def raft_forward(sd, image1, image2, iters=20, flow_init=None, alternate=False, return_lowres=False):
    """raft.py:87-146 with test_mode=True: the upsampled flow of the last iteration (and the low-res flow)."""
    f1, f2, net, inp = features(sd, image1, image2)
    if alternate:
        lookup = lambda c: alt_corr_ref.corr_lookup_alt(f1, f2, c, radius=RADIUS)
    else:
        pyr = ops_ref.corr_pyramid(f1, f2)
        lookup = lambda c: ops_ref.corr_lookup(pyr, c, radius=RADIUS)
    N, _, H, W = image1.shape
    h, w = H // 8, W // 8
    ys, xs = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    c0 = torch.stack([xs, ys], 0).float()[None].repeat(N, 1, 1, 1).to(image1.device)
    c1 = c0.clone() if flow_init is None else c0 + flow_init
    for _ in range(iters):
        net, d = update_block(sd, net, inp, lookup(c1), c1 - c0)
        c1 = c1 + d
    up = upflow8(c1 - c0)                 # the reference upsamples every iteration and returns the last (raft.py:136-146)
    if return_lowres:
        return c1 - c0, up
    return up


def lookup_iter0(sd, image1, image2, alternate=False):
    """The 196-channel correlation lookup of iteration 0 (centres on the coordinate grid)."""
    f1, f2, _, _ = features(sd, image1, image2)
    N, _, h, w = f1.shape
    ys, xs = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    c0 = torch.stack([xs, ys], 0).float()[None].repeat(N, 1, 1, 1).to(image1.device)
    if alternate:
        return alt_corr_ref.corr_lookup_alt(f1, f2, c0, radius=RADIUS)
    return ops_ref.corr_lookup(ops_ref.corr_pyramid(f1, f2), c0, radius=RADIUS)


def raft_bi(sd, frames, iters=20, alternate=False):
    """flow_comp_raft.py:39-55 with the small model.  frames [b,l,3,h,w] -> (fwd, bwd) each [b,l-1,2,h,w]."""
    b, l, c, h, w = frames.shape
    a = frames[:, :-1].reshape(-1, c, h, w)
    bb = frames[:, 1:].reshape(-1, c, h, w)
    fw = raft_forward(sd, a, bb, iters, alternate=alternate)
    bw = raft_forward(sd, bb, a, iters, alternate=alternate)
    return fw.view(b, l - 1, 2, h, w), bw.view(b, l - 1, 2, h, w)
