"""RAFT optical flow (basic and small models) on the H100 hot path.

Drop-in for the reference's ``RAFT`` (RAFT/raft.py:24-146): same constructor argument, same
``forward(image1, image2, iters, flow_init, test_mode)`` result in test mode, same state_dict.
What differs is the execution plan:
  * features live pixel-major (channels-last); convs are cuDNN through torch
  * the all-pairs volume + pyramid (corr.py:13-27) is built by ``ops.corr_build`` (fp32-accurate
    3xTF32 tensor-core GEMM) into row-padded planes; the 4-level 9x9 lookup (corr.py:29-50) is one
    kernel writing the 324-channel pixel-major tensor the motion encoder consumes
  * where that volume cannot fit the device, or with the reference's ``args.alternate_corr``, the on-the-fly plan
    (AlternateCorrBlock, corr.py:83-111) pools the features instead and forms the window dot products at lookup time,
    writing the same 324-channel tensor (``corr_plan`` below)
  * z and r gates of the SepConvGRU share one conv (concatenated weights); eval BatchNorm is folded
    into the cnet convs; the mask head + convex upsampling run only on the last iteration (the
    reference computes them 20x and keeps one, raft.py:135-146)
  * ``flows_bidirectional`` encodes every frame once for both directions (the reference encodes each
    frame up to 4x, flow_comp_raft.py:48-49); per-sample InstanceNorm makes this exactly equivalent
  * ``args.small`` builds RAFT-small (raft.py:29-33,48-51): SmallEncoders, radius-3 lookups (196 channels) on either
    plan, the 3x3 ConvGRU with z and r sharing one conv, no mask head -- the flow is upsampled once, after the last
    iteration, by ``ops.upflow8`` (the reference upsamples every iteration and keeps the last in test mode,
    raft.py:136-146).  Captured graphs are cached per instance (ParamNet.graphs), so a basic and a small net never
    share one.
"""
import torch
import torch.nn.functional as F

from .. import config, ops
from .._params import ParamNet
from ..nn_util import as_nchw, as_pm, cl, conv, pad_in_channels
from ..schemas import raft_schema, raft_small_schema


ALL_PAIRS, ON_THE_FLY = "all_pairs", "on_the_fly"
# Bytes per input-frame pixel that one all-pairs RAFT call needs besides its correlation pyramid: encoder activations,
# context / GRU buffers, the 324-channel lookup output, the upsampled flows.  Measured by profiles/raft_mem.py on an
# H100 80GB HBM3 (700 W power limit): a 2-frame call (2 pairs, 20 iterations) peaked 2,676,002,816 bytes above its
# inputs at 1280x720, of which 2,200,320,000 are the two pyramids -> 258.1 B per pixel of the 2 frames (257.3 at
# 1920x1080).  Rounded up.  Measured on the basic model; RAFT-small is planned with the same constants: its pyramid has
# the same size (it depends on the feature grid only) and every other buffer is narrower (128-channel fmap, 196-channel
# lookup, 96-channel state), so they are upper bounds for it.
RAFT_WS_BYTES_PER_PX = 260
# Bytes per input-frame pixel that each pair of an on-the-fly call adds (the same buffers, no pyramid; the pooled
# feature levels are ~1/3 of fmap): same tool and card, the peak of a 4-frame call (6 pairs) minus that of a
# 2-frame call (2 pairs) over 4 pairs -> 243.6 B per pixel at 1280x720 and 1920x1080.  Rounded up.
OTF_BYTES_PER_PAIR_PX = 244


def pyramid_bytes(h, w):
    """Bytes of the 4-level all-pairs correlation pyramid of one pair on an h x w feature grid (ops.corr_alloc)."""
    n, hl, wl, total = h * w, h, w, 0
    for _ in range(4):
        total += n * hl * ops.corr_ld(wl) * 4
        hl, wl = hl // 2, wl // 2
    return total


def corr_plan(H, W, alternate=False, total_bytes=None):
    """The correlation plan of every RAFT call on H x W frames.  ON_THE_FLY (AlternateCorrBlock: no volume, the window
    dot products formed at lookup time) when the caller asks for it -- the reference's `args.alternate_corr` -- or when
    the smallest all-pairs call (2 frames: one pair per direction) with its working set exceeds the device's memory
    `total_bytes` (None: no limit).  ALL_PAIRS otherwise: it is the faster plan wherever it fits, and every size that
    runs all-pairs keeps its numerics."""
    if alternate:
        return ON_THE_FLY
    if total_bytes is not None and 2 * pyramid_bytes(H // 8, W // 8) + RAFT_WS_BYTES_PER_PX * 2 * H * W > total_bytes:
        return ON_THE_FLY
    return ALL_PAIRS


def device_bytes(device):
    """Total memory of a CUDA device, None elsewhere."""
    device = torch.device(device)
    return torch.cuda.get_device_properties(device).total_memory if device.type == "cuda" else None


class RAFT(ParamNet):
    hidden_dim = 128
    context_dim = 128

    def __init__(self, args=None, seed=None):
        small = bool(getattr(args, "small", False))
        super().__init__(raft_small_schema() if small else raft_schema(), seed=seed)
        self.small = small
        if small:                                                  # raft.py:29-33
            self.hidden_dim, self.context_dim = 96, 64
            args.corr_levels, args.corr_radius = 4, 3
        self.args = args

    # ------------------------------------------------------------------ weights
    def _wb(self, key, bn=None):
        """(weight, bias) of a conv, channels_last, with eval-BatchNorm `bn` folded in if given."""
        def build():
            w, b = self.P[key + ".weight"], self.P[key + ".bias"]
            if bn is not None and (bn + ".running_var") in self.P:
                s = self.P[bn + ".weight"] / torch.sqrt(self.P[bn + ".running_var"] + 1e-5)
                w = w * s.view(-1, 1, 1, 1)
                b = (b - self.P[bn + ".running_mean"]) * s + self.P[bn + ".bias"]
            return cl(w), b.contiguous()
        return self.packed("wb:" + key, build)

    def _motion_out(self):
        """update_block.encoder.conv with its 126 outputs padded to 128 (two zero filters): keeps the output
        rows 16-byte aligned; the pad slots are overwritten by the flow channels in raft_pack_motion."""
        def build():
            w, b = self.P["update_block.encoder.conv.weight"], self.P["update_block.encoder.conv.bias"]
            w = torch.cat([w, w.new_zeros(2, *w.shape[1:])], 0)
            return cl(w), torch.cat([b, b.new_zeros(2)]).contiguous()
        return self.packed("motion_out", build)

    def _gru(self, tag):
        """SepConvGRU weights of one pass (update.py:45-60), input channels [h(128) | inp(128) | motion(128)] (:129-130).
        z and r share one conv.  The `inp` (context) channels do not change over the refinement iterations, so their
        share of every gate conv is split off: (w_zr, w_q) act on the per-iteration [h | motion] buffers, (w_zr_inp,
        b_zr) / (w_q_inp, b_q) are convolved with `inp` once per clip and enter through the gate kernels' `pre` term."""
        def build():
            u = "update_block.gru."
            wzr = torch.cat([self.P[u + f"convz{tag}.weight"], self.P[u + f"convr{tag}.weight"]], 0)
            bzr = torch.cat([self.P[u + f"convz{tag}.bias"], self.P[u + f"convr{tag}.bias"]], 0)
            wq, bq = self.P[u + f"convq{tag}.weight"], self.P[u + f"convq{tag}.bias"]
            dyn = lambda w: cl(torch.cat([w[:, :128], w[:, 256:]], 1))
            ctx = lambda w: cl(w[:, 128:256])
            return dyn(wzr), dyn(wq), (ctx(wzr), bzr.contiguous()), (ctx(wq), bq.contiguous())
        return self.packed("gru" + tag, build)

    def _half(self, key, fn):
        """fp16 copy of packed weights `fn()` (biases, 1-D, stay fp32) for the half-operand refinement loop"""
        return self.packed("f16:" + key, lambda: tuple(t.half() if t.dim() == 4 else t for t in fn()))

    # ------------------------------------------------------------------ encoders (extractor.py:168-192)
    def _encode(self, p, x):
        """BasicEncoder.forward extractor.py:168-192.  fnet: conv -> InstanceNorm -> ReLU with the norm, the ReLU and the
        block's `relu(x + y)` as one pp_instance_norm call on the raw conv output (the conv bias cancels under the
        per-channel mean subtraction, so it is not even added).  cnet: eval BatchNorm folded into the conv; bias, ReLU
        and the residual add + ReLU are one pp_bias_act pass.
        cnet under config.half_convs() (CUDA tensors) runs on fp16 operands: frames rounded to fp16 and padded to 8 channels
        (zero weight columns), fp16 weights, cuDNN convs with fp32 accumulation writing fp16, pp_bias_act epilogues on fp16
        maps with an fp16 residual (fp32 arithmetic, each map rounded once); conv2 is widened on store, so the result is
        fp32 [n,256,h,w] channels_last either way and `net` / `inp` stay fp32.  fnet stays on TF32: every InstanceNorm it
        runs is held to the fp32 kernel's float64 bound, and on fp16 maps its outputs land up to ~1.4e3 times outside it."""
        inst = p == "fnet"
        half = not inst and x.is_cuda and config.half_convs()

        def wb(key, bn=None, cin_pad=None):
            if not half:
                return self._wb(key, bn)

            def build():
                w, b = self._wb(key, bn)
                return cl(pad_in_channels(w, cin_pad) if cin_pad else w).half(), b
            return self.packed(f"f16:{key}:{cin_pad}", build)

        def cn(key, bn, t, stride=1, pad=1, relu=True, res=None, cin_pad=None):
            if inst:
                w, _ = self._wb(key)
                y = as_pm(F.conv2d(t, w, None, stride=stride, padding=pad))
                return as_nchw(ops.instance_norm(y, relu=relu, res=None if res is None else as_pm(res),
                                                 post_relu=res is not None, out=y))
            return conv(t, wb(key, bn, cin_pad), stride, pad, act="relu" if relu else "none", res=res, post_relu=res is not None)

        if half:
            n, _, H, W = x.shape
            x16 = torch.zeros(n, H, W, 8, device=x.device, dtype=torch.float16)
            x16[..., :3].copy_(as_pm(x))
            x = as_nchw(x16)
        x = cn(p + ".conv1", p + ".norm1", x, 2, 3, cin_pad=8 if half else None)
        for li, stride in ((1, 1), (2, 2), (3, 2)):
            for bi in (0, 1):
                q = f"{p}.layer{li}.{bi}"
                s = stride if bi == 0 else 1
                y = cn(q + ".conv1", q + ".norm1", x, s, 1)
                if s != 1:
                    x = cn(q + ".downsample.0", q + ".norm3", x, s, 0, relu=False)
                x = cn(q + ".conv2", q + ".norm2", y, 1, 1, res=x)              # relu(x + relu(norm(conv2(y))))
        if half:
            m, _, h, w = x.shape
            return conv(x, wb(p + ".conv2"), out=as_nchw(torch.empty(m, h, w, 256, device=x.device)))
        return conv(x, self._wb(p + ".conv2"))

    def _encode_small(self, p, x):
        """SmallEncoder.forward extractor.py:244-267 with BottleneckBlocks (:60-115, 8/16/24 inner channels).  fnet: conv ->
        InstanceNorm -> ReLU as one pp_instance_norm call on the raw conv output (the bias cancels), the block's
        `relu(x + y)` fused into the last one.  cnet (norm_fn='none'): conv + bias + ReLU (+ residual + ReLU) through
        pp_bias_act."""
        inst = p == "fnet"

        def cn(key, t, stride=1, pad=0, relu=True, res=None):
            if inst:
                w, _ = self._wb(key)
                y = as_pm(F.conv2d(t, w, None, stride=stride, padding=pad))
                return as_nchw(ops.instance_norm(y, relu=relu, res=None if res is None else as_pm(res),
                                                 post_relu=res is not None, out=y))
            return conv(t, self._wb(key), stride, pad, act="relu" if relu else "none", res=res, post_relu=res is not None)

        x = cn(p + ".conv1", x, 2, 3)
        for li, stride in ((1, 1), (2, 2), (3, 2)):
            for bi in (0, 1):
                q = f"{p}.layer{li}.{bi}"
                s = stride if bi == 0 else 1
                y = cn(q + ".conv2", cn(q + ".conv1", x), s, 1)
                if s != 1:
                    x = cn(q + ".downsample.0", x, s, 0, relu=False)
                x = cn(q + ".conv3", y, res=x)                               # relu(x + relu(norm(conv3(y))))
        return conv(x, self._wb(p + ".conv2"))

    def encode_frames(self, frames):
        """frames [n,3,H,W] -> (fmap pixel-major [n, h*w, D], net [n,hdim,h,w], inp [n,cdim,h,w]); D = 256 / 128,
        (hdim, cdim) = (128, 128) / (96, 64) for the basic / small model."""
        x = frames.contiguous(memory_format=torch.channels_last)
        enc = self._encode_small if self.small else self._encode
        fmap = as_pm(enc("fnet", x).float())
        n, h, w, d = fmap.shape
        c = enc("cnet", x)
        hd = self.hidden_dim
        net, inp = torch.tanh(c[:, :hd]), torch.relu(c[:, hd:])
        return fmap.view(n, h * w, d), net, inp, (h, w)

    # ------------------------------------------------------------------ refinement loop (raft.py:122-146)
    def corr_plan(self, H, W, device):
        """corr_plan for this net's `args` (reference flag `alternate_corr`) on `device`."""
        return corr_plan(H, W, bool(getattr(self.args, "alternate_corr", False)), device_bytes(device))

    def _refine(self, fmap, idx1, idx2, net, inp, hw, iters, plan, flow_init=None):
        if self.small:
            return self._refine_small(fmap, idx1, idx2, net, inp, hw, iters, plan, flow_init)
        if plan == ALL_PAIRS and fmap.is_cuda and config.half_convs():      # cuDNN convs only: elsewhere there is no TF32
            return self._refine_half(fmap, idx1, idx2, net, inp, hw, iters, flow_init)
        h, w = hw
        B = idx1.numel()
        dev = fmap.device
        if plan == ON_THE_FLY:
            pooled = ops.corr_fmap_pyramid(fmap, h, w)
            lookup = lambda c, out: ops.corr_lookup_otf(fmap, pooled, idx1, idx2, c, out)
        else:
            levels = ops.corr_alloc(B, h, w, dev)
            ops.corr_build(fmap, idx1, idx2, levels, h, w)
            lookup = lambda c, out: ops.corr_lookup(levels, c, out)
        ys, xs = torch.meshgrid(torch.arange(h, device=dev), torch.arange(w, device=dev), indexing="ij")
        c0 = torch.stack([xs, ys], -1).float()[None].expand(B, h, w, 2).contiguous()     # coords_grid (utils.py:74-77)
        c1 = c0.clone()
        if flow_init is not None:
            c1 = c1 + as_pm(flow_init)
        u = "update_block."
        corr = torch.empty(B, h, w, 324, device=dev)
        # persistent GRU buffers (no torch.cat inside the loop):
        #   HX = [net | motion(126) flow(2)]  -> z/r gate convs;   RX = [r*net | motion flow] -> candidate conv
        # the context channels `inp` are iteration-invariant: their conv contributions (+ biases) are computed here, once
        HX = torch.empty(B, h, w, 256, device=dev)
        RX = torch.empty(B, h, w, 256, device=dev)
        HX[..., :128] = as_pm(net)
        pre = {}
        for tag, pad in (("1", (0, 2)), ("2", (2, 0))):
            _, _, zr_ctx, q_ctx = self._gru(tag)
            pre[tag] = (as_pm(conv(inp, zr_ctx, 1, pad)), as_pm(conv(inp, q_ctx, 1, pad)))
        netv, z = HX[..., :128], torch.empty(B, h, w, 128, device=dev)
        netc = torch.empty(B, h, w, 128, device=dev)            # dense copy of the state for the flow / mask heads
        mot_in = torch.empty(B, h, w, 256, device=dev)          # [cor(192) | flo(64)] without a torch.cat (update.py:95)
        mw, mb = self._motion_out()
        for _ in range(iters):
            lookup(c1, corr)
            flow_pm = c1 - c0
            flow = as_nchw(flow_pm)
            cor = conv(as_nchw(corr), self._wb(u + "encoder.convc1"), act="relu")
            conv(cor, self._wb(u + "encoder.convc2"), 1, 1, act="relu", out=as_nchw(mot_in[..., :192]))
            flo = conv(flow, self._wb(u + "encoder.convf1"), 1, 3, act="relu")
            conv(flo, self._wb(u + "encoder.convf2"), 1, 1, act="relu", out=as_nchw(mot_in[..., 192:]))
            mot = F.conv2d(as_nchw(mot_in), mw, None, padding=1)                   # 126 real + 2 pad channels, raw
            ops.raft_pack_motion(as_pm(mot), flow_pm, HX[..., 128:], RX[..., 128:], bias=mb)   # + bias + ReLU (update.py:96)
            for tag, pad in (("1", (0, 2)), ("2", (2, 0))):
                gw, qw, _, _ = self._gru(tag)
                ops.gru_gate(as_pm(F.conv2d(as_nchw(HX), gw, None, padding=pad)), None, netv, z, RX[..., :128], pre=pre[tag][0])
                ops.gru_update(as_pm(F.conv2d(as_nchw(RX), qw, None, padding=pad)), None, z, netv,
                               net_copy=netc if tag == "2" else None, pre=pre[tag][1])
            net = as_nchw(netc)
            d = conv(conv(net, self._wb(u + "flow_head.conv1"), 1, 1, act="relu"), self._wb(u + "flow_head.conv2"), 1, 1)
            c1 = c1 + as_pm(d)
        flow_lr = c1 - c0
        mask = conv(conv(net, self._wb(u + "mask.0"), 1, 1, act="relu"), self._wb(u + "mask.2"))
        up = ops.convex_upsample(as_pm(mask), flow_lr.contiguous(), 0.25)
        return as_nchw(flow_lr), up

    def _refine_half(self, fmap, idx1, idx2, net, inp, hw, iters, flow_init=None):
        """_refine on the all-pairs plan with half-precision operands (config.HALF_OPERANDS, DESIGN.md §4 "Precision"):
        the lookup output, the motion features, HX / RX and the inputs of convc1, convc2, convf2, the motion conv, the
        four SepConvGRU gate convs and flow_head.conv1 are fp16 (rounded to nearest by the producing kernel), the convs
        accumulate in fp32 and every epilogue computes in fp32.  The recurrent state (`netf`, HX / RX hold its fp16
        image), the coordinates, the context shares `pre`, convf1 (7x7 on the flow), flow_head.conv2 and the mask head
        stay fp32."""
        h, w = hw
        B = idx1.numel()
        dev = fmap.device
        f16 = torch.float16
        levels = ops.corr_alloc(B, h, w, dev)
        ops.corr_build(fmap, idx1, idx2, levels, h, w)
        ys, xs = torch.meshgrid(torch.arange(h, device=dev), torch.arange(w, device=dev), indexing="ij")
        c0 = torch.stack([xs, ys], -1).float()[None].expand(B, h, w, 2).contiguous()     # coords_grid (utils.py:74-77)
        c1 = c0.clone()
        if flow_init is not None:
            c1 = c1 + as_pm(flow_init)
        u = "update_block."
        corr = torch.zeros(B, h, w, 328, device=dev, dtype=f16)   # 324 taps + 4 zero channels: 16-byte pixel rows
        HX = torch.empty(B, h, w, 256, device=dev, dtype=f16)
        RX = torch.empty(B, h, w, 256, device=dev, dtype=f16)
        netf = torch.empty(B, h, w, 128, device=dev)
        netf.copy_(as_pm(net))
        HX[..., :128] = netf
        pre = {}
        for tag, pad in (("1", (0, 2)), ("2", (2, 0))):
            _, _, zr_ctx, q_ctx = self._gru(tag)
            pre[tag] = (as_pm(conv(inp, zr_ctx, 1, pad)), as_pm(conv(inp, q_ctx, 1, pad)))
        z = torch.empty(B, h, w, 128, device=dev)
        netc = torch.empty(B, h, w, 128, device=dev, dtype=f16)   # dense fp16 image of the state for flow_head.conv1
        mot_in = torch.empty(B, h, w, 256, device=dev, dtype=f16)
        mw, mb = self._half("motion_out", self._motion_out)
        c1w = self._half("convc1", lambda: (cl(pad_in_channels(self._wb(u + "encoder.convc1")[0], 328)),
                                            self._wb(u + "encoder.convc1")[1]))
        wb16 = lambda k: self._half(k, lambda: self._wb(u + k))

        def ep(x, wb, pad, out):
            """conv (no bias) + bias + ReLU into the pixel-major `out` (fp16 or fp32) through pp_bias_act_f16"""
            return as_nchw(ops.bias_act(as_pm(F.conv2d(x, wb[0], None, padding=pad)), wb[1], "relu", out=out))

        for _ in range(iters):
            ops.corr_lookup(levels, c1, corr)
            flow_pm = c1 - c0
            cor = ep(as_nchw(corr), c1w, 0, torch.empty(B, h, w, 256, device=dev, dtype=f16))
            ep(cor, wb16("encoder.convc2"), 1, mot_in[..., :192])
            flo = ep(as_nchw(flow_pm), self._wb(u + "encoder.convf1"), 3, torch.empty(B, h, w, 128, device=dev, dtype=f16))
            ep(flo, wb16("encoder.convf2"), 1, mot_in[..., 192:])
            mot = F.conv2d(as_nchw(mot_in), mw, None, padding=1)                   # 126 real + 2 pad channels, raw
            ops.raft_pack_motion(as_pm(mot), flow_pm, HX[..., 128:], RX[..., 128:], bias=mb)   # + bias + ReLU (update.py:96)
            for tag, pad in (("1", (0, 2)), ("2", (2, 0))):
                gw, qw = self._half("gru" + tag, lambda: self._gru(tag)[:2])
                ops.gru_gate(as_pm(F.conv2d(as_nchw(HX), gw, None, padding=pad)), None, netf, z, RX[..., :128], pre=pre[tag][0])
                ops.gru_update(as_pm(F.conv2d(as_nchw(RX), qw, None, padding=pad)), None, z, netf,
                               net_copy=netc if tag == "2" else None, pre=pre[tag][1], h_img=HX[..., :128])
            fh = ep(as_nchw(netc), wb16("flow_head.conv1"), 1, torch.empty(B, h, w, 256, device=dev))
            c1 = c1 + as_pm(conv(fh, self._wb(u + "flow_head.conv2"), 1, 1))
        flow_lr = c1 - c0
        net = as_nchw(netf)
        mask = conv(conv(net, self._wb(u + "mask.0"), 1, 1, act="relu"), self._wb(u + "mask.2"))
        up = ops.convex_upsample(as_pm(mask), flow_lr.contiguous(), 0.25)
        return as_nchw(flow_lr), up

    def _gru_small(self):
        """ConvGRU weights (update.py:16-31), input channels [h(96) | inp(64) | motion(80) | flow(2)] (:108-109); z and r
        share one conv.  As in _gru, the `inp` share of every gate is split off and convolved once per call; the per-
        iteration convs read [h | motion flow pad(2)] (180 channels, 16-byte rows), the pad weights are zero."""
        def build():
            u = "update_block.gru."
            wzr = torch.cat([self.P[u + "convz.weight"], self.P[u + "convr.weight"]], 0)
            bzr = torch.cat([self.P[u + "convz.bias"], self.P[u + "convr.bias"]], 0)
            wq, bq = self.P[u + "convq.weight"], self.P[u + "convq.bias"]
            dyn = lambda w: cl(torch.cat([w[:, :96], w[:, 160:], w.new_zeros(w.shape[0], 2, *w.shape[2:])], 1))
            ctx = lambda w: cl(w[:, 96:160])
            return dyn(wzr), dyn(wq), (ctx(wzr), bzr.contiguous()), (ctx(wq), bq.contiguous())
        return self.packed("gru_small", build)

    def _refine_small(self, fmap, idx1, idx2, net, inp, hw, iters, plan, flow_init=None):
        """SmallUpdateBlock refinement (raft.py:122-146, update.py:62-77,99-112) on radius-3 lookups; upflow8 once at the end."""
        h, w = hw
        B = idx1.numel()
        dev = fmap.device
        R = self.args.corr_radius
        if plan == ON_THE_FLY:
            pooled = ops.corr_fmap_pyramid(fmap, h, w)
            lookup = lambda c, out: ops.corr_lookup_otf_r(fmap, pooled, idx1, idx2, c, R, out)
        else:
            levels = ops.corr_alloc(B, h, w, dev)
            ops.corr_build(fmap, idx1, idx2, levels, h, w)
            lookup = lambda c, out: ops.corr_lookup_r(levels, c, R, out)
        ys, xs = torch.meshgrid(torch.arange(h, device=dev), torch.arange(w, device=dev), indexing="ij")
        c0 = torch.stack([xs, ys], -1).float()[None].expand(B, h, w, 2).contiguous()     # coords_grid (utils.py:74-77)
        c1 = c0.clone()
        if flow_init is not None:
            c1 = c1 + as_pm(flow_init)
        u = "update_block."
        corr = torch.empty(B, h, w, 4 * (2 * R + 1) ** 2, device=dev)
        # HX = [net(96) | motion(80) flow(2) pad(2)] -> z/r gate conv;  RX = [r*net | motion flow pad] -> candidate conv
        HX = torch.empty(B, h, w, 180, device=dev)
        RX = torch.empty(B, h, w, 180, device=dev)
        HX[..., :96] = as_pm(net)
        gw, qw, zr_ctx, q_ctx = self._gru_small()
        pre_zr, pre_q = as_pm(conv(inp, zr_ctx, 1, 1)), as_pm(conv(inp, q_ctx, 1, 1))
        netv, z = HX[..., :96], torch.empty(B, h, w, 96, device=dev)
        netc = torch.empty(B, h, w, 96, device=dev)             # dense copy of the state for the flow head
        mot_in = torch.empty(B, h, w, 128, device=dev)          # [cor(96) | flo(32)] without a torch.cat (update.py:74)
        mw, mb = cl(self.P[u + "encoder.conv.weight"]), self.P[u + "encoder.conv.bias"].contiguous()
        for _ in range(iters):
            lookup(c1, corr)
            flow_pm = c1 - c0
            flow = as_nchw(flow_pm)
            conv(as_nchw(corr), self._wb(u + "encoder.convc1"), act="relu", out=as_nchw(mot_in[..., :96]))
            flo = conv(flow, self._wb(u + "encoder.convf1"), 1, 3, act="relu")
            conv(flo, self._wb(u + "encoder.convf2"), 1, 1, act="relu", out=as_nchw(mot_in[..., 96:]))
            mot = F.conv2d(as_nchw(mot_in), mw, None, padding=1)                   # 80 channels, raw
            ops.raft_pack_motion_n(as_pm(mot), flow_pm, HX[..., 96:], RX[..., 96:], 80, bias=mb)   # + bias + ReLU (update.py:75)
            ops.gru_gate(as_pm(F.conv2d(as_nchw(HX), gw, None, padding=1)), None, netv, z, RX[..., :96], pre=pre_zr)
            ops.gru_update(as_pm(F.conv2d(as_nchw(RX), qw, None, padding=1)), None, z, netv, net_copy=netc, pre=pre_q)
            net = as_nchw(netc)
            d = conv(conv(net, self._wb(u + "flow_head.conv1"), 1, 1, act="relu"), self._wb(u + "flow_head.conv2"), 1, 1)
            c1 = c1 + as_pm(d)
        flow_lr = c1 - c0
        return as_nchw(flow_lr), ops.upflow8(flow_lr.contiguous())

    @torch.no_grad()
    def forward(self, image1, image2, iters=12, flow_init=None, test_mode=True):
        """raft.py:87-146.  image1/2 [N,3,H,W] in [-1,1] -> (flow_lowres [N,2,H/8,W/8], flow_up [N,2,H,W])."""
        if not test_mode:
            raise NotImplementedError("training-mode flow_predictions list is outside the inference hot path")
        n = image1.shape[0]
        plan = self.corr_plan(image1.shape[-2], image1.shape[-1], image1.device)
        fmap, net, inp, hw = self.encode_frames(torch.cat([image1, image2], 0))
        idx1 = torch.arange(n, device=image1.device, dtype=torch.int32)
        return self._refine(fmap, idx1, idx1 + n, net[:n], inp[:n], hw, iters, plan, flow_init)

    @torch.no_grad()
    def flows_bidirectional(self, frames, iters=20):
        """frames [l,3,H,W] -> (forward flows i->i+1, backward flows i+1->i), each [l-1,2,H,W].
        Encoders + 20 refinement iterations replay as one CUDA graph per clip shape."""
        plan = self.corr_plan(frames.shape[-2], frames.shape[-1], frames.device)
        return self.graphs(("raft_bi", iters, plan), lambda fr: self._flows_bidirectional(fr, iters, plan), frames.contiguous())

    def _flows_bidirectional(self, frames, iters, plan=ALL_PAIRS):
        l = frames.shape[0]
        fmap, net, inp, hw = self.encode_frames(frames)
        a = torch.arange(l - 1, device=frames.device, dtype=torch.int32)
        idx1, idx2 = torch.cat([a, a + 1]), torch.cat([a + 1, a])
        sel = idx1.long()
        _, up = self._refine(fmap, idx1, idx2, net[sel], inp[sel], hw, iters, plan)
        return up[:l - 1], up[l - 1:]
