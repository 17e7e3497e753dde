"""Recurrent flow completion network on the H100 hot path.

Drop-in for model/recurrent_flow_completion.py:203-347 of the reference (constructor, ``forward``,
``forward_bidirect_flow``, ``combine_flow``, state_dict incl. the training-only edge head).
Execution plan: every (1,k,k) Conv3d is a 2-D conv over the frame batch and every (3,1,1) dilated
temporal Conv3d one 1x1 conv over three time-shifted copies (both channels-last, cuDNN); the
second-order deformable alignment of the bidirectional scan (:9-44, :67-124) is
``ops.deform_align`` -- 5*tanh offset prep, sigmoid modulation, bilinear gather and the 2304-deep
GEMM in one kernel, reading the two previous states straight out of the scan buffer.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import autotune, config, ops
from .._params import ParamNet
from ..graphs import high_priority
from ..nn_util import as_nchw, as_pm, cl, conv, up2
from ..schemas import rfc_schema


def _lrelu(x, s=0.2):
    return F.leaky_relu_(x, s)


class RecurrentFlowCompleteNet(ParamNet):
    def __init__(self, model_path=None, seed=None):
        super().__init__(rfc_schema(), seed=seed)
        if model_path is not None:
            print("Pretrained flow completion model has loaded...")
            self.load_state_dict(torch.load(model_path, map_location="cpu"), strict=True)

    # ------------------------------------------------------------------ packed weights
    def _w2d(self, key):
        """spatial Conv3d (1,k,k) or Conv2d weight -> 2-D channels_last (weight, bias)."""
        def build():
            w = self.P[key + ".weight"]
            if w.dim() == 5:
                w = w[:, :, 0]
            return cl(w), self.P[key + ".bias"].contiguous()
        return self.packed("w2d:" + key, build)

    def _wt(self, key):
        """temporal Conv3d (3,1,1) weight [co,ci,3,1,1] -> 1x1 conv over [x(t-2) | x(t) | x(t+2)]."""
        def build():
            w = self.P[key + ".weight"][:, :, :, 0, 0]                      # [co,ci,3]
            w = w.permute(0, 2, 1).reshape(w.shape[0], -1, 1, 1)             # [co, 3*ci] tap-major
            return cl(w), self.P[key + ".bias"].contiguous()
        return self.packed("wt:" + key, build)

    def _offset_w0(self, name):
        """conv_offset.0 input channels reordered from [prop|cur|n2] (:96) to our scan-buffer order
        [prop|n2|cur] so deform input and condition share one buffer."""
        def build():
            w = self.P[f"feat_prop_module.deform_align.{name}.conv_offset.0.weight"]
            w = torch.cat([w[:, :128], w[:, 256:384], w[:, 128:256]], 1)
            return cl(w), self.P[f"feat_prop_module.deform_align.{name}.conv_offset.0.bias"].contiguous()
        return self.packed("off0:" + name, build)

    def _dcn(self, name):
        def build():
            p = f"feat_prop_module.deform_align.{name}"
            return ops.pack_deform_weight(self.P[p + ".weight"]), self.P[p + ".bias"].contiguous()
        return self.packed("dcn:" + name, build)

    # ------------------------------------------------------------------ blocks
    def _p3d(self, p, x, stride, act="leaky"):
        """P3DBlock :148-169 on a frame batch x [t,c,h,w] (channels_last)."""
        y = conv(x, self._w2d(p + ".conv1.0"), stride, 1, act="leaky", slope=0.2)
        t = y.shape[0]
        yp = F.pad(y, (0, 0, 0, 0, 0, 0, 2, 2))                             # zero-pad time by 2 (padding=(2,0,0))
        z = torch.cat([yp[0:t], yp[2:t + 2], yp[4:t + 4]], 1)                # dilation 2 taps
        return conv(z, self._wt(p + ".conv2.0"), act=act, slope=0.2)

    def _up2_conv(self, key, x, act="none", res=None):
        return conv(up2(x), self._w2d(key + ".conv"), 1, 1, act=act, slope=0.2, res=res)

    def _propagate(self, x, gather_gemm=False):
        """BidirectionalPropagation.forward :67-124.  x [t,128,h,w] channels_last -> same.
        gather_gemm: deformable conv = pp_deform_gather + one 1x1 wgmma GEMM (library convs around it unchanged)."""
        t, c, h, w = x.shape
        dev = x.device
        xs = as_pm(x)                                                         # [t,h,w,128]
        fp = "feat_prop_module."
        results = {}
        for di, name in enumerate(("backward_", "forward_")):
            order = list(range(t))[::-1] if di == 0 else list(range(t))
            hist = torch.zeros(t + 2, h, w, c, device=dev)                   # slots 0,1 = zero states
            # backbone input of every step, [cur | (backward feature) | aligned state] (:101-106), laid out once per scan:
            # the step-independent parts are filled by one copy, each step's deform-align writes its own last slot
            k = 2 + di
            fall = torch.empty(t, h, w, k * c, device=dev)
            fall[..., :c] = xs
            if di == 1:
                fall[..., c:2 * c] = results["backward_"]
            fall[order[0], :, :, -c:] = 0                                     # step 0 propagates the zero state
            dw, db = self._dcn(name)
            if gather_gemm:
                dwp = self.packed("dcnu:" + name, lambda: ops.pack_deform_weight_umma(self.P[f"{fp}deform_align.{name}.weight"]))
                cols = torch.empty(1, h, w, 9 * 256, device=dev)
            for i, idx in enumerate(order):
                pslot = fall[idx:idx + 1, :, :, -c:]                          # [1,h,w,128] view, pixel stride k*128
                if i > 0:
                    # deform input | cur: [state(i-1) | state(i-2) | cur]
                    buf = torch.cat([hist[i + 1:i + 2], hist[i:i + 1], xs[idx:idx + 1]], -1)
                    o = conv(as_nchw(buf), self._offset_w0(name), 1, 1, act="leaky", slope=0.1)
                    o = conv(o, self._w2d(f"{fp}deform_align.{name}.conv_offset.2"), 1, 1, act="leaky", slope=0.1)
                    o = conv(o, self._w2d(f"{fp}deform_align.{name}.conv_offset.4"), 1, 1, act="leaky", slope=0.1)
                    w6, b6 = self._w2d(f"{fp}deform_align.{name}.conv_offset.6")
                    o = as_pm(F.conv2d(o, w6, None, padding=1))             # bias folded into the tap-decoding pre-pass
                    if gather_gemm:
                        ops.deform_gather(buf[:, :, :, :256], o, None, 5.0, cols, o_bias=b6)
                        ops.conv_umma([cols], dwp, 1, 1, c, bias=db, out=pslot)
                    else:
                        ops.deform_align(buf[0, :, :, :256], o[0], None, 5.0, dw, db, pslot[0], o_bias=b6)
                y = conv(as_nchw(fall[idx:idx + 1]), self._w2d(f"{fp}backbone.{name}.0"), 1, 1, act="leaky", slope=0.1)
                # state(i) = aligned + backbone(...) (:108-110): bias, residual add and placement in one epilogue pass
                conv(y, self._w2d(f"{fp}backbone.{name}.2"), 1, 1, res=as_nchw(pslot), out=as_nchw(hist[i + 2:i + 3]))
            seq = hist[2:]
            results[name] = seq.flip(0) if di == 0 else seq
        return conv(as_nchw(torch.cat([results["backward_"], results["forward_"]], -1)), self._w2d(fp + "fusion"), res=x)

    def _uw(self, key, sel, segs, half=False):
        """packed weight of conv `key` restricted to the input channels `sel` (list of (lo, hi)), split into segments `segs`
        (half: fp16, for conv_umma_f16)"""
        def build():
            w = self.P[key + ".weight"]
            if w.dim() == 5:
                w = w[:, :, 0]
            return (ops.pack_conv_weight_f16 if half else ops.pack_conv_weight)(torch.cat([w[:, lo:hi] for lo, hi in sel], 1), segs)
        return self.packed(f"uw{16 if half else ''}:{key}:{sel}:{segs}", build)

    def _propagate_umma(self, x):
        """`_propagate` on the wgmma conv kernel (config.UMMA_CONV): every conv of the scan is one pp_conv2d_umma launch
        with its bias / LeakyReLU / residual / placement fused, the two previous states are read as two input segments straight
        from the history buffer (no torch.cat), the deformable conv is pp_deform_gather (split input) + a 1x1 conv over the
        sampled columns, and the shares of conv_offset.0 / backbone.0 that only see the current frame (and, in the forward
        scan, the finished backward features) are convolved for all frames at once before the scan starts and enter the step
        as a pre-activation addend (conv is linear in its input channels).  8 launches per step (before: ~17).
        Under config.half_convs() the per-step convs take fp16 operands (conv_umma_f16): backbone.2 writes each state in
        fp32 (hist) and its fp16 image (hist16) in one pass, the deformable GEMM writes the aligned features the same way,
        and the sampled columns and t1 / t2 / t3 / y are fp16; the states, the hoisted shares, o and the epilogues stay
        fp32 (DESIGN.md §4 "Precision")."""
        t, c, h, w = x.shape
        dev = x.device
        xs = as_pm(x)                                                         # [t,h,w,128]
        fp = "feat_prop_module."
        U = ops.conv_umma
        P = self.P
        half = x.is_cuda and config.half_convs()
        dt = torch.float16 if half else torch.float32                        # the per-step A operands
        t1, t2, t3, y = (torch.empty(1, h, w, c, device=dev, dtype=dt) for _ in range(4))
        o = torch.empty(1, h, w, 432, device=dev)
        cols = torch.empty(1, h, w, 9 * 2 * c, device=dev, dtype=dt)
        albuf = torch.empty(1, h, w, c, device=dev)
        zero = torch.zeros(1, h, w, c, device=dev)
        if half:                                                              # fp16 images of the aligned features and states
            al16 = torch.empty(1, h, w, c, device=dev, dtype=dt)
            zero16 = torch.zeros(1, h, w, c, device=dev, dtype=dt)
            hist16 = torch.zeros(t + 2, h, w, c, device=dev, dtype=dt)       # slots 0,1 = zero states, never written
        results = {}
        for di, name in enumerate(("backward_", "forward_")):
            order = list(range(t))[::-1] if di == 0 else list(range(t))
            po, pb = f"{fp}deform_align.{name}.conv_offset.", f"{fp}backbone.{name}."
            hist = torch.zeros(t + 2, h, w, c, device=dev)                   # slots 0,1 = zero states
            # conv_offset.0 input = [prop 0:128 | cur 128:256 | n2 256:384] (:93-96); backbone.0 input = [cur | (backward feats) | aligned] (:101-106)
            pre_off = U([xs], self._uw(po + "0", ((c, 2 * c),), (c,)), 3, 3, c, bias=P[po + "0.bias"])
            k = 1 + di
            hsegs = [xs] + ([results["backward_"]] if di == 1 else [])
            pre_bb = U(hsegs, self._uw(pb + "0", ((0, k * c),), (c,) * k), 3, 3, c, bias=P[pb + "0.bias"])
            dbias = P[f"{fp}deform_align.{name}.bias"]
            if half:
                self._scan_f16(hist, hist16, order, k, pre_off, pre_bb, po, pb, name, o, albuf, zero, (t1, t2, t3, y, cols, al16, zero16))
                seq = hist[2:]
                results[name] = seq.flip(0) if di == 0 else seq
                continue
            dwp = self.packed("dcnu:" + name, lambda: ops.pack_deform_weight_umma(P[f"{fp}deform_align.{name}.weight"]))
            for i, idx in enumerate(order):
                if i > 0:
                    s1, s2 = hist[i + 1:i + 2], hist[i:i + 1]                 # state(i-1), state(i-2)
                    U([s1, s2], self._uw(po + "0", ((0, c), (2 * c, 3 * c)), (c, c)), 3, 3, c, pre=pre_off[idx:idx + 1], act="leaky", slope=0.1,
                      out=t1, round_tf32=True)
                    U([t1], self._uw(po + "2", ((0, c),), (c,)), 3, 3, c, bias=P[po + "2.bias"], act="leaky", slope=0.1, out=t2, round_tf32=True)
                    U([t2], self._uw(po + "4", ((0, c),), (c,)), 3, 3, c, bias=P[po + "4.bias"], act="leaky", slope=0.1, out=t3, round_tf32=True)
                    U([t3], self._uw(po + "6", ((0, c),), (c,)), 3, 3, 432, bias=P[po + "6.bias"], out=o)
                    ops.deform_gather(s1, o, None, 5.0, cols, x2=s2)
                    al = U([cols], dwp, 1, 1, c, bias=dbias, out=albuf)
                else:
                    al = zero                                                # step 0 propagates the zero state
                U([al], self._uw(pb + "0", (((k) * c, (k + 1) * c),), (c,)), 3, 3, c, pre=pre_bb[idx:idx + 1], act="leaky", slope=0.1, out=y,
                  round_tf32=True)
                # state(i) = aligned + backbone(...) (:108-110)
                U([y], self._uw(pb + "2", ((0, c),), (c,)), 3, 3, c, bias=P[pb + "2.bias"], res=al, out=hist[i + 2:i + 3])
            seq = hist[2:]
            results[name] = seq.flip(0) if di == 0 else seq
        return as_nchw(U([results["backward_"], results["forward_"]], self._uw(fp + "fusion", ((0, 2 * c),), (c, c)), 1, 1, c,
                         bias=P[fp + "fusion.bias"], res=xs))

    def _scan_f16(self, hist, hist16, order, k, pre_off, pre_bb, po, pb, name, o, albuf, zero, bufs):
        """the sequential loop of `_propagate_umma` on fp16 operands: state(i) goes to hist[i + 2] (fp32) and hist16[i + 2]"""
        c = hist.shape[-1]
        fp = "feat_prop_module."
        H = ops.conv_umma_f16
        P = self.P
        t1, t2, t3, y, cols, al16, zero16 = bufs
        dwp = self.packed("dcnu16:" + name, lambda: ops.pack_deform_weight_umma_f16(P[f"{fp}deform_align.{name}.weight"]))
        dbias = P[f"{fp}deform_align.{name}.bias"]
        for i, idx in enumerate(order):
            if i > 0:
                H([hist16[i + 1:i + 2], hist16[i:i + 1]], self._uw(po + "0", ((0, c), (2 * c, 3 * c)), (c, c), True), 3, 3, c,
                  pre=pre_off[idx:idx + 1], act="leaky", slope=0.1, out16=t1)
                H([t1], self._uw(po + "2", ((0, c),), (c,), True), 3, 3, c, bias=P[po + "2.bias"], act="leaky", slope=0.1, out16=t2)
                H([t2], self._uw(po + "4", ((0, c),), (c,), True), 3, 3, c, bias=P[po + "4.bias"], act="leaky", slope=0.1, out16=t3)
                H([t3], self._uw(po + "6", ((0, c),), (c,), True), 3, 3, 432, bias=P[po + "6.bias"], out=o)
                ops.deform_gather(hist[i + 1:i + 2], o, None, 5.0, cols, x2=hist[i:i + 1])
                H([cols], dwp, 1, 1, c, bias=dbias, out=albuf, out16=al16)
                al, a16 = albuf, al16
            else:
                al, a16 = zero, zero16                                      # step 0 propagates the zero state
            H([a16], self._uw(pb + "0", ((k * c, (k + 1) * c),), (c,), True), 3, 3, c, pre=pre_bb[idx:idx + 1], act="leaky", slope=0.1,
              out16=y)
            H([y], self._uw(pb + "2", ((0, c),), (c,), True), 3, 3, c, bias=P[pb + "2.bias"], res=al, out=hist[i + 2:i + 3],
              out16=hist16[i + 2:i + 3])

    def _lw(self, key, sel, bias=True):
        """(channels_last 2-D conv weight, bias | None) of conv `key` restricted to the input channel ranges `sel`"""
        def build():
            w = self.P[key + ".weight"]
            if w.dim() == 5:
                w = w[:, :, 0]
            return cl(torch.cat([w[:, lo:hi] for lo, hi in sel], 1)), (self.P[key + ".bias"].contiguous() if bias else None)
        return self.packed(f"lw:{key}:{sel}:{bias}", build)

    def _propagate_hoisted(self, x, gather_gemm=False):
        """`_propagate` with library convs and the algebra of `_propagate_umma`: the shares of conv_offset.0 / backbone.0
        over the current frame (and, in the forward scan, the finished backward features) are one batched conv per scan;
        the per-step convs see only the state-dependent channels (K = 2304 instead of 3456, 1152 instead of 2304 / 3456)
        and add the hoisted share through pp_bias_act_pre."""
        t, c, h, w = x.shape
        dev = x.device
        xs = as_pm(x)                                                         # [t,h,w,128]
        fp = "feat_prop_module."
        albuf = torch.empty(1, h, w, c, device=dev)
        zero = torch.zeros(1, h, w, c, device=dev)
        results = {}
        for di, name in enumerate(("backward_", "forward_")):
            order = list(range(t))[::-1] if di == 0 else list(range(t))
            po, pb = f"{fp}deform_align.{name}.conv_offset.", f"{fp}backbone.{name}."
            hist = torch.zeros(t + 2, h, w, c, device=dev)                   # slots 0,1 = zero states
            # conv_offset.0 input = [prop 0:128 | cur 128:256 | n2 256:384] (:93-96); backbone.0 input = [cur | (backward feats) | aligned] (:101-106)
            pre_off = as_pm(conv(x, self._lw(po + "0", ((c, 2 * c),)), 1, 1))
            k = 1 + di
            hx = x if di == 0 else as_nchw(torch.cat([xs, results["backward_"]], -1))
            pre_bb = as_pm(conv(hx, self._lw(pb + "0", ((0, k * c),)), 1, 1))
            dw, db = self._dcn(name)
            if gather_gemm:
                dwp = self.packed("dcnu:" + name, lambda: ops.pack_deform_weight_umma(self.P[f"{fp}deform_align.{name}.weight"]))
                cols = torch.empty(1, h, w, 9 * 2 * c, device=dev)
            for i, idx in enumerate(order):
                if i > 0:
                    buf = torch.cat([hist[i + 1:i + 2], hist[i:i + 1]], -1)  # [state(i-1) | state(i-2)]
                    o = conv(as_nchw(buf), self._lw(po + "0", ((0, c), (2 * c, 3 * c)), False), 1, 1, act="leaky", slope=0.1,
                             pre=as_nchw(pre_off[idx:idx + 1]))
                    o = conv(o, self._w2d(po + "2"), 1, 1, act="leaky", slope=0.1)
                    o = conv(o, self._w2d(po + "4"), 1, 1, act="leaky", slope=0.1)
                    w6, b6 = self._w2d(po + "6")
                    o = as_pm(F.conv2d(o, w6, None, padding=1))             # bias folded into the tap decoding
                    if gather_gemm:
                        ops.deform_gather(buf, o, None, 5.0, cols, o_bias=b6)
                        ops.conv_umma([cols], dwp, 1, 1, c, bias=db, out=albuf)
                    else:
                        ops.deform_align(buf[0], o[0], None, 5.0, dw, db, albuf[0], o_bias=b6)
                    al = albuf
                else:
                    al = zero                                                # step 0 propagates the zero state
                y = conv(as_nchw(al), self._lw(pb + "0", ((k * c, (k + 1) * c),), False), 1, 1, act="leaky", slope=0.1,
                         pre=as_nchw(pre_bb[idx:idx + 1]))
                # state(i) = aligned + backbone(...) (:108-110)
                conv(y, self._w2d(pb + "2"), 1, 1, res=as_nchw(al), out=as_nchw(hist[i + 2:i + 3]))
            seq = hist[2:]
            results[name] = seq.flip(0) if di == 0 else seq
        return conv(as_nchw(torch.cat([results["backward_"], results["forward_"]], -1)), self._w2d(fp + "fusion"), res=x)

    # ------------------------------------------------------------------ API
    @torch.no_grad()
    def forward(self, masked_flows, masks):
        """:272-309 (eval).  masked_flows [b,t,2,h,w], masks [b,t,1,h,w] -> (flow [b,t,2,h,w], None)."""
        b, t, _, h, w = masked_flows.shape
        outs = [self.graphs("rfc", self._forward_one, masked_flows[bi].contiguous().float(), masks[bi].contiguous().float())
                for bi in range(b)]
        return torch.stack(outs, 0).view(b, t, 2, h, w).to(masked_flows.dtype), None

    def _forward_one(self, flows, masks):
        """one clip: flows [t,2,h,w], masks [t,1,h,w] -> [t,2,h,w]; captured as a CUDA graph per shape."""
        x = torch.cat([flows, masks], 1)                                         # [t,3,h,w]
        x = F.pad(x, (2, 2, 2, 2), mode="replicate").contiguous(memory_format=torch.channels_last)
        x = conv(x, self._w2d("downsample.0"), 2, 0, act="leaky", slope=0.2)
        e1 = self._p3d("encoder1.0", x, 1)
        e1 = self._p3d("encoder1.2", e1, 2)
        e2 = self._p3d("encoder2.0", e1, 1)
        e2 = self._p3d("encoder2.2", e2, 2)
        m = e2
        for i, d in ((0, 3), (2, 2), (4, 1)):
            m = conv(m, self._w2d(f"mid_dilation.{i}"), 1, d, d, act="leaky", slope=0.2)

        def scan():
            if config.UMMA_CONV == "auto":  # five plans of the same scan (TF32 products; plan 0 on fp16 operands under half_convs, part of the key): keep the fastest
                return autotune.pick(("rfc_prop", tuple(m.shape[1:]), config.half_convs()), (self._propagate_umma, self._propagate, lambda a: self._propagate(a, True),
                                                                        self._propagate_hoisted, lambda a: self._propagate_hoisted(a, True)),
                                     m, reps=2, graph_timed=True)
            if config.UMMA_CONV == "hoisted":
                return self._propagate_hoisted(m)
            if config.UMMA_CONV == "hybrid":
                return self._propagate(m, True)
            return self._propagate_umma(m) if config.UMMA_CONV else self._propagate(m)
        fpr = high_priority(scan)
        d2 = self._up2_conv("decoder2.2", conv(fpr, self._w2d("decoder2.0"), 1, 1, act="leaky", slope=0.2), "leaky", res=e1)
        d1 = self._up2_conv("decoder1.2", conv(d2, self._w2d("decoder1.0"), 1, 1, act="leaky", slope=0.2), "leaky")
        fl = self._up2_conv("upsample.2", conv(d1, self._w2d("upsample.0"), 1, 1, act="leaky", slope=0.2))
        return fl.contiguous()

    @torch.no_grad()
    def forward_bidirect_flow(self, masked_flows_bi, masks):
        """:312-337 (eval).  flows (f,b) each [b,t-1,2,h,w]; masks [b,t,1,h,w]."""
        mf, mb = masks[:, :-1].contiguous(), masks[:, 1:].contiguous()
        xf, xb = masked_flows_bi[0] * (1 - mf), torch.flip(masked_flows_bi[1] * (1 - mb), dims=[1])
        mbf = torch.flip(mb, dims=[1])
        b, t, _, h, w = xf.shape
        pf, pb = [], []
        for bi in range(b):
            f, g = self.graphs("rfc_bi", self._forward_pair, xf[bi].contiguous().float(), mf[bi].contiguous().float(),
                               xb[bi].contiguous().float(), mbf[bi].contiguous().float())
            pf.append(f)
            pb.append(g)
        dt = masked_flows_bi[0].dtype                              # fp16 storage in, fp16 out; the scan itself is fp32
        pf, pb = torch.stack(pf, 0).view(b, t, 2, h, w).to(dt), torch.stack(pb, 0).view(b, t, 2, h, w).to(dt)
        return [pf, torch.flip(pb, dims=[1])], [None, None]

    def _forward_pair(self, xf, mf, xb, mb):
        """The two directions are independent recurrent scans over 30x54 maps (312 strictly sequential, latency-bound
        deformable steps per 80-frame clip): run them on two streams so their kernels interleave on the GPU.  Inside a
        CUDA-graph capture this becomes two parallel branches of one graph."""
        if not xf.is_cuda:
            return self._forward_one(xf, mf), self._forward_one(xb, mb)
        cur = torch.cuda.current_stream()
        side = self.packed("side_stream", lambda: torch.cuda.Stream(device=xf.device))
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            ob = self._forward_one(xb, mb)
        of = self._forward_one(xf, mf)
        cur.wait_stream(side)
        if not torch.cuda.is_current_stream_capturing():
            ob.record_stream(cur)            # allocated on `side`, consumed on `cur`: keep the block until cur is done with it
        return of, ob

    @torch.no_grad()
    def combine_flow(self, masked_flows_bi, pred_flows_bi, masks):
        """:340-347."""
        mf, mb = masks[:, :-1].contiguous(), masks[:, 1:].contiguous()
        return (pred_flows_bi[0] * mf + masked_flows_bi[0] * (1 - mf),
                pred_flows_bi[1] * mb + masked_flows_bi[1] * (1 - mb))
