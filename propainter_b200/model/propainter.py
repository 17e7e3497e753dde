"""``InpaintGenerator``: image propagation, encoder, flow-guided deformable feature propagation,
mask-guided sparse transformer, decoder -- H100 execution plan.

Drop-in for the generator half of model/propainter.py (:256-372) of the reference: same constructor,
``img_propagation`` / ``forward`` signatures and results, same state_dict (216 tensors).  The GAN
discriminators (:378-532) are training-only and not part of the inference path.
"""
import torch
import torch.nn.functional as F

from .. import autotune, config, ops
from .._params import ParamNet
from ..graphs import high_priority
from ..nn_util import as_nchw, as_pm, cl, conv, pad_in_channels, up2
from ..schemas import generator_schema
from ..window_index import padded_grid, token_grid
from .modules.sparse_transformer import WIN, TransformerExec


def _flow_in(f):
    """a window's completed flows as gen_prep reads them: fp16 clip storage as it is (pp_gen_prep_f16 widens it on load),
    anything else as fp32"""
    return f.contiguous() if f.dtype == torch.float16 else f.contiguous().float()


def _lrelu(x, s=0.2):
    return F.leaky_relu_(x, s)


class InpaintGenerator(ParamNet):
    def __init__(self, init_weights=True, model_path=None, seed=None):
        # `init_weights` is kept for signature compatibility; a fresh net is always given a seeded
        # synthetic init (the reference's N(0,0.02) init is a training detail, base_module.py:22-56).
        super().__init__(generator_schema(), seed=seed)
        self.tx = TransformerExec(self)
        if model_path is not None:
            print("Pretrained ProPainter has loaded...")
            self.load_state_dict(torch.load(model_path, map_location="cpu"), strict=True)

    # ------------------------------------------------------------------ packed weights
    def _wb(self, key, cin_pad=None):
        def build():
            w = self.P[key + ".weight"]
            if cin_pad is not None:
                w = pad_in_channels(w, cin_pad)
            return cl(w), self.P[key + ".bias"].contiguous()
        return self.packed(f"wb:{key}:{cin_pad}", build)

    def _wb16(self, key, cin_pad=None):
        """_wb with an fp16 weight (the bias stays fp32) for the half-operand convs"""
        return self.packed(f"f16:{key}:{cin_pad}", lambda: (self._wb(key, cin_pad)[0].half(), self._wb(key, cin_pad)[1]))

    def _wb_group(self, key, j, g):
        """(weight, bias) of group j of a grouped conv, as a dense conv."""
        def build():
            w, b = self.P[key + ".weight"], self.P[key + ".bias"]
            co = w.shape[0] // g
            return cl(w[j * co:(j + 1) * co]), b[j * co:(j + 1) * co].contiguous()
        return self.packed(f"wbg:{key}:{j}", build)

    def _dcn(self, name):
        def build():
            p = f"feat_prop_module.deform_align.{name}"
            return ops.pack_deform_weight(self.P[p + ".weight"]), self.P[p + ".bias"].contiguous()
        return self.packed("dcn:" + name, build)

    # ------------------------------------------------------------------ image propagation
    @torch.no_grad()
    def img_propagation(self, masked_frames, completed_flows, masks, interpolation="nearest"):
        """propainter.py:315-317 -> BidirectionalPropagation(3, learnable=False) :104-190, as one fused scan."""
        if interpolation not in ("nearest", "bilinear"):
            raise ValueError(f"unsupported interpolation {interpolation!r}")
        if tuple(masked_frames.shape[-2:]) != tuple(completed_flows[0].shape[-2:]):
            raise ValueError("The spatial sizes of input and flow are not the same.")     # flow_loss_utils.py:25-27
        b = masked_frames.shape[0]
        fr, mk = [], []
        for i in range(b):
            f, m = ops.img_prop_scan(masked_frames[i].contiguous().float(), completed_flows[0][i].contiguous().float(),
                                     completed_flows[1][i].contiguous().float(), masks[i].contiguous().float(),
                                     interpolation == "nearest")
            fr.append(f)
            mk.append(m)
        dt = masked_frames.dtype                                   # fp16 callers (--fp16) get fp16 back; math is fp32
        return torch.stack(fr, 0).to(dt), torch.stack(mk, 0).to(dt)

    # ------------------------------------------------------------------ conv trunk
    def _encoder(self, x):
        """Encoder.forward propainter.py:218-232; x [n,8,H,W] channels_last (5 real + 3 zero channels)."""
        L = dict(act="leaky", slope=0.2)
        out = conv(x, self._wb("encoder.layers.0", 8), 2, 1, **L)
        out = conv(out, self._wb("encoder.layers.2"), 1, 1, **L)
        out = conv(out, self._wb("encoder.layers.4"), 2, 1, **L)
        out = conv(out, self._wb("encoder.layers.6"), 1, 1, **L)
        x0 = as_pm(out)                                                       # [n,h,w,256]
        n, h, w, _ = x0.shape
        out = conv(out, self._wb("encoder.layers.8"), 1, 1, **L)
        for i, g in ((10, 2), (12, 4), (14, 8), (16, 1)):
            key = f"encoder.layers.{i}"

            def grouped(x0, o, key=key, g=g):               # one grouped conv over the interleaved [x0_j | o_j] groups
                mix = torch.cat([x0.view(n, h, w, g, -1), o.view(n, h, w, g, -1)], -1).view(n, h, w, -1)
                return conv(as_nchw(mix), self._wb(key), 1, 1, 1, g, **L)

            def per_group(x0, o, key=key, g=g):             # the same math as g dense convs (cuDNN's grouped kernels are
                a, b = x0.shape[-1] // g, o.shape[-1] // g  # several times slower than its dense ones at these shapes)
                co = self.P[key + ".weight"].shape[0] // g
                res = torch.empty(n, h, w, g * co, device=x0.device)
                for j in range(g):
                    xin = torch.cat([x0[..., j * a:(j + 1) * a], o[..., j * b:(j + 1) * b]], -1)
                    conv(as_nchw(xin), self._wb_group(key, j, g), 1, 1, out=as_nchw(res[..., j * co:(j + 1) * co]), **L)
                return as_nchw(res)

            o = as_pm(out)
            if g == 1:
                out = grouped(x0, o)
            else:
                out = autotune.pick(("enc_group", i, tuple(x0.shape), tuple(o.shape)), (grouped, per_group), x0, o)
        return out

    def _encoder_half(self, x):
        """_encoder on fp16 operands (config.half_convs): x [n,8,H,W] fp16 channels_last; fp16 weights and maps, cuDNN convs
        with fp32 accumulation, bias + LeakyReLU in fp32 by pp_bias_act, each map rounded once to fp16; layers.16 is widened
        on store, so the result is fp32 [n,128,h,w] channels_last as on the fp32 path."""
        L = dict(act="leaky", slope=0.2)
        out = conv(x, self._wb16("encoder.layers.0", 8), 2, 1, **L)
        out = conv(out, self._wb16("encoder.layers.2"), 1, 1, **L)
        out = conv(out, self._wb16("encoder.layers.4"), 2, 1, **L)
        x0 = as_pm(conv(out, self._wb16("encoder.layers.6"), 1, 1, **L))                # [n,h,w,256]
        raw = as_pm(F.conv2d(as_nchw(x0), self._wb16("encoder.layers.8")[0], None, 1, 1))  # layers.8 before its epilogue
        return autotune.pick(("enc_group", torch.float16, tuple(x0.shape), tuple(raw.shape)),
                             (lambda a, b: self._enc_groups_half(a, b, True), lambda a, b: self._enc_groups_half(a, b, False)),
                             x0, raw)

    def _enc_groups_half(self, x0, raw, interleaved):
        """layers.8's epilogue and the grouped layers 10 / 12 / 14 / 16 on fp16 operands.  Group j of a layer with g groups
        reads [x0_j | o_j] (a = 256/g channels of x0, b of the previous output o).  These inputs are not concatenated: each
        layer's input buffer is allocated in the layout its conv reads -- interleaved [n,h,w,g,a+b] for one grouped conv, or
        group-major [g][n,h,w,a+b] for g dense convs (the per-group plan) -- x0 is copied into its slots once, and the
        previous layer's bias + LeakyReLU (pp_bias_act, one call per group slot it reaches) writes o into the rest."""
        n, h, w, c0 = x0.shape
        pieces, bias = [(raw, 0)], self.P["encoder.layers.8.bias"]        # raw conv outputs and their first output channel
        for i, g in ((10, 2), (12, 4), (14, 8), (16, 1)):
            key = f"encoder.layers.{i}"
            a, b = c0 // g, bias.shape[0] // g
            if interleaved:
                buf = torch.empty(n, h, w, g, a + b, device=x0.device, dtype=torch.float16)
                buf[..., :a].copy_(x0.view(n, h, w, g, a))
                slots = [buf[..., k, :] for k in range(g)]
            else:
                buf = torch.empty(g, n, h, w, a + b, device=x0.device, dtype=torch.float16)
                buf[..., :a].copy_(x0.view(n, h, w, g, a).permute(3, 0, 1, 2, 4))
                slots = list(buf)
            for y, cs in pieces:                   # output channel c of the previous layer -> slot c // b, column a + c % b
                for k in range(cs // b, (cs + y.shape[-1] - 1) // b + 1):
                    lo, hi = max(cs, k * b), min(cs + y.shape[-1], (k + 1) * b)
                    ops.bias_act(y[..., lo - cs:hi - cs], bias[lo:hi], "leaky", 0.2,
                                 out=slots[k][..., a + lo - k * b:a + hi - k * b])
            wt, bias = self._wb16(key)
            co = wt.shape[0] // g
            if interleaved:
                pieces = [(as_pm(F.conv2d(as_nchw(buf.view(n, h, w, -1)), wt, None, 1, 1, 1, g)), 0)]
            else:
                wg = [self.packed(f"f16:wbg:{key}:{j}", lambda j=j: self._wb_group(key, j, g)[0].half()) for j in range(g)]
                pieces = [(as_pm(F.conv2d(as_nchw(slots[j]), wg[j], None, 1, 1)), j * co) for j in range(g)]
        (y, _), = pieces
        return as_nchw(ops.bias_act(y, bias, "leaky", 0.2, out=torch.empty(y.shape, device=y.device)))   # widened to fp32

    def _decoder(self, x):
        """x [lt,128,h,w] channels_last -> the pre-tanh image [lt,3,4h,4w], fp32.  fp16 x (half-operand trunk): fp16 weights
        and maps, fp32 accumulation and epilogues; decoder.6 gets a zero fourth output channel so that its bias is added as
        the fp16 conv output is widened to the fp32 image."""
        L = dict(act="leaky", slope=0.2)
        if x.dtype != torch.float16:
            x = conv(up2(x), self._wb("decoder.0.conv"), 1, 1, **L)
            x = conv(x, self._wb("decoder.2"), 1, 1, **L)
            x = conv(up2(x), self._wb("decoder.4.conv"), 1, 1, **L)
            return conv(x, self._wb("decoder.6"), 1, 1)
        x = conv(up2(x), self._wb16("decoder.0.conv"), 1, 1, **L)
        x = conv(x, self._wb16("decoder.2"), 1, 1, **L)
        x = conv(up2(x), self._wb16("decoder.4.conv"), 1, 1, **L)
        w6, b6 = self.packed("f16:decoder.6", lambda: (cl(F.pad(self.P["decoder.6.weight"], (0, 0, 0, 0, 0, 0, 0, 1))).half(),
                                                       F.pad(self.P["decoder.6.bias"], (0, 1)).contiguous()))
        n, _, H, W = x.shape
        out = torch.empty(n, H, W, 4, device=x.device)
        return conv(x, (w6, b6), 1, 1, out=as_nchw(out))[:, :3]

    # ------------------------------------------------------------------ learnable feature propagation
    def _feat_propagation(self, x, dsf, dsb, pmask, interpolation, gather_gemm=False):
        """BidirectionalPropagation(128, learnable=True).forward propainter.py:104-190.
        x [lt,h,w,128] pixel-major; dsf/dsb [lt-1,h,w,2]; pmask [lt,h,w,2] -> fused [lt,128,h,w].
        gather_gemm: the deformable conv as pp_deform_gather + one 1x1 wgmma GEMM over the sampled columns instead of
        the tap pre-pass + split-K mma.sync kernel + reduce (the library convs around it stay)."""
        if interpolation != "bilinear":
            raise NotImplementedError("the feature propagation path uses bilinear warping (propainter.py:319 default)")
        lt, h, w, C = x.shape
        dev = x.device
        fp = "feat_prop_module."
        cond = torch.empty(1, h, w, 2 * C + 8, device=dev)      # 261 -> 264 channels
        bb = torch.empty(1, h, w, 2 * C + 4, device=dev)        # 258 -> 260 channels
        src = x
        outs = {}
        for name in ("backward_1", "forward_1"):
            bwd = name == "backward_1"
            order = list(range(lt))[::-1] if bwd else list(range(lt))
            dst = torch.empty(lt, h, w, C, device=dev)
            dw, db = self._dcn(name)
            if gather_gemm:
                dwp = self.packed("dcnu:" + name, lambda: ops.pack_deform_weight_umma(self.P[f"{fp}deform_align.{name}.weight"]))
                cols = torch.empty(1, h, w, 9 * C, device=dev)
            prev = None
            for i, idx in enumerate(order):
                if i == 0:
                    ops.prop_cond(src[idx], None, None, None, pmask[idx], None, bb[0], True)
                else:
                    fprop, fchk = (dsf[idx], dsb[idx]) if bwd else (dsb[idx - 1], dsf[idx - 1])
                    ops.prop_cond(src[idx], prev, fprop, fchk, pmask[idx], cond[0], bb[0], False)
                    p = f"{fp}deform_align.{name}.conv_offset."
                    o = conv(as_nchw(cond), self._wb(p + "0", 2 * C + 8), 1, 1, act="leaky", slope=0.1)
                    o = conv(o, self._wb(p + "2"), 1, 1, act="leaky", slope=0.1)
                    o = conv(o, self._wb(p + "4"), 1, 1, act="leaky", slope=0.1)
                    w6, b6 = self._wb(p + "6")
                    o = as_pm(F.conv2d(o, w6, None, padding=1))             # bias folded into the tap-decoding pre-pass
                    if gather_gemm:
                        ops.deform_gather(prev[None], o, fprop[None], 3.0, cols, o_bias=b6)
                        ops.conv_umma([cols], dwp, 1, 1, C, bias=db, out=bb[:, :, :, C:2 * C])
                    else:
                        ops.deform_align(prev, o[0], fprop, 3.0, dw, db, bb[0, :, :, C:2 * C], o_bias=b6)
                y = conv(as_nchw(bb), self._wb(f"{fp}backbone.{name}.0", 2 * C + 4), 1, 1, act="leaky", slope=0.2)
                # feat(idx) = aligned + backbone(...) (:173-176): bias, residual add and placement in one epilogue pass
                conv(y, self._wb(f"{fp}backbone.{name}.2"), 1, 1, res=as_nchw(bb[:, :, :, C:2 * C]), out=as_nchw(dst[idx:idx + 1]))
                prev = dst[idx]
            outs[name] = dst
            src = dst                                            # forward scan consumes the backward features (:138)
        z = torch.cat([outs["backward_1"], outs["forward_1"], pmask, pmask.new_zeros(lt, h, w, 2)], -1)
        z = conv(as_nchw(z), self._wb(fp + "fuse.0", 2 * C + 4), 1, 1, act="leaky", slope=0.2)
        return conv(z, self._wb(fp + "fuse.2"), 1, 1, res=as_nchw(x))

    # ---- the same scan on the wgmma conv kernel (config.UMMA_CONV)
    def _uw(self, key, sel, segs, half=False):
        """packed weight of conv `key` restricted to the input channels `sel` (list of (lo, hi)) split into segments `segs`
        (half: fp16, for conv_umma_f16)"""
        def build():
            w = self.P[key + ".weight"]
            return (ops.pack_conv_weight_f16 if half else ops.pack_conv_weight)(torch.cat([w[:, lo:hi] for lo, hi in sel], 1), segs)
        return self.packed(f"uw{16 if half else ''}:{key}:{sel}:{segs}", build)

    def _ub(self, key):
        return self.P[key + ".bias"]

    def _feat_propagation_umma(self, x, dsf, dsb, pmask):
        """`_feat_propagation` with every conv of the scan on pp_conv2d_umma (wgmma, TF32 products, fused bias /
        activation / residual / placement epilogues, multi-segment inputs instead of concat buffers) and the deformable
        conv as pp_deform_gather + a 1x1 pp_conv2d_umma.  Only the part of each conv that depends on the recurrent state
        stays inside the sequential loop: conv(cat[a, b]) = conv_a(a) + conv_b(b), so the shares of conv_offset.0 and
        backbone.0 that see the current frame, the flow / validity / mask channels (all known before the scan starts) are
        convolved once per scan for all frames in one batched launch and enter the step as a pre-activation addend.
        Per step: 1 warp + 4 offset convs + gather + GEMM + 2 backbone convs = 9 launches (before: ~17), K on the critical
        path 7 x 1152 (before: 2376 + 3 x 1152 + 1152 + 2340 + 1152).
        Under config.half_convs() the per-step convs take fp16 operands (conv_umma_f16): the warped features, the sampled
        columns and the conv outputs t1 / t2 / t3 / y are fp16; the state, the aligned features (backbone.2's residual), the
        hoisted shares, the offset-net output o and all epilogue arithmetic stay fp32 (DESIGN.md §4 "Precision")."""
        lt, h, w, C = x.shape
        dev = x.device
        fp = "feat_prop_module."
        U = ops.conv_umma
        half = x.is_cuda and config.half_convs()
        aux = torch.zeros(lt, h, w, 8, device=dev)                  # [fx fy valid m0 m1 0 0 0]: step-independent condition channels
        aux[..., 3:5] = pmask
        mpad = torch.zeros(lt, h, w, 4, device=dev)                 # mask as a 16-byte aligned segment
        mpad[..., :2] = pmask
        dt = torch.float16 if half else torch.float32                # the per-step A operands
        warp = torch.empty(1, h, w, C, device=dev, dtype=dt)
        t1, t2, t3, y = (torch.empty(1, h, w, C, device=dev, dtype=dt) for _ in range(4))
        o = torch.empty(1, h, w, 432, device=dev)
        cols = torch.empty(1, h, w, 9 * C, device=dev, dtype=dt)
        albuf = torch.empty(1, h, w, C, device=dev)
        al16 = torch.empty(1, h, w, C, device=dev, dtype=dt) if half else None
        src, outs = x, {}
        for name in ("backward_1", "forward_1"):
            bwd = name == "backward_1"
            order = list(range(lt))[::-1] if bwd else list(range(lt))
            po, pb = f"{fp}deform_align.{name}.conv_offset.", f"{fp}backbone.{name}."
            if lt > 1:                                              # (fx, fy, valid) of every frame that has a flow in this direction
                if bwd:
                    ops.flow_warp_fbcheck(None, dsf, dsb, aux=aux[:lt - 1, :, :, :3], want_warp=False)
                else:
                    ops.flow_warp_fbcheck(None, dsb, dsf, aux=aux[1:, :, :, :3], want_warp=False)
            # conv_offset.0 input = [cur 0:128 | warped 128:256 | flow 256:258 | valid 258 | mask 259:261] (propainter.py:151);
            # backbone.0 input = [cur 0:128 | aligned 128:256 | mask 256:258] (:171)
            pre_off = U([src, aux[..., :5]], self._uw(po + "0", ((0, C), (2 * C, 2 * C + 5)), (C, 5)), 3, 3, C, bias=self._ub(po + "0"))
            pre_bb = U([src, mpad[..., :2]], self._uw(pb + "0", ((0, C), (2 * C, 2 * C + 2)), (C, 2)), 3, 3, C, bias=self._ub(pb + "0"))
            dst = torch.empty(lt, h, w, C, device=dev)
            if half:
                self._feat_scan_f16(src, dst, order, bwd, dsf, dsb, pre_off, pre_bb, po, pb, name, o, albuf, (warp, t1, t2, t3, y, cols, al16))
                outs[name] = dst
                src = dst
                continue
            dwp = self.packed("dcnu:" + name, lambda: ops.pack_deform_weight_umma(self.P[f"{fp}deform_align.{name}.weight"]))
            dbias = self.P[f"{fp}deform_align.{name}.bias"]
            prev = None
            for i, idx in enumerate(order):
                if i == 0:
                    al = src[idx:idx + 1]                            # feat_prop = feat_current (:141-143)
                else:
                    fprop = (dsf[idx] if bwd else dsb[idx - 1])[None]
                    ops.flow_warp_fbcheck(prev, fprop, warped=warp, round_tf32=True)
                    U([warp], self._uw(po + "0", ((C, 2 * C),), (C,)), 3, 3, C, pre=pre_off[idx:idx + 1], act="leaky", slope=0.1,
                      out=t1, round_tf32=True)
                    U([t1], self._uw(po + "2", ((0, C),), (C,)), 3, 3, C, bias=self._ub(po + "2"), act="leaky", slope=0.1, out=t2, round_tf32=True)
                    U([t2], self._uw(po + "4", ((0, C),), (C,)), 3, 3, C, bias=self._ub(po + "4"), act="leaky", slope=0.1, out=t3, round_tf32=True)
                    U([t3], self._uw(po + "6", ((0, C),), (C,)), 3, 3, 432, bias=self._ub(po + "6"), out=o)
                    ops.deform_gather(prev, o, fprop, 3.0, cols)
                    al = U([cols], dwp, 1, 1, C, bias=dbias, out=albuf)
                U([al], self._uw(pb + "0", ((C, 2 * C),), (C,)), 3, 3, C, pre=pre_bb[idx:idx + 1], act="leaky", slope=0.2, out=y, round_tf32=True)
                # feat(idx) = aligned + backbone(...) (:173-176)
                prev = U([y], self._uw(pb + "2", ((0, C),), (C,)), 3, 3, C, bias=self._ub(pb + "2"), res=al, out=dst[idx:idx + 1])
            outs[name] = dst
            src = dst                                            # forward scan consumes the backward features (:138)
        z = U([outs["backward_1"], outs["forward_1"], mpad[..., :2]], self._uw(fp + "fuse.0", ((0, 2 * C + 2),), (C, C, 2)), 3, 3, C,
              bias=self._ub(fp + "fuse.0"), act="leaky", slope=0.2, round_tf32=True)
        return as_nchw(U([z], self._uw(fp + "fuse.2", ((0, C),), (C,)), 3, 3, C, bias=self._ub(fp + "fuse.2"), res=x))

    def _feat_scan_f16(self, src, dst, order, bwd, dsf, dsb, pre_off, pre_bb, po, pb, name, o, albuf, bufs):
        """the sequential loop of `_feat_propagation_umma` on fp16 operands; dst (fp32) receives the states"""
        C = src.shape[-1]
        fp = "feat_prop_module."
        H = ops.conv_umma_f16
        warp16, t1, t2, t3, y16, cols16, al16 = bufs
        dwp = self.packed("dcnu16:" + name, lambda: ops.pack_deform_weight_umma_f16(self.P[f"{fp}deform_align.{name}.weight"]))
        dbias = self.P[f"{fp}deform_align.{name}.bias"]
        prev = None
        for i, idx in enumerate(order):
            if i == 0:
                al = src[idx:idx + 1]                                # feat_prop = feat_current (:141-143)
                a16 = al.to(torch.float16)
            else:
                fprop = (dsf[idx] if bwd else dsb[idx - 1])[None]
                ops.flow_warp_fbcheck(prev, fprop, warped=warp16)
                H([warp16], self._uw(po + "0", ((C, 2 * C),), (C,), True), 3, 3, C, pre=pre_off[idx:idx + 1], act="leaky", slope=0.1, out16=t1)
                H([t1], self._uw(po + "2", ((0, C),), (C,), True), 3, 3, C, bias=self._ub(po + "2"), act="leaky", slope=0.1, out16=t2)
                H([t2], self._uw(po + "4", ((0, C),), (C,), True), 3, 3, C, bias=self._ub(po + "4"), act="leaky", slope=0.1, out16=t3)
                H([t3], self._uw(po + "6", ((0, C),), (C,), True), 3, 3, 432, bias=self._ub(po + "6"), out=o)
                ops.deform_gather(prev, o, fprop, 3.0, cols16)
                al, a16 = albuf, al16
                H([cols16], dwp, 1, 1, C, bias=dbias, out=albuf, out16=al16)     # fp32 residual + fp16 operand, one pass
            H([a16], self._uw(pb + "0", ((C, 2 * C),), (C,), True), 3, 3, C, pre=pre_bb[idx:idx + 1], act="leaky", slope=0.2, out16=y16)
            prev = H([y16], self._uw(pb + "2", ((0, C),), (C,), True), 3, 3, C, bias=self._ub(pb + "2"), res=al, out=dst[idx:idx + 1])

    def _lw(self, key, sel, bias=True):
        """(channels_last conv weight, bias | None) of conv `key` restricted to input channels `sel`: list of (lo, hi) ranges
        of the original weight, or ("zero", n) for n zero-weight pad channels, concatenated in that order."""
        def build():
            w = self.P[key + ".weight"]
            parts = [w.new_zeros(w.shape[0], s[1], *w.shape[2:]) if s[0] == "zero" else w[:, s[0]:s[1]] for s in sel]
            return cl(torch.cat(parts, 1)), (self.P[key + ".bias"].contiguous() if bias else None)
        return self.packed(f"lw:{key}:{sel}:{bias}", build)

    def _feat_propagation_hoisted(self, x, dsf, dsb, pmask):
        """`_feat_propagation` with the algebra of `_feat_propagation_umma` but library convs: conv(cat[a, b]) = conv_a(a) +
        conv_b(b), so the shares of conv_offset.0 and backbone.0 over step-independent inputs (current frame, flow, validity,
        mask: 133 of 261 and 130 of 258 input channels) are one batched conv per scan, and the per-step convs see only the
        128 state-dependent channels (K = 1152 instead of 2376 / 2340); their result enters through pp_bias_act_pre.  The
        deformable conv is pp_deform_gather + a 1x1 wgmma GEMM."""
        lt, h, w, C = x.shape
        dev = x.device
        fp = "feat_prop_module."
        hin = torch.zeros(lt, h, w, C + 8, device=dev)            # [cur 0:128 | fx fy valid m0 m1 0 0 0]: everything known before the scan
        aux = hin[..., C:]
        aux[..., 3:5] = pmask
        warp, albuf = torch.empty(1, h, w, C, device=dev), torch.empty(1, h, w, C, device=dev)
        cols = torch.empty(1, h, w, 9 * C, device=dev)
        src, outs = x, {}
        for name in ("backward_1", "forward_1"):
            bwd = name == "backward_1"
            order = list(range(lt))[::-1] if bwd else list(range(lt))
            po, pb = f"{fp}deform_align.{name}.conv_offset.", f"{fp}backbone.{name}."
            hin[..., :C] = src
            aux[..., :3] = 0
            if lt > 1:                                              # (fx, fy, valid) of every frame that has a flow in this direction
                if bwd:
                    ops.flow_warp_fbcheck(None, dsf, dsb, aux=aux[:lt - 1, :, :, :3], want_warp=False)
                else:
                    ops.flow_warp_fbcheck(None, dsb, dsf, aux=aux[1:, :, :, :3], want_warp=False)
            # conv_offset.0 input = [cur 0:128 | warped 128:256 | flow 256:258 | valid 258 | mask 259:261] (propainter.py:151);
            # backbone.0 input = [cur 0:128 | aligned 128:256 | mask 256:258] (:171)
            pre_off = as_pm(conv(as_nchw(hin), self._lw(po + "0", ((0, C), (2 * C, 2 * C + 5), ("zero", 3))), 1, 1))
            pre_bb = as_pm(conv(as_nchw(hin), self._lw(pb + "0", ((0, C), ("zero", 3), (2 * C, 2 * C + 2), ("zero", 3))), 1, 1))
            dst = torch.empty(lt, h, w, C, device=dev)
            dwp = self.packed("dcnu:" + name, lambda: ops.pack_deform_weight_umma(self.P[f"{fp}deform_align.{name}.weight"]))
            dbias = self.P[f"{fp}deform_align.{name}.bias"]
            prev = None
            for i, idx in enumerate(order):
                if i == 0:
                    al = src[idx:idx + 1]                            # feat_prop = feat_current (:141-143)
                else:
                    fprop = (dsf[idx] if bwd else dsb[idx - 1])[None]
                    ops.flow_warp_fbcheck(prev, fprop, warped=warp)
                    o = conv(as_nchw(warp), self._lw(po + "0", ((C, 2 * C),), False), 1, 1, act="leaky", slope=0.1,
                             pre=as_nchw(pre_off[idx:idx + 1]))
                    o = conv(o, self._wb(po + "2"), 1, 1, act="leaky", slope=0.1)
                    o = conv(o, self._wb(po + "4"), 1, 1, act="leaky", slope=0.1)
                    w6, b6 = self._wb(po + "6")
                    o = as_pm(F.conv2d(o, w6, None, padding=1))             # bias folded into the tap decoding
                    ops.deform_gather(prev, o, fprop, 3.0, cols, o_bias=b6)
                    al = ops.conv_umma([cols], dwp, 1, 1, C, bias=dbias, out=albuf)
                y = conv(as_nchw(al), self._lw(pb + "0", ((C, 2 * C),), False), 1, 1, act="leaky", slope=0.2,
                         pre=as_nchw(pre_bb[idx:idx + 1]))
                # feat(idx) = aligned + backbone(...) (:173-176)
                conv(y, self._wb(pb + "2"), 1, 1, res=as_nchw(al), out=as_nchw(dst[idx:idx + 1]))
                prev = dst[idx:idx + 1]
            outs[name] = dst
            src = dst                                            # forward scan consumes the backward features (:138)
        z = torch.cat([outs["backward_1"], outs["forward_1"], pmask, pmask.new_zeros(lt, h, w, 2)], -1)
        z = conv(as_nchw(z), self._wb(fp + "fuse.0", 2 * C + 4), 1, 1, act="leaky", slope=0.2)
        return conv(z, self._wb(fp + "fuse.2"), 1, 1, res=as_nchw(x))

    # ------------------------------------------------------------------ forward
    @torch.no_grad()
    def encode(self, masked_frames, masks_in, masks_updated, chunk=40, out=None):
        """Encoder features of a set of frames: [n,3,H,W], [n,1,H,W], [n,1,H,W] -> [n,128,H/4,W/4].
        The encoder output of a frame depends only on (frame, mask_in, mask_updated), so the sliding-window
        driver calls this once per clip and feeds ``forward_features``; the reference re-encodes every frame
        in each of the ~3.5 windows that select it (propainter.py:330-333, 58 % of the generator's conv FLOPs).
        `out` (fp16 pixel-major [n,H/4,W/4,128], half-precision clip storage): each chunk's features are rounded once
        into it instead of being concatenated, and `out` is returned."""
        outs = []
        for s in range(0, masked_frames.shape[0], chunk):
            o = self.graphs("gen_enc", self._encode_frames, masked_frames[s:s + chunk].contiguous().float(),
                            masks_in[s:s + chunk].contiguous().float(), masks_updated[s:s + chunk].contiguous().float())
            if out is None:
                outs.append(o)
            else:
                out[s:s + o.shape[0]].copy_(o.permute(0, 2, 3, 1))
        return torch.cat(outs, 0) if out is None else out

    def _encode_frames(self, fr, mi, mu):
        n, _, H, W = fr.shape
        if fr.is_cuda and config.half_convs():
            x = torch.zeros(n, H, W, 8, device=fr.device, dtype=torch.float16)
            for c0, t in ((0, fr), (3, mi), (4, mu)):
                x[..., c0:c0 + t.shape[1]].copy_(as_pm(t))
            return self._encoder_half(as_nchw(x))
        x = torch.cat([fr, mi, mu, fr.new_zeros(n, 3, H, W)], 1).contiguous(memory_format=torch.channels_last)
        return self._encoder(x).contiguous(memory_format=torch.channels_last)

    @torch.no_grad()
    def forward_features(self, enc_feat, completed_flows, masks_in, masks_updated, num_local_frames,
                         interpolation="bilinear", t_dilation=2, slot=0):
        """``forward`` minus the encoder: enc_feat [t,128,h,w] (local frames first), flows 2x[lt-1,2,H,W] (fp16 or fp32),
        masks [t,1,H,W] -> [lt,3,H,W].  `slot` selects an independent captured-graph instance so that several
        windows can be in flight on different streams."""
        lt = num_local_frames
        return self.graphs(("gen_feat", lt, interpolation, t_dilation, slot),
                           lambda *a: self._forward_features(*a, lt, interpolation, t_dilation),
                           enc_feat.contiguous(memory_format=torch.channels_last), _flow_in(completed_flows[0]),
                           _flow_in(completed_flows[1]), masks_in.contiguous().float(),
                           masks_updated.contiguous().float())

    @torch.no_grad()
    def forward(self, masked_frames, completed_flows, masks_in, masks_updated, num_local_frames,
                interpolation="bilinear", t_dilation=2):
        """propainter.py:319-372 (eval).  masked_frames [b,t,3,H,W], flows 2x[b,lt-1,2,H,W],
        masks [b,t,1,H,W] -> [b,lt,3,H,W] in (-1,1)."""
        lt = num_local_frames
        b, t, _, H, W = masked_frames.shape
        if H % 8 or W % 8:
            raise ValueError("H and W must be multiples of 8 (inference_propainter.py:34-45)")
        res = []
        for bi in range(b):
            enc = self.encode(masked_frames[bi], masks_in[bi], masks_updated[bi])
            res.append(self.forward_features(enc, (completed_flows[0][bi], completed_flows[1][bi]), masks_in[bi],
                                             masks_updated[bi], lt, interpolation, t_dilation))
        return torch.stack(res, 0).view(b, lt, 3, H, W).to(masked_frames.dtype)

    @torch.no_grad()
    def forward_parts(self, masked_frames, completed_flows, masks_in, masks_updated, num_local_frames, interpolation="bilinear",
                      t_dilation=2):
        """`forward` for one clip (b = 1), run eagerly, that also returns the intermediate tensors the oracle exposes
        (oracle/generator_ref.generator_forward(return_parts=True)): the propagated local features, the tokens entering and
        leaving the transformer and the features handed to the decoder -- so parity tests can localise an error instead of
        only seeing it after the tanh."""
        lt = num_local_frames
        enc = self._encode_frames(masked_frames[0].contiguous().float(), masks_in[0].contiguous().float(),
                                  masks_updated[0].contiguous().float())
        parts = {}
        out = self._forward_features(enc, completed_flows[0][0].contiguous().float(), completed_flows[1][0].contiguous().float(),
                                     masks_in[0].contiguous().float(), masks_updated[0].contiguous().float(), lt, interpolation, t_dilation,
                                     parts=parts)
        return out.unsqueeze(0), parts

    def _forward_features(self, enc, flows_f, flows_b, mi, mu, lt, interpolation, t_dilation, parts=None):
        """one window after the encoder; captured as one CUDA graph per shape signature."""
        h, w = enc.shape[-2:]
        dsf, dsb, pmask = ops.gen_prep(flows_f, flows_b, mi, mu, lt)
        fh, fw = token_grid((h, w))
        H2, W2 = padded_grid(fh, fw, WIN)
        flags = ops.window_mask(pmask, fh, fw, H2 // WIN[0], W2 // WIN[1])
        enc_pm = as_pm(enc)
        if interpolation != "bilinear":
            raise NotImplementedError("the feature propagation path uses bilinear warping (propainter.py:319 default)")
        xl = enc_pm[:lt]

        def scan():
            if config.UMMA_CONV == "auto":  # four plans of the same scan (TF32 products; plan 0 on fp16 operands under half_convs, part of the key): keep the fastest
                return autotune.pick(("gen_prop", tuple(xl.shape[1:]), config.half_convs()), (lambda a, b, c, d: self._feat_propagation_umma(a, b, c, d),
                                                                          lambda a, b, c, d: self._feat_propagation(a, b, c, d, interpolation),
                                                                          lambda a, b, c, d: self._feat_propagation(a, b, c, d, interpolation, True),
                                                                          lambda a, b, c, d: self._feat_propagation_hoisted(a, b, c, d)),
                                     xl, dsf, dsb, pmask, reps=2, graph_timed=True)
            if config.UMMA_CONV == "hoisted":
                return self._feat_propagation_hoisted(xl, dsf, dsb, pmask)
            if config.UMMA_CONV == "hybrid":
                return self._feat_propagation(xl, dsf, dsb, pmask, interpolation, True)
            if config.UMMA_CONV:
                return self._feat_propagation_umma(xl, dsf, dsb, pmask)
            return self._feat_propagation(xl, dsf, dsb, pmask, interpolation)
        local = high_priority(scan)
        # half-operand trunk (config.half_convs): SoftSplit, SoftComp, sc.bias_conv and the decoder take fp16 operands with
        # fp32 accumulation; the transformer's residual stream and SoftComp's residual (the fp32 scan output) stay fp32
        half = enc.is_cuda and config.half_convs()
        if half:
            t = enc.shape[0]
            enc2 = torch.empty(t, h, w, enc.shape[1], device=enc.device, dtype=torch.float16)
            enc2[:lt].copy_(as_pm(local))
            enc2[lt:].copy_(enc_pm[lt:])
            enc2 = as_nchw(enc2)
        else:
            enc2 = torch.cat([local, enc[lt:]], 0).contiguous(memory_format=torch.channels_last)
        tok_in = self.tx.soft_split(enc2)
        tok = self.tx.run(tok_in, (h, w), flags, t_dilation)
        # trans_feat + enc_feat (:365-366).  Only the local frames reach the decoder, so SoftComp runs for them alone; the
        # parity path computes every frame, in fp32, for parts["enc_out"]
        if parts is None:
            enc3 = self.tx.soft_comp(tok, (h, w), local, lt, half, torch.float16 if half else torch.float32)
        else:
            res = torch.cat([local, enc[lt:]], 0).contiguous(memory_format=torch.channels_last)
            enc3 = self.tx.soft_comp(tok, (h, w), res, enc.shape[0], half)
            parts.update(prop_feat=local.contiguous(), tokens_in=tok_in, tokens_out=tok, enc_out=enc3.contiguous())
            enc3 = enc3[:lt].half() if half else enc3[:lt]
        return torch.tanh(self._decoder(enc3)).contiguous()
