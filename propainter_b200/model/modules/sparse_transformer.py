"""Soft split / composition and the mask-guided sparse temporal transformer (H100 execution plan).

Reference: model/modules/sparse_transformer.py (SoftSplit :7-31, SoftComp :34-61, FusionFeedForward
:64-101, SparseWindowAttention :117-281, TemporalSparseTransformer(Block) :284-344).  Parameters live in
the owning ``InpaintGenerator`` (a ParamNet); these helpers only execute.

  * SoftSplit  = unfold(7,3,3) + Linear(6272->512) == one strided 7x7 conv  (no 325 MB im2col buffer)
  * SoftComp   = Linear(512->6272) + fold == one transposed conv + a constant (folded-bias) map
  * attention  = LayerNorm, fused QKV GEMM, pooled K/V, then ``ops.sparse_window_attn`` which gathers
                 own / rolled / pooled keys arithmetically (no roll / window_partition / cat / index copies,
                 no score matrix in HBM) and handles masked and unmasked windows in one call
  * fusion FFN = GEMM, ``ops.ffn_overlap_add`` (fold -> normalise -> unfold -> GELU as two stencil
                 kernels on tap-major columns), GEMM
"""
import torch
import torch.nn.functional as F

from ... import autotune, config, ops
from ...nn_util import as_nchw, as_pm, cl, conv
from ...window_index import padded_grid, token_grid, window_key_table

WIN = (5, 9)
POOL = (4, 4)
KS, ST, PD = 7, 3, 3


class TransformerExec:
    def __init__(self, net, depths=8, hidden=512, channel=128, ffn_ch=40):
        self.net, self.depths, self.hidden, self.channel, self.ffn_ch = net, depths, hidden, channel, ffn_ch

    # ------------------------------------------------------------------ packed weights
    def _ss(self):
        def build():
            P = self.net.P
            return cl(P["ss.embedding.weight"].view(self.hidden, self.channel, KS, KS)), P["ss.embedding.bias"].contiguous()
        return self.net.packed("ss", build)

    def _sc(self):
        def build():
            P = self.net.P
            w = P["sc.embedding.weight"].view(self.channel, KS, KS, self.hidden).permute(3, 0, 1, 2).contiguous()
            return w
        return self.net.packed("sc", build)

    def _sc_bias_map(self, hw):
        """fold of the Linear bias: constant per (h,w); sparse_transformer.py:52-59."""
        def build():
            fh, fw = token_grid(hw)
            b = self.net.P["sc.embedding.bias"].view(1, -1, 1).expand(1, -1, fh * fw)
            return F.fold(b, hw, (KS, KS), stride=ST, padding=PD).contiguous(memory_format=torch.channels_last)
        return self.net.packed(f"scb:{hw}", build)

    def _qkv(self, i):
        def build():
            P, p = self.net.P, f"transformers.transformer.{i}.attention."
            w = torch.cat([P[p + "query.weight"], P[p + "key.weight"], P[p + "value.weight"]], 0).contiguous()
            b = torch.cat([P[p + "query.bias"], P[p + "key.bias"], P[p + "value.bias"]], 0).contiguous()
            wkv = torch.cat([P[p + "key.weight"], P[p + "value.weight"]], 0).contiguous()
            bkv = torch.cat([P[p + "key.bias"], P[p + "value.bias"]], 0).contiguous()
            wpool = P[p + "pool_layer.weight"]                                     # [C,1,kh,kw] -> tap-major [kh*kw, C]
            return w, b, wkv, bkv, wpool.reshape(wpool.shape[0], -1).t().contiguous(), P[p + "pool_layer.bias"].contiguous()
        return self.net.packed(f"qkv{i}", build)

    def _ffn(self, i):
        def build():
            P, p = self.net.P, f"transformers.transformer.{i}.mlp."
            ch = self.ffn_ch
            perm = torch.arange(49 * ch, device=P[p + "fc1.0.weight"].device).view(ch, 49).t().reshape(-1)
            return (P[p + "fc1.0.weight"][perm].contiguous(), P[p + "fc1.0.bias"][perm].contiguous(),
                    P[p + "fc2.1.weight"][:, perm].contiguous(), P[p + "fc2.1.bias"].contiguous())
        return self.net.packed(f"ffn{i}", build)

    def _qkv_half(self, i):
        """fp16 copies of the fused QKV and pooled K/V weights and biases; the depthwise pooling weights stay fp32"""
        return self.net.packed(f"f16:qkv{i}", lambda: tuple(t.half() for t in self._qkv(i)[:4]) + self._qkv(i)[4:])

    def _proj_half(self, i):
        P, p = self.net.P, f"transformers.transformer.{i}.attention.proj."
        return self.net.packed(f"f16:proj{i}", lambda: (P[p + "weight"].half(), P[p + "bias"].half()))

    def _ffn_half(self, i):
        """fp16 copies of fc1 / fc2 weights and biases"""
        return self.net.packed(f"f16:ffn{i}", lambda: tuple(t.half() for t in self._ffn(i)))

    def _ss_half(self):
        """fp16 copy of the SoftSplit conv weight; the bias stays fp32"""
        return self.net.packed("f16:ss", lambda: (self._ss()[0].half(), self._ss()[1]))

    def _sc_half(self):
        """fp16 SoftComp weights: the transposed-conv weight, and the Linear weight with its output rows tap-major
        (row tap*C + c; the Linear's own rows are c*49 + tap, fold's channel-major order) for the GEMM + fold plan"""
        def build():
            W = self.net.P["sc.embedding.weight"]
            wcol = W.view(self.channel, KS * KS, self.hidden).transpose(0, 1).reshape(-1, self.hidden)
            return self._sc().half(), wcol.half().contiguous()
        return self.net.packed("f16:sc", build)

    def _scbc(self, half):
        P = self.net.P
        wb = self.net.packed("scbc", lambda: (cl(P["sc.bias_conv.weight"]), P["sc.bias_conv.bias"].contiguous()))
        return self.net.packed("f16:scbc", lambda: (wb[0].half(), wb[1])) if half else wb

    # ------------------------------------------------------------------ soft split / composition
    def soft_split(self, feat):
        """feat [t,c,h,w] channels_last -> tokens [t,fh,fw,hidden] pixel-major, fp32 (SoftSplit.forward :19-31).  fp16 feat
        (half-operand trunk): fp16 weight, fp32 accumulation, and the bias is added as the fp16 conv output is widened."""
        if feat.dtype == torch.float16:
            t, _, h, w = feat.shape
            fh, fw = token_grid((h, w))
            out = torch.empty(t, fh, fw, self.hidden, device=feat.device)
            conv(feat, self._ss_half(), ST, PD, out=as_nchw(out))
            return out
        return as_pm(conv(feat, self._ss(), ST, PD))

    def soft_comp(self, tokens, hw, res, frames, half=False, out_dtype=torch.float32):
        """tokens [t,fh,fw,hidden] -> [frames,c,h,w] for the first `frames` frames (SoftComp.forward :49-61); `res` [frames,c,h,w]
        = skip added in the last conv's epilogue.  half: fp16 operands with fp32 accumulation -- the Linear + fold as either a
        fp16 transposed conv or a fp16 GEMM into tap-major columns + pp_sc_fold_f16 (whichever measures faster), then
        sc.bias_conv on the fp16 result; the output is written in `out_dtype`."""
        fh, fw = tokens.shape[1:3]
        tok = tokens[:frames]
        bmap = self._sc_bias_map(tuple(hw))
        if not half:
            op = (hw[0] + 2 - 3 * fh, hw[1] + 2 - 3 * fw)
            y = F.conv_transpose2d(as_nchw(tok), self._sc(), None, stride=ST, padding=PD, output_padding=op)
            y = y + bmap
        else:
            tok16 = tok.half()
            wt, wcol = self._sc_half()

            def tconv(tok16):
                op = (hw[0] + 2 - 3 * fh, hw[1] + 2 - 3 * fw)
                y = F.conv_transpose2d(as_nchw(tok16), wt, None, stride=ST, padding=PD, output_padding=op)
                return torch.add(y, bmap, out=torch.empty_like(y))            # fp32 sum, rounded once to fp16

            def fold(tok16):
                with config.fp32_reductions():
                    cols = torch.mm(tok16.view(-1, self.hidden), wcol.t())
                return as_nchw(ops.sc_fold(cols, as_pm(bmap)[0], frames, hw[0], hw[1]))
            y = autotune.pick(("sc_half", tuple(tok16.shape), tuple(hw)), (fold, tconv), tok16)
        out = torch.empty(frames, hw[0], hw[1], self.channel, device=tokens.device, dtype=out_dtype)
        return conv(y, self._scbc(half), 1, 1, res=res, out=as_nchw(out))

    # ------------------------------------------------------------------ transformer
    def run(self, tokens, hw, flags, t_dilation=2):
        """tokens [t,fh,fw,C]; flags int32 [n_windows] (1 = masked window).  :294-344."""
        assert self.depths % t_dilation == 0, "wrong t_dilation input."
        with config.linear_precision():
            if tokens.is_cuda and config.half_linears():              # cuBLAS only: elsewhere there is no TF32
                with config.fp32_reductions():
                    return self._run(tokens, hw, flags, t_dilation, True)
            return self._run(tokens, hw, flags, t_dilation, False)

    def _run(self, tokens, hw, flags, t_dilation, half):
        t, fh, fw, C = tokens.shape
        H2, W2 = padded_grid(fh, fw, WIN)
        NT = H2 * W2
        key_tok = self.net.packed(f"ktab:{H2}x{W2}", lambda: torch.from_numpy(window_key_table(H2, W2, WIN)).to(tokens.device))
        P = self.net.P
        x = tokens.contiguous()
        pad = (H2 != fh) or (W2 != fw)
        norm = lambda i, k: (P[f"transformers.transformer.{i}.norm{k}.weight"], P[f"transformers.transformer.{i}.norm{k}.bias"])
        yd = {"y_dtype": torch.float16} if half else {}                # half: every LayerNorm output is a GEMM operand
        _, y = ops.add_layernorm(x, None, *norm(0, 1), **yd)
        for i in range(self.depths):
            p = f"transformers.transformer.{i}."
            wqkv, bqkv, wkv, bkv, wpool, bpool = self._qkv_half(i) if half else self._qkv(i)
            wproj, bproj = self._proj_half(i) if half else (P[p + "attention.proj.weight"], P[p + "attention.proj.bias"])
            if pad:                                                    # zeros are padded *before* q/k/v (:168-176)
                y = F.pad(y, (0, 0, 0, W2 - fw, 0, H2 - fh))
            qkv = F.linear(y, wqkv, bqkv).view(t, NT, 3 * C)
            pooled = ops.pool_depthwise(y, wpool, bpool, POOL[0], POOL[1])                      # [t,ph,pw,C]
            pool_kv = F.linear(pooled.reshape(t, -1, C), wkv, bkv)                              # [t,NP,2C]
            att = ops.sparse_window_attn(qkv, pool_kv, key_tok, flags, t, NT, i % t_dilation, t_dilation,
                                         WN=WIN[0] * WIN[1], C=C).view(t, H2, W2, C)
            if pad:
                att = att[:, :fh, :fw]
            # x = x + proj(att); y = norm2(x)   (residual add fused into the LayerNorm pass)
            x, y = ops.add_layernorm(x, F.linear(att, wproj, bproj), *norm(i, 2), **yd)
            w1, b1, w2, b2 = self._ffn_half(i) if half else self._ffn(i)
            hdn = F.linear(y.reshape(t * fh * fw, C), w1, b1)
            hdn = ops.ffn_overlap_add(hdn, t, hw[0], hw[1], self.ffn_ch)
            d = F.linear(hdn, w2, b2).view(t, fh, fw, C)
            if i + 1 < self.depths:                                    # x = x + mlp(y); y = norm1 of the next block
                x, y = ops.add_layernorm(x, d, *norm(i + 1, 1), **yd)
            else:
                x = x + d                                              # fp16 d is widened exactly
        return x
