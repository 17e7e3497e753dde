"""Cutie, the web demo's video object segmentation network (web-demos/hugging_face/tracker/model/cutie.py), on the H100 path.

Drop-in for the reference's ``CUTIE`` at tracker/config CONFIG (multi-object): same state_dict (``cutie-base-mega.pth``
loads through ``load_weights`` with the same single-object conversion and non-strict semantics), and the inference
methods ``MemoryManager`` / ``InferenceCore`` call: ``encode_image``, ``transform_key``, ``encode_mask``,
``pixel_fusion``, ``readout_query`` and ``segment``.  Training losses, ``read_memory`` and ``compute_aux`` are not
provided (the aux head's weights stay in the state_dict so checkpoints load).

Every convolution is a cuDNN call with eval BatchNorm folded into its weights once per device; the grouped ``GConv2d``
over objects is the same conv over objects flattened into the batch.  The memory read itself is
``ops.cutie_topk_readout`` (propainter_b200/tracker.py), and the frame / label ends are ``ops.cutie_frame_in`` /
``ops.cutie_labels``.
"""
import logging
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from .._params import ParamNet
from ..schemas import CUTIE_DIMS, cutie_schema

log = logging.getLogger(__name__)

PIXEL_MEAN = (0.485, 0.456, 0.406)
PIXEL_STD = (0.229, 0.224, 0.225)
_BN_EPS = 1e-5
_PE_SCALE = 32                                           # model.pixel_pe_scale


def aggregate(prob, dim):
    """tracker/utils/tensor_utils.py:46-53: soft aggregation of per-object probabilities into logits with a background"""
    prob = prob.float()
    new_prob = torch.cat([torch.prod(1 - prob, dim=dim, keepdim=True), prob], dim).clamp(1e-7, 1 - 1e-7)
    return torch.log(new_prob / (1 - new_prob))


def _others(masks):
    """CUTIE._get_others (cutie.py:47-57): per object, the clamped sum of every other object's mask"""
    if masks.shape[1] >= 1:
        return (masks.sum(dim=1, keepdim=True) - masks).clamp(0, 1)
    return torch.zeros_like(masks)


def _recurrent_update(h, values):
    """modules.py:35-43"""
    dim = values.shape[2] // 3
    forget_gate = torch.sigmoid(values[:, :, :dim])
    update_gate = torch.sigmoid(values[:, :, dim:dim * 2])
    new_value = torch.tanh(values[:, :, dim * 2:])
    return forget_gate * h * (1 - update_gate) + update_gate * new_value


def _groups(fn, g):
    """apply an [n,C,H,W] function to a grouped tensor [B,objects,C,H,W] (GConv2d, group_modules.py:33-37)"""
    B, K = g.shape[:2]
    y = fn(g.flatten(0, 1))
    return y.view(B, K, *y.shape[1:])


def positional_encoding(h, w, inv_freq):
    """PositionalEncoding.forward (transformer/positional_encoding.py:33-90), normalize=True, as an [h, w, 4 * len(inv_freq)]
    table; inv_freq is the module's state_dict buffer"""
    d, device = 2 * inv_freq.numel(), inv_freq.device
    pos_y = torch.arange(h, device=device, dtype=torch.float32)
    pos_x = torch.arange(w, device=device, dtype=torch.float32)
    pos_y = pos_y / (pos_y[-1] + 1e-6) * _PE_SCALE
    pos_x = pos_x / (pos_x[-1] + 1e-6) * _PE_SCALE

    def emb(sin_inp):
        return torch.stack((sin_inp.sin(), sin_inp.cos()), dim=-1).flatten(-2, -1)

    out = torch.zeros((h, w, d * 2), device=device, dtype=torch.float32)
    out[:, :, :d] = emb(torch.einsum("i,j->ij", pos_x, inv_freq))
    out[:, :, d:] = emb(torch.einsum("i,j->ij", pos_y, inv_freq)).unsqueeze(1)
    return out


class CUTIE(ParamNet):
    def __init__(self, cfg=None, *, single_object=False, seed=None):
        if single_object:
            raise ValueError("CUTIE(single_object=True) is not supported: the web demo builds the multi-object network")
        super().__init__(cutie_schema(), seed=seed)
        d = CUTIE_DIMS
        self.ms_dims = list(d["ms_dims"])
        self.key_dim, self.value_dim, self.sensory_dim = d["key_dim"], d["value_dim"], d["sensory_dim"]
        self.pixel_dim, self.embed_dim = d["pixel_dim"], d["embed_dim"]
        self.num_queries, self.num_heads, self.num_blocks = d["num_queries"], d["num_heads"], d["num_blocks"]
        self.single_object = False

    # ------------------------------------------------------------------ weights
    def load_weights(self, src_dict, init_as_zero_if_needed=False):
        """CUTIE.load_weights (cutie.py:202-247): single-object checkpoints gain the extra input channel of
        mask_encoder.conv1 / pixel_fuser.sensory_compress (orthogonal or zero init), then a non-strict load."""
        src_dict = dict(src_dict)
        for k in list(src_dict.keys()):
            if k == "mask_encoder.conv1.weight" and src_dict[k].shape[1] == 4:
                pads = torch.zeros((64, 1, 7, 7), device=src_dict[k].device)
                if not init_as_zero_if_needed:
                    nn.init.orthogonal_(pads)
                src_dict[k] = torch.cat([src_dict[k], pads], 1)
            elif k == "pixel_fuser.sensory_compress.weight" and src_dict[k].shape[1] == self.sensory_dim + 1:
                pads = torch.zeros((self.value_dim, 1, 1, 1), device=src_dict[k].device)
                if not init_as_zero_if_needed:
                    nn.init.orthogonal_(pads)
                src_dict[k] = torch.cat([src_dict[k], pads], 1)
        own = self.state_dict()
        for k in src_dict:
            if k not in own:
                log.info(f"Key {k} found in src_dict but not in self.state_dict()!!!")
        for k in own:
            if k not in src_dict:
                log.info(f"Key {k} found in self.state_dict() but not in src_dict!!!")
        self.load_state_dict(src_dict, strict=False)

    def _bnconv(self, conv, bn):
        """bias-free conv `conv` with eval BatchNorm `bn` folded in: (weight * scale, shift)"""
        def build():
            P = self.P
            s = P[bn + ".weight"] / torch.sqrt(P[bn + ".running_var"] + _BN_EPS)
            return (P[conv + ".weight"] * s.view(-1, 1, 1, 1)).contiguous(), (P[bn + ".bias"] - P[bn + ".running_mean"] * s)
        return self.packed("bn:" + conv, build)

    def _conv(self, x, key, stride=1, padding=0):
        P = self.P
        return F.conv2d(x, P[key + ".weight"], P.get(key + ".bias"), stride=stride, padding=padding)

    def _cbr(self, x, conv, bn, stride=1, padding=0, relu=True):
        w, b = self._bnconv(conv, bn)
        y = F.conv2d(x, w, b, stride=stride, padding=padding)
        return F.relu_(y) if relu else y

    def _linear(self, x, key):
        P = self.P
        return F.linear(x, P[key + ".weight"], P[key + ".bias"])

    # ------------------------------------------------------------------ backbones (resnet.py)
    def _bottleneck(self, x, p, stride):
        out = self._cbr(x, p + ".conv1", p + ".bn1")
        out = self._cbr(out, p + ".conv2", p + ".bn2", stride=stride, padding=1)
        out = self._cbr(out, p + ".conv3", p + ".bn3", relu=False)
        res = self._cbr(x, p + ".downsample.0", p + ".downsample.1", stride=stride, relu=False) \
            if p + ".downsample.0.weight" in self.P else x
        return F.relu_(out + res)

    def _basic(self, x, p, stride):
        out = self._cbr(x, p + ".conv1", p + ".bn1", stride=stride, padding=1)
        out = self._cbr(out, p + ".conv2", p + ".bn2", padding=1, relu=False)
        res = self._cbr(x, p + ".downsample.0", p + ".downsample.1", stride=stride, relu=False) \
            if p + ".downsample.0.weight" in self.P else x
        return F.relu_(out + res)

    def _layer(self, x, p, n, stride, block):
        for b in range(n):
            x = block(x, f"{p}.{b}", stride if b == 0 else 1)
        return x

    def _pixel_encoder(self, x):
        """PixelEncoder.forward (big_modules.py:43-52): ResNet-50 through layer3 -> (f16, f8, f4)"""
        p = "pixel_encoder"
        x = self._cbr(x, p + ".conv1", p + ".bn1", stride=2, padding=3)
        x = F.max_pool2d(x, 3, 2, 1)
        f4 = self._layer(x, p + ".res2", 3, 1, self._bottleneck)
        f8 = self._layer(f4, p + ".layer2", 4, 2, self._bottleneck)
        f16 = self._layer(f8, p + ".layer3", 6, 2, self._bottleneck)
        return f16, f8, f4

    # ------------------------------------------------------------------ shared blocks
    def _ca_block(self, x, p):
        """CAResBlock.forward (channel_attn.py:27-39), in_dim == out_dim"""
        r = x
        x = self._conv(F.relu(x), p + ".conv1", padding=1)
        x = self._conv(F.relu_(x), p + ".conv2", padding=1)
        b, c = x.shape[:2]
        w = x.mean(dim=(2, 3)).view(b, 1, c)
        w = F.conv1d(w, self.P[p + ".conv.weight"], padding=2).transpose(-1, -2).unsqueeze(-1).sigmoid()
        return x * w + r

    def _fusion(self, x, g, p):
        """GroupFeatureFusionBlock.forward (group_modules.py:120-131)"""
        B, K = g.shape[:2]
        g = self._conv(x, p + ".distributor.x_transform").unsqueeze(1) + \
            _groups(lambda t: self._conv(t, p + ".distributor.g_transform"), g)
        g = g.flatten(0, 1)
        g = self._ca_block(g, p + ".block1")
        g = self._ca_block(g, p + ".block2")
        return g.view(B, K, *g.shape[1:])

    def _gru(self, g, h, key):
        """SensoryDeepUpdater / the transform of SensoryUpdater (modules.py:63-85): GConv 3x3 + recurrent update"""
        values = _groups(lambda t: self._conv(t, key, padding=1), torch.cat([g.float(), h.float()], dim=2))
        return _recurrent_update(h.float(), values)

    # ------------------------------------------------------------------ CUTIE inference methods (cutie.py)
    def normalize(self, image):
        mean = torch.tensor(PIXEL_MEAN, device=image.device).view(-1, 1, 1)
        std = torch.tensor(PIXEL_STD, device=image.device).view(-1, 1, 1)
        return (image - mean) / std

    @torch.no_grad()
    def encode_image(self, image):
        """image [B,3,H,W] in [0, 1] -> ((f16, f8, f4), pix_feat)"""
        return self.encode_normalized(self.normalize(image))

    @torch.no_grad()
    def encode_normalized(self, x):
        """encode_image on an already normalised image (ops.cutie_frame_in's output)"""
        ms = self._pixel_encoder(x)
        return ms, self._conv(ms[0], "pix_feat_proj")

    @torch.no_grad()
    def transform_key(self, final_pix_feat, *, need_sk=True, need_ek=True):
        """KeyProjection.forward (big_modules.py:76-82) -> (key, shrinkage, selection)"""
        x = self._conv(final_pix_feat, "key_proj.pix_feat_proj")
        shrinkage = self._conv(x, "key_proj.d_proj", padding=1) ** 2 + 1 if need_sk else None
        selection = torch.sigmoid(self._conv(x, "key_proj.e_proj", padding=1)) if need_ek else None
        return self._conv(x, "key_proj.key_proj", padding=1), shrinkage, selection

    @torch.no_grad()
    def encode_mask(self, image, ms_features, sensory, masks, *, deep_update=True, chunk_size=-1, need_weights=False):
        """CUTIE.encode_mask (cutie.py:64-87) with image in [0, 1]"""
        return self.encode_mask_normalized(self.normalize(image), ms_features, sensory, masks, deep_update=deep_update,
                                           need_weights=need_weights)

    @torch.no_grad()
    def encode_mask_normalized(self, x, pix_feat, sensory, masks, *, deep_update=True, need_weights=False):
        """MaskEncoder.forward (big_modules.py:122-177, one chunk) + ObjectSummarizer on a normalised image x"""
        others = _others(masks)
        g = torch.stack([masks, others], dim=2)
        B, K = g.shape[:2]
        g = torch.cat([x.unsqueeze(1).expand(-1, K, -1, -1, -1), g], 2).flatten(0, 1)
        p = "mask_encoder"
        w, b = self._bnconv(p + ".conv1", p + ".bn1")
        g = F.conv2d(g, w, b, stride=2, padding=3)
        g = F.relu_(F.max_pool2d(g, 3, 2, 1))
        g = self._layer(g, p + ".layer1", 2, 1, self._basic)
        g = self._layer(g, p + ".layer2", 2, 2, self._basic)
        g = self._layer(g, p + ".layer3", 2, 2, self._basic)
        g = g.view(B, K, *g.shape[1:])
        g = self._fusion(pix_feat, g, p + ".fuser")
        new_sensory = self._gru(g, sensory, p + ".sensory_update.transform") if deep_update else sensory
        summaries, logits = self._summarize(masks, g, need_weights)
        return g, new_sensory, summaries, logits

    def _summarize(self, masks, value, need_weights=False):
        """ObjectSummarizer.forward (transformer/object_summarizer.py:46-88)"""
        h, w = value.shape[-2:]
        masks = F.interpolate(masks, size=(h, w), mode="area").unsqueeze(-1)
        half = self.num_queries // 2
        repeated = torch.cat([masks.expand(-1, -1, -1, -1, half), (1 - masks).expand(-1, -1, -1, -1, half)], dim=-1)
        p = "object_summarizer"
        value = self._linear(value.permute(0, 1, 3, 4, 2), p + ".input_proj")
        value = value + positional_encoding(h, w, self.P[p + ".pos_enc.inv_freq"])
        feature = self._linear(F.relu(self._linear(value, p + ".feature_pred.0")), p + ".feature_pred.2")
        logits = self._linear(F.relu(self._linear(value, p + ".weights_pred.0")), p + ".weights_pred.2")
        weights = logits.sigmoid() * repeated
        sums = torch.einsum("bkhwq,bkhwc->bkqc", weights, feature)
        area = weights.flatten(start_dim=2, end_dim=3).sum(2).unsqueeze(-1)
        return torch.cat([sums, area], dim=-1), (logits if need_weights else None)

    @torch.no_grad()
    def pixel_fusion(self, pix_feat, pixel, sensory, last_mask, *, chunk_size=-1):
        """CUTIE.pixel_fusion + PixelFeatureFuser.forward (cutie.py:134-151, big_modules.py:206-235, one chunk)"""
        last_mask = F.interpolate(last_mask, size=sensory.shape[-2:], mode="area")
        last_mask = torch.stack([last_mask, _others(last_mask)], dim=2)
        sensory_readout = _groups(lambda t: self._conv(t, "pixel_fuser.sensory_compress"), torch.cat([sensory, last_mask], 2))
        return self._fusion(pix_feat, pixel + sensory_readout, "pixel_fuser.fuser")

    # ------------------------------------------------------------------ object transformer (transformer/object_transformer.py)
    def _mha(self, q, k, v, p, attn_mask=None):
        """nn.MultiheadAttention(batch_first=True) forward, eval, boolean attn_mask (True = blocked) per (batch*head)"""
        P = self.P
        E, nh = self.embed_dim, self.num_heads
        w, b = P[p + ".in_proj_weight"], P[p + ".in_proj_bias"]
        q = F.linear(q, w[:E], b[:E])
        k = F.linear(k, w[E:2 * E], b[E:2 * E])
        v = F.linear(v, w[2 * E:], b[2 * E:])
        n, L, S = q.shape[0], q.shape[1], k.shape[1]
        q = q.view(n, L, nh, E // nh).transpose(1, 2)
        k = k.view(n, S, nh, E // nh).transpose(1, 2)
        v = v.view(n, S, nh, E // nh).transpose(1, 2)
        a = (q * (1.0 / math.sqrt(E // nh))) @ k.transpose(-2, -1)
        if attn_mask is not None:
            a = a.masked_fill(attn_mask.view(n, nh, L, S), float("-inf"))
        o = (a.softmax(-1) @ v).transpose(1, 2).reshape(n, L, E)
        return F.linear(o, P[p + ".out_proj.weight"], P[p + ".out_proj.bias"])

    def _ln(self, x, p):
        return F.layer_norm(x, (self.embed_dim,), self.P[p + ".weight"], self.P[p + ".bias"])

    def _aux_mask(self, logits):
        """QueryTransformer._get_aux_mask (object_transformer.py:159-185), selector None"""
        logits = aggregate(logits.sigmoid(), dim=1)
        fg = (logits[:, 1:] >= logits.max(dim=1, keepdim=True)[0]).flatten(start_dim=2)
        half = self.num_queries // 2
        a = (~fg).unsqueeze(2).unsqueeze(2).repeat(1, 1, self.num_heads, half, 1).flatten(start_dim=0, end_dim=2)
        b = fg.unsqueeze(2).unsqueeze(2).repeat(1, 1, self.num_heads, half, 1).flatten(start_dim=0, end_dim=2)
        m = torch.cat([a, b], dim=1)
        m[torch.where(m.sum(-1) == m.shape[-1])] = False
        return m

    def _mask_pred(self, pixel, i):
        return _groups(lambda t: self._conv(F.relu(t), f"object_transformer.mask_pred.{i}.1"), pixel).squeeze(2)

    @torch.no_grad()
    def readout_query(self, pixel_readout, obj_memory, *, selector=None, need_weights=False):
        """QueryTransformer.forward (object_transformer.py:94-157) at inference: returns (pixel, {})"""
        if selector is not None or need_weights:
            raise ValueError("readout_query: selector / need_weights are training-time options")
        t = "object_transformer"
        T = obj_memory.shape[2]
        bs, K, _, H, W = pixel_readout.shape
        E = self.embed_dim
        obj = obj_memory.view(bs * K, T, self.num_queries, E + 1)
        obj_values = obj[:, :, :, :-1].sum(dim=1) / (obj[:, :, :, -1:].sum(dim=1) + 1e-4)
        query = self.P[t + ".query_init.weight"].unsqueeze(0) + self._linear(obj_values, t + ".summary_to_query_init")
        query_emb = self.P[t + ".query_emb.weight"].unsqueeze(0) + self._linear(obj_values, t + ".summary_to_query_emb")
        pixel = _groups(lambda x: self._conv(x, t + ".pixel_init_proj"), pixel_readout)
        pixel_emb = _groups(lambda x: self._conv(x, t + ".pixel_emb_proj"), pixel_readout)
        pixel_emb = pixel_emb.flatten(3, 4).flatten(0, 1).transpose(1, 2)
        pixel_pe = positional_encoding(H, W, self.P[t + ".spatial_pe.inv_freq"]).flatten(0, 1).unsqueeze(0) + pixel_emb
        attn_mask = self._aux_mask(self._mask_pred(pixel, 0))
        for i in range(self.num_blocks):
            p = f"{t}.blocks.{i}"
            pixel_flat = pixel.flatten(3, 4).flatten(0, 1).transpose(1, 2).contiguous()
            x = self._ln(query, p + ".read_from_pixel.norm")                    # CrossAttention, norm=True
            query = x + self._mha(x + query_emb, pixel_flat + pixel_pe, pixel_flat, p + ".read_from_pixel.cross_attn", attn_mask)
            x = self._ln(query, p + ".self_attn.norm")                          # SelfAttention
            query = x + self._mha(x + query_emb, x + query_emb, x, p + ".self_attn.self_attn")
            x = self._ln(query, p + ".ffn.norm")                                # FFN
            query = query + self._linear(F.relu(self._linear(x, p + ".ffn.linear1")), p + ".ffn.linear2")
            pixel_flat = pixel_flat + self._mha(pixel_flat + pixel_pe, query + query_emb, query,
                                                p + ".read_from_query.cross_attn")   # output_norm=False
            pf = pixel_flat.view(bs * K, H, W, E).permute(0, 3, 1, 2).contiguous()
            pixel = self._ca_block(pf, p + ".pixel_ffn.conv").view(bs, K, E, H, W)
            if i < self.num_blocks - 1:                                         # the last block's mask is never read
                attn_mask = self._aux_mask(self._mask_pred(pixel, i + 1))
        return pixel, {}

    # ------------------------------------------------------------------ decoder (big_modules.py:238-304, modules.py)
    def _group_res(self, g, p):
        """GroupResBlock.forward (group_modules.py:55-62)"""
        out = _groups(lambda t: self._conv(F.relu(t), p + ".conv1", padding=1), g)
        out = _groups(lambda t: self._conv(F.relu(t), p + ".conv2", padding=1), out)
        if p + ".downsample.weight" in self.P:
            g = _groups(lambda t: self._conv(t, p + ".downsample"), g)
        return out + g

    def _up(self, g, skip, p):
        """MaskUpsampleBlock.forward (modules.py:16-20)"""
        g = _groups(lambda t: F.interpolate(t, scale_factor=2, mode="bilinear", align_corners=False), g)
        return self._group_res(skip.unsqueeze(1) + g, p + ".out_conv")

    @torch.no_grad()
    def segment(self, ms_image_feat, memory_readout, sensory, *, selector=None, chunk_size=-1, update_sensory=True):
        """CUTIE.segment (cutie.py:165-196) + MaskDecoder.forward (one chunk) -> (sensory, logits, prob)"""
        d = "mask_decoder"
        bs, K = memory_readout.shape[:2]
        f8 = self._conv(ms_image_feat[1], d + ".decoder_feat_proc.transforms.0")
        f4 = self._conv(ms_image_feat[2], d + ".decoder_feat_proc.transforms.1")
        p16 = memory_readout
        p8 = self._up(p16, f8, d + ".up_16_8")
        p4 = self._up(p8, f4, d + ".up_8_4")
        logits = self._conv(F.relu(p4.flatten(start_dim=0, end_dim=1).float()), d + ".pred", padding=1)
        new_sensory = sensory
        if update_sensory:
            p4 = torch.cat([p4, logits.view(bs, K, 1, *logits.shape[-2:])], 2)
            u = d + ".sensory_update"
            g = _groups(lambda t: self._conv(t, u + ".g16_conv"), p16) + \
                _groups(lambda t: self._conv(F.interpolate(t, scale_factor=1 / 2, mode="area"), u + ".g8_conv"), p8) + \
                _groups(lambda t: self._conv(F.interpolate(t, scale_factor=1 / 4, mode="area"), u + ".g4_conv"), p4)
            new_sensory = self._gru(g, sensory, u + ".transform")
        logits = logits.view(bs, K, *logits.shape[-2:])
        prob = torch.sigmoid(logits)
        if selector is not None:
            prob = prob * selector
        logits = F.interpolate(aggregate(prob, dim=1), scale_factor=4, mode="bilinear", align_corners=False)
        return new_sensory, logits, F.softmax(logits, dim=1)

    def forward(self, *args, **kwargs):
        raise NotImplementedError
