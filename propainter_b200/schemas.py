"""state_dict schemas of the three nets on the hot path (key names / shapes == reference).

RAFT:  RAFT/raft.py:48-56, RAFT/extractor.py:6-58,118-165, RAFT/update.py:6-14,33-43,79-97,114-125
RFC :  model/recurrent_flow_completion.py:9-28,46-65,148-160,172-190,203-264
GEN :  model/propainter.py:34-54,72-101,193-216,235-304; model/modules/sparse_transformer.py:7-17,
       34-47,64-72,117-153,284-292,321-329
The golden manifest ``tests/golden/state_dict_manifest.json`` (dumped from the reference modules in
the authoring container) pins these in the CPU test-suite; ``tests/golden/state_dict_manifest_raft_small.json`` pins
``raft_small_schema``.
I3D (the VFID feature network): core/metrics.py:221-256,289-531, pinned by ``tests/golden/state_dict_manifest_i3d.json``.
"""
import torch

from ._params import Schema


def raft_schema():
    S = Schema()
    for enc, bn in (("fnet", False), ("cnet", True)):
        def norm(p, c):
            if bn:
                S.batchnorm(p, c)          # InstanceNorm2d (fnet) has no parameters / buffers
        S.conv(f"{enc}.conv1", 3, 64, 7, gain=1.4)
        norm(f"{enc}.norm1", 64)
        cin = 64
        for li, dim, stride in ((1, 64, 1), (2, 96, 2), (3, 128, 2)):
            for bi in (0, 1):
                p = f"{enc}.layer{li}.{bi}"
                S.conv(p + ".conv1", cin, dim, 3, gain=1.4)
                S.conv(p + ".conv2", dim, dim, 3, gain=1.4)
                norm(p + ".norm1", dim)
                norm(p + ".norm2", dim)
                if bi == 0 and stride != 1:
                    norm(p + ".norm3", dim)
                    S.conv(p + ".downsample.0", cin, dim, 1)
                    if bn:
                        S.alias(p + ".downsample.1", p + ".norm3")   # same module object upstream
                cin = dim
        S.conv(f"{enc}.conv2", 128, 256, 1)
    u = "update_block."
    S.conv(u + "encoder.convc1", 324, 256, 1, gain=1.4)
    S.conv(u + "encoder.convc2", 256, 192, 3, gain=1.4)
    S.conv(u + "encoder.convf1", 2, 128, 7, gain=1.4)
    S.conv(u + "encoder.convf2", 128, 64, 3, gain=1.4)
    S.conv(u + "encoder.conv", 256, 126, 3, gain=1.4)
    for tag, k in (("1", (1, 5)), ("2", (5, 1))):
        for gate in "zrq":
            S.conv(f"{u}gru.conv{gate}{tag}", 384, 128, k)
    S.conv(u + "flow_head.conv1", 128, 256, 3, gain=1.4)
    S.conv(u + "flow_head.conv2", 256, 2, 3, gain=0.05)   # keeps random-init flow within a few px
    S.conv(u + "mask.0", 128, 256, 3, gain=1.4)
    S.conv(u + "mask.2", 256, 576, 1)
    return S


def raft_small_schema():
    """RAFT(args.small=True): RAFT/raft.py:29-33,48-51, SmallEncoder RAFT/extractor.py:195-267 with BottleneckBlock :60-115,
    SmallUpdateBlock RAFT/update.py:16-31,62-77,99-112.  No norm parameters: fnet's InstanceNorm2d has no affine and cnet
    uses norm_fn='none' (nn.Sequential()), so a strided block's downsample is Sequential(conv, Sequential()) -> key
    `.downsample.0` only."""
    S = Schema()
    for enc, out in (("fnet", 128), ("cnet", 160)):
        S.conv(f"{enc}.conv1", 3, 32, 7, gain=1.4)
        cin = 32
        for li, dim, stride in ((1, 32, 1), (2, 64, 2), (3, 96, 2)):
            for bi in (0, 1):
                p = f"{enc}.layer{li}.{bi}"
                S.conv(p + ".conv1", cin, dim // 4, 1, gain=1.4)
                S.conv(p + ".conv2", dim // 4, dim // 4, 3, gain=1.4)
                S.conv(p + ".conv3", dim // 4, dim, 1, gain=1.4)
                if bi == 0 and stride != 1:
                    S.conv(p + ".downsample.0", cin, dim, 1)
                cin = dim
        S.conv(f"{enc}.conv2", 96, out, 1)
    u = "update_block."
    S.conv(u + "encoder.convc1", 196, 96, 1, gain=1.4)
    S.conv(u + "encoder.convf1", 2, 64, 7, gain=1.4)
    S.conv(u + "encoder.convf2", 64, 32, 3, gain=1.4)
    S.conv(u + "encoder.conv", 128, 80, 3, gain=1.4)
    for gate in "zrq":
        S.conv(f"{u}gru.conv{gate}", 96 + 146, 96, 3)
    S.conv(u + "flow_head.conv1", 96, 128, 3, gain=1.4)
    S.conv(u + "flow_head.conv2", 128, 2, 3, gain=0.05)   # keeps random-init flow within a few px
    return S


# InceptionI3d's Inception blocks (core/metrics.py:449-517): name, input channels, (b0, b1a, b1b, b2a, b2b, b3b) outputs.
# The pooling endpoints between them carry no parameters.
I3D_INCEPTION = (
    ("Mixed_3b", 192, (64, 96, 128, 16, 32, 32)),
    ("Mixed_3c", 256, (128, 128, 192, 32, 96, 64)),
    ("Mixed_4b", 480, (192, 96, 208, 16, 48, 64)),
    ("Mixed_4c", 512, (160, 112, 224, 24, 64, 64)),
    ("Mixed_4d", 512, (128, 128, 256, 24, 64, 64)),
    ("Mixed_4e", 512, (112, 144, 288, 32, 64, 64)),
    ("Mixed_4f", 528, (256, 160, 320, 32, 128, 128)),
    ("Mixed_5b", 832, (256, 160, 320, 32, 128, 128)),
    ("Mixed_5c", 832, (384, 192, 384, 48, 128, 128)),
)


def _unit3d(S, p, cin, cout, k):
    """Unit3D (core/metrics.py:221-256): bias-free conv3d + BatchNorm3d(eps=1e-3).  Seeded init: Kaiming-normal conv weights
    (ReLU gain) so the signal survives 57 layers, and BN statistics / affine spread so that folding them is exercised."""
    S.conv(p + ".conv3d", cin, cout, k, bias=False, nd=3, gain=2 ** 0.5)
    S.add(p + ".bn.weight", (cout,), init=("uniform", 0.5, 1.5))
    S.add(p + ".bn.bias", (cout,), init=("normal", 0.1))
    S.add(p + ".bn.running_mean", (cout,), kind="buffer", init=("normal", 0.1))
    S.add(p + ".bn.running_var", (cout,), kind="buffer", init=("uniform", 0.5, 2.0))
    S.add(p + ".bn.num_batches_tracked", (), kind="buffer", dtype=torch.int64, init=("zeros",))


def i3d_schema(num_classes=400, in_channels=3):
    """InceptionI3d(final_endpoint='Logits') core/metrics.py:334-531 in its state_dict order: `logits` first (it is assigned
    in __init__ before build() registers the endpoints), then the endpoints; the unused classifier head stays so that
    pytorch-i3d checkpoints load strict."""
    S = Schema()
    S.conv("logits.conv3d", 1024, num_classes, 1, nd=3)
    _unit3d(S, "Conv3d_1a_7x7", in_channels, 64, 7)
    _unit3d(S, "Conv3d_2b_1x1", 64, 64, 1)
    _unit3d(S, "Conv3d_2c_3x3", 64, 192, 3)
    for name, cin, (c0, c1a, c1b, c2a, c2b, c3b) in I3D_INCEPTION:
        _unit3d(S, name + ".b0", cin, c0, 1)
        _unit3d(S, name + ".b1a", cin, c1a, 1)
        _unit3d(S, name + ".b1b", c1a, c1b, 3)
        _unit3d(S, name + ".b2a", cin, c2a, 1)
        _unit3d(S, name + ".b2b", c2a, c2b, 3)
        _unit3d(S, name + ".b3b", cin, c3b, 1)
    return S


def _offset_net(S, p, cond_ch, ch=128, groups=16):
    S.conv(p + ".conv_offset.0", cond_ch, ch, 3, gain=1.3)
    S.conv(p + ".conv_offset.2", ch, ch, 3, gain=1.3)
    S.conv(p + ".conv_offset.4", ch, ch, 3, gain=1.3)
    # the reference zero-initialises this layer (offsets == 0, modulation == 0.5), which never
    # exercises the deformable gather; our synthetic init keeps it live (SURVEY.md §7 "hard parts").
    S.conv(p + ".conv_offset.6", ch, 27 * groups, 3, gain=0.7)


def rfc_schema():
    S = Schema()
    S.conv("downsample.0", 3, 32, (1, 5, 5), gain=1.3)
    for enc, specs in (("encoder1", ((0, 32, 32), (2, 32, 64))), ("encoder2", ((0, 64, 64), (2, 64, 128)))):
        for i, cin, cout in specs:
            S.conv(f"{enc}.{i}.conv1.0", cin, cout, (1, 3, 3), gain=1.3)
            S.conv(f"{enc}.{i}.conv2.0", cout, cout, (3, 1, 1), gain=1.3)
    for i in (0, 2, 4):
        S.conv(f"mid_dilation.{i}", 128, 128, (1, 3, 3), gain=1.3)
    fp = "feat_prop_module."
    for i, name in enumerate(("backward_", "forward_")):
        S.conv(fp + "deform_align." + name, 256, 128, 3)
        _offset_net(S, fp + "deform_align." + name, 384)
        S.conv(fp + f"backbone.{name}.0", (2 + i) * 128, 128, 3, gain=1.3)
        S.conv(fp + f"backbone.{name}.2", 128, 128, 3, gain=0.5)
    S.conv(fp + "fusion", 256, 128, 1)
    S.conv("decoder2.0", 128, 128, 3, gain=1.3)
    S.conv("decoder2.2.conv", 128, 64, 3, gain=1.3)
    S.conv("decoder1.0", 64, 64, 3, gain=1.3)
    S.conv("decoder1.2.conv", 64, 32, 3, gain=1.3)
    S.conv("upsample.0", 32, 32, 3, gain=1.3)
    S.conv("upsample.2.conv", 32, 2, 3)
    # edge head: training-only upstream (:301-305) but part of the strict state_dict
    S.conv("edgeDetector.projection.0", 2, 16, 3)
    S.conv("edgeDetector.mid_layer_1.0", 16, 16, 3)
    S.conv("edgeDetector.mid_layer_2.0", 16, 16, 3)
    S.conv("edgeDetector.out_layer", 16, 1, 1)
    return S


def generator_schema(depths=8, hidden=512, channel=128):
    S = Schema()
    enc = ((0, 5, 64, 1), (2, 64, 64, 1), (4, 64, 128, 1), (6, 128, 256, 1), (8, 256, 384, 1),
           (10, 640, 512, 2), (12, 768, 384, 4), (14, 640, 256, 8), (16, 512, 128, 1))
    for i, cin, cout, g in enc:
        S.conv(f"encoder.layers.{i}", cin, cout, 3, groups=g, gain=1.3)
    S.conv("decoder.0.conv", channel, 128, 3, gain=1.3)
    S.conv("decoder.2", 128, 64, 3, gain=1.3)
    S.conv("decoder.4.conv", 64, 64, 3, gain=1.3)
    S.conv("decoder.6", 64, 3, 3, gain=0.7)
    S.linear("ss.embedding", 49 * channel, hidden)
    S.linear("sc.embedding", hidden, 49 * channel, gain=1.0)
    S.conv("sc.bias_conv", channel, channel, 3, gain=0.6)
    fp = "feat_prop_module."
    for name in ("backward_1", "forward_1"):
        S.conv(fp + "deform_align." + name, channel, channel, 3)
        _offset_net(S, fp + "deform_align." + name, 2 * channel + 5)
    for name in ("backward_1", "forward_1"):
        S.conv(fp + f"backbone.{name}.0", 2 * channel + 2, channel, 3, gain=1.3)
        S.conv(fp + f"backbone.{name}.2", channel, channel, 3, gain=0.5)
    S.conv(fp + "fuse.0", 2 * channel + 2, channel, 3, gain=1.3)
    S.conv(fp + "fuse.2", channel, channel, 3, gain=0.5)
    from .window_index import rolled_valid_index
    for i in range(depths):
        p = f"transformers.transformer.{i}."
        S.add(p + "attention.valid_ind_rolled", (148,), kind="buffer", dtype=torch.int64,
              init=("const", rolled_valid_index((5, 9))))
        for n in ("key", "query", "value", "proj"):
            S.linear(p + "attention." + n, hidden, hidden, gain=1.0 if n != "proj" else 0.5)
        S.add(p + "attention.pool_layer.weight", (hidden, 1, 4, 4), init=("normal_mean", 1.0 / 16, 0.02))
        S.add(p + "attention.pool_layer.bias", (hidden,), init=("normal", 0.02))
        S.affine(p + "norm1", hidden)
        S.affine(p + "norm2", hidden)
        S.linear(p + "mlp.fc1.0", hidden, 1960)
        S.linear(p + "mlp.fc2.1", 1960, hidden, gain=0.5)
    return S


# ---------------------------------------------------------------------------------------------------------------- Cutie
# The web demo's mask tracker (web-demos/hugging_face/tracker/model/cutie.py:18-45 at tracker/config CONFIG), pinned by
# tests/golden/state_dict_manifest_cutie.json: resnet.py:38-121 (the two ResNets, through layer3), big_modules.py,
# modules.py, group_modules.py, channel_attn.py, transformer/*.py and aux_modules.py (the aux head is kept so that
# cutie-base-mega.pth loads strict; inference does not use it).
def _bn(S, p, c, lo=0.4, hi=0.9):
    S.add(p + ".weight", (c,), init=("uniform", lo, hi))
    S.add(p + ".bias", (c,), init=("normal", 0.1))
    S.add(p + ".running_mean", (c,), kind="buffer", init=("normal", 0.1))
    S.add(p + ".running_var", (c,), kind="buffer", init=("uniform", 0.5, 2.0))
    S.add(p + ".num_batches_tracked", (), kind="buffer", dtype=torch.int64, init=("zeros",))


def _resnet(S, p, cin, bottleneck, blocks, layer_names):
    """ResNet.__init__ / _make_layer (resnet.py:86-121) for layer1..layer3: bias-free convs (Kaiming-normal), BatchNorm2d"""
    S.conv(p + ".conv1", cin, 64, 7, bias=False, gain=2 ** 0.5)
    _bn(S, p + ".bn1", 64)
    inplanes = 64
    for name, planes, n, stride in zip(layer_names, (64, 128, 256), blocks, (1, 2, 2)):
        out = planes * (4 if bottleneck else 1)
        for b in range(n):
            q = f"{p}.{name}.{b}"
            if bottleneck:
                S.conv(q + ".conv1", inplanes, planes, 1, bias=False, gain=2 ** 0.5)
                _bn(S, q + ".bn1", planes)
                S.conv(q + ".conv2", planes, planes, 3, bias=False, gain=2 ** 0.5)
                _bn(S, q + ".bn2", planes)
                S.conv(q + ".conv3", planes, out, 1, bias=False, gain=2 ** 0.5)
                _bn(S, q + ".bn3", out, 0.2, 0.5)
            else:
                S.conv(q + ".conv1", inplanes, planes, 3, bias=False, gain=2 ** 0.5)
                _bn(S, q + ".bn1", planes)
                S.conv(q + ".conv2", planes, planes, 3, bias=False, gain=2 ** 0.5)
                _bn(S, q + ".bn2", planes, 0.2, 0.5)
            if b == 0 and (stride != 1 or inplanes != out):
                S.conv(q + ".downsample.0", inplanes, out, 1, bias=False, gain=2 ** 0.5)
                _bn(S, q + ".downsample.1", out, 0.2, 0.5)
            inplanes = out


def _ca_block(S, p, dim):
    """CAResBlock (channel_attn.py:7-25) with in_dim == out_dim: two 3x3 convs + the ECA conv1d (k = 5 at 256 channels)"""
    S.conv(p + ".conv1", dim, dim, 3)
    S.conv(p + ".conv2", dim, dim, 3)
    S.add(p + ".conv.weight", (1, 1, 5), init=("normal", 5 ** -0.5))


def _fusion(S, p, x_dim, g_dim, out_dim):
    """GroupFeatureFusionBlock (group_modules.py:107-118)"""
    S.conv(p + ".distributor.x_transform", x_dim, out_dim, 1)
    S.conv(p + ".distributor.g_transform", g_dim, out_dim, 1)
    _ca_block(S, p + ".block1", out_dim)
    _ca_block(S, p + ".block2", out_dim)


def _mha(S, p, dim):
    """nn.MultiheadAttention(dim, heads, batch_first=True): packed in-projection + out_proj"""
    S.add(p + ".in_proj_weight", (3 * dim, dim), init=("normal", dim ** -0.5))
    S.add(p + ".in_proj_bias", (3 * dim,), init=("normal", 0.02))
    S.linear(p + ".out_proj", dim, dim)


def cutie_pe_inv_freq(dim=256, temperature=128):
    """PositionalEncoding.inv_freq (transformer/positional_encoding.py:21-23), a persistent buffer of the state_dict"""
    d = int(-(-dim // 4) * 2)
    return (1.0 / (temperature ** (torch.arange(0, d, 2).float() / d))).tolist()


CUTIE_DIMS = dict(pixel_dim=256, key_dim=64, value_dim=256, sensory_dim=256, embed_dim=256, ms_dims=(1024, 512, 256),
                  num_queries=16, num_heads=8, num_blocks=3, ff_dim=2048, up_dims=(256, 128, 128))


def cutie_schema():
    """CUTIE(cfg) (tracker/model/cutie.py:18-45) at tracker/config CONFIG, multi-object, in its state_dict order"""
    d = CUTIE_DIMS
    E, V, SD, K = d["embed_dim"], d["value_dim"], d["sensory_dim"], d["key_dim"]
    S = Schema()
    _resnet(S, "pixel_encoder", 3, True, (3, 4, 6), ("res2", "layer2", "layer3"))
    S.conv("pix_feat_proj", 1024, d["pixel_dim"], 1)
    S.conv("key_proj.pix_feat_proj", 1024, d["pixel_dim"], 1)
    S.conv("key_proj.key_proj", d["pixel_dim"], K, 3)
    S.conv("key_proj.d_proj", d["pixel_dim"], 1, 3)
    S.conv("key_proj.e_proj", d["pixel_dim"], K, 3)
    _resnet(S, "mask_encoder", 5, False, (2, 2, 2), ("layer1", "layer2", "layer3"))
    _fusion(S, "mask_encoder.fuser", d["pixel_dim"], 256, V)
    S.conv("mask_encoder.sensory_update.transform", V + SD, SD * 3, 3)
    u0, u1, u2 = d["up_dims"]
    S.conv("mask_decoder.sensory_update.g16_conv", u0, SD, 1)
    S.conv("mask_decoder.sensory_update.g8_conv", u1, SD, 1)
    S.conv("mask_decoder.sensory_update.g4_conv", u2 + 1, SD, 1)
    S.conv("mask_decoder.sensory_update.transform", SD + SD, SD * 3, 3)
    S.conv("mask_decoder.decoder_feat_proc.transforms.0", d["ms_dims"][1], u0, 1)
    S.conv("mask_decoder.decoder_feat_proc.transforms.1", d["ms_dims"][2], u1, 1)
    S.conv("mask_decoder.up_16_8.out_conv.downsample", u0, u1, 1)
    S.conv("mask_decoder.up_16_8.out_conv.conv1", u0, u1, 3)
    S.conv("mask_decoder.up_16_8.out_conv.conv2", u1, u1, 3)
    S.conv("mask_decoder.up_8_4.out_conv.conv1", u1, u2, 3)
    S.conv("mask_decoder.up_8_4.out_conv.conv2", u2, u2, 3)
    S.conv("mask_decoder.pred", u2, 1, 3)
    _fusion(S, "pixel_fuser.fuser", d["pixel_dim"], V, E)
    S.conv("pixel_fuser.sensory_compress", SD + 2, V, 1)
    t = "object_transformer"
    Q = d["num_queries"]
    S.add(t + ".query_init.weight", (Q, E), init=("normal", 1.0))
    S.add(t + ".query_emb.weight", (Q, E), init=("normal", 1.0))
    S.linear(t + ".summary_to_query_init", E, E)
    S.linear(t + ".summary_to_query_emb", E, E)
    S.conv(t + ".pixel_init_proj", E, E, 1)
    S.conv(t + ".pixel_emb_proj", E, E, 1)
    S.add(t + ".spatial_pe.inv_freq", (E // 4,), kind="buffer", init=("const", cutie_pe_inv_freq(E)))
    for b in range(d["num_blocks"]):
        q = f"{t}.blocks.{b}"
        _mha(S, q + ".read_from_pixel.cross_attn", E)
        S.affine(q + ".read_from_pixel.norm", E)
        _mha(S, q + ".self_attn.self_attn", E)
        S.affine(q + ".self_attn.norm", E)
        S.linear(q + ".ffn.linear1", E, d["ff_dim"])
        S.linear(q + ".ffn.linear2", d["ff_dim"], E)
        S.affine(q + ".ffn.norm", E)
        _mha(S, q + ".read_from_query.cross_attn", E)
        _ca_block(S, q + ".pixel_ffn.conv", E)
    for i in range(d["num_blocks"] + 1):
        S.conv(f"{t}.mask_pred.{i}.1", E, 1, 1)
    s = "object_summarizer"
    S.add(s + ".pos_enc.inv_freq", (E // 4,), kind="buffer", init=("const", cutie_pe_inv_freq(E)))
    S.linear(s + ".input_proj", V, E)
    S.linear(s + ".feature_pred.0", E, E)
    S.linear(s + ".feature_pred.2", E, E)
    S.linear(s + ".weights_pred.0", E, E)
    S.linear(s + ".weights_pred.2", E, Q)
    S.conv("aux_computer.sensory_aux.projection", SD, E + 1, 1)
    return S
