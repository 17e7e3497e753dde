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
