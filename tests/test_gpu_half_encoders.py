"""The clip encoders on fp16 operands (config.HALF_OPERANDS where cuDNN may use TF32): the generator's frame encoder
(InpaintGenerator._encoder_half) and RAFT's context encoder (RAFT._encode("cnet")), against the float64 oracle on a
slice of the C2 clip shape (240 x 432 frames), next to the TF32 path's error; the grouped layers' slot placement against
torch.cat; the largest fp16 value the encoders store; RAFT's feature encoder left on TF32; and bit identity of a
strict-fp32 run with the switch on and off."""
import contextlib
import types

import pytest
import torch
import torch.nn.functional as F

from oracle import generator_ref, raft_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
H, W = 240, 432


@contextlib.contextmanager
def _switches(half, tf32=True):
    from propainter_b200 import config
    prev = config.HALF_OPERANDS, torch.backends.cudnn.allow_tf32
    config.HALF_OPERANDS, torch.backends.cudnn.allow_tf32 = half, tf32
    try:
        yield
    finally:
        config.HALF_OPERANDS, torch.backends.cudnn.allow_tf32 = prev


def _sd64(net):
    return {k: v.detach().to(DEV, torch.float64) for k, v in net.state_dict().items()}


def _gen_inputs(n=3, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    fr = torch.rand(n, 3, H, W, generator=g) * 2 - 1
    mi = (torch.rand(n, 1, H // 8, W // 8, generator=g) > 0.7).float()
    mi = F.interpolate(mi, size=(H, W), mode="nearest")
    mu = (torch.rand(n, 1, H // 8, W // 8, generator=g) > 0.8).float()
    mu = F.interpolate(mu, size=(H, W), mode="nearest")
    return fr.to(DEV), mi.to(DEV), mu.to(DEV)


def _rel_rms(got, ref):
    return ((got.double() - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item()


def _generator():
    import __graft_entry__ as ge
    ge.build()
    from propainter_b200.model.propainter import InpaintGenerator
    return InpaintGenerator(seed=3).to(DEV)


def _raft():
    import __graft_entry__ as ge
    ge.build()
    from propainter_b200.RAFT.raft import RAFT
    return RAFT(types.SimpleNamespace(small=False, mixed_precision=False, alternate_corr=False), seed=1).to(DEV)


@contextlib.contextmanager
def _record_f16_max(store):
    """the largest |value| of every fp16 map pp_bias_act writes while the block runs"""
    from propainter_b200 import ops
    orig = ops.bias_act

    def rec(*a, **k):
        out = orig(*a, **k)
        if out.dtype == torch.float16:
            store.append(out.detach().abs().max().item())
        return out
    ops.bias_act = rec
    try:
        yield
    finally:
        ops.bias_act = orig


def test_generator_encoder_fp16_against_oracle():
    net = _generator()
    fr, mi, mu = _gen_inputs()
    ref = generator_ref.encoder(_sd64(net), torch.cat([fr, mi, mu], 1).double())
    err, peaks = {}, []
    with torch.no_grad():
        for half in (False, True):
            with _switches(half), (_record_f16_max(peaks) if half else contextlib.nullcontext()):
                out = net._encode_frames(fr, mi, mu)
            assert out.dtype == torch.float32 and out.shape == ref.shape
            assert out.is_contiguous(memory_format=torch.channels_last)
            err[half] = _rel_rms(out, ref)
    print(f"generator encoder rel. RMS error: TF32 {err[False]:.3e}, fp16 {err[True]:.3e}; largest fp16 value {max(peaks):.1f}")
    assert err[True] <= 1.5 * err[False] and err[True] < 5e-3
    assert len(peaks) > 0 and all(v == v for v in peaks) and max(peaks) < 6e4


def test_raft_context_encoder_fp16_against_oracle():
    net = _raft()
    fr = _gen_inputs(seed=1)[0]
    ref = raft_ref.encoder(_sd64(net), "cnet", fr.double(), "batch")
    err, peaks = {}, []
    x = fr.contiguous(memory_format=torch.channels_last)
    with torch.no_grad():
        for half in (False, True):
            with _switches(half), (_record_f16_max(peaks) if half else contextlib.nullcontext()):
                out = net._encode("cnet", x)
            assert out.dtype == torch.float32 and out.shape == ref.shape
            err[half] = _rel_rms(out, ref)
    print(f"RAFT cnet rel. RMS error: TF32 {err[False]:.3e}, fp16 {err[True]:.3e}; largest fp16 value {max(peaks):.1f}")
    assert err[True] <= 1.5 * err[False] and err[True] < 5e-3
    assert len(peaks) > 0 and all(v == v for v in peaks) and max(peaks) < 6e4


def test_raft_feature_encoder_stays_tf32():
    """fnet keeps the TF32 path under the switch: its InstanceNorms are held to the fp32 kernel's float64 bound"""
    net = _raft()
    x = _gen_inputs(n=2, seed=5)[0].contiguous(memory_format=torch.channels_last)
    with torch.no_grad():
        outs = []
        for half in (False, True):
            with _switches(half):
                outs.append(net._encode("fnet", x))
    assert outs[0].dtype == torch.float32 and torch.equal(outs[0], outs[1])


def test_encoders_strict_fp32_unchanged_by_switch():
    gen, raft = _generator(), _raft()
    fr, mi, mu = _gen_inputs(n=2, seed=2)
    x = fr.contiguous(memory_format=torch.channels_last)
    outs = {}
    with torch.no_grad():
        for half in (False, True):
            with _switches(half, tf32=False):
                outs[half] = (gen._encode_frames(fr, mi, mu), *raft.encode_frames(x)[:3])
    for a, b in zip(outs[False], outs[True]):
        assert torch.equal(a, b)


def test_grouped_slot_placement_matches_cat():
    """both plans of the grouped layers (one grouped conv over interleaved slots, g dense convs over group-major slots) give
    exactly what the same fp16 convs give on torch.cat-built inputs: the placement moves bits, it computes nothing"""
    from propainter_b200 import ops
    from propainter_b200.nn_util import as_nchw, as_pm
    net = _generator()
    n, h, w = 2, H // 4, W // 4
    g0 = torch.Generator(device="cpu").manual_seed(4)
    x0 = torch.randn(n, h, w, 256, generator=g0).half().to(DEV)
    raw = torch.randn(n, h, w, 384, generator=g0).half().to(DEV)
    with torch.no_grad():
        o = ops.bias_act(raw.clone(), net.P["encoder.layers.8.bias"], "leaky", 0.2)
        ref = {}
        for grouped in (True, False):
            y = o
            for i, g in ((10, 2), (12, 4), (14, 8), (16, 1)):
                wt, b = net._wb16(f"encoder.layers.{i}")
                if grouped:
                    mix = torch.cat([x0.view(n, h, w, g, -1), y.view(n, h, w, g, -1)], -1).view(n, h, w, -1)
                    r = as_pm(F.conv2d(as_nchw(mix), wt, None, 1, 1, 1, g))
                else:
                    a, c, co = 256 // g, y.shape[-1] // g, wt.shape[0] // g
                    r = torch.cat([as_pm(F.conv2d(as_nchw(torch.cat([x0[..., j * a:(j + 1) * a], y[..., j * c:(j + 1) * c]], -1)),
                                                  net._wb_group(f"encoder.layers.{i}", j, g)[0].half(), None, 1, 1))
                                   for j in range(g)], -1)
                y = ops.bias_act(r, b, "leaky", 0.2, out=torch.empty(r.shape, device=DEV, dtype=torch.float32 if i == 16 else torch.float16))
            ref[grouped] = as_nchw(y)
        for grouped in (True, False):
            got = net._enc_groups_half(x0, raw, grouped)
            assert got.dtype == torch.float32 and torch.equal(got, ref[grouped])
