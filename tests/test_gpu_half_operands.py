"""RAFT's refinement loop on half-precision operands (config.HALF_OPERANDS) against the oracle.

fp16 has TF32's 10 explicit mantissa bits, so the half-operand path must stay in the error class of the TF32 library
path it replaces: each test runs both on the same inputs and weights, with cuDNN TF32 allowed (the shipping setting),
and compares their errors against the fp32 oracle.  The tests set the switches themselves and restore them.
"""
import contextlib

import pytest
import torch

from oracle import pipeline_ref, raft_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"


@contextlib.contextmanager
def _switches(half, tf32=True):
    from propainter_b200 import config
    prev = config.HALF_OPERANDS, torch.backends.cudnn.allow_tf32
    config.HALF_OPERANDS, torch.backends.cudnn.allow_tf32 = half, tf32
    try:
        yield
    finally:
        config.HALF_OPERANDS, torch.backends.cudnn.allow_tf32 = prev


def cpu_sd(m):
    return {k: v.detach().cpu() for k, v in m.state_dict().items()}


def _errors(fw, bw, rf, rb):
    rel = max((a.cpu() - b).abs().max().item() / max(b.abs().max().item(), 1e-12) for a, b in ((fw, rf), (bw, rb)))
    epe = max(((a.cpu() - b) ** 2).sum(2).sqrt().mean().item() for a, b in ((fw, rf), (bw, rb)))
    return rel, epe


def _compare(net, frames, iters, label):
    rf, rb = raft_ref.raft_bi(cpu_sd(net.fix_raft), frames, iters)
    out = {}
    for half in (False, True):
        with _switches(half):
            fw, bw = net(frames.to(DEV), iters=iters)
        out[half] = _errors(fw, bw, rf, rb)
    (r32, e32), (r16, e16) = out[False], out[True]
    print(f"{label}: TF32 rel {r32:.2e} EPE {e32:.4f}px | fp16 operands rel {r16:.2e} EPE {e16:.4f}px | "
          f"|flow|max {max(rf.abs().max().item(), rb.abs().max().item()):.2f}")
    # the TF32 path itself measures 1.6e-3 of a 1.4 px flow at 2 iterations on the small clip: the bar that separates the
    # two precision classes is the ratio, the absolute one only catches a broken path
    assert r16 <= 5e-3 and e16 <= 0.05
    assert r16 <= 1.5 * r32 and e16 <= 1.5 * e32


def test_raft_half_operands_small_clip():
    from propainter_b200 import synth
    from propainter_b200.model.modules.flow_comp_raft import RAFT_bi
    net = RAFT_bi(None, DEV, seed=1)
    u8, _, _ = synth.make_clip(4, 128, 144, seed=3)
    frames = pipeline_ref.to_float_frames(u8)
    for iters in (2, 12):
        _compare(net, frames, iters, f"4x128x144 iters={iters}")


def test_raft_half_operands_c2_slice():
    """12 frames of the benchmark's C2 clip at its 240x432 size, 20 iterations"""
    from propainter_b200 import synth
    from propainter_b200.model.modules.flow_comp_raft import RAFT_bi
    net = RAFT_bi(None, DEV, seed=1)
    u8, _, _ = synth.make_clip(80, 240, 432, mask="ellipse", seed=0)
    frames = pipeline_ref.to_float_frames(u8[:12])
    _compare(net, frames, 20, "C2 12x240x432 iters=20")


def test_raft_half_operands_range():
    """C2 slice, eager: the fp32 state stays finite and no fp16 operand comes near the fp16 maximum (65504)"""
    from propainter_b200 import ops, synth
    from propainter_b200.model.modules.flow_comp_raft import RAFT_bi
    net = RAFT_bi(None, DEV, seed=1)
    u8, _, _ = synth.make_clip(80, 240, 432, mask="ellipse", seed=0)
    frames = pipeline_ref.to_float_frames(u8[:12])[0].to(DEV)
    peak, state_finite = {}, []

    def watch(name, fn, pick):
        def wrapped(*a, **kw):
            r = fn(*a, **kw)
            for t in pick(a, kw, r):
                if t is not None and t.dtype == torch.float16:
                    peak[name] = max(peak.get(name, 0.0), t.abs().max().item())
            return r
        return wrapped

    def update(*a, **kw):
        r = gru_update(*a, **kw)
        state_finite.append(bool(torch.isfinite(a[3]).all()))
        return r
    mp = pytest.MonkeyPatch()
    try:
        mp.setattr(ops, "corr_lookup", watch("corr", ops.corr_lookup, lambda a, kw, r: [r]))
        mp.setattr(ops, "bias_act", watch("bias_act", ops.bias_act, lambda a, kw, r: [a[0], r]))
        mp.setattr(ops, "raft_pack_motion", watch("motion", ops.raft_pack_motion, lambda a, kw, r: [a[0], a[2]]))
        mp.setattr(ops, "gru_gate", watch("gate", ops.gru_gate, lambda a, kw, r: [a[0], a[4]]))
        gru_update = watch("update", ops.gru_update, lambda a, kw, r: [a[0], kw.get("h_img")])
        mp.setattr(ops, "gru_update", update)
        with _switches(True), torch.no_grad():
            net.fix_raft._flows_bidirectional(frames, 20)
            torch.cuda.synchronize()
    finally:
        mp.undo()
    print("max |fp16 operand|:", {k: round(v, 2) for k, v in peak.items()})
    assert set(peak) == {"corr", "bias_act", "motion", "gate", "update"}
    assert state_finite and all(state_finite)
    assert max(peak.values()) < 6e4


def test_half_operands_follow_cudnn_tf32():
    """with cuDNN TF32 off the switch changes nothing: strict-fp32 runs stay strict"""
    from propainter_b200 import synth
    from propainter_b200.model.modules.flow_comp_raft import RAFT_bi
    net = RAFT_bi(None, DEV, seed=1)
    u8, _, _ = synth.make_clip(4, 128, 144, seed=3)
    frames = pipeline_ref.to_float_frames(u8).to(DEV)
    outs = []
    for half in (False, True):
        with _switches(half, tf32=False):
            outs.append(net(frames, iters=2))
    assert all(torch.equal(a, b) for a, b in zip(*outs))
