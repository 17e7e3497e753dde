"""The generator's transformer on half-precision operands (config.HALF_OPERANDS) against the oracle.

Its Linear layers take fp16 operands where they would run TF32 anyway, so the half-operand generator must stay in the
error class of the TF32 path it replaces: each comparison runs both settings on the same inputs and weights and compares
their errors against the fp32 oracle (run on the GPU with TF32 off).  The fp16 overlap-add and LayerNorm kernels are
checked bit for bit against their fp32 instantiations, the attention kernels against float64 in
tests/test_gpu_half_attention_f64.py.  The tests set the switches themselves and restore them.
"""
import contextlib

import pytest
import torch
import torch.nn.functional as F

from oracle import generator_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"


@contextlib.contextmanager
def _switches(half, tf32=True, graphs=None):
    from propainter_b200 import config
    prev = (config.HALF_OPERANDS, config.LINEAR_TF32, config.CUDA_GRAPHS, torch.backends.cuda.matmul.allow_tf32,
            torch.backends.cudnn.allow_tf32)
    config.HALF_OPERANDS, config.LINEAR_TF32 = half, tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = tf32
    if graphs is not None:
        config.CUDA_GRAPHS = graphs
    try:
        yield
    finally:
        (config.HALF_OPERANDS, config.LINEAR_TF32, config.CUDA_GRAPHS, torch.backends.cuda.matmul.allow_tf32,
         torch.backends.cudnn.allow_tf32) = prev


def rel_err(a, b):
    return (a.float() - b.float()).abs().max().item() / max(b.abs().max().item(), 1e-12)


def _inputs(H, W, t, lt, seed=1):
    gen = torch.Generator().manual_seed(seed)
    frames = torch.rand(1, t, 3, H, W, generator=gen) * 2 - 1
    sm = lambda z: F.avg_pool2d(z.view(-1, 2, H, W), 9, 1, 4).view(z.shape)
    flows = (sm(torch.randn(1, lt - 1, 2, H, W, generator=gen) * 12), sm(torch.randn(1, lt - 1, 2, H, W, generator=gen) * 12))
    masks = torch.zeros(1, t, 1, H, W)
    masks[..., H // 4:H // 2, W // 3:2 * W // 3] = 1
    upd = masks * (torch.rand(1, t, 1, H, W, generator=gen) > 0.5).float()
    mf = frames * (1 - masks)
    return mf.to(DEV), (flows[0].to(DEV), flows[1].to(DEV)), masks.to(DEV), upd.to(DEV)


# (128, 128): an 11 x 11 token grid, padded to 15 x 18 for the windows (the F.pad path of y); (240, 432): the C2 window shape
@pytest.mark.parametrize("H,W,t,lt", [(128, 128, 5, 3), (240, 432, 18, 11)])
def test_half_transformer_error_vs_tf32(H, W, t, lt):
    from propainter_b200.model.propainter import InpaintGenerator
    net = InpaintGenerator(seed=3).to(DEV)
    mf, flows, masks, upd = _inputs(H, W, t, lt)
    sd = {k: v.detach() for k, v in net.state_dict().items()}
    with _switches(False, tf32=False):
        ref, rparts = generator_ref.generator_forward(sd, mf, flows, masks, upd, lt, return_parts=True)
    errs = {}
    for half in (False, True):
        with _switches(half):
            out, parts = net.forward_parts(mf, flows, masks, upd, lt)
        fh, fw = parts["tokens_in"].shape[1:3]
        errs[half] = {"tokens_out": rel_err(parts["tokens_out"], rparts["tokens_out"].view(t, fh, fw, -1)),
                      "enc_out": rel_err(parts["enc_out"], rparts["enc_out"][0]), "out": rel_err(out, ref)}
    print(f"generator {H}x{W} t={t}: TF32 " + " ".join(f"{k}={v:.2e}" for k, v in errs[False].items()) +
          " | fp16 operands " + " ".join(f"{k}={v:.2e}" for k, v in errs[True].items()))
    for k in errs[True]:
        assert errs[True][k] < 5e-3                                    # catches a broken path
        assert errs[True][k] <= 1.5 * errs[False][k] + 1e-5, k


def test_half_transformer_range():
    """every fp16 tensor of the transformer (LayerNorm outputs y, qkv, pooled tokens, pool_kv, attention output, proj / fc1 /
    fc2 outputs -- the last block's fc2 output included -- and Z) stays far inside fp16's range on a C2 window"""
    from propainter_b200 import ops
    from propainter_b200.model.propainter import InpaintGenerator
    peak, finite = {}, []

    def note(k, v):
        if v is not None and v.dtype == torch.float16:
            peak[k] = max(peak.get(k, 0.0), v.float().abs().max().item())
            finite.append(bool(torch.isfinite(v).all()))
    names = {(1536, 512): "qkv", (1024, 512): "pool_kv", (512, 512): "proj out", (1960, 512): "fc1 out", (512, 1960): "fc2 out"}
    real = {"linear": F.linear, "ffn": ops.ffn_overlap_add, "ln": ops.add_layernorm, "pool": ops.pool_depthwise,
            "attn": ops.sparse_window_attn}

    def linear(x, w, b=None):
        y = real["linear"](x, w, b)
        note(names.get(tuple(w.shape), "other linear"), y)
        return y

    def wrap(key, label, pick):
        def fn(*a, **k):
            r = real[key](*a, **k)
            note(label, pick(r))
            return r
        return fn
    net = InpaintGenerator(seed=3).to(DEV)
    mf, flows, masks, upd = _inputs(240, 432, 18, 11)
    with _switches(True, graphs=False), pytest.MonkeyPatch.context() as mp:
        mp.setattr(F, "linear", linear)
        mp.setattr(ops, "ffn_overlap_add", wrap("ffn", "Z", lambda r: r))
        mp.setattr(ops, "add_layernorm", wrap("ln", "y", lambda r: r[1]))
        mp.setattr(ops, "pool_depthwise", wrap("pool", "pooled", lambda r: r))
        mp.setattr(ops, "sparse_window_attn", wrap("attn", "attention out", lambda r: r))
        out = net(mf, flows, masks, upd, 11)
    print("max |fp16 operand|:", {k: round(v, 2) for k, v in peak.items()})
    assert set(peak) == {"y", "qkv", "pooled", "pool_kv", "attention out", "proj out", "fc1 out", "Z", "fc2 out"}
    assert all(finite) and bool(torch.isfinite(out).all())
    assert max(peak.values()) < 6e4


def test_strict_fp32_unchanged():
    """with LINEAR_TF32 and matmul TF32 off the switch changes nothing: the transformer of a strict-fp32 run is bit for bit
    the same with it on and off, on a padded (11 x 11 tokens) and the C2 (20 x 36) token grid, masked and unmasked windows
    mixed"""
    from propainter_b200.model.propainter import InpaintGenerator
    net = InpaintGenerator(seed=3).to(DEV)
    gen = torch.Generator(device=DEV).manual_seed(0)
    for t, fh, fw, hw in ((5, 11, 11, (32, 32)), (6, 20, 36, (60, 108))):
        tokens = torch.randn(t, fh, fw, 512, device=DEV, generator=gen)
        nwin = -(-fh // 5) * -(-fw // 9)
        flags = (torch.arange(nwin, device=DEV) % 3 == 0).int()
        outs = []
        for half in (False, True):
            with _switches(half, tf32=False):
                outs.append(net.tx.run(tokens, hw, flags))
        assert torch.equal(outs[0], outs[1])
        with _switches(True):
            assert not torch.equal(outs[0], net.tx.run(tokens, hw, flags))


def test_switch_recaptures():
    """the graph key carries the switch: flipping it captures again, and each capture replays bit for bit"""
    from propainter_b200 import graphs
    from propainter_b200.model.propainter import InpaintGenerator
    net = InpaintGenerator(seed=3).to(DEV)
    mf, flows, masks, upd = _inputs(128, 128, 5, 3)
    keys, res = [], {}
    for half in (False, True):
        with _switches(half, graphs=True):
            keys.append(graphs._switches())
            res[half] = (net(mf, flows, masks, upd, 3).clone(), net(mf, flows, masks, upd, 3).clone())
    assert keys[0] != keys[1]
    assert not torch.equal(res[False][0], res[True][0])
    assert all(torch.equal(a, b) for a, b in res.values())


def test_ffn_overlap_add_f16_bit_identical():
    from propainter_b200 import ops
    gen = torch.Generator(device=DEV).manual_seed(0)
    for frames, h, w in ((1, 7, 5), (3, 60, 108), (18, 60, 108)):
        fh, fw = (h - 1) // 3 + 1, (w - 1) // 3 + 1
        Y16 = (torch.randn(frames * fh * fw, 1960, device=DEV, generator=gen) * 3).half()
        Z16 = ops.ffn_overlap_add(Y16, frames, h, w, 40)
        Z32 = ops.ffn_overlap_add(Y16.float(), frames, h, w, 40)
        assert Z16.dtype == torch.float16 and torch.equal(Z16, Z32.half())


def test_add_layernorm_f16_bit_identical():
    from propainter_b200 import ops
    gen = torch.Generator(device=DEV).manual_seed(0)
    for rows in (1, 7, 18 * 720):
        x = torch.randn(rows, 512, device=DEV, generator=gen) * 4
        d16 = (torch.randn(rows, 512, device=DEV, generator=gen) * 2).half()
        g, b = torch.randn(512, device=DEV, generator=gen), torch.randn(512, device=DEV, generator=gen)
        for delta in (d16, d16.float()):
            for yd in (torch.float16, torch.float32):
                if delta.dtype == torch.float32 and yd == torch.float32:
                    continue
                xo, y = ops.add_layernorm(x, delta, g, b, y_dtype=yd)
                xr, yr = ops.add_layernorm(x, delta.float(), g, b)
                assert y.dtype == yd and torch.equal(xo, xr) and torch.equal(y, yr.to(yd))
        _, y = ops.add_layernorm(x, None, g, b, y_dtype=torch.float16)
        assert torch.equal(y, ops.add_layernorm(x, None, g, b)[1].half())


def test_half_entries_refuse_misaligned_and_accept_empty():
    from propainter_b200 import _lib
    L = _lib.lib()
    s = torch.cuda.current_stream().cuda_stream
    Y = torch.zeros(64 * 1960 + 8, device=DEV, dtype=torch.float16)
    ws = torch.zeros(1 << 20, device=DEV)
    assert L.pp_ffn_overlap_add_f16(Y.data_ptr() + 2, 1960, Y.data_ptr(), 1960, 1, 7, 5, 40, ws.data_ptr(), ws.numel() * 4, s) == -5
    assert L.pp_ffn_overlap_add_f16(Y.data_ptr(), 1964, Y.data_ptr(), 1960, 1, 7, 5, 40, ws.data_ptr(), ws.numel() * 4, s) == -5
    assert L.pp_ffn_overlap_add_f16(Y.data_ptr(), 1960, Y.data_ptr(), 1960, 0, 7, 5, 40, ws.data_ptr(), ws.numel() * 4, s) == 0
    x = torch.zeros(4 * 512 + 8, device=DEV)
    assert L.pp_add_layernorm_f16(x.data_ptr(), x.data_ptr(), 0, x.data_ptr(), x.data_ptr(), x.data_ptr(), Y.data_ptr() + 2, 1,
                                  4, 512, 1e-5, s) == -5
    assert L.pp_add_layernorm_f16(x.data_ptr(), None, 0, x.data_ptr(), x.data_ptr(), None, Y.data_ptr(), 1, 0, 512, 1e-5, s) == 0
    torch.cuda.synchronize()


def test_pool_depthwise_f16_bit_identical():
    from propainter_b200 import ops
    gen = torch.Generator(device=DEV).manual_seed(0)
    for n, H, W in ((1, 4, 4), (5, 15, 18), (18, 20, 36)):
        x = (torch.randn(n, H, W, 512, device=DEV, generator=gen) * 2).half()
        w, b = torch.randn(16, 512, device=DEV, generator=gen), torch.randn(512, device=DEV, generator=gen)
        p16 = ops.pool_depthwise(x, w, b, 4, 4)
        assert p16.dtype == torch.float16 and torch.equal(p16, ops.pool_depthwise(x.float(), w, b, 4, 4).half())
