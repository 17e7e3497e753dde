"""The generator's conv trunk (SoftSplit, SoftComp, sc.bias_conv, decoder) on half-precision operands (config.HALF_OPERANDS
while cuDNN may use TF32) against the oracle, and its two fp16 kernels against float64.

The trunk's convs take fp16 operands where they would run TF32 anyway, so the half-operand trunk must stay in the error class
of the TF32 trunk it replaces: the generator runs with the trunk on fp16 and with everything on TF32, on the same inputs and
weights, and both errors are taken against the fp32 oracle (run on the GPU with TF32 off).  The transformer keeps its own
setting (TF32 here) so that the comparison sees the trunk alone; tests/test_gpu_half_transformer.py flips both together.
The tests set the switches themselves and restore them.
"""
import contextlib
import gc

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import generator_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(autouse=True)
def _release_graph_pools():
    """each test builds its own generator, whose captured C2-sized graphs hold private memory pools until the net is
    collected: release them after the test so that later tests in the same process get the memory back"""
    yield
    gc.collect()
    torch.cuda.empty_cache()


@contextlib.contextmanager
def _switches(half, tf32=True, graphs=None, half_transformer=False):
    from propainter_b200 import config
    prev = (config.HALF_OPERANDS, config.LINEAR_TF32, config.CUDA_GRAPHS, torch.backends.cuda.matmul.allow_tf32,
            torch.backends.cudnn.allow_tf32)
    config.HALF_OPERANDS, config.LINEAR_TF32 = half, tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = tf32
    if graphs is not None:
        config.CUDA_GRAPHS = graphs
    try:
        with pytest.MonkeyPatch.context() as mp:
            if not half_transformer:
                mp.setattr(config, "half_linears", lambda: False)
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


def _net():
    from propainter_b200.model.propainter import InpaintGenerator
    return InpaintGenerator(seed=3).to(DEV)


# (240, 432): the C2 window shape; (248, 424): a 62 x 106 feature map (neither a multiple of 3 nor of 8)
@pytest.mark.parametrize("H,W,t,lt", [(240, 432, 18, 11), (248, 424, 7, 4)])
def test_half_trunk_error_vs_tf32(H, W, t, lt):
    net = _net()
    mf, flows, masks, upd = _inputs(H, W, t, lt)
    sd = {k: v.detach() for k, v in net.state_dict().items()}
    with _switches(False, tf32=False):
        ref, rparts = generator_ref.generator_forward(sd, mf, flows, masks, upd, lt, return_parts=True)
    errs = {}
    for half in (False, True):
        with _switches(half):
            out, parts = net.forward_parts(mf, flows, masks, upd, lt)
            shipped = net(mf, flows, masks, upd, lt)
        errs[half] = {"enc_out": rel_err(parts["enc_out"], rparts["enc_out"][0]), "out": rel_err(out, ref),
                      "out (graph)": rel_err(shipped, ref)}
    print(f"generator {H}x{W} t={t}: TF32 trunk " + " ".join(f"{k}={v:.2e}" for k, v in errs[False].items()) +
          " | fp16 trunk " + " ".join(f"{k}={v:.2e}" for k, v in errs[True].items()))
    for k in errs[True]:
        assert errs[True][k] < 5e-3                                    # catches a broken path
        assert errs[True][k] <= 1.5 * errs[False][k] + 1e-5, k


def test_half_trunk_range():
    """every fp16 tensor of the trunk (enc2, the SoftSplit conv output, the SoftComp result, the decoder's input, the decoder's
    conv and up-sampling outputs, decoder.6's raw output) stays far inside fp16's range on a C2 window"""
    from propainter_b200 import ops
    peak, finite = {}, []

    def note(k, v):
        if v is not None and v.dtype == torch.float16:
            peak[k] = max(peak.get(k, 0.0), v.float().abs().max().item())
            finite.append(bool(torch.isfinite(v).all()))
    real = {"conv2d": F.conv2d, "tconv": F.conv_transpose2d, "fold": ops.sc_fold, "up": ops.upsample2x, "ba": ops.bias_act,
            "mm": torch.mm}

    def wrap(key, label):
        def fn(*a, **k):
            r = real[key](*a, **k)
            note(label(a, k) if callable(label) else label, r)
            return r
        return fn

    def conv_label(a, k):
        x, w = a[0], a[1]
        if x.dtype == torch.float16 and x.shape[0] == 18 and x.shape[1] == 128 and w.shape[-1] == 7:
            note("enc2", x)
        return f"conv {w.shape[1]}->{w.shape[0]} {w.shape[-1]}x{w.shape[-1]}"
    net = _net()
    mf, flows, masks, upd = _inputs(240, 432, 18, 11)
    with _switches(True, graphs=False, half_transformer=True), pytest.MonkeyPatch.context() as mp:
        mp.setattr(F, "conv2d", wrap("conv2d", conv_label))
        mp.setattr(F, "conv_transpose2d", wrap("tconv", "SoftComp (transposed conv)"))
        mp.setattr(torch, "mm", wrap("mm", "SoftComp columns"))
        mp.setattr(ops, "sc_fold", wrap("fold", "SoftComp (fold)"))
        mp.setattr(ops, "upsample2x", wrap("up", lambda a, k: f"up2 {a[0].shape[-1]} ch"))
        mp.setattr(ops, "bias_act", wrap("ba", lambda a, k: f"epilogue {a[0].shape[-1]} ch"))
        out = net(mf, flows, masks, upd, 11)
    print("max |fp16 tensor|:", {k: round(v, 2) for k, v in peak.items()})
    assert {"enc2", "conv 128->512 7x7", "conv 128->128 3x3", "epilogue 128 ch", "up2 128 ch", "conv 128->64 3x3",
            "conv 64->64 3x3", "up2 64 ch", "conv 64->4 3x3", "epilogue 64 ch"} <= set(peak)
    assert {"SoftComp (transposed conv)", "SoftComp (fold)"} & set(peak)
    assert all(finite) and bool(torch.isfinite(out).all())
    assert max(peak.values()) < 6e4


def test_strict_fp32_unchanged():
    """with cuDNN TF32 (and the Linear layers' TF32) off, the switch changes nothing: SoftSplit, SoftComp with sc.bias_conv,
    and the decoder as the generator calls them are bit for bit the same with it on and off, with cuDNN held to
    deterministic algorithms (the whole generator is not compared: its propagation scans do not repeat bit for bit from
    run to run)"""
    from propainter_b200 import config
    net = _net()
    gen = torch.Generator(device=DEV).manual_seed(0)
    t, lt, hw = 7, 4, (62, 106)
    feat = torch.randn(t, 128, *hw, device=DEV, generator=gen).contiguous(memory_format=torch.channels_last)
    tok = torch.randn(t, 21, 36, 512, device=DEV, generator=gen)
    res = {}
    for half in (False, True):
        with _switches(half, tf32=False, half_transformer=True), torch.backends.cudnn.flags(
                enabled=True, benchmark=False, deterministic=True, allow_tf32=False):
            h = feat.is_cuda and config.half_convs()
            assert not h
            enc3 = net.tx.soft_comp(tok, hw, feat[:lt], lt, h)
            res[half] = (net.tx.soft_split(feat), enc3, net._decoder(enc3))
    assert all(torch.equal(a, b) for a, b in zip(res[False], res[True]))


@pytest.mark.parametrize("half", [False, True])
def test_soft_comp_local_frames_only(half):
    """SoftComp for the first lt frames gives the first lt frames of SoftComp over all t frames: exactly per frame in the fold
    kernel, and through the library GEMM / conv and sc.bias_conv to fp32 summation-order level (fp32 path) or to a one-ulp
    flip of a fp16-rounded fold output (half path: the two frame counts may take different GEMM kernels or plans)"""
    from propainter_b200 import ops
    from propainter_b200.nn_util import as_pm
    net = _net()
    gen = torch.Generator(device=DEV).manual_seed(0)
    t, lt, hw = 18, 11, (60, 108)
    tok = torch.randn(t, 20, 36, 512, device=DEV, generator=gen)
    res = torch.randn(t, 128, *hw, device=DEV, generator=gen).contiguous(memory_format=torch.channels_last)
    with _switches(half):
        full = net.tx.soft_comp(tok, hw, res, t, half)
        part = net.tx.soft_comp(tok, hw, res[:lt], lt, half)
    assert part.shape == (lt, 128, *hw)
    assert rel_err(part, full[:lt]) < (1e-3 if half else 1e-5)
    cols = torch.randn(t * 720, 49 * 128, device=DEV, generator=gen).half()
    bmap = as_pm(net.tx._sc_bias_map(hw))[0]
    assert torch.equal(ops.sc_fold(cols[:lt * 720], bmap, lt, *hw), ops.sc_fold(cols, bmap, t, *hw)[:lt])


def _fold64(cols, bmap, frames, h, w):
    C = bmap.shape[-1]
    fh, fw = (h - 1) // 3 + 1, (w - 1) // 3 + 1
    y = cols.double().view(frames, fh * fw, 49, C).permute(0, 3, 2, 1).reshape(frames, C * 49, fh * fw)
    s = F.fold(y, (h, w), 7, stride=3, padding=3).permute(0, 2, 3, 1)
    a = F.fold(y.abs(), (h, w), 7, stride=3, padding=3).permute(0, 2, 3, 1)
    return s + bmap.double(), a + bmap.double().abs()


def _check_rn16(got, ref, mag, nterms):
    """got (fp16) is ref (float64) rounded to nearest, up to the fp32 arithmetic error of an `nterms`-term sum"""
    ulp = torch.from_numpy(np.spacing(np.abs(ref.cpu().numpy()).astype(np.float16)).astype(np.float64)).to(ref.device)
    bound = 0.5 * ulp + nterms * 2.0 ** -24 * mag
    err = (got.double() - ref).abs()
    assert bool((err <= bound).all()), (err - bound).max().item()
    return (err / ulp.clamp_min(2.0 ** -24)).max().item()


@pytest.mark.parametrize("frames,h,w", [(11, 60, 108), (3, 61, 107), (2, 25, 34), (1, 4, 5)])
def test_sc_fold_f16_vs_float64(frames, h, w):
    """pp_sc_fold_f16 element by element against a float64 F.fold + bias map, on the C2 map, ragged maps (61 x 107: neither a
    multiple of 3 nor of 8) and maps smaller than one patch; columns sit in a wider NaN-padded buffer (ldc > 49*C)"""
    from propainter_b200 import ops
    gen = torch.Generator(device=DEV).manual_seed(frames * 1000 + h)
    C = 128
    fh, fw = (h - 1) // 3 + 1, (w - 1) // 3 + 1
    wide = torch.full((frames * fh * fw, 49 * C + 8), float("nan"), device=DEV, dtype=torch.float16)
    cols = wide[:, :49 * C]
    cols.copy_(torch.randn(frames * fh * fw, 49 * C, device=DEV, generator=gen) * 2)
    bmap = torch.randn(h, w, C, device=DEV, generator=gen)
    out = torch.full((frames + 1, h, w, C), float("nan"), device=DEV, dtype=torch.float16)
    got = ops.sc_fold(cols, bmap, frames, h, w, out=out[:frames])
    ref, mag = _fold64(cols, bmap, frames, h, w)
    worst = _check_rn16(got, ref, mag, 10)
    assert torch.isnan(out[frames]).all()
    print(f"sc_fold {frames}x{h}x{w}: max error {worst:.3f} fp16 ulp")


def _up2_weights(n_out, n_in):
    """the kernel's fp32 source index and weights (pp_up2_coord), as float64"""
    f = np.float32
    s = f(f(n_in - 1) / f(2 * n_in - 1)) * np.arange(n_out, dtype=f)
    i0 = s.astype(np.int64)
    l1 = (s - i0.astype(f)).astype(f)
    return i0, np.minimum(i0 + 1, n_in - 1), (f(1) - l1).astype(np.float64), l1.astype(np.float64)


@pytest.mark.parametrize("n,h,w,C", [(11, 60, 108, 128), (11, 120, 216, 64), (2, 31, 27, 64), (1, 2, 3, 8)])
def test_upsample2x_f16_vs_float64(n, h, w, C):
    """the fp16 instance of k_upsample2x against a float64 bilinear blend (align_corners=True) at the kernel's own fp32
    source coordinates, which the fp32 instance shares"""
    from propainter_b200 import ops
    gen = torch.Generator(device=DEV).manual_seed(n * 100 + h)
    x = (torch.randn(n, h, w, C, device=DEV, generator=gen) * 3).half()
    got = ops.upsample2x(x)
    assert got.dtype == torch.float16
    y0, y1, a0, a1 = (torch.from_numpy(v).to(DEV) for v in _up2_weights(2 * h, h))
    x0, x1, b0, b1 = (torch.from_numpy(v).to(DEV) for v in _up2_weights(2 * w, w))
    xd = x.double()
    row = lambda yi: xd[:, yi][:, :, x0] * b0[:, None] + xd[:, yi][:, :, x1] * b1[:, None]
    ref = row(y0) * a0[:, None, None] + row(y1) * a1[:, None, None]
    _check_rn16(got, ref, xd.abs().amax().expand_as(ref), 8)


def test_half_trunk_entries_refuse_misaligned_and_accept_empty():
    from propainter_b200 import _lib
    L = _lib.lib()
    s = torch.cuda.current_stream().cuda_stream
    cols = torch.zeros(720 * 49 * 128 + 8, device=DEV, dtype=torch.float16)
    bmap = torch.zeros(60 * 108 * 128 + 4, device=DEV)
    out = torch.zeros(60 * 108 * 128 + 8, device=DEV, dtype=torch.float16)
    ldc = 49 * 128
    assert L.pp_sc_fold_f16(cols.data_ptr() + 2, ldc, bmap.data_ptr(), out.data_ptr(), 1, 60, 108, 128, s) == -5
    assert L.pp_sc_fold_f16(cols.data_ptr(), ldc, bmap.data_ptr() + 4, out.data_ptr(), 1, 60, 108, 128, s) == -5
    assert L.pp_sc_fold_f16(cols.data_ptr(), ldc + 2, bmap.data_ptr(), out.data_ptr(), 1, 60, 108, 128, s) == -5
    assert L.pp_sc_fold_f16(cols.data_ptr(), ldc - 4, bmap.data_ptr(), out.data_ptr(), 1, 60, 108, 128, s) != 0
    assert L.pp_sc_fold_f16(cols.data_ptr(), ldc, bmap.data_ptr(), out.data_ptr(), 0, 60, 108, 128, s) == 0
    assert L.pp_upsample2x_bilinear_f16(cols.data_ptr() + 2, out.data_ptr(), 1, 4, 4, 8, s) == -5
    assert L.pp_upsample2x_bilinear_f16(cols.data_ptr(), out.data_ptr(), 1, 4, 4, 12, s) == -5
    assert L.pp_upsample2x_bilinear_f16(cols.data_ptr(), out.data_ptr(), 0, 4, 4, 8, s) == 0
    torch.cuda.synchronize()
