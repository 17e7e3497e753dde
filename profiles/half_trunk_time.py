"""Stage 4 (generator) of one clip with the half-operand switch off and on (config.HALF_OPERANDS), and the generator's conv
trunk (SoftSplit, SoftComp, sc.bias_conv, decoder) op by op at the C2 window shape.

usage: python profiles/half_trunk_time.py [c2|c1] [reps] > half_trunk.txt

One run prints: the card's name, power limit and max SM clock; warm stage-4 ms (CUDA events) for the switch off and on,
alternated, `reps` repetitions each, with min / median / max; a torch.profiler kernel table of stage 4 per setting; at the
C2 window shape (t = 18 frames, lt = 11 local frames, 60 x 108 feature map) each trunk op alone in fp32 (TF32) and fp16
operands, with ms and TFLOP/s against the H100 SXM data-sheet rates (495 TF32, 989 dense fp16), CUDA events, 256 MiB L2
flush before each launch.  The switch also covers RAFT and the transformer, so stages 1-3 run once per setting before the
timed stage-4 calls and the stage-4 difference includes the transformer's fp16 operands."""
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as g  # noqa: E402

g.build()
from bench import WORKLOADS  # noqa: E402
from propainter_b200 import config, ops, synth  # noqa: E402
from propainter_b200.inference_propainter import InferenceConfig, ProPainterPipeline  # noqa: E402

wl = WORKLOADS[sys.argv[1] if len(sys.argv) > 1 else "c2"]
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
modes = (False, True)
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
except OSError:
    card = "nvidia-smi unavailable"
print("card:", card, "|", torch.cuda.get_device_name(0))

u8, fm, md = synth.make_clip(wl["T"], wl["H"], wl["W"], mask=wl["mask"], seed=0)
u8d, fmd, mdd = torch.from_numpy(u8).cuda(), fm.cuda(), md.cuda()
pipe = ProPainterPipeline(device="cuda")
cfg = InferenceConfig(raft_iter=wl["raft_iter"])
inputs = {}
with torch.no_grad():
    for m in modes:
        config.HALF_OPERANDS = m
        frames = ops.u8_to_frames(u8d).unsqueeze(0)
        pred = pipe.complete_flows(pipe.compute_flows(frames, cfg), fmd, cfg)
        inputs[m] = pipe.propagate_images(frames, mdd, pred, cfg), pred
torch.cuda.synchronize()


def stage4(m):
    config.HALF_OPERANDS = m
    upd, pred = inputs[m]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.no_grad():
        e0.record()
        pipe.generate(upd[0], mdd, upd[1], pred, u8d, cfg)
        e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


for m in modes:                                            # capture + autotune the window graphs of both settings
    for _ in range(2):
        stage4(m)
runs = {m: [] for m in modes}
for _ in range(reps):
    for m in modes:
        runs[m].append(stage4(m))
for m in modes:
    v = runs[m]
    print(f"HALF_OPERANDS={m}: stage 4 ms over {reps} reps (min / median / max) {min(v):8.2f} {statistics.median(v):8.2f} {max(v):8.2f}")

from torch.profiler import ProfilerActivity, profile  # noqa: E402

for m in modes:
    config.HALF_OPERANDS = m
    upd, pred = inputs[m]
    with torch.no_grad(), profile(activities=[ProfilerActivity.CUDA]) as prof:
        pipe.generate(upd[0], mdd, upd[1], pred, u8d, cfg)
        torch.cuda.synchronize()
    print(f"\nHALF_OPERANDS={m}: stage 4 kernels")
    print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=30, max_name_column_width=90))

# ---------------------------------------------------------------- trunk ops alone at the C2 window shape
t, lt, h, w, C, HID = 18, 11, 60, 108, 128, 512
fh, fw = (h - 1) // 3 + 1, (w - 1) // 3 + 1
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
torch.backends.cudnn.allow_tf32 = True
torch.backends.cudnn.benchmark = True
torch.backends.cuda.matmul.allow_tf32 = True
torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction = False


def timed(fn, n=20):
    fn()
    ts = []
    for _ in range(n):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return statistics.median(ts)


def cl4(*shape, dt):
    return torch.randn(*shape, device="cuda").to(dt).contiguous(memory_format=torch.channels_last)


def report(name, flop, fn, dt):
    ms = timed(fn)
    peak = 989 if dt == torch.float16 else 495
    tf = flop / (ms * 1e-3) / 1e12
    print(f"  {name:34s} {str(dt):14s} {ms:7.3f} ms {tf:7.1f} TFLOP/s ({100 * tf / peak:.0f} % of {peak})")
    return ms


print(f"\ntrunk ops at the C2 window shape (t = {t}, lt = {lt}, {h} x {w} features, {fh} x {fw} tokens), median of 20, L2 flushed")
for dt in (torch.float32, torch.float16):
    s = 0.0
    x = cl4(t, C, h, w, dt=dt)
    wss = cl4(HID, C, 7, 7, dt=dt) / 80
    s += report("SoftSplit conv 7x7/s3 128->512, t", 2 * t * fh * fw * HID * C * 49, lambda: F.conv2d(x, wss, None, 3, 3), dt)
    tok = cl4(t, HID, fh, fw, dt=dt)
    wsc = torch.randn(HID, C, 7, 7, device="cuda").to(dt) / 23
    for n in (t, lt):
        s_ = report(f"SoftComp conv_transpose2d, {n} frames", 2 * n * fh * fw * HID * C * 49,
                    lambda: F.conv_transpose2d(tok[:n], wsc, None, 3, 3, (h + 2 - 3 * fh, w + 2 - 3 * fw)), dt)
    s += s_
    if dt == torch.float16:
        tok2 = torch.randn(lt * fh * fw, HID, device="cuda").half()
        wcol = torch.randn(49 * C, HID, device="cuda").half() / 23
        bmap = torch.randn(h, w, C, device="cuda")
        cols = torch.empty(lt * fh * fw, 49 * C, device="cuda", dtype=dt)
        fold_out = torch.empty(lt, h, w, C, device="cuda", dtype=dt)
        report(f"SoftComp GEMM (fold plan), {lt} frames", 2 * lt * fh * fw * HID * C * 49, lambda: torch.mm(tok2, wcol.t(), out=cols), dt)
        ms = timed(lambda: ops.sc_fold(cols, bmap, lt, h, w, out=fold_out))
        nbytes = cols.numel() * 2 + bmap.numel() * 4 + fold_out.numel() * 2
        print(f"  {'SoftComp fold kernel, ' + str(lt) + ' frames':34s} {str(dt):14s} {ms:7.3f} ms {nbytes / (ms * 1e-3) / 1e9:7.1f} GB/s "
              f"({100 * nbytes / (ms * 1e-3) / 3.35e12:.0f} % of 3.35 TB/s)")
    wbc = cl4(C, C, 3, 3, dt=dt) / 34
    s += report(f"sc.bias_conv 3x3 128->128, {lt} frames", 2 * lt * h * w * C * C * 9, lambda: F.conv2d(x[:lt], wbc, None, 1, 1), dt)
    d0 = cl4(lt, C, 2 * h, 2 * w, dt=dt)
    w0 = cl4(64, C, 3, 3, dt=dt) / 34
    s += report("decoder.0 3x3 128->64 @120x216", 2 * lt * 4 * h * w * 64 * C * 9, lambda: F.conv2d(d0, w0, None, 1, 1), dt)
    d2 = cl4(lt, 64, 2 * h, 2 * w, dt=dt)
    w2 = cl4(64, 64, 3, 3, dt=dt) / 24
    s += report("decoder.2 3x3 64->64 @120x216", 2 * lt * 4 * h * w * 64 * 64 * 9, lambda: F.conv2d(d2, w2, None, 1, 1), dt)
    d4 = cl4(lt, 64, 4 * h, 4 * w, dt=dt)
    s += report("decoder.4 3x3 64->64 @240x432", 2 * lt * 16 * h * w * 64 * 64 * 9, lambda: F.conv2d(d4, w2, None, 1, 1), dt)
    w6 = cl4(3, 64, 3, 3, dt=dt) / 24
    w6p = cl4(4, 64, 3, 3, dt=dt) / 24
    s += report("decoder.6 3x3 64->3 @240x432", 2 * lt * 16 * h * w * 3 * 64 * 9, lambda: F.conv2d(d4, w6, None, 1, 1), dt)
    report("decoder.6 padded to 64->4", 2 * lt * 16 * h * w * 4 * 64 * 9, lambda: F.conv2d(d4, w6p, None, 1, 1), dt)
    print(f"  {'library convs above, summed':34s} {str(dt):14s} {s:7.3f} ms per window, {16 * s:7.2f} ms per 16 windows")
    for name, src in (("upsample2x 128 ch @60x108", torch.randn(lt, h, w, C, device="cuda").to(dt)),
                      ("upsample2x 64 ch @120x216", torch.randn(lt, 2 * h, 2 * w, 64, device="cuda").to(dt))):
        ms = timed(lambda: ops.upsample2x(src))
        nbytes = src.numel() * src.element_size() * 5
        print(f"  {name:34s} {str(dt):14s} {ms:7.3f} ms {nbytes / (ms * 1e-3) / 1e9:7.1f} GB/s ({100 * nbytes / (ms * 1e-3) / 3.35e12:.0f} % of 3.35 TB/s)")
