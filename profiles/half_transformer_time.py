"""Stage 4 (generator) of one clip with the transformer's half-operand feed-forward off and on (config.HALF_OPERANDS).

usage: python profiles/half_transformer_time.py [c2|c1] [reps] > half_transformer.txt

One run prints: the card's name, power limit and max SM clock; warm stage-4 ms (CUDA events) for the switch off and on,
alternated, `reps` repetitions each, with min / median / max; a torch.profiler kernel table of stage 4 per setting; at the
C2 window shape (t = 18, 20 x 36 tokens per frame) the achieved TFLOP/s of each transformer Linear layer in fp32 (TF32) and fp16
operands, against the H100 SXM data-sheet rates (495 TF32, 989 dense fp16), and the fused overlap-add's GB/s against the
3.35 TB/s HBM3 peak (CUDA events, 256 MiB L2 flush before each launch).  RAFT is switched with the same flag, so stages
1-3 run once per setting before the timed stage-4 calls."""
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
    print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=25, max_name_column_width=90))

# ---------------------------------------------------------------- kernels alone at the C2 window shape
t, h, w, C, HID = 18, 60, 108, 512, 1960                  # feature map 60 x 108 -> 20 x 36 tokens per frame
N = t * ((h - 1) // 3 + 1) * ((w - 1) // 3 + 1)
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")


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


torch.backends.cuda.matmul.allow_tf32 = True
torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction = False
print(f"\nLinear layers at the C2 window shape ({N} tokens), median of 20, L2 flushed")
for name, k, n in (("qkv", C, 3 * C), ("proj", C, C), ("fc1", C, HID), ("fc2", HID, C)):
    for dt, peak in ((torch.float32, 495), (torch.float16, 989)):
        a = torch.randn(N, k, device="cuda").to(dt)
        wt = torch.randn(n, k, device="cuda").to(dt) / k ** 0.5
        b = torch.randn(n, device="cuda").to(dt)
        ms = timed(lambda: F.linear(a, wt, b))
        tf = 2 * N * k * n / (ms * 1e-3) / 1e12
        print(f"  {name:5s} {str(dt):14s} {ms:7.3f} ms {tf:7.1f} TFLOP/s ({100 * tf / peak:.0f} % of {peak})")

print("\nFFN overlap-add (fold + unfold) at the C2 window shape, median of 20, L2 flushed")
for dt in (torch.float32, torch.float16):
    Y = torch.randn(N, HID, device="cuda").to(dt)
    ms = timed(lambda: ops.ffn_overlap_add(Y, t, h, w, 40))
    es = Y.element_size()
    nbytes = 2 * N * HID * es + 2 * t * h * w * 40 * 4      # Y read, Z written, fp32 workspace written and read once
    print(f"  {str(dt):14s} {ms:7.3f} ms {nbytes / (ms * 1e-3) / 1e9:7.1f} GB/s ({100 * nbytes / (ms * 1e-3) / 3.35e12:.0f} % of 3.35 TB/s)")

print("\nwindow attention alone at the C2 window shape (t = 18, key frames 0, 2, .., 16), median of 20, L2 flushed")
from propainter_b200.window_index import window_key_table  # noqa: E402

ktab = torch.from_numpy(window_key_table(20, 36)).cuda()
NT, NP, NKO, nwin, nkf = 720, 45, ktab.shape[1], ktab.shape[0], 9
qkv = torch.randn(t, NT, 3 * C, device="cuda")
pkv = torch.randn(t, NP, 2 * C, device="cuda")
for label, masked in (("masked windows (wgmma)", 1), ("unmasked windows (mma.sync)", 0)):
    flags = torch.full((nwin,), masked, dtype=torch.int32, device="cuda")
    per_head = 2 * 2 * (t * 45) * (nkf * (NKO + NP)) * 128 if masked else t * 2 * 2 * 45 * 45 * 128
    flop = per_head * nwin * (C // 128)
    for dt, peak in ((torch.float32, 495), (torch.float16, 989)):
        a, b = qkv.to(dt), pkv.to(dt)
        ms = timed(lambda: ops.sparse_window_attn(a, b, ktab, flags, t, NT, 0, 2))
        tf = flop / (ms * 1e-3) / 1e12
        print(f"  {label:28s} {str(dt):14s} {ms:7.3f} ms {tf:7.1f} TFLOP/s ({100 * tf / peak:.0f} % of {peak})")
