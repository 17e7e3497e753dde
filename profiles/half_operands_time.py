"""Stage times and kernel split of one C2 step with half-precision operands off and on (config.HALF_OPERANDS).

usage: python profiles/half_operands_time.py [c2|c1] [reps] > half_operands.txt

One run prints: the card's name, power limit and max SM clock; warm stage ms (CUDA events) for the switch off and on,
alternated, `reps` repetitions each, with min / median / max; a torch.profiler kernel table of stage 1 (RAFT) and stage 4
(generator) per setting; the achieved TFLOP/s of RAFT's refinement-loop convs, computed from their shapes over the
profiled time of the library conv kernels of stage 1, against the H100 SXM data-sheet rates (989 TFLOP/s dense fp16,
495 TF32)."""
import os
import statistics
import subprocess
import sys

import torch

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


def refine_flops(T, H, W, iters):
    """Refinement-loop conv FLOPs of RAFT_bi over a T-frame clip (2 MAC = 2 FLOP): convc1 1x1 324->256, convc2 3x3 256->192,
    convf2 3x3 128->64, motion 3x3 256->128, per GRU pass z/r 5-tap 256->256 and q 5-tap 256->128, flow_head.conv1 3x3
    128->256.  convf1 (7x7 on 2 channels), flow_head.conv2 and the context shares are left out."""
    px = 2 * (T - 1) * (H // 8) * (W // 8)
    macs = 324 * 256 + 9 * 256 * 192 + 9 * 128 * 64 + 9 * 256 * 128 + 2 * (5 * 256 * 256 + 5 * 256 * 128) + 9 * 128 * 256
    return 2 * px * macs * iters


u8, fm, md = synth.make_clip(wl["T"], wl["H"], wl["W"], mask=wl["mask"], seed=0)
u8d, fmd, mdd = torch.from_numpy(u8).cuda(), fm.cuda(), md.cuda()
pipe = ProPainterPipeline(device="cuda")
cfg = InferenceConfig(raft_iter=wl["raft_iter"])


def set_mode(m):
    config.HALF_OPERANDS = m


def stages():
    frames = ops.u8_to_frames(u8d).unsqueeze(0)
    out = {}

    def timed(name, fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        r = fn()
        e1.record()
        torch.cuda.synchronize()
        out[name] = e0.elapsed_time(e1)
        return r
    with torch.no_grad():
        gt = timed("1 raft", lambda: pipe.compute_flows(frames, cfg))
        pred = timed("2 flow completion", lambda: pipe.complete_flows(gt, fmd, cfg))
        upd = timed("3 image propagation", lambda: pipe.propagate_images(frames, mdd, pred, cfg))
        timed("4 generator+composite", lambda: pipe.generate(upd[0], mdd, upd[1], pred, u8d, cfg))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        pipe(u8d, fmd, mdd, cfg)
        e1.record()
        torch.cuda.synchronize()
        out["step"] = e0.elapsed_time(e1)
    return out


for m in modes:                                            # capture + autotune every graph of both settings first
    set_mode(m)
    for _ in range(2):
        stages()
runs = {m: [] for m in modes}
for _ in range(reps):
    for m in modes:
        set_mode(m)
        runs[m].append(stages())
for m in modes:
    print(f"\nHALF_OPERANDS={m}: stage ms over {reps} reps (min / median / max)")
    for k in runs[m][0]:
        v = [r[k] for r in runs[m]]
        print(f"  {k:24s} {min(v):8.2f} {statistics.median(v):8.2f} {max(v):8.2f}")

from torch.profiler import ProfilerActivity, profile  # noqa: E402

LIB = ("cudnn", "xmma", "cutlass", "sm90", "sm80", "gemm", "conv", "implicit", "ampere", "hopper", "nchw", "nhwc", "nvjet")
HALF = ("f16", "_hsh", "h1688", "h16816")                  # fp16-operand library kernels (cuDNN convs, cuBLAS GEMMs of 1x1 convs)


def own(name):
    return name.startswith("k_") or name.startswith("void k_")


tf = refine_flops(wl["T"], wl["H"], wl["W"], wl["raft_iter"])
for m in modes:
    set_mode(m)
    frames = ops.u8_to_frames(u8d).unsqueeze(0)
    with torch.no_grad():
        gt = pipe.compute_flows(frames, cfg)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            pipe.compute_flows(frames, cfg)
            torch.cuda.synchronize()
        ka = prof.key_averages()
        lib = [e for e in ka if not own(e.key) and "convertTensor" not in e.key and any(s in e.key.lower() for s in LIB)]
        lib_us = sum(e.device_time_total for e in lib)
        h_us = sum(e.device_time_total for e in lib if any(s in e.key.lower() for s in HALF))
        own_us = sum(e.device_time_total for e in ka if own(e.key))
        all_us = sum(e.device_time_total for e in ka)
        print(f"\nHALF_OPERANDS={m}: stage 1 kernels: total {all_us / 1e3:.2f} ms, library conv/GEMM {lib_us / 1e3:.2f} ms "
              f"(fp16-operand ones {h_us / 1e3:.2f} ms), own k_* {own_us / 1e3:.2f} ms")
        print(f"  refinement-loop convs: {tf / 1e12:.2f} TFLOP; over all library conv time {tf / (lib_us * 1e-6) / 1e12:.1f} TFLOP/s "
              f"(includes the encoders' and heads' convs)" +
              (f", over the fp16-operand conv time {tf / (h_us * 1e-6) / 1e12:.1f} TFLOP/s" if h_us else "") +
              " (data sheet: 989 fp16, 495 TF32)")
        print(ka.table(sort_by="cuda_time_total", row_limit=25, max_name_column_width=90))
        pred = pipe.complete_flows(gt, fmd, cfg)
        upd = pipe.propagate_images(frames, mdd, pred, cfg)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            pipe.generate(upd[0], mdd, upd[1], pred, u8d, cfg)
            torch.cuda.synchronize()
        print(f"\nHALF_OPERANDS={m}: stage 4 kernels")
        print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=25, max_name_column_width=90))
