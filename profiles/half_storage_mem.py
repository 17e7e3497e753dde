"""Device memory and clip time of the pipeline with fp32 and half-precision clip storage (InferenceConfig.half_storage).

usage: python profiles/half_storage_mem.py [reps] > half_storage_mem.txt

One run prints the card's name and power limit, then for 432x240 (120 and 200 frames, subvideo_length 40, raft_clip_frames
12) and 1920x1080 (30 and 40 frames, subvideo_length 10, raft_clip_frames 4), raft_iter 2:
- the growth of torch.cuda.max_memory_allocated over one call (inputs already on the device, CUDA graphs off so no
  captured pool is counted), in both modes;
- the per-frame slope between the two clip lengths and the clip length that slope puts at the card's total memory
  (an extrapolation: the out-of-memory point is not searched for).  The two lengths of a size have the same RAFT chunk
  and the same largest flow-completion and propagation sub-video, so the slope is the clip-resident bytes per frame alone
  (with the default raft_clip_frames RAFT takes as many frames per call as an 8 GB pyramid allows, and its workspace
  would grow with the clip);
- the warm clip time (CUDA events, default switches and InferenceConfig, raft_iter 20) of 1920x1080 x 20 and
  432x240 x 80, the two modes alternated `reps` times.
Seeded synthetic weights and clips."""
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as g  # noqa: E402

g.build()
from propainter_b200 import config, synth  # noqa: E402
from propainter_b200.inference_propainter import InferenceConfig, ProPainterPipeline  # noqa: E402

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
except OSError:
    card = "nvidia-smi unavailable"
total = torch.cuda.get_device_properties(0).total_memory
print("card:", card, "|", torch.cuda.get_device_name(0), f"| {total / 2**30:.1f} GiB")

SIZES = [((240, 432), (120, 200), 40, 12), ((1080, 1920), (30, 40), 10, 4)]
TIMED = [((1080, 1920), 20), ((240, 432), 80)]
MODES = (False, True)
pipe = ProPainterPipeline(device="cuda")


def clip(T, H, W):
    u8, fm, md = synth.make_clip(T, H, W, mask="ellipse", seed=0)
    return torch.from_numpy(u8).cuda(), fm.cuda(), md.cuda()


def growth(inputs, half, sub, clip_frames):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    with torch.no_grad():
        out = pipe(*inputs, InferenceConfig(raft_iter=2, subvideo_length=sub, raft_clip_frames=clip_frames,
                                              half_storage=half))
    torch.cuda.synchronize()
    del out
    return torch.cuda.max_memory_allocated() - base


def timed(inputs, half):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.no_grad():
        e0.record()
        out = pipe(*inputs, InferenceConfig(half_storage=half))
        e1.record()
    torch.cuda.synchronize()
    del out
    return e0.elapsed_time(e1)


print("\n== peak growth of max_memory_allocated over one call (CUDA graphs off)")
print(f"{'size':>10} {'frames':>6} {'fp32 MiB':>10} {'half MiB':>10} {'ratio':>6}")
graphs = config.CUDA_GRAPHS
config.CUDA_GRAPHS = False
slopes = {}
for (H, W), lengths, sub, clip_frames in SIZES:
    peaks = {}
    for T in lengths:
        inputs = clip(T, H, W)
        for half in MODES:
            growth(inputs, half, sub, clip_frames)                 # lazy weight packing, cuDNN / plan selection
        peaks[T] = {half: growth(inputs, half, sub, clip_frames) for half in MODES}
        print(f"{W}x{H:<5} {T:>6} {peaks[T][False] / 2**20:>10.0f} {peaks[T][True] / 2**20:>10.0f} "
              f"{peaks[T][True] / peaks[T][False]:>6.3f}")
        del inputs
        torch.cuda.empty_cache()
    a, b = lengths
    slopes[(H, W)] = {half: ((peaks[b][half] - peaks[a][half]) / (b - a), peaks[a][half]) for half in MODES}
config.CUDA_GRAPHS = graphs

print("\n== per-frame slope between the two lengths, and the clip length it extrapolates to at the card's memory")
for (H, W), (a, _), _, _ in SIZES:
    row = []
    for half in MODES:
        s, pa = slopes[(H, W)][half]
        inp = 11 * H * W                                           # uint8 frames + two fp32 masks, resident before the call
        cap = a + (total - torch.cuda.memory_allocated() - pa - inp * a) / (s + inp)
        row.append(f"{'half' if half else 'fp32'}: {s / 2**20:.1f} MiB/frame ({s / (H * W):.1f} B/px), ~{cap:.0f} frames")
    print(f"{W}x{H}: " + " | ".join(row))

print(f"\n== clip time, ms (CUDA events, modes alternated, {reps} reps, CUDA graphs {'on' if config.CUDA_GRAPHS else 'off'})")
for (H, W), T in TIMED:
    inputs = clip(T, H, W)
    for half in MODES:
        timed(inputs, half)                                        # warm-up (graph capture, plan selection)
    ts = {half: [] for half in MODES}
    for _ in range(reps):
        for half in MODES:
            ts[half].append(timed(inputs, half))
    print(f"{W}x{H} x {T}: " + " | ".join(
        f"{'half' if half else 'fp32'} median {statistics.median(v):.1f} (min {min(v):.1f}, max {max(v):.1f})"
        for half, v in ts.items()))
    del inputs
    torch.cuda.empty_cache()
