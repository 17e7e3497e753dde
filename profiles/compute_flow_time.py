"""Pairs per second of evaluate.compute_flow_video, the port of scripts/compute_flow.py, against the script's own schedule
run on this package's kernels: per pair, the two frames prepared on the device (ops.u8_to_frames_resized), then two
batch-1 RAFT.forward calls (forward, backward), each followed by a blocking .cpu() as the script's flowwrite needs.  The
batched arm also copies its fp16 flows to the host.  Seeded synthetic videos (synth.make_clip) resized to 432x240, 20
iterations, seeded random RAFT weights, shipping precision switches.  Both arms run in one process, alternated, after one
warm-up pass each; the median of REPEATS timed passes is reported.  Also: the time of pp_u8_to_frames_resized on one
video (CUDA events over many launches) with its bytes (uint8 input read + fp32 output written) over that time as a share
of the H100 SXM's 3.35 TB/s, and the peak device memory of compute_flow_video.

    python profiles/compute_flow_time.py [--workloads 4x36x720x1280 2x70x480x854] [--repeats 3] [OUT.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HBM_PEAK = 3.35e12                                        # bytes/s, H100 SXM data sheet


def script_schedule(raft, videos, size, iters, dev):
    """compute_flow.py:62-108 on this package's kernels: per pair, two batch-1 RAFT calls, each ending in .cpu()"""
    from propainter_b200 import ops
    for u8 in videos:
        for i in range(len(u8) - 1):
            pair = ops.u8_to_frames_resized(torch.from_numpy(u8[i:i + 2]).to(dev), size)
            _, f = raft(pair[:1], pair[1:], iters=iters, test_mode=True)
            f[0].permute(1, 2, 0).cpu()
            _, b = raft(pair[1:], pair[:1], iters=iters, test_mode=True)
            b[0].permute(1, 2, 0).cpu()


def batched(pipe, videos, size, iters):
    from propainter_b200.evaluate import compute_flow_video
    for u8 in videos:
        fw, bw = compute_flow_video(pipe, u8, size, iters)
        fw.cpu(), bw.cpu()


def timed(fn, dev):
    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize(dev)
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="*", default=["4x36x720x1280", "2x70x480x854"])
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("out", nargs="?")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("compute_flow_time: needs a CUDA device")
    import __graft_entry__
    __graft_entry__.build()
    from propainter_b200 import ops, synth
    from propainter_b200.evaluate import compute_flow_video
    from propainter_b200.inference_propainter import ProPainterPipeline
    dev = torch.device("cuda:0")
    q = lambda k: subprocess.run(["nvidia-smi", f"--query-gpu={k}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                                 text=True).stdout.strip()
    size = (432, 240)
    out = {"card": torch.cuda.get_device_name(dev), "power_limit": q("power.limit"), "sm_clock_max": q("clocks.max.sm"),
           "size": list(size), "iters": a.iters, "runs": []}
    print(json.dumps({k: out[k] for k in ("card", "power_limit", "sm_clock_max")}), flush=True)
    pipe = ProPainterPipeline(device=dev)
    raft = pipe.fix_raft.fix_raft
    for wl in a.workloads:
        n, T, H0, W0 = (int(x) for x in wl.split("x"))
        videos = [synth.make_clip(T, H0, W0, seed=s)[0] for s in range(n)]
        pairs = n * (T - 1)
        with torch.no_grad():
            batched(pipe, videos[:1], size, a.iters)                          # warm-up of every shape
            script_schedule(raft, [videos[0][:3]], size, a.iters, dev)
            t_batched, t_script = [], []
            for _ in range(a.repeats):
                t_batched.append(timed(lambda: batched(pipe, videos, size, a.iters), dev))
                t_script.append(timed(lambda: script_schedule(raft, videos, size, a.iters, dev), dev))
            torch.cuda.synchronize(dev)
            torch.cuda.reset_peak_memory_stats(dev)
            base = torch.cuda.memory_allocated(dev)
            compute_flow_video(pipe, videos[0], size, a.iters)
            torch.cuda.synchronize(dev)
            peak = torch.cuda.max_memory_allocated(dev)
            src = torch.from_numpy(videos[0]).to(dev)
            dst = ops.u8_to_frames_resized(src, size)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            launches = 200
            e0.record()
            for _ in range(launches):
                ops.u8_to_frames_resized(src, size)
            e1.record()
            torch.cuda.synchronize(dev)
            kt = e0.elapsed_time(e1) / 1e3 / launches
        nbytes = src.numel() + dst.numel() * 4
        mb, ms = float(np.median(t_batched)), float(np.median(t_script))
        r = {"workload": wl, "videos": n, "frames": T, "source": [H0, W0], "pairs": pairs,
             "batched_seconds": t_batched, "script_seconds": t_script,
             "batched_pairs_per_s": pairs / mb, "script_pairs_per_s": pairs / ms, "speedup": ms / mb,
             "peak_allocated_gib": peak / 2 ** 30, "resident_before_gib": base / 2 ** 30,
             "resize_kernel_us": kt * 1e6, "resize_kernel_bytes": nbytes, "resize_kernel_hbm_share": nbytes / kt / HBM_PEAK}
        print(json.dumps(r), flush=True)
        out["runs"].append(r)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
