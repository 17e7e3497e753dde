"""Seconds per frame and peak device memory of evaluate.evaluate_video, the evaluation script's video-completion protocol
(scripts/evaluate_propainter.py::main_worker), on DAVIS-shaped synthetic clips: 432x240 (the script's default size),
neighbor_length 20, ref_stride 10, raft_iter 20, with loaded flows (--load_flow, how the published numbers were made) and
with RAFT in 60-frame chunks.  Seeded random weights, shipping precision switches.  `seconds` is the script's timer
(synchronised, upload excluded); each configuration runs once to warm up and REPEATS times timed.  Whole-clip flow
completion and propagation grow linearly with T, so the peak is reported per clip length measured, never extrapolated.

    python profiles/eval_protocol_time.py [--frames 70 90] [--repeats 3] [OUT.json]     (JSON lines on stdout; the whole
    result also to OUT.json when given)"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, nargs="*", default=[70, 90])
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("out", nargs="?")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eval_protocol_time: needs a CUDA device")
    import __graft_entry__
    __graft_entry__.build()
    from propainter_b200 import ops, synth
    from propainter_b200.evaluate import evaluate_video
    from propainter_b200.inference_propainter import ProPainterPipeline
    dev = torch.device("cuda:0")
    q = lambda k: subprocess.run(["nvidia-smi", f"--query-gpu={k}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                                 text=True).stdout.strip()
    out = {"card": torch.cuda.get_device_name(dev), "power_limit": q("power.limit"), "sm_clock_max": q("clocks.max.sm"),
           "size": [432, 240], "neighbor_length": 20, "ref_stride": 10, "raft_iter": 20, "runs": []}
    pipe = ProPainterPipeline(device=dev)
    for T in a.frames:
        u8, fm, _ = synth.make_clip(T, 240, 432, mask="ellipse", seed=0)
        fr = torch.from_numpy(u8).to(dev)
        mk = ops.mask_dilate((fm[0, :, 0] > 0).to(torch.uint8).to(dev), 4).unsqueeze(0)
        rng = np.random.default_rng(T)
        loaded = tuple(torch.from_numpy((rng.standard_normal((T - 1, 2, 240, 432)) * 2).astype(np.float32)).to(dev)
                       for _ in range(2))
        for mode, flows in (("loaded_flows", loaded), ("raft_60", None)):
            evaluate_video(pipe, fr, mk, flows, task="object_removal")            # warm-up of every shape
            torch.cuda.synchronize(dev)
            torch.cuda.reset_peak_memory_stats(dev)
            base = torch.cuda.memory_allocated(dev)
            secs = [evaluate_video(pipe, fr, mk, flows, task="object_removal")["seconds"] for _ in range(a.repeats)]
            peak = torch.cuda.max_memory_allocated(dev)
            r = {"frames": T, "mode": mode, "seconds": secs, "seconds_per_frame_median": float(np.median(secs)) / T,
                 "peak_allocated_gib": peak / 2 ** 30, "resident_before_gib": base / 2 ** 30}
            print(json.dumps(r), flush=True)
            out["runs"].append(r)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps({k: out[k] for k in ("card", "power_limit", "sm_clock_max")}))


if __name__ == "__main__":
    main()
