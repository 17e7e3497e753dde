"""I3D feature extraction (VFID) on the device: time per call, peak memory, the cuDNN / own-kernel split and the max-pool
kernel's share of the HBM peak.

  python profiles/i3d_time.py [OUT.json]

Seeded random weights (InceptionI3d(seed=5)), shipping precision (cuDNN TF32).  Workloads: C2's real and composited
videos as one B=2 call (two 80x240x432 clips from synth.make_clip, seeds 0 and 1) and one 50-frame 1280x720 video (B=1),
both through evaluate.i3d_activations (uint8 frames on the device -> float32 numpy features, including that copy).
Each: 2 warm-up calls, then 7 calls timed one by one between CUDA events -> min / median / max ms.  Peak memory:
torch.cuda.max_memory_allocated above the inputs during one call.  Split: one more C2 call under torch.profiler (a run of
its own), CUDA kernel time summed by name, own kernels (k_*) vs the rest (cuDNN convolutions and their helpers).
k_maxpool3d_same alone at three C2 (B=2) layers, 50 launches each: bytes = input read once + output written once
(4 bytes per element, from the shapes), over the H100 SXM data-sheet 3.35 TB/s.  The card's name, power limit and SM
clock are read in the same run."""
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HBM_PEAK = 3.35e12


def main():
    import numpy as np
    import torch
    import __graft_entry__ as g
    g.build()
    from propainter_b200 import ops, synth
    from propainter_b200.evaluate import i3d_activations
    from propainter_b200.model.i3d import InceptionI3d
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    net = InceptionI3d(seed=5).to(dev)
    ev = lambda: torch.cuda.Event(enable_timing=True)
    q = lambda k: subprocess.run(["nvidia-smi", f"--query-gpu={k}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                                 text=True).stdout.strip()
    out = {"card": torch.cuda.get_device_name(dev), "power_limit": q("power.limit"), "sm_clock_max": q("clocks.max.sm"),
           "cudnn_allow_tf32": torch.backends.cudnn.allow_tf32, "timed_calls": 7, "rows": []}
    print(out, flush=True)

    c2 = [synth.make_clip(80, 240, 432, mask="ellipse", seed=s)[0] for s in (0, 1)]
    rng = np.random.default_rng(0)
    workloads = {"C2 real+comp 80x240x432 B=2": torch.from_numpy(np.stack(c2)).to(dev),
                 "50x1280x720 B=1": torch.from_numpy(rng.integers(0, 256, (1, 50, 720, 1280, 3), dtype=np.uint8)).to(dev)}
    for name, video in workloads.items():
        run = lambda: i3d_activations(net, video)
        for _ in range(2):
            run()
        torch.cuda.synchronize()
        ms = []
        for _ in range(out["timed_calls"]):
            a, b = ev(), ev()
            a.record()
            run()
            b.record()
            torch.cuda.synchronize()
            ms.append(a.elapsed_time(b))
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        run()
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated(dev) - base
        B, T, H, W, _ = video.shape
        row = {"workload": name, "ms_min": min(ms), "ms_median": statistics.median(ms), "ms_max": max(ms),
               "ms_per_video": statistics.median(ms) / B, "peak_bytes": peak, "frames": B * T}
        out["rows"].append(row)
        print(row, flush=True)

    # kernel-time split of one C2 call
    video = workloads["C2 real+comp 80x240x432 B=2"]
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        i3d_activations(net, video)
        torch.cuda.synchronize()
    per = {}
    for e in prof.events():
        if e.device_type.name == "CUDA" and e.device_time_total > 0:
            per[e.name] = per.get(e.name, 0.0) + e.device_time_total / 1e3
    own = {k: v for k, v in per.items() if k.startswith("k_") or k.startswith("void k_")}
    total = sum(per.values())
    out["split_c2_ms"] = {"total_kernel_ms": total, "own_kernels_ms": sum(own.values()),
                          "library_ms": total - sum(own.values()),
                          "own": {k: round(v, 3) for k, v in sorted(own.items(), key=lambda kv: -kv[1])}}
    out["split_c2_ms"]["top_library"] = dict(sorted(((k[:90], round(v, 3)) for k, v in per.items() if k not in own),
                                                    key=lambda kv: -kv[1])[:8])
    print(out["split_c2_ms"], flush=True)

    # k_maxpool3d_same alone at C2 layers (B=2): (T, H, W, C), kernel, stride
    layers = {"MaxPool3d_2a_3x3": ((40, 120, 216, 64), (1, 3, 3), (1, 2, 2)),
              "Mixed_3b.b3a": ((40, 30, 54, 192), (3, 3, 3), (1, 1, 1)),
              "MaxPool3d_4a_3x3": ((40, 30, 54, 480), (3, 3, 3), (2, 2, 2))}
    mp = {}
    for lname, ((T, H, W, C), k, s) in layers.items():
        x = torch.randn(2, T, H, W, C, device=dev)
        o = ops.maxpool3d_same(x, k, s)
        for _ in range(3):
            ops.maxpool3d_same(x, k, s, out=o)
        torch.cuda.synchronize()
        a, b = ev(), ev()
        a.record()
        for _ in range(50):
            ops.maxpool3d_same(x, k, s, out=o)
        b.record()
        torch.cuda.synchronize()
        t = a.elapsed_time(b) / 50
        nbytes = (x.numel() + o.numel()) * 4
        mp[lname] = {"ms": t, "bytes": nbytes, "GB_per_s": nbytes / (t * 1e-3) / 1e9, "hbm_share": nbytes / (t * 1e-3) / HBM_PEAK}
        print(lname, mp[lname], flush=True)
        del x, o
    out["maxpool"] = mp
    print(json.dumps(out, indent=1))
    if len(sys.argv) > 1:
        os.makedirs(os.path.dirname(os.path.abspath(sys.argv[1])), exist_ok=True)
        with open(sys.argv[1], "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
