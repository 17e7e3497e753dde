"""RAFT's two correlation plans on each side of the plan rule (propainter_b200/RAFT/raft.py corr_plan), one JSON record.

  python profiles/raft_large.py [OUT.json]

  corr_otf    k_corr_lookup_otf timed live (CUDA events, L2 flushed) at the C2 shape (158 pairs of 30x54, next to the
              all-pairs lookup bench.py times) and on one 3840x2160 pair: algorithmic FLOP and bytes from shapes, share
              of the FP32 peak (the kernel is fp32 FFMA, L1-throughput limited)
  1280x720 / 1920x1080
              both plans on one 2-frame RAFT call (one pair per direction, 20 iterations, eager): ms per pair and peak
              memory above the inputs -- the crossover, at sizes where both fit
  3840x2160_8f
              RAFT_bi over an 8-frame 3840x2160 synthetic clip, plan chosen by size: frames/s and max_memory_allocated
  card        the card's name, power limit and max SM clock, read in the same run
Random-init weights, seeded synthetic frames."""
import gc
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FP32_PEAK_TFLOPS = 67.0     # H100 SXM data sheet, dense FP32 (non-tensor) at up to 700 W


def time_kernel(torch, fn, reps=10):
    """mean ms over `reps` launches, CUDA events, L2 flushed before each"""
    flush = torch.empty(64 * 1024 * 1024, device="cuda")
    for _ in range(3):
        fn()
    ts = []
    for _ in range(reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return statistics.mean(ts)


def corr_otf_probe(torch, dev, n_frames, bidirectional, h, w):
    """one lookup of every pair of n_frames random-feature frames on an h x w grid, pairs i -> i+1 (and back).
    FLOP: 4 levels x 100 dot products x 256 x 2 per query pixel; L1 bytes: the 400 KB of f2 each query reads;
    HBM bytes: fmap + pooled levels read once, the 324-channel output written."""
    from propainter_b200 import ops
    fmap = torch.randn(n_frames, h * w, 256, device=dev)
    a = torch.arange(n_frames - 1, device=dev, dtype=torch.int32)
    i1, i2 = (torch.cat([a, a + 1]), torch.cat([a + 1, a])) if bidirectional else (a, a + 1)
    B = i1.numel()
    ys, xs = torch.meshgrid(torch.arange(h, device=dev), torch.arange(w, device=dev), indexing="ij")
    coords = (torch.stack([xs, ys], -1).float()[None] + torch.randn(B, h, w, 2, device=dev) * 3).contiguous()
    pooled = ops.corr_fmap_pyramid(fmap, h, w)
    out = torch.empty(B, h, w, 324, device=dev)
    ms = time_kernel(torch, lambda: ops.corr_lookup_otf(fmap, pooled, i1, i2, coords, out))
    q = B * h * w
    flops = q * 4 * 100 * 256 * 2
    hbm_bytes = 4 * (fmap.numel() + sum(p.numel() for p in pooled) + q * 326)
    ach = flops / (ms * 1e-3) / 1e12
    return {"kernel": "k_corr_lookup_otf", "shape": f"{B} pairs x {h}x{w}", "bound": "fp32 FFMA (L1-throughput limited)",
            "achieved_tflops": ach, "peak_tflops": FP32_PEAK_TFLOPS, "frac": ach / FP32_PEAK_TFLOPS, "launch_ms": ms,
            "algorithmic_flops": flops, "l1_bytes": q * 4 * 100 * 256 * 4, "hbm_bytes": hbm_bytes,
            "hbm_gb_s": hbm_bytes / (ms * 1e-3) / 1e9}


def main(iters=20):
    import torch
    import __graft_entry__ as g
    g.build()
    from propainter_b200 import synth
    from propainter_b200.model.modules.flow_comp_raft import RAFT_bi
    from propainter_b200.RAFT.raft import ALL_PAIRS, ON_THE_FLY
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    out = {"card": {"name": torch.cuda.get_device_name(dev), "power_limit,clocks_max_sm": q}, "iters": iters}
    otf = corr_otf_probe(torch, dev, 80, True, 240 // 8, 432 // 8)
    otf["uhd_pair"] = corr_otf_probe(torch, dev, 2, False, 270, 480)
    out["corr_otf"] = otf
    gc.collect()
    torch.cuda.empty_cache()

    net = RAFT_bi(None, dev, seed=1)
    raft = net.fix_raft

    def run(fn, reps):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps, (torch.cuda.max_memory_allocated(dev) - base) / 1e9

    def frames(T, H, W):
        u8, _, _ = synth.make_clip(T, H, W, seed=3)
        return (torch.from_numpy(u8).to(dev).permute(0, 3, 1, 2).float() / 127.5 - 1).contiguous()

    for H, W in ((720, 1280), (1080, 1920)):
        fr = frames(2, H, W)
        row = {}
        for plan in (ALL_PAIRS, ON_THE_FLY):
            call = lambda: raft._flows_bidirectional(fr, iters, plan)          # eager, the same for both plans
            run(call, 1)
            ms, peak = run(call, 3)
            row[plan] = {"ms_per_pair": ms / 2, "peak_mem_gb": peak}
        out[f"{W}x{H}"] = row
        del fr
        gc.collect()
        torch.cuda.empty_cache()
    fr = frames(8, 2160, 3840)[None]
    plan = raft.corr_plan(2160, 3840, dev)
    net(fr, iters=iters)
    ms, _ = run(lambda: net(fr, iters=iters), 1)
    out["3840x2160_8f"] = {"plan": plan, "frames_per_s": 8 / (ms * 1e-3), "ms_per_clip": ms,
                           "max_memory_allocated_gb": torch.cuda.max_memory_allocated(dev) / 1e9}
    print(json.dumps(out, indent=1))
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
