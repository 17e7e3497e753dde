"""Basic vs small RAFT: ms per frame pair and peak device memory, and the radius-3 lookup kernels' share of peak.

  python profiles/raft_small_time.py [OUT.json]

One flows_bidirectional call per size (2 frames: one pair per direction), 20 iterations, seeded random weights,
warm-up 2 calls, then 5 timed calls between CUDA events around synchronised work; ms per pair = call time / 2.  Peak
memory: torch.cuda.max_memory_allocated above the inputs during one eager call.  432x240, 1280x720 and 1920x1080 run
all-pairs, 3840x2160 on the fly.  Lookup kernels at 1920x1080 (TMA, share of the HBM peak: bytes = the staged boxes,
4 levels x 8 x 12 floats, plus coords and the 196-float output per query) and at 3840x2160 (on the fly, share of the FP32
peak: FLOP = 2 x 4 levels x 64 dot products x D = 128 per query).  The card's name, power limit and SM clock are read in
the same run; the peaks are the H100 SXM data-sheet figures (3.35 TB/s, 67 TFLOP/s FP32)."""
import json
import subprocess
import sys
import os
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HBM_PEAK, FP32_PEAK = 3.35e12, 67e12


def main():
    import torch
    import __graft_entry__ as g
    g.build()
    from propainter_b200 import ops, synth
    from propainter_b200.RAFT.raft import ALL_PAIRS, ON_THE_FLY, RAFT
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    nets = {"basic": RAFT(seed=1).to(dev),
            "small": RAFT(types.SimpleNamespace(small=True, mixed_precision=False, alternate_corr=False), seed=4).to(dev)}
    ev = lambda: torch.cuda.Event(enable_timing=True)

    def timed(fn, reps):
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        a, b = ev(), ev()
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / reps

    q = lambda k: subprocess.run(["nvidia-smi", f"--query-gpu={k}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                                 text=True).stdout.strip()
    out = {"card": torch.cuda.get_device_name(dev), "power_limit": q("power.limit"), "sm_clock_max": q("clocks.max.sm"),
           "iters": 20, "pairs_per_call": 2, "timed_calls": 5, "rows": []}
    for (W, H, plan) in ((432, 240, ALL_PAIRS), (1280, 720, ALL_PAIRS), (1920, 1080, ALL_PAIRS), (3840, 2160, ON_THE_FLY)):
        u8, _, _ = synth.make_clip(2, H, W, seed=3)
        fr = (torch.from_numpy(u8).to(dev).permute(0, 3, 1, 2).float() / 127.5 - 1).contiguous()
        for name, net in nets.items():
            run = lambda: net._flows_bidirectional(fr, 20, plan)
            with torch.no_grad():
                ms = timed(run, 5 if W < 3840 else 2)
                torch.cuda.synchronize()
                torch.cuda.empty_cache()
                torch.cuda.reset_peak_memory_stats(dev)
                base = torch.cuda.memory_allocated(dev)
                run()
                torch.cuda.synchronize()
                peak = torch.cuda.max_memory_allocated(dev) - base
            out["rows"].append({"model": name, "size": f"{W}x{H}", "plan": plan, "ms_per_pair": ms / 2, "peak_bytes": peak})
            print(out["rows"][-1], flush=True)
            torch.cuda.empty_cache()
    # radius-3 lookup kernels alone
    lk = {}
    for (h, w, plan) in ((135, 240, ALL_PAIRS), (270, 480, ON_THE_FLY)):
        B, D = 2, 128
        gen = torch.Generator(device=dev).manual_seed(0)
        fmap = torch.randn(B + 1, h * w, D, device=dev, generator=gen)
        i1 = torch.arange(B, dtype=torch.int32, device=dev)
        i2 = i1 + 1
        ys, xs = torch.meshgrid(torch.arange(h, device=dev), torch.arange(w, device=dev), indexing="ij")
        coords = (torch.stack([xs, ys], -1).float()[None] + torch.randn(B, h, w, 2, device=dev, generator=gen) * 4).contiguous()
        outb = torch.empty(B, h, w, 196, device=dev)
        npix = B * h * w
        if plan == ALL_PAIRS:
            levels = ops.corr_alloc(B, h, w, dev)
            ops.corr_build(fmap, i1, i2, levels, h, w)
            ms = timed(lambda: ops.corr_lookup_r(levels, coords, 3, outb), 50)
            ms_ldg = timed(lambda: ops.corr_lookup_r(levels, coords, 3, outb, tma=False), 50)
            nbytes = npix * (4 * 8 * 12 * 4 + 8 + 196 * 4)
            lk["tma_1920x1080"] = {"ms": ms, "bytes": nbytes, "hbm_share": nbytes / (ms * 1e-3) / HBM_PEAK, "ldg_ms": ms_ldg}
            del levels
        else:
            pooled = ops.corr_fmap_pyramid(fmap, h, w)
            ms = timed(lambda: ops.corr_lookup_otf_r(fmap, pooled, i1, i2, coords, 3, outb), 5)
            flop = npix * 2 * 4 * 64 * D
            lk["otf_3840x2160"] = {"ms": ms, "flop": flop, "fp32_share": flop / (ms * 1e-3) / FP32_PEAK}
        print(lk, flush=True)
    out["lookup_kernels"] = lk
    print(json.dumps(out, indent=1))
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
