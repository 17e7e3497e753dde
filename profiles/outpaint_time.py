"""Video outpainting on the C2 clip, one JSON record (outside bench.py's line).

  python profiles/outpaint_time.py [OUT.json] [--steps K] [--warmup W]

  outpaint_1.0x1.2   ProPainterPipeline.outpaint of the C2 source (80 x 240 x 432, raft_iter 20) at the script's default
                     scale: a 240 x 512 canvas.  frames/s from CUDA events over K whole calls after W warm-up calls, with
                     the uint8 source resident on the device; peak memory (max_memory_allocated) over the timed calls.
  outpaint_1.2x1.2   the same at (1.2, 1.2): a 288 x 512 canvas
  inpaint_c2         C2 inpainting (bench.py's workload, ellipse mask) timed the same way in the same run, for comparison
  front_end          k_extrapolate_u8 (default scale) and k_mask_overlay_u8 (on its canvas) alone: mean us per launch
                     over 50 launches, and the bytes each must move over that time
  card               the card's name, power limit and max SM clock, read in the same run
Random-init weights, seeded synthetic frames, shipping defaults."""
import argparse
import gc
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out", nargs="?")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import torch
    import __graft_entry__ as g
    g.build()
    from propainter_b200 import ops, synth
    from propainter_b200.inference_propainter import InferenceConfig, ProPainterPipeline, outpaint_geometry
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    out = {"card": {"name": torch.cuda.get_device_name(dev), "power_limit,clocks_max_sm": q},
           "steps": a.steps, "warmup": a.warmup, "raft_iter": 20}
    T, H, W = 80, 240, 432
    u8_np, fm, md = synth.make_clip(T, H, W, mask="ellipse", seed=0)
    u8 = torch.from_numpy(u8_np).to(dev)
    fm, md = fm.to(dev), md.to(dev)
    cfg = InferenceConfig(raft_iter=20)

    def fresh():
        """a new pipeline (same seeded weights) per arm: each frame size captures its own CUDA graphs, whose memory pools
        stay with the pipeline object, so one object over three sizes would also measure the graphs of the others"""
        gc.collect()
        torch.cuda.empty_cache()
        return ProPainterPipeline(device=dev)

    def timed(fn):
        for _ in range(a.warmup):
            fn()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.steps):
            res = fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / a.steps
        return res, {"ms_per_clip": ms, "frames_per_s": T / (ms * 1e-3),
                     "peak_mem_gb": torch.cuda.max_memory_allocated(dev) / 1e9}

    for sh, sw in ((1.0, 1.2), (1.2, 1.2)):
        pipe = fresh()
        comp, row = timed(lambda: pipe.outpaint(u8, sh, sw, cfg))
        row["canvas"] = list(comp.shape[1:3])
        out[f"outpaint_{sh}x{sw}"] = row
        del pipe, comp
    pipe = fresh()
    _, out["inpaint_c2"] = timed(lambda: pipe(u8, fm, md, cfg))
    del pipe

    geo = outpaint_geometry(H, W, 1.0, 1.2)
    canvas, _, mdo = ops.extrapolate_u8(u8, geo)
    n_canvas = canvas.numel() // 3

    def kernel_us(fn, reps=50):
        for _ in range(3):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e3 / reps

    fe = {}
    for name, fn, nbytes in (("k_extrapolate_u8", lambda: ops.extrapolate_u8(u8, geo), u8.numel() + n_canvas * (3 + 8)),
                             ("k_mask_overlay_u8", lambda: ops.mask_overlay_u8(canvas, mdo), n_canvas * (3 + 4 + 3))):
        us = kernel_us(fn)
        fe[name] = {"us_per_launch": us, "bytes": nbytes, "gb_s": nbytes / (us * 1e-6) / 1e9}
    out["front_end"] = fe
    print(json.dumps(out, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
