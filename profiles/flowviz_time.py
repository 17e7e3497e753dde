"""Flow colour coding and flow-completion evaluation, one JSON record (outside bench.py's line).

  python profiles/flowviz_time.py [OUT.json] [--reps R]

  kernels      k_flow_maxrad and k_flow_to_image_u8 alone, each variant ("frame": flow_viz.py, "clip": flow_viz_pt.py):
               mean us per launch over R launches (CUDA events, buffers preallocated), the bytes each must move (maxrad
               8 B/pixel read; colour pass 8 B read + 3 B written per pixel), GB/s and the share of the H100 SXM's
               3.35 TB/s HBM3 peak.  Shapes: the C2 clip's 158 flows (both directions of 80 x 240 x 432, the completed
               flows of ProPainterPipeline.flows) and a 6-flow 3840 x 2160 clip (smooth random flow).
  evaluate     evaluate_flow_clip on C2 (raft_iter 20, shipping defaults): stage-2 seconds per frame after one warm-up
               call, as evaluate_flow_completion.py measures it, and the EPE
  card         the card's name, power limit and max SM clock, read in the same run
Random-init weights, seeded synthetic frames."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HBM_PEAK = 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out", nargs="?")
    ap.add_argument("--reps", type=int, default=50)
    a = ap.parse_args()
    import torch
    import __graft_entry__ as g
    g.build()
    from propainter_b200 import _lib, ops, synth
    from propainter_b200.evaluate import evaluate_flow_clip
    from propainter_b200.inference_propainter import InferenceConfig, ProPainterPipeline
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    out = {"card": {"name": torch.cuda.get_device_name(dev), "power_limit,clocks_max_sm": q}, "reps": a.reps}

    T, H, W = 80, 240, 432
    u8, fm, _ = synth.make_clip(T, H, W, mask="ellipse", seed=0)
    pipe = ProPainterPipeline(device=dev)
    _, pred = pipe.flows(torch.from_numpy(u8), fm)
    c2 = torch.cat([pred[0][0], pred[1][0]]).contiguous()                     # [158,2,240,432]
    gen = torch.Generator(device=dev).manual_seed(0)
    k4 = torch.nn.functional.interpolate(torch.randn(6, 2, 34, 60, device=dev, generator=gen) * 20, size=(2160, 3840),
                                         mode="bilinear", align_corners=False).contiguous()

    def us(fn):
        for _ in range(3):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e3 / a.reps

    L = _lib.lib()
    st = lambda: ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    ptr = lambda t: ctypes.c_void_p(t.data_ptr())
    rows = {}
    for name, f in (("c2_158x240x432", c2), ("4k_6x2160x3840", k4)):
        N, _, h, w = f.shape
        img = torch.empty(N, h, w, 3, dtype=torch.uint8, device=dev)
        for norm, variant in ops.FLOWVIZ_NORMALIZE.items():
            per_frame = int(norm == "frame")
            mx = torch.empty(N if per_frame else 1, device=dev)
            t_max = us(lambda: L.pp_flow_maxrad(ptr(f), ptr(mx), N, h, w, per_frame, 0, ctypes.c_float(0), st()))
            t_img = us(lambda: L.pp_flow_to_image_u8(ptr(f), ptr(mx), ptr(img), N, h, w, variant, 0, ctypes.c_float(0), 0,
                                                     st()))
            assert torch.equal(img, ops.flow_to_image_u8(f, norm))
            px = N * h * w
            r = {}
            for kname, t, nbytes in (("k_flow_maxrad", t_max, 8 * px), ("k_flow_to_image_u8", t_img, 11 * px)):
                r[kname] = {"us": t, "bytes": nbytes, "gb_s": nbytes / (t * 1e-6) / 1e9,
                            "hbm_peak_fraction": nbytes / (t * 1e-6) / HBM_PEAK}
            rows[f"{name}_{norm}"] = r
    out["kernels"] = rows

    cfg = InferenceConfig(raft_iter=20)
    masks = (fm[0, :, 0] > 0).to(torch.uint8).numpy()
    evaluate_flow_clip(pipe, u8, masks, cfg=cfg)                                # warm-up: graphs, plans
    res = evaluate_flow_clip(pipe, u8, masks, cfg=cfg)
    out["evaluate_c2"] = {"stage2_seconds": res["seconds"], "stage2_seconds_per_frame": res["seconds_per_frame"],
                          "epe": res["epe"], "epe_forward": res["epe_forward"], "epe_backward": res["epe_backward"]}
    print(json.dumps(out, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
