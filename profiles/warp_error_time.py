"""Temporal warping error (E_warp) kernels, one JSON record (outside bench.py's line).

  python profiles/warp_error_time.py [OUT.json] [--reps R]

  kernels   mean us per call over R calls (CUDA events, buffers preallocated, 3 warm-up calls) of
              pp_flow_occlusion             k_flow_occlusion: reads F_t and B_t (16 B/px), writes O_t (1 B/px)
              pp_warp_error (occ given)     k_warp_error + k_warp_error_reduce: F_t (8), O_t (1), frames t and t+1 (6)
              pp_warp_error (fused)         the occlusion test in the same pass: F_t (8), B_t (8), frames t and t+1 (6)
            per pair, with bytes computed from shapes (neighbouring taps counted once, the partial sums neglected),
            GB/s and the share of the H100 SXM's 3.35 TB/s HBM3 peak.
  evaluate  evaluate.warp_error (one fused pass + the per-pair numbers to the host), synchronised wall time
  card      the card's name, power limit and max SM clock, read in the same run
Shapes: C2's 80 x 240 x 432 clip (79 pairs) and a 30-frame 1920 x 1080 clip (29 pairs); seeded random frames and smooth
random flows (bw = -fw + noise, so a good share of the pixels passes the occlusion test and is warped)."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HBM_PEAK = 3.35e12
BYTES_PER_PX = {"pp_flow_occlusion": 17, "pp_warp_error_occ": 15, "pp_warp_error_fused": 22}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out", nargs="?")
    ap.add_argument("--reps", type=int, default=50)
    a = ap.parse_args()
    import torch
    import __graft_entry__ as g
    g.build()
    from propainter_b200 import _lib, ops
    from propainter_b200.evaluate import warp_error
    if not torch.cuda.is_available():
        raise SystemExit("warp_error_time.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    out = {"card": {"name": torch.cuda.get_device_name(dev), "power_limit,clocks_max_sm": q}, "reps": a.reps}

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
    for name, (T, H, W) in (("c2_80x240x432", (80, 240, 432)), ("fhd_30x1080x1920", (30, 1080, 1920))):
        gen = torch.Generator(device=dev).manual_seed(T)
        lo = torch.rand(T, 3, H // 8, W // 8, device=dev, generator=gen) * 255
        img = torch.nn.functional.interpolate(lo, size=(H, W), mode="bilinear", align_corners=False)
        img = img + torch.randn(T, 3, H, W, device=dev, generator=gen) * 8
        frames = img.clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous()
        fw = torch.nn.functional.interpolate(torch.randn(T - 1, 2, 4, 6, device=dev, generator=gen) * W / 40, size=(H, W),
                                             mode="bilinear", align_corners=False).contiguous()
        bw = (-fw + torch.randn(fw.shape, device=dev, generator=gen) * 0.3).contiguous()
        del lo, img
        occ = torch.empty(T - 1, H, W, dtype=torch.uint8, device=dev)
        ws = torch.empty(L.pp_warp_error_workspace_bytes(T, H, W), dtype=torch.uint8, device=dev)
        res = torch.empty(T - 1, 2, dtype=torch.float64, device=dev)
        t = {"pp_flow_occlusion": us(lambda: L.pp_flow_occlusion(ptr(fw), ptr(bw), ptr(occ), T - 1, H, W, st())),
             "pp_warp_error_occ": us(lambda: L.pp_warp_error(ptr(frames), ptr(fw), None, ptr(occ), ptr(res), T, H, W, ptr(ws),
                                                             ws.numel(), st())),
             "pp_warp_error_fused": us(lambda: L.pp_warp_error(ptr(frames), ptr(fw), ptr(bw), None, ptr(res), T, H, W, ptr(ws),
                                                               ws.numel(), st()))}
        assert torch.equal(occ, ops.flow_occlusion(fw, bw))
        assert torch.equal(res, ops.warp_error_sums(frames, fw, bw=bw))
        px = (T - 1) * H * W
        r = {"pairs": T - 1, "occluded_fraction": occ.float().mean().item()}
        for k, us_k in t.items():
            nbytes = BYTES_PER_PX[k] * px
            r[k] = {"us": us_k, "us_per_pair": us_k / (T - 1), "bytes": nbytes, "bytes_per_px": BYTES_PER_PX[k],
                    "gb_s": nbytes / (us_k * 1e-6) / 1e9, "hbm_peak_fraction": nbytes / (us_k * 1e-6) / HBM_PEAK}
        warp_error(frames, (fw, bw))
        torch.cuda.synchronize()
        walls = []
        for _ in range(5):
            t0 = time.perf_counter()
            ew = warp_error(frames, (fw, bw))
            torch.cuda.synchronize()
            walls.append(time.perf_counter() - t0)
        r["evaluate_warp_error_ms_median"] = sorted(walls)[2] * 1e3
        r["ewarp"] = ew["ewarp"]
        rows[name] = r
        del frames, fw, bw, occ, ws
        torch.cuda.empty_cache()
    out["kernels"] = rows
    print(json.dumps(out, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
