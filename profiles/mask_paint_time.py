"""The tracking preview on the device: ops.mask_paint_u8 (k_mask_paint_partial + k_mask_paint_maxima + k_mask_paint_u8)
alone, and MaskTracker.track with return_painted against track alone.

  python profiles/mask_paint_time.py [OUT.json]

Clips: 40 frames from tests/cutie_inputs.make_clip at 854x480 and 1920x1080, 1 and 3 objects (the templates of
profiles/cutie_time.py), tracked once by MaskTracker (CUTIE(seed=4), shipping precision); the painter then runs on those
labels.  Painter: the three kernels through the C entry point with preallocated buffers (kernels_*), and the ops
wrapper with its argument checks and allocations (op_*), 5 warm-up + 50 timed calls between CUDA events each, median
and minimum per call.  Bytes moved: what the painting needs, 7 B per pixel (frame 3 + labels 1 in, 3 out; the labels'
3-pixel tile halo and the per-frame maxima are not counted), over the median kernel time.  A 1920x1080 clip of random labels 0..3
(every pixel near a boundary, so pass 1 reduces the per-object maxima over the whole frame) is timed the same way.
The share of peak is kernel time against the least time the bytes need at 3.35 TB/s (memory is the bound that applies).
Tracking: track and track(return_painted=True) on the same clip, alternating, 3 timed runs each after one warm-up, the
median per clip and the difference.  The card's name, power limit and max SM clock are read in the same run."""
import ctypes
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(1, os.path.join(ROOT, "tests"))

HBM_PEAK = 3.35e12
BYTES_PER_PX = 7


def main():
    import numpy as np
    import torch
    import __graft_entry__ as g
    g.build()
    from cutie_inputs import make_clip
    from propainter_b200 import _lib, ops
    from propainter_b200.model.cutie import CUTIE
    from propainter_b200.tracker import MaskTracker
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    ev = lambda: torch.cuda.Event(enable_timing=True)
    q = lambda k: subprocess.run(["nvidia-smi", f"--query-gpu={k}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                                 text=True).stdout.strip()
    out = {"card": torch.cuda.get_device_name(dev), "power_limit": q("power.limit"), "max_sm_clock": q("clocks.max.sm"),
           "painter": [], "tracking": []}

    def time_calls(fn, warm=5, n=50):
        for _ in range(warm):
            fn()
        ts = []
        for _ in range(n):
            a, b = ev(), ev()
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        return statistics.median(ts), min(ts)

    L = _lib.lib()

    def painter(name, fr, lab):
        T, H, W = lab.shape
        pal = torch.from_numpy(ops.paint_palette()).to(dev)
        img = torch.empty_like(fr)
        ws = torch.empty(L.pp_mask_paint_workspace_bytes(T, H, W), dtype=torch.uint8, device=dev)
        ptr = lambda t: ctypes.c_void_p(t.data_ptr())
        alpha = (ctypes.c_double * 2)(0.7, 1 - 0.7)
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        kernels = lambda: L.pp_mask_paint_u8(ptr(fr), ptr(lab), ptr(pal), 257, alpha, ptr(img), T, H, W, ptr(ws), ws.numel(),
                                             stream)
        med, mn = time_calls(kernels)
        op_med, _ = time_calls(lambda: ops.mask_paint_u8(fr, lab))
        assert torch.equal(img, ops.mask_paint_u8(fr, lab))
        nbytes = BYTES_PER_PX * T * H * W
        r = {"case": name, "frames": T, "size": f"{W}x{H}", "kernels_ms_median": round(med, 4), "kernels_ms_min": round(mn, 4),
             "op_ms_median": round(op_med, 4), "GB_per_s": round(nbytes / (med * 1e-3) / 1e9, 1),
             "share_of_hbm_peak": round(nbytes / (med * 1e-3) / HBM_PEAK, 3)}
        out["painter"].append(r)
        print(r, flush=True)

    tr = MaskTracker(CUTIE(seed=4), dev)
    T = 40
    for H, W in ((480, 854), (1080, 1920)):
        frames, masks = make_clip(T, H, W, 1)
        fr = torch.from_numpy(frames).to(dev)
        for nobj in (1, 3):
            tmpl = masks[0].copy()
            if nobj == 1:
                tmpl[tmpl == 2] = 0
            else:
                ys, xs = np.nonzero(masks[0] == 2)
                tmpl[np.clip(ys - H // 4, 0, H - 1), np.clip(xs - W // 3, 0, W - 1)] = 3
            lab = tr.track(fr, tmpl)
            torch.cuda.synchronize()
            painter(f"tracked, {nobj} object(s)", fr, lab)
            times = {"track": [], "track_painted": []}
            fns = {"track": lambda: tr.track(fr, tmpl), "track_painted": lambda: tr.track(fr, tmpl, return_painted=True)}
            for _ in range(4):
                for name, fn in fns.items():
                    a, b = ev(), ev()
                    a.record()
                    fn()
                    b.record()
                    torch.cuda.synchronize()
                    times[name].append(a.elapsed_time(b))
            med = {k: statistics.median(v[1:]) for k, v in times.items()}
            r = {"size": f"{W}x{H}", "objects": nobj, "frames": T, "track_ms": round(med["track"], 2),
                 "track_painted_ms": round(med["track_painted"], 2),
                 "painted_extra_ms": round(med["track_painted"] - med["track"], 2)}
            out["tracking"].append(r)
            print(r, flush=True)
        del fr
    gen = torch.Generator(device=dev).manual_seed(0)
    lab = torch.randint(0, 4, (T, 1080, 1920), generator=gen, device=dev, dtype=torch.uint8)
    fr = torch.randint(0, 256, (T, 1080, 1920, 3), generator=gen, device=dev, dtype=torch.uint8)
    painter("random labels 0..3", fr, lab)
    print(json.dumps(out, indent=1))
    if len(sys.argv) > 1:
        os.makedirs(os.path.dirname(os.path.abspath(sys.argv[1])), exist_ok=True)
        with open(sys.argv[1], "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
