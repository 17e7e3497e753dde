"""The Cutie mask tracker on the device: per-frame tracking time and peak memory, and the fused top-k readout against the
reference's dense memory read on the same inputs.

  python profiles/cutie_time.py [OUT.json]

Seeded random weights (CUTIE(seed=4)), shipping precision (cuDNN TF32 as torch defaults it).  Tracking: 40-frame clips from
tests/cutie_inputs.make_clip at 854x480 and 1920x1080 with 1 and 3 objects (ids 1..3; the third object is the second's
square shifted), through MaskTracker.track; per-frame time = (one timed clip between CUDA events) / frames after one
warm-up clip, peak memory = torch.cuda.max_memory_allocated above the clip's inputs during the timed clip.  Readout: working
memory full (1 permanent + 4 FIFO frames, N = 5 HW), 2 objects, random keys / values at HW = 30x54 (854x480) and
68x120 (1920x1080); ops.cutie_topk_readout vs oracle.cutie_ref.memory_read (get_similarity + do_softmax(top_k=30) +
the dense bmm, fp32, what MemoryManager.read runs), 3 warm-up + 20 timed calls each between CUDA events, alternating.
The card's name and power limit are read in the same run."""
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(1, os.path.join(ROOT, "tests"))


def main():
    import numpy as np
    import torch
    import __graft_entry__ as g
    g.build()
    from cutie_inputs import make_clip
    from oracle import cutie_ref
    from propainter_b200 import ops
    from propainter_b200.model.cutie import CUTIE
    from propainter_b200.tracker import MaskTracker
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    ev = lambda: torch.cuda.Event(enable_timing=True)
    q = lambda k: subprocess.run(["nvidia-smi", f"--query-gpu={k}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                                 text=True).stdout.strip()
    out = {"card": torch.cuda.get_device_name(dev), "power_limit": q("power.limit"), "tracking": [], "readout": []}
    tr = MaskTracker(CUTIE(seed=4), dev)
    T = 40
    for H, W in ((480, 854), (1080, 1920)):
        frames, masks = make_clip(T, H, W, 1)
        for nobj in (1, 3):
            tmpl = masks[0].copy()
            if nobj == 1:
                tmpl[tmpl == 2] = 0
            else:
                ys, xs = np.nonzero(masks[0] == 2)
                tmpl[np.clip(ys - H // 4, 0, H - 1), np.clip(xs - W // 3, 0, W - 1)] = 3
            fr = torch.from_numpy(frames).to(dev)
            tr.track(fr, tmpl)
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            a, b = ev(), ev()
            a.record()
            tr.track(fr, tmpl)
            b.record()
            torch.cuda.synchronize()
            ms = a.elapsed_time(b) / T
            peak = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
            out["tracking"].append({"size": f"{W}x{H}", "objects": nobj, "ms_per_frame": round(ms, 3), "peak_mib": round(peak, 1)})
            print(out["tracking"][-1], flush=True)
            del fr
    for h, w in ((30, 54), (68, 120)):
        HW, nf, K = h * w, 5, 2
        gen = torch.Generator(device=dev).manual_seed(0)
        keys = torch.randn(nf * HW, 64, device=dev, generator=gen) * 0.5
        shrink = 1 + torch.randn(nf * HW, device=dev, generator=gen) ** 2 * 0.1
        values = torch.randn(K, nf * HW, 256, device=dev, generator=gen)
        qk = torch.randn(64, HW, device=dev, generator=gen) * 0.5
        qe = torch.rand(64, HW, device=dev, generator=gen)
        mk, ms_, mv = keys.t()[None].contiguous(), shrink[None, None], values.transpose(1, 2)[None].contiguous()
        fused = lambda: ops.cutie_topk_readout(keys, shrink, values, nf, 0, nf - 1, qk, qe, 30)
        dense = lambda: cutie_ref.memory_read(mk, ms_, qk[None], qe[None], mv, 30)
        times = {"fused": [], "dense": []}
        for _ in range(3):
            fused(), dense()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        peaks = {}
        for name, fn in (("fused", fused), ("dense", dense)):
            torch.cuda.reset_peak_memory_stats()
            fn()
            torch.cuda.synchronize()
            peaks[name] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
        for _ in range(20):
            for name, fn in (("fused", fused), ("dense", dense)):
                a, b = ev(), ev()
                a.record()
                fn()
                b.record()
                torch.cuda.synchronize()
                times[name].append(a.elapsed_time(b))
        err = (fused().permute(0, 2, 1) - dense()[0]).abs().max().item()
        r = {"HW": HW, "N": nf * HW, "objects": K, "max_abs_diff": err}
        for name in times:
            r[f"{name}_ms_median"] = round(statistics.median(times[name]), 4)
            r[f"{name}_ms_min"] = round(min(times[name]), 4)
            r[f"{name}_peak_mib"] = peaks[name]
        out["readout"].append(r)
        print(r, flush=True)
    print(json.dumps(out, indent=1))
    if len(sys.argv) > 1:
        os.makedirs(os.path.dirname(os.path.abspath(sys.argv[1])), exist_ok=True)
        with open(sys.argv[1], "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
