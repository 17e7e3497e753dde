"""Time pp_instance_norm of two builds of the library on the same call: the fnet conv1 norm (in place, + ReLU) and a
residual-block norm (+ residual + ReLU) at the C2 clip (80 frames of 240 x 432: 120 x 216 x 64 maps) and at 720p (2
frames: 360 x 640 x 64).  The builds alternate, so both see the same clocks and neighbours.

    python profiles/inorm_time.py --before /path/to/old/libpropainter_b200.so [--after this tree's library]

Prints the card's name and power limit, then one line per shape: median ms of each build and their ratio."""
import argparse
import ctypes
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def load(path):
    from propainter_b200._lib import SIGNATURES
    lib = ctypes.CDLL(path)
    for name in ("pp_instance_norm_workspace_bytes", "pp_instance_norm"):
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = SIGNATURES[name]
    return lib


def call(lib, x, res, ws, n, HW, C, stream):
    r = lib.pp_instance_norm(x.data_ptr(), res.data_ptr() if res is not None else None, x.data_ptr(), n, HW, C,
                             ctypes.c_float(1e-5), 1, int(res is not None), ws.data_ptr(), ws.numel(), stream)
    assert r == 0, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--before", required=True)
    ap.add_argument("--after", default=os.path.join(ROOT, "propainter_b200", "libpropainter_b200.so"))
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=7)
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print("card:", q.stdout.strip())
    libs = {"before": load(a.before), "after": load(a.after)}
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    for label, n, H, W, C in (("C2 fnet 80x120x216x64", 80, 120, 216, 64), ("720p fnet 2x360x640x64", 2, 360, 640, 64)):
        HW = H * W
        gen = torch.Generator(device="cuda").manual_seed(0)
        x0 = torch.randn(n, HW, C, generator=gen, device="cuda") + 3
        res = torch.randn(n, HW, C, generator=gen, device="cuda")
        nb = max(lib.pp_instance_norm_workspace_bytes(n, HW, C) for lib in libs.values())
        ws = torch.empty(nb, dtype=torch.uint8, device="cuda")
        x = x0.clone()
        for r in (None, res):
            times = {k: [] for k in libs}
            for k, lib in libs.items():                                   # warm-up
                call(lib, x, r, ws, n, HW, C, stream)
            for _ in range(a.rounds):
                for k, lib in libs.items():
                    x.copy_(x0)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(a.reps):
                        call(lib, x, r, ws, n, HW, C, stream)
                    e1.record()
                    torch.cuda.synchronize()
                    times[k].append(e0.elapsed_time(e1) / a.reps)
            med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
            print(f"{label}{' +res' if r is not None else ''}: before {med['before']:.4f} ms, after {med['after']:.4f} ms, "
                  f"after/before {med['after'] / med['before']:.3f}")


if __name__ == "__main__":
    main()
