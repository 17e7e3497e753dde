"""The two recurrent propagation scans with TF32 and with fp16 operands (config.half_convs), at the C2 shapes.

usage: python profiles/half_scans_time.py [reps] > half_scans.txt

One run prints: the card's name, power limit and max SM clock; each per-step conv of both scans, the deformable gather and
the flow warp alone at the C2 map sizes (generator 60 x 108, flow completion 30 x 54) in TF32 and fp16, median of `reps`
launches timed with CUDA events after a 256 MiB L2 flush each, with the algorithmic FLOPs and bytes and their share of the
H100 SXM data-sheet rates (495 TF32 / 989 dense fp16 TFLOP/s, 3.35 TB/s); one generator window's scan (plan 0, 11 frames)
and the flow-completion scan of a stage-2 call (80 frames, both directions, plan 0) as replayed CUDA graphs in both
precisions; and the graph-timed candidates of the `gen_prop` / `rfc_prop` autotune keys in both precisions."""
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as g  # noqa: E402

g.build()
from propainter_b200 import autotune, config, ops  # noqa: E402
from propainter_b200.model.propainter import InpaintGenerator  # noqa: E402
from propainter_b200.model.recurrent_flow_completion import RecurrentFlowCompleteNet  # noqa: E402

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
DEV = "cuda"
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
except OSError:
    card = "nvidia-smi unavailable"
print("card:", card, "|", torch.cuda.get_device_name(0))
torch.backends.cudnn.allow_tf32 = True
flush = torch.empty(256 << 20, dtype=torch.uint8, device=DEV)


def timed(fn, n=reps):
    fn()
    ts = []
    for _ in range(n):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return statistics.median(ts)


def report(name, ms, flops, nbytes, peak_tflops):
    tf, bw = flops / ms / 1e9, nbytes / ms / 1e6
    bound = max(flops / (peak_tflops * 1e12), nbytes / 3.35e12) * 1e3
    print(f"  {name:58s} {ms * 1e3:8.1f} us  {tf:6.1f} TFLOP/s ({tf / peak_tflops:5.1%})  {bw:7.1f} GB/s  "
          f"bound/time {bound / ms:5.1%}")


gen = torch.Generator(device=DEV).manual_seed(0)
print(f"\n== per-step kernels at the C2 shapes (median of {reps}, L2 flushed; FLOP share of the TF32 / fp16 data-sheet rate)")
# (label, map h, w, input segment channels, Cout, KH)
CONVS = [("generator 3x3 128->128 (offset net, backbone)", 60, 108, [128], 128, 3),
         ("generator conv_offset.6 3x3 128->432", 60, 108, [128], 432, 3),
         ("generator deformable GEMM 1x1 1152->128", 60, 108, [1152], 128, 1),
         ("flow completion conv_offset.0 3x3 [128|128]->128", 30, 54, [128, 128], 128, 3),
         ("flow completion 3x3 128->128", 30, 54, [128], 128, 3),
         ("flow completion conv_offset.6 3x3 128->432", 30, 54, [128], 432, 3),
         ("flow completion deformable GEMM 1x1 2304->128", 30, 54, [2304], 128, 1)]
for label, h, w, segC, Cout, KH in CONVS:
    Cin = sum(segC)
    wt = torch.randn(Cout, Cin, KH, KH, device=DEV, generator=gen) * 0.05
    bias = torch.randn(Cout, device=DEV, generator=gen)
    flops = 2.0 * h * w * Cout * Cin * KH * KH
    for half in (False, True):
        dt, esz = (torch.float16, 2) if half else (torch.float32, 4)
        segs = [torch.randn(1, h, w, C, device=DEV, generator=gen).to(dt) for C in segC]
        if half:
            wp = ops.pack_conv_weight_f16(wt, segC)
            out16 = torch.empty(1, h, w, Cout, device=DEV, dtype=dt)
            fn = lambda: ops.conv_umma_f16(segs, wp, KH, KH, Cout, bias=bias, act="leaky", slope=0.1, out16=out16)
        else:
            wp = ops.pack_conv_weight(wt, segC)
            out = torch.empty(1, h, w, Cout, device=DEV)
            fn = lambda: ops.conv_umma(segs, wp, KH, KH, Cout, bias=bias, act="leaky", slope=0.1, out=out, round_tf32=True)
        plan = ops.conv_plan(segs, KH, KH, Cout, half=half)
        nbytes = (h * w * Cin + Cout * Cin * KH * KH + h * w * Cout) * esz
        report(f"{label} {'fp16' if half else 'TF32'} bn{plan.bn} {plan.tile_h}x{plan.tile_w} ({plan.ctas} CTAs)", timed(fn),
               flops, nbytes, 989.0 if half else 495.0)
for label, h, w, Cin, x2, flow in (("generator deform gather Cin 128", 60, 108, 128, False, True),
                                  ("flow completion deform gather Cin 256 (x | x2)", 30, 54, 256, True, False)):
    xc = Cin // 2 if x2 else Cin
    x = torch.randn(1, h, w, xc, device=DEV, generator=gen)
    xx = torch.randn(1, h, w, xc, device=DEV, generator=gen) if x2 else None
    o = torch.randn(1, h, w, 432, device=DEV, generator=gen)
    fl = torch.randn(1, h, w, 2, device=DEV, generator=gen) if flow else None
    for half in (False, True):
        cols = torch.empty(1, h, w, 9 * Cin, device=DEV, dtype=torch.float16 if half else torch.float32)
        # least HBM traffic: x and o read once, the columns written (the 9 x 4 corner reads per pixel mostly hit L2)
        nbytes = h * w * (Cin * 4 + 432 * 4 + 9 * Cin * (2 if half else 4))
        report(f"{label} -> {'fp16' if half else 'TF32'} columns", timed(lambda: ops.deform_gather(x, o, fl, 3.0, cols, x2=xx)), 0.0,
               nbytes, 989.0 if half else 495.0)
feat = torch.randn(1, 60, 108, 128, device=DEV, generator=gen)
fprop = torch.randn(1, 60, 108, 2, device=DEV, generator=gen) * 3
for half in (False, True):
    warped = torch.empty(1, 60, 108, 128, device=DEV, dtype=torch.float16 if half else torch.float32)
    nbytes = 60 * 108 * (128 * 4 + 8 + 128 * (2 if half else 4))     # map and flow read once, warped written
    report(f"generator flow warp 128 ch -> {'fp16' if half else 'TF32'}", timed(lambda: ops.flow_warp_fbcheck(feat, fprop, warped=warped,
                                                                                                           round_tf32=True)),
           0.0, nbytes, 989.0 if half else 495.0)


def graph_ms(fn, n=reps):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
        fn()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fn()
    return timed(graph.replay, n)


print("\n== scans as replayed CUDA graphs (plan 0)")
config.UMMA_CONV = True
net = InpaintGenerator(seed=3).to(DEV)
lt = 11
xl = torch.randn(lt, 60, 108, 128, device=DEV, generator=gen)
dsf, dsb = (torch.randn(lt - 1, 60, 108, 2, device=DEV, generator=gen) * 3 for _ in range(2))
pmask = (torch.rand(lt, 60, 108, 2, device=DEV, generator=gen) > 0.5).float()
rfc = RecurrentFlowCompleteNet(None, seed=2).to(DEV)
m = torch.randn(80, 128, 30, 54, device=DEV, generator=gen).contiguous(memory_format=torch.channels_last)
res = {}
with torch.no_grad():
    for rnd in range(3):                                           # alternated
        for half in (False, True):
            config.HALF_OPERANDS = half
            res.setdefault(("gen", half), []).append(graph_ms(lambda: net._feat_propagation_umma(xl, dsf, dsb, pmask), 5))
            res.setdefault(("rfc", half), []).append(graph_ms(lambda: rfc._propagate_umma(m), 3))
            torch.cuda.empty_cache()
for (what, half), v in sorted(res.items()):
    name = "generator window scan (11 frames, 60x108)" if what == "gen" else "flow-completion scan (80 frames, 30x54, both directions)"
    print(f"  {name:58s} {'fp16' if half else 'TF32'}: {statistics.median(v):8.3f} ms (runs {', '.join(f'{x:.3f}' for x in v)})")

print("\n== autotune candidates (graph-timed, ms per run; #0 = plan 0)")
config.UMMA_CONV = "auto"
flows = tuple(torch.randn(1, 79, 2, 240, 432, device=DEV, generator=gen) for _ in range(2))
masks = (torch.rand(1, 80, 1, 240, 432, device=DEV, generator=gen) > 0.8).float()
with torch.no_grad():
    for half in (False, True):
        config.HALF_OPERANDS = half
        rfc.forward_bidirect_flow(flows, masks)
        net.forward_features(torch.randn(18, 128, 60, 108, device=DEV, generator=gen), (flows[0][0, :lt - 1].contiguous(),
                             flows[1][0, :lt - 1].contiguous()), masks[0, :18], masks[0, :18], lt)
torch.cuda.synchronize()
for (key, i), ms in sorted(autotune._timings.items(), key=lambda kv: str(kv[0])):
    if key[0] in ("gen_prop", "rfc_prop"):
        print(f"  {key[0]} {key[1]} half={key[2]} #{i}: {ms:.3f} ms")
print("  picks:", {str(k): v for k, v in autotune._choice.items() if k[0] in ("gen_prop", "rfc_prop")})
