"""The clip encoders of one C2 clip with the half-operand switch off and on (config.HALF_OPERANDS): the generator's frame
encoder (InpaintGenerator.encode, captured graph gen_enc, 2 chunks of 40 frames) and RAFT's feature and context encoders
(RAFT.encode_frames, fnet + cnet, over the clip's RAFT chunks), then every conv of both encoders alone.

usage: python profiles/half_encoders_time.py [c2|c1] [reps] > half_encoders.txt

One run prints: the card's name, power limit and max SM clock; for each encoder the wall time over the clip (CUDA events,
256 MiB L2 flush before each call, warm) with the switch off (TF32 convs) and on (fp16 operands), the two settings
alternated in one process, `reps` repetitions each, min / median / max, and TFLOP/s from the encoder's FLOP count against
the H100 SXM data-sheet rates (495 TF32, 989 dense fp16).  Then each conv layer alone at the clip shape, in fp32 (TF32) and
fp16 operands (cuDNN, channels_last, no epilogue), median of 20 with the L2 flushed, with TFLOP/s.  cuDNN TF32 is allowed
throughout, as in a default run.  The switch moves only cnet of RAFT's two encoders (fnet stays TF32), so the RAFT line's
share of the fp16 rate mixes the two."""
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as g  # noqa: E402

g.build()
from bench import WORKLOADS  # noqa: E402
from propainter_b200 import config, ops, synth  # noqa: E402
from propainter_b200.inference_propainter import (InferenceConfig, ProPainterPipeline, auto_clip_frames,  # noqa: E402
                                                  flow_chunks)

wl = WORKLOADS[sys.argv[1] if len(sys.argv) > 1 else "c2"]
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 7
T, H, W = wl["T"], wl["H"], wl["W"]
modes = (False, True)
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
except OSError:
    card = "nvidia-smi unavailable"
print("card:", card, "|", torch.cuda.get_device_name(0))
torch.backends.cudnn.allow_tf32 = True
torch.backends.cudnn.benchmark = True

u8, fm, md = synth.make_clip(T, H, W, mask=wl["mask"], seed=0)
u8d, mdd = torch.from_numpy(u8).cuda(), md.cuda()[0]                  # masks [T,1,H,W]
pipe = ProPainterPipeline(device="cuda")
gen, raft = pipe.model, pipe.fix_raft.fix_raft
cfg = InferenceConfig(raft_iter=wl["raft_iter"])
frames = ops.u8_to_frames(u8d)                                      # [T,3,H,W] in [-1,1]
masked = frames * (1 - mdd[:, 0:1])
clip = auto_clip_frames(T, H, W, raft.corr_plan(H, W, frames.device))
chunks = flow_chunks(T, clip)
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")


def conv_flops(shapes):
    return sum(2 * n * ho * wo * co * ci * kh * kw for n, ho, wo, co, ci, kh, kw, _, _ in shapes)


def gen_layers(n):
    """(n, Ho, Wo, Cout, Cin per group, kh, kw, stride, groups) of the generator encoder's convs over n frames"""
    h, w = H // 4, W // 4
    out = [(n, H // 2, W // 2, 64, 8, 3, 3, 2, 1), (n, H // 2, W // 2, 64, 64, 3, 3, 1, 1), (n, h, w, 128, 64, 3, 3, 2, 1),
           (n, h, w, 256, 128, 3, 3, 1, 1), (n, h, w, 384, 256, 3, 3, 1, 1)]
    for i, gr, cin in ((10, 2, 640), (12, 4, 768), (14, 8, 640), (16, 1, 512)):
        co = gen.P[f"encoder.layers.{i}.weight"].shape[0]
        out.append((n, h, w, co, cin // gr, 3, 3, 1, gr))
    return out


def raft_layers(n):
    """the same for one BasicEncoder (fnet and cnet have the same convs)"""
    out = [(n, H // 2, W // 2, 64, 3, 7, 7, 2, 1)]
    cin, h, w = 64, H // 2, W // 2
    for co, s in ((64, 1), (96, 2), (128, 2)):
        h, w = (h - 1) // s + 1, (w - 1) // s + 1
        out += [(n, h, w, co, cin, 3, 3, s, 1), (n, h, w, co, co, 3, 3, 1, 1)]
        if s != 1:
            out.append((n, h, w, co, cin, 1, 1, s, 1))
        out += [(n, h, w, co, co, 3, 3, 1, 1), (n, h, w, co, co, 3, 3, 1, 1)]
        cin = co
    out.append((n, h, w, 256, cin, 1, 1, 1, 1))
    return out


def timed(fn):
    flush.zero_()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def gen_enc():
    gen.encode(masked, mdd, mdd)


def raft_enc():
    for s, e in chunks:
        raft.encode_frames(frames[s:e])


encoders = {"generator encoder (gen_enc)": (gen_enc, conv_flops(gen_layers(T))),
            "RAFT fnet + cnet (encode_frames)": (raft_enc, 2 * conv_flops(raft_layers(sum(e - s for s, e in chunks))))}
with torch.no_grad():
    for m in modes:                                  # warm: graph capture, cuDNN algorithm choice, autotune.pick
        config.HALF_OPERANDS = m
        for fn, _ in encoders.values():
            for _ in range(3):
                fn()
    torch.cuda.synchronize()
    runs = {(k, m): [] for k in encoders for m in modes}
    for _ in range(reps):
        for m in modes:
            config.HALF_OPERANDS = m
            for k, (fn, _) in encoders.items():
                runs[(k, m)].append(timed(fn))
config.HALF_OPERANDS = True
print(f"\nencoders over the {wl['name'][:3]} clip ({T} frames {W}x{H}; RAFT chunks {chunks}), {reps} reps, L2 flushed, "
      "ms min / median / max")
for k, (_, flop) in encoders.items():
    for m in modes:
        v = runs[(k, m)]
        med = statistics.median(v)
        tf = flop / (med * 1e-3) / 1e12
        peak = 989 if m else 495
        print(f"  {k:34s} {'fp16' if m else 'tf32'}  {min(v):8.3f} {med:8.3f} {max(v):8.3f}   {flop / 1e12:.2f} TFLOP "
              f"{tf:6.1f} TFLOP/s ({100 * tf / peak:.0f} % of {peak})")


# ---------------------------------------------------------------- each conv alone at the clip shape
def layer_ms(fn, n=20):
    fn()
    return statistics.median(timed(fn) for _ in range(n))


def conv_alone(n, ho, wo, co, ci, kh, kw, s, gr, dt):
    """a grouped layer runs as `gr` dense convs (the per-group plan of InpaintGenerator._encoder)"""
    ci = 8 if ci == 3 and dt == torch.float16 else ci              # RAFT conv1: fp16 frames padded to 8 channels
    xs = [torch.randn(n, ci, ho * s, wo * s, device="cuda").to(dt).contiguous(memory_format=torch.channels_last)
          for _ in range(gr)]
    w = (torch.randn(co // gr, ci, kh, kw, device="cuda") / (ci * kh * kw) ** 0.5).to(dt).contiguous(memory_format=torch.channels_last)
    return lambda: [F.conv2d(x, w, None, s, kh // 2) for x in xs]


for title, layers in (("generator encoder", gen_layers(T // 2)), ("RAFT BasicEncoder (one of fnet / cnet)", raft_layers(T))):
    print(f"\n{title}: each conv alone, median of 20, L2 flushed (n, Ho, Wo, Cout, Cin/group, kh, kw, stride, groups)")
    tot = {dt: 0.0 for dt in (torch.float32, torch.float16)}
    for sh in layers:
        line = f"  {str(sh):44s}"
        for dt in (torch.float32, torch.float16):
            ms = layer_ms(conv_alone(*sh, dt))
            tot[dt] += ms
            tf = conv_flops([sh]) / (ms * 1e-3) / 1e12
            peak = 989 if dt == torch.float16 else 495
            line += f"  {'fp16' if dt == torch.float16 else 'tf32'} {ms:7.3f} ms {tf:6.1f} TFLOP/s ({100 * tf / peak:3.0f} %)"
        print(line)
    print(f"  {'sum':44s}  tf32 {tot[torch.float32]:7.3f} ms                          fp16 {tot[torch.float16]:7.3f} ms")
