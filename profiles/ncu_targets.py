"""Launches the hot kernels once each at BASELINE configs[1] (C2, 432x240) shapes for ncu:

  ncu --set full --clock-control none --import-source on \
      -k regex:'k_conv_umma|k_deform|k_flow_warp|k_sparse_attn|k_corr_lookup|k_inorm|k_add_layernorm|k_pool_depthwise|k_bias_act|k_gru' \
      -o gpurun_out/prof python profiles/ncu_targets.py          (then profiles/ncu_summarize.py on the report)

and, with --time, prints CUDA-event timings of the same launches (never report numbers taken under ncu)."""
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from propainter_b200 import ops  # noqa: E402
from propainter_b200.window_index import window_key_table  # noqa: E402

dev = "cuda"
torch.manual_seed(0)
TIME = "--time" in sys.argv
results = {}


def run(name, fn, reps=20):
    fn()
    torch.cuda.synchronize()
    if not TIME:
        return
    flush = torch.empty(64 * 1024 * 1024, device=dev)
    ts = []
    for _ in range(reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    results[name] = (statistics.median(ts), min(ts))


# ---- deformable alignment: generator step (60x108, Cin 128, flow-guided) and flow-completion step (30x54, Cin 256)
for tag, (H, W, Cin, use_flow, mr) in {"gen": (60, 108, 128, True, 3.0), "rfc": (30, 54, 256, False, 5.0)}.items():
    x = torch.randn(H, W, Cin, device=dev)
    o = torch.randn(H, W, 432, device=dev)
    fl = torch.randn(H, W, 2, device=dev) if use_flow else None
    wp = torch.randn(9 * Cin, 128, device=dev) * 0.03
    b = torch.randn(128, device=dev)
    out = torch.empty(H, W, 128, device=dev)
    run(f"deform_align_{tag}", lambda: ops.deform_align(x, o, fl, mr, wp, b, out))

# ---- wgmma conv kernel + deformable gather + flow warp at the two propagation-scan shapes
for tag, (H, W) in {"gen": (60, 108), "rfc": (30, 54)}.items():
    xc = torch.randn(1, H, W, 128, device=dev)
    wpk = ops.pack_conv_weight(torch.randn(128, 128, 3, 3, device=dev) * 0.03)
    bc, prec, resc = torch.randn(128, device=dev), torch.randn(1, H, W, 128, device=dev), torch.randn(1, H, W, 128, device=dev)
    oc = torch.empty(1, H, W, 128, device=dev)
    run(f"conv_umma_3x3_128_{tag}", lambda: ops.conv_umma([xc], wpk, 3, 3, 128, bias=bc, act="leaky", slope=0.1, pre=prec, res=resc, out=oc))
    w432 = ops.pack_conv_weight(torch.randn(432, 128, 3, 3, device=dev) * 0.03)
    o432 = torch.empty(1, H, W, 432, device=dev)
    run(f"conv_umma_3x3_432_{tag}", lambda: ops.conv_umma([xc], w432, 3, 3, 432, out=o432))
    cin = 128 if tag == "gen" else 256
    xd = torch.randn(1, H, W, cin, device=dev)
    od = torch.randn(1, H, W, 432, device=dev)
    fld = torch.randn(1, H, W, 2, device=dev) if tag == "gen" else None
    colsd = torch.empty(1, H, W, 9 * cin, device=dev)
    run(f"deform_gather_{tag}", lambda: ops.deform_gather(xd, od, fld, 3.0 if tag == "gen" else 5.0, colsd))
    wdp = ops.pack_deform_weight_umma(torch.randn(128, cin, 3, 3, device=dev) * 0.03)
    run(f"conv_umma_1x1_deform_gemm_{tag}", lambda: ops.conv_umma([colsd], wdp, 1, 1, 128, bias=bc, out=oc))
fw_feat, fw_flow = torch.randn(1, 60, 108, 128, device=dev), torch.randn(1, 60, 108, 2, device=dev)
fw_out = torch.empty(1, 60, 108, 128, device=dev)
run("flow_warp_gen", lambda: ops.flow_warp_fbcheck(fw_feat, fw_flow, warped=fw_out, round_tf32=True))

# ---- sparse window attention: t=18 frames, 20x36 tokens, 5 of 16 windows masked (ellipse mask of C2), layer parity 0
t, H2, W2, C = 18, 20, 36, 512
qkv = torch.randn(t, H2 * W2, 3 * C, device=dev)
pool = torch.randn(t, 45, 2 * C, device=dev)
ktab = torch.from_numpy(window_key_table(H2, W2)).to(dev)
for nm, masked in (("5of16", [5, 6, 9, 10, 11]), ("16of16", list(range(16)))):
    flags = torch.zeros(16, dtype=torch.int32, device=dev)
    flags[masked] = 1
    run(f"sparse_attn_umma_{nm}", lambda: ops.sparse_window_attn(qkv, pool, ktab, flags, t, H2 * W2, 0, 2, impl="umma"))
    run(f"sparse_attn_mma_{nm}", lambda: ops.sparse_window_attn(qkv, pool, ktab, flags, t, H2 * W2, 0, 2, impl="mma"))

# ---- RAFT correlation: build + lookup for one refinement batch (22 pairs at 30x54)
B, h, w = 22, 30, 54
fmap = torch.randn(12, h * w, 256, device=dev)
a = torch.arange(11, device=dev, dtype=torch.int32)
levels = ops.corr_alloc(B, h, w, dev)
run("corr_build", lambda: ops.corr_build(fmap, torch.cat([a, a + 1]), torch.cat([a + 1, a]), levels, h, w), reps=5)
ys, xs = torch.meshgrid(torch.arange(h, device=dev), torch.arange(w, device=dev), indexing="ij")
coords = (torch.stack([xs, ys], -1).float()[None] + torch.randn(B, h, w, 2, device=dev) * 3).contiguous()
out = torch.empty(B, h, w, 324, device=dev)
run("corr_lookup_tma", lambda: ops.corr_lookup(levels, coords, out, tma=True))
run("corr_lookup_ldg", lambda: ops.corr_lookup(levels, coords, out, tma=False))

# ---- propagation prologue + FFN stencils
cur, prop = torch.randn(60, 108, 128, device=dev), torch.randn(60, 108, 128, device=dev)
f1, f2, m = torch.randn(60, 108, 2, device=dev), torch.randn(60, 108, 2, device=dev), torch.zeros(60, 108, 2, device=dev)
cond, bb = torch.empty(60, 108, 264, device=dev), torch.empty(60, 108, 260, device=dev)
run("prop_cond", lambda: ops.prop_cond(cur, prop, f1, f2, m, cond, bb, False))
Y = torch.randn(18 * 720, 1960, device=dev)
run("ffn_overlap_add", lambda: ops.ffn_overlap_add(Y, 18, 60, 108, 40))
fr = torch.randn(80, 3, 240, 432, device=dev)
ff, fb, mk = torch.randn(79, 2, 240, 432, device=dev), torch.randn(79, 2, 240, 432, device=dev), torch.zeros(80, 1, 240, 432, device=dev)
mk[:, :, 80:160, 150:280] = 1
run("img_prop_scan_80f", lambda: ops.img_prop_scan(fr, ff, fb, mk, True), reps=5)

# ---- epilogue / glue kernels at their largest call sites
B2 = 158
zr, pz = torch.randn(B2, 30, 54, 256, device=dev), torch.randn(B2, 30, 54, 256, device=dev)
HX, RX = torch.randn(B2, 30, 54, 256, device=dev), torch.randn(B2, 30, 54, 256, device=dev)
zb, qv, pq = torch.empty(B2, 30, 54, 128, device=dev), torch.randn(B2, 30, 54, 128, device=dev), torch.randn(B2, 30, 54, 128, device=dev)
run("gru_gate_158pairs", lambda: ops.gru_gate(zr, None, HX[..., :128], zb, RX[..., :128], pre=pz))
run("gru_update_158pairs", lambda: ops.gru_update(qv, None, zb, HX[..., :128], pre=pq))
xin = torch.randn(80, 120, 216, 64, device=dev)
res = torch.randn(80, 120, 216, 64, device=dev)
run("instance_norm_80x120x216x64", lambda: ops.instance_norm(xin, relu=True, res=res, post_relu=True, out=xin), reps=5)
cb = torch.randn(B2, 30, 54, 256, device=dev)
bias256 = torch.randn(256, device=dev)
run("bias_act_158x30x54x256", lambda: ops.bias_act(cb, bias256, "relu"))
tok, dl = torch.randn(18, 20, 36, 512, device=dev), torch.randn(18, 20, 36, 512, device=dev)
gam, bet = torch.randn(512, device=dev), torch.randn(512, device=dev)
run("add_layernorm_18x720x512", lambda: ops.add_layernorm(tok, dl, gam, bet))
wt, bp = torch.randn(16, 512, device=dev), torch.randn(512, device=dev)
run("pool_depthwise_18x20x36x512", lambda: ops.pool_depthwise(tok, wt, bp, 4, 4))

if TIME:
    for k, (med, mn) in results.items():
        print(f"{k:24s} median {med:9.1f} us   min {mn:9.1f} us")
