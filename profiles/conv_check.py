"""Hardware check + timing of the wgmma conv kernel (pp_conv2d_umma) and the deformable gather (pp_deform_gather).

    python profiles/conv_check.py [group]        group in {basic, shapes, deform, step}; default all, one subprocess each

Correctness is checked twice per case: (i) *exact* -- inputs and weights rounded to TF32-representable values, so every
product is exact in fp32 and only the accumulation order differs from torch's fp32 conv (error ~1e-6: any indexing /
layout / swizzle mistake shows up as O(1)); (ii) *plain* -- arbitrary fp32 inputs (activations reach the tensor core
truncated to TF32), error relative to the output scale.  Timings: CUDA events, L2 flushed between repetitions, next to
cuDNN (TF32 allowed) + pp_bias_act for the same math.  Not part of the test-suite (tests/test_gpu_ops.py has the parity
tests); this is the script the numbers in profiles/README.md come from."""
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

GROUPS = ["basic", "shapes", "deform", "step"]


def main(group):
    import torch
    import torch.nn.functional as F
    from propainter_b200 import ops
    dev = "cuda"
    torch.manual_seed(0)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    flush = torch.empty(64 * 1024 * 1024, device=dev)

    def timeit(fn, reps=20):
        for _ in range(3):
            fn()
        ts = []
        for _ in range(reps):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) * 1e3)
        return statistics.median(ts)

    def conv_case(name, n, H, W, segC, Cout, KH=3, KW=3, act="none", slope=0.1, use_bias=True, use_pre=False, use_res=False,
                  post_relu=False, bn=0, tile_w=0, time_it=True, exact=True, tile_m=0):
        Cin = sum(segC)
        w = torch.randn(Cout, Cin, KH, KW, device=dev) / (Cin * KH * KW) ** 0.5
        b = torch.randn(Cout, device=dev) if use_bias else None
        # segments live as channel slices of wider buffers (like the scan buffers of the product)
        bufs = [torch.randn(n, H, W, (C + 11) // 4 * 4, device=dev) for C in segC]   # pixel stride: multiple of 16 bytes
        pre = torch.randn(n, H, W, Cout + 4, device=dev)[..., :Cout] if use_pre else None
        res = torch.randn(n, H, W, Cout + 8, device=dev)[..., 4:4 + Cout] if use_res else None
        outbuf = torch.zeros(n, H, W, Cout + 12, device=dev)
        out = outbuf[..., 8:8 + Cout]
        errs = []
        for mode in (("exact", "plain") if exact else ("plain",)):
            if mode == "exact":
                xs = [ops.tf32_round(bf)[..., 4:4 + C] for bf, C in zip(bufs, segC)]
                wr = ops.tf32_round(w)
            else:
                xs = [bf[..., 4:4 + C] for bf, C in zip(bufs, segC)]
                wr = w
            wp = ops.pack_conv_weight(wr, segC)
            outbuf.zero_()
            ops.conv_umma(xs, wp, KH, KW, Cout, bias=b, act=act, slope=slope, pre=pre, res=res, post_relu=post_relu, out=out, bn=bn,
                          tile_w=tile_w, tile_m=tile_m)
            torch.cuda.synchronize()
            xin = torch.cat(xs, -1).permute(0, 3, 1, 2)
            ref = F.conv2d(xin, wr, b, padding=(KH // 2, KW // 2)).permute(0, 2, 3, 1)
            if pre is not None:
                ref = ref + pre
            ref = {"none": lambda v: v, "relu": torch.relu, "leaky": lambda v: F.leaky_relu(v, slope), "sigmoid": torch.sigmoid,
                   "tanh": torch.tanh}[act](ref)
            if res is not None:
                ref = ref + res
            if post_relu:
                ref = torch.relu(ref)
            e = ((out - ref).abs().max() / ref.abs().max()).item()
            errs.append(e)
            pad_ok = outbuf[..., :8].abs().max().item() == 0 and outbuf[..., 8 + Cout:].abs().max().item() == 0
            if not pad_ok:
                errs.append(float("nan"))
        msg = f"{name:34s} n={n} {H}x{W} segC={segC} Cout={Cout} {KH}x{KW} act={act} bn={bn} tw={tile_w} tm={tile_m}: " + \
              " ".join(f"{m}={e:.2e}" for m, e in zip(("exact", "plain") if exact else ("plain",), errs))
        if time_it:
            xs = [bf[..., 4:4 + C] for bf, C in zip(bufs, segC)]
            wp = ops.pack_conv_weight(w, segC)
            t_own = timeit(lambda: ops.conv_umma(xs, wp, KH, KW, Cout, bias=b, act=act, slope=slope, pre=pre, res=res, post_relu=post_relu,
                                                 out=out, bn=bn, tile_w=tile_w, tile_m=tile_m))
            torch.backends.cudnn.allow_tf32 = True
            xin = torch.cat(xs, -1).permute(0, 3, 1, 2).contiguous(memory_format=torch.channels_last)
            wcl = w.contiguous(memory_format=torch.channels_last)
            with torch.backends.cudnn.flags(enabled=True, benchmark=True):
                def lib():
                    y = F.conv2d(xin, wcl, None, padding=(KH // 2, KW // 2))
                    return ops.bias_act(y.permute(0, 2, 3, 1), b, act, slope, res=res, post_relu=post_relu, out=out)
                t_lib = timeit(lib)
            torch.backends.cudnn.allow_tf32 = False
            flops = 2.0 * n * H * W * Cin * KH * KW * Cout
            msg += f" | own {t_own:7.1f} us ({flops / t_own * 1e-6:6.1f} TF/s)  cudnn+bias_act {t_lib:7.1f} us"
        print(msg, flush=True)

    if group == "basic":
        conv_case("1x1 K=32", 1, 16, 8, [32], 32, 1, 1, use_bias=False, time_it=False)
        conv_case("1x1 K=128 bn64", 1, 30, 54, [128], 64, 1, 1, time_it=False)
        conv_case("3x3 single block", 1, 16, 8, [32], 32, time_it=False)
        conv_case("3x3 128->128 rfc map", 1, 30, 54, [128], 128)
        conv_case("3x3 128->128 gen map", 1, 60, 108, [128], 128)
        conv_case("3x3 leaky+pre+res", 1, 30, 54, [128], 128, act="leaky", use_pre=True, use_res=True)
    elif group == "shapes":
        for bn in (32, 64, 128):
            conv_case(f"3x3 gen map bn={bn}", 1, 60, 108, [128], 128, bn=bn, exact=False)
        for bn in (32, 64, 128):
            conv_case(f"3x3 rfc map bn={bn}", 1, 30, 54, [128], 128, bn=bn, exact=False)
        for bn in (32, 64, 128):
            conv_case(f"3x3 gen map M=64 bn={bn}", 1, 60, 108, [128], 128, bn=bn, tile_m=64, exact=(bn == 128))
        for bn in (32, 64, 128):
            conv_case(f"3x3 rfc map M=64 bn={bn}", 1, 30, 54, [128], 128, bn=bn, tile_m=64, exact=(bn == 64))
        conv_case("3x3 M=64 tile_w=16 leaky pre res", 2, 30, 54, [128, 128], 128, act="leaky", use_pre=True, use_res=True, tile_m=64, tile_w=16)
        conv_case("1x1 M=64 K=1152", 1, 60, 108, [1152], 128, 1, 1, tile_m=64)
        conv_case("3x3 rfc map tile_w=16", 1, 30, 54, [128], 128, tile_w=16)
        conv_case("3x3 gen map tile_w=16", 1, 60, 108, [128], 128, tile_w=16)
        conv_case("3x3 3 segments", 1, 30, 54, [128, 128, 128], 128, act="leaky")
        conv_case("3x3 2 segments rfc x2", 2, 30, 54, [128, 128], 128, act="leaky")
        conv_case("3x3 ragged channels 264", 1, 60, 108, [264], 128, act="leaky")
        conv_case("3x3 ragged segs 128+5", 1, 60, 108, [128, 5], 128, act="leaky", use_pre=True)
        conv_case("3x3 Cout=432", 1, 60, 108, [128], 432)
        conv_case("3x3 Cout=432 rfc", 1, 30, 54, [128], 432)
        conv_case("1x1 ragged segments 160+96", 1, 30, 54, [160, 96], 128, 1, 1, use_res=True)
        conv_case("1x1 K=1152 (deform gemm gen)", 1, 60, 108, [1152], 128, 1, 1)
        conv_case("1x1 K=2304 (deform gemm rfc)", 1, 30, 54, [2304], 128, 1, 1)
        conv_case("1x5 gru 256->256 n=8", 8, 30, 54, [256], 256, 1, 5)
        conv_case("5x1 gru 256->256 n=8", 8, 30, 54, [256], 256, 5, 1)
        conv_case("3x3 relu post_relu res", 2, 30, 54, [64], 64, act="relu", use_res=True, post_relu=True)
        conv_case("3x3 sigmoid", 1, 17, 23, [40], 36, act="sigmoid")
        conv_case("7x7 64->64", 1, 40, 40, [64], 64, 7, 7, bn=32)
        conv_case("3x3 batch 11 gen (fuse)", 11, 60, 108, [128, 128, 4], 128, act="leaky", exact=False)
        conv_case("3x3 158x30x54 256->128 (raft)", 158, 30, 54, [256], 128, act="relu", exact=False)
    elif group == "deform":
        for tag, (n, H, W, Cin, use_flow, mr) in {"gen": (1, 60, 108, 128, True, 3.0), "rfc": (1, 30, 54, 256, False, 5.0),
                                                   "rfc x2": (2, 30, 54, 256, False, 5.0)}.items():
            x = torch.randn(n, H, W, Cin + 128, device=dev)[..., :Cin]
            o = torch.randn(n, H, W, 432, device=dev)
            fl = torch.randn(n, H, W, 2, device=dev) * 2 if use_flow else None
            w = torch.randn(128, Cin, 3, 3, device=dev) * 0.03
            b, ob = torch.randn(128, device=dev), torch.randn(432, device=dev) * 0.1
            wp_old = ops.pack_deform_weight(w)
            wp_new = ops.pack_deform_weight_umma(w)
            ref = torch.empty(n, H, W, 128, device=dev)
            for i in range(n):
                ops.deform_align(x[i], o[i], None if fl is None else fl[i], mr, wp_old, b, ref[i], o_bias=ob)
            cols = torch.empty(n, H, W, 9 * Cin, device=dev)
            out = torch.empty(n, H, W, 128, device=dev)

            def new():
                ops.deform_gather(x, o, fl, mr, cols, o_bias=ob)
                ops.conv_umma([cols], wp_new, 1, 1, 128, bias=b, out=out)
            new()
            torch.cuda.synchronize()
            e = ((out - ref).abs().max() / ref.abs().max()).item()
            t_new = timeit(new)
            t_g = timeit(lambda: ops.deform_gather(x, o, fl, mr, cols, o_bias=ob))
            t_old = timeit(lambda: [ops.deform_align(x[i], o[i], None if fl is None else fl[i], mr, wp_old, b, ref[i], o_bias=ob) for i in range(n)])
            print(f"deform {tag}: gather+umma vs mma.sync kernel rel {e:.2e} | new {t_new:.1f} us (gather {t_g:.1f}) vs old {t_old:.1f} us", flush=True)
    elif group == "step":
        # one propagation step's conv chain, back to back inside a CUDA graph (launch gaps included): new kernels vs cuDNN + bias_act
        for tag, (H, W, cin0) in {"gen": (60, 108, 128), "rfc": (30, 54, 256)}.items():
            C = 128
            xs0 = torch.randn(1, H, W, cin0, device=dev)
            ws = [torch.randn(128, cin0, 3, 3, device=dev) * 0.02, torch.randn(128, 128, 3, 3, device=dev) * 0.03,
                  torch.randn(128, 128, 3, 3, device=dev) * 0.03, torch.randn(432, 128, 3, 3, device=dev) * 0.03]
            bs = [torch.randn(w.shape[0], device=dev) * 0.1 for w in ws]
            wps = [ops.pack_conv_weight(w) for w in ws]
            pre = torch.randn(1, H, W, 128, device=dev)
            t1, t2, t3 = (torch.empty(1, H, W, 128, device=dev) for _ in range(3))
            o = torch.empty(1, H, W, 432, device=dev)
            dcin = cin0
            xd = torch.randn(1, H, W, dcin, device=dev)
            wd = torch.randn(128, dcin, 3, 3, device=dev) * 0.03
            wdp, wdo = ops.pack_deform_weight_umma(wd), ops.pack_deform_weight(wd)
            cols = torch.empty(1, H, W, 9 * dcin, device=dev)
            al = torch.empty(1, H, W, 128, device=dev)
            wb0, wb2 = torch.randn(128, 128, 3, 3, device=dev) * 0.03, torch.randn(128, 128, 3, 3, device=dev) * 0.03
            wb0p, wb2p = ops.pack_conv_weight(wb0), ops.pack_conv_weight(wb2)
            st = torch.empty(1, H, W, 128, device=dev)
            fl = torch.randn(1, H, W, 2, device=dev) if tag == "gen" else None
            mr = 3.0 if tag == "gen" else 5.0

            def new_step():
                ops.conv_umma([xs0], wps[0], 3, 3, 128, bias=bs[0], act="leaky", slope=0.1, pre=pre, out=t1, round_tf32=True)
                ops.conv_umma([t1], wps[1], 3, 3, 128, bias=bs[1], act="leaky", slope=0.1, out=t2, round_tf32=True)
                ops.conv_umma([t2], wps[2], 3, 3, 128, bias=bs[2], act="leaky", slope=0.1, out=t3, round_tf32=True)
                ops.conv_umma([t3], wps[3], 3, 3, 432, bias=bs[3], out=o)
                ops.deform_gather(xd, o, fl, mr, cols)
                ops.conv_umma([cols], wdp, 1, 1, 128, bias=bs[0], out=al)
                ops.conv_umma([al], wb0p, 3, 3, 128, bias=bs[1], act="leaky", slope=0.2, pre=pre, out=t1, round_tf32=True)
                ops.conv_umma([t1], wb2p, 3, 3, 128, bias=bs[2], res=al, out=st)

            wcl = [w.contiguous(memory_format=torch.channels_last) for w in ws + [wb0, wb2]]
            torch.backends.cudnn.allow_tf32 = True

            def lib_conv(x, w, b, act, slope=0.0, res=None, out=None):
                y = F.conv2d(x.permute(0, 3, 1, 2), w, None, padding=1)
                return ops.bias_act(y.permute(0, 2, 3, 1), b, act, slope, res=res, out=out)

            def old_step():
                a = lib_conv(xs0, wcl[0], bs[0], "leaky", 0.1)
                a = lib_conv(a, wcl[1], bs[1], "leaky", 0.1)
                a = lib_conv(a, wcl[2], bs[2], "leaky", 0.1)
                oo = F.conv2d(a.permute(0, 3, 1, 2), wcl[3], None, padding=1).permute(0, 2, 3, 1)
                ops.deform_align(xd[0], oo[0], None if fl is None else fl[0], mr, wdo, bs[0], al[0], o_bias=bs[3])
                a = lib_conv(al, wcl[4], bs[1], "leaky", 0.2)
                lib_conv(a, wcl[5], bs[2], "none", res=al, out=st)

            for nm, fn in (("new", new_step), ("old", old_step)):
                with torch.backends.cudnn.flags(enabled=True, benchmark=True):
                    for _ in range(3):
                        fn()
                    torch.cuda.synchronize()
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g):
                        for _ in range(10):
                            fn()
                t = timeit(g.replay, reps=10) / 10
                print(f"step chain {tag} [{nm}]: {t:.1f} us per step (10 steps per graph replay)", flush=True)


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] in GROUPS:
        main(sys.argv[1])
    else:
        for g in GROUPS:                       # one process per group: a trapped kernel must not take the others with it
            print(f"==== {g}", flush=True)
            try:
                r = subprocess.run([sys.executable, os.path.abspath(__file__), g], timeout=600)
                print(f"==== {g}: exit {r.returncode}", flush=True)
            except subprocess.TimeoutExpired:
                print(f"==== {g}: TIMEOUT", flush=True)
