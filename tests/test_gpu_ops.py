"""GPU parity: every C-ABI op vs the oracle on seeded inputs (through propainter_b200.ops -> ctypes -> .so).

Tolerances: gather / stencil kernels are fp32 -> 1e-5 abs (discontinuous outputs: mismatch fraction);
the TF32 tensor-core kernels (deform GEMM, attention) -> 2e-3 of the output scale; the correlation
GEMM uses the 3xTF32 split -> 1e-5.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import generator_ref, ops_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(autouse=True)
def _exact_library_math():
    """Keep torch's own convs / matmuls in fp32 so differences isolate our kernels."""
    a, b = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = a, b



def smooth_flow(gen, n, H, W, amp=4.0):
    z = torch.randn(n, 2, H // 8 + 2, W // 8 + 2, generator=gen) * amp
    return F.interpolate(z, size=(H, W), mode="bicubic", align_corners=False).contiguous()


def test_img_prop_scan():
    from propainter_b200 import ops
    gen = torch.Generator().manual_seed(0)
    for (T, H, W) in ((6, 40, 56), (9, 128, 136)):
        frames = torch.rand(1, T, 3, H, W, generator=gen) * 2 - 1
        ff = smooth_flow(gen, T - 1, H, W).view(1, T - 1, 2, H, W)
        fb = (-ff + 0.3 * smooth_flow(gen, T - 1, H, W).view(1, T - 1, 2, H, W)).contiguous()
        masks = torch.zeros(1, T, 1, H, W)
        masks[..., H // 4:3 * H // 4, W // 4:3 * W // 4] = 1
        masked = (frames * (1 - masks)).contiguous()
        for nearest in (True, False):
            ref_f, ref_m = generator_ref.img_propagation(masked, ff, fb, masks, "nearest" if nearest else "bilinear")
            of, om = ops.img_prop_scan(masked[0].to(DEV), ff[0].to(DEV), fb[0].to(DEV), masks[0].to(DEV), nearest)
            assert 0.02 < ref_m.mean() < masks.mean()
            assert (om.cpu() != ref_m[0]).float().mean() < 2e-3
            assert ((of.cpu() - ref_f[0]).abs() > 1e-5).float().mean() < 5e-3


def test_prop_cond():
    from propainter_b200 import ops
    gen = torch.Generator().manual_seed(1)
    h, w, C = 30, 54, 128
    cur, prop = torch.randn(h, w, C, generator=gen), torch.randn(h, w, C, generator=gen)
    f1 = smooth_flow(gen, 1, h * 8, w * 8, 3.0)[0, :, ::8, ::8].contiguous()
    f2 = (-f1 + 0.4 * torch.randn(2, h, w, generator=gen)).contiguous()
    m = (torch.rand(h, w, 2, generator=gen) > 0.5).float()
    cond = torch.full((h, w, 2 * C + 8), 7.0, device=DEV)
    bb = torch.full((h, w, 2 * C + 4), 7.0, device=DEV)
    fpi, fci = f1.permute(1, 2, 0).contiguous().to(DEV), f2.permute(1, 2, 0).contiguous().to(DEV)
    ops.prop_cond(cur.to(DEV), prop.to(DEV), fpi, fci, m.to(DEV), cond, bb, False)
    valid = ops_ref.fb_consistency(f1[None], f2[None])[0, 0]
    warped = ops_ref.flow_warp(prop.permute(2, 0, 1)[None], f1.permute(1, 2, 0)[None])[0].permute(1, 2, 0)
    c, b = cond.cpu(), bb.cpu()
    assert torch.equal(c[..., :C], cur) and torch.allclose(c[..., C:2 * C], warped, atol=1e-5)
    assert torch.equal(c[..., 2 * C:2 * C + 2], fpi.cpu()) and (c[..., 2 * C + 2] != valid).float().mean() < 5e-3
    assert torch.equal(c[..., 2 * C + 3:2 * C + 5], m) and (c[..., 2 * C + 5:] == 0).all()
    assert torch.equal(b[..., :C], cur) and torch.equal(b[..., 2 * C:2 * C + 2], m) and (b[..., 2 * C + 2:] == 0).all()
    assert (b[..., C:2 * C] == 7).all()
    ops.prop_cond(cur.to(DEV), None, None, None, m.to(DEV), None, bb, True)
    assert torch.equal(bb.cpu()[..., C:2 * C], cur)


def test_corr_build_pool_lookup():
    from propainter_b200 import ops
    gen = torch.Generator().manual_seed(2)
    for (h, w) in ((16, 22), (30, 54)):
        F_, D = 3, 256
        fm = torch.randn(F_, D, h, w, generator=gen)
        idx1, idx2 = [0, 1, 1, 2], [1, 0, 2, 1]
        pyr = ops_ref.corr_pyramid(fm[idx1], fm[idx2])
        fmap = fm.permute(0, 2, 3, 1).reshape(F_, h * w, D).contiguous().to(DEV)
        levels = ops.corr_alloc(len(idx1), h, w, DEV)
        ops.corr_build(fmap, torch.tensor(idx1, dtype=torch.int32, device=DEV), torch.tensor(idx2, dtype=torch.int32, device=DEV),
                       levels, h, w)
        hl, wl = h, w
        for l in range(4):
            got = levels[l].cpu()[:, :, :wl]
            ref = pyr[l][:, 0]
            assert torch.allclose(got, ref, atol=2e-5 * ref.abs().max().item(), rtol=1e-5), (l, (got - ref).abs().max())
            hl, wl = hl // 2, wl // 2
        B = len(idx1)
        ys, xs = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
        coords = torch.stack([xs, ys], 0).float()[None].repeat(B, 1, 1, 1) + torch.randn(B, 2, h, w, generator=gen) * 6
        ref = ops_ref.corr_lookup(pyr, coords)
        cpm = coords.permute(0, 2, 3, 1).contiguous().to(DEV)
        for tma in (True, False):
            got = ops.corr_lookup(levels, cpm, tma=tma).cpu().permute(0, 3, 1, 2)
            assert torch.allclose(got, ref, atol=1e-4, rtol=1e-4), (tma, (got - ref).abs().max())
        far = cpm.clone()
        far[0, :2] += 500.0                      # centres far outside the image -> all-zero windows, no faults
        far[1, :2] -= 500.0
        a, b = ops.corr_lookup(levels, far, tma=True), ops.corr_lookup(levels, far, tma=False)
        assert torch.allclose(a, b, atol=1e-5, rtol=1e-5) and (a[0, :2] == 0).all() and (a[1, :2] == 0).all()


def test_convex_upsample():
    from propainter_b200 import ops
    gen = torch.Generator().manual_seed(3)
    n, h, w = 3, 16, 18
    flow = torch.randn(n, 2, h, w, generator=gen) * 3
    mask = torch.randn(n, 576, h, w, generator=gen) * 4
    ref = ops_ref.convex_upsample(flow, 0.25 * mask)
    got = ops.convex_upsample(mask.permute(0, 2, 3, 1).contiguous().to(DEV), flow.permute(0, 2, 3, 1).contiguous().to(DEV), 0.25)
    assert torch.allclose(got.cpu(), ref, atol=1e-5, rtol=1e-5)


def test_gen_prep_and_window_mask():
    from propainter_b200 import ops
    from propainter_b200.window_index import padded_grid, token_grid
    gen = torch.Generator().manual_seed(4)
    for (H, W) in ((240, 432), (128, 128)):
        t, lt = 5, 3
        ff, fb = torch.randn(lt - 1, 2, H, W, generator=gen), torch.randn(lt - 1, 2, H, W, generator=gen)
        mi = torch.zeros(t, 1, H, W)
        mi[:, :, H // 3:H // 3 + 30, W // 2:W // 2 + 40] = 1
        mu = (torch.rand(t, 1, H, W, generator=gen) > 0.7).float() * mi
        dsf, dsb, pmask = ops.gen_prep(ff.to(DEV), fb.to(DEV), mi.to(DEV), mu.to(DEV), lt)
        ref_f = F.interpolate(ff, scale_factor=0.25, mode="bilinear", align_corners=False) / 4.0
        assert torch.allclose(dsf.cpu().permute(0, 3, 1, 2), ref_f, atol=1e-6)
        ref_b = F.interpolate(fb, scale_factor=0.25, mode="bilinear", align_corners=False) / 4.0
        assert torch.allclose(dsb.cpu().permute(0, 3, 1, 2), ref_b, atol=1e-6)
        dm = F.interpolate(mi[:lt], scale_factor=0.25, mode="nearest")
        du = F.interpolate(mu[:lt], scale_factor=0.25, mode="nearest")
        assert torch.equal(pmask.cpu()[..., 0], dm[:, 0]) and torch.equal(pmask.cpu()[..., 1], du[:, 0])
        h, w = H // 4, W // 4
        fh, fw = token_grid((h, w))
        H2, W2 = padded_grid(fh, fw)
        flags = ops.window_mask(pmask, fh, fw, H2 // 5, W2 // 9).cpu()
        mp = F.max_pool2d(dm, (7, 7), (3, 3), (3, 3))
        mp = F.pad(mp, (0, W2 - fw, 0, H2 - fh))
        ref = (F.max_pool2d(mp, (5, 9), (5, 9)).view(lt, -1).sum(0) > 0).int()
        assert torch.equal(flags, ref) and 0 < ref.sum() < ref.numel()


def test_deform_align():
    from propainter_b200 import ops
    gen = torch.Generator().manual_seed(5)
    for Cin, use_flow, max_res, (H, W) in ((128, True, 3.0, (60, 108)), (256, False, 5.0, (30, 54)), (128, True, 3.0, (7, 10))):
        Co = 128
        x = torch.randn(1, Cin, H, W, generator=gen)
        o = torch.randn(1, 432, H, W, generator=gen) * 1.5
        flow = torch.randn(1, 2, H, W, generator=gen) * 2
        wgt = torch.randn(Co, Cin, 3, 3, generator=gen) / (Cin * 9) ** 0.5
        bias = torch.randn(Co, generator=gen)
        o1, o2, m = torch.chunk(o, 3, dim=1)
        offset = max_res * torch.tanh(torch.cat((o1, o2), 1))
        if use_flow:
            offset = offset + flow.flip(1).repeat(1, 144, 1, 1)
        ref = ops_ref.deform_conv3x3(x, offset, torch.sigmoid(m), wgt, bias)[0]
        # x lives inside a wider buffer (channel slice) like in the scan, output goes into a slice too
        xbuf = torch.zeros(H, W, Cin + 128, device=DEV)
        xbuf[..., :Cin] = x[0].permute(1, 2, 0).to(DEV)
        out = torch.zeros(H, W, 260, device=DEV)
        fl = flow[0].permute(1, 2, 0).contiguous().to(DEV) if use_flow else None
        ops.deform_align(xbuf[..., :Cin], o[0].permute(1, 2, 0).contiguous().to(DEV), fl, max_res,
                         ops.pack_deform_weight(wgt).to(DEV), bias.to(DEV), out[..., 128:256])
        got = out[..., 128:256].cpu().permute(2, 0, 1)
        scale = ref.abs().max().item()
        assert (got - ref).abs().max().item() < 2e-3 * scale, ((got - ref).abs().max().item(), scale)
        assert (out[..., :128] == 0).all() and (out[..., 256:] == 0).all()
        # same result when the offset-net bias is folded into the tap pre-pass instead of being pre-added
        ob = torch.randn(432, generator=gen) * 0.3
        out2 = torch.zeros(H, W, 128, device=DEV)
        ops.deform_align(xbuf[..., :Cin], (o[0].permute(1, 2, 0) - ob).contiguous().to(DEV), fl, max_res,
                         ops.pack_deform_weight(wgt).to(DEV), bias.to(DEV), out2, o_bias=ob.to(DEV))
        assert (out2.cpu().permute(2, 0, 1) - ref).abs().max().item() < 2e-3 * scale


def test_conv_umma_matches_torch_conv():
    """pp_conv2d_umma (wgmma implicit GEMM, TMA-staged shifted halo boxes) vs F.conv2d in fp32.  `exact`: operands that are
    exactly representable in TF32, so every product is exact and only the fp32 accumulation order differs (1e-5 of the
    output scale: any indexing / swizzle / segment-order mistake is O(1)); `plain`: arbitrary fp32 activations reach the
    tensor core truncated to TF32 (3e-3 of the output scale; 1.7e-3 measured at K = 1280)."""
    from propainter_b200 import ops
    gen = torch.Generator().manual_seed(11)
    cases = [  # n, H, W, segment channels, Cout, KH, KW, act, pre, res, post_relu, bn, tile_w (negative: 64-pixel tiles of that width)
        (1, 30, 54, [128], 128, 3, 3, "leaky", True, True, False, 0, 0),          # flow-completion step conv
        (1, 60, 108, [128], 432, 3, 3, "none", False, False, False, 0, 0),        # conv_offset.6 (ragged last N tile)
        (2, 30, 54, [128, 128], 128, 3, 3, "leaky", True, False, False, 64, 16),  # two state segments, 8x16 tiles
        (3, 17, 23, [128, 5], 36, 3, 3, "relu", False, True, True, 32, 0),        # ragged map, 5-channel segment, Cout < BN
        (1, 60, 108, [264], 128, 3, 3, "sigmoid", False, False, False, 128, 0),   # channels not a multiple of 32
        (1, 30, 54, [2304], 128, 1, 1, "none", False, False, False, 0, 0),        # deformable-conv GEMM over sampled columns
        (2, 30, 54, [256], 128, 1, 5, "tanh", False, False, False, 0, 0),         # SepConvGRU shapes
        (2, 30, 54, [256], 128, 5, 1, "none", False, False, False, 0, 0),
        (1, 30, 54, [160, 96], 128, 1, 1, "none", False, True, False, 0, 0),       # 1x1, grouped k-blocks, ragged segment ends
        (1, 30, 54, [128, 128], 128, 3, 3, "leaky", True, True, False, 64, -8),   # M = 64 tiles (8x8 pixels)
        (2, 33, 21, [128], 432, 3, 3, "none", False, False, False, 128, -16),     # M = 64 tiles (4x16 pixels), ragged map
    ]
    for (n, H, W, segC, Cout, KH, KW, act, use_pre, use_res, post_relu, bn, tile_w) in cases:
        Cin = sum(segC)
        w = torch.randn(Cout, Cin, KH, KW, generator=gen) / (Cin * KH * KW) ** 0.5
        b = torch.randn(Cout, generator=gen)
        bufs = [torch.randn(n, H, W, (C + 11) // 4 * 4, generator=gen).to(DEV) for C in segC]      # segments = channel slices of wider buffers
        pre = torch.randn(n, H, W, Cout + 4, generator=gen).to(DEV)[..., :Cout] if use_pre else None
        res = torch.randn(n, H, W, Cout + 8, generator=gen).to(DEV)[..., 4:4 + Cout] if use_res else None
        for mode, tol in (("exact", 3e-5), ("plain", 3e-3)):
            if mode == "exact":
                xs = [ops.tf32_round(bf)[..., 4:4 + C] for bf, C in zip(bufs, segC)]
                wr = ops.tf32_round(w)
            else:
                xs, wr = [bf[..., 4:4 + C] for bf, C in zip(bufs, segC)], w
            outbuf = torch.zeros(n, H, W, Cout + 12, device=DEV)
            out = outbuf[..., 8:8 + Cout]
            ops.conv_umma(xs, ops.pack_conv_weight(wr, segC).to(DEV), KH, KW, Cout, bias=b.to(DEV), act=act, slope=0.1, pre=pre, res=res,
                          post_relu=post_relu, out=out, bn=bn, tile_w=abs(tile_w), tile_m=64 if tile_w < 0 else 0)
            ref = F.conv2d(torch.cat(xs, -1).permute(0, 3, 1, 2), wr.to(DEV), b.to(DEV), padding=(KH // 2, KW // 2)).permute(0, 2, 3, 1)
            if pre is not None:
                ref = ref + pre
            ref = {"none": lambda v: v, "relu": torch.relu, "leaky": lambda v: F.leaky_relu(v, 0.1), "sigmoid": torch.sigmoid,
                   "tanh": torch.tanh}[act](ref)
            if res is not None:
                ref = ref + res
            if post_relu:
                ref = torch.relu(ref)
            err = ((out - ref).abs().max() / ref.abs().max()).item()
            assert err < tol, (mode, n, H, W, segC, Cout, KH, KW, err)
            assert (outbuf[..., :8] == 0).all() and (outbuf[..., 8 + Cout:] == 0).all()      # nothing written outside the slice
    # round_tf32: stored activations are TF32 values (the next conv's operands are then round-to-nearest, not truncated)
    x = torch.randn(1, 16, 8, 32, generator=gen).to(DEV)
    w = torch.randn(32, 32, 3, 3, generator=gen) * 0.1
    y = ops.conv_umma([x], ops.pack_conv_weight(w).to(DEV), 3, 3, 32, round_tf32=True)
    assert torch.equal(y, ops.tf32_round(y))
    with pytest.raises(RuntimeError):
        ops.conv_umma([x], ops.pack_conv_weight(torch.randn(32, 64, 3, 3)).to(DEV), 3, 3, 32)   # packed weight / segment mismatch


def test_deform_gather_plus_gemm():
    """pp_deform_gather + 1x1 pp_conv2d_umma = torchvision.ops.deform_conv2d as DeformableAlignment /
    SecondOrderDeformableAlignment call it (same cases as test_deform_align, plus the split two-state input)."""
    from propainter_b200 import ops
    gen = torch.Generator().manual_seed(5)
    for Cin, use_flow, max_res, (H, W), split in ((128, True, 3.0, (60, 108), False), (256, False, 5.0, (30, 54), True),
                                                  (256, False, 5.0, (30, 54), False), (128, True, 3.0, (7, 10), False)):
        x = torch.randn(2, Cin, H, W, generator=gen)
        o = torch.randn(2, 432, H, W, generator=gen) * 1.5
        flow = torch.randn(2, 2, H, W, generator=gen) * 2
        wgt = torch.randn(128, Cin, 3, 3, generator=gen) / (Cin * 9) ** 0.5
        bias, ob = torch.randn(128, generator=gen), torch.randn(432, generator=gen) * 0.3
        o1, o2, m = torch.chunk(o, 3, dim=1)
        offset = max_res * torch.tanh(torch.cat((o1, o2), 1))
        if use_flow:
            offset = offset + flow.flip(1).repeat(1, 144, 1, 1)
        ref = ops_ref.deform_conv3x3(x, offset, torch.sigmoid(m), wgt, bias).permute(0, 2, 3, 1)
        xp = x.permute(0, 2, 3, 1).contiguous().to(DEV)
        op = (o.permute(0, 2, 3, 1) - ob).contiguous().to(DEV)
        fl = flow.permute(0, 2, 3, 1).contiguous().to(DEV) if use_flow else None
        if split:
            a, b = xp[..., :Cin // 2].contiguous(), xp[..., Cin // 2:].contiguous()
            cols = ops.deform_gather(a, op, fl, max_res, o_bias=ob.to(DEV), x2=b)
        else:
            cols = ops.deform_gather(xp, op, fl, max_res, o_bias=ob.to(DEV))
        out = ops.conv_umma([cols], ops.pack_deform_weight_umma(wgt).to(DEV), 1, 1, 128, bias=bias.to(DEV))
        scale = ref.abs().max().item()
        assert (out.cpu() - ref).abs().max().item() < 2e-3 * scale, ((out.cpu() - ref).abs().max().item(), scale)


def test_flow_warp_fbcheck():
    from propainter_b200 import ops
    gen = torch.Generator().manual_seed(6)
    n, h, w, C = 3, 30, 54, 128
    feat = torch.randn(n, h, w, C, generator=gen)
    f1 = smooth_flow(gen, n, h, w, 2.0)
    f2 = (-f1 + 0.5 * torch.randn(n, 2, h, w, generator=gen)).contiguous()
    ref_w = ops_ref.flow_warp(feat.permute(0, 3, 1, 2), f1.permute(0, 2, 3, 1)).permute(0, 2, 3, 1)
    ref_v = ops_ref.fb_consistency(f1, f2)[:, 0]
    aux = torch.zeros(n, h, w, 8, device=DEV)
    warped, _ = ops.flow_warp_fbcheck(feat.to(DEV), f1.permute(0, 2, 3, 1).contiguous().to(DEV), f2.permute(0, 2, 3, 1).contiguous().to(DEV),
                                      aux=aux[..., :3])
    assert (warped.cpu() - ref_w).abs().max() < 1e-5
    assert torch.equal(aux[..., :2].cpu(), f1.permute(0, 2, 3, 1)) and (aux[..., 3:] == 0).all()
    assert 0.02 < ref_v.mean() < 0.98 and (aux[..., 2].cpu() != ref_v).float().mean() < 2e-3
    w2, none = ops.flow_warp_fbcheck(feat.to(DEV), f1.permute(0, 2, 3, 1).contiguous().to(DEV), round_tf32=True)
    assert none is None and torch.equal(w2, ops.tf32_round(warped))


def test_sparse_window_attention():
    """Attention core vs the oracle's window_attention with identity-free weights: we feed q/k/v projections
    computed by torch on the device and compare the pre-`proj` output through the oracle's own formula."""
    from propainter_b200 import ops
    from propainter_b200.window_index import padded_grid, window_key_table
    gen = torch.Generator().manual_seed(6)
    C = 512
    for (t, lt, fh, fw, masked_cols) in ((4, 3, 20, 36, (10, 20)), (5, 2, 11, 11, (0, 5)), (3, 3, 20, 36, None)):
        sd = {}
        for n in ("query", "key", "value", "proj"):
            sd[f"a.{n}.weight"] = torch.randn(C, C, generator=gen) / math.sqrt(C)
            sd[f"a.{n}.bias"] = torch.randn(C, generator=gen) * 0.1
        sd["a.proj.weight"] = torch.eye(C)
        sd["a.proj.bias"] = torch.zeros(C)
        sd["a.pool_layer.weight"] = torch.randn(C, 1, 4, 4, generator=gen) / 4
        sd["a.pool_layer.bias"] = torch.randn(C, generator=gen) * 0.1
        x = torch.randn(1, t, fh, fw, C, generator=gen)
        mask = torch.zeros(1, lt, fh, fw, 1)
        if masked_cols is not None:
            mask[:, :, 2:9, masked_cols[0]:masked_cols[1]] = 1
        H2, W2 = padded_grid(fh, fw)
        for layer in (0, 1):
            t_ind = torch.arange(layer % 2, t, 2)
            ref = generator_ref.window_attention(sd, "a", x, mask, t_ind)[0]          # [t,fh,fw,C] (proj = identity)
            xp = F.pad(x[0], (0, 0, 0, W2 - fw, 0, H2 - fh)).to(DEV)
            wqkv = torch.cat([sd["a.query.weight"], sd["a.key.weight"], sd["a.value.weight"]], 0).to(DEV)
            bqkv = torch.cat([sd["a.query.bias"], sd["a.key.bias"], sd["a.value.bias"]], 0).to(DEV)
            qkv = F.linear(xp, wqkv, bqkv).view(t, H2 * W2, 3 * C)
            pooled = F.conv2d(xp.permute(0, 3, 1, 2), sd["a.pool_layer.weight"].to(DEV), sd["a.pool_layer.bias"].to(DEV),
                              stride=4, groups=C).permute(0, 2, 3, 1).reshape(t, -1, C)
            pool_kv = F.linear(pooled, wqkv[C:], bqkv[C:]).contiguous()
            mp = F.pad(mask[0, ..., 0], (0, W2 - fw, 0, H2 - fh))
            flags = (F.max_pool2d(mp[:, None], (5, 9), (5, 9)).view(lt, -1).sum(0) > 0).int().to(DEV)
            ktab = torch.from_numpy(window_key_table(H2, W2)).to(DEV)
            for impl in ("umma", "mma"):
                got = ops.sparse_window_attn(qkv, pool_kv, ktab, flags, t, H2 * W2, layer % 2, 2, impl=impl)
                got = got.view(t, H2, W2, C)[:, :fh, :fw].cpu()
                scale = ref.abs().max().item()
                err = (got - ref).abs().max().item()
                assert err < 3e-3 * scale, (impl, t, fh, fw, layer, err, scale)


def test_ffn_overlap_add():
    from propainter_b200 import ops
    gen = torch.Generator().manual_seed(7)
    for (h, w) in ((60, 108), (32, 32)):
        frames, CH = 3, 40
        fh, fw = (h - 1) // 3 + 1, (w - 1) // 3 + 1
        n = frames * fh * fw
        Y = torch.randn(n, 49 * CH, generator=gen)
        norm = F.fold(torch.ones(frames, 49, fh * fw), (h, w), (7, 7), padding=3, stride=3)
        y = F.fold(Y.view(frames, fh * fw, 49 * CH).permute(0, 2, 1), (h, w), (7, 7), padding=3, stride=3)
        ref = F.gelu(F.unfold(y / norm, (7, 7), padding=3, stride=3).permute(0, 2, 1).reshape(n, 49 * CH))
        perm = torch.arange(49 * CH).view(CH, 49).t().reshape(-1)
        Z = ops.ffn_overlap_add(Y[:, perm].contiguous().to(DEV), frames, h, w, CH).cpu()
        assert torch.allclose(Z, ref[:, perm], atol=1e-5, rtol=1e-5)


def test_bias_act_and_upsample2x():
    from propainter_b200 import ops
    gen = torch.Generator().manual_seed(10)
    x = torch.randn(3, 17, 23, 64, generator=gen)
    b = torch.randn(64, generator=gen)
    refs = {"none": x + b, "relu": F.relu(x + b), "leaky": F.leaky_relu(x + b, 0.1), "sigmoid": torch.sigmoid(x + b),
            "tanh": torch.tanh(x + b)}
    for act, ref in refs.items():
        got = ops.bias_act_(x.clone().to(DEV), b.to(DEV), act, 0.1).cpu()
        assert torch.allclose(got, ref, atol=2e-6, rtol=1e-6), act
    for (n, h, w, C) in ((2, 30, 54, 128), (1, 15, 27, 32)):
        z = torch.randn(n, C, h, w, generator=gen)
        ref = F.interpolate(z, scale_factor=2, mode="bilinear", align_corners=True)
        got = ops.upsample2x(z.permute(0, 2, 3, 1).contiguous().to(DEV)).cpu().permute(0, 3, 1, 2)
        assert torch.allclose(got, ref, atol=1e-6, rtol=1e-6)


def test_bias_act_strided_residual_and_instance_norm():
    """pp_bias_act with channel-slice views (x / res / out each a slice of a wider pixel-major buffer), residual add and
    final ReLU vs plain torch; pp_instance_norm vs F.instance_norm (+ReLU, +residual, in place) on the three channel
    counts of the RAFT feature encoder.  Tolerance 2e-5 abs on O(1) values (fp32 sums, double fold of the partials)."""
    from propainter_b200 import ops
    g = torch.Generator().manual_seed(5)
    X, R, O = (torch.randn(2, 9, 13, 48, generator=g).to(DEV) for _ in range(3))
    bias = torch.randn(16, generator=g).to(DEV)
    for act, fn in (("leaky", lambda t: F.leaky_relu(t, 0.1)), ("relu", F.relu), ("none", lambda t: t), ("tanh", torch.tanh)):
        for post in (False, True):
            x, r, o = X[..., 16:32], R[..., 32:48], O.clone()
            want = fn(x + bias) + r
            want = F.relu(want) if post else want
            ops.bias_act(x, bias, act, 0.1, res=r, post_relu=post, out=o[..., 0:16])
            assert torch.allclose(o[..., 0:16], want, atol=1e-6) and torch.equal(o[..., 16:], O[..., 16:])
            # pp_bias_act_pre: per-pixel pre-activation addend (a hoisted conv share), also a channel slice
            pre = R[..., 0:16]
            want = fn(x + bias + pre) + r
            want = F.relu(want) if post else want
            o = O.clone()
            ops.bias_act(x, bias, act, 0.1, res=r, post_relu=post, out=o[..., 0:16], pre=pre)
            assert torch.allclose(o[..., 0:16], want, atol=1e-6) and torch.equal(o[..., 16:], O[..., 16:])
    y = X[..., :16].clone()
    assert torch.allclose(ops.bias_act(y, None, "relu"), F.relu(X[..., :16]), atol=0)          # no bias, in place
    for n, h, w, C in ((3, 40, 56, 64), (2, 20, 27, 96), (5, 9, 14, 128), (1, 3, 5, 64)):
        x = (torch.randn(n, h, w, C, generator=g) * 2 + torch.randn(1, 1, 1, C, generator=g) * 3).to(DEV)
        res = torch.randn(n, h, w, C, generator=g).to(DEV)
        ref = F.instance_norm(x.permute(0, 3, 1, 2), eps=1e-5).permute(0, 2, 3, 1)
        assert torch.allclose(ops.instance_norm(x), ref, atol=2e-5)
        assert torch.allclose(ops.instance_norm(x, relu=True), F.relu(ref), atol=2e-5)
        want = F.relu(res + F.relu(ref))
        xin = x.clone()
        got = ops.instance_norm(xin, relu=True, res=res, post_relu=True, out=xin)
        assert got.data_ptr() == xin.data_ptr() and torch.allclose(got, want, atol=2e-5)


def test_transformer_glue_kernels():
    """pp_pool_depthwise vs F.conv2d(groups=C, kernel=stride) (sparse_transformer.py:131-133) and pp_add_layernorm vs
    x + d followed by F.layer_norm (:322-334); fp32, 1e-5."""
    from propainter_b200 import ops
    g = torch.Generator().manual_seed(6)
    for (n, H, W, C, kh, kw) in ((3, 20, 36, 512, 4, 4), (2, 15, 18, 128, 4, 4), (1, 10, 9, 64, 2, 3)):
        x = torch.randn(n, H, W, C, generator=g)
        w, b = torch.randn(C, 1, kh, kw, generator=g) * 0.3, torch.randn(C, generator=g)
        ref = F.conv2d(x.permute(0, 3, 1, 2), w, b, stride=(kh, kw), groups=C).permute(0, 2, 3, 1)
        got = ops.pool_depthwise(x.to(DEV), w.reshape(C, -1).t().contiguous().to(DEV), b.to(DEV), kh, kw).cpu()
        assert got.shape == ref.shape and torch.allclose(got, ref, atol=1e-5, rtol=1e-5)
    for (rows, C) in (((3, 20, 36), 512), ((7, 5), 128), ((1, 1), 1024)):
        x, d = torch.randn(*rows, C, generator=g) * 2 + 0.5, torch.randn(*rows, C, generator=g)
        ga, be = torch.randn(C, generator=g), torch.randn(C, generator=g)
        xo, y = ops.add_layernorm(x.to(DEV), d.to(DEV), ga.to(DEV), be.to(DEV))
        assert torch.equal(xo.cpu(), x + d) and torch.allclose(y.cpu(), F.layer_norm(x + d, (C,), ga, be), atol=1e-5, rtol=1e-5)
        x2, y2 = ops.add_layernorm(x.to(DEV), None, ga.to(DEV), be.to(DEV))
        assert torch.equal(x2.cpu(), x) and torch.allclose(y2.cpu(), F.layer_norm(x, (C,), ga, be), atol=1e-5, rtol=1e-5)


def test_gru_fusion_kernels():
    """SepConvGRU elementwise rules (RAFT/update.py:45-60) on slices of the persistent HX / RX buffers."""
    from propainter_b200 import ops
    gen = torch.Generator().manual_seed(11)
    B, h, w, C = 2, 9, 13, 128
    HX, RX = torch.randn(B, h, w, 384, generator=gen), torch.randn(B, h, w, 384, generator=gen)
    zr, q = torch.randn(B, h, w, 2 * C, generator=gen) * 2, torch.randn(B, h, w, C, generator=gen) * 2
    bzr, bq = torch.randn(2 * C, generator=gen), torch.randn(C, generator=gen)
    mot, flow = torch.randn(B, h, w, 128, generator=gen), torch.randn(B, h, w, 2, generator=gen)
    hx, rx = HX.to(DEV), RX.to(DEV)
    z = torch.empty(B, h, w, C, device=DEV)
    ops.gru_gate(zr.to(DEV), bzr.to(DEV), hx[..., :C], z, rx[..., :C])
    g = torch.sigmoid(zr + bzr)
    assert torch.allclose(z.cpu(), g[..., :C], atol=2e-6) and torch.allclose(rx.cpu()[..., :C], g[..., C:] * HX[..., :C], atol=5e-6)
    assert torch.equal(rx.cpu()[..., C:], RX[..., C:]) and torch.equal(hx.cpu(), HX)
    netc = torch.empty(B, h, w, C, device=DEV)
    ops.gru_update(q.to(DEV), bq.to(DEV), z, hx[..., :C], net_copy=netc)
    ref = (1 - g[..., :C]) * HX[..., :C] + g[..., :C] * torch.tanh(q + bq)
    assert torch.allclose(hx.cpu()[..., :C], ref, atol=5e-6) and torch.equal(hx.cpu()[..., C:], HX[..., C:])
    assert torch.equal(netc, hx[..., :C])
    ops.raft_pack_motion(mot.to(DEV), flow.to(DEV), hx[..., 256:], rx[..., 256:])
    want = torch.cat([mot[..., :126], flow], -1)
    assert torch.equal(hx.cpu()[..., 256:], want) and torch.equal(rx.cpu()[..., 256:], want)
    assert torch.equal(hx.cpu()[..., C:256], HX[..., C:256])
    # iteration-invariant addend `pre` instead of the per-channel bias (context-channel share of the gate convs)
    pz, pq = torch.randn(B, h, w, 2 * C, generator=gen), torch.randn(B, h, w, C, generator=gen)
    hx2, rx2, z2 = HX.to(DEV), RX.to(DEV), torch.empty(B, h, w, C, device=DEV)
    ops.gru_gate(zr.to(DEV), None, hx2[..., :C], z2, rx2[..., :C], pre=pz.to(DEV))
    g2 = torch.sigmoid(zr + pz)
    assert torch.allclose(z2.cpu(), g2[..., :C], atol=2e-6) and torch.allclose(rx2.cpu()[..., :C], g2[..., C:] * HX[..., :C], atol=5e-6)
    ops.gru_update(q.to(DEV), None, z2, hx2[..., :C], pre=pq.to(DEV))
    assert torch.allclose(hx2.cpu()[..., :C], (1 - g2[..., :C]) * HX[..., :C] + g2[..., :C] * torch.tanh(q + pq), atol=5e-6)
    bm = torch.randn(128, generator=gen)
    ops.raft_pack_motion(mot.to(DEV), flow.to(DEV), hx[..., 256:], rx[..., 256:], bias=bm.to(DEV))   # raw conv output in
    want = torch.cat([F.relu(mot + bm)[..., :126], flow], -1)
    assert torch.allclose(hx.cpu()[..., 256:], want, atol=1e-6) and torch.equal(rx[..., 256:], hx[..., 256:])


def test_u8_and_composite():
    from oracle import pipeline_ref
    from propainter_b200 import ops
    gen = torch.Generator().manual_seed(8)
    T, H, W = 5, 24, 40
    u8 = torch.randint(0, 256, (T, H, W, 3), generator=gen, dtype=torch.uint8)
    assert torch.equal(ops.u8_to_frames(u8.to(DEV)).cpu(), pipeline_ref.to_float_frames(u8.numpy())[0])
    masks = (torch.rand(T, 1, H, W, generator=gen) > 0.5).float()
    comp = torch.zeros(T, H, W, 3, dtype=torch.uint8, device=DEV)
    ref = [None] * T
    for ids in ([0, 1, 2], [1, 2, 3], [2, 3, 4], [2]):
        pred = torch.rand(len(ids), 3, H, W, generator=gen) * 2 - 1
        first = [ref[i] is None for i in ids]
        pr = ((pred + 1) / 2).permute(0, 2, 3, 1).numpy() * 255
        bm = masks[ids].permute(0, 2, 3, 1).numpy().astype(np.uint8)
        for k, i in enumerate(ids):
            img = np.array(pr[k]).astype(np.uint8) * bm[k] + u8[i].numpy() * (1 - bm[k])
            ref[i] = img if ref[i] is None else (ref[i].astype(np.float32) * 0.5 + img.astype(np.float32) * 0.5)
            ref[i] = ref[i].astype(np.uint8)
        ops.composite_blend(pred.to(DEV), masks.to(DEV), u8.to(DEV), comp, ids, first)
    assert np.array_equal(comp.cpu().numpy(), np.stack(ref, 0))


def test_mask_dilate():
    import scipy.ndimage
    from propainter_b200 import ops
    gen = torch.Generator().manual_seed(12)
    T, H, W = 3, 240, 432
    m = (torch.rand(T, H, W, generator=gen) > 0.999).to(torch.uint8) * 255
    for it in (0, 4):
        ref = np.stack([scipy.ndimage.binary_dilation(m[i].numpy(), iterations=it) if it else m[i].numpy() > 0 for i in range(T)])
        out = ops.mask_dilate(m.to(DEV), it).cpu()[:, 0].numpy()
        assert np.array_equal(out > 0.5, ref) and set(np.unique(out)) <= {0.0, 1.0}


def test_resize_kernels():
    """Device resizing vs the host libraries the reference calls: PIL.Image.resize (BICUBIC default) for the frames,
    Image.NEAREST for the masks, cv2.resize (INTER_LINEAR) for the output (inference_propainter.py:34-45, :95-96, :469-470)."""
    cv2 = pytest.importorskip("cv2")
    Image = pytest.importorskip("PIL.Image")
    from propainter_b200 import ops
    rng = np.random.default_rng(0)
    for (H, W, size) in ((243, 437, (432, 240)), (100, 150, (72, 48)), (37, 53, (160, 96)), (240, 432, (432, 240))):
        fr = rng.integers(0, 256, (3, H, W, 3), dtype=np.uint8)
        got = ops.resize_frames_u8(torch.from_numpy(fr).to(DEV), size).cpu().numpy()
        ref = np.stack([np.array(Image.fromarray(f, mode="RGB").resize(size)) for f in fr])
        assert np.array_equal(got, ref), (H, W, size)
        m = (rng.integers(0, 2, (2, H, W), dtype=np.uint8) * 255)
        gm = ops.resize_masks_u8(torch.from_numpy(m).to(DEV), size).cpu().numpy()
        rm = np.stack([np.array(Image.fromarray(x, mode="L").resize(size, Image.NEAREST)) for x in m])
        assert np.array_equal(gm, rm)
    for (H, W, size) in ((240, 432, (437, 243)), (64, 96, (101, 77)), (120, 200, (150, 90))):
        fr = rng.integers(0, 256, (2, H, W, 3), dtype=np.uint8)
        got = ops.resize_output_u8(torch.from_numpy(fr).to(DEV), size).cpu().numpy()
        ref = np.stack([cv2.resize(f, size) for f in fr])
        d = np.abs(got.astype(int) - ref.astype(int))
        assert d.max() <= 1 and (d > 0).mean() < 1e-3, (d.max(), (d > 0).mean())
