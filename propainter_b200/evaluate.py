"""Evaluation harness for the hot path (scripts/evaluate_propainter.py:37-257, core/metrics.py:12-62): per-frame PSNR / SSIM of
the composited video against the ground-truth frames and flow end-point error, computed on the device.

    from propainter_b200.evaluate import evaluate_clip
    res = evaluate_clip(pipe, frames_u8, masks_u8)        # {"psnr": ..., "ssim": ..., "frames_per_s": ..., per-frame lists}

PSNR: 20 log10(255 / sqrt(MSE)) over float64 (core/metrics.py:20-36).  SSIM: skimage.measure.compare_ssim(data_range=255,
multichannel=True, win_size=65) as core/metrics.py:44-47 calls it -- uniform 65x65 windows, sample covariance
(N/(N-1)), K1 = 0.01, K2 = 0.03, mean over the positions whose window lies inside the image and over the channels; restated
from scikit-image's published `structural_similarity` (third-party dependency, not installed here; pinned against a direct
numpy evaluation of the same definition in tests/test_evaluate.py).  VFID: `evaluate_clip` takes an `i3d_activations`
callable; `i3d_activations(model, frames_u8)` below is the reference's calculate_i3d_activations (core/metrics.py:70-82)
on this package's InceptionI3d (propainter_b200.model.i3d), and `video_completion_summary` gives the script's final
PSNR / SSIM / VFID line, FID computed as core/metrics.py:85-150 does.

    i3d = InceptionI3d(400, in_channels=3, final_endpoint='Logits').to("cuda")
    i3d.load_state_dict(torch.load("weights/i3d_rgb_imagenet.pt"), strict=True)
    res = [evaluate_clip(pipe, f, m, i3d_activations=functools.partial(i3d_activations, i3d)) for f, m in clips]
    video_completion_summary(res)                         # {"psnr", "ssim", "vfid", "seconds_per_frame", "videos"}"""
import time

import numpy as np
import torch
import torch.nn.functional as F


def psnr_frames(a_u8, b_u8):
    """[T,H,W,3] uint8 x2 (tensors) -> float64 tensor [T] (inf where identical)"""
    d = (a_u8.double() - b_u8.double()) ** 2
    mse = d.flatten(1).mean(1)
    return torch.where(mse == 0, torch.full_like(mse, float("inf")), 20.0 * torch.log10(255.0 / mse.sqrt()))


def ssim_frames(a_u8, b_u8, win_size=65, data_range=255.0):
    """skimage compare_ssim(multichannel=True, win_size=65, data_range=255) per frame: [T,H,W,3] uint8 x2 -> float64 [T]"""
    T, H, W, C = a_u8.shape
    if min(H, W) < win_size:
        raise ValueError("win_size exceeds image extent")
    x = a_u8.permute(0, 3, 1, 2).double().reshape(T * C, 1, H, W)
    y = b_u8.permute(0, 3, 1, 2).double().reshape(T * C, 1, H, W)
    npx = win_size * win_size
    cov_norm = npx / (npx - 1.0)
    box = lambda z: F.avg_pool2d(z, win_size, stride=1)                       # windows fully inside the image = skimage's crop
    ux, uy = box(x), box(y)
    vx = cov_norm * (box(x * x) - ux * ux)
    vy = cov_norm * (box(y * y) - uy * uy)
    vxy = cov_norm * (box(x * y) - ux * uy)
    c1, c2 = (0.01 * data_range) ** 2, (0.03 * data_range) ** 2
    s = ((2 * ux * uy + c1) * (2 * vxy + c2)) / ((ux * ux + uy * uy + c1) * (vx + vy + c2))
    return s.flatten(1).mean(1).view(T, C).mean(1)


def epe(flow1, flow2):
    """core/metrics.py:12-17: mean end-point error of two flow fields [..,2,H,W]"""
    return ((flow1 - flow2) ** 2).sum(-3).sqrt().mean().item()


def fid_from_activations(real, fake):
    """core/metrics.py:122-160 (Frechet distance of two activation sets [n, d])"""
    from scipy import linalg
    m1, m2 = real.mean(0), fake.mean(0)
    s1, s2 = np.cov(real, rowvar=False), np.cov(fake, rowvar=False)
    covmean = linalg.sqrtm(s1.dot(s2))                                     # (scipy >= 1.18 dropped the `disp` argument)
    if not np.isfinite(covmean).all():
        off = np.eye(s1.shape[0]) * 1e-6
        covmean = linalg.sqrtm((s1 + off).dot(s2 + off))
    covmean = covmean.real if np.iscomplexobj(covmean) else covmean
    d = m1 - m2
    return float(d.dot(d) + np.trace(s1) + np.trace(s2) - 2 * np.trace(covmean))


@torch.no_grad()
def evaluate_clip(pipe, frames_u8, masks_u8, cfg=None, mask_dilation=0, i3d_activations=None):
    """The per-video body of scripts/evaluate_propainter.py:95-215 for the `video_completion` task: inpaint `frames_u8`
    ([T,H,W,3] uint8, numpy or tensor) under `masks_u8` ([T,H,W], non-zero = hole) and score the result against the input
    frames.  Returns metrics + timing (synchronised wall time of stages 1-4 incl. compositing, as :100-101,181-184)."""
    from .inference_propainter import InferenceConfig, prepare_masks
    dev = pipe.device
    fr = torch.as_tensor(frames_u8).to(dev)
    mk = torch.as_tensor(masks_u8).to(dev)
    mk = ((mk != 0).to(torch.uint8) * 255).contiguous()
    fm, md = prepare_masks(mk, mask_dilation, dev)
    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    comp = pipe(fr, fm, md, cfg or InferenceConfig())
    torch.cuda.synchronize(dev)
    dt = time.perf_counter() - t0
    ps, ss = psnr_frames(fr, comp), ssim_frames(fr, comp)
    out = {"psnr": ps[torch.isfinite(ps)].mean().item() if torch.isfinite(ps).any() else float("inf"), "ssim": ss.mean().item(),
           "psnr_per_frame": ps.tolist(), "ssim_per_frame": ss.tolist(), "seconds": dt, "frames_per_s": fr.shape[0] / dt, "comp": comp}
    if i3d_activations is not None:
        out["i3d"] = (i3d_activations(fr), i3d_activations(comp))
    return out


@torch.no_grad()
def i3d_activations(model, frames_u8):
    """calculate_i3d_activations (core/metrics.py:70-82) for one video: uint8 frames [T,H,W,3] (numpy or tensor) -> float32
    numpy [1024], the I3D features of the to_tensors video on `model`'s device.  A batch [B,T,H,W,3] of equally long
    videos -> [B,1024] in one pass (eval BatchNorm is per sample, so a row does not depend on the others beyond the
    rounding of the convolution algorithm cuDNN picks for that batch size)."""
    fr = torch.as_tensor(frames_u8)
    single = fr.dim() == 4
    fr = fr[None] if single else fr
    if fr.dtype != torch.uint8:
        raise ValueError(f"i3d_activations: expected uint8 frames, got {fr.dtype}")
    feats = model.features_u8(fr.to(model.device).contiguous()).cpu().numpy()
    return feats[0] if single else feats


def video_completion_summary(results):
    """The final line of scripts/evaluate_propainter.py:245-251 over evaluate_clip results (each with its "i3d" pair):
    PSNR and SSIM averaged over all frames of all videos (total_frame_psnr / total_frame_ssim, so an identical frame's inf
    carries through), VFID = calculate_vfid of the stacked per-video activations (core/metrics.py:85-96), and the mean over
    videos of seconds per frame (time_all)."""
    psnr = [p for r in results for p in r["psnr_per_frame"]]
    ssim = [s for r in results for s in r["ssim_per_frame"]]
    out = {"psnr": sum(psnr) / len(psnr), "ssim": sum(ssim) / len(ssim),
           "seconds_per_frame": sum(r["seconds"] / len(r["psnr_per_frame"]) for r in results) / len(results),
           "videos": len(results)}
    if all("i3d" in r for r in results):
        real = np.stack([np.asarray(r["i3d"][0]) for r in results])
        fake = np.stack([np.asarray(r["i3d"][1]) for r in results])
        out["vfid"] = fid_from_activations(real, fake)
    return out


def epe64(flow1, flow2):
    """calculate_epe (core/metrics.py:12-17) accumulated in float64: mean over pixels of |flow1 - flow2| for [..,2,H,W]"""
    return ((flow1.double() - flow2.double()) ** 2).sum(-3).sqrt().mean().item()


@torch.no_grad()
def evaluate_flow_clip(pipe, frames_u8, masks_u8, reference_flows=None, cfg=None, mask_dilation=4):
    """The per-video body of scripts/evaluate_flow_completion.py:88-160: RAFT flows of `frames_u8` ([T,H,W,3] uint8,
    numpy or tensor), completed by the recurrent flow-completion net under `masks_u8` ([T,H,W], non-zero = hole; made
    binary and dilated `mask_dilation` times with the 3x3 cross, as TestDataset's cv2.dilate), scored by end-point error.

    As in the script, flow completion runs once over the whole clip (no sub-video chunks), then combine_flow.
    `reference_flows` (forward, backward), each [1,T-1,2,H,W] or [T-1,2,H,W], are what EPE is measured against; without
    them the reference is the RAFT flows of the unmasked frames, what scripts/compute_flow.py stores for them.
    `seconds` is the synchronised wall time of stage 2 alone (:113-137).  Deviation: the script's short-clip branch
    hard-codes iters=20 where this uses cfg.raft_iter throughout (the default is 20).  EPE is accumulated in float64."""
    from . import ops
    from .inference_propainter import InferenceConfig, prepare_masks
    cfg = cfg or InferenceConfig()
    dev = pipe.device
    fr = torch.as_tensor(frames_u8).to(dev)
    mk = torch.as_tensor(masks_u8).to(dev)
    fm, _ = prepare_masks(((mk != 0).to(torch.uint8) * 255).contiguous(), mask_dilation, dev)
    if cfg.half_storage:                       # fp16 RAFT flows in, fp16 completed flows out (InferenceConfig.half_storage)
        gt = pipe.compute_flows_half(fr.contiguous(), cfg)
    else:
        gt =pipe.compute_flows(ops.u8_to_frames(fr).unsqueeze(0), cfg)
    net = pipe.fix_flow_complete
    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    pred, _ = net.forward_bidirect_flow(gt, fm)
    pred = net.combine_flow(gt, pred, fm)
    if cfg.half_storage:
        pred = tuple(p.half() for p in pred)
    torch.cuda.synchronize(dev)
    dt = time.perf_counter() - t0
    ref = gt if reference_flows is None else tuple(torch.as_tensor(r).to(dev).float().reshape(p.shape)
                                                   for r, p in zip(reference_flows, pred))
    ef, eb = epe64(ref[0], pred[0]), epe64(ref[1], pred[1])
    T = fr.shape[0]
    return {"epe": (ef + eb) / 2, "epe_forward": ef, "epe_backward": eb, "frames": T, "seconds": dt,
            "seconds_per_frame": dt / T, "pred_flows": pred}


def flow_epe_summary(results):
    """The dataset line of evaluate_flow_completion.py:141-178 over evaluate_flow_clip results: `epe` is the
    frame-weighted average (total_frame_epe: each direction's EPE counted once per flow), `seconds_per_frame` the mean
    stage-2 time per frame (time_all)."""
    flows = [r["frames"] - 1 for r in results]
    epe = sum(n * (r["epe_forward"] + r["epe_backward"]) for n, r in zip(flows, results)) / (2 * sum(flows))
    return {"epe": epe, "seconds_per_frame": sum(r["seconds"] for r in results) / sum(r["frames"] for r in results),
            "videos": len(results)}
