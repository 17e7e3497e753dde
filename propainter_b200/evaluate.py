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
    """[T,H,W,3] uint8 x2 (tensors) -> float64 tensor [T] (inf where identical).  Float frames (the evaluation protocol's
    blended video) are widened to float64 as they are, as calc_psnr_and_ssim does."""
    d = (a_u8.double() - b_u8.double()) ** 2
    mse = d.flatten(1).mean(1)
    return torch.where(mse == 0, torch.full_like(mse, float("inf")), 20.0 * torch.log10(255.0 / mse.sqrt()))


def ssim_frames(a_u8, b_u8, win_size=65, data_range=255.0):
    """skimage compare_ssim(multichannel=True, win_size=65, data_range=255) per frame: [T,H,W,3] uint8 x2 -> float64 [T]
    (float frames are taken at their float64 value, as for psnr_frames)"""
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
    return _complete_and_score(pipe, gt, fm, reference_flows, cfg.half_storage)


def _complete_and_score(pipe, gt, fm, reference_flows, half):
    """evaluate_flow_completion.py:111-137 + :141-147: flow completion once over the whole clip, then combine_flow, timed
    with synchronisations around it; then the EPE of each direction against `reference_flows` (None: against `gt`)."""
    dev = pipe.device
    net = pipe.fix_flow_complete
    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    pred, _ = net.forward_bidirect_flow(gt, fm)
    pred = net.combine_flow(gt, pred, fm)
    if half:
        pred = tuple(p.half() for p in pred)
    torch.cuda.synchronize(dev)
    dt = time.perf_counter() - t0
    ref = gt if reference_flows is None else tuple(torch.as_tensor(r).to(dev).float().reshape(p.shape)
                                                   for r, p in zip(reference_flows, pred))
    ef, eb = epe64(ref[0], pred[0]), epe64(ref[1], pred[1])
    T = fm.shape[1]
    return {"epe": (ef + eb) / 2, "epe_forward": ef, "epe_backward": eb, "frames": T, "seconds": dt,
            "seconds_per_frame": dt / T, "pred_flows": pred}


@torch.no_grad()
def evaluate_flow_video(pipe, masks, flows):
    """The per-video body of scripts/evaluate_flow_completion.py:88-160 with --load_flow, on prepare_test_video's outputs:
    masks float {0,1} [1,T,1,h,w], flows the loaded (forward, backward) pair [T-1,2,h,w] or [1,T-1,2,h,w].  The loaded
    flows are completed (forward_bidirect_flow + combine_flow over the whole clip) and are also what EPE is measured
    against.  Returns the record of evaluate_flow_clip: EPE per direction (float64), `seconds` = the synchronised wall
    time of the completion alone (:111-137), and the completed flows."""
    dev = pipe.device
    fm = torch.as_tensor(masks).to(dev).float()
    T, H, W = fm.shape[1], fm.shape[-2], fm.shape[-1]
    fm = fm.reshape(1, T, 1, H, W).contiguous()
    gt = tuple(torch.as_tensor(f).to(dev).float().reshape(1, T - 1, 2, H, W).contiguous() for f in flows)
    return _complete_and_score(pipe, gt, fm, None, False)


def flow_epe_summary(results):
    """The dataset line of evaluate_flow_completion.py:141-178 over evaluate_flow_clip results: `epe` is the
    frame-weighted average (total_frame_epe: each direction's EPE counted once per flow), `seconds_per_frame` the mean
    stage-2 time per frame (time_all)."""
    flows = [r["frames"] - 1 for r in results]
    epe = sum(n * (r["epe_forward"] + r["epe_backward"]) for n, r in zip(flows, results)) / (2 * sum(flows))
    return {"epe": epe, "seconds_per_frame": sum(r["seconds"] for r in results) / sum(r["frames"] for r in results),
            "videos": len(results)}


# ---------------------------------------------------------------- the evaluation script's video-completion protocol
PROTOCOL_RAFT_CLIP = 60                 # evaluate_propainter.py:108 short_len: RAFT chunks of 60 frames, 1-frame overlap


def prepare_test_video(frames_u8, masks_u8, size, flows=None, device="cuda"):
    """TestDataset.__getitem__ (core/dataset.py:173-231) after file I/O, on the device.  size = (w, h), the script's
    args.size.  frames_u8 uint8 [T,H0,W0,3] (RGB) -> [T,h,w,3] by cv2.resize(INTER_LINEAR) -- these frames are both the
    network input and the ground truth; masks_u8 uint8 [T,H0,W0] -> float {0,1} [1,T,1,h,w]: PIL NEAREST resize, > 0,
    cv2.dilate with the 3x3 cross x4; flows: an optional (forward, backward) pair of float32 [T-1,2,Hf,Wf] -> [T-1,2,h,w]
    through resize_flow (utils/flow_util.py:6-11).  Returns (frames, masks, flows or None); frames_u8 = None skips the
    frames (the flow-completion protocol reads none) and returns None in their place.  An exact 2x down-scaling of
    the frames, where OpenCV switches the 8-bit resize to INTER_AREA, raises (the uint8 kernel does not implement it)."""
    from . import ops
    w, h = (int(s) for s in size)
    dev = torch.device(device)
    fr = None if frames_u8 is None else ops.resize_output_u8(torch.as_tensor(frames_u8).to(dev).contiguous(), (w, h))
    mk = ops.resize_masks_u8(torch.as_tensor(masks_u8).to(dev).contiguous(), (w, h))
    mk = ops.mask_dilate(mk, 4).unsqueeze(0)
    if flows is not None:
        flows = tuple(ops.resize_flow(torch.as_tensor(f).to(dev).float().contiguous(), (w, h)) for f in flows)
    return fr, mk, flows


@torch.no_grad()
def warp_error(result_u8, flows):
    """The temporal warping error E_warp of Lai et al., "Learning Blind Video Temporal Consistency" (ECCV 2018), which the
    reference's README defers to for --save_results output, with the occlusion test of Ruder et al. (GCPR 2016).
    result_u8 uint8 [T,H,W,3] (the saved frames; values / 255), flows the (forward, backward) pair of the ground-truth
    clip, each [T-1,2,H,W] or [1,T-1,2,H,W] in fp32 or fp16 (RAFT's, or compute_flow_video's).  Per pair t, frame t+1
    is warped to frame t along the forward flow (border-clamped bilinear), and E_t is the mean squared RGB difference
    over the pixels the occlusion test keeps (0 if it keeps none).  One device pass (ops.warp_error_sums).

    Returns {"ewarp": mean over pairs of E_t, "ewarp_per_pair": [E_t], "occluded_fraction": share of occluded pixels
    over all pairs}, raw values (no x 1e-3).  Comparable across methods scored by this package; not digit for digit
    with published tables, which used FlowNet2 flows on frames resized to multiples of 64 (INTEGRATION.md §3)."""
    from . import ops
    fw, bw = flows
    dev = result_u8.device if isinstance(result_u8, torch.Tensor) else torch.device("cuda")
    fr = torch.as_tensor(result_u8).to(dev)
    fw, bw = (torch.as_tensor(f).to(dev) for f in (fw, bw))
    sums = ops.warp_error_sums(fr, fw, bw=bw).cpu()
    s, n = sums[:, 0].tolist(), sums[:, 1].tolist()
    per_pair = [a / (3 * k) if k > 0 else 0.0 for a, k in zip(s, n)]
    T, H, W = fr.shape[0], fr.shape[1], fr.shape[2]
    return {"ewarp": sum(per_pair) / len(per_pair), "ewarp_per_pair": per_pair,
            "occluded_fraction": 1.0 - sum(n) / ((T - 1) * H * W)}


_warp_error = warp_error            # evaluate_video's argument of the same name shadows it there


@torch.no_grad()
def evaluate_video(pipe, frames_u8, masks, flows=None, task="video_completion", neighbor_length=20, ref_stride=10,
                   raft_iter=20, i3d=None, cfg=None, warp_error=False):
    """The per-video body of scripts/evaluate_propainter.py::main_worker (:92-210) on prepare_test_video's outputs:
    frames_u8 uint8 [T,h,w,3], masks float {0,1} [1,T,1,h,w] (one mask set for flow completion, propagation, the
    generator and compositing), flows the loaded (forward, backward) pair [T-1,2,h,w] or [1,T-1,2,h,w] (--load_flow),
    or None: RAFT with `raft_iter` iterations in chunks of 60 frames overlapping by one (:108-124).

    Unlike the inference schedule (ProPainterPipeline.__call__): flow completion and image propagation run once over the
    whole clip; windows of `neighbor_length` (stride neighbor_length // 2) take every `ref_stride`-th frame of the clip
    as reference, with no cap; and the composited video stays float32 (ops.composite_blend_f32), a frame seen by several
    windows holding multiples of 1/2 or 1/4.  `seconds` is the synchronised wall time from after the upload to after
    compositing (:100-101, :181-184).  video_completion: per-frame PSNR / SSIM in float64 of the float frames against
    the input frames, and with `i3d` (an InceptionI3d) the pair (real, comp truncated to uint8) of I3D activations.
    object_removal only times.  `cfg`: an InferenceConfig for what the script leaves open (windows_in_flight); its
    schedule fields are replaced by the protocol's, and half_storage raises ValueError (the script has no such mode).
    `warp_error`: also the temporal warping error of the result (the module's warp_error, keys ewarp / ewarp_per_pair /
    occluded_fraction) on comp truncated to uint8, with the protocol's ground-truth flows (RAFT's or the loaded ones),
    which are then kept until after the timed region; either task."""
    from dataclasses import replace
    from . import ops
    from .inference_propainter import InferenceConfig
    if task not in ("video_completion", "object_removal"):
        raise ValueError(f"task must be 'video_completion' or 'object_removal', got {task!r}")
    cfg = cfg or InferenceConfig()
    if cfg.half_storage:
        raise ValueError("evaluate_video: the evaluation protocol keeps fp32 clip storage (half_storage is not supported)")
    dev = pipe.device
    ori = torch.as_tensor(frames_u8).to(dev).contiguous()
    T, H, W, _ = ori.shape
    mk = torch.as_tensor(masks).to(dev).float().reshape(1, T, 1, H, W).contiguous()
    cfg = replace(cfg, raft_iter=raft_iter, neighbor_length=neighbor_length, ref_stride=ref_stride,
                  subvideo_length=max(T, 1), raft_clip_frames=PROTOCOL_RAFT_CLIP)
    frames = ops.u8_to_frames(ori).unsqueeze(0)                  # the dataset's frame_tensors
    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    if flows is not None:
        gt = tuple(torch.as_tensor(f).to(dev).float().reshape(1, T - 1, 2, H, W) for f in flows)
    else:
        gt = pipe.compute_flows(frames, cfg)
    pred = pipe.complete_flows(gt, mk, cfg)                       # subvideo_length >= T: one pass over the clip
    gt = (gt[0][0], gt[1][0]) if warp_error else None
    prop, upd_m = pipe.model.img_propagation(frames * (1 - mk), pred, mk, "nearest")
    upd_f = frames * (1 - mk) + prop * mk
    del prop, frames
    comp = torch.zeros(T, H, W, 3, device=dev, dtype=torch.float32)
    pipe.generate(upd_f, mk, upd_m, pred, ori, cfg, comp=comp, composite=ops.composite_blend_f32)
    torch.cuda.synchronize(dev)
    dt = time.perf_counter() - t0
    out = {"frames": T, "seconds": dt, "seconds_per_frame": dt / T, "comp": comp}
    if task == "video_completion":
        ps, ss = psnr_frames(ori, comp).tolist(), ssim_frames(ori, comp).tolist()
        out.update(psnr_per_frame=ps, ssim_per_frame=ss, psnr=sum(ps) / len(ps), ssim=sum(ss) / len(ss))
        if i3d is not None:
            out["i3d"] = (i3d_activations(i3d, ori), i3d_activations(i3d, comp.to(torch.uint8)))
    if warp_error:
        out.update(_warp_error(comp.to(torch.uint8), gt))
    return out


def protocol_video_line(index, count, name, rec, avg_psnr, avg_ssim, avg_time):
    """the per-video line evaluate_propainter.py:219-226 prints and writes (its backslash continuation keeps the next
    source line's indentation inside the string)"""
    if "psnr" not in rec:
        return f'[{index + 1:3}/{count}] Name: {str(name):25} | Time: {avg_time:.4f}'
    return (f'[{index + 1:3}/{count}] Name: {str(name):25} | PSNR/SSIM: {rec["psnr"]:.4f}/{rec["ssim"]:.4f} '
            f'                    | Avg PSNR/SSIM: {avg_psnr:.4f}/{avg_ssim:.4f} | Time: {avg_time:.4f}')


def evaluate_propainter(pipe, videos, size=(432, 240), task="video_completion", neighbor_length=20, ref_stride=10,
                        raft_iter=20, i3d=None, cfg=None, log=None, warp_error=False):
    """scripts/evaluate_propainter.py::main_worker's dataset loop over `videos`, an iterable of (name, frames_u8,
    masks_u8, flows) the caller has read (frames uint8 [T,H0,W0,3] RGB, masks uint8 [T,H0,W0], flows None or the
    (forward, backward) pair of float32 [T-1,2,Hf,Wf] .flo contents), each prepared by prepare_test_video at
    size = (w, h) (the script's --width / --height defaults) and scored by evaluate_video.

    Returns {"videos": per-video records (name, psnr / ssim of the video, the running frame averages avg_psnr /
    avg_ssim, the running mean time per frame avg_time, per-frame metrics, seconds, line = the script's text),
    "summary": video_completion_summary of the records (PSNR / SSIM over all frames, VFID with `i3d`, mean time per
    frame), "line": the script's final line}.  `log(text)` receives each line as it is produced.  The composited
    videos are not kept.  `warp_error`: each record also holds evaluate_video's warping-error keys, summary["ewarp"] is
    their mean over videos (not frame-weighted), and out["ewarp_line"] = "Average Warping Error = ..." follows the final
    line; the script's lines are unchanged."""
    recs = []
    videos = list(videos)
    frame_psnr, frame_ssim, times = [], [], []
    for index, (name, frames_u8, masks_u8, flows) in enumerate(videos):
        torch.cuda.empty_cache()
        fr, mk, fl = prepare_test_video(frames_u8, masks_u8, size, flows, pipe.device)
        r = evaluate_video(pipe, fr, mk, fl, task, neighbor_length, ref_stride, raft_iter, i3d, cfg, warp_error)
        r.pop("comp")
        times.append(r["seconds_per_frame"])
        avg_time = sum(times) / len(times)
        r.update(name=name, avg_time=avg_time)
        if task == "video_completion":
            frame_psnr += r["psnr_per_frame"]
            frame_ssim += r["ssim_per_frame"]
            r.update(avg_psnr=sum(frame_psnr) / len(frame_psnr), avg_ssim=sum(frame_ssim) / len(frame_ssim))
        r["line"] = protocol_video_line(index, len(videos), name, r, r.get("avg_psnr"), r.get("avg_ssim"), avg_time)
        if log:
            log(r["line"])
        recs.append(r)
    out = {"videos": recs}
    if task == "video_completion":
        s = video_completion_summary(recs)
        vfid = f'{s["vfid"]:.3f}' if "vfid" in s else "n/a"
        line = (f'Finish evaluation... Average Frame PSNR/SSIM/VFID: {s["psnr"]:.2f}/{s["ssim"]:.4f}/{vfid} '
                f'| Time: {s["seconds_per_frame"]:.4f}')
    else:
        s = {"seconds_per_frame": sum(times) / len(times), "videos": len(recs)}
        line = f'Finish evaluation... Time: {s["seconds_per_frame"]:.4f}'
    out.update(summary=s, line=line)
    if log:
        log(line)
    if warp_error:
        s["ewarp"] = sum(r["ewarp"] for r in recs) / len(recs)
        out["ewarp_line"] = f'Average Warping Error = {s["ewarp"]:.6f}'
        if log:
            log(out["ewarp_line"])
    return out


# ---------------------------------------------------------------- scripts/compute_flow.py and the flow-completion protocol
@torch.no_grad()
def compute_flow_video(pipe, frames_u8, size=(432, 240), iters=20):
    """scripts/compute_flow.py:62-108 for one video after file I/O: the flow ground truth both evaluation scripts load
    with --load_flow.  frames_u8 uint8 RGB [T,H0,W0,3] (numpy or tensor, T >= 2), size = (w, h), the script's
    --width / --height (default 432 x 240).  Each frame is resized as the script does (ToTensor, torch bilinear
    F.interpolate with align_corners=False, *2 - 1: ops.u8_to_frames_resized), then RAFT with `iters` iterations gives
    the forward flow of every pair (i, i+1) and the backward flow of (i+1, i).

    Returns (forward, backward), each fp16 [T-1,2,h,w] on the pipeline's device: what flowwrite stores, in planar layout
    (`.float()` of it is flowread's array, transposed to [2,h,w] per pair).  The script runs RAFT once per pair and
    direction at batch 1; this runs pipe.compute_flows over the whole clip (RAFT's batched chunks and correlation plan),
    which differs from it only by floating-point summation order.  The result plugs into prepare_test_video(flows=...),
    evaluate_propainter's and evaluate_flow_completion's videos and evaluate_flow_clip(reference_flows=...)."""
    from . import ops
    from .inference_propainter import InferenceConfig
    w, h = (int(s) for s in size)
    if w % 8 or h % 8 or w < 128 or h < 128:
        raise ValueError(f"compute_flow_video: size must be multiples of 8 and at least 128 on both sides (RAFT), got {size}")
    fr = torch.as_tensor(frames_u8)
    if fr.dtype != torch.uint8 or fr.dim() != 4 or fr.shape[-1] != 3 or fr.shape[0] < 2:
        raise ValueError(f"compute_flow_video: expected uint8 frames [T>=2,H,W,3], got {fr.dtype} {tuple(fr.shape)}")
    frames = ops.u8_to_frames_resized(fr.to(pipe.device).contiguous(), (w, h)).unsqueeze(0)
    fwd, bwd = pipe.compute_flows(frames, InferenceConfig(raft_iter=iters))
    return fwd[0].half(), bwd[0].half()


def flow_completion_video_line(index, count, name, epe, avg_time):
    """the per-video line evaluate_flow_completion.py:150-155 prints and writes.  The script prints the name its
    DataLoader collated (batch_size=1): default_collate transposes the batch with zip, so the name is a one-element
    tuple and video 'bear' appears as ('bear',).  This prints the same."""
    return f'[{index + 1:3}/{count}] Name: {str((name,)):25} | EPE: {epe:.4f} | Time: {avg_time:.4f}'


def evaluate_flow_completion(pipe, videos, size=(432, 240), log=None):
    """scripts/evaluate_flow_completion.py::main_worker with --load_flow (:55-179) over `videos`, an iterable of
    (name, masks_u8, flows) the caller has read: masks uint8 [T,H0,W0], flows the (forward, backward) pair of float32
    [T-1,2,Hf,Wf] .flo contents (compute_flow_video's output, or flowread's arrays transposed).  Frames are not an input:
    the script computes nothing from them.  Masks and flows are prepared by prepare_test_video at size = (w, h) and each
    video is scored by evaluate_flow_video.  flows = None raises ValueError: the script cannot run without --load_flow.

    Returns {"videos": per-video records (name, EPE per direction and their mean `epe`, seconds, the running mean time
    per frame avg_time, line = the script's text), "summary": flow_epe_summary of the records, "line": the script's
    final line}.  `log(text)` receives each line as it is produced.  The completed flows are not kept."""
    recs = []
    videos = list(videos)
    for name, _, flows in videos:
        if flows is None:
            raise ValueError(f"evaluate_flow_completion: video {name!r} has no flows (the protocol runs on loaded flows)")
    frames = seconds = 0
    for index, (name, masks_u8, flows) in enumerate(videos):
        torch.cuda.empty_cache()
        _, mk, fl = prepare_test_video(None, masks_u8, size, flows, pipe.device)
        r = evaluate_flow_video(pipe, mk, fl)
        r.pop("pred_flows")
        frames += r["frames"]
        seconds += r["seconds"]
        r.update(name=name, avg_time=seconds / frames)
        r["line"] = flow_completion_video_line(index, len(videos), name, r["epe"], r["avg_time"])
        if log:
            log(r["line"])
        recs.append(r)
    s = flow_epe_summary(recs)
    line = f'Finish evaluation... Average Frame EPE: {s["epe"]:.4f} | | Time: {s["seconds_per_frame"]:.4f}'
    if log:
        log(line)
    return {"videos": recs, "summary": s, "line": line}
