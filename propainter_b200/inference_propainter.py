"""The inference driver: stage scheduling of inference_propainter.py:298-452 as a library call.

The reference keeps this logic under ``__main__`` with file I/O around it; here it is a class that
takes frames / masks as tensors (uint8 frames may come from pinned host memory), keeps everything
on the device, and replaces the per-window ``.cpu()`` + numpy compositing (:437-450) with one kernel,
so a clip needs exactly one host->device and one device->host copy.  Chunk boundaries, halo lengths,
reference-frame selection and the order-dependent blend follow the reference exactly.
"""
import math
from dataclasses import dataclass

import torch

from . import config, ops
from .RAFT.raft import ON_THE_FLY, OTF_BYTES_PER_PAIR_PX
from .model.modules.flow_comp_raft import RAFT_bi
from .model.propainter import InpaintGenerator
from .model.recurrent_flow_completion import RecurrentFlowCompleteNet


@dataclass
class InferenceConfig:
    """argparse flags of inference_propainter.py:181-217 that shape the hot path."""
    raft_iter: int = 20
    ref_stride: int = 10
    neighbor_length: int = 10
    subvideo_length: int = 80
    # frames per RAFT call.  None = as many as an 8 GB correlation pyramid allows (never fewer than the reference's
    # 12/8/4/2, inference_propainter.py:302-309).  Frame pairs are independent, so this only changes batching.
    raft_clip_frames: int = None
    # generator windows computed concurrently on side streams (compositing stays ordered); > 1 needs CUDA_GRAPHS off
    windows_in_flight: int = 1
    # --fp16 (inference_propainter.py:211, :268-270, :323-330) halves the two nets and every tensor after RAFT.  The
    # kernels here compute in fp32 whatever the storage dtype (a `.half()` net is widened once, fp16 inputs are widened at
    # entry and results handed back in the caller's dtype), so the flag is accepted and changes nothing in the pipeline.
    fp16: bool = False
    # Half-precision clip storage: the four clip-resident stage outputs (RAFT flows, completed flows, updated frames and
    # masks, encoder features) are rounded once to fp16 where a stage hands them on, and widened to fp32 on load; all
    # arithmetic stays fp32.  A clip then holds about 35 instead of 95 bytes per pixel and frame (DESIGN.md §7), for a small
    # change of the result, so it is the caller's explicit choice (the reference's --fp16 "to reduce running memory cost").
    half_storage: bool = False


def get_ref_index(mid_neighbor_id, neighbor_ids, length, ref_stride=10, ref_num=-1):
    """inference_propainter.py:159-173 (incl. its `> ref_num` early-exit quirk)."""
    nb = set(neighbor_ids)
    if ref_num == -1:
        return [i for i in range(0, length, ref_stride) if i not in nb]
    half = ref_stride * (ref_num // 2)
    picked = []
    for i in range(max(0, mid_neighbor_id - half), min(length, mid_neighbor_id + half), ref_stride):
        if i in nb:
            continue
        if len(picked) > ref_num:
            break
        picked.append(i)
    return picked


def raft_clip_len(width):
    """:302-309"""
    for limit, n in ((640, 12), (720, 8), (1280, 4)):
        if width <= limit:
            return n
    return 2


def auto_clip_frames(T, H, W, plan):
    """Frames per RAFT call when InferenceConfig.raft_clip_frames is None: as many as fit an 8 GB budget for the
    plan's per-pair memory (all-pairs: the 4-level pyramid, ~1.34 N^2 floats; on-the-fly: the lookup output, GRU
    buffers and encoder activations, RAFT.OTF_BYTES_PER_PAIR_PX per input pixel), never fewer than the reference's."""
    if plan == ON_THE_FLY:
        pairs = int(8e9 // (OTF_BYTES_PER_PAIR_PX * H * W))
    else:
        n = (H // 8) * (W // 8)
        pairs = int(8e9 // (5.4 * n * n))
    return max(raft_clip_len(W), min(T, pairs // 2 + 1))


def flow_chunks(T, clip):
    """Frame ranges [s,e) handed to RAFT_bi, with the 1-frame overlap of :314-319."""
    if T <= clip:
        return [(0, T)]
    return [(max(f - 1, 0), min(T, f + clip)) for f in range(0, T, clip)]


def halo_chunks(L, sub, pad):
    """(s, e, keep_lo, keep_hi) for the recompute-halo chunking of :342-364 / :373-398."""
    out = []
    for f in range(0, L, sub):
        s, e = max(0, f - pad), min(L, f + sub + pad)
        out.append((s, e, f - s, (e - s) - (e - min(L, f + sub))))
    return out


def window_plan(T, cfg):
    """[(neighbor_ids, ref_ids)] of the sliding-window loop :406-421."""
    stride = cfg.neighbor_length // 2
    ref_num = cfg.subvideo_length // cfg.ref_stride if T > cfg.subvideo_length else -1
    plan = []
    for f in range(0, T, stride):
        nb = list(range(max(0, f - stride), min(T, f + stride + 1)))
        plan.append((nb, get_ref_index(f, nb, T, cfg.ref_stride, ref_num)))
    return plan


def prepare_masks(masks_u8, mask_dilation=4, device="cuda"):
    """read_mask (inference_propainter.py:77-114) after file I/O: uint8 masks [T,H,W] (or [1,H,W], repeated by the
    caller) -> (flow_masks, masks_dilated), both float {0,1} [1,T,1,H,W] on the device.  Both use `mask_dilation`
    (the script passes args.mask_dilation for both, :238-240)."""
    m = masks_u8.to(device)
    d = ops.mask_dilate(m, mask_dilation).unsqueeze(0)
    return d, d.clone()


def outpaint_geometry(h, w, scale_h, scale_w):
    """extrapolation's geometry (inference_propainter.py:123-128, :142-143) for an h x w source:
    ((H, W), (top, left), (rim_h, rim_w)) = the canvas, the source's offset in it and the flow-mask rim.

    The reference's expressions in Python doubles: int(scale * size) rounded down to a multiple of 8, offset
    int((H - h) / 2), rim 4 if offset > 10 else 0 (1.4 * 360 = 503.99999999999994 gives 496, not 504).  Deviation: a
    canvas smaller than the source in either dimension, where the reference's negative offset makes the numpy slice
    fail or misplace the frame, and a non-finite scale raise ValueError."""
    sh, sw = float(scale_h), float(scale_w)
    if not (math.isfinite(sh) and math.isfinite(sw)):
        raise ValueError(f"outpainting scale must be finite, got ({scale_h}, {scale_w})")
    H, W = int(sh * h), int(sw * w)
    H, W = H - H % 8, W - W % 8
    if H < h or W < w:
        raise ValueError(f"outpainting canvas {H}x{W} is smaller than the {h}x{w} source (scale ({scale_h}, {scale_w}))")
    top, left = int((H - h) / 2), int((W - w) / 2)
    return (H, W), (top, left), (4 if top > 10 else 0, 4 if left > 10 else 0)


def prepare_outpainting(frames_u8, scale_h=1.0, scale_w=1.2, device="cuda"):
    """extrapolation (inference_propainter.py:117-156) + to_tensors of its masks (:265-266) on the device: uint8 frames
    [T,h,w,3] (host or device) -> (canvas uint8 [T,H,W,3], flow_masks, masks_dilated float {0,1} [1,T,1,H,W], (W, H)),
    the reference's return order and its --scale_h / --scale_w defaults (:206-209).  mask_dilation plays no part."""
    src = torch.as_tensor(frames_u8).to(device).contiguous()
    geo = outpaint_geometry(src.shape[1], src.shape[2], scale_h, scale_w)
    canvas, fm, md = ops.extrapolate_u8(src, geo)
    H, W = geo[0]
    return canvas, fm.unsqueeze(0), md.unsqueeze(0), (W, H)


class ProPainterPipeline:
    """RAFT flow -> flow completion -> image propagation -> sliding-window generator -> compositing."""

    def __init__(self, fix_raft=None, fix_flow_complete=None, model=None, device="cuda", seeds=(1, 2, 3),
                 weights=(None, None, None)):
        self.device = torch.device(device)
        self.fix_raft = fix_raft if fix_raft is not None else RAFT_bi(weights[0], device, seed=seeds[0])
        self.fix_flow_complete = (fix_flow_complete if fix_flow_complete is not None
                                  else RecurrentFlowCompleteNet(weights[1], seed=seeds[1]).to(device))
        self.model = model if model is not None else InpaintGenerator(model_path=weights[2], seed=seeds[2]).to(device)

    def index(self, ids):
        """device int64 index tensor for a frame list, built once per distinct list (the window plan repeats every clip)"""
        cache = self.__dict__.setdefault("_index_cache", {})
        key = tuple(ids)
        if key not in cache:
            cache[key] = torch.tensor(list(ids), dtype=torch.long, device=self.device)
        return cache[key]

    def state_dicts(self):
        return {"raft": self.fix_raft.fix_raft.state_dict(), "rfc": self.fix_flow_complete.state_dict(),
                "gen": self.model.state_dict()}

    # ---- stage 1 (:302-330)
    def compute_flows(self, frames, cfg):
        T, H, W = frames.shape[1], frames.shape[-2], frames.shape[-1]
        clip = cfg.raft_clip_frames
        if clip is None:
            clip = auto_clip_frames(T, H, W, self.fix_raft.fix_raft.corr_plan(H, W, frames.device))
        ff, bb = [], []
        for s, e in flow_chunks(T, clip):
            f, b = self.fix_raft(frames[:, s:e], iters=cfg.raft_iter)
            ff.append(f)
            bb.append(b)
        return torch.cat(ff, 1), torch.cat(bb, 1)

    # ---- stage 2 (:341-368)
    def complete_flows(self, gt_flows, flow_masks, cfg):
        net, L = self.fix_flow_complete, gt_flows[0].shape[1]
        if L <= cfg.subvideo_length:
            pred, _ = net.forward_bidirect_flow(gt_flows, flow_masks)
            return net.combine_flow(gt_flows, pred, flow_masks)
        pf, pb = [], []
        for s, e, lo, hi in halo_chunks(L, cfg.subvideo_length, 5):
            sub = (gt_flows[0][:, s:e], gt_flows[1][:, s:e])
            pred, _ = net.forward_bidirect_flow(sub, flow_masks[:, s:e + 1])
            pred = net.combine_flow(sub, pred, flow_masks[:, s:e + 1])
            pf.append(pred[0][:, lo:hi])
            pb.append(pred[1][:, lo:hi])
        return torch.cat(pf, 1), torch.cat(pb, 1)

    # ---- stage 3 (:371-404)
    def propagate_images(self, frames, masks_dilated, pred_flows, cfg):
        T = frames.shape[1]
        masked = frames * (1 - masks_dilated)
        sub = min(100, cfg.subvideo_length)
        if T <= sub:
            prop, um = self.model.img_propagation(masked, pred_flows, masks_dilated, "nearest")
            return frames * (1 - masks_dilated) + prop * masks_dilated, um
        uf, umk = [], []
        for s, e, lo, hi in halo_chunks(T, sub, 10):
            prop, um = self.model.img_propagation(masked[:, s:e], (pred_flows[0][:, s:e - 1], pred_flows[1][:, s:e - 1]),
                                                  masks_dilated[:, s:e], "nearest")
            upd = frames[:, s:e] * (1 - masks_dilated[:, s:e]) + prop * masks_dilated[:, s:e]
            uf.append(upd[:, lo:hi])
            umk.append(um[:, lo:hi])
        return torch.cat(uf, 1), torch.cat(umk, 1)

    # ---- stages 1-3 on half-precision clip storage (InferenceConfig.half_storage): each stage's clip-sized output is
    # rounded once to fp16 (R1: RAFT flows, R2: completed flows, R3: updated frames / masks) into a preallocated clip
    # buffer, chunk by chunk; every consumer widens it to fp32
    def compute_flows_half(self, ori_u8, cfg):
        """stage 1 on uint8 frames [T,H,W,3]: RAFT on fp32 frames built per chunk -> fp16 (forward, backward) [1,T-1,2,H,W]"""
        T, H, W = ori_u8.shape[0], ori_u8.shape[1], ori_u8.shape[2]
        clip = cfg.raft_clip_frames
        if clip is None:
            clip = auto_clip_frames(T, H, W, self.fix_raft.fix_raft.corr_plan(H, W, ori_u8.device))
        gf = torch.empty(1, max(T - 1, 0), 2, H, W, device=ori_u8.device, dtype=torch.float16)
        gb = torch.empty_like(gf)
        for s, e in flow_chunks(T, clip):
            f, b = self.fix_raft(ops.u8_to_frames(ori_u8[s:e]).unsqueeze(0), iters=cfg.raft_iter)
            gf[:, s:e - 1].copy_(f)
            gb[:, s:e - 1].copy_(b)
        return gf, gb

    def complete_flows_half(self, gt_flows, flow_masks, cfg):
        """stage 2 on fp16 RAFT flows: each sub-video is widened inside the net, and its kept range of the combined flows is
        rounded into fp16 clip buffers"""
        net, L = self.fix_flow_complete, gt_flows[0].shape[1]
        out = (torch.empty_like(gt_flows[0]), torch.empty_like(gt_flows[1]))
        units = [(0, L, 0, L)] if L <= cfg.subvideo_length else halo_chunks(L, cfg.subvideo_length, 5)
        for s, e, lo, hi in units:
            sub = (gt_flows[0][:, s:e], gt_flows[1][:, s:e])
            pred, _ = net.forward_bidirect_flow(sub, flow_masks[:, s:e + 1])
            pred = net.combine_flow(sub, pred, flow_masks[:, s:e + 1])
            out[0][:, s + lo:s + hi].copy_(pred[0][:, lo:hi])
            out[1][:, s + lo:s + hi].copy_(pred[1][:, lo:hi])
        return out

    def propagate_images_half(self, ori_u8, masks_dilated, pred_flows, cfg):
        """stage 3 on the clip's uint8 frames and fp16 completed flows: one pp_img_prop_scan_u8h call per sub-video masks the
        frames, runs the fp32 scan and writes its kept frames, composited, into fp16 clip buffers [1,T,3,H,W] / [1,T,1,H,W]"""
        T, H, W = ori_u8.shape[0], ori_u8.shape[1], ori_u8.shape[2]
        md = masks_dilated[0].contiguous()
        uf = torch.empty(1, T, 3, H, W, device=ori_u8.device, dtype=torch.float16)
        um = torch.empty(1, T, 1, H, W, device=ori_u8.device, dtype=torch.float16)
        sub = min(100, cfg.subvideo_length)
        units = [(0, T, 0, T)] if T <= sub else halo_chunks(T, sub, 10)
        for s, e, lo, hi in units:
            ops.img_prop_scan_u8h(ori_u8[s:e], md[s:e], pred_flows[0][0, s:e - 1], pred_flows[1][0, s:e - 1],
                                  uf[0, s + lo:s + hi], um[0, s + lo:s + hi], lo, hi)
        return uf, um

    # ---- stage 4 (:406-452)
    def generate(self, upd_frames, masks_dilated, upd_masks, pred_flows, ori_u8, cfg, windows=None, comp=None,
                 visited=None, composite=None):
        """`composite(pred, masks, ori_u8, comp, frame_ids, first_flags)` writes a window's prediction into `comp`:
        ops.composite_blend (uint8, the inference script's) unless given; the evaluation protocol passes
        ops.composite_blend_f32 with a float32 `comp`."""
        composite = composite or ops.composite_blend
        T = upd_frames.shape[1]
        plan = window_plan(T, cfg)
        comp = torch.zeros_like(ori_u8) if comp is None else comp
        visited = [False] * T if visited is None else visited
        md = masks_dilated[0].contiguous()
        # encoder features depend only on (frame, mask, updated mask): computed once per clip, not once per window
        if cfg.half_storage:                                       # R4: fp16 pixel-major clip buffer, widened per window
            H, W = upd_frames.shape[-2:]
            enc_all = self.model.encode(upd_frames[0], md, upd_masks[0], out=torch.empty(
                T, H // 4, W // 4, 128, device=upd_frames.device, dtype=torch.float16))
        else:
            enc_all = self.model.encode(upd_frames[0], md, upd_masks[0]).permute(0, 2, 3, 1)  # pixel-major rows: cheap frame gather
        todo = [(wi, nb, refs) for wi, (nb, refs) in enumerate(plan) if windows is None or wi in windows]

        um0 = upd_masks[0]

        def job(nb, refs):
            # frame selections as cached device index tensors / slices: indexing with a Python list builds the index on the
            # host and copies it with a blocking cudaMemcpy, which stalls the issuing thread until the stream has drained
            # (measured: generate() blocked the host for the whole clip, so nothing could be queued behind it)
            idx = self.index(nb + refs)
            a, b = nb[0], nb[-1]                                   # neighbour frames are a contiguous range
            return lambda slot: self.model.forward_features(enc_all.index_select(0, idx).float().permute(0, 3, 1, 2),
                                                            (pred_flows[0][0, a:b], pred_flows[1][0, a:b]),
                                                            md.index_select(0, idx), um0.index_select(0, idx), len(nb), slot=slot)

        def consume(k, pred):
            nb = todo[k][1]
            composite(pred, md, ori_u8, comp, nb, [not visited[i] for i in nb])
            for i in nb:
                visited[i] = True
        self.run_windows([job(nb, refs) for _, nb, refs in todo], consume, cfg, upd_frames.is_cuda)
        return comp

    def run_windows(self, jobs, consume, cfg, cuda=True):
        """Windows are independent given the stage-3 outputs: keep `cfg.windows_in_flight` of them in flight on side streams
        (each slot owns its own captured graph instance); `consume(k, pred)` -- the compositing -- is replayed on the main stream
        in ascending window order because the 1/2-1/2 blend of inference_propainter.py:445-450 is order-dependent.
        jobs[k](slot) launches window k and returns its prediction."""
        nfl = max(1, int(cfg.windows_in_flight)) if cuda else 1
        if nfl > 1 and config.CUDA_GRAPHS:
            # concurrently replayed window graphs give a wrong, run-to-run different video (also with library convs and the
            # mma.sync attention); run eagerly, windows in flight give exactly the one-at-a-time result
            raise ValueError("windows_in_flight > 1 requires config.CUDA_GRAPHS = False")
        if nfl == 1:
            for k, jb in enumerate(jobs):
                consume(k, jb(0))
            return
        main = torch.cuda.current_stream()
        if not hasattr(self, "_side_streams") or len(self._side_streams) < nfl:
            self._side_streams = [torch.cuda.Stream(device=self.device) for _ in range(nfl)]
        pending = []

        def drain(keep):
            while len(pending) > keep:
                slot, k, pred = pending.pop(0)
                main.wait_stream(self._side_streams[slot])
                pred.record_stream(main)
                consume(k, pred)
        for k, jb in enumerate(jobs):
            slot = k % nfl
            drain(nfl - 1)
            st = self._side_streams[slot]
            st.wait_stream(main)
            with torch.cuda.stream(st):
                pred = jb(slot)
            pending.append((slot, k, pred))
        drain(0)

    # ---- whole path
    @torch.no_grad()
    def __call__(self, frames_u8, flow_masks, masks_dilated, cfg=None, return_stages=False):
        """frames_u8 uint8 [T,H,W,3] (host or device); masks float {0,1} [1,T,1,H,W].
        Returns composited uint8 frames [T,H,W,3] on the device."""
        cfg = cfg or InferenceConfig()
        dev = self.device
        ori = frames_u8.to(dev, non_blocking=True)
        flow_masks = flow_masks.to(dev, non_blocking=True).float()
        masks_dilated = masks_dilated.to(dev, non_blocking=True).float()
        if cfg.half_storage:
            # no clip-sized fp32 frames: RAFT builds them per chunk, stage 3 masks the uint8 frames in its kernel
            gt = self.compute_flows_half(ori, cfg)
            pred = self.complete_flows_half(gt, flow_masks, cfg)
            stages = {"gt_flows": gt} if return_stages else {}
            del gt                                                 # released after stage 2 unless it is returned
            upd_f, upd_m = self.propagate_images_half(ori, masks_dilated, pred, cfg)
            comp = self.generate(upd_f, masks_dilated, upd_m, pred, ori, cfg)
            if return_stages:
                return comp, dict(stages, pred_flows=pred, updated_frames=upd_f, updated_masks=upd_m)
            return comp
        frames = ops.u8_to_frames(ori).unsqueeze(0)
        gt = self.compute_flows(frames, cfg)
        pred = self.complete_flows(gt, flow_masks, cfg)
        upd_f, upd_m = self.propagate_images(frames, masks_dilated, pred, cfg)
        comp = self.generate(upd_f, masks_dilated, upd_m, pred, ori, cfg)
        if return_stages:
            return comp, {"gt_flows": gt, "pred_flows": pred, "updated_frames": upd_f, "updated_masks": upd_m}
        return comp

    @torch.no_grad()
    def outpaint(self, frames_u8, scale_h=1.0, scale_w=1.2, cfg=None, return_stages=False):
        """--mode video_outpainting (inference_propainter.py:243-246): prepare_outpainting, then the four stages on the
        widened canvas.  frames_u8 uint8 [T,h,w,3] (host or device).  Returns the composited canvas uint8 [T,H,W,3] on
        the device (the script's final cv2.resize to the source size, :469-470, is ops.resize_output_u8(comp, (w, h)))."""
        canvas, flow_masks, masks_dilated, _ = prepare_outpainting(frames_u8, scale_h, scale_w, self.device)
        return self(canvas, flow_masks, masks_dilated, cfg, return_stages)

    def masked_preview(self, frames_u8, masks_dilated):
        """The script's second video (inference_propainter.py:250-261), in either mode: the holes of `masks_dilated`
        ([1,T,1,H,W] or [T,1,H,W] float) tinted green over uint8 frames [T,H,W,3].  Returns uint8 [T,H,W,3] on the device."""
        dev = self.device
        frames = torch.as_tensor(frames_u8).to(dev, non_blocking=True).contiguous()
        return ops.mask_overlay_u8(frames, masks_dilated.to(dev, non_blocking=True).float().contiguous())

    @torch.no_grad()
    def flows(self, frames_u8, flow_masks, cfg=None):
        """Stages 1-2 only (inference_propainter.py:302-368): RAFT flows and the completed flows, with the chunking of
        __call__ and without image propagation or the generator.  frames_u8 uint8 [T,H,W,3] (host or device), flow_masks
        float {0,1} [1,T,1,H,W].  Returns (gt_flows, pred_flows), each a (forward, backward) pair of [1,T-1,2,H,W],
        bit-identical to the stage outputs of __call__(..., return_stages=True); fp16 with cfg.half_storage."""
        cfg = cfg or InferenceConfig()
        dev = self.device
        ori = torch.as_tensor(frames_u8).to(dev, non_blocking=True)
        flow_masks = flow_masks.to(dev, non_blocking=True).float()
        if cfg.half_storage:
            gt = self.compute_flows_half(ori, cfg)
            return gt, self.complete_flows_half(gt, flow_masks, cfg)
        frames = ops.u8_to_frames(ori).unsqueeze(0)
        gt = self.compute_flows(frames, cfg)
        return gt, self.complete_flows(gt, flow_masks, cfg)

    def flow_preview(self, flows, normalize="frame", clip_flow=None, bgr=False):
        """One direction of a flow pair ([1,T-1,2,H,W] or [T-1,2,H,W] float32) as a colour-coded uint8 video
        [T-1,H,W,3] on the device; see ops.flow_to_image_u8 for `normalize` ("frame": flow_viz.py, "clip":
        flow_viz_pt.py), `clip_flow` and `bgr`."""
        f = flows.to(self.device, non_blocking=True)
        if f.dim() == 5:
            if f.shape[0] != 1:
                raise ValueError(f"flow_preview: expected one clip [1,T-1,2,H,W], got {tuple(flows.shape)}")
            f = f[0]
        return ops.flow_to_image_u8(f, normalize, clip_flow, bgr)
