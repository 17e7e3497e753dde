"""``ProInpainter``: the reference's high-level wrapper (web-demos/hugging_face/inpainter/base_inpainter.py:163-374) over the
H100 pipeline.  Same constructor arguments and ``inpaint`` signature / result (list of uint8 frames at the output size);
what differs is where the work happens: frame resizing (PIL BICUBIC), mask resizing (PIL NEAREST) + binarise + dilation
(scipy binary_dilation), uint8 -> float conversion, the four inference stages, compositing and the output resize
(cv2 INTER_LINEAR) all run on the device (propainter_b200.ops / ProPainterPipeline), so a call costs one host -> device
copy of the raw frames / masks and one device -> host copy of the result.

``use_half`` is accepted for signature compatibility: the kernels compute in fp32 whatever the storage dtype (INTEGRATION.md).

``track`` is the demo's Cutie stage (web-demos/hugging_face/track_anything.py:21-36, app.py:264-290): label masks for
every frame from the first frame's template, on the device, ready for ``inpaint``.  The tracker is built on first use.
"""
import numpy as np
import torch

from . import ops
from .inference_propainter import InferenceConfig, ProPainterPipeline
from .model.modules.flow_comp_raft import RAFT_bi
from .model.propainter import InpaintGenerator
from .model.recurrent_flow_completion import RecurrentFlowCompleteNet


def process_sizes(size, ratio=1.0):
    """base_inpainter.py:207-213 + resize_frames :20-31: (out_size, process_size) as (w, h) pairs."""
    out = (int(ratio * size[0]) // 2 * 2, int(ratio * size[1]) // 2 * 2)          # even, so that libx264 can encode it
    return out, (out[0] - out[0] % 8, out[1] - out[1] % 8)


class ProInpainter:
    def __init__(self, propainter_checkpoint=None, raft_checkpoint=None, flow_completion_checkpoint=None, device="cuda:0", use_half=True,
                 seeds=(1, 2, 3), cutie_checkpoint=None, cutie_seed=4):
        self.device = torch.device(device)
        self.cutie_checkpoint, self.cutie_seed = cutie_checkpoint, cutie_seed
        self.tracker = None
        self.use_half = bool(use_half) and self.device.type != "cpu"
        self.fix_raft = RAFT_bi(raft_checkpoint, self.device, seed=seeds[0])
        self.fix_flow_complete = RecurrentFlowCompleteNet(flow_completion_checkpoint, seed=seeds[1]).to(self.device)
        self.model = InpaintGenerator(model_path=propainter_checkpoint, seed=seeds[2]).to(self.device)
        self.pipe = ProPainterPipeline(self.fix_raft, self.fix_flow_complete, self.model, device=self.device)

    @torch.no_grad()
    def inpaint(self, npframes, masks, ratio=1.0, dilate_radius=4, raft_iter=20, subvideo_length=80, neighbor_length=10, ref_stride=10,
                half_storage=False):
        """npframes: T x [H,W,3] uint8 (array or list); masks: T (or 1) x [H,W] (non-zero = hole), as arrays or as one
        torch tensor [T,H,W] (on the device: no host round trip).  Returns a list of T uint8
        frames [H_out, W_out, 3] (base_inpainter.py:190-374).  half_storage: keep the clip's stage outputs in fp16
        (InferenceConfig.half_storage)."""
        fr = torch.from_numpy(np.ascontiguousarray(np.stack([np.asarray(f).astype(np.uint8) for f in npframes]))).to(self.device)
        T, H, W, _ = fr.shape
        out_size, size = process_sizes((W, H), ratio)
        if size != (W, H):
            fr = ops.resize_frames_u8(fr, size)                                     # resize_frames: PIL BICUBIC
        if torch.is_tensor(masks):                                                  # e.g. track()'s label masks, on the device
            mk = masks.to(self.device)
        else:
            mk = torch.from_numpy(np.ascontiguousarray(np.stack([np.asarray(m) for m in masks]))).to(self.device)
        mk = (mk != 0).to(torch.uint8) * 255 if mk.dtype != torch.uint8 else mk
        if mk.shape[-2:] != (size[1], size[0]):
            mk = ops.resize_masks_u8(mk.contiguous(), size)                          # read_mask_demo: Image.NEAREST
        dil = ops.mask_dilate(mk.contiguous(), dilate_radius).unsqueeze(0)          # binary_dilation (or binarise if radius 0)
        if dil.shape[1] == 1 and T > 1:
            dil = dil.expand(1, T, 1, size[1], size[0]).contiguous()
        cfg = InferenceConfig(raft_iter=raft_iter, ref_stride=ref_stride, neighbor_length=neighbor_length, subvideo_length=subvideo_length,
                              fp16=self.use_half, half_storage=half_storage)
        comp = self.pipe(fr, dil, dil.clone(), cfg)                                  # both masks use dilate_radius (:214)
        if out_size != size:
            comp = ops.resize_output_u8(comp, out_size)                              # cv2.resize(f, out_size)
        return list(comp.cpu().numpy())

    @torch.no_grad()
    def track(self, npframes, template_mask, return_probs=False):
        """The demo's tracking stage: frames T x [H,W,3] uint8 and the first frame's label mask [H,W] (object ids, 0 =
        background) -> uint8 label masks [T,H,W] on the device (plus probabilities [T,objects+1,H,W] if return_probs).
        Zeroing the objects that should not be removed before ``inpaint`` is the caller's step, as in the demo."""
        if self.tracker is None:
            from .model.cutie import CUTIE
            from .tracker import MaskTracker
            net = CUTIE(seed=self.cutie_seed)
            if self.cutie_checkpoint is not None:
                net.load_weights(torch.load(self.cutie_checkpoint, map_location="cpu"))
            self.tracker = MaskTracker(net, self.device)
        return self.tracker.track(npframes, template_mask, return_probs=return_probs)
