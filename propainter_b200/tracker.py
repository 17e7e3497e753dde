"""The web demo's mask tracker on the device: per-frame object masks from one annotated frame.

``MaskTracker`` follows ``BaseTracker`` + ``InferenceCore.step`` (web-demos/hugging_face/tracker/base_tracker.py:20-93,
tracker/inference/inference_core.py:18-328) at the demo's configuration (tracker/config CONFIG): working memory only, a
permanent first frame plus a FIFO of ``max_mem_frames - 1`` memory frames (MemoryManager subtracts the permanent frame,
memory_manager.py:27-34), a new memory frame every ``mem_every`` frames, sensory updates on the ``stagger_ti`` offsets and
a top-k (30) readout.  What differs is where the work happens:
  * the memory keys, shrinkage and values live in preallocated ring buffers on the device; eviction moves a ring index
    instead of the reference's torch.cat and slicing (kv_memory_store.py)
  * the memory read is one kernel (``ops.cutie_topk_readout``): no N x HW similarity, no dense affinity
  * frame conversion + padding + normalisation and argmax + unpad + id remapping are single kernels
    (``ops.cutie_frame_in`` / ``ops.cutie_labels``), so ``track`` returns the label masks on the device
Long-term memory, flip augmentation, internal resizing and object chunking are not supported (ValueError).
"""
import logging

import numpy as np
import torch
import torch.nn.functional as F

from . import ops
from .model.cutie import aggregate

log = logging.getLogger(__name__)

# tracker/config CONFIG, as BaseTracker uses it
DEMO_CONFIG = dict(mem_every=5, max_mem_frames=5, top_k=30, stagger_updates=5, chunk_size=-1, use_long_term=None,
                   flip_aug=False, max_internal_size=-1)


class MaskMapper:
    """tracker/utils/mask_mapper.py:15-67 (default, non-exhaustive mode): the user's label ids -> consecutive object ids"""

    def __init__(self):
        self.clear_labels()

    def clear_labels(self):
        self.labels = []
        self.remappings = {}
        self.coherent = True

    def convert_mask(self, mask, exhaustive=False):
        """returns (mask, new_mapped_labels) as the reference does: the mask itself is not remapped"""
        labels = np.unique(mask).astype(np.uint8)
        labels = labels[labels != 0].tolist()
        new_labels = list(set(labels) - set(self.labels))
        if not exhaustive:
            assert len(new_labels) == len(labels), 'Old labels found in non-exhaustive mode'
        for i, l in enumerate(new_labels):
            self.remappings[l] = i + len(self.labels) + 1
            if self.coherent and i + len(self.labels) + 1 != l:
                self.coherent = False
        if exhaustive:
            new_mapped_labels = range(1, len(self.labels) + len(new_labels) + 1)
        elif self.coherent:
            new_mapped_labels = new_labels
        else:
            new_mapped_labels = range(len(self.labels) + 1, len(self.labels) + len(new_labels) + 1)
        self.labels.extend(new_labels)
        return mask, list(new_mapped_labels)

    def input_lut(self):
        """uint8 [256]: user id -> object id (0 elsewhere)"""
        lut = np.zeros(256, np.uint8)
        for k, v in self.remappings.items():
            lut[k] = v
        return lut

    def output_lut(self, num_objects):
        """uint8 [num_objects + 1]: object id (argmax channel) -> user id, background 0 (base_tracker.py:82-87)"""
        lut = np.zeros(num_objects + 1, np.uint8)
        for k, v in self.remappings.items():
            if v <= num_objects:
                lut[v] = k
        return lut


class Schedule:
    """The per-frame decisions of InferenceCore.step (inference_core.py:211-226) and the working memory's FIFO
    (MemoryManager.add_memory + KeyValueMemoryStore.remove_old_memory, memory_manager.py:223-275,
    kv_memory_store.py:153-200) as ring-buffer slots: slot 0 holds the permanent first memory frame, slots 1..fifo_cap
    the FIFO, `head` being the slot (minus one) of the oldest FIFO frame.  Host-side bookkeeping only."""

    def __init__(self, mem_every, stagger_updates, fifo_cap):
        self.mem_every, self.fifo_cap = mem_every, fifo_cap
        if stagger_updates >= mem_every:
            self.stagger_ti = set(range(1, mem_every + 1))
        else:
            self.stagger_ti = set(np.round(np.linspace(1, mem_every, stagger_updates)).astype(int).tolist())
        self.clear()

    def clear(self):
        self.curr_ti, self.last_mem_ti = -1, 0
        self.has_perm, self.head, self.count = False, 0, 0
        self.frames = {}                     # slot -> frame index it holds

    def begin(self, has_mask, need_segment_with_mask=False):
        """advance to the next frame -> (is_mem_frame, need_segment, update_sensory)"""
        self.curr_ti += 1
        d = self.curr_ti - self.last_mem_ti
        is_mem_frame = d >= self.mem_every or has_mask
        need_segment = (not has_mask) or need_segment_with_mask
        return is_mem_frame, need_segment, d in self.stagger_ti

    def add(self):
        """slot for a new memory frame (evicting the oldest FIFO frame when full); records last_mem_ti"""
        if not self.has_perm:
            self.has_perm, slot = True, 0
        elif self.count < self.fifo_cap:
            slot = 1 + (self.head + self.count) % self.fifo_cap
            self.count += 1
        else:
            slot = 1 + self.head
            self.head = (self.head + 1) % self.fifo_cap
        self.frames[slot] = self.curr_ti
        self.last_mem_ti = self.curr_ti
        return slot

    @property
    def n_frames(self):
        return int(self.has_perm) + self.count

    def memory_frames(self):
        """frame indices in memory, in the reference's token order (permanent, then FIFO oldest first)"""
        order = ([0] if self.has_perm else []) + [1 + (self.head + i) % self.fifo_cap for i in range(self.count)]
        return [self.frames[s] for s in order]


class MaskTracker:
    """BaseTracker + InferenceCore on the device.  ``step`` takes one uint8 frame [H,W,3] (and, on the first frame, the
    template label mask [H,W]) and returns the probabilities [objects+1,H,W]; ``track`` runs the demo's generator loop."""

    def __init__(self, cutie, device="cuda:0", **cfg):
        c = dict(DEMO_CONFIG)
        unknown = set(cfg) - set(c)
        if unknown:
            raise ValueError(f"MaskTracker: unknown options {sorted(unknown)}")
        c.update(cfg)
        if c["use_long_term"]:
            raise ValueError("MaskTracker: long-term memory is not supported (working memory only)")
        if c["flip_aug"]:
            raise ValueError("MaskTracker: flip augmentation is not supported")
        if c["max_internal_size"] > 0:
            raise ValueError("MaskTracker: max_internal_size (internal resizing) is not supported")
        if c["chunk_size"] >= 1:
            raise ValueError("MaskTracker: chunk_size is not supported (all objects are processed together)")
        if not 1 <= c["top_k"] <= ops.CUTIE_TOPK_MAX:
            raise ValueError(f"MaskTracker: top_k must be in [1, {ops.CUTIE_TOPK_MAX}]")
        if c["max_mem_frames"] < 2 or c["mem_every"] < 1:
            raise ValueError("MaskTracker: max_mem_frames >= 2 and mem_every >= 1 are required")
        self.cfg = c
        self.device = torch.device(device)
        self.network = cutie.to(self.device).eval()
        self.top_k = c["top_k"]
        self.fifo_cap = c["max_mem_frames"] - 1
        self.schedule = Schedule(c["mem_every"], c["stagger_updates"], self.fifo_cap)
        self.mapper = MaskMapper()
        self.clear_memory()

    def clear_memory(self):
        """BaseTracker.clear_memory: forget every object and memory frame"""
        self.schedule.clear()
        self.mapper.clear_labels()
        self.objects = []
        self.keys = self.shrink = self.values = None
        self.sensory = self.obj_v = self.last_mask = None
        self.out_lut = None
        self.log = []                        # per step: (is_mem_frame, need_segment, update_sensory, memory frame indices)

    # ------------------------------------------------------------------ memory
    def _alloc(self, HW):
        slots = 1 + self.fifo_cap
        self.keys = torch.empty(slots * HW, 64, device=self.device)
        self.shrink = torch.empty(slots * HW, device=self.device)
        self.values = torch.empty(len(self.objects), slots * HW, 256, device=self.device)

    def _add_memory(self, x, pix_feat, prob, key, shrinkage):
        """InferenceCore._add_memory (inference_core.py:53-104) + MemoryManager.add_memory into the ring slots"""
        if prob.shape[1] == 0:
            log.warning('Trying to add an empty object mask to memory!')
            return
        h, w = key.shape[-2:]
        HW = h * w
        if self.sensory is None:
            self.sensory = torch.zeros(1, len(self.objects), 256, h, w, device=self.device)
        msk_value, sensory, obj_value, _ = self.network.encode_mask_normalized(x, pix_feat, self.sensory, prob)
        if self.obj_v is None:
            self.obj_v = obj_value.clone()
        else:                                # streaming sum (memory_manager.py:246-262): sums and areas add
            self.obj_v += obj_value
        if self.keys is None:
            self._alloc(HW)
        slot = self.schedule.add()
        rows = slice(slot * HW, (slot + 1) * HW)
        self.keys[rows] = key.view(64, HW).t()
        self.shrink[rows] = shrinkage.view(HW)
        self.values[:, rows] = msk_value[0].flatten(2).transpose(1, 2)
        self.sensory = sensory

    def _segment(self, key, selection, pix_feat, ms_feat, update_sensory):
        """InferenceCore._segment (inference_core.py:106-153) with MemoryManager.read (one bucket, no chunks)"""
        if self.schedule.n_frames == 0:
            log.warning('Trying to segment without any memory!')
            return torch.zeros((1, key.shape[-2] * 16, key.shape[-1] * 16), device=self.device)
        h, w = key.shape[-2:]
        K = len(self.objects)
        s = self.schedule
        rd = ops.cutie_topk_readout(self.keys, self.shrink, self.values, s.n_frames, s.head, self.fifo_cap,
                                    key.view(64, h * w), selection.view(64, h * w), self.top_k)
        visual = rd.view(K, h, w, 256).permute(0, 3, 1, 2).unsqueeze(0)
        pixel = self.network.pixel_fusion(pix_feat, visual, self.sensory, self.last_mask)
        readout, _ = self.network.readout_query(pixel, self.obj_v.unsqueeze(2))
        sensory, _, prob = self.network.segment(ms_feat, readout, self.sensory, update_sensory=update_sensory)
        if update_sensory:
            self.sensory = sensory
        return prob[0]

    # ------------------------------------------------------------------ steps
    def _pad(self, H, W):
        Hp, Wp = -(-H // 16) * 16, -(-W // 16) * 16
        return (Hp - H) // 2, (Wp - W) // 2, Hp, Wp

    def _mask_objects(self, mask_u8):
        """MaskMapper.convert_mask of the template -> (object-id mask on the device, object ids).  The mask is remapped
        to the consecutive object ids before the one-hot split; the reference splits the unmapped mask by the mapped ids,
        which is the same whenever the ids are already 1..n (the demo's masks) and would lose non-consecutive ones."""
        if self.objects:
            raise ValueError("MaskTracker.step: a mask is accepted on the first frame only (call clear_memory first)")
        m = mask_u8.cpu().numpy() if torch.is_tensor(mask_u8) else np.asarray(mask_u8)
        if m.dtype != np.uint8:
            m = m.astype(np.uint8)
        _, objects = self.mapper.convert_mask(m)
        mapped = torch.from_numpy(self.mapper.input_lut()).to(self.device)[torch.as_tensor(m, device=self.device).long()]
        return mapped, objects

    @torch.no_grad()
    def step_padded(self, frame_u8, mask_u8=None):
        """InferenceCore.step (inference_core.py:155-328, idx_mask=True, end=False) -> probabilities [objects+1,Hp,Wp]
        on the padded frame"""
        frame = torch.as_tensor(frame_u8).to(self.device)
        H, W = frame.shape[:2]
        top, left, Hp, Wp = self._pad(H, W)
        x = ops.cutie_frame_in(frame.contiguous())
        is_mem_frame, need_segment, update_sensory = self.schedule.begin(mask_u8 is not None)
        ms_feat, pix_feat = self.network.encode_normalized(x)
        key, shrinkage, selection = self.network.transform_key(ms_feat[0])
        entry = (is_mem_frame, need_segment, update_sensory and need_segment)
        if need_segment:
            pred = self._segment(key, selection, pix_feat, ms_feat, update_sensory)
        if mask_u8 is not None:
            mapped, objects = self._mask_objects(mask_u8)
            if len(objects) == 0:
                log.warning('Trying to insert an empty mask as memory!')
                self.out_lut = torch.zeros(1, dtype=torch.uint8, device=self.device)
                self.log.append(entry + (self.schedule.memory_frames(),))
                return torch.zeros((1, Hp, Wp), device=self.device)
            self.objects = objects
            self.out_lut = torch.from_numpy(self.mapper.output_lut(len(objects))).to(self.device)
            mp = F.pad(mapped, (left, Wp - W - left, top, Hp - H - top))
            pred = torch.softmax(aggregate(torch.stack([mp == o for o in objects], dim=0), dim=0), dim=0)
        self.last_mask = pred[1:].unsqueeze(0)
        if is_mem_frame:
            self._add_memory(x, pix_feat, self.last_mask, key, shrinkage)
        self.log.append(entry + (self.schedule.memory_frames(),))
        return pred

    def step(self, frame_u8, mask_u8=None):
        """one frame -> probabilities [objects+1,H,W] (background first), as InferenceCore.step returns them"""
        H, W = frame_u8.shape[:2]
        top, left, _, _ = self._pad(H, W)
        return self.step_padded(frame_u8, mask_u8)[:, top:top + H, left:left + W]

    @torch.no_grad()
    def track(self, frames_u8, template_mask_u8, return_probs=False):
        """TrackingAnything.generator (track_anything.py:21-36) from a cleared memory: frames T x [H,W,3] uint8 (array,
        list or device tensor), the first frame's label mask [H,W] -> uint8 label masks [T,H,W] on the device, plus the
        probabilities [T,objects+1,H,W] when return_probs."""
        self.clear_memory()
        if torch.is_tensor(frames_u8):
            frames = frames_u8.to(self.device)
        else:
            frames = torch.from_numpy(np.ascontiguousarray(np.stack([np.asarray(f, dtype=np.uint8) for f in frames_u8])))
            frames = frames.to(self.device)
        if frames.dtype != torch.uint8 or frames.dim() != 4 or frames.shape[-1] != 3:
            raise ValueError(f"track: expected uint8 frames [T,H,W,3], got {frames.dtype} {tuple(frames.shape)}")
        T, H, W, _ = frames.shape
        if tuple(np.shape(template_mask_u8)) != (H, W):
            raise ValueError(f"track: template mask {tuple(np.shape(template_mask_u8))} != frame size {(H, W)}")
        top, left, _, _ = self._pad(H, W)
        out = torch.empty(T, H, W, dtype=torch.uint8, device=self.device)
        probs = []
        for i in range(T):
            pred = self.step_padded(frames[i], template_mask_u8 if i == 0 else None)
            ops.cutie_labels(pred.contiguous(), self.out_lut, H, W, out=out[i])
            if return_probs:
                probs.append(pred[:, top:top + H, left:left + W])
        if return_probs:
            return out, torch.stack(probs)
        return out
