"""One long clip across several GPUs (one process per GPU, torch.distributed; NCCL over NVLink, gloo in the CPU tests).

The reference's inference is single-device (SURVEY.md section 0.3); what it *does* have is a decomposition of every stage
into independent units with recompute halos (inference_propainter.py:302-319, :342-364, :373-398, :417-452).  Those units
are the shard boundary here, so every unit is the same math as in the single-GPU run:

  stage 1  RAFT          unit = frame pair; rank r owns the pairs that start at its frames (+1 halo frame of input)
  stage 2  completion    unit = (sub-video of `subvideo_length` flows + 5-flow input halo, flow direction): the forward- and
                         backward-flow nets are independent, so even a single sub-video gives two ranks work
  stage 3  image prop.   unit = sub-video of min(100, subvideo_length) frames (+10 halo), owned by the rank of its centre frame
  encoder               every rank encodes its own frames once
  stage 4  generator     unit = sliding window, rank r owns the windows centred on its frames
  merge                  the 1/2-1/2 blend (:445-450) is order dependent: compositing runs in ascending window order, a rank
                         first receives the <= 11 uint8 seam frames its first windows share with the previous rank

What crosses ranks -- always point to point, batched per (source, destination) pair, never a collective over the data:
raw flows into the completion units, completed flows into the propagation units and the windows, propagated frames + masks
to the frame owners, encoder features + masks of the neighbour / reference frames a rank's windows use (reference frames are
every `ref_stride`-th frame within +-(ref_num/2)*ref_stride of the window, inference_propainter.py:159-173, so that is a few
frames per neighbour, not the +-40-frame range), and the uint8 seam frames.  `last_bytes` reports the traffic per stage.
Every rank keeps the input clip and masks (they are inputs); the composited video stays sharded: rank r returns the frames
whose final value it holds.
"""
import torch
import torch.distributed as dist

from . import ops
from .inference_propainter import InferenceConfig, halo_chunks, window_plan


def split_range(n, parts):
    """[lo, hi) of `n` items for each of `parts` owners, contiguous and as even as possible."""
    base, rem = divmod(n, parts)
    out, lo = [], 0
    for r in range(parts):
        hi = lo + base + (1 if r < rem else 0)
        out.append((lo, hi))
        lo = hi
    return out


def frame_owner(T, world):
    """owner rank of every frame (contiguous runs, ascending)"""
    own = [0] * T
    for r, (lo, hi) in enumerate(split_range(T, world)):
        for i in range(lo, hi):
            own[i] = r
    return own


def window_owner(n_windows, world):
    """even split of the sliding windows into contiguous runs (ShardPlan instead assigns a window to the owner of its
    centre frame, so that most of its neighbour frames are local)."""
    owner = [0] * n_windows
    for r, (lo, hi) in enumerate(split_range(n_windows, world)):
        for i in range(lo, hi):
            owner[i] = r
    return owner


def final_frame_owner(plan, owner):
    """rank holding the final value of each frame = owner of the last window that visits it."""
    last = {}
    for wi, (nb, _) in enumerate(plan):
        for f in nb:
            last[f] = owner[wi]
    return last


class ShardPlan:
    """Who computes what and who needs what, derived from (T, world, cfg) alone: identical on every rank, no negotiation."""

    def __init__(self, T, world, cfg):
        self.T, self.world, self.cfg = T, world, cfg
        L = T - 1
        self.fown = frame_owner(T, world)
        self.pair_owner = [self.fown[i] for i in range(L)]                      # pair i = (frame i, frame i+1)
        # ---- stage 2: (sub-video, direction) tasks
        units = halo_chunks(L, cfg.subvideo_length, 5) if L > cfg.subvideo_length else [(0, L, 0, L)]
        self.s2_tasks = [(u, d) for u in units for d in (0, 1)]
        nt = len(self.s2_tasks)
        if nt >= world:
            self.s2_owner = [k * world // nt for k in range(nt)]
        else:                                                                    # fewer tasks than ranks: spread them out
            self.s2_owner = [k * world // nt for k in range(nt)]
        self.pred_owner = [[None] * L, [None] * L]                               # who holds completed flow (d, pair) afterwards
        for (u, d), o in zip(self.s2_tasks, self.s2_owner):
            s, e, lo, hi = u
            for i in range(s + lo, s + hi):
                self.pred_owner[d][i] = o
        # ---- stage 3: image-propagation units
        sub = min(100, cfg.subvideo_length)
        self.s3_units = halo_chunks(T, sub, 10) if T > sub else [(0, T, 0, T)]
        self.s3_owner = [self.fown[(s + lo + s + hi - 1) // 2] for s, e, lo, hi in self.s3_units]
        self.upd_owner = [None] * T
        for (s, e, lo, hi), o in zip(self.s3_units, self.s3_owner):
            for i in range(s + lo, s + hi):
                self.upd_owner[i] = o
        # ---- stage 4: windows
        self.plan = window_plan(T, cfg)
        stride = max(1, cfg.neighbor_length // 2)
        self.win_owner = [self.fown[min(T - 1, wi * stride)] for wi in range(len(self.plan))]
        self.final_owner = final_frame_owner(self.plan, self.win_owner)

    # needs[r] = sorted list of item indices rank r must hold for the stage
    def needs_gt(self, d):
        out = [set() for _ in range(self.world)]
        for (u, dd), o in zip(self.s2_tasks, self.s2_owner):
            if dd == d:
                out[o].update(range(u[0], u[1]))
        return [sorted(x) for x in out]

    def needs_pred(self):
        out = [set() for _ in range(self.world)]
        for (s, e, lo, hi), o in zip(self.s3_units, self.s3_owner):
            out[o].update(range(s, e - 1))
        for (nb, _), o in zip(self.plan, self.win_owner):
            out[o].update(nb[:-1])
        return [sorted(x) for x in out]

    def needs_upd(self):
        """propagated frame + updated mask of frame i go to the rank that encodes it (= its owner)"""
        out = [set() for _ in range(self.world)]
        for i in range(self.T):
            out[self.fown[i]].add(i)
        return [sorted(x) for x in out]

    def needs_enc(self):
        out = [set() for _ in range(self.world)]
        for (nb, refs), o in zip(self.plan, self.win_owner):
            out[o].update(nb + refs)
        return [sorted(x) for x in out]


class ShardedProPainter:
    def __init__(self, pipe, group=None):
        self.pipe, self.group = pipe, group
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        self.last_bytes = {}

    # ------------------------------------------------------------------ point-to-point exchange of per-item tensors
    def _exchange(self, stage, have, producer, needs, like, shape):
        """have {item: tensor} on this rank; producer[item] = rank that holds it; needs[r] = items rank r must end up with.
        One message per (source, destination) pair (items stacked), all posted as one batch.  Returns {item: tensor}."""
        rank, world = self.rank, self.world
        p2p, recv, sent = [], [], 0
        for dst in range(world):
            if dst == rank:
                continue
            idx = [i for i in needs[dst] if producer[i] == rank]
            if idx:
                buf = torch.stack([have[i] for i in idx]).contiguous()
                sent += buf.numel() * buf.element_size()
                p2p.append(dist.P2POp(dist.isend, buf, dst, self.group))
        for src in range(world):
            if src == rank:
                continue
            idx = [i for i in needs[rank] if producer[i] == src]
            if idx:
                buf = like.new_empty((len(idx),) + tuple(shape))
                recv.append((idx, buf))
                p2p.append(dist.P2POp(dist.irecv, buf, src, self.group))
        if p2p:
            for req in dist.batch_isend_irecv(p2p):
                req.wait()
        out = {i: have[i] for i in needs[rank] if producer[i] == rank}
        for idx, buf in recv:
            for j, i in enumerate(idx):
                out[i] = buf[j]
        self.last_bytes[stage] = self.last_bytes.get(stage, 0) + sent
        return out

    @staticmethod
    def _stack(d, idx):
        return torch.stack([d[i] for i in idx], 0)

    @torch.no_grad()
    def __call__(self, frames_u8, flow_masks, masks_dilated, cfg=None, gather=False):
        """Returns (comp_u8 [n,H,W,3], frame_ids): the composited frames whose final value this rank holds (ascending).
        gather=True additionally assembles the whole video on every rank (tests; costs a collective over the output)."""
        cfg = cfg or InferenceConfig()
        if getattr(cfg, "half_storage", False):
            raise ValueError("the sharded runner keeps fp32 clip storage: InferenceConfig.half_storage is not supported here")
        pipe, dev, rank = self.pipe, self.pipe.device, self.rank
        self.last_bytes = {}
        ori = frames_u8.to(dev, non_blocking=True)
        flow_masks, masks_dilated = flow_masks.to(dev, non_blocking=True).float(), masks_dilated.to(dev, non_blocking=True).float()
        T, H, W = ori.shape[0], ori.shape[1], ori.shape[2]
        sp = ShardPlan(T, self.world, cfg)
        L = T - 1
        net = pipe.fix_flow_complete

        # ---- stage 1: RAFT on the pairs that start at this rank's frames (clip-length logic of compute_flows applies)
        mine = [i for i in range(L) if sp.pair_owner[i] == rank]
        gt = [{}, {}]
        if mine:
            a, b = mine[0], mine[-1] + 1                                         # frames a .. b (b = halo)
            fr = ops.u8_to_frames(ori[a:b + 1]).unsqueeze(0)
            ff, fb = pipe.compute_flows(fr, cfg)
            for j, i in enumerate(mine):
                gt[0][i], gt[1][i] = ff[0, j], fb[0, j]
            del fr, ff, fb
        like = masks_dilated
        for d in (0, 1):
            gt[d] = self._exchange("raw_flows", gt[d], sp.pair_owner, sp.needs_gt(d), like, (2, H, W))

        # ---- stage 2: (sub-video, direction) completion tasks (recurrent_flow_completion.py:312-347, one direction each)
        pred = [{}, {}]
        for (u, d), o in zip(sp.s2_tasks, sp.s2_owner):
            if o != rank:
                continue
            s, e, lo, hi = u
            g = self._stack(gt[d], range(s, e)).unsqueeze(0)                     # [1, e-s, 2, H, W]
            m = flow_masks[:, s:e] if d == 0 else flow_masks[:, s + 1:e + 1]
            if d == 0:
                p, _ = net(g * (1 - m), m)
            else:
                p, _ = net(torch.flip(g * (1 - m), dims=[1]), torch.flip(m, dims=[1]))
                p = torch.flip(p, dims=[1])
            p = p * m + g * (1 - m)                                              # combine_flow :340-347
            for j in range(lo, hi):
                pred[d][s + j] = p[0, j]
        del gt
        need_pred = sp.needs_pred()
        for d in (0, 1):
            pred[d] = self._exchange("completed_flows", pred[d], sp.pred_owner[d], need_pred, like, (2, H, W))

        # ---- stage 3: image propagation units (:373-398) -> propagated frames + updated masks, sent to the frame owners
        upd = {}
        for (s, e, lo, hi), o in zip(sp.s3_units, sp.s3_owner):
            if o != rank:
                continue
            fr = ops.u8_to_frames(ori[s:e]).unsqueeze(0)
            md = masks_dilated[:, s:e]
            pf = (self._stack(pred[0], range(s, e - 1)).unsqueeze(0), self._stack(pred[1], range(s, e - 1)).unsqueeze(0))
            prop, um = pipe.model.img_propagation(fr * (1 - md), pf, md, "nearest")
            u_f = fr * (1 - md) + prop * md
            for j in range(lo, hi):
                upd[s + j] = torch.cat([u_f[0, j], um[0, j]], 0)                # [3+1, H, W]
            del fr, prop, u_f
        upd = self._exchange("propagated_frames", upd, sp.upd_owner, sp.needs_upd(), like, (4, H, W))

        # ---- encoder: every rank encodes its own frames once; windows fetch the neighbour / reference frames they use
        own = sorted(upd)
        md_all = masks_dilated[0]
        enc = {}
        if own:
            u = self._stack(upd, own)
            e_own = pipe.model.encode(u[:, :3], md_all[own[0]:own[-1] + 1], u[:, 3:4]).permute(0, 2, 3, 1)   # pixel-major [n,h,w,128]; own is a contiguous range
            for j, i in enumerate(own):
                enc[i] = e_own[j]
            eshape = tuple(e_own.shape[1:])
        else:
            eshape = (H // 4, W // 4, 128)
        need_enc = sp.needs_enc()
        enc = self._exchange("encoder_features", enc, sp.fown, need_enc, like, eshape)
        um1 = self._exchange("updated_masks", {i: upd[i][3:4] for i in own}, sp.fown, need_enc, like, (1, H, W))
        del upd

        # ---- stage 4: this rank's windows, then ordered compositing across the seams
        plan, owner = sp.plan, sp.win_owner
        mine_w = [wi for wi in range(len(plan)) if owner[wi] == rank]
        touched = sorted({f for wi in mine_w for f in plan[wi][0]})
        pos = {f: j for j, f in enumerate(touched)}
        comp = ori.new_zeros((len(touched), H, W, 3))
        visited = {f: False for f in touched}
        preds = {}

        def job(wi):
            nb, refs = plan[wi]
            ids = nb + refs
            empty = like.new_empty(0, 2, H, W)
            return lambda slot: pipe.model.forward_features(
                self._stack(enc, ids).permute(0, 3, 1, 2),
                (self._stack(pred[0], nb[:-1]) if len(nb) > 1 else empty, self._stack(pred[1], nb[:-1]) if len(nb) > 1 else empty),
                md_all.index_select(0, pipe.index(ids)), self._stack(um1, ids), len(nb), slot=slot)
        # the window predictions do not depend on the seam: compute them all (several in flight), composite afterwards in order
        pipe.run_windows([job(wi) for wi in mine_w], lambda k, p: preds.__setitem__(mine_w[k], p), cfg, ori.is_cuda)
        earlier = {f for wi in range(len(plan)) if owner[wi] < rank for f in plan[wi][0]}
        need = sorted(set(touched) & earlier)
        prev = max([owner[wi] for wi in range(len(plan)) if owner[wi] < rank], default=None)
        if need and prev is not None:
            buf = comp.new_empty(len(need), H, W, 3)
            dist.recv(buf, src=prev, group=self.group)
            comp.index_copy_(0, pipe.index([pos[f] for f in need]), buf)
            for f in need:
                visited[f] = True
            self.last_bytes["seam_frames"] = self.last_bytes.get("seam_frames", 0)
        ori_t = ori[touched[0]:touched[-1] + 1] if touched else ori[:0]          # a rank's windows touch a contiguous frame range
        md_t = md_all[touched[0]:touched[-1] + 1] if touched else md_all[:0]
        for wi in mine_w:
            nb = plan[wi][0]
            ops.composite_blend(preds[wi], md_t, ori_t, comp, [pos[i] for i in nb], [not visited[i] for i in nb])
            for i in nb:
                visited[i] = True
        nxt = min([owner[wi] for wi in range(len(plan)) if owner[wi] > rank], default=None)
        if nxt is not None and mine_w:
            later = {f for wi in range(len(plan)) if owner[wi] == nxt for f in plan[wi][0]}
            send = sorted(later & set(touched))
            if send:
                sb = comp.index_select(0, pipe.index([pos[f] for f in send]))
                dist.send(sb, dst=nxt, group=self.group)
                self.last_bytes["seam_frames"] = self.last_bytes.get("seam_frames", 0) + sb.numel()
        final = [f for f in touched if sp.final_owner[f] == rank]
        out = comp.index_select(0, pipe.index([pos[f] for f in final])) if final else comp[:0]
        if not gather:
            return out, final
        # tests only: assemble the whole video everywhere (padded to T frames per rank)
        full = ori.new_zeros((T, H, W, 3))
        if final:
            full.index_copy_(0, pipe.index(final), out)
        allc = [torch.empty_like(full) for _ in range(self.world)]
        dist.all_gather(allc, full, group=self.group)
        res = torch.empty_like(full)
        for f in range(T):
            res[f] = allc[sp.final_owner[f]][f]
        return res
