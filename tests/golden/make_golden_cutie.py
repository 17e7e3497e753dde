"""Generates tests/golden/cutie_track.npz and tests/golden/state_dict_manifest_cutie.json by running the UNMODIFIED
reference tracker (web-demos/hugging_face/tracker, imported read-only from /root/reference) on the CPU in the authoring
container.  Not runnable on the GPU box (no /root/reference there); the committed fixture is what travels.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_cutie.py

No download, ever: the reference builds its ResNets with pretrained=True, which calls torch.utils.model_zoo.load_url
(tracker/model/utils/resnet.py:168-178).  Before anything of the tracker is constructed, load_url / hub downloads and
load_weights_add_extra_dim are replaced by stand-ins that raise, and resnet18 / resnet50 by wrappers that build the
networks with pretrained=False; the seeded state_dict then overwrites every parameter with strict=True.  omegaconf is not
installed: a sys.modules stub provides DictConfig, and the config is an attribute dict with the ${...} interpolations of
tracker/config CONFIG resolved.

Weights: the seeded synthetic state_dict of the product's ParamNet(cutie_schema(), seed=SEED).  Stored:
  * pair_*: one frame pair (tests/cutie_inputs.PAIR) through InferenceCore.step: encode_image / transform_key /
    encode_mask on frame 0, pixel_fusion / readout_query / segment on frame 1.  The memory readouts and the sensory memory
    enter their modules rounded to fp16 (stored exactly as *16); outputs are subsampled by OUT_STEPS
  * track_*: a whole tracking run (tests/cutie_inputs.CLIP, 32 frames at 250x430, ids {1, 2}, object 2 leaves the frame):
    the probabilities of every frame at spatial step TRACK_STEP (fp16), the labels there, and the schedule -- per frame
    whether it was a memory frame, whether it was segmented, whether the sensory memory was updated, and the frame
    indices held in working memory afterwards
"""
import copy
import json
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(1, os.path.join(ROOT, "tests"))
sys.path.insert(2, "/root/reference/web-demos/hugging_face")


def _no_download(*a, **k):
    raise RuntimeError("make_golden_cutie: a weight download was attempted")


import torch.hub  # noqa: E402
import torch.utils.model_zoo as _mz  # noqa: E402

_mz.load_url = _no_download
torch.hub.load_state_dict_from_url = _no_download
_om = types.ModuleType("omegaconf")


class DictConfig(dict):
    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k)


_om.DictConfig = DictConfig
sys.modules["omegaconf"] = _om

from tracker.model.utils import resnet  # noqa: E402

_r18, _r50 = resnet.resnet18, resnet.resnet50
resnet.resnet18 = lambda pretrained=True, extra_dim=0: _r18(False, extra_dim)
resnet.resnet50 = lambda pretrained=True, extra_dim=0: _r50(False, extra_dim)
resnet.load_weights_add_extra_dim = _no_download
resnet.model_zoo = types.SimpleNamespace(load_url=_no_download)

from tracker.config import CONFIG  # noqa: E402
from tracker.inference.inference_core import InferenceCore  # noqa: E402
from tracker.model.cutie import CUTIE as RefCUTIE  # noqa: E402
from tracker.utils.mask_mapper import MaskMapper  # noqa: E402
from tracker.utils.tensor_utils import pad_divide_by  # noqa: E402

from cutie_inputs import CLIP, PAIR, make_clip  # noqa: E402
from propainter_b200 import schemas  # noqa: E402
from propainter_b200._params import ParamNet  # noqa: E402

SEED = 13
TRACK_STEP = 10
# (channel step, spatial step) of the stored module outputs; the tests read the same table from the fixture
OUT_STEPS = {"f16": (32, 2), "f8": (16, 2), "f4": (8, 2), "pix_feat": (8, 1), "mask_value": (8, 1), "sensory": (8, 1),
             "readout": (8, 1), "prob": (1, 4)}
GOLD = os.path.dirname(os.path.abspath(__file__))


def config():
    c = copy.deepcopy(CONFIG)
    c["model"]["object_transformer"]["embed_dim"] = c["model"]["embed_dim"]
    c["model"]["object_summarizer"]["embed_dim"] = c["model"]["object_transformer"]["embed_dim"]
    c["model"]["object_summarizer"]["num_summaries"] = c["model"]["object_transformer"]["num_queries"]

    def wrap(d):
        return DictConfig({k: wrap(v) if isinstance(v, dict) else v for k, v in d.items()})
    return wrap(c)


def image_to_torch(frame):
    """BaseTracker.image_to_torch (base_tracker.py:46-51), on the CPU"""
    return torch.from_numpy(frame.transpose(2, 0, 1)).float() / 255


class Recorder:
    """wraps the reference InferenceCore's network / memory calls to record what a step did"""

    def __init__(self, core):
        self.core, self.calls = core, {}
        net = core.network
        for name in ("encode_image", "transform_key", "encode_mask", "segment", "readout_query"):
            self._wrap(net, name)
        self._wrap(core.memory, "_readout")
        self._wrap(core, "_add_memory")

    def _wrap(self, obj, name):
        orig = getattr(obj, name)

        def f(*a, **k):
            out = orig(*a, **k)
            self.calls.setdefault(name, []).append((a, k, out))
            return out
        setattr(obj, name, f)

    def reset(self):
        self.calls = {}


def sub(x, c=1, s=1):
    """[..., C, H, W] subsampled by channel step c and spatial step s"""
    return np.ascontiguousarray(x[..., ::c, ::s, ::s].numpy())


def half(x):
    """x rounded to fp16 and widened back: a module input the fixture can store exactly"""
    return x.half().float()


def store16(x):
    return x.half().numpy()


@torch.no_grad()
def main():
    torch.set_num_threads(8)
    cfg = config()
    sd = ParamNet(schemas.cutie_schema(), seed=SEED).state_dict()
    net = RefCUTIE(cfg).eval()
    net.load_state_dict(sd, strict=True)
    out = {"seed": np.int64(SEED), "track_step": np.int64(TRACK_STEP), "out_steps_keys": np.array(list(OUT_STEPS)),
           "out_steps": np.array(list(OUT_STEPS.values()), np.int64)}

    # ---------------------------------------------------------------- one frame pair, function by function
    # Each module is called on the inputs InferenceCore.step gives it, except that the inputs a test cannot recompute
    # itself (the memory readouts and the sensory memory) are first rounded to fp16 and the reference module is called
    # again on the rounded values: stored as fp16 they are then exact, and the stored outputs are what the reference
    # computes from them.  Outputs are stored in fp32, subsampled by (channel step, spatial step) of OUT_STEPS.
    frames, masks = make_clip(2, PAIR["H"], PAIR["W"], PAIR["seed"])
    core = InferenceCore(net, cfg)
    rec = Recorder(core)
    mapper = MaskMapper()
    m, labels = mapper.convert_mask(masks[0])
    core.step(image_to_torch(frames[0]), torch.Tensor(m), labels)
    (img0,), _, (ms, pix) = rec.calls["encode_image"][0]
    (f16,), _, (key, shrinkage, selection) = rec.calls["transform_key"][0]
    (_, _, sens_in, prob_in), _, (mval, sens_out, summ, _) = rec.calls["encode_mask"][0]
    assert torch.equal(img0[0], pad_divide_by(image_to_torch(frames[0]), 16)[0])     # the tests restate the input
    assert not sens_in.any()
    for name, t in (("f16", ms[0]), ("f8", ms[1]), ("f4", ms[2]), ("pix_feat", pix)):
        out[f"pair_{name}"] = sub(t, *OUT_STEPS[name])
    out["pair_key"], out["pair_shrinkage"], out["pair_selection"] = key.numpy(), shrinkage.numpy(), selection.numpy()
    out["pair_mask_value"] = sub(mval, *OUT_STEPS["mask_value"])
    out["pair_mask_sensory"] = sub(sens_out, *OUT_STEPS["sensory"])
    out["pair_summaries"] = summ.numpy()
    rec.reset()
    core.step(image_to_torch(frames[1]))
    ms1, pix1 = rec.calls["encode_image"][0][2]
    visual = half(rec.calls["_readout"][0][2])
    sens16 = half(sens_out)
    pr = net.pixel_fusion(pix1, visual.view(*visual.shape[:3], *pix1.shape[-2:]), sens16, prob_in)
    out["pair_visual_readout16"], out["pair_sensory16"] = store16(visual), store16(sens16)
    out["pair_pixel_readout"] = sub(pr, *OUT_STEPS["readout"])
    (pr_in, obj_mem), _, _ = rec.calls["readout_query"][0]
    pr16, obj16 = half(pr_in), half(obj_mem)
    mem, _ = net.readout_query(pr16, obj16)
    out["pair_pixel_readout16"], out["pair_obj_mem16"] = store16(pr16), store16(obj16)
    out["pair_mem_readout"] = sub(mem, *OUT_STEPS["readout"])
    mem16 = half(mem)
    (_, _, sens_seg_in), kw, _ = rec.calls["segment"][0]
    assert kw["update_sensory"] and torch.equal(sens_seg_in, sens_out)
    sens_seg, logits, prob = net.segment(ms1, mem16, sens16, update_sensory=True)
    out["pair_mem_readout16"] = store16(mem16)
    out["pair_seg_sensory"] = sub(sens_seg, *OUT_STEPS["sensory"])
    out["pair_seg_logits"], out["pair_seg_prob"] = sub(logits, *OUT_STEPS["prob"]), sub(prob, *OUT_STEPS["prob"])

    # ---------------------------------------------------------------- a whole tracking run
    T, H, W = CLIP["T"], CLIP["H"], CLIP["W"]
    frames, masks = make_clip(T, H, W, CLIP["seed"])
    core = InferenceCore(net, cfg)
    rec = Recorder(core)
    mapper = MaskMapper()
    probs, lbls, sched, mem_frames, adds = [], [], [], [], []
    for t in range(T):
        rec.reset()
        if t == 0:
            m, labels = mapper.convert_mask(masks[0])
            p = core.step(image_to_torch(frames[t]), torch.Tensor(m), labels)
        else:
            p = core.step(image_to_torch(frames[t]))
        is_mem = "_add_memory" in rec.calls
        seg = "segment" in rec.calls
        upd = bool(seg and rec.calls["segment"][0][1]["update_sensory"])
        if is_mem:
            adds.append(t)
        HW = core.memory.HW
        n = core.memory.work_mem.size(0) // HW
        assert core.memory.work_mem.perm_size(0) == HW
        mem_frames.append(([adds[0]] + adds[len(adds) - (n - 1):]) if n > 1 else adds[:1])
        sched.append((is_mem, seg, upd, n))
        lbl = torch.argmax(p, dim=0).numpy().astype(np.uint8)
        final = np.zeros_like(lbl)
        for k, v in mapper.remappings.items():
            final[lbl == v] = k
        probs.append(p[:, ::TRACK_STEP, ::TRACK_STEP].numpy().astype(np.float16))
        lbls.append(final[::TRACK_STEP, ::TRACK_STEP])
    out["track_probs"] = np.stack(probs)
    out["track_labels"] = np.stack(lbls)
    out["track_schedule"] = np.array(sched, np.int64)
    out["track_mem_frames"] = np.array([f + [-1] * (8 - len(f)) for f in mem_frames], np.int64)
    print("schedule (mem, seg, upd, n):", [tuple(int(v) for v in s) for s in sched])
    print("memory frames:", mem_frames[-1], "label counts last frame:", np.bincount(lbls[-1].ravel(), minlength=3))
    print("prob range", float(out["track_probs"].min()), float(out["track_probs"].max()))
    np.savez_compressed(os.path.join(GOLD, "cutie_track.npz"), **out)

    man = {"cutie": {k: [list(v.shape), str(v.dtype).replace("torch.", "")] for k, v in net.state_dict().items()}}
    with open(os.path.join(GOLD, "state_dict_manifest_cutie.json"), "w") as f:
        f.write(json.dumps(man, indent=0))


if __name__ == "__main__":
    main()
