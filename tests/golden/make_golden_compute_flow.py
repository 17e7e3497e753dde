"""Generates tests/golden/compute_flow_2v_128x160.npz by running the UNMODIFIED scripts/compute_flow.py (its __main__
body) and then scripts/evaluate_flow_completion.py::main_worker with --load_flow on the .flo files that run wrote, read-only
from the reference checkout at REF.  The committed fixture is what the tests read.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_compute_flow.py

A small dataset tree is written to a temporary directory from tests/compute_flow_inputs.py: PNG frames (lossless, BGR as
cv2.imwrite stores them) at each video's native size (200 x 240, down-scaled, and 96 x 120, up-scaled, to the 160 x 128
eval size) and PNG masks (mode L, 0 / 255).  compute_flow.py runs with -i <frames> -o <flows> --height 128 --width 160;
its module-level definitions (initialize_RAFT, imwrite, the imports) are compiled as they stand, and so is its __main__
body except for its first statement.  main_worker is taken from evaluate_flow_completion.py with `ast` and compiled as it
stands, with TestDataset from core/dataset.py and Stack / ToTorchFormatTensor from core/utils.py (core.utils imports
matplotlib at module level, which the fixture's environment need not have), run with --dataset davis --load_flow and
its defaults otherwise.

Substitutions, none of which touches what the scripts compute:
  * compute_flow.py's `device = 'cuda'`: device is bound to 'cpu' instead (the assignment is the one statement of the
    __main__ body not executed; the run is on the CPU);
  * weights/raft-things.pth (loaded by initialize_RAFT from the working directory) and the flow-completion checkpoint:
    make_golden's seeded state_dicts (RAFT seed 1 with DataParallel's `module.` prefix, flow completion seed 2) saved to
    temporary checkpoints;
  * torch.cuda.synchronize: a no-op (main_worker runs on the CPU);
  * main_worker's `time`: a clock that advances by 1/16 s per reading, so the text's times, and the whole fixture,
    are the same on every run;
  * RecurrentFlowCompleteNet: a subclass whose combine_flow records its inputs and output, unchanged.
Stored, to keep the fixture small: every 4th pixel in each direction (`[..., ::4, ::4]`, as the other RAFT fixtures)
of the fp16 flows of every .flo file (flowread's array, planar [T-1,2,h,w]) and of the completed flows (fp16); the
per-video EPE of each direction as main_worker computes it over the full frames (from the recorded tensors, by its own
expression); and the metrics-file text.
"""
import ast
import os
import sys
import tempfile
import types

import cv2
import numpy as np
import torch
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden  # noqa: E402  (puts the repository and the reference on sys.path)
from make_golden_eval_protocol import reference_defs  # noqa: E402

from tests.compute_flow_inputs import GOLD_NAME, SIZE, VIDEOS, video_inputs  # noqa: E402

REF = "/root/reference"


def write_dataset(root):
    for name, T, mask, seed, native in VIDEOS:
        fr, mk = video_inputs(T, mask, seed, native)
        for d in ("JPEGImages", "masks"):
            os.makedirs(os.path.join(root, d, name), exist_ok=True)
        for t in range(T):
            cv2.imwrite(os.path.join(root, "JPEGImages", name, f"{t:05d}.png"), cv2.cvtColor(fr[t], cv2.COLOR_RGB2BGR))
            Image.fromarray(mk[t], mode="L").save(os.path.join(root, "masks", name, f"{t:05d}.png"))


def run_compute_flow(tmp):
    """compute_flow.py's module body, then its __main__ body after `device = 'cuda'` with device = 'cpu'"""
    path = os.path.join(REF, "scripts", "compute_flow.py")
    tree = ast.parse(open(path).read(), path)
    main = [n for n in tree.body if isinstance(n, ast.If)]
    assert len(main) == 1 and ast.unparse(main[0].test) == "__name__ == '__main__'"
    first = main[0].body[0]
    assert ast.unparse(first) == "device = 'cuda'", ast.unparse(first)
    defs = [n for n in tree.body if not isinstance(n, ast.If)]
    ns = {"__name__": "compute_flow"}
    exec(compile(ast.Module(body=defs, type_ignores=[]), path, "exec"), ns)
    ns["device"] = "cpu"
    argv = sys.argv
    sys.argv = ["compute_flow.py", "-i", os.path.join(tmp, "JPEGImages"), "-o", os.path.join(tmp, "flows"),
                "--height", str(SIZE[1]), "--width", str(SIZE[0])]
    try:
        exec(compile(ast.Module(body=main[0].body[1:], type_ignores=[]), path, "exec"), ns)
    finally:
        sys.argv = argv


def main():
    import argparse
    torch.set_num_threads(8)
    tmp = tempfile.mkdtemp(prefix="compute_flow_")
    write_dataset(tmp)
    raft, rfc, _ = make_golden.build_reference()
    os.makedirs(os.path.join(tmp, "weights"))
    ck_raft = os.path.join(tmp, "weights", "raft-things.pth")
    ck_rfc = os.path.join(tmp, "weights", "recurrent_flow_completion.pth")
    torch.save({"module." + k: v for k, v in raft.state_dict().items()}, ck_raft)
    torch.save(rfc.state_dict(), ck_rfc)

    cwd = os.getcwd()
    os.chdir(tmp)
    try:
        run_compute_flow(tmp)
    finally:
        os.chdir(cwd)

    cu = types.ModuleType("core.utils")
    import torchvision.transforms as transforms
    ns_u = {"np": np, "torch": torch, "Image": Image, "transforms": transforms}
    reference_defs(os.path.join(REF, "core", "utils.py"), ["Stack", "ToTorchFormatTensor", "to_tensors"], ns_u)
    for k in ("Stack", "ToTorchFormatTensor", "to_tensors"):
        setattr(cu, k, ns_u[k])
    sys.modules["core.utils"] = cu
    from utils.file_client import FileClient
    from utils.flow_util import flowread, resize_flow
    from utils.img_util import imfrombytes
    from model.modules.flow_comp_raft import RAFT_bi
    from model.recurrent_flow_completion import RecurrentFlowCompleteNet
    ns_d = {"os": os, "cv2": cv2, "np": np, "torch": torch, "Image": Image, "transforms": transforms,
            "FileClient": FileClient, "imfrombytes": imfrombytes, "resize_flow": resize_flow, "flowread": flowread,
            "Stack": cu.Stack, "ToTorchFormatTensor": cu.ToTorchFormatTensor}
    reference_defs(os.path.join(REF, "core", "dataset.py"), ["TestDataset"], ns_d)

    combined = []

    class RecordingRFC(RecurrentFlowCompleteNet):
        def combine_flow(self, gt, pred, masks):
            out = super().combine_flow(gt, pred, masks)
            combined.append((tuple(g.clone() for g in gt), tuple(o.clone() for o in out)))
            return out

    from torch.utils.data import DataLoader
    readings = iter(range(1 << 20))
    time = lambda: next(readings) / 16
    torch.cuda.synchronize = lambda *a, **k: None
    ns = {"os": os, "np": np, "torch": torch, "DataLoader": DataLoader, "TestDataset": ns_d["TestDataset"],
          "RAFT_bi": RAFT_bi, "RecurrentFlowCompleteNet": RecordingRFC, "time": time}
    reference_defs(os.path.join(REF, "scripts", "evaluate_flow_completion.py"), ["main_worker"], ns)
    args = argparse.Namespace(height=SIZE[1], width=SIZE[0], raft_model_path=ck_raft, fc_model_path=ck_rfc,
                              dataset="davis", video_root=os.path.join(tmp, "JPEGImages"),
                              mask_root=os.path.join(tmp, "masks"), flow_root=os.path.join(tmp, "flows"), load_flow=True,
                              raft_iter=20, save_results=False, num_workers=0)
    os.chdir(tmp)
    try:
        ns["main_worker"](args)
    finally:
        os.chdir(cwd)
    summary = open(os.path.join(tmp, "results_flow", "davis", "davis_metrics.txt")).read()

    out = {"names": np.array([v[0] for v in VIDEOS]), "lengths": np.array([v[1] for v in VIDEOS]),
           "masks_kind": np.array([v[2] for v in VIDEOS]), "seeds": np.array([v[3] for v in VIDEOS]),
           "native": np.array([v[4] for v in VIDEOS]), "size": np.array(SIZE), "raft_iter": np.array(20),
           "summary": np.array(summary)}
    for vi, (name, T, _, _, _) in enumerate(VIDEOS):
        flo = {}
        for d in ("f", "b"):
            fl = []
            for t in range(T - 1):
                a, b = (t, t + 1) if d == "f" else (t + 1, t)
                fl.append(flowread(os.path.join(tmp, "flows", name, f"{a:05d}_{b:05d}_{d}.flo"), quantize=False))
            flo[d] = np.stack(fl).transpose(0, 3, 1, 2)                        # [T-1,2,h,w]
            assert np.array_equal(flo[d].astype(np.float16).astype(np.float32), flo[d])
            out[f"{name}_flow_{d}_sub4"] = flo[d][..., ::4, ::4].astype(np.float16)
        gt, pred = combined[vi]
        assert np.array_equal(gt[0][0].numpy(), flo["f"]) and np.array_equal(gt[1][0].numpy(), flo["b"])
        out[f"{name}_pred_f_sub4"] = pred[0][0, ..., ::4, ::4].numpy().astype(np.float16)
        out[f"{name}_pred_b_sub4"] = pred[1][0, ..., ::4, ::4].numpy().astype(np.float16)
        # main_worker's own expression (evaluate_flow_completion.py:141-142) on the tensors it used
        epe1 = torch.mean(torch.sum((gt[0].cpu() - pred[0].cpu()) ** 2, dim=2).sqrt())
        epe2 = torch.mean(torch.sum((gt[1].cpu() - pred[1].cpu()) ** 2, dim=2).sqrt())
        out[f"{name}_epe"] = np.array([epe1.item(), epe2.item()])
        print(name, "T", T, "EPE", out[f"{name}_epe"], "|flow|max", np.abs(flo["f"]).max(), np.abs(flo["b"]).max())
    path = os.path.join(HERE, GOLD_NAME + ".npz")
    np.savez_compressed(path, **out)
    print(summary)
    print(GOLD_NAME, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
