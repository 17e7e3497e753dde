"""CPU tests of the evaluation script's video-completion protocol (propainter_b200.evaluate.evaluate_video): the float
compositing rule pp_composite_f32 (host build of pp_elem.cuh) against a numpy restatement of
scripts/evaluate_propainter.py:166-179, the flow-resize rule of pp_resize_flow_linear_cv (its host tables + the oracle's
numpy emulation) against cv2.resize + the in-place rescale, the protocol's window plan against the script's, and the
oracle protocol (oracle/eval_protocol_ref.py) against the fixture made by the unmodified script
(tests/golden/make_golden_eval_protocol.py).  The kernels run on the GPU in test_gpu_eval_protocol.py."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from oracle import eval_protocol_ref as epr

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "eval_protocol_2v_128x224.npz")

# (H, W) -> (Wo, Ho): down, non-integer, up, exact 2x (INTER_AREA), same size, one axis only, odd shapes
RESIZE_CASES = [((480, 854), (432, 240)), ((720, 1280), (432, 240)), ((200, 300), (128, 128)), ((128, 128), (256, 256)),
                ((256, 256), (128, 128)), ((144, 240), (224, 128)), ((60, 60), (60, 60)), ((64, 96), (50, 64)),
                ((64, 96), (96, 40)), ((37, 53), (53, 37)), ((33, 17), (70, 9))]


@pytest.fixture(scope="module")
def hs(tmp_path_factory):
    lib = os.path.join(str(tmp_path_factory.mktemp("hostsim_eval")), "libhostsim_eval.so")
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", lib,
                           os.path.join(HERE, "hostsim", "hostsim_eval.cpp")])
    return ctypes.CDLL(lib)


def script_blend(preds, masks, ori, visits):
    """:166-179 verbatim on numpy: preds {window: [n,3,H,W] float32}, visits [(window, nb)]"""
    comp = [None] * len(ori)
    for w, nb in visits:
        p = (preds[w] + np.float32(1)) / np.float32(2)
        p = p.transpose(0, 2, 3, 1) * 255
        bm = masks[nb].transpose(0, 2, 3, 1).astype(np.uint8)
        for i, idx in enumerate(nb):
            img = np.array(p[i]).astype(np.uint8) * bm[i] + ori[idx] * (1 - bm[i])
            if comp[idx] is None:
                comp[idx] = img
            else:
                comp[idx] = comp[idx].astype(np.float32) * 0.5 + img.astype(np.float32) * 0.5
    return comp


def test_composite_f32_rule_matches_script(hs):
    rng = np.random.default_rng(3)
    T, H, W = 7, 9, 11
    ori = rng.integers(0, 256, (T, H, W, 3), dtype=np.uint8)
    masks = (rng.random((T, 1, H, W)) < 0.6).astype(np.float32)
    masks[0] = 0
    masks[1] = 1
    # frames 0-1 seen once, 2-3 twice, 4-6 three times
    visits = [(0, [0, 2, 3, 4, 5]), (1, [1, 2, 4, 5, 6]), (2, [3, 4, 6]), (3, [5, 6])]
    preds = {}
    for w, nb in visits:
        p = rng.uniform(-1, 1, (len(nb), 3, H, W)).astype(np.float32)
        # values whose ((p + 1) / 2) * 255 lands on or next to an integer: the truncation boundaries
        k = rng.integers(0, 256, p.shape)
        edge = (k / 255.0 * 2 - 1).astype(np.float32)
        sel = rng.random(p.shape) < 0.5
        p[sel] = np.nextafter(edge, rng.choice([-2, 2], p.shape).astype(np.float32))[sel]
        p[0, 0, 0, :2] = (-1.0, 1.0)
        preds[w] = p
    ref = script_blend(preds, masks[:, :, :, :], ori, visits)
    got = np.zeros((T, H, W, 3), np.float32)
    seen = [False] * T
    fp = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))
    for w, nb in visits:
        p = np.ascontiguousarray(preds[w])
        fr = (ctypes.c_int * len(nb))(*nb)
        first = (ctypes.c_int * len(nb))(*[int(not seen[i]) for i in nb])
        hs.hs_composite_f32(fp(p), fp(masks), ori.ctypes.data_as(ctypes.c_void_p), fp(got), len(nb), fr, first, H, W)
        for i in nb:
            seen[i] = True
    for t in range(T):
        assert np.array_equal(got[t], ref[t].astype(np.float32)), t
    assert (got[4:] * 4 % 2 == 1).any()                                      # three visits: quarter values occur
    assert np.array_equal(got[1] % 1, np.zeros_like(got[1]))                  # one visit: integers


@pytest.mark.parametrize("src,size", RESIZE_CASES, ids=[f"{s[0]}x{s[1]}-{d[1]}x{d[0]}" for s, d in RESIZE_CASES])
def test_resize_flow_emulation_matches_cv2(src, size):
    cv2 = pytest.importorskip("cv2")
    H, W = src
    Wo, Ho = size
    f = (np.random.default_rng(H * W).standard_normal((3, 2, H, W)) * 20).astype(np.float32)
    ref = []
    for fl in f:
        r = cv2.resize(np.ascontiguousarray(fl.transpose(1, 2, 0)), (Wo, Ho), interpolation=cv2.INTER_LINEAR)
        r[:, :, 0] *= Wo / W                                                   # utils/flow_util.py:9-10
        r[:, :, 1] *= Ho / H
        ref.append(r.transpose(2, 0, 1))
    assert np.array_equal(epr.resize_flow(f, size), np.stack(ref))


@pytest.mark.parametrize("n_in,n_out", [(854, 432), (480, 240), (128, 256), (240, 224), (144, 128), (17, 70), (60, 60)])
def test_resize_flow_tables_match_oracle(n_in, n_out):
    """the library's host tables (pp_resample_coeffs_linear_f32) are the oracle's coordinate rule"""
    from propainter_b200 import ops
    try:
        tabs = {h: ops.resample_tables("linear_f32", n_in, n_out, None, h) for h in (True, False)}
    except RuntimeError as e:
        pytest.skip(str(e))                                                    # library not built
    for h, (ofs, coef) in tabs.items():
        o, c = epr.linear_f32_tables(n_in, n_out, h)
        assert np.array_equal(ofs.numpy(), o) and np.array_equal(coef.numpy(), c)


def test_protocol_window_plan_matches_script():
    from propainter_b200.inference_propainter import InferenceConfig, window_plan

    def script_plan(T, nl=20, rs=10):                                         # evaluate_propainter.py:29-34, :148-154
        out = []
        for f in range(0, T, nl // 2):
            nb = [i for i in range(max(0, f - nl // 2), min(T, f + nl // 2 + 1))]
            out.append((nb, [i for i in range(0, T, rs) if i not in nb]))
        return out
    for T in (1, 5, 11, 17, 24, 61, 80, 81, 90, 157, 230):
        for nl, rs in ((20, 10), (10, 5), (20, 7)):
            cfg = InferenceConfig(neighbor_length=nl, ref_stride=rs, subvideo_length=max(T, 1))
            assert window_plan(T, cfg) == script_plan(T, nl, rs) == epr.window_plan(T, nl, rs), (T, nl, rs)


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLD))


def golden_inputs(g, vi):
    from tests.eval_protocol_inputs import video_inputs
    name, T = str(g["names"][vi]), int(g["lengths"][vi])
    return name, video_inputs(T, str(g["masks_kind"][vi]), int(g["seeds"][vi]))


def test_oracle_inputs_match_fixture(gold):
    """the oracle's TestDataset restatement gives the script's frames, masks and resized flows bit for bit"""
    pytest.importorskip("cv2")
    from tests.eval_protocol_inputs import digest
    size = tuple(int(s) for s in gold["size"])
    for vi in range(len(gold["names"])):
        name, (fr, mk, fl) = golden_inputs(gold, vi)
        f, m, flows = epr.test_inputs(fr, mk, size, fl)
        assert digest(f) == str(gold[f"{name}_sha_frames"])
        assert digest(m.astype(np.float32)) == str(gold[f"{name}_sha_masks"])
        assert digest(np.stack(flows)) == str(gold[f"{name}_sha_flows"])


def test_oracle_protocol_reproduces_fixture(gold):
    """oracle/eval_protocol_ref.py's fp32 CPU restatement against the unmodified script: the float composited video
    (all but < 0.01 % of the values equal), per-frame PSNR / SSIM, and the summary lines (the times aside)"""
    pytest.importorskip("cv2")
    from propainter_b200 import schemas
    from propainter_b200._params import ParamNet
    from propainter_b200.evaluate import fid_from_activations
    sds = {"rfc": ParamNet(schemas.rfc_schema(), seed=2).state_dict(), "gen": ParamNet(schemas.generator_schema(), seed=3).state_dict()}
    size = tuple(int(s) for s in gold["size"])
    n = len(gold["names"])
    lines, all_p, all_s = [], [], []
    for vi in range(n):
        name, (fr, mk, fl) = golden_inputs(gold, vi)
        f, m, flows = epr.test_inputs(fr, mk, size, fl)
        comp = np.stack(epr.run_video(sds, f, m, flows)).astype(np.float64)
        hole = m[0, :, 0] > 0
        ref = f.astype(np.float64)
        ref[hole] = gold[f"{name}_comp4_holes"] / 4.0
        # the oracle's convolutions round differently from the reference modules': a few values move by a level
        bad = comp != ref
        assert bad.mean() < 1e-4 and np.abs(comp - ref).max() <= 2, (name, int(bad.sum()), np.abs(comp - ref).max())
        ps = [epr.psnr(f[t], comp[t]) for t in range(len(f))]
        ss = [epr.ssim(f[t], comp[t]) for t in range(len(f))]
        assert np.allclose(ps, gold[f"{name}_psnr"], rtol=0, atol=1e-3)
        assert np.allclose(ss, gold[f"{name}_ssim"], rtol=0, atol=1e-5)
        # the lines' arithmetic on the script's own per-frame values
        ps, ss = list(gold[f"{name}_psnr"]), list(gold[f"{name}_ssim"])
        all_p += ps
        all_s += ss
        lines.append(epr.video_line(vi, n, name, sum(ps) / len(ps), sum(ss) / len(ss), sum(all_p) / len(all_p),
                                    sum(all_s) / len(all_s), 0.0))
    real = np.stack([gold[f"{gold['names'][vi]}_i3d_real"] for vi in range(n)])
    fake = np.stack([gold[f"{gold['names'][vi]}_i3d_comp"] for vi in range(n)])
    lines.append(epr.final_line(sum(all_p) / len(all_p), sum(all_s) / len(all_s), fid_from_activations(real, fake), 0.0))
    untimed = lambda s: re.sub(r"Time: [0-9.]+", "Time: -", s)
    assert [untimed(x) for x in lines] == [untimed(x) for x in str(gold["summary"]).strip().split("\n")]


def test_protocol_lines_match_oracle():
    from propainter_b200.evaluate import protocol_video_line
    rec = {"psnr": 20.67171, "ssim": 0.778712}
    assert protocol_video_line(0, 2, "bear", rec, 20.5, 0.7, 0.72461) == epr.video_line(0, 2, "bear", 20.67171, 0.778712,
                                                                                         20.5, 0.7, 0.72461)


def test_evaluate_video_refuses_half_storage_and_unknown_task():
    from propainter_b200.evaluate import evaluate_video
    from propainter_b200.inference_propainter import InferenceConfig

    class Pipe:
        device = torch.device("cpu")
    with pytest.raises(ValueError):
        evaluate_video(Pipe(), np.zeros((3, 8, 8, 3), np.uint8), np.zeros((1, 3, 1, 8, 8), np.float32),
                       cfg=InferenceConfig(half_storage=True))
    with pytest.raises(ValueError):
        evaluate_video(Pipe(), np.zeros((3, 8, 8, 3), np.uint8), np.zeros((1, 3, 1, 8, 8), np.float32), task="inpaint")


def test_resize_flow_refuses_bad_arguments():
    from propainter_b200 import ops
    with pytest.raises(ValueError):
        ops.resize_flow(torch.zeros(2, 3, 8, 8), (4, 4))
    with pytest.raises(ValueError):
        ops.resize_flow(torch.zeros(2, 2, 8, 8, dtype=torch.float16), (4, 4))
    with pytest.raises(ValueError):
        ops.resize_flow(torch.zeros(2, 2, 8, 8), (0, 4))
