"""Oracle (test infrastructure): the video-completion protocol of scripts/evaluate_propainter.py::main_worker (:88-254)
and its dataset (core/dataset.py::TestDataset.__getitem__, :173-231), restated on the CPU in fp32 from the oracle
pipeline pieces.  File I/O is outside this path: frames / masks / flows come in as the arrays the files hold.

  * test_inputs: TestDataset after file I/O -- cv2.resize(INTER_LINEAR) of the RGB frames, PIL NEAREST of the masks,
    > 0, cv2.dilate (3x3 cross, 4 iterations), resize_flow of the loaded flows;
  * resize_flow: utils/flow_util.py:6-11 restated in numpy (OpenCV's float32 INTER_LINEAR: float coefficients, unfused
    separable passes, exact 2x down-scaling as INTER_AREA; then the float32 in-place rescale) -- pinned to cv2 itself in
    tests/test_eval_protocol_host.py;
  * run_video: flow completion and image propagation once over the whole clip, windows of neighbor_length with every
    ref_stride-th frame of the clip as reference, and the float-valued 1/2-1/2 blend (:166-179);
  * metrics / summary lines (:186-254), SSIM as propainter_b200.evaluate.ssim_frames restates it.
"""
import numpy as np
import torch

from . import flowcomp_ref, generator_ref, pipeline_ref


def linear_f32_tables(in_size, out_size, horizontal):
    """OpenCV's INTER_LINEAR coordinate rule for one axis (resize.cpp): fx = float((d + 0.5) * scale - 0.5) with
    scale = 1 / (out / in) in double, sx = floor(fx), fx -= sx; horizontally sx < 0 -> (0, 0) and sx >= n - 1 ->
    (n - 1, 0).  -> (ofs int [out], coef float32 [out, 2] = (1 - fx, fx))"""
    scale = 1.0 / (out_size / in_size)
    ofs = np.empty(out_size, np.int64)
    coef = np.empty((out_size, 2), np.float32)
    for d in range(out_size):
        f = np.float32((d + 0.5) * scale - 0.5)
        s = int(np.floor(f))
        f = np.float32(f - np.float32(s))
        if horizontal:
            if s < 0:
                f, s = np.float32(0), 0
            if s >= in_size - 1:
                f, s = np.float32(0), in_size - 1
        ofs[d] = s
        coef[d] = (np.float32(1) - f, f)
    return ofs, coef


def resize_flow(flows, size):
    """resize_flow of planar float32 flows [N,2,H,W] -> [N,2,Ho,Wo], size = (Wo, Ho)"""
    flows = np.asarray(flows, np.float32)
    N, _, H, W = flows.shape
    Wo, Ho = size
    f32 = np.float32
    if (Ho, Wo) == (H, W):
        out = flows.copy()
    elif W == 2 * Wo and H == 2 * Ho:
        a, b = flows[..., 0::2, 0::2], flows[..., 0::2, 1::2]
        c, d = flows[..., 1::2, 0::2], flows[..., 1::2, 1::2]
        out = (((a + b) + c) + d) * f32(0.25)
    else:
        xo, xa = linear_f32_tables(W, Wo, True)
        yo, ya = linear_f32_tables(H, Ho, False)
        edge = xo + 1 >= W
        x1 = np.minimum(xo + 1, W - 1)
        rows = np.where(edge, flows[..., xo] * xa[:, 0], flows[..., xo] * xa[:, 0] + flows[..., x1] * xa[:, 1])
        y0, y1 = np.clip(yo, 0, H - 1), np.clip(yo + 1, 0, H - 1)
        out = rows[..., y0, :] * ya[:, 0, None] + rows[..., y1, :] * ya[:, 1, None]
    out = out.astype(np.float32)
    out[:, 0] *= f32(Wo / W)
    out[:, 1] *= f32(Ho / H)
    return out


def test_inputs(frames_rgb, masks_u8, size, flows=None):
    """TestDataset.__getitem__ after file I/O.  frames_rgb uint8 [T,H0,W0,3], masks_u8 uint8 [T,H0,W0], flows None or
    (forward, backward) float32 [T-1,2,Hf,Wf].  -> (frames uint8 [T,h,w,3], masks float32 {0,1} [1,T,1,h,w], flows)"""
    import cv2
    from PIL import Image
    w, h = size
    frames = np.stack([cv2.resize(f, (w, h), interpolation=cv2.INTER_LINEAR) for f in frames_rgb])
    cross = cv2.getStructuringElement(cv2.MORPH_CROSS, (3, 3))
    masks = []
    for m in masks_u8:
        m = np.asarray(Image.fromarray(m).resize((w, h), Image.NEAREST).convert('L'))
        masks.append(cv2.dilate((m > 0).astype(np.uint8), cross, iterations=4))
    masks = np.stack(masks).astype(np.float32)[None, :, None]
    if flows is not None:
        flows = tuple(resize_flow(f, (w, h)) for f in flows)
    return frames, masks, flows


def float_blend(comp, idx, pred01_255, bm, ori):
    """:170-178 for one local frame: pred01_255 float32 [H,W,3] = ((p + 1) / 2) * 255, bm uint8 [H,W,1]"""
    img = np.array(pred01_255).astype(np.uint8) * bm + ori * (1 - bm)
    if comp[idx] is None:
        comp[idx] = img
    else:
        comp[idx] = comp[idx].astype(np.float32) * 0.5 + img.astype(np.float32) * 0.5


def window_plan(T, neighbor_length=20, ref_stride=10):
    """:148-154 with get_ref_index :29-34: every ref_stride-th frame of the whole clip not among the neighbours"""
    ns = neighbor_length // 2
    plan = []
    for f in range(0, T, ns):
        nb = list(range(max(0, f - ns), min(T, f + ns + 1)))
        plan.append((nb, [i for i in range(0, T, ref_stride) if i not in nb]))
    return plan


@torch.no_grad()
def run_video(sds, frames_u8, masks, flows, neighbor_length=20, ref_stride=10):
    """:103-179 with loaded flows: frames_u8 [T,h,w,3] uint8, masks [1,T,1,h,w] float {0,1}, flows (forward, backward)
    [T-1,2,h,w].  Returns the composited frames as a list (uint8 where visited once, float32 otherwise)."""
    frames = pipeline_ref.to_float_frames(frames_u8)
    masks = torch.as_tensor(masks).float()
    T, H, W = frames.shape[1], frames.shape[-2], frames.shape[-1]
    gt = tuple(torch.as_tensor(f).float().reshape(1, T - 1, 2, H, W) for f in flows)
    pred = flowcomp_ref.forward_bidirect_flow(sds["rfc"], gt, masks)
    pred = flowcomp_ref.combine_flow(gt, pred, masks)
    prop, upd_m = generator_ref.img_propagation(frames * (1 - masks), pred[0], pred[1], masks, "nearest")
    upd_f = frames * (1 - masks) + prop * masks
    comp = [None] * T
    ori = np.asarray(frames_u8)
    for nb, refs in window_plan(T, neighbor_length, ref_stride):
        ids = nb + refs
        p = generator_ref.generator_forward(sds["gen"], upd_f[:, ids], (pred[0][:, nb[:-1]], pred[1][:, nb[:-1]]),
                                            masks[:, ids], upd_m[:, ids], len(nb))
        p = ((p[0] + 1) / 2).permute(0, 2, 3, 1).numpy() * 255
        bm = masks[0, nb].permute(0, 2, 3, 1).numpy().astype(np.uint8)
        for i, idx in enumerate(nb):
            float_blend(comp, idx, p[i], bm[i], ori[idx])
    return comp


def psnr(ori, comp):
    """calculate_psnr (core/metrics.py:20-36) in float64"""
    mse = np.mean((ori.astype(np.float64) - comp.astype(np.float64)) ** 2)
    return float('inf') if mse == 0 else 20. * np.log10(255. / np.sqrt(mse))


def ssim(ori, comp):
    from propainter_b200.evaluate import ssim_frames
    return ssim_frames(torch.from_numpy(ori.astype(np.float64))[None], torch.from_numpy(comp.astype(np.float64))[None]).item()


def video_line(index, count, name, cur_psnr, cur_ssim, avg_psnr, avg_ssim, avg_time):
    """:219-226 (the backslash continuation keeps the next source line's 20 leading blanks in the string)"""
    return (f'[{index + 1:3}/{count}] Name: {str(name):25} | PSNR/SSIM: {cur_psnr:.4f}/{cur_ssim:.4f} '
            + ' ' * 20 + f'| Avg PSNR/SSIM: {avg_psnr:.4f}/{avg_ssim:.4f} | Time: {avg_time:.4f}')


def final_line(avg_psnr, avg_ssim, vfid, avg_time):
    """:250-251"""
    return f'Finish evaluation... Average Frame PSNR/SSIM/VFID: {avg_psnr:.2f}/{avg_ssim:.4f}/{vfid:.3f} | Time: {avg_time:.4f}'
