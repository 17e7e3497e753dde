"""Inputs of the compute_flow fixture (tests/golden/make_golden_compute_flow.py), regenerated from seeds by the tests:
synth.make_clip frames / masks at each video's native size, one down-scaled and one up-scaled to the 160 x 128 eval size."""
import numpy as np

from propainter_b200 import synth

GOLD_NAME = "compute_flow_2v_128x160"
SIZE = (160, 128)                                                    # (width, height), the scripts' --width / --height
VIDEOS = [("bear", 8, "ellipse", 0, (200, 240)), ("swing", 6, "square", 1, (96, 120))]   # name, T, mask, seed, (H0, W0)


def video_inputs(T, mask, seed, native):
    """-> (frames uint8 [T,H0,W0,3] RGB, masks uint8 [T,H0,W0] 0 / 255)"""
    u8, fm, _ = synth.make_clip(T, native[0], native[1], mask=mask, seed=seed)
    return u8, (fm[0, :, 0].numpy() > 0).astype(np.uint8) * 255
