"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/hist_match.pt by running the UNMODIFIED MMCM `hist_match_video_bcthw`
(MMCM/mmcm/vision/process/correct_color.py:91-100, executed by oracle/hist_match_oracle.py with the restated skimage
`match_histograms`) the way the predictor calls it (pipeline_controlnet_predictor.py:745-749): on float32 slices
video[:, :, 1:] and video[:, :, :1] of one array, the float64 result stored back into it.

Run in the build container only:  python -m oracle.make_golden_hist_match
The fixture (~145 KB) keeps the seeded inputs and the float32 result. Frames: seeded noise, three distinct values, and
values at fl32(k / 255), which quantise to k, or one ulp below, which quantise to k - 1; batch item 1's template holds
k / 255 values.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.hist_match_oracle import mmcm_hist_match_video_bcthw  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "hist_match.pt")
SPEC = dict(B=2, C=3, F=3, H=24, W=31, seed=5)


def make_inputs(spec=SPEC):
    """video [B, C, 1 + F, H, W] float32: frame 0 is the template (H x W here), frames 1.. are matched to it."""
    B, C, F, H, W = (spec[k] for k in ("B", "C", "F", "H", "W"))
    rng = np.random.default_rng(spec["seed"])
    v = np.clip(rng.normal(0.45, 0.22, (B, C, 1 + F, H, W)), 0, 1).astype(np.float32)
    v[:, :, 2] = rng.choice(np.array([0.1, 0.5, 0.93], np.float32), size=(B, C, H, W))
    v[:, :, 3] = (rng.integers(0, 256, (B, C, H, W)) / np.float32(255)).astype(np.float32)
    below = rng.random((B, C, H, W)) < 0.5
    v[:, :, 3][below] = np.nextafter(v[:, :, 3][below], np.float32(0))
    v[1, :, 0] = (rng.integers(40, 200, (C, H, W)) / np.float32(255)).astype(np.float32)
    return v


def main():
    video = make_inputs()
    ref = mmcm_hist_match_video_bcthw()
    out = video.copy()
    out[:, :, 1:, :, :] = ref(out[:, :, 1:, :, :], out[:, :, :1, :, :], value=255.0)
    torch.save({"spec": SPEC, "video": torch.from_numpy(video), "out": torch.from_numpy(out)}, GOLDEN)
    print(GOLDEN, os.path.getsize(GOLDEN), "bytes")


if __name__ == "__main__":
    main()
