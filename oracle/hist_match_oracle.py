"""numpy restatement of the `need_hist_match` colour correction of text2video
(musev/pipelines/pipeline_controlnet_predictor.py:745-749):

  MMCM `hist_match_video_bcthw` (MMCM/mmcm/vision/process/correct_color.py:91-100): channels last, q = (x * value)
      .astype(uint8), one `match_histograms(frame, target[b], channel_axis=-1)` per batch item and frame, then / value.
      Pinned: `mmcm_hist_match_video_bcthw()` executes the unmodified file (through oracle/ref_shim.py's module stubs)
      with the restated `match_histograms` below standing in for `skimage.exposure`, and tests/golden/hist_match.pt
      (oracle/make_golden_hist_match.py) holds what it returns.
  skimage 0.22 `exposure.match_histograms` / `_match_cumulative_cdf` (skimage/exposure/histogram_matching.py; MMCM pins
      scikit-image==0.22.0, MMCM/requirements.txt:213) on uint8 images: **parity unpinned** -- scikit-image is not a
      dependency of this project or of its build, so this restatement of its uint8 branch is the specification and no
      test runs skimage itself. Per channel: bincount of source and template, the template's non-empty bins as the
      ordinates, cumulative counts over the pixel count as the quantiles, `np.interp` of the source quantiles, gathered
      per pixel; the channels are assembled as float64.
"""
from __future__ import annotations

import importlib.util
import os
import sys

import numpy as np


def match_cumulative_cdf(source: np.ndarray, template: np.ndarray) -> np.ndarray:
    """skimage 0.22 `_match_cumulative_cdf`, unsigned-integer branch: float64 image of source's shape."""
    if source.dtype.kind != "u" or template.dtype.kind != "u":
        raise TypeError("the restatement covers the unsigned-integer branch only (uint8 frames)")
    src_lookup = source.reshape(-1)
    src_counts = np.bincount(src_lookup)
    tmpl_counts = np.bincount(template.reshape(-1))
    tmpl_values = np.nonzero(tmpl_counts)[0]          # omit values where the count was 0
    tmpl_counts = tmpl_counts[tmpl_values]
    src_quantiles = np.cumsum(src_counts) / source.size
    tmpl_quantiles = np.cumsum(tmpl_counts) / template.size
    interp_a_values = np.interp(src_quantiles, tmpl_quantiles, tmpl_values)
    return interp_a_values[src_lookup].reshape(source.shape)


def match_histograms(image: np.ndarray, reference: np.ndarray, *, channel_axis=None) -> np.ndarray:
    """skimage 0.22 `exposure.match_histograms` for uint8 images: each channel matched on its own (channel_axis=-1, the
    only use MMCM makes of it), or the whole image as one channel (None)."""
    if image.ndim != reference.ndim:
        raise ValueError("Image and reference must have the same number of channels.")
    if channel_axis is None:
        return match_cumulative_cdf(image, reference)
    if channel_axis != -1:
        raise ValueError("the restatement covers channel_axis=-1 and None")
    if image.shape[-1] != reference.shape[-1]:
        raise ValueError("Number of channels in the input image and reference image must match!")
    matched = np.empty(image.shape, dtype=np.float64)
    for channel in range(image.shape[-1]):
        matched[..., channel] = match_cumulative_cdf(image[..., channel], reference[..., channel])
    return matched


def hist_match_video_bcthw(video: np.ndarray, target: np.ndarray, value: float = 255.0) -> np.ndarray:
    """MMCM `hist_match_video_bcthw` restated without einops: video [b, c, t, h, w], target [b, c, 1, h', w'] -> float64
    [b, c, t, h, w]. Equal to the unmodified function (tests/test_hist_match_host.py)."""
    v = (np.transpose(video, (0, 2, 3, 4, 1)) * value).astype(np.uint8)            # b t h w c
    tg = np.transpose(target, (0, 2, 3, 4, 1))
    tg = (tg.reshape(-1, *tg.shape[2:]) * value).astype(np.uint8)                    # (b t) h w c
    out = np.stack([np.stack([match_histograms(v[b, t], tg[b], channel_axis=-1) for t in range(v.shape[1])])
                    for b in range(v.shape[0])])
    return np.transpose(out / value, (0, 4, 1, 2, 3))


def hist_match_video_f32(video: np.ndarray, target: np.ndarray) -> np.ndarray:
    """What the predictor keeps: the float64 result stored into its float32 video array."""
    return hist_match_video_bcthw(video, target, 255.0).astype(np.float32)


def mmcm_hist_match_video_bcthw():
    """The unmodified MMCM `hist_match_video_bcthw`, executed from the reference tree with `skimage.exposure` bound to the
    restated `match_histograms` and MMCM's package imports stubbed (the module only imports `DecordVideoDataset` for a
    function not used here). sys.modules is left as it was found. Needs the reference tree (ref_shim.available())."""
    from oracle import ref_shim
    path = os.path.join(ref_shim.REFERENCE_ROOT, "MMCM", "mmcm", "vision", "process", "correct_color.py")
    if not os.path.isfile(path):
        raise RuntimeError(f"reference file not found: {path}")
    names = ("mmcm", "mmcm.vision", "mmcm.vision.process", "mmcm.vision.data", "mmcm.vision.data.video_dataset",
             "skimage", "skimage.exposure", "mmcm.vision.process.correct_color")
    saved = {n: sys.modules.get(n) for n in names}
    try:
        for n in names[:4]:
            ref_shim._stub(n)
        ref_shim._stub("mmcm.vision.data.video_dataset", DecordVideoDataset=type("DecordVideoDataset", (), {}))
        ref_shim._stub("skimage").exposure = ref_shim._stub("skimage.exposure", match_histograms=match_histograms)
        spec = importlib.util.spec_from_file_location("mmcm.vision.process.correct_color", path)
        mod = importlib.util.module_from_spec(spec)
        sys.modules[spec.name] = mod
        spec.loader.exec_module(mod)
    finally:
        for n, m in saved.items():
            if m is None:
                sys.modules.pop(n, None)
            else:
                sys.modules[n] = m
    return mod.hist_match_video_bcthw
