"""Drop-in for MMCM's `mmcm.vision.process.correct_color.hist_match_video_bcthw` (MMCM/mmcm/vision/process/correct_color.py:
91-100), the colour correction behind text2video's `--need_hist_match`: every generated frame's per-channel histogram
is matched to the vision-condition frame's, on the device (`musev_b200.ops.hist_match`).

    import musev.pipelines.pipeline_controlnet_predictor as pcp
    import musev_b200.correct_color
    pcp.hist_match_video_bcthw = musev_b200.correct_color.hist_match_video_bcthw
"""
from __future__ import annotations

import numpy as np
import torch

from . import ops


def hist_match_video_bcthw(video, target, value: float = 255.0):
    """video [B, C, F, H, W] and target [B, C, 1, H', W'], float32 with values in [0, 1], both numpy arrays or both CUDA
    tensors. Returns the matched video as float32 [B, C, F, H, W]: the values the reference's float64 result becomes when
    its caller stores it into its float32 array, bit for bit. numpy in, numpy out (the frames go to the device and back);
    CUDA tensors in, a new CUDA tensor out.

    Only value = 255.0 is taken: the engine quantises as uint8(fl32(x * 255)). A float64 input is refused too, since the
    reference would quantise fl64(x * 255) instead. Values outside [0, 1] saturate (NaN maps to 0) where the reference's
    uint8 cast is undefined."""
    if value != 255.0:
        raise ValueError(f"hist_match_video_bcthw: value must be 255.0 (the uint8 quantisation the engine implements), "
                         f"got {value}")
    if isinstance(video, np.ndarray) and isinstance(target, np.ndarray):
        for name, a in (("video", video), ("target", target)):
            if a.dtype != np.float32:
                raise TypeError(f"hist_match_video_bcthw: {name} must be float32 (another dtype quantises differently), "
                                f"got {a.dtype}")
        dev = torch.device("cuda", torch.cuda.current_device())
        v = torch.from_numpy(np.ascontiguousarray(video)).to(dev)
        t = torch.from_numpy(np.ascontiguousarray(target)).to(dev)
        return ops.hist_match(v, t, out=v).cpu().numpy()
    if isinstance(video, torch.Tensor) and isinstance(target, torch.Tensor):
        for name, a in (("video", video), ("target", target)):
            if not a.is_cuda or a.dtype != torch.float32:
                raise TypeError(f"hist_match_video_bcthw: {name} must be a float32 CUDA tensor (another dtype quantises "
                                f"differently; pass host data as numpy arrays), got {a.dtype} on {a.device}")
        return ops.hist_match(video, target)
    raise TypeError(f"hist_match_video_bcthw: video and target must both be numpy arrays or both CUDA tensors, got "
                    f"{type(video).__name__} and {type(target).__name__}")
