"""TEST INFRASTRUCTURE ONLY -- plain-torch fp32 restatement of `musev.models.controlnet.PoseGuider.forward`
(musev/models/controlnet.py:308-371) driven by a reference-format state dict, and the two places its output enters the
denoiser: `UNet3DPoseOracle` (the UNet's `pose_guider_emb` add) and `denoise_loop_with_pose` (the window loop). Pinned to the
imported, unmodified reference by tests/golden/pose_guider_{narrow,full}.pt and unet_pose_narrow.pt
(oracle/make_golden_pose_guider.py).

Only tests/ and tools/ may import this file; the product (musev_b200/) never does.
"""
from __future__ import annotations

from typing import Callable, Dict

import torch
import torch.nn.functional as F

from musev_b200.schema import PoseGuiderConfig, pose_guider_layers
from oracle.pipeline_oracle import denoise_loop, prepare_global_context
from oracle.unet3d_oracle import UNet3DOracle


class PoseGuiderOracle(torch.nn.Module):
    """conv_in + SiLU, (stride-1 conv + SiLU, stride-2 conv + SiLU) per block, conv_out; every conv 3x3 pad 1 and applied
    per frame (InflatedConv3d, :308-316). `forward` takes [b, c, t, H, W] like the reference; `frames` takes [N, c, H, W].
    An nn.Module so that eager fp16 timing (cuDNN) and FlopCounterMode can run it as is."""

    def __init__(self, cfg: PoseGuiderConfig, state_dict: Dict[str, torch.Tensor], device="cpu", dtype=torch.float32):
        super().__init__()
        self.cfg = cfg
        self.layers = pose_guider_layers(cfg)
        for name, _, _, _ in self.layers:
            self.register_buffer(name.replace(".", "_") + "_w", state_dict[name + ".weight"].to(device, dtype))
            self.register_buffer(name.replace(".", "_") + "_b", state_dict[name + ".bias"].to(device, dtype))

    def frames(self, x: torch.Tensor) -> torch.Tensor:
        n = len(self.layers)
        for i, (name, _, _, stride) in enumerate(self.layers):
            key = name.replace(".", "_")
            x = F.conv2d(x, getattr(self, key + "_w"), getattr(self, key + "_b"), stride=stride, padding=1)
            if i != n - 1:
                x = F.silu(x)
        return x

    def forward(self, conditioning: torch.Tensor) -> torch.Tensor:
        b, c, t, H, W = conditioning.shape
        x = conditioning.permute(0, 2, 1, 3, 4).reshape(b * t, c, H, W)
        e = self.frames(x)
        return e.reshape(b, t, *e.shape[1:]).permute(0, 2, 1, 3, 4)


class UNet3DPoseOracle(UNet3DOracle):
    """`UNet3DOracle` with the reference's `pose_guider_emb` add (unet_3d_condition.py:1011-1016):
    `sample = conv_in(sample) + pose_guider_emb` on the `(b t) c h w` output of conv_in, before transformer_in.

    The base forward is reused unchanged. conv_in is its only reader of `conv_in.bias`, and the residual-stream rounding
    `_qs` it applies to conv_in's output is the next `_qs` call, so `_w` arms the add and `_qs` performs it, once per
    forward. Without `pose_guider_emb` the forward is the base one."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._pose = None
        self._pose_armed = self._pose_added = False

    def _w(self, name):
        if name == "conv_in.bias" and self._pose is not None:
            self._pose_armed = True
        return super()._w(name)

    def _qs(self, x):
        if self._pose_armed:
            self._pose_armed, self._pose_added = False, True
            x = x + self._pose.to(x.device, x.dtype)
        return super()._qs(x)

    @torch.no_grad()
    def forward(self, sample, timestep, encoder_hidden_states, pose_guider_emb=None, **kwargs):
        self._pose, self._pose_armed, self._pose_added = pose_guider_emb, False, False
        try:
            out = super().forward(sample, timestep, encoder_hidden_states, **kwargs)
        finally:
            self._pose, self._pose_armed = None, False
        if pose_guider_emb is not None and not self._pose_added:
            raise RuntimeError("pose_guider_emb was not added after conv_in")
        return out

    __call__ = forward


def denoise_loop_with_pose(unet: Callable, scheduler, latents: torch.Tensor, condition_latents: torch.Tensor,
                           prompt_embeds: torch.Tensor, num_inference_steps: int, guidance_scale: float,
                           pose_guider_emb: torch.Tensor, context_frames: int = 12, context_overlap: int = 4,
                           context_schedule: str = "uniform_v2", context_stride: int = 1, **kwargs):
    """`oracle.pipeline_oracle.denoise_loop` with `pose_guider_emb` [2B, C0, n_vc + T, h, w] (vision-condition frames first)
    passed to every UNet call sliced to the window: the vision-condition frames, then the window's frames (duplicates
    included), as `(b t) c h w`. With one window over the whole video this is the reference's whole-video tensor
    (pipeline_controlnet.py:1774-1783, :2066); with several windows the reference's add cannot broadcast.

    The loop visits its windows in `prepare_global_context` order on every step; the wrapper walks the same list."""
    n_vc = condition_latents.shape[2]
    T, h, w = latents.shape[2:]
    contexts = [c[0] for c in prepare_global_context(context_schedule, num_inference_steps, T, context_frames,
                                                     context_stride, context_overlap, 1)]
    calls = [0]

    def unet_pose(sample, t, enc, **k):
        c = contexts[calls[0] % len(contexts)]
        calls[0] += 1
        assert sample.shape[2] == n_vc + len(c), "window order differs from prepare_global_context"
        pe = pose_guider_emb[:, :, list(range(n_vc)) + [ci + n_vc for ci in c]]
        return unet(sample, t, enc, pose_guider_emb=pe.permute(0, 2, 1, 3, 4).reshape(-1, pe.shape[1], h, w), **k)

    out = denoise_loop(unet_pose, scheduler, latents, condition_latents, prompt_embeds, num_inference_steps, guidance_scale,
                       context_frames=context_frames, context_overlap=context_overlap, context_schedule=context_schedule,
                       context_stride=context_stride, **kwargs)
    assert calls[0] == num_inference_steps * len(contexts)
    return out
