"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the Multi-ControlNet path of the reference.

  * multi_controlnet_forward   diffusers `MultiControlNetModel.forward`
                               (diffusers/src/diffusers/pipelines/controlnet/multicontrolnet.py:31-72) over
                               `ControlNetOracle`s: every net on the same sample, maps summed in net order (:64-70)
  * denoise_loop_multi         `oracle.pipeline_oracle.denoise_loop` with several ControlNets per window-step:
                               per-net condition latents, scales (:1548-1553) and keep lists (:1229-1235,1700-1711)
Pinned against the unmodified diffusers class by oracle/make_golden_multicontrolnet.py -> tests/golden/multicontrolnet_narrow.pt.
Not imported by the product path.
"""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence, Union

import torch

from oracle.pipeline_oracle import denoise_loop


@torch.no_grad()
def multi_controlnet_forward(nets: List[Callable], sample, timestep, encoder_hidden_states,
                             controlnet_cond: Optional[List[torch.Tensor]], conditioning_scale: List[float],
                             guess_mode=False, controlnet_cond_latents: Optional[List[torch.Tensor]] = None):
    """MultiControlNetModel.forward (multicontrolnet.py:31-72): each net with its own image (or condition latents) and
    scale, the maps summed in net order (:64-70), here in the oracles' dtype."""
    down, mid = None, None
    for k, net in enumerate(nets):
        d, m = net(sample, timestep, encoder_hidden_states,
                   controlnet_cond=None if controlnet_cond is None else controlnet_cond[k],
                   conditioning_scale=conditioning_scale[k], guess_mode=guess_mode,
                   controlnet_cond_latents=None if controlnet_cond_latents is None else controlnet_cond_latents[k])
        if down is None:
            down, mid = d, m
        else:
            down = [a + b for a, b in zip(down, d)]
            mid = mid + m
    return down, mid


def denoise_loop_multi(unet: Callable, scheduler, latents: torch.Tensor, condition_latents: torch.Tensor,
                       prompt_embeds: torch.Tensor, num_inference_steps: int, guidance_scale: float,
                       controlnets: Sequence[Callable], controlnet_latents: Sequence[torch.Tensor],
                       controlnet_conditioning_scale: Union[float, Sequence[float]] = 1.0,
                       controlnet_keep: Optional[Sequence[Sequence[float]]] = None, **kwargs):
    """`denoise_loop` with a Multi-ControlNet in every window-step (pipeline_controlnet.py:1992-2038, :1202-1291).

    controlnet_latents: one [2B, C0, n_vc + T, h, w] tensor per net. controlnet_conditioning_scale: a float for every
    net (:1548-1553) or one per net. controlnet_keep: one list per step (:1700-1711). As in the reference, every net runs
    in every window-step with scale * keep (:1229-1235).

    The per-net latents travel through `denoise_loop`'s single `controlnet_latents` argument concatenated on the channel
    axis, so the loop slices every net's frames exactly as it slices one net's; the callable splits them again and maps
    the timestep back to its step index for the keep list."""
    n = len(controlnets)
    if len(controlnet_latents) != n:
        raise ValueError(f"{len(controlnet_latents)} controlnet_latents for {n} ControlNets")
    scales = list(controlnet_conditioning_scale) if isinstance(controlnet_conditioning_scale, (list, tuple)) \
        else [controlnet_conditioning_scale] * n
    widths = [lat.shape[1] for lat in controlnet_latents]
    scheduler.set_timesteps(num_inference_steps)
    step_of = {int(t): i for i, t in enumerate(scheduler.timesteps)}

    def multi(x2, t, enc2, controlnet_cond_latents, conditioning_scale=1.0):
        keep = [1.0] * n if controlnet_keep is None else controlnet_keep[step_of[int(t)]]
        return multi_controlnet_forward(controlnets, x2, t, enc2, None, [s * k for s, k in zip(scales, keep)],
                                        controlnet_cond_latents=list(controlnet_cond_latents.split(widths, dim=1)))

    return denoise_loop(unet, scheduler, latents, condition_latents, prompt_embeds, num_inference_steps, guidance_scale,
                        controlnet=multi, controlnet_latents=torch.cat(list(controlnet_latents), dim=1), **kwargs)
