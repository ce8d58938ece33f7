"""Visual-Conditioned Parallel-Denoise loop on the CUDA engine.

Mirrors the loop body of `MusevControlNetPipeline.__call__` (musev/pipelines/pipeline_controlnet.py:1846-2147):
per step, every window -> UNet -> accumulate eps; overlap mean; CFG; scheduler.step. What changes:
  * the UNet forward is the CUDA engine (musev_b200.unet.UNet3DConditionModel);
  * the ~12 pointwise launches of mean / CFG / DDIM are ONE kernel (`mvb_fuse_cfg_ddim`);
  * windows are sharded over the ranks of a torch.distributed process group (one process per GPU) with exactly one
    all-reduce (sum) of the eps accumulator per step -- the reference loops over windows on a single GPU. Every
    rank keeps the full latents and applies the identical fused update, so latents stay replicated bit-exactly.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Sequence, Union

import torch

from . import ops
from .context import assign_windows, prepare_global_context
from .samplers import multistep_update
from .scheduler import DDIMScheduler, _PRED, _variance_noise
from .unet import UNet3DConditionModel


@dataclass
class DenoiseOutput:
    latents: torch.Tensor
    windows: List[List[int]]
    windows_per_rank: List[List[int]]


class ParallelDenoiser:
    def __init__(self, unet, scheduler, process_group=None, device_ops=None):
        """scheduler: musev_b200 `DDIMScheduler` (any prediction type / clipping / eta), one of the affine samplers of
        musev_b200.samplers (`EulerDiscreteScheduler`, the predictor's default; `LCMScheduler`) or any scheduler with a
        `multistep_plan` (`DPMSolverMultistepScheduler`, `EulerAncestralDiscreteScheduler`, `DDPMScheduler`)."""
        # device_ops: module providing accumulate_window / fuse_cfg_*; the CUDA library unless a test injects a double
        self.ops = device_ops if device_ops is not None else ops
        self.unet = unet
        # The engine UNet runs the layers before the first per-half input once for both CFG halves when told that their
        # samples are equal; any other callable (a reference model, a test double) is called as the reference calls it.
        self._shares_cfg_prefix = isinstance(unet, UNet3DConditionModel)
        self.scheduler = scheduler
        self.pg = process_group
        self._dist = None
        if process_group is not None or (torch.distributed.is_available() and torch.distributed.is_initialized()):
            import torch.distributed as dist
            self._dist = dist
        self.rank = self._dist.get_rank(self.pg) if self._dist else 0
        self.world = self._dist.get_world_size(self.pg) if self._dist else 1

    @torch.no_grad()
    def __call__(
        self,
        latents: torch.Tensor,                 # [B, 4, T, h, w] initial noise * init_noise_sigma
        condition_latents: torch.Tensor,       # [B, 4, n_vc, h, w] vision-condition latents
        prompt_embeds: torch.Tensor,           # [2B, 77, 768] = cat([negative, positive]) (pipeline_controlnet.py:1565-1577)
        num_inference_steps: int = 20,
        guidance_scale: float = 3.5,
        context_frames: int = 12,
        context_overlap: int = 4,
        context_schedule: str = "uniform_v2",
        context_stride: int = 1,
        motion_speed: float = 8.0,
        eta: float = 0.0,
        unet_kwargs: Optional[dict] = None,    # down_block_refer_embs / mid_block_refer_emb / vision_clip_emb / ip_adapter_scale
        controlnet_fn: Optional[Callable] = None,  # (window frame list, latent_model_input, t, step index) -> (down_res, mid_res); see make_controlnet_fn
        callback: Optional[Callable] = None,
        guidance_scale_lst: Optional[Sequence[float]] = None,
        generator: Optional[torch.Generator] = None,   # eta > 0 / LCM / Euler churn: source of the per-step noise
        noise_type: str = "random",                    # or "video_fusion" (pipeline_controlnet.py:1690-1696)
        w_ind_noise: float = 0.5,
        cfg_split: bool = False,                       # pair the ranks: each rank of a pair runs ONE half of the CFG batch
        pose_guider_emb: Optional[torch.Tensor] = None,  # [2B, C0, n_vc + T, h, w], vision-condition frames first
    ) -> DenoiseOutput:
        if guidance_scale <= 1.0:
            # the reference's CFG-off branch feeds the wrong vis-cond tensor (pipeline_controlnet.py:1922-1926, Q14)
            raise NotImplementedError("parallel denoise is implemented for classifier-free guidance (guidance_scale > 1)")
        unet_kwargs = dict(unet_kwargs or {})
        dev = latents.device
        B, C, T, h, w = latents.shape
        n_vc = condition_latents.shape[2]
        if pose_guider_emb is not None:
            # the PoseGuider output (pipeline_controlnet.py:1774-1783, UNet :2066), on the frame axis of make_controlnet_fn's
            # controlnet_latents; every window gets its own frames (see DESIGN.md section 5)
            pg = pose_guider_emb
            if pg.dim() != 5 or pg.shape[0] != 2 * B or tuple(pg.shape[2:]) != (n_vc + T, h, w):
                raise ValueError(f"pose_guider_emb must be [2B, C0, n_vc + T, h, w] = [{2 * B}, C0, {n_vc + T}, {h}, {w}], "
                                 f"got {tuple(pg.shape)}")
        sch = self.scheduler
        sch.set_timesteps(num_inference_steps, device="cpu")
        contexts = [c[0] for c in prepare_global_context(context_schedule, num_inference_steps, T, context_frames,
                                                         context_stride, context_overlap, 1)]
        # CFG split (SURVEY.md 8e, last row): the unconditional and the text half of the CFG batch never interact inside the
        # UNet (Q3: the only cross-half code is dead), so ranks 2p and 2p+1 can share the windows of pair p, each running a
        # B-row forward and filling only its half of the eps accumulator. The halves are disjoint, so the SAME single
        # all-reduce(SUM) per step that merges the windows also merges the halves -- no extra collective. This lets a video
        # with fewer windows than GPUs (config 2: one window) use twice the GPUs, and halves the critical path when the
        # window count is not a multiple of the GPU count (config 4: 11 windows on 8 GPUs -> 3 half-cost forwards, not 2).
        if cfg_split:
            if self.world % 2:
                raise ValueError("cfg_split needs an even number of ranks")
            per_rank = assign_windows([len(c) for c in contexts], self.world // 2)
            mine = per_rank[self.rank // 2]
            half = self.rank % 2
            rows = slice(half * B, (half + 1) * B)
            for k, v in list(unet_kwargs.items()):               # per-batch conditioning: keep this half's rows
                if torch.is_tensor(v) and v.dim() > 0 and v.shape[0] == 2 * B:
                    unet_kwargs[k] = v[rows].contiguous()
                elif isinstance(v, (list, tuple)) and v and torch.is_tensor(v[0]) and v[0].shape[0] == 2 * B:
                    unet_kwargs[k] = [x[rows].contiguous() for x in v]
        else:
            per_rank = assign_windows([len(c) for c in contexts], self.world)
            mine = per_rank[self.rank]
        # A closed-loop `uniform` window with context_stride >= 2 can name a frame twice (e % num_frames, context.py:46).
        # The reference's `noise_pred[:, :, c] = noise_pred[:, :, c] + noise_pred_c; counter[:, :, c] += 1` (:2076-2077) is
        # an indexed assignment: for a repeated index the LAST occurrence wins and the counter grows by one. The
        # accumulate kernel adds every listed frame exactly once, so duplicates are resolved here, on the host.
        counter = torch.zeros(T, dtype=torch.float32)
        keep_pos: List[Optional[torch.Tensor]] = []
        uniq_frames: List[List[int]] = []
        for c in contexts:
            last = {}
            for k, fidx in enumerate(c):
                last[fidx] = k
            pos = sorted(last.values())
            uniq_frames.append([c[k] for k in pos])
            keep_pos.append(None if len(pos) == len(c) else torch.tensor(pos, dtype=torch.long, device=dev) + n_vc)
            for fidx in last:
                counter[fidx] += 1                                                  # :2077, static per call
        counter = counter.to(dev)
        frame_idx_dev = [torch.tensor(c, dtype=torch.int32, device=dev) for c in uniq_frames]
        frame_idx_long = [torch.tensor(c, dtype=torch.long, device=dev) for c in contexts]
        cond2 = torch.cat([condition_latents] * 2).to(latents.dtype)                # :1921-1926
        vis_idx = torch.arange(n_vc)
        eps_sum = torch.zeros((2 * B, C, T, h, w), dtype=torch.float32, device=dev)
        latents = latents.contiguous()
        is_ddim = isinstance(sch, DDIMScheduler)
        is_multistep = not is_ddim and hasattr(sch, "multistep_plan")
        if is_multistep:
            # m1 / m2 of the multistep kernel (DPM-Solver's `model_outputs`). Every rank applies the same plan and kernel to
            # the same all-reduced eps, so the histories stay replicated bit-exactly, like the latents.
            history = [torch.zeros((B, C, T, h, w), dtype=torch.float32, device=dev) for _ in range(2)]
        if is_ddim:
            pred = _PRED[sch.config.prediction_type]
            clip = sch.config.clip_sample_range if sch.config.clip_sample else 0.0

        def step_noise():
            """Per-step noise [B,C,T,h,w] fp32, identical on every rank (drawn on rank 0, broadcast): scheduling_ddim.py
            :266-295, scheduling_euler_discrete.py:116-127, scheduling_lcm.py:291-300, scheduling_euler_ancestral_discrete.py
            :303-314, scheduling_ddpm.py:220-241."""
            nz = _variance_noise(latents, generator, noise_type, w_ind_noise).float().contiguous()
            if self.world > 1:
                self._dist.broadcast(nz, src=0, group=self.pg)
            return nz

        for i, t in enumerate(sch.timesteps.tolist()):
            eps_sum.zero_()                                                         # :1870-1876
            for wi in mine:                                                         # :1900 (this rank's windows)
                c = contexts[wi]
                lat_c = latents.index_select(2, frame_idx_long[wi])                 # :1902
                if not is_ddim:
                    scale = sch.model_input_scale(t)                                # scale_model_input, :1911
                    if scale != 1.0:
                        lat_c = lat_c * scale
                sub_idx = torch.arange(len(c)) + n_vc                               # :1914-1920
                # batch_concat_two_tensor_with_index: vis-cond frames first, then the window, duplicated for CFG
                if cfg_split:
                    model_in = torch.cat([cond2[:B], lat_c], dim=2)                 # this rank's half of the CFG batch
                else:
                    model_in = torch.cat([cond2, torch.cat([lat_c] * 2)], dim=2)    # :1908-1946
                kw = dict(unet_kwargs)
                if pose_guider_emb is not None:
                    # vision-condition frames + this window's frames (duplicates included), (b t) c h w like model_in
                    ctx = torch.tensor(list(range(n_vc)) + [ci + n_vc for ci in c], dtype=torch.long,
                                       device=pose_guider_emb.device)
                    pe = pose_guider_emb.index_select(2, ctx)
                    if cfg_split:
                        pe = pe[rows]
                    nb, c0, tc = pe.shape[:3]
                    kw["pose_guider_emb"] = pe.permute(0, 2, 1, 3, 4).reshape(nb * tc, c0, h, w)
                if controlnet_fn is not None:
                    if cfg_split:      # the callback gets this rank's half of the CFG batch and which rows it is
                        down_res, mid_res = controlnet_fn(c, model_in, t, i, rows)
                    else:
                        down_res, mid_res = controlnet_fn(c, model_in, t, i)        # :2022-2038
                    kw["down_block_additional_residuals"] = down_res
                    kw["mid_block_additional_residual"] = mid_res
                if self._shares_cfg_prefix:
                    kw["cfg_shared_sample"] = not cfg_split    # cond2 and [lat_c] * 2: both halves of model_in are equal
                eps = self.unet(model_in, t, prompt_embeds[rows] if cfg_split else prompt_embeds, sample_index=sub_idx,
                                vision_conditon_frames_sample_index=vis_idx, sample_frame_rate=motion_speed,
                                do_classifier_free_guidance=True, return_dict=False, **kw)[0]   # :2045-2067
                acc = eps_sum[rows] if cfg_split else eps_sum                            # contiguous leading-dim slice
                if keep_pos[wi] is None:
                    self.ops.accumulate_window(acc, eps, n_vc, frame_idx_dev[wi])        # :2068-2078
                else:                                                                    # window with repeated frames
                    self.ops.accumulate_window(acc, eps.index_select(2, keep_pos[wi]).contiguous(), 0, frame_idx_dev[wi])
            if self.world > 1:
                self._dist.all_reduce(eps_sum, op=self._dist.ReduceOp.SUM, group=self.pg)
            g = guidance_scale_lst[i] if guidance_scale_lst is not None else guidance_scale
            if is_ddim:
                a_t, a_p, std = sch.step_scalars(t, eta)
                if std > 0.0:
                    latents = self.ops.fuse_cfg_ddim(eps_sum, counter, latents, float(g), a_t, a_p, pred, clip, std_dev=std,
                                                     noise=step_noise())                 # eta > 0: scheduling_ddim.py:266-295
                else:
                    latents = self.ops.fuse_cfg_ddim(eps_sum, counter, latents, float(g), a_t, a_p, pred, clip)  # :2079,2101-2117
            elif is_multistep:
                p = sch.multistep_plan(t)                                           # DPM-Solver / Euler ancestral / DDPM
                latents = multistep_update(self.ops, p, eps_sum, counter, latents, g, history,
                                           step_noise() if p.needs_noise else None)
            else:
                a = sch.affine_step(t)                                              # Euler / LCM: scalars on the host
                latents = self.ops.fuse_cfg_affine(eps_sum, counter, latents, float(g), a.c_x, a.c_e, a.c_n,
                                                   step_noise() if a.c_n != 0.0 else None)
            if callback is not None:
                callback(i, t, latents)
        return DenoiseOutput(latents=latents, windows=contexts, windows_per_rank=per_rank)



def controlnet_keep_schedule(num_inference_steps: int, control_guidance_start: Union[float, Sequence[float]] = 0.0,
                             control_guidance_end: Union[float, Sequence[float]] = 1.0,
                             num_controlnets: Optional[int] = None) -> list:
    """`controlnet_keep` of the reference: per step, 1.0 while a net's guidance window [start, end] covers the step and 0.0
    outside it (musev/pipelines/pipeline_controlnet.py:1700-1711), after the start / end lists are aligned
    (:1060-1083). num_controlnets: None for one `ControlNetModel` (a float per step), N for a Multi-ControlNet of N nets
    (a list of N per step). The checks and their wording are diffusers' check_inputs
    (pipelines/controlnet/pipeline_controlnet.py:601-615)."""
    start, end = control_guidance_start, control_guidance_end
    if not isinstance(start, (list, tuple)) and isinstance(end, (list, tuple)):          # :1060-1083
        start = len(end) * [start]
    elif not isinstance(end, (list, tuple)) and isinstance(start, (list, tuple)):
        end = len(start) * [end]
    elif not isinstance(start, (list, tuple)) and not isinstance(end, (list, tuple)):
        mult = 1 if num_controlnets is None else num_controlnets
        start, end = mult * [start], mult * [end]
    if len(start) != len(end):
        raise ValueError(f"`control_guidance_start` has {len(start)} elements, but `control_guidance_end` has {len(end)} "
                         "elements. Make sure to provide the same number of elements to each list.")
    n = 1 if num_controlnets is None else num_controlnets
    if len(start) != n:
        raise ValueError(f"`control_guidance_start`: {list(start)} has {len(start)} elements but there are {n} controlnets "
                         f"available. Make sure to provide {n}.")
    for s, e in zip(start, end):
        if s >= e:
            raise ValueError(f"control guidance start: {s} cannot be larger or equal to control guidance end: {e}.")
        if s < 0.0:
            raise ValueError(f"control guidance start: {s} can't be smaller than 0.")
        if e > 1.0:
            raise ValueError(f"control guidance end: {e} can't be larger than 1.0.")
    keep = []
    for i in range(num_inference_steps):                                                  # :1700-1711
        keeps = [1.0 - float(i / num_inference_steps < s or (i + 1) / num_inference_steps > e) for s, e in zip(start, end)]
        keep.append(keeps[0] if num_controlnets is None else keeps)
    return keep


def make_controlnet_fn(controlnet, controlnet_latents, prompt_embeds: torch.Tensor, n_vision_cond: int,
                       controlnet_conditioning_scale: Union[float, Sequence[float]] = 1.0, guess_mode: bool = False,
                       controlnet_keep: Optional[Sequence] = None) -> Callable:
    """The per-window-step ControlNet call of the reference loop as a `controlnet_fn` for `ParallelDenoiser`
    (musev/pipelines/pipeline_controlnet.py:1992-2038 window slicing, :1202-1291 `get_controlnet_emb`).

    controlnet_latents: [2B, C0, n_vc + T, h, w] -- the condition embedding of every frame, vision-condition frame(s) first,
    already duplicated for CFG ([B, ...] in guess mode); computed once per call (`controlnet_cond_latents`, :1258).
    Returns residuals shaped `(b t) c h w` with b = 2B, which is what `UNet3DConditionModel.forward` takes.

    Several ControlNets (a `MultiControlNetModel` or a list of nets, the reference's multi-net branch): controlnet_latents
    is a list with one such tensor per net, controlnet_conditioning_scale a float for every net (:1548-1553) or a list,
    and controlnet_keep[i] a float or a list per net (`controlnet_keep_schedule`). Each net's slice of its own latents
    is taken as for one net; the nets' maps are summed on the device. A net whose keep is 0 in a step is not run (the
    reference runs it and scales its maps by 0, which only differs where a map is not finite); when every net is off the
    function returns (None, None) and the UNet adds no residuals."""
    from .controlnet import MultiControlNetModel
    multi = isinstance(controlnet, (MultiControlNetModel, list, tuple))
    if multi:
        mc = controlnet if isinstance(controlnet, MultiControlNetModel) else MultiControlNetModel(controlnet)
        nets = mc.nets
        all_lat = mc.check_list("controlnet_latents", controlnet_latents)
        scales = mc.check_list("controlnet_conditioning_scale", controlnet_conditioning_scale) \
            if isinstance(controlnet_conditioning_scale, (list, tuple)) else [controlnet_conditioning_scale] * len(nets)
    else:
        nets, all_lat, scales = [controlnet], [controlnet_latents], [controlnet_conditioning_scale]
    vis = list(range(n_vision_cond))

    def fn(c, latent_model_input, t, i=0, rows=None):
        """rows: with `ParallelDenoiser(cfg_split=True)` the slice of the CFG batch this rank runs (`latent_model_input` then
        holds only those rows); the prompt and condition latents are sliced to match."""
        ctx = vis + [ci + n_vision_cond for ci in c]                                       # :1997-2000
        b2 = latent_model_input.shape[0]
        if rows is not None:
            if guess_mode:
                raise NotImplementedError("guess_mode runs the ControlNet on the conditional half only; not combined with cfg_split")
            x, enc = latent_model_input, prompt_embeds[rows]
        elif guess_mode:                                                                   # :1219-1225: cond half only
            x = latent_model_input[b2 // 2:]
            enc = prompt_embeds[prompt_embeds.shape[0] // 2:]
        else:
            x, enc = latent_model_input, prompt_embeds
        nb, ch, tc, hh, ww = x.shape
        x2 = x.permute(0, 2, 1, 3, 4).reshape(nb * tc, ch, hh, ww)                           # b c t h w -> (b t) c h w
        enc2 = enc.repeat_interleave(tc, dim=0)                                            # align_repeat_tensor_single_dim

        def net_latents(lat):
            idx = torch.tensor(ctx, dtype=torch.long, device=lat.device)
            lat_c = lat.index_select(2, idx)                                               # :2008-2010
            if rows is not None:
                lat_c = lat_c[rows]
            return lat_c.permute(0, 2, 1, 3, 4).reshape(nb * tc, lat_c.shape[1], hh, ww)

        if not multi:
            keep = 1.0 if controlnet_keep is None else float(controlnet_keep[i])
            down, mid = controlnet(x2, t, enc2, controlnet_cond_latents=net_latents(controlnet_latents),
                                   conditioning_scale=controlnet_conditioning_scale * keep, guess_mode=guess_mode,
                                   return_dict=False)
        else:
            keep = [1.0] * len(nets) if controlnet_keep is None else controlnet_keep[i]
            if not isinstance(keep, (list, tuple)):
                keep = [float(keep)] * len(nets)
            if len(keep) != len(nets):
                raise ValueError(f"controlnet_keep[{i}] has {len(keep)} entries for {len(nets)} ControlNets")
            res = None
            for net, lat, scale, kp in zip(nets, all_lat, scales, keep):                    # :1229-1235, cond_scale per net
                if float(kp) == 0.0:
                    continue
                res = net(x2, t, enc2, controlnet_cond_latents=net_latents(lat), conditioning_scale=scale * float(kp),
                          guess_mode=guess_mode, return_dict=False, accumulate_into=res)
            if res is None:
                return None, None
            down, mid = res
        if guess_mode:                                                                     # :1275-1286: zeros for uncond
            def pad(r):
                r5 = r.view(nb, tc, *r.shape[1:])
                return torch.cat([torch.zeros_like(r5), r5]).view(2 * nb * tc, *r.shape[1:])
            down, mid = [pad(d) for d in down], pad(mid)
        return list(down), mid
    return fn
