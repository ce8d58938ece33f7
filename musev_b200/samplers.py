"""Host mirrors of the other samplers of SURVEY.md 8(f)-4 on the fused step kernels.

  * `EulerDiscreteScheduler`  musev/schedulers/scheduling_euler_discrete.py:21-293 over diffusers
                              schedulers/scheduling_euler_discrete.py:135-463 -- the predictor's DEFAULT sampler
                              (musev/pipelines/pipeline_controlnet_predictor.py:258-261).
  * `LCMScheduler`            musev/schedulers/scheduling_lcm.py:44-312 over diffusers schedulers/scheduling_lcm.py:196-547.
Both keep the reference's constructor / `set_timesteps` / `timesteps` / `sigmas` / `init_noise_sigma` /
`scale_model_input` / `step` / `add_noise` surface (the pipeline probes `inspect.signature(step)` for `generator` /
`noise_type`, pipeline_controlnet.py:1690-1696). Every step of these samplers is affine in (sample, model_output, noise),
so `step` and the fused loop (`ParallelDenoiser`) run ONE kernel (`mvb_fuse_cfg_affine`) with host-computed scalars
(`affine_step`). Integer / float bookkeeping restated from the reference; the tensor arithmetic is on the GPU only.

The multistep samplers run on `mvb_fuse_cfg_multistep` with host-computed scalars (`multistep_plan`, see below):
  * `DPMSolverMultistepScheduler`      musev/schedulers/scheduling_dpmsolver_multistep.py:66-815 (DPM-Solver / DPM-Solver++,
                                       orders 1-3, midpoint / heun, Karras sigmas on by default in this copy)
  * `EulerAncestralDiscreteScheduler`  musev/schedulers/scheduling_euler_ancestral_discrete.py:90-356
  * `DDPMScheduler`                    musev/schedulers/scheduling_ddpm.py:42-262 (clip_sample through the kernel's clamp)
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from types import SimpleNamespace
from typing import List, Optional, Tuple, Union

import numpy as np
import torch

from . import ops
from .scheduler import _rescale_zero_terminal_snr, _variance_noise


def _betas(beta_schedule, beta_start, beta_end, n, trained_betas, cls):
    if trained_betas is not None:
        return torch.tensor(trained_betas, dtype=torch.float32)
    if beta_schedule == "linear":
        return torch.linspace(beta_start, beta_end, n, dtype=torch.float32)
    if beta_schedule == "scaled_linear":
        return torch.linspace(beta_start ** 0.5, beta_end ** 0.5, n, dtype=torch.float32) ** 2
    raise NotImplementedError(f"{beta_schedule} does is not implemented for {cls}")


@dataclass
class AffineStep:
    """x_prev = c_x x + c_e eps + c_n noise; aux (pred_original_sample / denoised) = a_x x + a_e eps."""
    c_x: float
    c_e: float
    c_n: float
    a_x: float
    a_e: float


@dataclass
class EulerDiscreteSchedulerOutput:
    prev_sample: torch.Tensor
    pred_original_sample: Optional[torch.Tensor] = None


@dataclass
class LCMSchedulerOutput:
    prev_sample: torch.Tensor
    denoised: Optional[torch.Tensor] = None


def _run_affine(a: AffineStep, model_output, sample, noise):
    if not sample.is_cuda:
        raise RuntimeError("musev_b200 samplers run on the GPU only")
    shape = sample.shape
    x = sample.contiguous()
    if x.dtype not in (torch.float16, torch.float32):
        x = x.float()
    x5 = x.view(shape[0], shape[1], 1, 1, -1) if x.dim() != 5 else x
    eps = model_output.contiguous().float().view(x5.shape)
    nz = None if noise is None else noise.to(sample.device).contiguous().float().view(x5.shape)
    aux = torch.empty(x5.shape, dtype=torch.float32, device=x.device)
    prev = ops.fuse_cfg_affine(eps, None, x5, 1.0, a.c_x, a.c_e, a.c_n, nz, a.a_x, a.a_e, aux, cfg=False)
    return prev.view(shape).to(sample.dtype), aux.view(shape).to(sample.dtype)


class EulerDiscreteScheduler:
    order = 1

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.0001, beta_end: float = 0.02,
                 beta_schedule: str = "linear", trained_betas=None, prediction_type: str = "epsilon",
                 interpolation_type: str = "linear", use_karras_sigmas: Optional[bool] = False,
                 timestep_spacing: str = "linspace", steps_offset: int = 0):
        self.config = SimpleNamespace(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                                      beta_schedule=beta_schedule, trained_betas=trained_betas, prediction_type=prediction_type,
                                      interpolation_type=interpolation_type, use_karras_sigmas=use_karras_sigmas,
                                      timestep_spacing=timestep_spacing, steps_offset=steps_offset)
        self.betas = _betas(beta_schedule, beta_start, beta_end, num_train_timesteps, trained_betas, self.__class__)
        self.alphas = 1.0 - self.betas
        self.alphas_cumprod = torch.cumprod(self.alphas, dim=0)
        sig = (((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5).numpy()
        self.sigmas = torch.from_numpy(np.concatenate([sig[::-1], [0.0]]).astype(np.float32))
        self.num_inference_steps = None
        self.timesteps = torch.from_numpy(np.linspace(0, num_train_timesteps - 1, num_train_timesteps, dtype=float)[::-1].copy())
        self.is_scale_input_called = False
        self.use_karras_sigmas = use_karras_sigmas
        self._step_index = None

    @property
    def init_noise_sigma(self):
        if self.config.timestep_spacing in ["linspace", "trailing"]:
            return self.sigmas.max()
        return (self.sigmas.max() ** 2 + 1) ** 0.5

    @property
    def step_index(self):
        return self._step_index

    def _init_step_index(self, timestep):
        t = float(timestep)
        cand = (self.timesteps == t).nonzero()
        if len(cand) == 0:
            raise ValueError(f"timestep {t} is not one of scheduler.timesteps")
        self._step_index = (cand[1] if len(cand) > 1 else cand[0]).item()

    def model_input_scale(self, timestep) -> float:
        """1 / sqrt(sigma^2 + 1) of `scale_model_input` as a host scalar."""
        if self._step_index is None:
            self._init_step_index(timestep)
        sigma = float(self.sigmas[self._step_index])
        self.is_scale_input_called = True
        return 1.0 / (sigma * sigma + 1.0) ** 0.5

    def scale_model_input(self, sample: torch.Tensor, timestep) -> torch.Tensor:
        return sample * self.model_input_scale(timestep)

    def set_timesteps(self, num_inference_steps: int, device=None):
        c = self.config
        self.num_inference_steps = num_inference_steps
        if c.timestep_spacing == "linspace":
            ts = np.linspace(0, c.num_train_timesteps - 1, num_inference_steps, dtype=np.float32)[::-1].copy()
        elif c.timestep_spacing == "leading":
            ratio = c.num_train_timesteps // num_inference_steps
            ts = (np.arange(0, num_inference_steps) * ratio).round()[::-1].copy().astype(np.float32)
            ts += c.steps_offset
        elif c.timestep_spacing == "trailing":
            ratio = c.num_train_timesteps / num_inference_steps
            ts = (np.arange(c.num_train_timesteps, 0, -ratio)).round().copy().astype(np.float32)
            ts -= 1
        else:
            raise ValueError(f"{c.timestep_spacing} is not supported. Please make sure to choose one of 'linspace', 'leading' or 'trailing'.")
        sig = (((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5).numpy()
        log_sig = np.log(sig)
        if c.interpolation_type == "linear":
            sig = np.interp(ts, np.arange(0, len(sig)), sig)
        elif c.interpolation_type == "log_linear":
            sig = torch.linspace(np.log(sig[-1]), np.log(sig[0]), num_inference_steps + 1).exp().numpy()
        else:
            raise ValueError(f"{c.interpolation_type} is not implemented. Please specify interpolation_type to either 'linear' or 'log_linear'")
        if self.use_karras_sigmas:
            smin, smax, rho = float(sig[-1]), float(sig[0]), 7.0
            ramp = np.linspace(0, 1, num_inference_steps)
            sig = (smax ** (1 / rho) + ramp * (smin ** (1 / rho) - smax ** (1 / rho))) ** rho
            ts = np.array([self._sigma_to_t(s, log_sig) for s in sig])
        self.sigmas = torch.from_numpy(np.concatenate([sig, [0.0]]).astype(np.float32))
        self.timesteps = torch.from_numpy(ts)
        self._step_index = None

    @staticmethod
    def _sigma_to_t(sigma, log_sigmas):
        log_sigma = np.log(np.maximum(sigma, 1e-10))
        dists = log_sigma - log_sigmas[:, np.newaxis]
        low_idx = np.cumsum((dists >= 0), axis=0).argmax(axis=0).clip(max=log_sigmas.shape[0] - 2)
        high_idx = low_idx + 1
        low, high = log_sigmas[low_idx], log_sigmas[high_idx]
        w = np.clip((low - log_sigma) / (low - high), 0, 1)
        return ((1 - w) * low_idx + w * high_idx).reshape(np.shape(sigma))

    def affine_step(self, timestep, s_churn: float = 0.0, s_tmin: float = 0.0, s_tmax: float = float("inf"),
                    s_noise: float = 1.0) -> AffineStep:
        """Scalars of `step` (scheduling_euler_discrete.py:107-166) at the current step index; advances the index."""
        if self._step_index is None:
            self._init_step_index(timestep)
        sigma = float(self.sigmas[self._step_index])
        gamma = min(s_churn / (len(self.sigmas) - 1), 2 ** 0.5 - 1) if s_tmin <= sigma <= s_tmax else 0.0
        sigma_hat = sigma * (gamma + 1)
        c_n = s_noise * (sigma_hat ** 2 - sigma ** 2) ** 0.5 if gamma > 0 else 0.0
        dt = float(self.sigmas[self._step_index + 1]) - sigma_hat
        pt = self.config.prediction_type
        # x0 = a_x x' + a_e e  (x' = x + c_n noise);  prev = x' + (x' - x0) / sigma_hat * dt
        if pt in ("original_sample", "sample"):
            a_x, a_e = 0.0, 1.0
        elif pt == "epsilon":
            a_x, a_e = 1.0, -sigma_hat
        elif pt == "v_prediction":
            a_x, a_e = 1.0 / (sigma ** 2 + 1), -sigma / (sigma ** 2 + 1) ** 0.5
        else:
            raise ValueError(f"prediction_type given as {pt} must be one of `epsilon`, or `v_prediction`")
        r = dt / sigma_hat
        c_x = 1.0 + r * (1.0 - a_x)
        c_e = -r * a_e
        self._step_index += 1
        # the churn noise enters through x': prev = c_x (x + c_n z) + c_e e, aux = a_x (x + c_n z) + a_e e; with the default
        # s_churn = 0 there is no noise. (aux ignores the churn term: it is only reported, never fed back.)
        return AffineStep(c_x, c_e, c_x * c_n, a_x, a_e)

    def step(self, model_output: torch.Tensor, timestep, sample: torch.Tensor, s_churn: float = 0.0, s_tmin: float = 0.0,
             s_tmax: float = float("inf"), s_noise: float = 1.0, generator=None, return_dict: bool = True,
             w_ind_noise: float = 0.5, noise_type: str = "random"):
        if isinstance(timestep, int) or isinstance(timestep, (torch.IntTensor, torch.LongTensor)):
            raise ValueError("Passing integer indices (e.g. from `enumerate(timesteps)`) as timesteps to"
                             " `EulerDiscreteScheduler.step()` is not supported. Make sure to pass"
                             " one of the `scheduler.timesteps` as a timestep.")
        a = self.affine_step(timestep, s_churn, s_tmin, s_tmax, s_noise)
        # the reference draws the noise on every step (scheduling_euler_discrete.py:116-127) even when gamma = 0, which
        # advances the generator; keep that side effect
        noise = _variance_noise(model_output, generator, noise_type, w_ind_noise)
        prev, x0 = _run_affine(a, model_output, sample, noise if a.c_n != 0.0 else None)
        if not return_dict:
            return (prev,)
        return EulerDiscreteSchedulerOutput(prev_sample=prev, pred_original_sample=x0)

    def add_noise(self, original_samples: torch.Tensor, noise: torch.Tensor, timesteps: torch.Tensor) -> torch.Tensor:
        sigmas = self.sigmas.to(device=original_samples.device, dtype=original_samples.dtype)
        sched_t = self.timesteps.to(original_samples.device)
        idx = [(sched_t == t).nonzero().item() for t in timesteps.to(original_samples.device)]
        sigma = sigmas[idx].flatten()
        while sigma.dim() < original_samples.dim():
            sigma = sigma.unsqueeze(-1)
        return original_samples + noise * sigma

    def __len__(self):
        return self.config.num_train_timesteps


class LCMScheduler:
    order = 1

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.00085, beta_end: float = 0.012,
                 beta_schedule: str = "scaled_linear", trained_betas=None, original_inference_steps: int = 50,
                 clip_sample: bool = False, clip_sample_range: float = 1.0, set_alpha_to_one: bool = True,
                 steps_offset: int = 0, prediction_type: str = "epsilon", thresholding: bool = False,
                 dynamic_thresholding_ratio: float = 0.995, sample_max_value: float = 1.0,
                 timestep_spacing: str = "leading", timestep_scaling: float = 10.0, rescale_betas_zero_snr: bool = False):
        if thresholding or clip_sample:
            raise NotImplementedError("musev_b200.LCMScheduler runs the affine fused step: clip_sample / thresholding are not supported")
        self.config = SimpleNamespace(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                                      beta_schedule=beta_schedule, trained_betas=trained_betas,
                                      original_inference_steps=original_inference_steps, clip_sample=clip_sample,
                                      clip_sample_range=clip_sample_range, set_alpha_to_one=set_alpha_to_one,
                                      steps_offset=steps_offset, prediction_type=prediction_type, thresholding=thresholding,
                                      dynamic_thresholding_ratio=dynamic_thresholding_ratio, sample_max_value=sample_max_value,
                                      timestep_spacing=timestep_spacing, timestep_scaling=timestep_scaling,
                                      rescale_betas_zero_snr=rescale_betas_zero_snr)
        self.betas = _betas(beta_schedule, beta_start, beta_end, num_train_timesteps, trained_betas, self.__class__)
        if rescale_betas_zero_snr:
            self.betas = _rescale_zero_terminal_snr(self.betas)
        self.alphas = 1.0 - self.betas
        self.alphas_cumprod = torch.cumprod(self.alphas, dim=0)
        self.final_alpha_cumprod = torch.tensor(1.0) if set_alpha_to_one else self.alphas_cumprod[0]
        self.init_noise_sigma = 1.0
        self.num_inference_steps = None
        self.timesteps = torch.from_numpy(np.arange(0, num_train_timesteps)[::-1].copy().astype(np.int64))
        self._step_index = None

    @property
    def step_index(self):
        return self._step_index

    def _init_step_index(self, timestep):
        cand = (self.timesteps == int(timestep)).nonzero()
        if len(cand) == 0:
            raise ValueError(f"timestep {int(timestep)} is not one of scheduler.timesteps")
        self._step_index = (cand[1] if len(cand) > 1 else cand[0]).item()

    def scale_model_input(self, sample: torch.Tensor, timestep=None) -> torch.Tensor:
        return sample

    def model_input_scale(self, timestep) -> float:
        return 1.0

    def set_timesteps(self, num_inference_steps: int, device=None, original_inference_steps: Optional[int] = None,
                      strength: float = 1.0):
        c = self.config
        if num_inference_steps > c.num_train_timesteps:
            raise ValueError(f"`num_inference_steps`: {num_inference_steps} cannot be larger than `self.config.train_timesteps`:"
                             f" {c.num_train_timesteps} as the unet model trained with this scheduler can only handle"
                             f" maximal {c.num_train_timesteps} timesteps.")
        self.num_inference_steps = num_inference_steps
        original_steps = original_inference_steps if original_inference_steps is not None else c.original_inference_steps
        if original_steps > c.num_train_timesteps:
            raise ValueError(f"`original_steps`: {original_steps} cannot be larger than `self.config.train_timesteps`:"
                             f" {c.num_train_timesteps}")
        if num_inference_steps > original_steps:
            raise ValueError(f"`num_inference_steps`: {num_inference_steps} cannot be larger than `original_inference_steps`:"
                             f" {original_steps}")
        k = c.num_train_timesteps // original_steps
        origin = np.asarray(list(range(1, int(original_steps * strength) + 1))) * k - 1
        if len(origin) // num_inference_steps < 1:
            raise ValueError(f"The combination of `original_steps x strength`: {original_steps} x {strength} is smaller than"
                             f" `num_inference_steps`: {num_inference_steps}.")
        origin = origin[::-1].copy()
        idx = np.floor(np.linspace(0, len(origin), num=num_inference_steps, endpoint=False)).astype(np.int64)
        self.timesteps = torch.from_numpy(origin[idx]).to(dtype=torch.long)
        self._step_index = None

    def get_scalings_for_boundary_condition_discrete(self, timestep) -> Tuple[float, float]:
        sigma_data = 0.5
        st = float(timestep) * self.config.timestep_scaling
        return sigma_data ** 2 / (st ** 2 + sigma_data ** 2), st / (st ** 2 + sigma_data ** 2) ** 0.5

    def affine_step(self, timestep) -> AffineStep:
        """Scalars of `step` (musev/schedulers/scheduling_lcm.py:232-305); advances the step index."""
        if self.num_inference_steps is None:
            raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after creating the scheduler")
        if self._step_index is None:
            self._init_step_index(timestep)
        t = int(timestep)
        nxt = self._step_index + 1
        prev_t = int(self.timesteps[nxt]) if nxt < len(self.timesteps) else t
        a_t = float(self.alphas_cumprod[t])
        a_p = float(self.alphas_cumprod[prev_t]) if prev_t >= 0 else float(self.final_alpha_cumprod)
        sa, sb = a_t ** 0.5, (1 - a_t) ** 0.5
        c_skip, c_out = self.get_scalings_for_boundary_condition_discrete(t)
        pt = self.config.prediction_type
        if pt == "epsilon":
            x0_x, x0_e = 1.0 / sa, -sb / sa
        elif pt == "sample":
            x0_x, x0_e = 0.0, 1.0
        elif pt == "v_prediction":
            x0_x, x0_e = sa, -sb
        else:
            raise ValueError(f"prediction_type given as {pt} must be one of `epsilon`, `sample` or `v_prediction` for `LCMScheduler`.")
        d_x, d_e = c_out * x0_x + c_skip, c_out * x0_e                       # denoised = d_x x + d_e e
        last = self._step_index == self.num_inference_steps - 1
        self._step_index += 1
        if last:
            return AffineStep(d_x, d_e, 0.0, d_x, d_e)
        return AffineStep(a_p ** 0.5 * d_x, a_p ** 0.5 * d_e, (1 - a_p) ** 0.5, d_x, d_e)

    def step(self, model_output: torch.Tensor, timestep, sample: torch.Tensor, generator=None, return_dict: bool = True):
        a = self.affine_step(timestep)
        noise = None
        if a.c_n != 0.0:
            noise = torch.randn(model_output.shape, generator=generator, device=model_output.device, dtype=model_output.dtype)
        prev, den = _run_affine(a, model_output, sample, noise)
        if not return_dict:
            return (prev, den)
        return LCMSchedulerOutput(prev_sample=prev, denoised=den)

    def add_noise(self, original_samples: torch.Tensor, noise: torch.Tensor, timesteps: torch.Tensor) -> torch.Tensor:
        a = self.alphas_cumprod.to(device=original_samples.device, dtype=original_samples.dtype)[timesteps.to(original_samples.device)]
        sa, sb = (a ** 0.5).flatten(), ((1 - a) ** 0.5).flatten()
        while sa.dim() < original_samples.dim():
            sa, sb = sa.unsqueeze(-1), sb.unsqueeze(-1)
        return sa * original_samples + sb * noise

    def __len__(self):
        return self.config.num_train_timesteps


# ------------------------------------------------------------------------------------------------ multistep samplers
# DPM-Solver multistep, Euler ancestral and DDPM are not affine in (x, eps): DPM-Solver's update reads the converted model
# outputs of earlier steps and DDPM clamps x0. They run on `mvb_fuse_cfg_multistep`:
#   m0 = clamp(a_x x + a_e eps, +-clip);  x_prev = c_x x + c0 m0 + c1 m1 + c2 m2 + c_n noise
# with m1 / m2 the m0 of the previous one / two steps. Each mirror's `multistep_plan(t)` gives those scalars and advances
# the host bookkeeping exactly as the reference `step` does; the scheduler (standalone `step`) or `ParallelDenoiser` owns
# the two fp32 history buffers and rotates them with `rotate_history`.

@dataclass
class MultistepPlan:
    a_x: float
    a_e: float
    clip: float
    c_x: float
    c0: float
    c1: float = 0.0
    c2: float = 0.0
    c_n: float = 0.0
    needs_noise: bool = False      # the reference draws noise on this step (even when c_n is 0, it advances the generator)


@dataclass
class DPMSolverMultistepSchedulerOutput:
    prev_sample: torch.Tensor

    def __getitem__(self, i):
        return (self.prev_sample,)[i]


@dataclass
class EulerAncestralDiscreteSchedulerOutput:
    prev_sample: torch.Tensor
    pred_original_sample: Optional[torch.Tensor] = None

    def __getitem__(self, i):
        return (self.prev_sample, self.pred_original_sample)[i]


@dataclass
class DDPMSchedulerOutput:
    prev_sample: torch.Tensor
    pred_original_sample: Optional[torch.Tensor] = None

    def __getitem__(self, i):
        return (self.prev_sample, self.pred_original_sample)[i]


def multistep_update(device_ops, p: MultistepPlan, eps_sum, counter, latents, guidance, history: List[torch.Tensor],
                     noise=None, cfg=True):
    """One `fuse_cfg_multistep` launch for plan `p`. history = [m1, m2] (fp32, shaped like latents); the new m0 is written
    over m2 (the kernel reads m2 first) and the list is rotated in place, so that afterwards history[0] is this step's m0."""
    m1 = history[0] if p.c1 != 0.0 else None
    m2 = history[1] if p.c2 != 0.0 else None
    out = device_ops.fuse_cfg_multistep(eps_sum, counter, latents, float(guidance), p.a_x, p.a_e, p.clip, p.c_x, p.c0,
                                        p.c1, p.c2, p.c_n, m1, m2, noise if p.c_n != 0.0 else None, m0_out=history[1], cfg=cfg)
    history[0], history[1] = history[1], history[0]
    return out


class _MultistepMirror:
    """`step` on the GPU for the three multistep mirrors: one kernel launch with cfg = 0 and the scheduler's own history."""

    def _reset_history(self):
        self._history: Optional[List[torch.Tensor]] = None

    def _step_tensors(self, p: MultistepPlan, model_output, sample, noise):
        if not sample.is_cuda:
            raise RuntimeError("musev_b200 samplers run on the GPU only")
        shape = sample.shape
        x = sample.contiguous()
        if x.dtype not in (torch.float16, torch.float32):
            x = x.float()
        x5 = x.view(shape[0], shape[1], 1, 1, -1) if x.dim() != 5 else x
        if self._history is None or self._history[0].shape != x5.shape or self._history[0].device != x5.device:
            # allocated lazily to the sample shape; zeros, so a history read before it is written is harmless
            self._history = [torch.zeros(x5.shape, dtype=torch.float32, device=x5.device) for _ in range(2)]
        eps = model_output.contiguous().float().view(x5.shape)
        nz = None if noise is None else noise.to(sample.device).contiguous().float().view(x5.shape)
        prev = multistep_update(ops, p, eps, None, x5, 1.0, self._history, nz, cfg=False)
        return prev.view(shape).to(sample.dtype), self._history[0].view(shape)


def _betas_cos(beta_schedule, beta_start, beta_end, n, trained_betas, cls):
    if trained_betas is None and beta_schedule == "squaredcos_cap_v2":
        # Glide cosine schedule (betas_for_alpha_bar, scheduling_dpmsolver_multistep.py:34-63)
        def alpha_bar(t):
            return math.cos((t + 0.008) / 1.008 * math.pi / 2) ** 2
        return torch.tensor([min(1 - alpha_bar((i + 1) / n) / alpha_bar(i / n), 0.999) for i in range(n)],
                            dtype=torch.float32)
    return _betas(beta_schedule, beta_start, beta_end, n, trained_betas, cls)


def _as_index(timestep):
    return timestep.item() if torch.is_tensor(timestep) else timestep


class DPMSolverMultistepScheduler(_MultistepMirror):
    """musev/schedulers/scheduling_dpmsolver_multistep.py:66-815 (the musev copy: `use_karras_sigmas` defaults to True,
    the last step goes to timestep 0, `step` has `generator` / `w_ind_noise` and no `noise_type` / `eta`)."""
    order = 1

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.0001, beta_end: float = 0.02,
                 beta_schedule: str = "linear", trained_betas=None, solver_order: int = 2, prediction_type: str = "epsilon",
                 thresholding: bool = False, dynamic_thresholding_ratio: float = 0.995, sample_max_value: float = 1.0,
                 algorithm_type: str = "dpmsolver++", solver_type: str = "midpoint", lower_order_final: bool = True,
                 use_karras_sigmas: Optional[bool] = True, lambda_min_clipped: float = -float("inf"),
                 variance_type: Optional[str] = None):
        if thresholding:
            raise NotImplementedError("dynamic thresholding is unsuitable for latent diffusion and is not supported")
        if algorithm_type == "deis":
            algorithm_type = "dpmsolver++"
        if algorithm_type in ("sde-dpmsolver", "sde-dpmsolver++"):
            raise NotImplementedError(
                f"algorithm_type {algorithm_type!r} cannot run in the reference either: its step calls `.to(device)` with no "
                "`device` in scope (musev/schedulers/scheduling_dpmsolver_multistep.py:728-730) and raises NameError")
        if algorithm_type not in ("dpmsolver", "dpmsolver++"):
            raise NotImplementedError(f"{algorithm_type} does is not implemented for {self.__class__}")
        if solver_type in ("logrho", "bh1", "bh2"):
            solver_type = "midpoint"
        if solver_type not in ("midpoint", "heun"):
            raise NotImplementedError(f"{solver_type} does is not implemented for {self.__class__}")
        if solver_order not in (1, 2, 3):
            raise ValueError(f"solver_order must be 1, 2 or 3, got {solver_order}")
        if prediction_type not in ("epsilon", "sample", "v_prediction"):
            raise ValueError(f"prediction_type given as {prediction_type} must be one of `epsilon`, `sample`, or"
                             " `v_prediction` for the DPMSolverMultistepScheduler.")
        self.config = SimpleNamespace(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                                      beta_schedule=beta_schedule, trained_betas=trained_betas, solver_order=solver_order,
                                      prediction_type=prediction_type, thresholding=thresholding,
                                      dynamic_thresholding_ratio=dynamic_thresholding_ratio, sample_max_value=sample_max_value,
                                      algorithm_type=algorithm_type, solver_type=solver_type,
                                      lower_order_final=lower_order_final, use_karras_sigmas=use_karras_sigmas,
                                      lambda_min_clipped=lambda_min_clipped, variance_type=variance_type)
        self.betas = _betas_cos(beta_schedule, beta_start, beta_end, num_train_timesteps, trained_betas, self.__class__)
        self.alphas = 1.0 - self.betas
        self.alphas_cumprod = torch.cumprod(self.alphas, dim=0)
        self.alpha_t = torch.sqrt(self.alphas_cumprod)
        self.sigma_t = torch.sqrt(1 - self.alphas_cumprod)
        self.lambda_t = torch.log(self.alpha_t) - torch.log(self.sigma_t)
        self.init_noise_sigma = 1.0
        self.num_inference_steps = None
        self.timesteps = torch.from_numpy(np.linspace(0, num_train_timesteps - 1, num_train_timesteps,
                                                      dtype=np.float32)[::-1].copy())
        self.lower_order_nums = 0
        self.use_karras_sigmas = use_karras_sigmas
        self._reset_history()

    def set_timesteps(self, num_inference_steps: int = None, device: Union[str, torch.device] = None):
        c = self.config
        clipped_idx = torch.searchsorted(torch.flip(self.lambda_t, [0]), c.lambda_min_clipped)
        ts = (np.linspace(0, c.num_train_timesteps - 1 - int(clipped_idx), num_inference_steps + 1)
              .round()[::-1][:-1].copy().astype(np.int64))
        if self.use_karras_sigmas:
            sig = (((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5).numpy()
            log_sig = np.log(sig)
            smin, smax, rho = sig[-1].item(), sig[0].item(), 7.0
            ramp = np.linspace(0, 1, num_inference_steps)
            sig = (smax ** (1 / rho) + ramp * (smin ** (1 / rho) - smax ** (1 / rho))) ** rho
            ts = np.array([self._sigma_to_t(s, log_sig) for s in sig]).round()
            ts = np.flip(ts).copy().astype(np.int64)
        _, uniq = np.unique(ts, return_index=True)          # Karras timesteps can repeat (:276-279)
        ts = ts[np.sort(uniq)]
        self.timesteps = torch.from_numpy(ts).to(device)
        self.num_inference_steps = len(ts)
        self.lower_order_nums = 0                            # with `model_outputs = [None] * order` (:285-288)
        self._reset_history()

    @staticmethod
    def _sigma_to_t(sigma, log_sigmas):
        log_sigma = np.log(sigma)
        dists = log_sigma - log_sigmas[:, np.newaxis]
        low_idx = np.cumsum((dists >= 0), axis=0).argmax(axis=0).clip(max=log_sigmas.shape[0] - 2)
        high_idx = low_idx + 1
        low, high = log_sigmas[low_idx], log_sigmas[high_idx]
        w = np.clip((low - log_sigma) / (low - high), 0, 1)
        return ((1 - w) * low_idx + w * high_idx).reshape(sigma.shape)

    def scale_model_input(self, sample: torch.Tensor, *args, **kwargs) -> torch.Tensor:
        return sample

    def model_input_scale(self, timestep) -> float:
        return 1.0

    def _convert_coefs(self, t):
        """m0 = a_x x + a_e e: `convert_model_output` (:396-446); fp32 0-d tensors as the reference computes them."""
        c = self.config
        al, sg = self.alpha_t[t], self.sigma_t[t]
        one, zero = torch.tensor(1.0), torch.tensor(0.0)
        if c.algorithm_type == "dpmsolver++":                # x0 prediction
            return {"epsilon": (1.0 / al, -sg / al), "sample": (zero, one), "v_prediction": (al, -sg)}[c.prediction_type]
        return {"epsilon": (zero, one), "sample": (1.0 / sg, -al / sg), "v_prediction": (sg, al)}[c.prediction_type]

    def multistep_plan(self, timestep) -> MultistepPlan:
        """Scalars of `step` (:655-769) for `timestep`; advances `lower_order_nums` like the reference."""
        if self.num_inference_steps is None:
            raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after creating the scheduler")
        c = self.config
        ts = self.timesteps.cpu()
        found = (ts == _as_index(timestep)).nonzero()
        idx = len(ts) - 1 if len(found) == 0 else found.item()
        last = len(ts) - 1
        t = int(_as_index(timestep))
        prev_t = 0 if idx == last else int(ts[idx + 1])
        short = c.lower_order_final and len(ts) < 15
        lower_final, lower_second = idx == last and short, idx == last - 1 and short
        a_x, a_e = self._convert_coefs(t)
        if c.solver_order == 1 or self.lower_order_nums < 1 or lower_final:
            order = 1
        elif c.solver_order == 2 or self.lower_order_nums < 2 or lower_second:
            order = 2
        else:
            order = 3
        lam, alpha, sigma = self.lambda_t, self.alpha_t, self.sigma_t
        s0 = t
        h = lam[prev_t] - lam[s0]
        pp = c.algorithm_type == "dpmsolver++"
        if pp:
            c_x = sigma[prev_t] / sigma[s0]
            u0 = -(alpha[prev_t] * (torch.exp(-h) - 1.0))
        else:
            c_x = alpha[prev_t] / alpha[s0]
            u0 = -(sigma[prev_t] * (torch.exp(h) - 1.0))
        zero = torch.tensor(0.0)
        # x_prev = c_x x + u0 D0 + u1 D1 + u2 D2, each D a combination of (m0, m1, m2)
        D0 = (torch.tensor(1.0), zero, zero)
        D1, D2, u1, u2 = (zero, zero, zero), (zero, zero, zero), zero, zero
        if order == 2:                                                        # :499-593
            s1 = int(ts[idx - 1])
            r0 = (lam[s0] - lam[s1]) / h
            D1 = (1.0 / r0, -1.0 / r0, zero)
            if c.solver_type == "midpoint":
                u1 = 0.5 * u0
            elif pp:
                u1 = alpha[prev_t] * ((torch.exp(-h) - 1.0) / h + 1.0)
            else:
                u1 = -(sigma[prev_t] * ((torch.exp(h) - 1.0) / h - 1.0))
        elif order == 3:                                                      # :595-653
            s1, s2 = int(ts[idx - 1]), int(ts[idx - 2])
            r0, r1 = (lam[s0] - lam[s1]) / h, (lam[s1] - lam[s2]) / h
            d10 = (1.0 / r0, -1.0 / r0, zero)                                 # D1_0 = (m0 - m1) / r0
            d11 = (zero, 1.0 / r1, -1.0 / r1)                                 # D1_1 = (m1 - m2) / r1
            k, q = r0 / (r0 + r1), 1.0 / (r0 + r1)
            D1 = tuple(a + k * (a - b) for a, b in zip(d10, d11))
            D2 = tuple(q * (a - b) for a, b in zip(d10, d11))
            if pp:
                u1 = alpha[prev_t] * ((torch.exp(-h) - 1.0) / h + 1.0)
                u2 = -(alpha[prev_t] * ((torch.exp(-h) - 1.0 + h) / h ** 2 - 0.5))
            else:
                u1 = -(sigma[prev_t] * ((torch.exp(h) - 1.0) / h - 1.0))
                u2 = -(sigma[prev_t] * ((torch.exp(h) - 1.0 - h) / h ** 2 - 0.5))
        coef = [u0 * D0[j] + u1 * D1[j] + u2 * D2[j] for j in range(3)]
        if self.lower_order_nums < c.solver_order:
            self.lower_order_nums += 1
        return MultistepPlan(float(a_x), float(a_e), 0.0, float(c_x), float(coef[0]), float(coef[1]), float(coef[2]))

    def step(self, model_output: torch.Tensor, timestep: int, sample: torch.Tensor, generator=None, return_dict: bool = True,
             w_ind_noise: float = 0.5):
        p = self.multistep_plan(timestep)
        prev, _ = self._step_tensors(p, model_output, sample, None)
        if not return_dict:
            return (prev,)
        return DPMSolverMultistepSchedulerOutput(prev_sample=prev)

    def add_noise(self, original_samples: torch.Tensor, noise: torch.Tensor, timesteps: torch.Tensor) -> torch.Tensor:
        a = self.alphas_cumprod.to(device=original_samples.device, dtype=original_samples.dtype)[timesteps.to(original_samples.device)]
        sa, sb = (a ** 0.5).flatten(), ((1 - a) ** 0.5).flatten()
        while sa.dim() < original_samples.dim():
            sa, sb = sa.unsqueeze(-1), sb.unsqueeze(-1)
        return sa * original_samples + sb * noise

    def __len__(self):
        return self.config.num_train_timesteps


class EulerAncestralDiscreteScheduler(_MultistepMirror):
    """musev/schedulers/scheduling_euler_ancestral_discrete.py:90-356."""
    order = 1

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.0001, beta_end: float = 0.02,
                 beta_schedule: str = "linear", trained_betas=None, prediction_type: str = "epsilon"):
        self.config = SimpleNamespace(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                                      beta_schedule=beta_schedule, trained_betas=trained_betas, prediction_type=prediction_type)
        self.betas = _betas_cos(beta_schedule, beta_start, beta_end, num_train_timesteps, trained_betas, self.__class__)
        self.alphas = 1.0 - self.betas
        self.alphas_cumprod = torch.cumprod(self.alphas, dim=0)
        sig = (((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5).numpy()
        self.sigmas = torch.from_numpy(np.concatenate([sig[::-1], [0.0]]).astype(np.float32))
        self.init_noise_sigma = self.sigmas.max()
        self.num_inference_steps = None
        self.timesteps = torch.from_numpy(np.linspace(0, num_train_timesteps - 1, num_train_timesteps, dtype=float)[::-1].copy())
        self.is_scale_input_called = False
        self._reset_history()

    def _index(self, timestep) -> int:
        return (self.timesteps.cpu() == _as_index(timestep)).nonzero().item()

    def model_input_scale(self, timestep) -> float:
        """1 / sqrt(sigma^2 + 1) of `scale_model_input` (:172-191) as a host scalar."""
        sigma = self.sigmas[self._index(timestep)].cpu()
        self.is_scale_input_called = True
        return float(1.0 / ((sigma ** 2 + 1) ** 0.5))

    def scale_model_input(self, sample: torch.Tensor, timestep) -> torch.Tensor:
        sigma = self.sigmas[self._index(timestep)].to(sample.device)
        self.is_scale_input_called = True
        return sample / ((sigma ** 2 + 1) ** 0.5)

    def set_timesteps(self, num_inference_steps: int, device: Union[str, torch.device] = None):
        self.num_inference_steps = num_inference_steps
        ts = np.linspace(0, self.config.num_train_timesteps - 1, num_inference_steps, dtype=float)[::-1].copy()
        sig = (((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5).numpy()
        sig = np.interp(ts, np.arange(0, len(sig)), sig)
        self.sigmas = torch.from_numpy(np.concatenate([sig, [0.0]]).astype(np.float32)).to(device=device)
        self.timesteps = torch.from_numpy(ts).to(device=device)
        self._reset_history()

    def multistep_plan(self, timestep) -> MultistepPlan:
        """Scalars of `step` (:271-316): x0 (:274-287), then prev = x + (x - x0) / sigma * dt + sigma_up noise."""
        pt = self.config.prediction_type
        if pt == "sample":
            raise NotImplementedError("prediction_type not implemented yet: sample")
        if pt not in ("epsilon", "v_prediction"):
            raise ValueError(f"prediction_type given as {pt} must be one of `epsilon`, or `v_prediction`")
        i = self._index(timestep)
        sig = self.sigmas.cpu()
        sigma, sigma_to = sig[i], sig[i + 1]
        if pt == "epsilon":
            a_x, a_e = torch.tensor(1.0), -sigma
        else:
            a_x, a_e = 1.0 / (sigma ** 2 + 1), -sigma / (sigma ** 2 + 1) ** 0.5
        sigma_up = (sigma_to ** 2 * (sigma ** 2 - sigma_to ** 2) / sigma ** 2) ** 0.5
        sigma_down = (sigma_to ** 2 - sigma_up ** 2) ** 0.5
        r = (sigma_down - sigma) / sigma
        return MultistepPlan(float(a_x), float(a_e), 0.0, float(1.0 + r), float(-r), c_n=float(sigma_up), needs_noise=True)

    def step(self, model_output: torch.Tensor, timestep, sample: torch.Tensor, generator=None, return_dict: bool = True,
             w_ind_noise: float = 0.5, noise_type: str = "random"):
        if isinstance(timestep, int) or isinstance(timestep, (torch.IntTensor, torch.LongTensor)):
            raise ValueError("Passing integer indices (e.g. from `enumerate(timesteps)`) as timesteps to"
                             " `EulerDiscreteScheduler.step()` is not supported. Make sure to pass"
                             " one of the `scheduler.timesteps` as a timestep.")
        p = self.multistep_plan(timestep)
        noise = _variance_noise(model_output, generator, noise_type, w_ind_noise)     # drawn on every step (:303-314)
        prev, x0 = self._step_tensors(p, model_output, sample, noise)
        if not return_dict:
            return (prev,)
        return EulerAncestralDiscreteSchedulerOutput(prev_sample=prev, pred_original_sample=x0.to(sample.dtype, copy=True))

    def add_noise(self, original_samples: torch.Tensor, noise: torch.Tensor, timesteps: torch.Tensor) -> torch.Tensor:
        sigmas = self.sigmas.to(device=original_samples.device, dtype=original_samples.dtype)
        sched_t = self.timesteps.to(original_samples.device)
        idx = [(sched_t == t).nonzero().item() for t in timesteps.to(original_samples.device)]
        sigma = sigmas[idx].flatten()
        while sigma.dim() < original_samples.dim():
            sigma = sigma.unsqueeze(-1)
        return original_samples + noise * sigma

    def __len__(self):
        return self.config.num_train_timesteps


class DDPMScheduler(_MultistepMirror):
    """musev/schedulers/scheduling_ddpm.py:42-262 over diffusers schedulers/scheduling_ddpm.py:140-318,453-512."""
    order = 1

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.0001, beta_end: float = 0.02,
                 beta_schedule: str = "linear", trained_betas=None, variance_type: str = "fixed_small",
                 clip_sample: bool = True, prediction_type: str = "epsilon", thresholding: bool = False,
                 dynamic_thresholding_ratio: float = 0.995, clip_sample_range: float = 1, sample_max_value: float = 1,
                 timestep_spacing: str = "leading", steps_offset: int = 0):
        if thresholding:
            raise NotImplementedError("dynamic thresholding is unsuitable for latent diffusion and is not supported")
        if clip_sample and not clip_sample_range > 0:
            # the kernel clamps only for a positive range; the reference would clamp x0 to 0 (range 0) or to a degenerate
            # interval (negative range), which no sampler run wants
            raise ValueError(f"clip_sample_range must be > 0 when clip_sample is set, got {clip_sample_range}")
        if variance_type in ("learned", "learned_range"):
            raise NotImplementedError(f"variance_type {variance_type!r} needs a model that predicts its variance (2x the "
                                      "sample channels); the MuseV UNet outputs 4 channels")
        if variance_type not in ("fixed_small", "fixed_small_log", "fixed_large", "fixed_large_log"):
            raise ValueError(f"unknown variance_type {variance_type}")
        if prediction_type not in ("epsilon", "sample", "v_prediction"):
            raise ValueError(f"prediction_type given as {prediction_type} must be one of `epsilon`, `sample` or"
                             " `v_prediction`  for the DDPMScheduler.")
        self.config = SimpleNamespace(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                                      beta_schedule=beta_schedule, trained_betas=trained_betas, variance_type=variance_type,
                                      clip_sample=clip_sample, prediction_type=prediction_type, thresholding=thresholding,
                                      dynamic_thresholding_ratio=dynamic_thresholding_ratio,
                                      clip_sample_range=clip_sample_range, sample_max_value=sample_max_value,
                                      timestep_spacing=timestep_spacing, steps_offset=steps_offset)
        if trained_betas is None and beta_schedule == "sigmoid":
            self.betas = torch.sigmoid(torch.linspace(-6, 6, num_train_timesteps)) * (beta_end - beta_start) + beta_start
        else:
            self.betas = _betas_cos(beta_schedule, beta_start, beta_end, num_train_timesteps, trained_betas, self.__class__)
        self.alphas = 1.0 - self.betas
        self.alphas_cumprod = torch.cumprod(self.alphas, dim=0)
        self.one = torch.tensor(1.0)
        self.init_noise_sigma = 1.0
        self.custom_timesteps = False
        self.num_inference_steps = None
        self.timesteps = torch.from_numpy(np.arange(0, num_train_timesteps)[::-1].copy())
        self.variance_type = variance_type
        self._reset_history()

    def scale_model_input(self, sample: torch.Tensor, timestep: Optional[int] = None) -> torch.Tensor:
        return sample

    def model_input_scale(self, timestep) -> float:
        return 1.0

    def set_timesteps(self, num_inference_steps: Optional[int] = None, device: Union[str, torch.device] = None,
                      timesteps: Optional[List[int]] = None):
        c = self.config
        if num_inference_steps is not None and timesteps is not None:
            raise ValueError("Can only pass one of `num_inference_steps` or `custom_timesteps`.")
        if timesteps is not None:
            for i in range(1, len(timesteps)):
                if timesteps[i] >= timesteps[i - 1]:
                    raise ValueError("`custom_timesteps` must be in descending order.")
            if timesteps[0] >= c.num_train_timesteps:
                raise ValueError(f"`timesteps` must start before `self.config.train_timesteps`: {c.num_train_timesteps}.")
            ts = np.array(timesteps, dtype=np.int64)
            self.custom_timesteps = True
        else:
            if num_inference_steps > c.num_train_timesteps:
                raise ValueError(
                    f"`num_inference_steps`: {num_inference_steps} cannot be larger than `self.config.train_timesteps`:"
                    f" {c.num_train_timesteps} as the unet model trained with this scheduler can only handle"
                    f" maximal {c.num_train_timesteps} timesteps.")
            self.num_inference_steps = num_inference_steps
            self.custom_timesteps = False
            if c.timestep_spacing == "linspace":
                ts = np.linspace(0, c.num_train_timesteps - 1, num_inference_steps).round()[::-1].copy().astype(np.int64)
            elif c.timestep_spacing == "leading":
                ratio = c.num_train_timesteps // self.num_inference_steps
                ts = (np.arange(0, num_inference_steps) * ratio).round()[::-1].copy().astype(np.int64)
                ts += c.steps_offset
            elif c.timestep_spacing == "trailing":
                ratio = c.num_train_timesteps / self.num_inference_steps
                ts = np.round(np.arange(c.num_train_timesteps, 0, -ratio)).astype(np.int64)
                ts -= 1
            else:
                raise ValueError(f"{c.timestep_spacing} is not supported. Please make sure to choose one of 'linspace', "
                                 "'leading' or 'trailing'.")
        self.timesteps = torch.from_numpy(ts).to(device)
        self._reset_history()

    def previous_timestep(self, timestep):
        if self.custom_timesteps:
            index = (self.timesteps.cpu() == timestep).nonzero(as_tuple=True)[0][0]
            return -1 if index == self.timesteps.shape[0] - 1 else int(self.timesteps[index + 1])
        n = self.num_inference_steps if self.num_inference_steps else self.config.num_train_timesteps
        return timestep - self.config.num_train_timesteps // n

    def multistep_plan(self, timestep) -> MultistepPlan:
        """Scalars of `step` (:156-255): x0 with clip_sample, the posterior mean coefficients, the noise scale."""
        c = self.config
        t = int(_as_index(timestep))
        prev_t = self.previous_timestep(t)
        a_t = self.alphas_cumprod[t]
        a_p = self.alphas_cumprod[prev_t] if prev_t >= 0 else self.one
        b_t, b_p = 1 - a_t, 1 - a_p
        cur_a = a_t / a_p
        cur_b = 1 - cur_a
        if c.prediction_type == "epsilon":
            a_x, a_e = 1.0 / a_t ** 0.5, -(b_t ** 0.5) / a_t ** 0.5
        elif c.prediction_type == "sample":
            a_x, a_e = 0.0, 1.0
        else:
            a_x, a_e = a_t ** 0.5, -(b_t ** 0.5)
        c0 = (a_p ** 0.5 * cur_b) / b_t
        c_x = cur_a ** 0.5 * b_p / b_t
        c_n = 0.0
        if t > 0:
            var = torch.clamp(b_p / b_t * cur_b, min=1e-20)                  # _get_variance (diffusers :280-318)
            vt = c.variance_type
            if vt == "fixed_small":
                c_n = var ** 0.5
            elif vt == "fixed_small_log":
                c_n = torch.exp(0.5 * torch.log(var))                         # multiplied as is (:242-246)
            elif vt == "fixed_large":
                c_n = cur_b ** 0.5
            else:
                # fixed_large_log: the reference takes sqrt(log(beta_t)) of a negative number -> NaN, as here
                c_n = torch.log(cur_b) ** 0.5
        return MultistepPlan(float(a_x), float(a_e), float(c.clip_sample_range) if c.clip_sample else 0.0, float(c_x),
                             float(c0), c_n=float(c_n), needs_noise=t > 0)

    def step(self, model_output: torch.Tensor, timestep: int, sample: torch.Tensor, generator=None, return_dict: bool = True,
             w_ind_noise: float = 0.5, noise_type: str = "random"):
        if model_output.shape[1] != sample.shape[1]:
            raise NotImplementedError("a model output with a predicted variance is not supported")
        p = self.multistep_plan(timestep)
        noise = _variance_noise(model_output, generator, noise_type, w_ind_noise) if p.needs_noise else None
        prev, x0 = self._step_tensors(p, model_output, sample, noise)
        if not return_dict:
            return (prev,)
        return DDPMSchedulerOutput(prev_sample=prev, pred_original_sample=x0.to(sample.dtype, copy=True))

    def add_noise(self, original_samples: torch.Tensor, noise: torch.Tensor, timesteps: torch.Tensor) -> torch.Tensor:
        a = self.alphas_cumprod.to(device=original_samples.device, dtype=original_samples.dtype)[timesteps.to(original_samples.device)]
        sa, sb = (a ** 0.5).flatten(), ((1 - a) ** 0.5).flatten()
        while sa.dim() < original_samples.dim():
            sa, sb = sa.unsqueeze(-1), sb.unsqueeze(-1)
        return sa * original_samples + sb * noise

    def __len__(self):
        return self.config.num_train_timesteps
