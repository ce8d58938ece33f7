"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/samplers_multistep.pt and tests/golden/loop_musev_narrow_dpm.pt by running
the UNMODIFIED musev schedulers (imported through ref_shim):

  * DPMSolverMultistepScheduler      musev/schedulers/scheduling_dpmsolver_multistep.py:66-815
  * EulerAncestralDiscreteScheduler  musev/schedulers/scheduling_euler_ancestral_discrete.py:90-356
  * DDPMScheduler                    musev/schedulers/scheduling_ddpm.py:42-262

Per configuration the fixture holds the constructor kwargs, the timesteps (and sigmas / init_noise_sigma), the seeded start
sample and, per step, the model output fed to `step` (a deterministic dummy model of the current sample), the noise the
reference drew and its `prev_sample`. The loop fixture is `oracle.pipeline_oracle.denoise_loop` around the imported
narrow UNet with the imported DPM-Solver++ 2M Karras scheduler, 10 steps.

Run in the build container only:  python -m oracle.make_golden_samplers_multistep
"""
from __future__ import annotations

import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shim  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
SD15 = dict(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")

# name -> (class name, constructor kwargs, steps, step kwargs)
CONFIGS = {
    "dpmpp_2m_karras_10": ("DPMSolverMultistepScheduler", dict(SD15), 10, {}),
    "dpmpp_2m_karras_20": ("DPMSolverMultistepScheduler", dict(SD15), 20, {}),
    "dpmpp_3m": ("DPMSolverMultistepScheduler", dict(SD15, solver_order=3, use_karras_sigmas=False), 12, {}),
    "dpm_heun": ("DPMSolverMultistepScheduler", dict(SD15, algorithm_type="dpmsolver", solver_type="heun"), 10, {}),
    "dpmpp_2m_vpred": ("DPMSolverMultistepScheduler", dict(SD15, prediction_type="v_prediction"), 10, {}),
    "dpmpp_cos_clipped": ("DPMSolverMultistepScheduler", dict(beta_schedule="squaredcos_cap_v2", use_karras_sigmas=False,
                                                              lambda_min_clipped=-5.1), 10, {}),
    "ddpm_clip": ("DDPMScheduler", dict(clip_sample=True, clip_sample_range=1.0), 10, {}),
    "euler_a_random": ("EulerAncestralDiscreteScheduler", dict(SD15), 10, dict(noise_type="random")),
    "euler_a_video_fusion": ("EulerAncestralDiscreteScheduler", dict(SD15), 10,
                             dict(noise_type="video_fusion", w_ind_noise=0.5)),
    "ddpm_small_log": ("DDPMScheduler", dict(variance_type="fixed_small_log", clip_sample=False), 10, {}),
    "ddpm_large_vpred": ("DDPMScheduler", dict(variance_type="fixed_large", prediction_type="v_prediction"), 10, {}),
    "ddpm_sample_trailing": ("DDPMScheduler", dict(SD15, prediction_type="sample", timestep_spacing="trailing",
                                                   clip_sample=False), 10, dict(noise_type="video_fusion")),
}
SHAPE = (1, 4, 2, 4, 4)


def load_classes():
    """The three reference classes. `set_timesteps` of the DPM scheduler passes the 0-d tensor `torch.searchsorted` returns as
    `np.linspace`'s stop (:251-263), which numpy 2 rejects; the module sees a `torch` whose `searchsorted` returns that
    index as a Python int (same value)."""
    ref_shim.load()
    import musev.schedulers.scheduling_dpmsolver_multistep as dpm_mod
    from musev.schedulers.scheduling_ddpm import DDPMScheduler
    from musev.schedulers.scheduling_euler_ancestral_discrete import EulerAncestralDiscreteScheduler

    class _Torch:
        def __getattr__(self, name):
            return getattr(torch, name)

        @staticmethod
        def searchsorted(*a, **k):
            return int(torch.searchsorted(*a, **k))

    dpm_mod.torch = _Torch()
    return dict(DPMSolverMultistepScheduler=dpm_mod.DPMSolverMultistepScheduler, DDPMScheduler=DDPMScheduler,
                EulerAncestralDiscreteScheduler=EulerAncestralDiscreteScheduler)


def dummy_model(x, t):
    """Deterministic stand-in for the UNet: depends on the sample and the timestep."""
    return 0.8 * torch.tanh(0.7 * x) + 0.05 * torch.sin(3.0 * x + 0.01 * float(t))


def golden_steps(classes):
    out = {}
    for ci, (name, (cls_name, kw, steps, step_kw)) in enumerate(CONFIGS.items()):
        s = classes[cls_name](**kw)
        s.set_timesteps(steps)
        g = torch.Generator().manual_seed(100 + ci)
        x = torch.randn(SHAPE, generator=g) * float(getattr(s, "init_noise_sigma", 1.0))
        x_start = x.clone()
        noise_gen = torch.Generator().manual_seed(200 + ci)
        eps_seq, prev_seq, noise_seq = [], [], []
        for t in s.timesteps:
            xin = s.scale_model_input(x, t)
            eps = dummy_model(xin, t)
            state = noise_gen.get_state()
            kwargs = dict(step_kw)
            if cls_name != "DPMSolverMultistepScheduler":
                kwargs["generator"] = noise_gen
            prev = s.step(eps, t, x, return_dict=True, **kwargs).prev_sample
            # the noise this step drew: replay the generator from its state before the step
            used = noise_gen.get_state()
            noise = None
            if not torch.equal(state, used):
                rg = torch.Generator()
                rg.set_state(state)
                from musev_b200.scheduler import _variance_noise
                noise = _variance_noise(eps, rg, step_kw.get("noise_type", "random"), step_kw.get("w_ind_noise", 0.5))
                assert torch.equal(rg.get_state(), used), name
            eps_seq.append(eps.clone())
            prev_seq.append(prev.clone())
            noise_seq.append(noise)
            x = prev
        entry = dict(cls=cls_name, kwargs=kw, steps=steps, step_kwargs=step_kw, timesteps=s.timesteps.clone(),
                     init_noise_sigma=float(getattr(s, "init_noise_sigma", 1.0)), x=x_start, eps=eps_seq, prev=prev_seq,
                     noise=noise_seq, noise_seed=200 + ci)
        if hasattr(s, "sigmas"):
            entry["sigmas"] = s.sigmas.clone()
        out[name] = entry
        print(f"{name}: {len(s.timesteps)} steps, timesteps {s.timesteps.tolist()[:4]}..., final std {x.std().item():.4f}")
    out["source"] = "imported musev.schedulers DPMSolverMultistep / EulerAncestralDiscrete / DDPM on CPU fp32"
    torch.save(out, os.path.join(GOLDEN, "samplers_multistep.pt"))


def golden_loop(classes, steps=10, T=20, h=8, w=8, wseed=0, iseed=77):
    """denoise_loop (pipeline_oracle) around the imported narrow UNet and the imported DPM-Solver++ 2M Karras."""
    from musev_b200.schema import preset_config
    from musev_b200.synth import make_inputs, make_state_dict
    from oracle.make_golden import NARROW, build_reference
    from oracle.pipeline_oracle import denoise_loop
    preset = "musev"
    cfg = preset_config(preset, block_out_channels=NARROW)
    m, cfg = build_reference(preset, NARROW, make_state_dict(cfg, seed=wseed))
    sched = classes["DPMSolverMultistepScheduler"](**SD15)
    g = torch.Generator().manual_seed(iseed)
    latents = torch.randn(1, 4, T, h, w, generator=g)
    cond = torch.randn(1, 4, 1, h, w, generator=g) * 0.5
    prompt = torch.randn(2, 77, cfg.cross_attention_dim, generator=g)
    extra = make_inputs(cfg, batch=2, frames=1, h=h, w=w, seed=iseed)
    kw = {k: extra[k] for k in ("down_block_refer_embs", "mid_block_refer_emb", "vision_clip_emb") if k in extra}
    kw["ip_adapter_scale"] = 1.0

    def unet(sample, t, enc, **k):
        return m(sample, t, enc, do_classifier_free_guidance=True, **k)[0]

    with torch.no_grad():
        out = denoise_loop(unet, sched, latents, cond, prompt, steps, 3.5, context_frames=8, context_overlap=2, unet_kwargs=kw)
    meta = dict(preset=preset, block_out_channels=list(NARROW), T=T, h=h, w=w, steps=steps, weight_seed=wseed, input_seed=iseed,
                context_frames=8, context_overlap=2, guidance_scale=3.5, scheduler_kwargs=SD15,
                timesteps=sched.timesteps.tolist(),
                source="imported reference UNet + musev DPMSolverMultistepScheduler (++ 2M Karras) in pipeline_oracle.denoise_loop")
    path = os.path.join(GOLDEN, "loop_musev_narrow_dpm.pt")
    torch.save({"meta": meta, "latents": out.clone()}, path)
    print(path, "final latents std", out.std().item())


if __name__ == "__main__":
    cls = load_classes()
    golden_steps(cls)
    if "--steps-only" not in sys.argv:
        golden_loop(cls)
