"""CPU tests of the multistep sampler mirrors (musev_b200.samplers: DPMSolverMultistepScheduler, EulerAncestralDiscreteScheduler,
DDPMScheduler) and of their dispatch in ParallelDenoiser. The device kernel `mvb_fuse_cfg_multistep` is replaced by a plain
torch double of its documented arithmetic (`CPUOps`); the kernel itself is tested against the same restatement on the GPU
(test_gpu_samplers_multistep.py).

References: tests/golden/samplers_multistep.pt and loop_musev_narrow_dpm.pt (the imported musev schedulers, written by
oracle/make_golden_samplers_multistep.py), and the upstream known-answer tests where the musev copy and the upstream config
coincide."""
import inspect
import os
import socket

import pytest
import torch
import torch.multiprocessing as mp

from conftest import GOLDEN
from musev_b200.samplers import (DDPMScheduler, DPMSolverMultistepScheduler, EulerAncestralDiscreteScheduler, MultistepPlan,
                                 multistep_update)
from musev_b200.scheduler import _variance_noise

CLASSES = dict(DPMSolverMultistepScheduler=DPMSolverMultistepScheduler, DDPMScheduler=DDPMScheduler,
               EulerAncestralDiscreteScheduler=EulerAncestralDiscreteScheduler)


class CPUOps:
    """torch restatement of mvb_fuse_cfg_multistep and mvb_accumulate_window (include/musev_b200.h), in `dtype`."""
    dtype = torch.float32

    @classmethod
    def fuse_cfg_multistep(cls, eps_sum, counter, latents, g, a_x, a_e, clip, c_x, c0, c1=0.0, c2=0.0, c_n=0.0, m1=None,
                           m2=None, noise=None, m0_out=None, cfg=True, out=None):
        dt = cls.dtype
        e = eps_sum.to(dt)
        if counter is not None:
            e = e / counter.to(dt).view(1, 1, -1, *([1] * (e.dim() - 3)))
        if cfg:
            u, tx = e.chunk(2)
            e = u + g * (tx - u)
        x = latents.to(dt)
        m0 = a_x * x + a_e * e
        if clip > 0:
            m0 = m0.clamp(-clip, clip)
        prev = c_x * x + c0 * m0
        if m1 is not None:
            prev = prev + c1 * m1.to(dt)
        if m2 is not None:
            prev = prev + c2 * m2.to(dt)
        if noise is not None:
            prev = prev + c_n * noise.to(dt)
        if m0_out is not None:
            m0_out.copy_(m0)
        return prev.to(latents.dtype)

    @staticmethod
    def accumulate_window(eps_sum, eps, src_t0, frames_dev):
        idx = frames_dev.long()
        eps_sum[:, :, idx] += eps[:, :, src_t0:src_t0 + idx.numel()].float()


def cpu_step(sched, model_output, t, sample, history, generator=None, noise_type="random", w_ind_noise=0.5):
    """The mirror's `step` with the kernel replaced by CPUOps (same plan, same noise draw, same history rotation)."""
    p = sched.multistep_plan(t)
    noise = _variance_noise(model_output, generator, noise_type, w_ind_noise) if p.needs_noise else None
    return multistep_update(CPUOps, p, model_output, None, sample, 1.0, history, noise, cfg=False)


def new_history(x):
    return [torch.zeros(x.shape, dtype=torch.float32) for _ in range(2)]


def load_fixture():
    return torch.load(os.path.join(GOLDEN, "samplers_multistep.pt"))


def make(entry):
    s = CLASSES[entry["cls"]](**entry["kwargs"])
    s.set_timesteps(entry["steps"])
    return s


CONFIG_NAMES = ["dpmpp_2m_karras_10", "dpmpp_2m_karras_20", "dpmpp_3m", "dpm_heun", "dpmpp_2m_vpred", "dpmpp_cos_clipped",
                "ddpm_clip", "euler_a_random", "euler_a_video_fusion", "ddpm_small_log", "ddpm_large_vpred",
                "ddpm_sample_trailing"]


@pytest.mark.parametrize("name", CONFIG_NAMES)
def test_timesteps_sigmas_and_init_noise_sigma_match_reference(name):
    e = load_fixture()[name]
    s = make(e)
    assert torch.equal(s.timesteps, e["timesteps"]), (s.timesteps, e["timesteps"])
    assert abs(float(s.init_noise_sigma) - e["init_noise_sigma"]) < 1e-6
    if "sigmas" in e:
        assert torch.equal(s.sigmas, e["sigmas"])


@pytest.mark.parametrize("name", CONFIG_NAMES)
def test_plan_reproduces_reference_step_sequence(name):
    """Each step fed the reference's model output and sample; the plan's scalars through the kernel arithmetic reproduce the
    reference `prev_sample` of every step, with the noise drawn from the same generator in the same order."""
    e = load_fixture()[name]
    s = make(e)
    hist = new_history(e["x"])
    gen = torch.Generator().manual_seed(e["noise_seed"])
    x = e["x"]
    sk = e["step_kwargs"]
    for i, t in enumerate(s.timesteps):
        prev = cpu_step(s, e["eps"][i], t, x, hist, gen, sk.get("noise_type", "random"), sk.get("w_ind_noise", 0.5))
        ref = e["prev"][i]
        err = (prev - ref).abs().max().item()
        assert err <= 2e-6 * max(1.0, ref.abs().max().item()), (name, i, err)
        x = ref


# ------------------------------------------------------------------------------ upstream known-answer tests
def _dummy_sample_deter():
    """diffusers tests/schedulers/test_schedulers.py:283-295."""
    n = 4 * 3 * 8 * 8
    return (torch.arange(n).reshape(3, 8, 8, 4) / n).permute(3, 0, 1, 2)


def _dummy_model(sample, t):
    """diffusers tests/schedulers/test_schedulers.py:300-310."""
    if isinstance(t, torch.Tensor):
        t = t.reshape(-1, *(1,) * (sample.dim() - 1)).to(sample.dtype)
    return sample * t / (t + 1)


# test_scheduler_dpm_multi.py:19-38 without `euler_at_final` / `use_lu_lambdas` (absent from the musev copy, so the KATs that
# need them -- test_full_loop_with_lu_and_v_prediction, test_euler_at_final -- are not replayed) and with use_karras_sigmas
# passed explicitly, because the musev copy defaults it to True
DPM_KAT = dict(num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02, beta_schedule="linear", solver_order=2,
               prediction_type="epsilon", thresholding=False, sample_max_value=1.0, algorithm_type="dpmsolver++",
               solver_type="midpoint", lower_order_final=False, lambda_min_clipped=-float("inf"), variance_type=None,
               use_karras_sigmas=False)


@pytest.mark.parametrize("kw,mean", [({}, 0.3301),                                              # :215-219
                                     (dict(prediction_type="v_prediction"), 0.2251),            # :248-252
                                     (dict(prediction_type="v_prediction", use_karras_sigmas=True), 0.2096)])  # :254-258
def test_dpm_multistep_upstream_known_answers(kw, mean):
    s = DPMSolverMultistepScheduler(**{**DPM_KAT, **kw})
    s.set_timesteps(10)                                            # full_loop, test_scheduler_dpm_multi.py:102-117
    sample = _dummy_sample_deter()
    hist = new_history(sample)
    for t in s.timesteps:
        sample = cpu_step(s, _dummy_model(sample, t), t, sample, hist)
    assert abs(sample.abs().mean().item() - mean) < 1e-3


@pytest.mark.parametrize("pred,total,mean", [("epsilon", 152.3192, 0.1983), ("v_prediction", 108.4439, 0.1412)])
def test_euler_ancestral_upstream_known_answers(pred, total, mean):
    """test_scheduler_euler_ancestral.py:40-92 (1100 train steps, 10 inference steps, noise from torch.manual_seed(0))."""
    s = EulerAncestralDiscreteScheduler(num_train_timesteps=1100, beta_start=0.0001, beta_end=0.02, beta_schedule="linear",
                                        prediction_type=pred)
    s.set_timesteps(10)
    gen = torch.manual_seed(0)
    sample = _dummy_sample_deter() * s.init_noise_sigma
    hist = new_history(sample)
    for t in s.timesteps:
        sample = s.scale_model_input(sample, t)
        sample = cpu_step(s, _dummy_model(sample, t), t, sample, hist, gen)
    assert abs(sample.abs().sum().item() - total) < 1e-2
    assert abs(sample.abs().mean().item() - mean) < 1e-3


@pytest.mark.parametrize("pred,total,mean", [("epsilon", 258.9606, 0.3372), ("v_prediction", 202.0296, 0.2631)])
def test_ddpm_upstream_known_answers(pred, total, mean):
    """test_scheduler_ddpm.py:71-131: 1000 steps without set_timesteps, clip_sample, fixed_small, noise from manual_seed(0)."""
    s = DDPMScheduler(num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02, beta_schedule="linear",
                      variance_type="fixed_small", clip_sample=True, prediction_type=pred)
    gen = torch.manual_seed(0)
    sample = _dummy_sample_deter()
    hist = new_history(sample)
    for t in reversed(range(len(s))):
        sample = cpu_step(s, _dummy_model(sample, t), t, sample, hist, gen)
    assert abs(sample.abs().sum().item() - total) < 1e-2
    assert abs(sample.abs().mean().item() - mean) < 1e-3


# ------------------------------------------------------------------------------ surface and errors
def test_step_signatures_and_errors():
    assert list(inspect.signature(DPMSolverMultistepScheduler.step).parameters) == [
        "self", "model_output", "timestep", "sample", "generator", "return_dict", "w_ind_noise"]
    for cls in (EulerAncestralDiscreteScheduler, DDPMScheduler):         # the reference order, positional use included
        assert list(inspect.signature(cls.step).parameters) == [
            "self", "model_output", "timestep", "sample", "generator", "return_dict", "w_ind_noise", "noise_type"]
    for algo in ("sde-dpmsolver", "sde-dpmsolver++"):
        with pytest.raises(NotImplementedError, match="728-730"):
            DPMSolverMultistepScheduler(algorithm_type=algo)
    with pytest.raises(NotImplementedError):
        DPMSolverMultistepScheduler(thresholding=True)
    with pytest.raises(NotImplementedError):
        DDPMScheduler(thresholding=True)
    for vt in ("learned", "learned_range"):
        with pytest.raises(NotImplementedError):
            DDPMScheduler(variance_type=vt)
    for rng in (0.0, -1.0):
        with pytest.raises(ValueError, match="clip_sample_range"):
            DDPMScheduler(clip_sample=True, clip_sample_range=rng)
    DDPMScheduler(clip_sample=False, clip_sample_range=0.0)              # the range is unused without clip_sample
    s = EulerAncestralDiscreteScheduler()
    s.set_timesteps(4)
    with pytest.raises(ValueError, match="integer indices"):
        s.step(torch.zeros(1, 4, 1, 2, 2), 3, torch.zeros(1, 4, 1, 2, 2))
    with pytest.raises(ValueError):
        DPMSolverMultistepScheduler().multistep_plan(999)                 # set_timesteps not called
    # bookkeeping is reset by set_timesteps, like `model_outputs` / `lower_order_nums` (:285-288)
    d = DPMSolverMultistepScheduler()
    d.set_timesteps(10)
    first = [d.multistep_plan(t) for t in d.timesteps[:3]]
    d.set_timesteps(10)
    assert [d.multistep_plan(t) for t in d.timesteps[:3]] == first
    assert first[0].c1 == 0.0 and first[1].c1 != 0.0


def test_history_rotation_aliases_m0_into_m2():
    """multistep_update hands the kernel m0_out = history[1] (= m2) and rotates: afterwards history[0] is this step's m0."""
    calls = []

    class Spy:
        @staticmethod
        def fuse_cfg_multistep(*a, m0_out=None, **k):
            calls.append((a[12], a[13], m0_out))
            return a[2]

    h = [torch.zeros(2), torch.ones(2)]
    a, b = h
    p = MultistepPlan(1.0, 0.0, 0.0, 1.0, 0.0, c1=0.5, c2=0.25)
    multistep_update(Spy, p, torch.zeros(2), None, torch.zeros(2), 1.0, h)
    m1, m2, m0 = calls[0]
    assert m1 is a and m2 is b and m0 is b and h[0] is b and h[1] is a
    multistep_update(Spy, MultistepPlan(1.0, 0.0, 0.0, 1.0, 0.0), torch.zeros(2), None, torch.zeros(2), 1.0, h)
    assert calls[1][0] is None and calls[1][1] is None and calls[1][2] is a      # zero coefficients pass no history


# ------------------------------------------------------------------------------ ParallelDenoiser
def _loop_inputs(m, cfg):
    from musev_b200.synth import make_inputs
    gen = torch.Generator().manual_seed(m["input_seed"])
    latents = torch.randn(1, 4, m["T"], m["h"], m["w"], generator=gen)
    cond = torch.randn(1, 4, 1, m["h"], m["w"], generator=gen) * 0.5
    prompt = torch.randn(2, 77, cfg.cross_attention_dim, generator=gen)
    extra = make_inputs(cfg, batch=2, frames=1, h=m["h"], w=m["w"], seed=m["input_seed"])
    kw = {k: extra[k] for k in ("down_block_refer_embs", "mid_block_refer_emb", "vision_clip_emb") if k in extra}
    kw["ip_adapter_scale"] = 1.0
    return latents, cond, prompt, kw


def test_parallel_denoiser_dpm_matches_reference_loop():
    """10 DPM-Solver++ 2M Karras steps x 3 windows through ParallelDenoiser (kernel double, CPU UNet oracle) against the loop
    run with the imported reference UNet and scheduler."""
    from musev_b200.pipeline import ParallelDenoiser
    from musev_b200.schema import preset_config
    from musev_b200.synth import make_state_dict
    from oracle.unet3d_oracle import UNet3DOracle
    g = torch.load(os.path.join(GOLDEN, "loop_musev_narrow_dpm.pt"))
    m = g["meta"]
    cfg = preset_config(m["preset"], block_out_channels=tuple(m["block_out_channels"]))
    o = UNet3DOracle(cfg, make_state_dict(cfg, seed=m["weight_seed"]))
    latents, cond, prompt, kw = _loop_inputs(m, cfg)
    torch.set_num_threads(max(2, torch.get_num_threads()))
    seen = []
    den = ParallelDenoiser(lambda s, t, e, return_dict=False, do_classifier_free_guidance=True, **k: (o(s, t, e, **k),),
                           DPMSolverMultistepScheduler(**m["scheduler_kwargs"]), device_ops=CPUOps)
    res = den(latents, cond, prompt, num_inference_steps=m["steps"], guidance_scale=m["guidance_scale"],
              context_frames=m["context_frames"], context_overlap=m["context_overlap"], motion_speed=8, unet_kwargs=kw,
              callback=lambda i, t, x: seen.append(t))
    assert seen == m["timesteps"]
    err = (res.latents - g["latents"]).abs().max().item()
    assert err < 1e-3 * g["latents"].abs().max().item(), err


def _fake_unet(sample, t, enc, return_dict=False, do_classifier_free_guidance=True, **k):
    pos = torch.arange(sample.shape[2], dtype=sample.dtype).view(1, 1, -1, 1, 1)
    rows = enc.mean((1, 2)).view(-1, 1, 1, 1, 1)
    return (torch.tanh(sample * 0.9 + 0.001 * float(t) + 0.1 * pos) + 0.3 * rows,)


def _worker(rank, world, port, name, out_path, cfg_split):
    import torch.distributed as dist
    from musev_b200.pipeline import ParallelDenoiser
    if world > 1:
        dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    torch.set_num_threads(1)
    gen = torch.Generator().manual_seed(11)
    latents = torch.randn(1, 4, 20, 4, 4, generator=gen)
    cond = torch.randn(1, 4, 1, 4, 4, generator=gen)
    prompt = torch.randn(2, 77, 8, generator=gen)
    sched = {"dpm": lambda: DPMSolverMultistepScheduler(solver_order=3),
             "ddpm": lambda: DDPMScheduler(),
             "euler_a": lambda: EulerAncestralDiscreteScheduler()}[name]()
    den = ParallelDenoiser(_fake_unet, sched, device_ops=CPUOps)
    res = den(latents, cond, prompt, num_inference_steps=6, guidance_scale=3.0, context_frames=8, context_overlap=2,
              cfg_split=cfg_split, generator=torch.Generator().manual_seed(5))
    if rank == 0:
        torch.save({"latents": res.latents, "per_rank": res.windows_per_rank}, out_path)
    if world > 1:
        other = [torch.empty_like(res.latents) for _ in range(world)]
        dist.all_gather(other, res.latents)
        assert all(torch.equal(other[0], x) for x in other)
        dist.destroy_process_group()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.mark.parametrize("name", ["dpm", "ddpm", "euler_a"])
def test_parallel_denoise_multistep_two_ranks_gloo(tmp_path, name):
    """Two gloo ranks, window-sharded and CFG-split: both ranks end with identical latents (asserted in the worker), equal to a
    single-rank run up to the summation order of the overlap accumulation. The noisy samplers draw on rank 0 and broadcast."""
    p1, p2, p3 = (str(tmp_path / f"{i}.pt") for i in range(3))
    _worker(0, 1, 0, name, p1, False)
    mp.spawn(_worker, args=(2, _free_port(), name, p2, False), nprocs=2, join=True)
    mp.spawn(_worker, args=(2, _free_port(), name, p3, True), nprocs=2, join=True)
    single, double, split = (torch.load(p) for p in (p1, p2, p3))
    assert all(len(r) >= 1 for r in double["per_rank"]) and len(split["per_rank"]) == 1
    scale = max(1.0, single["latents"].abs().max().item())
    assert (double["latents"] - single["latents"]).abs().max().item() < 1e-5 * scale
    assert (split["latents"] - single["latents"]).abs().max().item() < 1e-5 * scale


# ------------------------------------------------------------------------------ C ABI
def test_multistep_args_layout_matches_ctypes_mirror(tmp_path):
    """`struct mvb_multistep_args` of include/musev_b200.h against `_capi.MvbMultistepArgs`: size and every field offset as
    gcc sees them, and the binding takes the struct by pointer. (tests/test_capi_symbols.py checks the `} name;` typedefs it
    lists; this struct is declared with a forward typedef and checked here the same way.)"""
    import ctypes
    import re
    import subprocess
    from conftest import ROOT
    from musev_b200 import _capi
    header = open(os.path.join(ROOT, "include", "musev_b200.h")).read()
    assert re.search(r"^struct mvb_multistep_args \{", header, flags=re.M)
    cls = _capi.MvbMultistepArgs
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "musev_b200.h"', "int main(void) {",
             '  printf(". %zu\\n", sizeof(mvb_multistep_args));']
    lines += [f'  printf("{f} %zu\\n", offsetof(mvb_multistep_args, {f}));' for f, *_ in cls._fields_]
    lines += ["  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    r = subprocess.run(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], capture_output=True,
                       text=True)
    assert r.returncode == 0, r.stderr
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout
    for line in out.strip().splitlines():
        name, value = line.split()
        assert int(value) == (ctypes.sizeof(cls) if name == "." else getattr(cls, name).offset), (name, value)
    proto = re.search(r"int mvb_fuse_cfg_multistep\(([^()]*)\);", header).group(1)
    assert proto.replace(" ", "") == "constmvb_multistep_args*args,void*stream"
