"""Times one sampler step of the parallel-denoise loop (overlap mean + CFG + update) on `mvb_fuse_cfg_multistep` against the
reference-form eager step on the same GPU, at the config-2 and config-5 latent shapes ([2,4,16,64,64] and [2,4,512,64,96]),
fp16 latents, fp32 eps accumulator [2B, ...] and fp32 histories as ParallelDenoiser holds them.

  * dpmpp_2m   a second-order DPM-Solver++ step: the kernel reads eps (both CFG halves), x, m1; writes x_prev and m0.
               Eager: `noise_pred / counter`, chunk, CFG (pipeline_controlnet.py:2079,2101-2105), then convert_model_output
               and multistep_dpm_solver_second_order_update (scheduling_dpmsolver_multistep.py:396-418,499-545) on fp16
               tensors with fp32 0-d scalars, as the reference runs them (the history kept as fp16 tensors).
  * euler_a    an Euler ancestral step with noise (scheduling_euler_ancestral_discrete.py:271-316): the kernel also reads the
               noise. Eager: the same CFG head, then the reference's step arithmetic.
Noise generation is outside all timings. Three times are taken, alternated for three rounds, best round reported:
  * kernel_ms   the kernel alone: `--iters` launches captured in one CUDA graph, CUDA events around its replay (no host
                work between launches); this is the number set against the byte bound;
  * call_ms     one `multistep_update` call as ParallelDenoiser issues it (host argument checks, ctypes, launch), CUDA
                events around `--iters` back-to-back calls: at small shapes this measures the host, not the GPU;
  * eager_fp16_ms  the reference-form step, launched eagerly as the reference runs it.
The byte bound is the kernel's HBM traffic at the data-sheet 3.35 TB/s. Prints one JSON line per case with the card's
name, power limit and SM clock.

  python tools/gpu_time_samplers.py [--iters 200]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.gpu_time_clip_vision import PEAK_TBS, card, time_ms  # noqa: E402

SHAPES = {"config2": (2, 4, 16, 64, 64), "config5": (2, 4, 512, 64, 96)}


def sm_clock():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        return "unknown"


def graph_ms(fn, iters):
    """ms per call of `fn` with `iters` calls captured in one CUDA graph and replayed (the launches alone)."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(iters):
            fn()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def kernel_bytes(n, history_reads, noise):
    # eps_sum (2 halves fp32) + x fp16 + x_prev fp16 + m0 fp32 + fp32 history / noise reads
    return n * (8 + 2 + 2 + 4 + 4 * history_reads + (4 if noise else 0))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from musev_b200 import ops
    from musev_b200.samplers import DPMSolverMultistepScheduler, EulerAncestralDiscreteScheduler, multistep_update
    dev = "cuda"
    name, power = card()
    sd15 = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
    for tag, shape in SHAPES.items():
        B, C, T, h, w = shape
        n = B * C * T * h * w
        g = torch.Generator(device=dev).manual_seed(0)
        eps_sum = torch.randn((2 * B, C, T, h, w), generator=g, device=dev)
        counter = torch.ones(T, device=dev) * 2
        x = torch.randn(shape, generator=g, device=dev).half()
        hist = [torch.randn(shape, generator=g, device=dev) for _ in range(2)]
        noise = torch.randn(shape, generator=g, device=dev)
        # plans at the second step of a 20-step run (second order for DPM-Solver++)
        d = DPMSolverMultistepScheduler(**sd15)
        d.set_timesteps(20)
        ts = d.timesteps.tolist()
        d.multistep_plan(ts[0])
        p_dpm = d.multistep_plan(ts[1])
        ea = EulerAncestralDiscreteScheduler(**sd15)
        ea.set_timesteps(20)
        p_ea = ea.multistep_plan(ea.timesteps[1])

        # reference-form eager steps (fp16 tensors, fp32 0-d scalars)
        t0, t1, tp = ts[1], ts[0], ts[2]
        lam, al, sg = d.lambda_t.to(dev), d.alpha_t.to(dev), d.sigma_t.to(dev)
        m1_16 = hist[0].half()
        eps_sum16, cnt16 = eps_sum.half(), counter.half().view(1, 1, T, 1, 1)
        sig = ea.sigmas.to(dev)
        noise16 = noise.half()

        def cfg_head():
            npred = eps_sum16 / cnt16
            u, tx = npred.chunk(2)
            return u + 7.5 * (tx - u)

        def eager_dpm():
            e = cfg_head()
            m0 = (x - sg[t0] * e) / al[t0]
            h_, h0 = lam[tp] - lam[t0], lam[t0] - lam[t1]
            r0 = h0 / h_
            D0, D1 = m0, (1.0 / r0) * (m0 - m1_16)
            return (sg[tp] / sg[t0]) * x - (al[tp] * (torch.exp(-h_) - 1.0)) * D0 - 0.5 * (al[tp] * (torch.exp(-h_) - 1.0)) * D1

        def eager_ea():
            e = cfg_head()
            s_, s_to = sig[1], sig[2]
            x0 = x - s_ * e
            s_up = (s_to ** 2 * (s_ ** 2 - s_to ** 2) / s_ ** 2) ** 0.5
            s_down = (s_to ** 2 - s_up ** 2) ** 0.5
            return x + (x - x0) / s_ * (s_down - s_) + noise16 * s_up

        cases = {
            "dpmpp_2m": (lambda: multistep_update(ops, p_dpm, eps_sum, counter, x, 7.5, hist), eager_dpm,
                         kernel_bytes(n, 1, False)),
            "euler_a": (lambda: multistep_update(ops, p_ea, eps_sum, counter, x, 7.5, hist, noise), eager_ea,
                        kernel_bytes(n, 0, True)),
        }
        for case, (kern, eager, nbytes) in cases.items():
            ms_k, ms_c, ms_e = [], [], []
            for _ in range(3):
                ms_k.append(graph_ms(kern, args.iters))
                ms_c.append(time_ms(kern, args.iters))
                ms_e.append(time_ms(eager, args.iters))
            k_ms, c_ms, e_ms = min(ms_k), min(ms_c), min(ms_e)
            bound_ms = nbytes / (PEAK_TBS * 1e12) * 1e3
            print(json.dumps(dict(case=case, shape=tag, dims=list(shape), gpu=name, power_limit=power, sm_clock=sm_clock(),
                                  elements=n, kernel_ms=round(k_ms, 4), call_ms=round(c_ms, 4), eager_fp16_ms=round(e_ms, 4),
                                  call_speedup_vs_eager=round(e_ms / c_ms, 2),
                                  kernel_bytes=nbytes, kernel_tb_per_s=round(nbytes / (k_ms * 1e-3) / 1e12, 3),
                                  byte_bound_ms=round(bound_ms, 4), of_byte_bound=round(bound_ms / k_ms, 3),
                                  rounds_kernel_ms=[round(v, 4) for v in ms_k], rounds_call_ms=[round(v, 4) for v in ms_c],
                                  rounds_eager_ms=[round(v, 4) for v in ms_e])),
                  flush=True)
        del eps_sum, eps_sum16, hist, noise, noise16, x
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
