#!/usr/bin/env python
"""Times the ControlNet part of one window-step at the config-4 window shape for N = 1, 2, 3 SD-1.5 ControlNets and
prints one JSON line per N (plus the card's name and power limit):

  * engine: `make_controlnet_fn` over N engine nets -- condition embeddings computed once per call (timed separately, per
    net, for the 1 + 128 frames of config 4), each window-step slices them, runs the nets and adds the second and later
    nets' maps into the first's on the device (`mvb_controlnet_args.accumulate`); with the last net's keep at 0 it is
    not run (`engine_ms_last_net_off`);
  * reference: the way MuseV's multi-net branch runs (pipeline_controlnet.py:1969-1982, multicontrolnet.py:31-72):
    eager fp16 torch nets (oracle/controlnet_oracle.py) that embed their 34 control images on every window-step, maps
    summed in torch.
Shape: 2B x (1 + 16) = 34 frames of 64 x 64 latents, 512 x 512 control images, fp16. Engine and reference alternate over
the rounds. A torch.profiler pass (after the timed rounds) gives the accumulate kernel's time; its bytes are the fp16 map
read, the destination read and the destination written, computed from the map shapes.

  python tools/gpu_time_controlnet.py [--nets 1 2 3] [--iters 10] [--rounds 3]
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


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(), "unknown"


def time_ms(fn, iters):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def map_bytes(net, NF, H, W, elem=2):
    """Bytes of one net's 12 + 1 residual maps at [NF, C, H / ds, W / ds]."""
    return sum(NF * c * (H // ds) * (W // ds) * elem for c, ds in net._maps)


def kernel_us(fn, names, reps):
    """Total CUDA time per call (us) of the kernels whose name contains each of `names`, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {n: 0.0 for n in names}
    for ev in prof.key_averages():
        for n in names:
            if n in ev.key:
                out[n] += ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
    return {n: v / reps for n, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nets", type=int, nargs="+", default=[1, 2, 3])
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from musev_b200.controlnet import ControlNetModel
    from musev_b200.pipeline import make_controlnet_fn
    from musev_b200.schema import ControlNetConfig
    from musev_b200.synth import make_state_dict
    from oracle.controlnet_oracle import ControlNetOracle
    dev, f16 = "cuda", torch.float16
    cfg = ControlNetConfig()
    B, n_vc, win, T, h, w = 1, 1, 16, 128, 64, 64
    tc = n_vc + win
    NF = 2 * B * tc                                                  # 34 frames per window-step
    g = torch.Generator().manual_seed(7)
    prompt = torch.randn(2, 77, 768, generator=g).to(dev, f16)
    x = torch.randn(2 * B, 4, tc, h, w, generator=g).to(dev, f16)   # latent_model_input of one window
    window = list(range(win))
    nmax = max(args.nets)
    nets, eager, lats, images = [], [], [], []
    for k in range(nmax):
        sd = make_state_dict(cfg, seed=3 + 10 * k, dtype=f16)
        n = ControlNetModel(cfg, device=dev, dtype=f16)
        n.load_state_dict(sd)
        nets.append(n)
        eager.append(ControlNetOracle(cfg, sd, device=dev, dtype=f16))
        imgs = torch.rand(n_vc + T, 3, 8 * h, 8 * w, generator=g).to(dev, f16)          # every frame's control image
        e = n.controlnet_cond_embedding(imgs)                                             # once per call
        lats.append(torch.cat([e.permute(1, 0, 2, 3).unsqueeze(0)] * 2 * B).contiguous())
        ctx = [0] + [c + n_vc for c in window]
        images.append(torch.cat([imgs[ctx]] * 2 * B))                                    # this window's 34 images
        del imgs, e
    torch.cuda.synchronize()
    embed_imgs = torch.rand(n_vc + T, 3, 8 * h, 8 * w, generator=g).to(dev, f16)
    embed_ms = time_ms(lambda: nets[0].controlnet_cond_embedding(embed_imgs), 3)
    del embed_imgs
    x2 = x.permute(0, 2, 1, 3, 4).reshape(NF, 4, h, w)
    enc2 = prompt.repeat_interleave(tc, dim=0)
    name, power = card()
    t = 501
    with torch.no_grad():
        for N in args.nets:
            scales = [1.0 - 0.1 * k for k in range(N)]
            fn = make_controlnet_fn(nets[:N] if N > 1 else nets[0], lats[:N] if N > 1 else lats[0], prompt, n_vc,
                                    controlnet_conditioning_scale=scales if N > 1 else scales[0])
            fn_off = make_controlnet_fn(nets[:N], lats[:N], prompt, n_vc, controlnet_conditioning_scale=scales,
                                        controlnet_keep=[[1.0] * (N - 1) + [0.0]]) if N > 1 else None

            def reference():
                down, mid = None, None
                for net, im, s in zip(eager[:N], images[:N], scales):
                    d, m = net(x2, t, enc2, controlnet_cond=im, conditioning_scale=s)   # embeds 34 images every time
                    down, mid = (d, m) if down is None else ([a + b for a, b in zip(down, d)], mid + m)
                return down, mid

            eng, ref, off = [], [], []
            for _ in range(args.rounds):                                 # alternate, so drift hits both the same way
                eng.append(time_ms(lambda: fn(window, x, t, 0), args.iters))
                ref.append(time_ms(reference, args.iters))
                if fn_off is not None:
                    off.append(time_ms(lambda: fn_off(window, x, t, 0), args.iters))
            ed, em = fn(window, x, t, 0)
            rd, rm = reference()
            diff = max((a.float() - b.float()).abs().max().item() for a, b in zip(list(ed) + [em], list(rd) + [rm]))
            scale_ref = max(b.abs().max().item() for b in list(rd) + [rm])
            k = kernel_us(lambda: fn(window, x, t, 0), ["tokens_to_ncthw_add_kernel", "tokens_to_ncthw_kernel"], 5)
            nbytes = 3 * map_bytes(nets[0], NF, h, w) * (N - 1)        # map read + destination read + destination write
            add_us = k["tokens_to_ncthw_add_kernel"]
            print(json.dumps({
                "gpu": name, "power_limit": power, "controlnets": N, "frames_per_window_step": NF, "latent_hw": [h, w],
                "image_hw": [8 * h, 8 * w],
                "engine_ms": min(eng), "reference_eager_fp16_ms": min(ref), "speedup_vs_reference": min(ref) / min(eng),
                "engine_ms_runs": [round(v, 3) for v in eng], "reference_ms_runs": [round(v, 3) for v in ref],
                "engine_ms_last_net_off": min(off) if off else None,
                "embedding_ms_per_net_per_call_129_frames": embed_ms,
                "accumulate_kernel_us": add_us, "accumulate_mbytes": nbytes / 1e6,
                "accumulate_gbs": nbytes / (add_us * 1e-6) / 1e9 if add_us > 0 else None,
                "write_kernel_us": k["tokens_to_ncthw_kernel"], "write_mbytes": 2 * map_bytes(nets[0], NF, h, w) / 1e6,
                "max_abs_engine_vs_reference": diff, "max_abs_reference": scale_ref,
            }), flush=True)


if __name__ == "__main__":
    main()
