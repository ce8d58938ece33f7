#!/usr/bin/env python
"""Runs one of BASELINE.json's configurations 2-5 end to end on the engine and prints one JSON line (rank 0).

  python tools/run_config.py --config 2                                   (1 GPU)
  python -m torch.distributed.run --nnodes=1 --nproc-per-node 4 --master-addr 127.0.0.1 --master-port 29511 \
         tools/run_config.py --config 3                                   (4 GPUs; config 4 / 5: 8 GPUs)

  2  image2video 16 frames 512x512, musev, 20 DDIM steps                        1 window
  3  image2video 48 frames 512x512, musev_referencenet + ReferenceNet one-shot + IP-Adapter tokens; window 16 overlap 4
     -> 4 windows (0-15, 12-27, 24-39, 36-47: the last one has 12 frames)
  4  pose video2video 128 frames 512x512, musev_referencenet + IP-Adapter + ControlNet encoder EVERY window-step;
     window 16 overlap 4 -> 11 windows (the last one has 8 frames); `--controlnets N` runs N ControlNets per
     window-step with their residuals summed on the device (Multi-ControlNet, e.g. `--controlnet_name dwpose,depth`)
  5  512 frames 512x768 (64x96 latents), musev, window 16 stride 8 -> 63 windows
Synthetic weights / inputs (no checkpoints offline). The one-shot side paths (ReferenceNet, image projection, ControlNet
condition embedding) run before the timed region, as in the metric definition (SURVEY.md 8d); the ControlNet encoder itself
is inside (it runs per window-step)."""
from __future__ import annotations

import argparse
import datetime
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONFIGS = {
    2: dict(preset="musev", T=16, h=64, w=64, overlap=4, refnet=False, controlnet=False),
    3: dict(preset="musev_referencenet", T=48, h=64, w=64, overlap=4, refnet=True, controlnet=False),
    4: dict(preset="musev_referencenet", T=128, h=64, w=64, overlap=4, refnet=True, controlnet=True),
    5: dict(preset="musev", T=512, h=64, w=96, overlap=8, refnet=False, controlnet=False),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, required=True, choices=sorted(CONFIGS))
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--repeat", type=int, default=1)
    ap.add_argument("--cfg-split", action="store_true")
    ap.add_argument("--frames", type=int, default=0, help="override the video length (smoke runs)")
    ap.add_argument("--controlnets", type=int, default=1,
                    help="config 4: number of ControlNets per window-step (2 = e.g. `--controlnet_name dwpose,depth`)")
    a = ap.parse_args()
    c = dict(CONFIGS[a.config])
    if a.controlnets != 1 and not c["controlnet"]:
        ap.error("--controlnets applies to the ControlNet configuration (4)")
    if a.frames:
        c["T"] = a.frames
    rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    import torch.distributed as dist
    if world > 1:
        if os.environ.get("NCCL_DEBUG", "").upper() in ("", "VERSION"):
            os.environ["NCCL_DEBUG"] = "WARN"
        dist.init_process_group("nccl", device_id=dev, timeout=datetime.timedelta(seconds=600))
    from musev_b200.context import prepare_global_context
    from musev_b200.pipeline import ParallelDenoiser, make_controlnet_fn
    from musev_b200.scheduler import SD15_DDIM_CONFIG, DDIMScheduler
    from musev_b200.schema import ControlNetConfig, ImageProjConfig, ReferenceNetConfig, preset_config
    from musev_b200.synth import make_state_dict
    from musev_b200.unet import UNet3DConditionModel

    cfg = preset_config(c["preset"])
    unet = UNet3DConditionModel(cfg, device=dev, dtype=torch.float16)
    unet.load_state_dict(make_state_dict(cfg, seed=0, dtype=torch.float16))
    g = torch.Generator().manual_seed(1234)
    T, h, w = c["T"], c["h"], c["w"]
    lat = torch.randn(1, 4, T, h, w, generator=g).half().to(dev)
    cond = (torch.randn(1, 4, 1, h, w, generator=g) * 0.18215).half().to(dev)
    prompt = torch.randn(2, 77, cfg.cross_attention_dim, generator=g).half().to(dev)
    kw, one_shot_ms = {}, {}
    if c["refnet"]:
        from musev_b200.referencenet import ImageProjModel, ReferenceNet2D, ip_adapter_image_emb
        e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        proj = ImageProjModel(ImageProjConfig(), device=dev, dtype=torch.float16)
        proj.load_state_dict(make_state_dict(ImageProjConfig(), seed=9))
        rcfg = ReferenceNetConfig()
        rnet = ReferenceNet2D(rcfg, device=dev, dtype=torch.float16)
        rnet.load_state_dict(make_state_dict(rcfg, seed=5, dtype=torch.float16))
        clip = torch.randn(1, 1, 1024, generator=g).half().to(dev)                   # CLIP-vision embedding of the reference image
        ref_lat = (torch.randn(1, 4, h, w, generator=g) * 0.18215).half().to(dev)    # its VAE latent
        e0.record()
        ip = ip_adapter_image_emb(proj, clip, n_images=1, batch_size=1)              # [2, 4, 768] (uncond first)
        e1.record()
        # uncond == cond for the reference latents (pipeline_controlnet.py:844-861); tokens = the IP-Adapter embedding
        down, mid, _ = rnet(torch.cat([ref_lat] * 2), 0, ip, num_frames=1, return_ndim=5)
        e2.record()
        torch.cuda.synchronize()
        one_shot_ms = {"image_proj": e0.elapsed_time(e1), "referencenet": e1.elapsed_time(e2)}
        kw = dict(down_block_refer_embs=list(down), mid_block_refer_emb=mid, vision_clip_emb=ip.half(), ip_adapter_scale=1.0)
        del rnet, proj
    cnet_fn = None
    if c["controlnet"]:
        from musev_b200.controlnet import ControlNetModel
        ccfg = ControlNetConfig()
        nets, lats = [], []
        for k in range(a.controlnets):
            cnet = ControlNetModel(ccfg, device=dev, dtype=torch.float16)
            cnet.load_state_dict(make_state_dict(ccfg, seed=3 + 10 * k, dtype=torch.float16))
            nets.append(cnet)
            lats.append((torch.randn(2, ccfg.block_out_channels[0], 1 + T, h, w, generator=g) * 0.3).half().to(dev))
        if a.controlnets == 1:
            cnet_fn = make_controlnet_fn(nets[0], lats[0], prompt, 1)
        else:                                        # Multi-ControlNet: the nets' residuals summed on the device
            cnet_fn = make_controlnet_fn(nets, lats, prompt, 1)
    den = ParallelDenoiser(unet, DDIMScheduler(**SD15_DDIM_CONFIG))

    def run(steps):
        return den(lat, cond, prompt, num_inference_steps=steps, guidance_scale=3.5, context_frames=16,
                   context_overlap=c["overlap"], context_schedule="uniform_v2", motion_speed=8.0, unet_kwargs=kw,
                   controlnet_fn=cnet_fn, cfg_split=a.cfg_split)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    res = run(2)                                     # warm-up: 2 steps over every window shape
    barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.repeat):
        res = run(a.steps)
    e1.record()
    barrier()
    ms = torch.tensor([e0.elapsed_time(e1) / a.repeat], device=dev)
    if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    if rank == 0:
        lens = [len(x) for x in res.windows]
        loads = [sum(lens[i] + 1 for i in r) for r in res.windows_per_rank]
        groups = len(res.windows_per_rank)
        print("RUN_CONFIG " + json.dumps({
            "config": a.config, "preset": c["preset"], "frames": T, "latent_hw": [h, w], "ddim_steps": a.steps, "n_gpus": world,
            "cfg_split": a.cfg_split, "windows": len(lens), "window_lengths": lens, "windows_per_rank": res.windows_per_rank,
            "computed_frames_per_rank_group": loads,
            "balance": (sum(loads) / groups) / max(loads) if loads else None,
            "ms_per_denoise": float(ms.item()), "frames_per_s": T / (float(ms.item()) * 1e-3),
            "one_shot_ms": one_shot_ms, "finite": bool(torch.isfinite(res.latents).all().item()),
            "referencenet": c["refnet"], "controlnet_per_window_step": c["controlnet"],
            "controlnets": a.controlnets if c["controlnet"] else 0}), flush=True)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
