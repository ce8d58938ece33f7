#!/usr/bin/env python
"""Times the SD-1.5 VAE's tiled mode on the engine per frame: `decode_latents` and `encode_video` with seeded weights,
fp16 latents / video, `--frames` frames per call (= frames_per_call), CUDA events around `--reps` calls after two warm-up
calls. Sizes: 704x704 tiled and untiled (it fits both ways), 1216x704 and 1280x704 tiled. Also prints the tile-count
overhead (latent pixels the tiles cover over the frame's) and the card's name and power limit, read in the same run.
Prints one JSON line per size; writes nothing to disk."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                               str(torch.cuda.current_device())], capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception as e:
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=4)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    from musev_b200 import vae_tiling
    from musev_b200.schema import VAEConfig
    from musev_b200.synth import make_state_dict, make_vae_images
    from musev_b200.vae import AutoencoderKL
    dev = "cuda"
    cfg = VAEConfig()
    vae = AutoencoderKL(cfg, device=dev, dtype=torch.float16, frames_per_call=a.frames)
    vae.load_state_dict(make_state_dict(cfg, seed=11, dtype=torch.float16))
    card = _card()

    def per_frame_ms(fn):
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / (a.reps * a.frames)

    for H, W, tiled in ((704, 704, False), (704, 704, True), (1216, 704, True), (1280, 704, True)):
        h, w = H // 8, W // 8
        video = make_vae_images(a.frames, H, W, seed=5).half().permute(1, 0, 2, 3)[None].contiguous().to(dev)
        lat = (torch.randn(1, 4, a.frames, h, w, generator=torch.Generator().manual_seed(6)) * 0.18215).half().to(dev)
        vae.enable_tiling(tiled)
        dec_ms = per_frame_ms(lambda: vae.decode_latents(lat))
        enc_ms = per_frame_ms(lambda: vae.encode_video(video))
        plan = vae_tiling.plan_decode(h, w, 512, 64, 0.25, 8) if tiled else None
        print(json.dumps({"workload": f"SD-1.5 VAE {H}x{W}, {'tiled' if tiled else 'untiled'}, seeded weights, fp16",
                          "card": card, "frames_per_call": a.frames, "reps": a.reps,
                          "decode_latents_ms_per_frame": dec_ms, "encode_video_ms_per_frame": enc_ms,
                          "tiles_per_frame": plan.tiles_per_frame if plan else 1,
                          "tile_pixel_overhead": plan.covered() / (H * W) if plan else 1.0}), flush=True)


if __name__ == "__main__":
    main()
