#!/usr/bin/env python
"""Times the SD-1.5 VAE on the engine per 512x512 frame: `AutoencoderKL.encode` and `.decode` with seeded weights, fp16
images / latents, `--frames` frames per call (= frames_per_call), CUDA events around `--reps` calls after two warm-up calls.
Prints one JSON line with ms per frame, the TFLOP/s that implies (musev_b200.flops) and the card's name and power limit.
Writes nothing to disk."""
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
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    from musev_b200.flops import vae_decoder_flops, vae_encoder_flops
    from musev_b200.schema import VAEConfig
    from musev_b200.synth import make_state_dict, make_vae_images
    from musev_b200.vae import AutoencoderKL
    dev = "cuda"
    cfg = VAEConfig()
    vae = AutoencoderKL(cfg, device=dev, dtype=torch.float16, frames_per_call=a.frames)
    vae.load_state_dict(make_state_dict(cfg, seed=11, dtype=torch.float16))
    x = make_vae_images(a.frames, 512, 512, seed=5).half().to(dev)
    z = (torch.randn(a.frames, 4, 64, 64, generator=torch.Generator().manual_seed(6)) * 0.18215).half().to(dev)

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

    enc_ms = per_frame_ms(lambda: vae.encode(x))
    dec_ms = per_frame_ms(lambda: vae.decode(z))
    enc_fl = vae_encoder_flops(cfg, 1, 64, 64)["total"]
    dec_fl = vae_decoder_flops(cfg, 1, 64, 64)["total"]
    print(json.dumps({"workload": "SD-1.5 VAE, 512x512 frames, seeded weights, fp16", "card": _card(),
                      "frames_per_call": a.frames, "reps": a.reps,
                      "encode_ms_per_frame": enc_ms, "decode_ms_per_frame": dec_ms,
                      "encode_tflops": enc_fl / (enc_ms * 1e-3) / 1e12, "decode_tflops": dec_fl / (dec_ms * 1e-3) / 1e12,
                      "encode_tflop_per_frame": enc_fl / 1e12, "decode_tflop_per_frame": dec_fl / 1e12}), flush=True)


if __name__ == "__main__":
    main()
