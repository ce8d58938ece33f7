#!/usr/bin/env python
"""Times the per-frame tail of a long video, VAE decode and encode, on one GPU and sharded over N:
`torchrun --nproc-per-node N tools/gpu_time_frames_sharded.py` (N = 1 gives the single-GPU numbers alone).

SD-1.5 VAE with seeded weights, fp16, frames_per_call 4, b = 1, `--frames` frames (128 and 512) at 512x512 and 512x768.
Per case, `decode_latents` and `encode_video` run once to warm up (workspace growth), then `--reps` timed calls: without
a group on every rank at once (the single-GPU time), and with N > 1 also with `process_group=WORLD`, the row exchange
included. A call is timed by the host clock from a barrier to a device synchronise; a sharded call counts as long as
its slowest rank. The sharded output is checked bit-equal to the unsharded one. Rank 0 prints one JSON line per case
with the median times and the card's name and power limit. Writes nothing to disk."""
import argparse
import datetime
import json
import os
import statistics
import subprocess
import sys
import time

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
    ap.add_argument("--frames", type=int, nargs="+", default=[128, 512])
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    import torch.distributed as dist
    from musev_b200.schema import VAEConfig
    from musev_b200.synth import make_state_dict, make_vae_images
    from musev_b200.vae import AutoencoderKL
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    group = None
    if world > 1:
        dist.init_process_group("nccl", device_id=dev, timeout=datetime.timedelta(seconds=600))
        group = dist.group.WORLD
    rank = dist.get_rank() if group is not None else 0
    cfg = VAEConfig()
    vae = AutoencoderKL(cfg, device=dev, dtype=torch.float16, frames_per_call=4)
    vae.load_state_dict(make_state_dict(cfg, seed=11, dtype=torch.float16))

    def timed(fn, pg):
        torch.cuda.synchronize()
        if group is not None:
            dist.barrier(device_ids=[local])
        t0 = time.perf_counter()
        out = fn(pg)
        torch.cuda.synchronize()
        dt = torch.tensor([time.perf_counter() - t0], dtype=torch.float64, device=dev)
        if pg is not None:
            dist.all_reduce(dt, op=dist.ReduceOp.MAX, group=pg)
        return out, dt.item() * 1e3

    for H, W in ((512, 512), (512, 768)):
        for f in a.frames:
            video = make_vae_images(f, H, W, seed=5).half().to(dev).permute(1, 0, 2, 3)[None]        # [1, 3, f, H, W]
            latents = (torch.randn(1, 4, f, H // 8, W // 8, generator=torch.Generator().manual_seed(6)) * 0.18215).half().to(dev)
            for stage, fn in (("decode_latents", lambda pg: vae.decode_latents(latents, process_group=pg)),
                              ("encode_video", lambda pg: vae.encode_video(video, process_group=pg))):
                modes = [None] + ([group] if group is not None else [])
                res = {}
                for pg in modes:
                    one = fn(pg)                                                               # warm-up
                    ms = []
                    for _ in range(a.reps):
                        one, t = timed(fn, pg)
                        ms.append(t)
                    res[pg is not None] = (one, ms)
                    del one
                rec = {"stage": stage, "frames": f, "size": f"{H}x{W}", "ranks": world, "reps": a.reps,
                       "single_gpu_ms": statistics.median(res[False][1]), "single_gpu_ms_all": res[False][1]}
                if group is not None:
                    assert torch.equal(res[True][0], res[False][0]), (stage, f, H, W)
                    rec.update(sharded_ms=statistics.median(res[True][1]), sharded_ms_all=res[True][1],
                               speedup=rec["single_gpu_ms"] / statistics.median(res[True][1]), bit_equal=True)
                res.clear()
                if rank == 0:
                    rec.update(workload="SD-1.5 VAE, seeded weights, fp16, frames_per_call 4", card=_card())
                    print(json.dumps(rec), flush=True)
            del video, latents
            torch.cuda.empty_cache()
    if group is not None:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
