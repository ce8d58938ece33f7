"""Times the PoseGuider per 512 x 512 frame on the engine and as eager torch fp16 (the oracle module on cuDNN) on the same
GPU and prints one JSON line: the card's name and power limit, ms per frame, achieved GB/s against a minimum-bytes model
(the image read once, every activation written once and read once, the embedding written once, the weights read once) and
TFLOP/s from musev_b200.flops, with the bound (memory or compute) the H100 SXM data sheet puts on that work.

  python tools/gpu_time_pose_guider.py [--frames 16] [--iters 20] [--config full|narrow]
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
from musev_b200.flops import pose_guider_flops  # noqa: E402
from musev_b200.schema import PoseGuiderConfig, pose_guider_layers  # noqa: E402
from musev_b200.synth import make_pose_guider_state_dict, make_pose_images  # noqa: E402

PEAK_TBS, PEAK_TFLOPS = 3.35, 989.0     # H100 SXM data sheet: HBM3 bandwidth, dense fp16 tensor rate (700 W)


def min_bytes(cfg, N, H, W):
    b = N * cfg.conditioning_channels * H * W * 2                      # the fp16 image, read once
    layers = pose_guider_layers(cfg)
    for i, (_, cin, cout, s) in enumerate(layers):
        H, W = (H - 1) // s + 1, (W - 1) // s + 1
        b += N * cout * H * W * 2 * (1 if i == len(layers) - 1 else 2)   # written once (and read once by the next layer)
        b += (cout * cin * 9) * 2 + cout * 4
    return b


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--config", default="full", choices=["full", "narrow"])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from musev_b200.controlnet import PoseGuider
    from oracle.pose_guider_oracle import PoseGuiderOracle
    cfg = PoseGuiderConfig(320, 3, (16, 32, 96, 256)) if args.config == "full" else PoseGuiderConfig(320, 3, (16, 32, 64, 128))
    N, H, W = args.frames, 512, 512
    sd = {k: v.half() for k, v in make_pose_guider_state_dict(cfg, seed=21).items()}
    pg = PoseGuider(cfg.conditioning_embedding_channels, 3, cfg.block_out_channels, device="cuda", dtype=torch.float16,
                    frames_per_call=N)
    pg.load_state_dict(sd)
    eager = PoseGuiderOracle(cfg, sd, device="cuda", dtype=torch.float16)
    x = make_pose_images(N, H, W, 5).cuda().half()
    torch.backends.cudnn.benchmark = True
    with torch.no_grad():
        ms_engine, ms_eager = [], []
        for _ in range(3):                                              # alternate, so drift hits both the same way
            ms_engine.append(time_ms(lambda: pg.embed_frames(x), args.iters))
            ms_eager.append(time_ms(lambda: eager.frames(x), args.iters))
        out = pg.embed_frames(x).float()
        ref = eager.frames(x).float()
    e, g = min(ms_engine), min(ms_eager)
    flops = pose_guider_flops(cfg, N, H, W)["total"]
    nbytes = min_bytes(cfg, N, H, W)
    t_mem, t_cmp = nbytes / (PEAK_TBS * 1e12), flops / (PEAK_TFLOPS * 1e12)
    name, power = card()
    print(json.dumps({
        "gpu": name, "power_limit": power, "config": list(cfg.block_out_channels), "emb": cfg.conditioning_embedding_channels,
        "frames": N, "size": [H, W],
        "engine_ms_per_frame": e / N, "eager_fp16_ms_per_frame": g / N, "speedup_vs_eager": g / e,
        "engine_ms_runs": [round(v / N, 4) for v in ms_engine], "eager_ms_runs": [round(v / N, 4) for v in ms_eager],
        "gflop_per_frame": flops / N / 1e9, "min_mbytes_per_frame": nbytes / N / 1e6,
        "engine_gbs": nbytes / (e * 1e-3) / 1e9, "engine_tflops": flops / (e * 1e-3) / 1e12,
        "bound": "memory" if t_mem > t_cmp else "compute",
        "engine_share_of_bound": max(t_mem, t_cmp) / (e * 1e-3),
        "max_abs_engine_vs_eager_fp16": (out - ref).abs().max().item(), "max_abs_eager": ref.abs().max().item(),
    }))


if __name__ == "__main__":
    main()
