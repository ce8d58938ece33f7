"""Times the IP-Adapter image encoder (CLIP ViT-H/14 + visual projection, seeded fp16 weights) per call on the engine and as
the eager fp16 oracle with SDPA attention (what transformers runs by default) on the same GPU, alternating the two, best of
three windows. Prints one JSON line per batch size: the card's name and power limit, ms per call, the engine's per-category
kernel time from the launch profiler, achieved TFLOP/s from musev_b200.flops, and the two data-sheet bounds of the work
(the fp16 weights read once per call at 3.35 TB/s; the FLOPs at 989 TFLOP/s).

  python tools/gpu_time_clip_vision.py [--batch 1 4] [--iters 20]
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
from musev_b200.flops import clip_vision_flops  # noqa: E402
from musev_b200.schema import ClipVisionConfig, clip_vision_param_shapes  # noqa: E402
from musev_b200.synth import make_clip_pixel_values, make_clip_vision_state_dict  # noqa: E402

PEAK_TBS, PEAK_TFLOPS = 3.35, 989.0     # H100 SXM data sheet: HBM3 bandwidth, dense fp16 tensor rate (700 W)


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
    ap.add_argument("--batch", type=int, nargs="+", default=[1, 4])
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from musev_b200 import _capi
    from musev_b200.clip_vision import CLIPVisionModelWithProjection
    from oracle.clip_vision_oracle import clip_vision_forward
    cfg = ClipVisionConfig()
    sd = {k: v.half() for k, v in make_clip_vision_state_dict(cfg, seed=7).items()}
    m = CLIPVisionModelWithProjection.from_state_dict(sd, cfg, device="cuda", dtype=torch.float16)
    sd_dev = {k: v.cuda() for k, v in sd.items()}
    weight_bytes = sum(2 * torch.Size(s).numel() for s in clip_vision_param_shapes(cfg).values())
    name, power = card()
    for N in args.batch:
        x = make_clip_pixel_values(N, cfg.image_size, seed=5).cuda().half()
        with torch.no_grad():
            ms_engine, ms_eager = [], []
            for _ in range(3):                                          # alternate, so drift hits both the same way
                ms_engine.append(time_ms(lambda: m(x), args.iters))
                ms_eager.append(time_ms(lambda: clip_vision_forward(sd_dev, cfg, x, dtype=torch.float16, sdpa=True),
                                        args.iters))
            _capi.profile_enable(True)
            for _ in range(args.iters):
                m(x)
            prof = _capi.profile_collect()
            _capi.profile_enable(False)
            got = m(x).image_embeds.float()
            ref = clip_vision_forward(sd_dev, cfg, x, dtype=torch.float16, sdpa=True)[0].float()
        e, g = min(ms_engine), min(ms_eager)
        flops = clip_vision_flops(cfg, N)["total"]
        t_mem, t_cmp = weight_bytes / (PEAK_TBS * 1e12), flops / (PEAK_TFLOPS * 1e12)
        print(json.dumps({
            "gpu": name, "power_limit": power, "model": "CLIP ViT-H/14 + projection", "images": N, "size": cfg.image_size,
            "engine_ms": e, "eager_fp16_sdpa_ms": g, "speedup_vs_eager": g / e,
            "engine_ms_runs": [round(v, 4) for v in ms_engine], "eager_ms_runs": [round(v, 4) for v in ms_eager],
            "engine_kernel_ms_per_call": {k: round(v["ms"] / args.iters, 4) for k, v in prof.items()},
            "launches_per_call": {k: v["launches"] // args.iters for k, v in prof.items()},
            "tflop_per_call": flops / 1e12, "engine_tflops": flops / (e * 1e-3) / 1e12,
            "weight_gbytes": weight_bytes / 1e9,
            "bound_ms_weights_at_3.35TBs": t_mem * 1e3, "bound_ms_flops_at_989TFLOPs": t_cmp * 1e3,
            "bound": "memory" if t_mem > t_cmp else "compute",
            "engine_share_of_bound": max(t_mem, t_cmp) / (e * 1e-3),
            "max_abs_engine_vs_eager_fp16": (got - ref).abs().max().item(), "max_abs_eager": ref.abs().max().item(),
        }), flush=True)


if __name__ == "__main__":
    main()
