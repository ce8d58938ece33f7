"""Times the prompt encoder (CLIP text model, SD-1.5 config, seeded fp16 weights) per call on the engine and as the eager
fp16 oracle with SDPA attention (what transformers runs by default) on the same GPU, alternating the two, best of three
windows. N = 2 is one classifier-free-guidance pair of 77-token chunks, N = 6 three chunks of each. Prints one JSON line
per N: the card's name and power limit, ms per call, launches per call and the engine's per-category kernel time from the
launch profiler, achieved TFLOP/s from musev_b200.flops, and the two data-sheet bounds of the work (the non-embedding fp16
weights read once per call at 3.35 TB/s; the FLOPs at 989 TFLOP/s).

  python tools/gpu_time_clip_text.py [--batch 2 6] [--iters 50]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from musev_b200.flops import clip_text_flops  # noqa: E402
from musev_b200.schema import ClipTextConfig, clip_text_param_shapes  # noqa: E402
from musev_b200.synth import make_clip_text_state_dict, make_input_ids  # noqa: E402
from tools.gpu_time_clip_vision import PEAK_TBS, PEAK_TFLOPS, card, time_ms  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[2, 6])
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from musev_b200 import _capi
    from musev_b200.clip_text import CLIPTextModel
    from oracle.clip_text_oracle import clip_text_forward
    cfg = ClipTextConfig()
    sd = {k: v.half() for k, v in make_clip_text_state_dict(cfg, seed=7).items()}
    m = CLIPTextModel.from_state_dict(sd, cfg, device="cuda", dtype=torch.float16)
    sd_dev = {k: v.cuda() for k, v in sd.items()}
    weight_bytes = sum(2 * torch.Size(s).numel() for n, s in clip_text_param_shapes(cfg).items() if ".embeddings." not in n)
    name, power = card()
    for N in args.batch:
        ids = make_input_ids(N, 77, cfg, seed=5).cuda()
        with torch.no_grad():
            ms_engine, ms_eager = [], []
            for _ in range(3):                                          # alternate, so drift hits both the same way
                ms_engine.append(time_ms(lambda: m(ids), args.iters))
                ms_eager.append(time_ms(lambda: clip_text_forward(sd_dev, cfg, ids, dtype=torch.float16, sdpa=True),
                                        args.iters))
            _capi.profile_enable(True)
            for _ in range(args.iters):
                m(ids)
            prof = _capi.profile_collect()
            _capi.profile_enable(False)
            n0 = _capi.launch_count()
            m(ids)
            torch.cuda.synchronize()
            launches = _capi.launch_count() - n0
            got = m(ids).last_hidden_state.float()
            ref = clip_text_forward(sd_dev, cfg, ids, dtype=torch.float16, sdpa=True)[0].float()
        e, g = min(ms_engine), min(ms_eager)
        flops = clip_text_flops(cfg, N, 77)["total"]
        t_mem, t_cmp = weight_bytes / (PEAK_TBS * 1e12), flops / (PEAK_TFLOPS * 1e12)
        print(json.dumps({
            "gpu": name, "power_limit": power, "model": "CLIP text (SD-1.5)", "sequences": N, "tokens": 77,
            "engine_ms": e, "eager_fp16_sdpa_ms": g, "speedup_vs_eager": g / e,
            "engine_ms_runs": [round(v, 4) for v in ms_engine], "eager_ms_runs": [round(v, 4) for v in ms_eager],
            "launches_per_call": launches,
            "engine_kernel_ms_per_call": {k: round(v["ms"] / args.iters, 4) for k, v in prof.items()},
            "launches_per_call_by_category": {k: v["launches"] // args.iters for k, v in prof.items()},
            "gflop_per_call": flops / 1e9, "engine_tflops": flops / (e * 1e-3) / 1e12,
            "weight_mbytes": weight_bytes / 1e6,
            "bound_us_weights_at_3.35TBs": t_mem * 1e6, "bound_us_flops_at_989TFLOPs": t_cmp * 1e6,
            "bound": "memory" if t_mem > t_cmp else "compute",
            "max_abs_engine_vs_eager_fp16": (got - ref).abs().max().item(), "max_abs_eager": ref.abs().max().item(),
        }), flush=True)


if __name__ == "__main__":
    main()
