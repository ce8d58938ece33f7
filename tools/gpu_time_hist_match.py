#!/usr/bin/env python
"""Times histogram matching (`need_hist_match`) on the engine: `musev_b200.ops.hist_match` on B = 1, 3 channels, F frames
of 512x512 fp32 matched to one 512x512 template, out of place, CUDA events around --iters calls after --warmup calls,
repeated --reps times (the median is reported). The bytes the op must move follow from the shapes: 4 B read per source
and template pixel by the histogram pass, 4 B read and 4 B written per source pixel by the apply pass; over the engine
time that is a rate, and over 3.35 TB/s (H100 SXM HBM3, data sheet) a share of the HBM bound.

Beside it, the reference's way on the same host: the device-to-host copy of the frames (what the reference's numpy
conversion of the decoded video costs) and the numpy restatement of the reference computation
(oracle/hist_match_oracle.py; a restatement of skimage's algorithm, not skimage itself), host clock.

--profile adds one torch.profiler pass per case with the three kernels' device times. Prints one JSON line with the
card's name and power limit; --out also writes it to a file."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12


def _card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                               str(torch.cuda.current_device())], capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception as e:
        return f"unknown ({e})"


def moved_bytes(B, C, F, hw, hw_t) -> int:
    return 4 * B * C * (F * hw + hw_t) + 8 * B * C * F * hw


def time_engine(video, target, out, warmup, iters, reps):
    from musev_b200 import ops
    for _ in range(warmup):
        ops.hist_match(video, target, out=out)
    torch.cuda.synchronize()
    per_call = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            ops.hist_match(video, target, out=out)
        e1.record()
        e1.synchronize()
        per_call.append(e0.elapsed_time(e1) / iters)
    return statistics.median(per_call), min(per_call), max(per_call)


def profile_kernels(video, target, out):
    from musev_b200 import ops
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            ops.hist_match(video, target, out=out)
        torch.cuda.synchronize()
    ms = {}
    for ev in prof.key_averages():
        if "hist_match" in ev.key:
            name = ev.key.split("hist_match_")[1].split("(")[0].split("<")[0]
            ms[name] = round(ev.device_time_total / 1e3 / 5, 4)     # us -> ms, per call
    return ms


def time_reference_way(video, target, reps):
    from oracle.hist_match_oracle import hist_match_video_bcthw
    d2h, cpu = [], []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        v = video.cpu().numpy()
        t = target.cpu().numpy()
        t1 = time.perf_counter()
        hist_match_video_bcthw(v, t, 255.0)
        t2 = time.perf_counter()
        d2h.append((t1 - t0) * 1e3)
        cpu.append((t2 - t1) * 1e3)
    return statistics.median(d2h), statistics.median(cpu)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, nargs="+", default=[16, 128])
    ap.add_argument("--size", type=int, nargs=2, default=[512, 512])
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ref-reps", type=int, default=1, help="runs of the host-side reference way per case")
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: times are only measured on the GPU")
    H, W = args.size
    B, C = 1, 3
    g = torch.Generator(device="cuda").manual_seed(0)
    res = {"card": _card(), "cases": []}
    for F in args.frames:
        video = (torch.randn(B, C, F, H, W, device="cuda", generator=g) * 0.22 + 0.45).clamp_(0, 1)
        target = (torch.randn(B, C, 1, H, W, device="cuda", generator=g) * 0.22 + 0.45).clamp_(0, 1)
        out = torch.empty_like(video)
        med, lo, hi = time_engine(video, target, out, args.warmup, args.iters, args.reps)
        nbytes = moved_bytes(B, C, F, H * W, H * W)
        case = {"B": B, "C": C, "F": F, "H": H, "W": W, "engine_ms": round(med, 4), "engine_ms_min": round(lo, 4),
                "engine_ms_max": round(hi, 4), "bytes": nbytes, "GB_per_s": round(nbytes / med / 1e6, 1),
                "share_of_3.35TBps": round(nbytes / med / 1e-3 / HBM_BYTES_PER_S, 3)}
        if args.profile:
            case["kernel_ms"] = profile_kernels(video, target, out)
        if args.ref_reps > 0:
            d2h, cpu = time_reference_way(video, target, args.ref_reps)
            case["reference_way"] = {"d2h_ms": round(d2h, 1), "numpy_restatement_ms": round(cpu, 1),
                                     "note": "numpy restatement of the reference algorithm on this host, not skimage"}
        res["cases"].append(case)
        print(json.dumps(case), file=sys.stderr, flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
