#!/usr/bin/env python
"""Times the spatial attention op (`ops.attention`, `attention_kernel`) at the shapes the config-2 UNet forward runs it
(CFG batch 2 x (16 + 1) frames = 34 frames, 8 heads, seeded fp16 inputs laid out as the engine lays them out):

  self_64x64   reference-only self attention at 64x64 latents: 4096 queries, 4096 own-frame + 4096 vision-condition
               keys, d 40 (padded to 48)
  cross_64x64  text cross attention at 64x64: 4096 queries, 77 keys, d 40
  self_32x32   self attention at 32x32: 1024 queries, 1024 + 1024 keys, d 80
  self_16x16   self attention at 16x16: 256 queries, 256 + 256 keys, d 160

Each shape is warmed up, then timed with CUDA events over enough back-to-back launches to fill at least --seconds. With
several libraries (--lib A B ...) every round times each library in turn, so that drift in clocks or in other work on the
machine hits all of them alike; outputs of every library are compared bit for bit with the first one's. One JSON line per
(library, shape): the card's name and power limit, ms per launch (best and every round), algorithmic TFLOP/s (4 d FLOP
per score element: the unpadded head dim), and score elements per SM clock (median SM clock sampled during the timing).

  python tools/gpu_time_attention.py [--lib old.so new.so] [--rounds 3] [--seconds 1] [--shapes self_64x64 ...]
"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import ClockSampler  # noqa: E402
from tools.gpu_compare_builds import _TolerantLib  # noqa: E402
from tools.gpu_time_clip_vision import card  # noqa: E402

NF, T, HEADS, N_TEXT = 34, 17, 8, 77      # CFG batch 2 x (16 window frames + 1 vision-condition frame)

# name: (Nq, d, dp, self attention with the vision-condition segment or text cross attention)
SHAPES = {
    "self_64x64": (4096, 40, 48, "self"),
    "cross_64x64": (4096, 40, 48, "cross"),
    "self_32x32": (1024, 80, 80, "self"),
    "self_16x16": (256, 160, 160, "self"),
}


def _head_padded(rows, heads, d, dp, g):
    x = torch.zeros(rows, heads, dp, dtype=torch.float16)
    x[:, :, :d] = torch.randn(rows, heads, d, generator=g).half()
    return x.reshape(rows, heads * dp)


def make_case(name, dev):
    """The op's arguments for one shape, laid out as the engine lays them out (engine_fwd.cuh) (fused q / k / v rows for self attention,
    q plus fused k / v of the B text sequences for cross attention). Returns (q, segs, Nq, d, dp, keys per query)."""
    Nq, d, dp, kind = SHAPES[name]
    hd = HEADS * dp
    g = torch.Generator().manual_seed(11)
    M = NF * Nq
    if kind == "self":
        qkv = torch.cat([_head_padded(M, HEADS, d, dp, g) for _ in range(3)], dim=1).to(dev)
        q, k, v = qkv[:, :hd], qkv[:, hd:2 * hd], qkv[:, 2 * hd:]
        # own frame, then the batch's vision-condition frame (frame 0 of each T-frame batch row)
        segs = [dict(k=k, v=v, nk=Nq, fdiv=1, fmul=Nq, fadd=0), dict(k=k, v=v, nk=Nq, fdiv=T, fmul=T * Nq, fadd=0)]
        return q, segs, Nq, d, dp, 2 * Nq
    q = _head_padded(M, HEADS, d, dp, g).to(dev)
    kv = torch.cat([_head_padded(2 * N_TEXT, HEADS, d, dp, g) for _ in range(2)], dim=1).to(dev)
    segs = [dict(k=kv[:, :hd], v=kv[:, hd:], nk=N_TEXT, fdiv=T, fmul=N_TEXT, fadd=0)]
    return q, segs, Nq, d, dp, N_TEXT


def use_lib(path):
    from musev_b200 import _capi
    lib = _TolerantLib(os.path.abspath(path))
    _capi._declare(lib)
    _capi._lib = lib


def time_case(case, out, seconds):
    """ms per launch over >= `seconds` of back-to-back launches, and the median SM clock (MHz) while they ran."""
    from musev_b200 import ops
    q, segs, Nq, d, dp, _ = case

    def launch():
        ops.attention(q, segs, NF, Nq, HEADS, d, dp, 1.0 / math.sqrt(d), out=out)

    for _ in range(3):                                        # module load, tensor-map encode, clocks up
        launch()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        launch()
    e1.record()
    torch.cuda.synchronize()
    iters = max(10, math.ceil(seconds * 1e3 / (e0.elapsed_time(e1) / 5)))
    sampler = ClockSampler(torch.cuda.current_device())
    sampler.start()
    e0.record()
    for _ in range(iters):
        launch()
    e1.record()
    torch.cuda.synchronize()
    sampler.stop_flag = True
    sampler.join()
    return e0.elapsed_time(e1) / iters, sampler.summary()["sm_mhz"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", nargs="+", default=None, help="libmusevb200.so builds to time, alternated (default: the in-tree one)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--seconds", type=float, default=1.0, help="least timed time per shape, library and round")
    ap.add_argument("--shapes", nargs="+", default=list(SHAPES), choices=list(SHAPES))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from musev_b200 import build
    libs = args.lib or [build.LIB_PATH]
    dev = torch.device("cuda", torch.cuda.current_device())
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    name, power = card()
    cases = {s: make_case(s, dev) for s in args.shapes}
    outs = {(lib, s): torch.zeros(NF * cases[s][2], HEADS * cases[s][3], dtype=torch.float16, device=dev)
            for lib in libs for s in args.shapes}
    ms = {key: [] for key in outs}
    mhz = {key: [] for key in outs}
    for _ in range(args.rounds):
        for lib in libs:
            use_lib(lib)
            for s in args.shapes:
                t, clk = time_case(cases[s], outs[(lib, s)], args.seconds)
                ms[(lib, s)].append(t)
                if clk:
                    mhz[(lib, s)].append(clk)
    for lib in libs:
        for s in args.shapes:
            _, _, Nq, d, dp, nk = cases[s]
            elems = NF * HEADS * Nq * nk                        # score elements per launch
            best = min(ms[(lib, s)])
            clk = sorted(mhz[(lib, s)])[len(mhz[(lib, s)]) // 2] if mhz[(lib, s)] else None
            print(json.dumps({
                "gpu": name, "power_limit": power, "lib": os.path.relpath(os.path.abspath(lib), ROOT), "shape": s,
                "NF": NF, "heads": HEADS, "Nq": Nq, "keys": nk, "d": d, "dp": dp,
                "ms": best, "ms_runs": [round(v, 4) for v in ms[(lib, s)]],
                "tflops": 4 * d * elems / (best * 1e-3) / 1e12,
                "sm_mhz_median": clk,
                "elements_per_clk_per_sm": elems / (best * 1e-3) / (sms * clk * 1e6) if clk else None,
                "equal_to_first_lib": bool(torch.equal(outs[(lib, s)].view(torch.int16), outs[(libs[0], s)].view(torch.int16))),
            }), flush=True)


if __name__ == "__main__":
    main()
