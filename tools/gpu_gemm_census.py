#!/usr/bin/env python
"""Lists every distinct conv_gemm launch of one config-2 UNet forward (`musev`, CFG batch 2 x (16 + 1) frames, 64x64
latents) and times each one on its own, so that the GEMM time of a forward can be split by shape and compared against
what the hardware could do.

The launch list comes from the library's MVB_TRACE lines: a child process runs the forward with MVB_TRACE set and
reports the distinct launches with their counts, and the GEMM time of that same forward from the library's per-launch
profile (the number `bench.py` reports as `step_share.gemm`, per forward instead of per 20-step denoise). Each entry is
then replayed through `musev_b200.ops.conv_gemm` on seeded inputs of its shape and options (taps, a concatenated
second A source, stride 2, bias, row-add, residual with alpha / beta, GEGLU, activation, fp32 output), warmed up and
timed with CUDA events over back-to-back launches filling at least --seconds. With several libraries (--lib A B ...)
every round times each library in turn so that clock drift and other work on the machine hit all of them alike, and
the outputs of every library are compared bit for bit with the first one's.

Per (library, shape) one JSON line: ms per launch (best of the rounds, and every round), launches per forward,
algorithmic TFLOP/s, the share of the forward's summed GEMM time, and the roofline bound: the larger of the FLOPs at
989 TFLOP/s (H100 SXM data sheet, dense FP16) and the least HBM bytes (A, weights and residual read once, the output
written once) at 3.35 TB/s. Per library a summary line with the summed ms per forward, the profiled GEMM time of the
forward, the card's name and power limit and the median SM clock sampled while the library was timed.

  python tools/gpu_gemm_census.py [--lib old.so new.so] [--rounds 3] [--seconds 1] [--out census.jsonl] [--part 1/2]
"""
from __future__ import annotations

import argparse
import json
import math
import os
import re
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_TFLOPS, PEAK_TBS = 989.0, 3.35
TRACE_RE = re.compile(r"MVB_TRACE gemm (.*)$")
# fields that describe a launch (block_n, tiles and epi are the library's choices, not the launch's)
KEY_FIELDS = ("N", "K", "geglu", "res", "f32", "W", "H", "NF", "c0", "c1", "offsets", "s2", "bias", "rowadd", "rpg",
              "alpha", "beta", "act", "ldc", "ld_res", "res_is_out")


def _parse(line):
    m = TRACE_RE.search(line)
    if not m:
        return None
    kv = dict(x.split("=", 1) for x in m.group(1).split())
    if "res_is_out" not in kv:
        raise SystemExit("the library's MVB_TRACE gemm lines lack the replay fields: capture with this tree's library")
    return kv


def distinct_entries(lines):
    """The distinct launches among MVB_TRACE lines, in first-seen order, each with its count."""
    counts, order = {}, []
    for line in lines:
        kv = _parse(line)
        if kv is None:
            continue
        key = tuple(kv[f] for f in KEY_FIELDS)
        if key not in counts:
            counts[key] = 0
            order.append(key)
        counts[key] += 1
    return [dict(zip(KEY_FIELDS, k), count=counts[k]) for k in order]


def capture_forward(preset: str, batch: int = 2, frames: int = 16, h: int = 64, w: int = 64, warmup: int = 2,
                    profile: bool = True):
    """In a process with MVB_TRACE set: the distinct GEMM launches of one UNet forward of `preset` on synthetic weights
    (batch x (frames + 1 vision-condition frame), h x w latents), and with `profile` the profiled GEMM time of a second
    forward (None otherwise)."""
    from musev_b200 import _capi
    from musev_b200.schema import preset_config
    from musev_b200.synth import make_inputs, make_state_dict
    from musev_b200.unet import UNet3DConditionModel
    dev = "cuda"
    cfg = preset_config(preset)
    m = UNet3DConditionModel(cfg, device=dev, dtype=torch.float16)
    m.load_state_dict(make_state_dict(cfg, seed=0, dtype=torch.float16))
    inp = make_inputs(cfg, batch=batch, frames=frames, h=h, w=w, n_vis_cond=1)
    kw = dict(sample_index=inp["sample_index"], vision_conditon_frames_sample_index=inp["vision_conditon_frames_sample_index"],
              sample_frame_rate=8)
    for k in ("down_block_refer_embs", "mid_block_refer_emb", "vision_clip_emb"):
        if k in inp:
            kw[k] = [x.half().to(dev) for x in inp[k]] if isinstance(inp[k], list) else inp[k].half().to(dev)
    x, enc = inp["sample"].half().to(dev), inp["encoder_hidden_states"].half().to(dev)
    prof = None
    sys.stderr.flush()
    saved = os.dup(2)
    with tempfile.TemporaryFile(mode="w+") as log:
        devnull = os.open(os.devnull, os.O_WRONLY)
        try:
            os.dup2(devnull, 2)                      # warm-up forwards: trace lines discarded
            for _ in range(warmup):
                m(x, 601, enc, **kw)
            torch.cuda.synchronize()
            os.dup2(log.fileno(), 2)                 # the traced forward
            m(x, 601, enc, **kw)
            torch.cuda.synchronize()
            os.dup2(devnull, 2)
            if profile:
                _capi.profile_enable(True)           # the profiled forward (same launches)
                m(x, 601, enc, **kw)
                prof = _capi.profile_collect()
                _capi.profile_enable(False)
        finally:
            os.dup2(saved, 2)
            os.close(saved)
            os.close(devnull)
        log.seek(0)
        lines = log.read().splitlines()
    del m
    torch.cuda.empty_cache()
    return distinct_entries(lines), prof


def capture(preset: str) -> None:
    """Child process (MVB_TRACE set): one forward's distinct GEMM launches and its profiled GEMM time, as JSON on stdout."""
    entries, prof = capture_forward(preset)
    print(json.dumps({"entries": entries, "profiled_gemm_ms": prof["gemm"]["ms"], "profiled_gemm_launches": prof["gemm"]["launches"]}))


def make_case(e, dev, g):
    """Seeded operands of one entry: the ops.conv_gemm keyword arguments, and (flops, least HBM bytes)."""
    W, H, NF, c0, c1, N, K = (int(e[k]) for k in ("W", "H", "NF", "c0", "c1", "N", "K"))
    s2 = int(e["s2"])
    geglu, f32 = int(e["geglu"]), int(e["f32"])
    M = W * H * NF
    Wi, Hi = (2 * W, 2 * H) if s2 else (W, H)

    def rnd(*shape, scale=1.0):
        return (torch.randn(*shape, generator=g) * scale).half().to(dev)

    a0 = rnd(NF, Hi, Wi, c0)
    kw = dict(a0=a0, weight=rnd(N, K, scale=1.0 / math.sqrt(K)))
    if s2:
        kw["stride2"] = s2
    else:
        kw["taps"] = tuple(tuple(int(v) for v in t.split(":")) for t in e["offsets"].split(","))
    if c1:
        kw["a1"] = rnd(NF, H, W, c1)
    if int(e["bias"]):
        kw["bias"] = torch.randn(N, generator=g).float().to(dev) * 0.1
    if int(e["rowadd"]):
        rpg = int(e["rpg"])
        kw["rowadd"] = torch.randn((M + rpg - 1) // rpg, N, generator=g).float().to(dev) * 0.1
        kw["rows_per_group"] = rpg
    nout = N // 2 if geglu else N
    if int(e["res"]):
        kw["residual"] = rnd(M, max(int(e["ld_res"]), nout))[:, :nout]   # the engine's row stride
    kw.update(alpha=float(e["alpha"]), beta=float(e["beta"]), geglu=bool(geglu), act=int(e["act"]), out_f32=bool(f32))
    flops = 2.0 * M * N * K
    nbytes = (NF * Hi * Wi * c0 + M * c1) * 2 + N * K * 2 + M * nout * (4 if f32 else 2) + (M * nout * 2 if int(e["res"]) else 0)
    return kw, flops, nbytes, (M, nout)


def make_out(e, kw, dev):
    """The output of one entry's replay as the engine passed it: the residual itself (res_is_out), or a [M, ldc] buffer
    whose leading columns are the output."""
    if int(e["res_is_out"]):
        return kw["residual"]
    M, nout = int(e["W"]) * int(e["H"]) * int(e["NF"]), int(e["N"]) // (2 if int(e["geglu"]) else 1)
    buf = torch.zeros(M, max(int(e["ldc"]), nout), dtype=torch.float32 if int(e["f32"]) else torch.float16, device=dev)
    return buf[:, :nout]


def _bits_equal(a, b):
    it = torch.int16 if a.dtype == torch.float16 else torch.int32
    return bool(torch.equal(a.view(it), b.view(it)))


def use_lib(path):
    from musev_b200 import _capi
    from tools.gpu_compare_builds import _TolerantLib
    lib = _TolerantLib(os.path.abspath(path))
    _capi._declare(lib)
    _capi._lib = lib


def time_case(kw, out, seconds):
    """ms per launch over >= `seconds` of back-to-back launches."""
    from musev_b200 import ops

    def launch():
        ops.conv_gemm(out=out, **kw)

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
    e0.record()
    for _ in range(iters):
        launch()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--capture", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--preset", default="musev")
    ap.add_argument("--lib", nargs="+", default=None, help="libmusevb200.so builds to time, alternated (default: the in-tree one)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--seconds", type=float, default=1.0, help="least timed time per shape, library and round")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    ap.add_argument("--part", default="1/1", help="K/N: time only every N-th shape from the K-th (a census split over "
                                                  "several runs; the summary then sums that part)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    if args.capture:
        capture(args.preset)
        return
    from bench import ClockSampler
    from musev_b200 import build
    from tools.gpu_time_clip_vision import card
    env = dict(os.environ, MVB_TRACE="1")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--capture", "--preset", args.preset], env=env,
                       capture_output=True, text=True)
    if r.returncode != 0:
        raise SystemExit(f"capture failed:\n{r.stderr[-4000:]}")
    cap = json.loads(r.stdout.strip().splitlines()[-1])
    k, n = (int(v) for v in args.part.split("/"))
    entries = cap["entries"][k - 1::n]
    libs = args.lib or [build.LIB_PATH]
    dev = torch.device("cuda", torch.cuda.current_device())
    name, power = card()
    g = torch.Generator().manual_seed(5)
    cases = [make_case(e, dev, g) for e in entries]
    outs = {(lib, i): torch.zeros(*c[3], dtype=torch.float32 if c[0]["out_f32"] else torch.float16, device=dev)
            for lib in libs for i, c in enumerate(cases)}
    ms = {key: [] for key in outs}
    mhz = {lib: [] for lib in libs}
    for _ in range(args.rounds):
        for lib in libs:
            use_lib(lib)
            sampler = ClockSampler(dev.index)
            sampler.start()
            for i, c in enumerate(cases):
                ms[(lib, i)].append(time_case(c[0], outs[(lib, i)], args.seconds))
            sampler.stop_flag = True
            sampler.join()
            s = sampler.summary()
            if s["sm_mhz"]:
                mhz[lib].append(s["sm_mhz"])
            mhz.setdefault(("reasons", lib), set()).update(s["reasons"])
    lines = []
    for lib in libs:
        rel = os.path.relpath(os.path.abspath(lib), ROOT)
        total = sum(min(ms[(lib, i)]) * e["count"] for i, e in enumerate(entries))
        for i, (e, c) in enumerate(zip(entries, cases)):
            best = min(ms[(lib, i)])
            _, flops, nbytes, _ = c
            bound_ms = max(flops / (PEAK_TFLOPS * 1e12), nbytes / (PEAK_TBS * 1e12)) * 1e3
            lines.append({
                "lib": rel, "shape": {k: e[k] for k in KEY_FIELDS}, "launches_per_forward": e["count"],
                "ms": best, "ms_runs": [round(v, 5) for v in ms[(lib, i)]],
                "tflops": flops / (best * 1e-3) / 1e12, "share_of_forward_gemm": best * e["count"] / total,
                "roofline_ms": bound_ms, "roofline_bound": "tensor" if flops / PEAK_TFLOPS > nbytes / PEAK_TBS * 1e3 else "hbm",
                "equal_to_first_lib": _bits_equal(outs[(lib, i)], outs[(libs[0], i)]),
            })
        clk = sorted(mhz[lib])[len(mhz[lib]) // 2] if mhz[lib] else None
        lines.append({
            "summary": True, "part": args.part, "lib": rel, "gpu": name, "power_limit": power, "sm_mhz_median": clk,
            "clock_event_reasons": sorted(mhz.get(("reasons", lib), set())),
            "distinct_shapes": len(entries), "launches_per_forward": sum(e["count"] for e in entries),
            "summed_ms_per_forward": total,
            "roofline_ms_per_forward": sum(max(c[1] / (PEAK_TFLOPS * 1e12), c[2] / (PEAK_TBS * 1e12)) * 1e3 * e["count"]
                                           for e, c in zip(entries, cases)),
            "profiled_gemm_ms_per_forward_in_tree_lib": cap["profiled_gemm_ms"],
            "profiled_gemm_launches": cap["profiled_gemm_launches"],
        })
    fh = open(args.out, "w") if args.out else None
    for ln in lines:
        s = json.dumps(ln)
        print(s, flush=True)
        if fh:
            fh.write(s + "\n")
    if fh:
        fh.close()


if __name__ == "__main__":
    main()
