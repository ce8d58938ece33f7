#!/usr/bin/env python
"""Times the LoRA merge on the engine: a seeded rank-64 kohya LoRA on every matrix and 4-D convolution of the SD-1.5
`musev_referencenet` UNet, applied (`update_pipeline_lora_model`, one `mvb_unet_merge_lora` call) and unloaded
(`unload_lora`), each call synchronous, host clock around `--reps` calls after one warm-up pair. For comparison it times
today's alternative, a full `load_state_dict` of the fp16 weights from device tensors. Prints one JSON line with the
card's name and power limit, ms per apply / unload, the packed weight bytes the merge reads and writes, and the GB/s that
implies. Writes nothing to disk."""
import argparse
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                               str(torch.cuda.current_device())], capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception as e:
        return f"unknown ({e})"


def packed_bytes(cfg, names) -> int:
    """fp16 bytes of the packed rows x columns the merge visits (the packer's head padding and conv_in / conv_out padding
    included), once read and once written."""
    from musev_b200.schema import unet_param_shapes
    shapes = unet_param_shapes(cfg)
    total = 0
    for n in names:
        s = shapes[n]
        rows, cols = s[0], 1
        for v in s[1:]:
            cols *= v
        if n.endswith((".to_q.weight", ".to_k.weight", ".to_v.weight", ".to_k_ip.weight", ".to_v_ip.weight")):
            d = rows // cfg.heads
            rows = cfg.heads * ((d + 15) // 16 * 16)
        if n == "conv_in.weight":
            cols = 64
        if n == "conv_out.weight":
            rows = 16
        total += rows * cols * 2
    return 2 * total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rank", type=int, default=64)
    a = ap.parse_args()
    from musev_b200 import lora
    from musev_b200.schema import preset_config, unet_param_shapes
    from musev_b200.synth import make_lora_state_dict, make_state_dict
    from musev_b200.unet import UNet3DConditionModel
    dev = "cuda"
    cfg = preset_config("musev_referencenet")
    sd16 = {k: v.to(dev) for k, v in make_state_dict(cfg, seed=0, dtype=torch.float16).items()}
    model = UNet3DConditionModel(cfg, device=dev)
    model.load_state_dict(sd16)
    targets = [n for n, s in unet_param_shapes(cfg).items() if len(s) in (2, 4)]
    lsd = {k: v.to(dev) for k, v in make_lora_state_dict(cfg, targets, rank=a.rank, seed=9).items()}
    pipe = SimpleNamespace(unet=model, text_encoder=None)

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, r

    _, (_, undo) = timed(lambda: lora.update_pipeline_lora_model(pipe, lsd, alpha=1.0, need_unload=True))
    lora.unload_lora(undo)
    apply_s, unload_s = [], []
    for _ in range(a.reps):
        s, (_, undo) = timed(lambda: lora.update_pipeline_lora_model(pipe, lsd, alpha=1.0, need_unload=True))
        apply_s.append(s)
        s, _ = timed(lambda: lora.unload_lora(undo))
        unload_s.append(s)
    # the engine call alone (factors already on the device, host-side parsing done): one mvb_unet_merge_lora each way
    args = ([u["name"] for u in undo], [u["up"] for u in undo], [u["down"] for u in undo], [u["scale"] for u in undo])
    call_s = []
    for _ in range(a.reps):
        call_s.append(timed(lambda: model._merge_lora(*args, subtract=False))[0])
        call_s.append(timed(lambda: model._merge_lora(*args, subtract=True))[0])
    load_s = [timed(lambda: model.load_state_dict(sd16))[0] for _ in range(max(2, a.reps // 2))]
    nbytes = packed_bytes(cfg, targets)
    apply_ms, unload_ms = 1e3 * min(apply_s), 1e3 * min(unload_s)
    print(json.dumps({"workload": f"SD-1.5 musev_referencenet UNet, rank-{a.rank} LoRA on every matrix and 4-D conv",
                      "card": _card(), "targets": len(targets), "reps": a.reps,
                      "apply_ms": apply_ms, "unload_ms": unload_ms,
                      "apply_ms_median": 1e3 * sorted(apply_s)[len(apply_s) // 2],
                      "unload_ms_median": 1e3 * sorted(unload_s)[len(unload_s) // 2],
                      "packed_bytes_read_and_written": nbytes,
                      "apply_gbps": nbytes / (apply_ms * 1e-3) / 1e9, "unload_gbps": nbytes / (unload_ms * 1e-3) / 1e9,
                      "engine_call_ms": 1e3 * min(call_s), "engine_call_gbps": nbytes / min(call_s) / 1e9,
                      "load_state_dict_ms": 1e3 * min(load_s)}), flush=True)


if __name__ == "__main__":
    main()
