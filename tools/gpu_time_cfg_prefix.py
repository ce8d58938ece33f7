#!/usr/bin/env python
"""Times one UNet forward at the config-2 shape (CFG batch 2 with equal sample halves, 16 + 1 frames, 64 x 64 latents,
full width, fp16) with and without `cfg_shared_sample`, in one process: rounds of N forwards alternate between the two
(CUDA events around each round), so the difference is the saving of running the shared prefix once. Checks that both
give the same bits, and prints the card, its power limit and the SM clock sampled after the timing."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--preset", default="musev")
    ap.add_argument("--iters", type=int, default=5, help="forwards per round")
    ap.add_argument("--rounds", type=int, default=4, help="rounds per setting, alternated")
    a = ap.parse_args()
    from musev_b200 import _capi
    from musev_b200.schema import preset_config
    from musev_b200.synth import make_inputs, make_state_dict
    from musev_b200.unet import UNet3DConditionModel
    dev = "cuda"
    cfg = preset_config(a.preset)
    m = UNet3DConditionModel(cfg, device=dev, dtype=torch.float16)
    m.load_state_dict(make_state_dict(cfg, seed=0, dtype=torch.float16))
    inp = make_inputs(cfg, batch=2, frames=16, h=64, w=64, n_vis_cond=1)
    kw = dict(sample_index=inp["sample_index"], vision_conditon_frames_sample_index=inp["vision_conditon_frames_sample_index"], sample_frame_rate=8)
    for k in ("vision_clip_emb",):
        if k in inp:
            kw[k] = inp[k].half().to(dev)
    s = inp["sample"].half()
    x, enc = torch.cat([s[:1], s[:1]]).to(dev), inp["encoder_hidden_states"].half().to(dev)

    def fwd(shared):
        return m(x, 601, enc, cfg_shared_sample=shared, **kw).sample

    same = torch.equal(fwd(False).clone(), fwd(True).clone())
    for shared in (False, True):
        for _ in range(2):
            fwd(shared)
    torch.cuda.synchronize()
    ms = {False: [], True: []}
    launches = {}
    for _ in range(a.rounds):
        for shared in (False, True):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            n0 = _capi.launch_count()
            e0.record()
            for _ in range(a.iters):
                fwd(shared)
            e1.record()
            torch.cuda.synchronize()
            ms[shared].append(e0.elapsed_time(e1) / a.iters)
            launches[shared] = (_capi.launch_count() - n0) // a.iters
    split = {}
    for shared in (False, True):
        _capi.profile_enable(True)
        fwd(shared)
        prof = _capi.profile_collect()
        _capi.profile_enable(False)
        split[shared] = {k: round(v["ms"], 2) for k, v in prof.items()}
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    med = {k: statistics.median(v) for k, v in ms.items()}
    print("CFG_PREFIX " + json.dumps({
        "preset": a.preset, "bit_identical": same, "card": card,
        "forward_ms": {"unflagged": [round(v, 3) for v in ms[False]], "flagged": [round(v, 3) for v in ms[True]]},
        "median_ms": {"unflagged": round(med[False], 3), "flagged": round(med[True], 3)},
        "saving_ms": round(med[False] - med[True], 3),
        "launches_per_forward": {"unflagged": launches[False], "flagged": launches[True]},
        "split_ms": {"unflagged": split[False], "flagged": split[True]}}), flush=True)


if __name__ == "__main__":
    main()
