"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/clip_vision_{narrow,full}.pt by running the UNMODIFIED
`transformers.CLIPVisionModelWithProjection` (eager attention, CPU fp32) on seeded weights and pixel values.

transformers is third-party arithmetic (the reference pins transformers==4.33.1, requirements.txt:15); it is pinned here by
executing it in the build container. Run there only:  python -m oracle.make_golden_clip_vision
Weights and inputs are regenerated from the seeds in each fixture's meta (musev_b200.synth, bit-identical CPU RNG).
"""
from __future__ import annotations

import os
import sys
import time
from dataclasses import asdict

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from musev_b200.schema import ClipVisionConfig, clip_vision_param_shapes  # noqa: E402
from musev_b200.synth import make_clip_pixel_values, make_clip_vision_state_dict  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
NARROW = {
    "gelu_d64": ClipVisionConfig(hidden_size=128, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2,
                                 image_size=56, patch_size=14, projection_dim=64, hidden_act="gelu"),
    # head dim 40 is stored padded to 48; 8 heads, since the hidden size must be a multiple of 64 (conv_gemm K)
    "quick_gelu_d40": ClipVisionConfig(hidden_size=320, intermediate_size=640, num_hidden_layers=2, num_attention_heads=8,
                                       image_size=56, patch_size=14, projection_dim=64, hidden_act="quick_gelu"),
}
FULL = ClipVisionConfig()            # the IP-Adapter SD-1.5 image encoder (ViT-H/14)
FULL_ROWS = [0, 1, 128, 256]         # token rows of last_hidden_state kept in the full fixture


def run_transformers(cfg: ClipVisionConfig, sd, pixel_values):
    import transformers
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection
    tc = CLIPVisionConfig(**asdict(cfg))
    m = CLIPVisionModelWithProjection(tc)
    m.config._attn_implementation = "eager"
    m.eval()
    ref_shapes = {k: tuple(v.shape) for k, v in m.state_dict().items() if not k.endswith("position_ids")}
    assert ref_shapes == dict(clip_vision_param_shapes(cfg)), "CLIP vision schema mismatch"
    res = m.load_state_dict(sd, strict=False)
    assert not res.missing_keys and all(k.endswith("position_ids") for k in res.unexpected_keys), res
    with torch.no_grad():
        out = m(pixel_values=pixel_values)
    return out.image_embeds.clone(), out.last_hidden_state.clone(), transformers.__version__


def golden(tag, cfgs, n=2, wseed=7, iseed=3131, rows=None):
    entries = {}
    version = None
    for name, cfg in cfgs.items():
        t0 = time.time()
        sd = make_clip_vision_state_dict(cfg, seed=wseed)
        x = make_clip_pixel_values(n, cfg.image_size, seed=iseed)
        emb, last, version = run_transformers(cfg, sd, x)
        entries[name] = dict(config=asdict(cfg), image_embeds=emb,
                             last_hidden_state=last if rows is None else last[:, rows].clone())
        print(f"{tag}/{name}: image_embeds std {emb.std().item():.4f}, last_hidden_state max|.| "
              f"{last.abs().max().item():.3f} ({time.time() - t0:.1f}s)", flush=True)
    meta = dict(n=n, weight_seed=wseed, input_seed=iseed, rows=rows, transformers_version=version,
                source="transformers.CLIPVisionModelWithProjection (attn_implementation eager), CPU fp32")
    path = os.path.join(GOLDEN, f"clip_vision_{tag}.pt")
    torch.save({"meta": meta, "configs": entries}, path)
    print(path, os.path.getsize(path), "bytes", flush=True)


if __name__ == "__main__":
    os.makedirs(GOLDEN, exist_ok=True)
    torch.set_num_threads(os.cpu_count() or 1)
    golden("narrow", NARROW)
    golden("full", {"vit_h14": FULL}, rows=FULL_ROWS)
