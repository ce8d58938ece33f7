"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/clip_text_{narrow,full}.pt by running the UNMODIFIED
`transformers.CLIPTextModel` (eager attention, CPU fp32) on seeded weights and input ids.

transformers is third-party arithmetic (the reference pins transformers==4.33.1, requirements.txt:15); it is pinned here by
executing it in the build container. Run there only:  python -m oracle.make_golden_clip_text
Weights and ids are regenerated from the seeds in each fixture's meta (musev_b200.synth, bit-identical CPU RNG); the
fixtures hold outputs only.
"""
from __future__ import annotations

import os
import sys
import time
from dataclasses import asdict

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from musev_b200.schema import ClipTextConfig, clip_text_param_shapes  # noqa: E402
from musev_b200.synth import make_clip_text_state_dict, make_input_ids  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
NARROW = {
    # legacy pooling (argmax of the ids), d = 64, one 77-row tile
    "a_quick_gelu_d64": (ClipTextConfig(vocab_size=1000, hidden_size=128, intermediate_size=512, num_hidden_layers=2,
                                        num_attention_heads=2, hidden_act="quick_gelu"), 77),
    # eos rule with content ids above eos (argmax would pick another row), d = 40 stored as 48, 150 tokens over two
    # 128-row query / key tiles
    "b_gelu_d40": (ClipTextConfig(vocab_size=1000, hidden_size=320, intermediate_size=640, num_hidden_layers=2,
                                  num_attention_heads=8, max_position_embeddings=160, hidden_act="gelu", bos_token_id=6,
                                  eos_token_id=7, pad_token_id=7), 150),
}
FULL = {"sd15": (ClipTextConfig(), 77)}       # SD-1.5 text_encoder/config.json
ROWS = {77: [0, 1, 6, 40, 76], 150: [0, 1, 4, 127, 128, 129, 149]}   # token rows of last_hidden_state kept per length
LENGTHS = {77: [5, 75, 30], 150: [3, 148, 120]}   # content tokens per sequence (0 = bos, eos... only)


def run_transformers(cfg: ClipTextConfig, sd, ids):
    import transformers
    from transformers import CLIPTextConfig, CLIPTextModel
    m = CLIPTextModel(CLIPTextConfig(**asdict(cfg)))
    m.config._attn_implementation = "eager"
    m.eval()
    ref_shapes = {k: tuple(v.shape) for k, v in m.state_dict().items() if not k.endswith("position_ids")}
    assert ref_shapes == dict(clip_text_param_shapes(cfg)), "CLIP text schema mismatch"
    res = m.load_state_dict(sd, strict=False)
    assert not res.missing_keys and all(k.endswith("position_ids") for k in res.unexpected_keys), res
    with torch.no_grad():
        out = m(input_ids=ids)
    return out.last_hidden_state.clone(), out.pooler_output.clone(), transformers.__version__


def golden(tag, cfgs, wseed=7, iseed=4747):
    entries = {}
    version = None
    for name, (cfg, L) in cfgs.items():
        t0 = time.time()
        sd = make_clip_text_state_dict(cfg, seed=wseed)
        ids = make_input_ids(len(LENGTHS[L]), L, cfg, seed=iseed, lengths=LENGTHS[L])
        last, pooled, version = run_transformers(cfg, sd, ids)
        entries[name] = dict(config=asdict(cfg), L=L, lengths=LENGTHS[L], rows=ROWS[L], pooler_output=pooled,
                             last_hidden_state=last[:, ROWS[L]].clone())
        print(f"{tag}/{name}: pooler std {pooled.std().item():.4f}, last_hidden_state max|.| "
              f"{last.abs().max().item():.3f} ({time.time() - t0:.1f}s)", flush=True)
    meta = dict(weight_seed=wseed, input_seed=iseed, transformers_version=version,
                source="transformers.CLIPTextModel (attn_implementation eager), CPU fp32")
    path = os.path.join(GOLDEN, f"clip_text_{tag}.pt")
    torch.save({"meta": meta, "configs": entries}, path)
    print(path, os.path.getsize(path), "bytes", flush=True)


if __name__ == "__main__":
    os.makedirs(GOLDEN, exist_ok=True)
    torch.set_num_threads(os.cpu_count() or 1)
    golden("narrow", NARROW)
    golden("full", FULL)
