"""CPU tests of the CLIP vision tower (IP-Adapter image encoder): the oracle against transformers and against the fixtures
(tests/golden/clip_vision_*.pt, produced by oracle/make_golden_clip_vision.py from the unmodified transformers model), the
state-dict schema, the FLOP counter and the config checks."""
import os
from dataclasses import asdict

import pytest
import torch

from conftest import GOLDEN
from musev_b200.schema import ClipVisionConfig, clip_vision_config, clip_vision_param_shapes
from musev_b200.synth import make_clip_pixel_values, make_clip_vision_state_dict
from oracle.clip_vision_oracle import clip_vision_forward

NARROW = {
    "gelu_d64": ClipVisionConfig(hidden_size=128, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2,
                                 image_size=56, patch_size=14, projection_dim=64, hidden_act="gelu"),
    "quick_gelu_d40": ClipVisionConfig(hidden_size=320, intermediate_size=640, num_hidden_layers=2, num_attention_heads=8,
                                       image_size=56, patch_size=14, projection_dim=64, hidden_act="quick_gelu"),
}


def _transformers_model(cfg, sd):
    transformers = pytest.importorskip("transformers")
    m = transformers.CLIPVisionModelWithProjection(transformers.CLIPVisionConfig(**asdict(cfg))).eval()
    m.config._attn_implementation = "eager"
    m.load_state_dict(sd, strict=False)
    return m


@pytest.mark.parametrize("name", list(NARROW) + ["vit_h14"])
def test_oracle_matches_transformers(name):
    cfg = NARROW.get(name, ClipVisionConfig())
    sd = make_clip_vision_state_dict(cfg, seed=11, outlier_channels=3)
    m = _transformers_model(cfg, sd)
    x = make_clip_pixel_values(2 if name in NARROW else 1, cfg.image_size, seed=5)
    with torch.no_grad():
        ref = m(pixel_values=x)
    emb, last = clip_vision_forward(sd, cfg, x)
    assert (emb - ref.image_embeds).abs().max().item() <= 1e-5 * max(1.0, ref.image_embeds.abs().max().item())
    assert (last - ref.last_hidden_state).abs().max().item() <= 1e-5 * max(1.0, ref.last_hidden_state.abs().max().item())


@pytest.mark.parametrize("tag", ["narrow", "full"])
def test_oracle_reproduces_fixture(tag):
    g = torch.load(os.path.join(GOLDEN, f"clip_vision_{tag}.pt"))
    m = g["meta"]
    for name, e in g["configs"].items():
        cfg = ClipVisionConfig(**e["config"])
        sd = make_clip_vision_state_dict(cfg, seed=m["weight_seed"])
        x = make_clip_pixel_values(m["n"], cfg.image_size, seed=m["input_seed"])
        emb, last = clip_vision_forward(sd, cfg, x)
        if m["rows"] is not None:
            last = last[:, m["rows"]]
        assert e["image_embeds"].abs().max().item() > 0.5, name        # the fixture carries signal
        assert (emb - e["image_embeds"]).abs().max().item() < 1e-5 * max(1.0, e["image_embeds"].abs().max().item()), name
        assert (last - e["last_hidden_state"]).abs().max().item() < 1e-5 * max(1.0, e["last_hidden_state"].abs().max().item())


@pytest.mark.parametrize("act", ["gelu", "quick_gelu"])
def test_param_shapes_match_transformers_state_dict(act):
    transformers = pytest.importorskip("transformers")
    for cfg in (ClipVisionConfig(hidden_act=act), ClipVisionConfig(**{**asdict(NARROW["quick_gelu_d40"]), "hidden_act": act})):
        with torch.device("meta"):
            m = transformers.CLIPVisionModelWithProjection(transformers.CLIPVisionConfig(**asdict(cfg)))
        got = {k: tuple(v.shape) for k, v in m.state_dict().items() if not k.endswith("position_ids")}
        assert list(got.items()) == list(clip_vision_param_shapes(cfg).items())


@pytest.mark.parametrize("name,N", [("gelu_d64", 2), ("quick_gelu_d40", 3), ("vit_h14", 1)])
def test_clip_vision_flops_match_flop_counter(name, N):
    from torch.utils.flop_counter import FlopCounterMode
    from musev_b200.flops import clip_vision_flops
    cfg = NARROW.get(name, ClipVisionConfig())
    sd = make_clip_vision_state_dict(cfg, seed=1)
    x = make_clip_pixel_values(N, cfg.image_size, seed=2)
    with FlopCounterMode(display=False) as fc:
        clip_vision_forward(sd, cfg, x)
    f = clip_vision_flops(cfg, N)
    assert f["total"] == fc.get_total_flops()
    if name == "vit_h14":
        assert abs(f["total"] / 1e12 - 0.3346) < 1e-4


def test_config_parsing():
    c = clip_vision_config({"hidden_size": 128, "num_attention_heads": 2, "hidden_act": "quick_gelu", "image_size": 56,
                            "unrelated_key": 1})
    assert (c.hidden_size, c.hidden_act, c.num_patches, c.patch_size) == (128, "quick_gelu", 16, 14)
    assert clip_vision_config(ClipVisionConfig()) == ClipVisionConfig()
    for bad in ({"hidden_act": "gelu_new"}, {"hidden_act": "relu"}, {"hidden_size": 1000},
                {"hidden_size": 128, "num_attention_heads": 32}, {"hidden_size": 256, "num_attention_heads": 1},
                {"image_size": 225}, {"num_channels": 5}):
        with pytest.raises(ValueError):
            clip_vision_config(bad)
    try:
        from transformers import CLIPVisionConfig
    except ImportError:
        return
    assert clip_vision_config(CLIPVisionConfig(hidden_size=1280, intermediate_size=5120, num_hidden_layers=32,
                                               num_attention_heads=16, patch_size=14, projection_dim=1024,
                                               hidden_act="gelu")) == ClipVisionConfig()
    with pytest.raises(ValueError, match="hidden_act"):
        clip_vision_config(CLIPVisionConfig(hidden_act="silu"))
