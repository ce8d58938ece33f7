"""CPU tests of the CLIP text encoder (the prompt encoder): the oracle against transformers and against the fixtures
(tests/golden/clip_text_*.pt, produced by oracle/make_golden_clip_text.py from the unmodified transformers model), the
state-dict schema, the FLOP counter, both pooling rules, the kohya text-encoder name map, the LoRA drop-in's routing of text
keys to an engine text encoder, and the config checks."""
import os
from dataclasses import asdict
from types import SimpleNamespace

import pytest
import torch

from conftest import GOLDEN
from musev_b200 import lora
from musev_b200.schema import (ClipTextConfig, clip_text_config, clip_text_param_shapes, kohya_text_name_map, preset_config)
from musev_b200.synth import make_clip_text_state_dict, make_input_ids, make_lora_state_dict
from oracle.clip_text_oracle import clip_text_forward, pool_index

NARROW = {
    "a_quick_gelu_d64": (ClipTextConfig(vocab_size=1000, hidden_size=128, intermediate_size=512, num_hidden_layers=2,
                                        num_attention_heads=2, hidden_act="quick_gelu"), 77),
    "b_gelu_d40": (ClipTextConfig(vocab_size=1000, hidden_size=320, intermediate_size=640, num_hidden_layers=2,
                                  num_attention_heads=8, max_position_embeddings=160, hidden_act="gelu", bos_token_id=6,
                                  eos_token_id=7, pad_token_id=7), 150),
}


def _transformers_model(cfg, sd):
    transformers = pytest.importorskip("transformers")
    m = transformers.CLIPTextModel(transformers.CLIPTextConfig(**asdict(cfg))).eval()
    m.config._attn_implementation = "eager"
    m.load_state_dict(sd, strict=False)
    return m


def _close(got, ref, tol=1e-5):
    return (got - ref).abs().max().item() <= tol * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("name", list(NARROW))
@pytest.mark.parametrize("outliers", [0, 3])
def test_oracle_matches_transformers(name, outliers):
    cfg, L = NARROW[name]
    sd = make_clip_text_state_dict(cfg, seed=11, outlier_channels=outliers)
    m = _transformers_model(cfg, sd)
    ids = make_input_ids(3, L, cfg, seed=5)
    with torch.no_grad():
        ref = m(input_ids=ids)
    last, pooled = clip_text_forward(sd, cfg, ids)
    assert _close(last, ref.last_hidden_state) and _close(pooled, ref.pooler_output)


@pytest.mark.parametrize("tag", ["narrow", "full"])
def test_oracle_reproduces_fixture(tag):
    g = torch.load(os.path.join(GOLDEN, f"clip_text_{tag}.pt"))
    m = g["meta"]
    assert m["transformers_version"]
    for name, e in g["configs"].items():
        cfg = ClipTextConfig(**e["config"])
        sd = make_clip_text_state_dict(cfg, seed=m["weight_seed"])
        ids = make_input_ids(len(e["lengths"]), e["L"], cfg, seed=m["input_seed"], lengths=e["lengths"])
        last, pooled = clip_text_forward(sd, cfg, ids)
        assert e["pooler_output"].abs().max().item() > 0.5, name        # the fixture carries signal
        assert _close(pooled, e["pooler_output"]), name
        assert _close(last[:, e["rows"]], e["last_hidden_state"]), name


def test_param_shapes_match_transformers_state_dict():
    transformers = pytest.importorskip("transformers")
    for cfg in [ClipTextConfig()] + [c for c, _ in NARROW.values()]:
        with torch.device("meta"):
            m = transformers.CLIPTextModel(transformers.CLIPTextConfig(**asdict(cfg)))
        got = {k: tuple(v.shape) for k, v in m.state_dict().items() if not k.endswith("position_ids")}
        assert list(got.items()) == list(clip_text_param_shapes(cfg).items())


@pytest.mark.parametrize("name,N,L", [("a_quick_gelu_d64", 2, 77), ("b_gelu_d40", 3, 150), ("sd15", 1, 77)])
def test_clip_text_flops_match_flop_counter(name, N, L):
    from torch.utils.flop_counter import FlopCounterMode
    from musev_b200.flops import clip_text_flops
    cfg = NARROW[name][0] if name in NARROW else ClipTextConfig()
    sd = make_clip_text_state_dict(cfg, seed=1)
    ids = make_input_ids(N, L, cfg, seed=2)
    with FlopCounterMode(display=False) as fc:
        clip_text_forward(sd, cfg, ids)
    f = clip_text_flops(cfg, N, L)
    assert f["total"] == fc.get_total_flops()
    if name == "sd15":
        assert abs(f["total"] / 1e9 - 13.30) < 0.01


def test_pooling_rules():
    """Legacy (eos_token_id == 2): argmax, first occurrence; otherwise the first eos, or 0 without one."""
    ids = torch.tensor([[49406, 5, 49407, 49407, 49407], [49406, 49407, 3, 49407, 9]])
    assert pool_index(ids, 2).tolist() == [2, 1]
    ids = torch.tensor([[6, 12, 30, 7, 7], [6, 7, 40, 7, 9], [6, 8, 9, 10, 11]])
    assert pool_index(ids, 7).tolist() == [3, 1, 0]
    assert pool_index(ids, 2).tolist() == [2, 2, 4]      # argmax picks other rows
    cfg, L = NARROW["b_gelu_d40"]
    gen = make_input_ids(3, L, cfg, seed=1, lengths=[3, 148, 120])
    assert pool_index(gen, 7).tolist() == [4, 149, 121]
    assert pool_index(gen, 2).tolist() != [4, 149, 121]
    sd = make_input_ids(2, 77, ClipTextConfig(), seed=1, lengths=[0, 75])
    assert sd[:, 0].tolist() == [49406, 49406] and pool_index(sd, 2).tolist() == [1, 76]
    assert (sd[0, 1:] == 49407).all()


def test_kohya_text_map_injective_and_complete():
    for cfg in [ClipTextConfig()] + [c for c, _ in NARROW.values()]:
        m = kohya_text_name_map(cfg)
        mats = [n for n, s in clip_text_param_shapes(cfg).items() if len(s) == 2 and ".encoder.layers." in n]
        assert sorted(m.values()) == sorted(mats) and len(set(m.values())) == len(m) == 6 * cfg.num_hidden_layers
        for k, n in m.items():
            assert n[:-7].replace(".", "_") == k
    assert kohya_text_name_map(ClipTextConfig())["text_model_encoder_layers_11_mlp_fc2"] == "text_model.encoder.layers.11.mlp.fc2.weight"


class _FakeEngine:
    """Records engine calls; stands in for an engine model on a machine without a GPU."""

    def __init__(self, cfg):
        self.cfg, self.device, self.calls = cfg, torch.device("cpu"), []

    def _merge_lora(self, targets, ups, downs, scales, subtract=False):
        self.calls.append((list(targets), list(scales), subtract))


def test_lora_text_keys_go_to_engine_text_encoder():
    cfg = preset_config("musev", block_out_channels=(64, 128, 128, 128))
    tcfg = ClipTextConfig(vocab_size=100, hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=1)
    targets = ["down_blocks.0.resnets.0.conv1.weight"]
    sd = make_lora_state_dict(cfg, targets, rank=4, seed=1,
                              text_targets=[("text_model_encoder_layers_0_self_attn_k_proj", 64, 64),
                                            ("text_model_encoder_layers_1_mlp_fc1", 128, 64)])
    pipe = SimpleNamespace(unet=_FakeEngine(cfg), text_encoder=_FakeEngine(tcfg))
    _, undo = lora.update_pipeline_lora_model(pipe, sd, alpha=0.6, lora_block_weight_str="DEFACE", need_unload=True)
    (names, scales, sub), = pipe.text_encoder.calls
    assert names == ["text_model.encoder.layers.0.self_attn.k_proj.weight", "text_model.encoder.layers.1.mlp.fc1.weight"]
    assert not sub and scales == [0.6 * 0.5, 0.6 * 0.5]               # DEFACE keeps weights[0] = 1; alpha = rank / 2
    assert [c[0] for c in pipe.unet.calls] == [targets]
    assert [u["layer"] for u in undo] == [pipe.unet, pipe.text_encoder, pipe.text_encoder]
    lora.unload_lora(undo)
    assert pipe.text_encoder.calls[-1] == (names, scales, True) and pipe.unet.calls[-1][2]
    # FACE gives the text encoder block weight 1 as well; a map miss or a wrong shape is rejected before any engine call
    bad = make_lora_state_dict(cfg, [], rank=2, seed=2, text_targets=[("text_model_encoder_layers_5_mlp_fc1", 128, 64)])
    pipe = SimpleNamespace(unet=_FakeEngine(cfg), text_encoder=_FakeEngine(tcfg))
    with pytest.raises(ValueError, match="no linear-layer weight"):
        lora.update_pipeline_lora_model(pipe, bad)
    bad = make_lora_state_dict(cfg, targets, rank=2, seed=2, text_targets=[("text_model_encoder_layers_0_mlp_fc1", 64, 64)])
    with pytest.raises(ValueError, match="does not match"):
        lora.update_pipeline_lora_model(pipe, bad)
    assert pipe.unet.calls == [] and pipe.text_encoder.calls == []


def test_config_parsing():
    c = clip_text_config({"hidden_size": 128, "num_attention_heads": 2, "hidden_act": "gelu", "eos_token_id": 7,
                          "unrelated_key": 1})
    assert (c.hidden_size, c.hidden_act, c.eos_token_id, c.max_position_embeddings) == (128, "gelu", 7, 77)
    assert clip_text_config(ClipTextConfig()) == ClipTextConfig()
    for bad in ({"hidden_act": "gelu_new"}, {"hidden_size": 1000}, {"hidden_size": 128, "num_attention_heads": 32},
                {"hidden_size": 256, "num_attention_heads": 1}, {"max_position_embeddings": 0},
                {"max_position_embeddings": 5000}, {"eos_token_id": -1}, {"intermediate_size": 100}):
        with pytest.raises(ValueError):
            clip_text_config(bad)
    try:
        from transformers import CLIPTextConfig
    except ImportError:
        return
    sd15 = CLIPTextConfig(vocab_size=49408, hidden_size=768, intermediate_size=3072, num_hidden_layers=12,
                          num_attention_heads=12, max_position_embeddings=77, hidden_act="quick_gelu", bos_token_id=0,
                          eos_token_id=2, pad_token_id=1)
    assert clip_text_config(sd15) == ClipTextConfig()
    with pytest.raises(ValueError, match="hidden_act"):
        clip_text_config(CLIPTextConfig(hidden_act="silu"))
