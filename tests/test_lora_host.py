"""CPU tests of the LoRA merge's host side: the kohya <-> reference name map, the plain-torch oracle against the unmodified
reference merge (tests/golden/lora_narrow.pt, oracle/make_golden_lora.py), and the rejections that happen before any
engine call."""
import os
from types import SimpleNamespace

import pytest
import torch

from conftest import GOLDEN
from musev_b200 import lora
from musev_b200.schema import preset_config, unet_param_shapes
from musev_b200.synth import make_lora_state_dict, make_state_dict, make_text_encoder

NARROW = (64, 128, 128, 128)


@pytest.mark.parametrize("preset", ["musev", "musev_referencenet"])
def test_name_map_covers_every_matrix_weight(preset):
    cfg = preset_config(preset)
    m = lora.kohya_name_map(cfg)
    mats = [n for n, s in unet_param_shapes(cfg).items() if len(s) >= 2]
    assert sorted(m.values()) == sorted(mats) and len(set(m.values())) == len(m)
    for k, n in m.items():
        assert n[:-7].replace(".", "_") == k


def _golden():
    return torch.load(os.path.join(GOLDEN, "lora_narrow.pt"))


def _spec_lora(cfg, meta):
    return make_lora_state_dict(cfg, meta["targets"], rank=meta["rank"], seed=meta["lora_seed"], amp=meta["amp"],
                                no_alpha=meta["no_alpha"], f32=meta["f32"], text_targets=[tuple(t) for t in meta["text_targets"]])


@pytest.mark.parametrize("case", ["all", "face", "unload"])
def test_oracle_reproduces_reference_merge_bits(case):
    from oracle.lora_oracle import deltas, merged, sha256
    g = _golden()
    meta = g["meta"]
    cfg = preset_config(meta["preset"], block_out_channels=tuple(meta["block_out_channels"]))
    sd16 = {k: v.half() for k, v in make_state_dict(cfg, seed=meta["weight_seed"]).items()}
    te = make_text_encoder(meta["text_width"], meta["text_seed"]).text_model.encoder.layers[0].self_attn.k_proj.weight.data
    block = "FACE" if case == "face" else "ALL"
    ds = deltas(cfg, _spec_lora(cfg, meta), meta["strength"], block)
    sd16[meta["text_weight"]] = te
    ds[meta["text_weight"]] = ds.pop("lora_te_" + meta["text_targets"][0][0])
    out = merged(sd16, ds)
    if case == "unload":
        out = merged(out, ds, subtract=True)
    want = g[f"sha256_{case}"]
    assert set(want) == set(meta["targets"]) | {meta["text_weight"]}
    for name, h in want.items():
        assert sha256(out[name]) == h, name
    if case == "face":   # FACE zeroes the down_blocks.0 attention targets and keeps resnets / up_blocks.1 attentions
        assert torch.equal(out["down_blocks.0.attentions.0.proj_in.weight"], sd16["down_blocks.0.attentions.0.proj_in.weight"])
        assert not torch.equal(out["down_blocks.0.resnets.0.conv1.weight"], sd16["down_blocks.0.resnets.0.conv1.weight"])
        assert not torch.equal(out["up_blocks.1.attentions.0.proj_out.weight"], sd16["up_blocks.1.attentions.0.proj_out.weight"])


class _FakeEngine:
    """Records engine calls; stands in for UNet3DConditionModel on a machine without a GPU."""

    def __init__(self, cfg):
        self.cfg, self.device, self.calls = cfg, torch.device("cpu"), []

    def _merge_lora(self, targets, ups, downs, scales, subtract=False):
        self.calls.append((list(targets), list(scales), subtract))


def _pipe(cfg):
    return SimpleNamespace(unet=_FakeEngine(cfg), text_encoder=make_text_encoder(64, 3))


def test_drop_in_scales_order_and_unload_batches():
    cfg = preset_config("musev_referencenet", block_out_channels=NARROW)
    targets = ["down_blocks.0.attentions.0.proj_in.weight", "down_blocks.0.resnets.0.conv1.weight",
               "up_blocks.1.attentions.0.transformer_blocks.0.attn2.to_k_ip.weight"]
    sd = make_lora_state_dict(cfg, targets, rank=4, seed=1, no_alpha=targets[1:2],
                              text_targets=[("text_model_encoder_layers_0_self_attn_k_proj", 64, 64)])
    pipe = _pipe(cfg)
    te_before = pipe.text_encoder.text_model.encoder.layers[0].self_attn.k_proj.weight.data.clone()
    _, undo = lora.update_pipeline_lora_model(pipe, sd, alpha=0.6, lora_block_weight_str="FACE", need_unload=True)
    (names, scales, sub), = pipe.unet.calls
    assert names == targets and not sub
    # alpha = rank / 2 -> 0.6 * 0.5; FACE zeroes down_blocks.0.attentions.*; resnets without alpha keep the strength
    assert scales == [0.0, 0.6, 0.6 * 0.5]
    te = pipe.text_encoder.text_model.encoder.layers[0].self_attn.k_proj.weight.data
    assert not torch.equal(te, te_before)
    lora.unload_lora(undo)
    assert pipe.unet.calls[-1] == (targets, scales, True)


def test_models_keep_reference_order_and_last_unload(tmp_path):
    from safetensors.torch import save_file
    cfg = preset_config("musev", block_out_channels=NARROW)
    paths = []
    for i, t in enumerate(["conv_in.weight", "mid_block.resnets.0.conv2.weight"]):
        p = str(tmp_path / f"l{i}.safetensors")
        save_file(dict(make_lora_state_dict(cfg, [t], rank=2, seed=i)), p)
        paths.append(p)
    pipe = _pipe(cfg)
    _, undo = lora.update_pipeline_lora_models(pipe, {paths[0]: {"strength": 0.5}, paths[1]: {"strength": 1.0, "strength_offset": -0.25}})
    assert [c[0] for c in pipe.unet.calls] == [["conv_in.weight"], ["mid_block.resnets.0.conv2.weight"]]
    assert pipe.unet.calls[1][1] == [0.75 * 0.5]
    assert [u["name"] for u in undo] == ["mid_block.resnets.0.conv2.weight"]    # model_util.py:464 keeps the last LoRA's


@pytest.mark.parametrize("what", ["unknown", "five_d", "rank", "peft", "shape"])
def test_rejections_name_the_key_and_merge_nothing(what):
    cfg = preset_config("musev", block_out_channels=NARROW)
    sd = make_lora_state_dict(cfg, ["down_blocks.0.resnets.0.conv1.weight", "conv_in.weight"], rank=4, seed=2)
    key = "lora_unet_conv_in.lora_down.weight"
    if what == "unknown":
        key = "lora_unet_down_blocks_0_nothing_here.lora_down.weight"
        sd[key] = torch.zeros(4, 8)
        sd[key.replace("lora_down", "lora_up")] = torch.zeros(8, 4)
    elif what == "five_d":
        key = "lora_unet_down_blocks_0_temp_convs_0_conv1_2"
        sd[key + ".lora_down.weight"] = torch.zeros(4, 64, 3, 1, 1)
        sd[key + ".lora_up.weight"] = torch.zeros(64, 4, 1, 1, 1)
    elif what == "rank":
        sd[key] = torch.zeros(3, 4, 3, 3)
        key = "lora_unet_conv_in"
    elif what == "peft":
        key = "unet.conv_in.lora_A.weight"
        sd[key] = torch.zeros(4, 36)
    elif what == "shape":
        sd[key] = torch.zeros(4, 5, 3, 3)
        key = "lora_unet_conv_in"
    pipe = _pipe(cfg)
    with pytest.raises(ValueError) as e:
        lora.update_pipeline_lora_model(pipe, sd, alpha=1.0)
    assert key.split(".")[0] in str(e.value)
    assert pipe.unet.calls == []
