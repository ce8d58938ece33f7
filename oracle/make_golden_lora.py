"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/lora_narrow.pt by running the UNMODIFIED reference LoRA merge
(musev/utils/model_util.py: `update_pipeline_lora_model`, `unload_lora`) on the imported reference UNet3D
(`musev_referencenet`, narrow width, CPU, `.half()`), with a seeded kohya LoRA and a small torch text encoder.

Run in the build container only:  python -m oracle.make_golden_lora
The reference's getattr walk stops at the first attribute that matches a prefix of the kohya name, so it cannot reach
`attn2.to_k_ip` / `to_v_ip` (it finds `to_k` / `to_v`) or `mid_block_refer_emb_attns` (it finds `mid_block`): those
targets are left out here and covered against oracle/lora_oracle.py on the GPU.
The fixture keeps the seeds and the key spec, the sha256 of every merged tensor (block weights ALL and FACE, and ALL
followed by unload_lora), and the fp32 UNet output after the ALL merge. Weights and factors are regenerated from the seeds.
"""
from __future__ import annotations

import os
import sys
import time
from types import SimpleNamespace

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from musev_b200.synth import make_inputs, make_lora_state_dict, make_state_dict, make_text_encoder  # noqa: E402
from oracle import ref_shim  # noqa: E402
from oracle.lora_oracle import sha256  # noqa: E402
from oracle.make_golden import GOLDEN, NARROW, build_reference, run_reference_unet  # noqa: E402

SPEC = dict(
    preset="musev_referencenet", block_out_channels=list(NARROW), weight_seed=0, lora_seed=21, rank=8, amp=0.25,
    strength=0.8, text_width=64, text_seed=3,
    targets=[
        "conv_in.weight",
        "down_blocks.0.resnets.0.conv1.weight",
        "down_blocks.0.resnets.0.time_emb_proj.weight",
        "down_blocks.0.attentions.0.proj_in.weight",
        "down_blocks.0.attentions.0.transformer_blocks.0.attn1.to_q.weight",
        "down_blocks.0.attentions.0.transformer_blocks.0.attn1.to_k.weight",
        "down_blocks.0.attentions.0.transformer_blocks.0.attn1.to_v.weight",
        "down_blocks.0.attentions.0.transformer_blocks.0.ff.net.0.proj.weight",
        "down_blocks.1.resnets.0.conv_shortcut.weight",
        "down_blocks.0.refer_emb_attns.0.to_q.weight",
        "mid_block.attentions.0.transformer_blocks.0.attn2.to_v.weight",
        "up_blocks.0.upsamplers.0.conv.weight",
        "up_blocks.1.attentions.0.proj_out.weight",
        "up_blocks.1.attentions.0.transformer_blocks.0.ff.net.2.weight",
        "up_blocks.2.temp_attentions.0.transformer_blocks.0.attn1.to_out.0.weight",
        "conv_out.weight",
    ],
    no_alpha=["down_blocks.0.resnets.0.time_emb_proj.weight", "up_blocks.1.attentions.0.proj_out.weight"],
    f32=["conv_in.weight", "down_blocks.0.attentions.0.transformer_blocks.0.attn1.to_q.weight",
         "up_blocks.0.upsamplers.0.conv.weight"],
    text_targets=[["text_model_encoder_layers_0_self_attn_k_proj", 64, 64]],
)
TEXT_WEIGHT = "text_model.encoder.layers.0.self_attn.k_proj.weight"


def lora_from_spec(cfg, spec):
    return make_lora_state_dict(cfg, spec["targets"], rank=spec["rank"], seed=spec["lora_seed"], amp=spec["amp"],
                                no_alpha=spec["no_alpha"], f32=spec["f32"], text_targets=[tuple(t) for t in spec["text_targets"]])


def main():
    t0 = time.time()
    ref_shim.load()
    from musev.utils.model_util import unload_lora, update_pipeline_lora_model
    sd = make_state_dict(__import__("musev_b200.schema", fromlist=["preset_config"]).preset_config(
        SPEC["preset"], block_out_channels=tuple(SPEC["block_out_channels"])), seed=SPEC["weight_seed"])
    m, cfg = build_reference(SPEC["preset"], tuple(SPEC["block_out_channels"]), sd)
    names = SPEC["targets"]

    def run(block, unload):
        m.load_state_dict(sd, strict=True)
        m.half()
        te = make_text_encoder(SPEC["text_width"], SPEC["text_seed"])
        pipe = SimpleNamespace(unet=m, text_encoder=te)
        _, undo = update_pipeline_lora_model(pipe, lora_from_spec(cfg, SPEC), alpha=SPEC["strength"], device="cpu",
                                             lora_block_weight_str=block, need_unload=True)
        if unload:
            unload_lora(undo)
        params = dict(m.named_parameters())
        hashes = {n: sha256(params[n]) for n in names}
        hashes[TEXT_WEIGHT] = sha256(te.text_model.encoder.layers[0].self_attn.k_proj.weight)
        return hashes

    out = {"meta": dict(SPEC, text_weight=TEXT_WEIGHT,
                        source="reference musev.utils.model_util.update_pipeline_lora_model / unload_lora on "
                               "musev.models.unet_3d_condition.UNet3DConditionModel (.half(), CPU)")}
    out["sha256_face"] = run("FACE", False)
    out["sha256_unload"] = run("ALL", True)
    out["sha256_all"] = run("ALL", False)
    g = torch.load(os.path.join(GOLDEN, "unet_musev_referencenet_narrow.pt"))["meta"]
    m.float()
    inp = make_inputs(cfg, batch=g["batch"], frames=g["frames"], h=g["h"], w=g["w"], n_vis_cond=1, seed=g["input_seed"])
    out["forward"] = dict(batch=g["batch"], frames=g["frames"], h=g["h"], w=g["w"], timestep=g["timestep"],
                          input_seed=g["input_seed"], sample_frame_rate=g["sample_frame_rate"],
                          ip_adapter_scale=g["ip_adapter_scale"])
    out["out"] = run_reference_unet(m, inp, g["timestep"], g["sample_frame_rate"], g["ip_adapter_scale"]).clone()
    path = os.path.join(GOLDEN, "lora_narrow.pt")
    torch.save(out, path)
    print(f"{path}: {os.path.getsize(path)} bytes, out std {out['out'].std().item():.4f} ({time.time() - t0:.1f}s)")


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count() or 1)
    main()
