"""LoRA / LCM-LoRA weights merged into the engine UNet on the device, with unload.

Drop-ins for musev/utils/model_util.py:98-475 (`LORA_BLOCK_WEIGHT_MAP`, `update_pipeline_lora_model`,
`update_pipeline_lora_models`, `unload_lora`), the two routes by which `DiffusersPipelinePredictor.__init__` applies a
base-model `lora_dict` and the LCM-LoRA of `lcm_lora_dct` (pipeline_controlnet_predictor.py:296-327).

Keys are kohya style, the only format the reference reads: `<prefix>_<module path with "_">.lora_down.weight`,
`.lora_up.weight` and an optional `.alpha`. UNet keys go to the engine (`mvb_unet_merge_lora`, musev_b200/csrc/lora.cu).
Keys containing "text" go to the engine too when `pipeline.text_encoder` is the engine `CLIPTextModel` (same entry point,
same arithmetic), and otherwise to the torch text encoder with the reference's own arithmetic. Per target:
    scale = strength * (alpha / rank if alpha is present else 1)
    delta16 = fp16(fl32(scale) * (up @ down)) * LORA_BLOCK_WEIGHT_MAP[...][block]
    W16 = fp16(W16 + delta16), and W16 = fp16(W16 - delta16) on unload (not guaranteed to restore the original bits).
"""
from __future__ import annotations

import gc
import os
from collections import OrderedDict
from typing import Dict, List, Optional, Tuple, Union

import torch

from .schema import ClipTextConfig, UNetConfig, clip_text_param_shapes, kohya_text_name_map, unet_param_shapes

# musev/utils/model_util.py:98-104. Entry 0 is the text encoder, entries 1..16 follow LORA_UNET_LAYERS.
LORA_BLOCK_WEIGHT_MAP = {
    "FACE": [1, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 0, 0, 0, 0, 0, 0],
    "DEFACE": [1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 1, 1, 1, 1, 1, 1],
    "ALL": [1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1],
    "MIDD": [1, 0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0],
    "OUTALL": [1, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 1, 1],
}
# model_util.py:115-132, matched as substrings of the key (so `temp_attentions` and resnets get weight 1)
LORA_UNET_LAYERS = (
    "lora_unet_down_blocks_0_attentions_0", "lora_unet_down_blocks_0_attentions_1",
    "lora_unet_down_blocks_1_attentions_0", "lora_unet_down_blocks_1_attentions_1",
    "lora_unet_down_blocks_2_attentions_0", "lora_unet_down_blocks_2_attentions_1",
    "lora_unet_mid_block_attentions_0",
    "lora_unet_up_blocks_1_attentions_0", "lora_unet_up_blocks_1_attentions_1", "lora_unet_up_blocks_1_attentions_2",
    "lora_unet_up_blocks_2_attentions_0", "lora_unet_up_blocks_2_attentions_1", "lora_unet_up_blocks_2_attentions_2",
    "lora_unet_up_blocks_3_attentions_0", "lora_unet_up_blocks_3_attentions_1", "lora_unet_up_blocks_3_attentions_2",
)
MAX_RANK = 256


def kohya_name_map(cfg: UNetConfig) -> "OrderedDict[str, str]":
    """kohya module name (without prefix) -> reference weight name, for every matrix / convolution weight of the UNet:
    the inverse of `name[:-len(".weight")].replace(".", "_")`."""
    out: "OrderedDict[str, str]" = OrderedDict()
    for name, shape in unet_param_shapes(cfg).items():
        if name.endswith(".weight") and len(shape) >= 2:
            k = name[:-7].replace(".", "_")
            assert k not in out, f"kohya names collide: {out[k]} and {name}"
            out[k] = name
    return out


def block_weights(lora_block_weight_str: Optional[str]) -> List[float]:
    w = LORA_BLOCK_WEIGHT_MAP[lora_block_weight_str.upper()] if lora_block_weight_str is not None else [1] * 17
    assert len(w) == 17
    return w


def _load(lora: Union[str, Dict[str, torch.Tensor]]) -> Dict[str, torch.Tensor]:
    if isinstance(lora, (str, os.PathLike)):
        from safetensors.torch import load_file
        return load_file(str(lora))
    return lora


class LoraTarget:
    """One (lora_up, lora_down[, alpha]) triple of a kohya state dict."""

    def __init__(self, module: str, up_key: str, down_key: str, alpha_key: Optional[str]):
        self.module, self.up_key, self.down_key, self.alpha_key = module, up_key, down_key, alpha_key


def pair_keys(state_dict: Dict[str, torch.Tensor]) -> List[LoraTarget]:
    """The reference's key walk (model_util.py:165-208, 255-257): targets in the order their first factor appears.
    Anything that is not a kohya factor or alpha is rejected by name."""
    for k in state_dict:
        if not (k.endswith(".lora_down.weight") or k.endswith(".lora_up.weight") or k.endswith(".alpha")):
            raise ValueError(f"unsupported LoRA key {k!r}: only kohya keys (`.lora_down.weight`, `.lora_up.weight`, "
                             "`.alpha`) are understood; PEFT / diffusers keys (lora_A / lora_B) are not")
    visited, out = set(), []
    for key in state_dict:
        if ".alpha" in key or key in visited:
            continue
        if "lora_down" in key:
            up, down, alpha = key.replace("lora_down", "lora_up"), key, key.replace("lora_down.weight", "alpha")
        else:
            up, down, alpha = key, key.replace("lora_up", "lora_down"), key.replace("lora_up.weight", "alpha")
        for k in (up, down):
            if k not in state_dict:
                raise ValueError(f"LoRA key {key!r} has no partner {k!r}")
        out.append(LoraTarget(key.split(".")[0], up, down, alpha if alpha in state_dict else None))
        visited.update((up, down))
    return out


def factors(state_dict, t: LoraTarget, target_shape=None) -> Tuple[torch.Tensor, torch.Tensor, int]:
    """(up, down, rank) of a target, checked the way the reference's arithmetic would accept them
    (model_util.py:211-240: 2-D x 2-D by torch.mm, 4-D x 4-D squeezed or by einsum; anything else raises there)."""
    up, down = state_dict[t.up_key], state_dict[t.down_key]
    if up.dim() == 5 or down.dim() == 5:
        raise ValueError(f"{t.module}: 5-D LoRA factors (temporal convolutions) cannot be merged "
                         f"(up {tuple(up.shape)}, down {tuple(down.shape)})")
    if not ((up.dim() == 2 and down.dim() == 2) or (up.dim() == 4 and down.dim() == 4 and up.shape[2:] == (1, 1))):
        raise ValueError(f"{t.module}: unsupported LoRA factor shapes up {tuple(up.shape)} / down {tuple(down.shape)}")
    r = up.shape[1]
    if down.shape[0] != r:
        raise ValueError(f"{t.module}: rank mismatch between lora_up {tuple(up.shape)} and lora_down {tuple(down.shape)}")
    if target_shape is not None:
        delta = (up.shape[0],) + tuple(down.shape[1:])
        if tuple(target_shape) != delta:
            raise ValueError(f"{t.module}: LoRA delta {delta} does not match the weight {tuple(target_shape)}")
    return up, down, int(r)


def target_scale(state_dict, t: LoraTarget, strength: float, rank: int) -> float:
    """`alpha * weight_scale` of model_util.py:216-226 (a Python double; the engine rounds it to fp32 as torch does)."""
    weight_scale = state_dict[t.alpha_key].item() / rank if t.alpha_key is not None else 1.0
    return strength * weight_scale


def block_weight(key: str, weights: List[float], lora_unet_layers) -> float:
    """model_util.py:242-249."""
    if "text" in key:
        return weights[0]
    for idx, layer in enumerate(lora_unet_layers):
        if layer in key:
            return weights[idx + 1]
    return 1


def _text_layer(root, key: str, prefix: str):
    """The reference's getattr walk over a torch module (model_util.py:176-198): module names may contain "_"."""
    infos = key.split(".")[0].split(prefix + "_")[-1].split("_")
    layer, temp = root, infos.pop(0)
    while True:
        try:
            layer = layer.__getattr__(temp)
            if not infos:
                return layer
            temp = infos.pop(0)
        except AttributeError:
            if not infos:
                raise ValueError(f"LoRA key {key!r}: no such text-encoder module")
            temp = temp + "_" + infos.pop(0) if temp else infos.pop(0)


def text_delta(up: torch.Tensor, down: torch.Tensor, scale: float, bw: float) -> torch.Tensor:
    """delta16 exactly as model_util.py:211-248 computes it."""
    if up.dim() == 4:
        u, d = up.squeeze(3).squeeze(2).to(torch.float32), down.squeeze(3).squeeze(2).to(torch.float32)
        if u.dim() == d.dim():
            delta = scale * torch.mm(u, d).unsqueeze(2).unsqueeze(3)
        else:
            delta = scale * torch.einsum("a b, b c h w -> a c h w", u, d)
    else:
        delta = scale * torch.mm(up.to(torch.float32), down.to(torch.float32))
    delta = delta.to(torch.float16)
    delta *= bw
    return delta


def update_pipeline_lora_model(pipeline, lora: Union[str, Dict[str, torch.Tensor]], alpha: float = 0.75, device: str = "cuda",
                               lora_prefix_unet: str = "lora_unet", lora_prefix_text_encoder: str = "lora_te",
                               lora_unet_layers=LORA_UNET_LAYERS, lora_block_weight_str: str = "ALL",
                               need_unload: bool = False):
    """Drop-in for musev/utils/model_util.py:108-262 with `pipeline.unet` a musev_b200 `UNet3DConditionModel`: the UNet
    targets of one LoRA are merged by one engine call. Text-encoder targets are merged by one more engine call when
    `pipeline.text_encoder` is the engine `CLIPTextModel` (block weight `weights[0]`), and into the torch module otherwise.
    `alpha` is the strength. Everything is validated before any weight changes."""
    weights = block_weights(lora_block_weight_str)
    sd = _load(lora)
    unet = pipeline.unet
    if not hasattr(unet, "_merge_lora"):
        raise TypeError("pipeline.unet is not a musev_b200 UNet3DConditionModel")
    names = kohya_name_map(unet.cfg)
    shapes = unet_param_shapes(unet.cfg)
    dev = unet.device
    te = getattr(pipeline, "text_encoder", None)
    te_engine = _is_engine_text_encoder(te)
    te_names = kohya_text_name_map(te.cfg) if te_engine else None
    te_shapes = clip_text_param_shapes(te.cfg) if te_engine else None
    eng, text, te_eng = [], [], []
    for t in pair_keys(sd):
        key = t.up_key
        if "text" in key and te_engine:
            mod = t.module
            name = te_names.get(mod[len(lora_prefix_text_encoder) + 1:]) if mod.startswith(lora_prefix_text_encoder + "_") else None
            if name is None:
                raise ValueError(f"LoRA key {key!r} names no linear-layer weight of this text encoder")
            up, down, r = factors(sd, t, te_shapes[name])
            if r > MAX_RANK:
                raise ValueError(f"{mod}: rank {r} exceeds {MAX_RANK}")
            s = target_scale(sd, t, alpha, r) * block_weight(key, weights, lora_unet_layers)
            te_eng.append((name, _dev(up, te.device), _dev(down, te.device), s))
            continue
        if "text" in key:
            up, down, r = factors(sd, t)
            text.append((t, up, down, r))
            continue
        mod = t.module
        name = names.get(mod[len(lora_prefix_unet) + 1:]) if mod.startswith(lora_prefix_unet + "_") else None
        if name is None:
            raise ValueError(f"LoRA key {key!r} names no matrix or convolution weight of this UNet")
        up, down, r = factors(sd, t, shapes[name])
        if r > MAX_RANK:
            raise ValueError(f"{mod}: rank {r} exceeds {MAX_RANK}")
        s = target_scale(sd, t, alpha, r) * block_weight(key, weights, lora_unet_layers)
        eng.append((name, _dev(up, dev), _dev(down, dev), s))
    text_layers = [(_text_layer(pipeline.text_encoder, t.up_key, lora_prefix_text_encoder), t, up, down, r)
                   for t, up, down, r in text]
    unload = []
    if eng:
        unet._merge_lora([e[0] for e in eng], [e[1] for e in eng], [e[2] for e in eng], [e[3] for e in eng], subtract=False)
        unload += [{"layer": unet, "name": n, "up": u, "down": d, "scale": s} for n, u, d, s in eng]
    if te_eng:
        te._merge_lora([e[0] for e in te_eng], [e[1] for e in te_eng], [e[2] for e in te_eng], [e[3] for e in te_eng],
                       subtract=False)
        unload += [{"layer": te, "name": n, "up": u, "down": d, "scale": s} for n, u, d, s in te_eng]
    for layer, t, up, down, r in text_layers:
        p = layer.weight
        delta = text_delta(up.to(p.device), down.to(p.device), target_scale(sd, t, alpha, r),
                           block_weight(t.up_key, weights, lora_unet_layers))
        layer.weight.data += delta
        unload.append({"layer": layer, "added_weight": delta})
    if need_unload:
        return pipeline, unload
    return pipeline


def update_pipeline_lora_models(pipeline, lora_dict: Dict[str, Dict], device: str = "cuda", need_unload: bool = True,
                                lora_prefix_unet: str = "lora_unet", lora_prefix_text_encoder: str = "lora_te",
                                lora_unet_layers=LORA_UNET_LAYERS):
    """Drop-in for musev/utils/model_util.py:401-465: one merge per LoRA, in `lora_dict` order, with strength
    `strength + strength_offset` and block weights `lora_block_weight` (default "ALL"). Like the reference (:464, after the
    loop), the returned unload list holds the entries of the LAST LoRA only."""
    unload_dict: list = []
    for lora, value in lora_dict.items():
        alpha = value.get("strength", 1.0) + value.get("strength_offset", 0.0)
        pipeline, unload_dict = update_pipeline_lora_model(
            pipeline, lora=_load(lora), device=device, alpha=alpha, lora_prefix_unet=lora_prefix_unet,
            lora_prefix_text_encoder=lora_prefix_text_encoder, lora_unet_layers=lora_unet_layers,
            lora_block_weight_str=value.get("lora_block_weight", "ALL"), need_unload=True)
    return pipeline, list(unload_dict)


def unload_lora(unload_dict: List[Dict]) -> None:
    """Drop-in for musev/utils/model_util.py:468-475: subtracts every recorded delta, in order. Consecutive engine entries
    go to the engine as one call each, split where a target repeats so that the order of subtractions is kept."""
    batch: list = []

    def flush():
        if batch:
            e = batch[0]["layer"]
            e._merge_lora([b["name"] for b in batch], [b["up"] for b in batch], [b["down"] for b in batch],
                          [b["scale"] for b in batch], subtract=True)
            batch.clear()

    for entry in unload_dict:
        if "added_weight" in entry:
            flush()
            entry["layer"].weight.data -= entry["added_weight"]
            continue
        if batch and (entry["layer"] is not batch[0]["layer"] or any(b["name"] == entry["name"] for b in batch)):
            flush()
        batch.append(entry)
    flush()
    gc.collect()
    torch.cuda.empty_cache()


def _is_engine_text_encoder(te) -> bool:
    """The engine `CLIPTextModel` (or a stand-in with its surface): LoRA factors go to its `_merge_lora`."""
    return te is not None and hasattr(te, "_merge_lora") and isinstance(getattr(te, "cfg", None), ClipTextConfig)


def _dev(t: torch.Tensor, dev) -> torch.Tensor:
    if t.dtype not in (torch.float16, torch.float32):
        t = t.float()
    return t.to(dev).contiguous()
