"""Plain-torch restatement of the reference LoRA merge (musev/utils/model_util.py:108-262, unload :468-475) over a
reference-named fp16 UNet state dict. Pinned bit for bit to the unmodified reference by tests/golden/lora_narrow.pt
(oracle/make_golden_lora.py); the GPU tests compare the engine's merged weights against it."""
from __future__ import annotations

from collections import OrderedDict
from typing import Dict

import torch

from musev_b200.schema import unet_param_shapes

BLOCK_WEIGHTS = {
    "FACE": [1, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 0, 0, 0, 0, 0, 0],
    "DEFACE": [1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 1, 1, 1, 1, 1, 1],
    "ALL": [1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1],
    "MIDD": [1, 0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0],
    "OUTALL": [1, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 1, 1],
}
LAYERS = [f"lora_unet_down_blocks_{i}_attentions_{j}" for i in range(3) for j in range(2)] + \
         ["lora_unet_mid_block_attentions_0"] + \
         [f"lora_unet_up_blocks_{i}_attentions_{j}" for i in range(1, 4) for j in range(3)]


def deltas(cfg, lora: Dict[str, torch.Tensor], strength: float = 1.0, block_weight_str: str = "ALL", device="cpu"):
    """OrderedDict target -> delta16, in the reference's key order. UNet targets are reference weight names, text-encoder
    targets keep their kohya module name (`lora_te_...`)."""
    names = {"lora_unet_" + n[:-7].replace(".", "_"): n for n, s in unet_param_shapes(cfg).items()
             if n.endswith(".weight") and len(s) >= 2}
    bw = BLOCK_WEIGHTS[block_weight_str.upper()]
    out: "OrderedDict[str, torch.Tensor]" = OrderedDict()
    visited = set()
    for key in lora:
        if ".alpha" in key or key in visited:
            continue
        if "lora_down" in key:
            pair = [key.replace("lora_down", "lora_up"), key]
            alpha_key = key.replace("lora_down.weight", "alpha")
        else:
            pair = [key, key.replace("lora_up", "lora_down")]
            alpha_key = key.replace("lora_up.weight", "alpha")
        up, down = lora[pair[0]].to(device), lora[pair[1]].to(device)
        if up.dim() == 4:
            u, d = up.squeeze(3).squeeze(2).to(torch.float32), down.squeeze(3).squeeze(2).to(torch.float32)
            ws = lora[alpha_key].item() / u.shape[1] if alpha_key in lora else 1.0
            if u.dim() == d.dim():
                delta = strength * ws * torch.mm(u, d).unsqueeze(2).unsqueeze(3)
            else:
                delta = strength * ws * torch.einsum("a b, b c h w -> a c h w", u, d)
        else:
            u, d = up.to(torch.float32), down.to(torch.float32)
            ws = lora[alpha_key].item() / u.shape[1] if alpha_key in lora else 1.0
            delta = strength * ws * torch.mm(u, d)
        delta = delta.to(torch.float16)
        if "text" in key:
            delta *= bw[0]
        else:
            for idx, layer in enumerate(LAYERS):
                if layer in key:
                    delta *= bw[idx + 1]
                    break
        mod = key.split(".")[0]
        out[mod if "text" in key else names[mod]] = delta
        visited.update(pair)
    return out


def merged(sd16: Dict[str, torch.Tensor], ds: Dict[str, torch.Tensor], subtract: bool = False) -> Dict[str, torch.Tensor]:
    """`weight.data += delta16` (or `-=`) on copies of the touched fp16 tensors; the others are shared."""
    out = dict(sd16)
    for name, d in ds.items():
        if name not in sd16:
            continue
        w = sd16[name].clone()
        if subtract:
            w -= d.to(w.device)
        else:
            w += d.to(w.device)
        out[name] = w
    return out


def sha256(t: torch.Tensor) -> str:
    """Digest of a tensor's bytes (its dtype and shape are compared separately)."""
    import hashlib
    return hashlib.sha256(t.detach().cpu().contiguous().numpy().tobytes()).hexdigest()
