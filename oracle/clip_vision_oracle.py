"""Plain-torch restatement of `transformers.CLIPVisionModelWithProjection.forward` (models/clip/modeling_clip.py; line numbers
below are transformers 5.5.0, whose arithmetic is the same as the 4.33.1 the reference pins, requirements.txt:15).

`clip_vision_forward(sd, cfg, pixel_values)` returns (image_embeds, last_hidden_state). By default it computes in fp32;
`dtype=torch.float16` runs it the way the reference runs the model (fp16 weights and activations, eager PyTorch), and
`sdpa=True` uses F.scaled_dot_product_attention, transformers' default attention implementation.
"""
from __future__ import annotations

from typing import Dict, Tuple

import torch
import torch.nn.functional as F

from musev_b200.schema import ClipVisionConfig


def _act(x: torch.Tensor, name: str) -> torch.Tensor:
    """ACT2FN (activations.py): "gelu" is the exact-erf GELU, "quick_gelu" is x * sigmoid(1.702 x) (QuickGELUActivation)."""
    if name == "gelu":
        return F.gelu(x)
    if name == "quick_gelu":
        return x * torch.sigmoid(1.702 * x)
    raise ValueError(f"unsupported hidden_act {name!r}")


def embeddings(w: Dict[str, torch.Tensor], cfg: ClipVisionConfig, pixel_values: torch.Tensor) -> torch.Tensor:
    """CLIPVisionEmbeddings.forward (:202-218): p x p conv with stride p and no bias, flatten to tokens, prepend
    class_embedding, add position_embedding."""
    e = "vision_model.embeddings."
    patch = F.conv2d(pixel_values, w[e + "patch_embedding.weight"], stride=cfg.patch_size)     # :209
    patch = patch.flatten(2).transpose(1, 2)                                                    # :210
    cls = w[e + "class_embedding"].expand(pixel_values.shape[0], 1, -1)                         # :212
    x = torch.cat([cls, patch], dim=1)                                                          # :213
    return x + w[e + "position_embedding.weight"].unsqueeze(0)                                  # :217


def attention(w: Dict[str, torch.Tensor], p: str, cfg: ClipVisionConfig, x: torch.Tensor, sdpa: bool = False) -> torch.Tensor:
    """CLIPAttention.forward (:300-336) with eager_attention_forward (:261-280): q / k / v with bias, per head
    softmax(q k^T * d^-0.5) v, out_proj."""
    N, T, C = x.shape
    H = cfg.num_attention_heads
    d = C // H

    def heads(n):
        return F.linear(x, w[f"{p}.{n}.weight"], w[f"{p}.{n}.bias"]).view(N, T, H, d).transpose(1, 2)
    q, k, v = heads("q_proj"), heads("k_proj"), heads("v_proj")                                # :310-316
    if sdpa:
        o = F.scaled_dot_product_attention(q, k, v, scale=d ** -0.5)
    else:
        s = torch.matmul(q, k.transpose(2, 3)) * d ** -0.5                                       # :271
        s = torch.softmax(s, dim=-1, dtype=torch.float32).to(q.dtype)                           # :274
        o = torch.matmul(s, v)                                                                   # :277
    o = o.transpose(1, 2).reshape(N, T, C)                                                      # :278, :333
    return F.linear(o, w[f"{p}.out_proj.weight"], w[f"{p}.out_proj.bias"])                      # :334


def encoder_layer(w: Dict[str, torch.Tensor], i: int, cfg: ClipVisionConfig, x: torch.Tensor, sdpa: bool = False) -> torch.Tensor:
    """CLIPEncoderLayer.forward (:363-386) with CLIPMLP (:347-351): pre-norm attention and MLP, each with a residual."""
    p = f"vision_model.encoder.layers.{i}"
    eps = cfg.layer_norm_eps
    C = x.shape[-1]
    h = F.layer_norm(x, (C,), w[f"{p}.layer_norm1.weight"], w[f"{p}.layer_norm1.bias"], eps)   # :369
    x = x + attention(w, f"{p}.self_attn", cfg, h, sdpa)                                       # :371-377
    h = F.layer_norm(x, (C,), w[f"{p}.layer_norm2.weight"], w[f"{p}.layer_norm2.bias"], eps)   # :380
    h = F.linear(h, w[f"{p}.mlp.fc1.weight"], w[f"{p}.mlp.fc1.bias"])                          # :348
    h = _act(h, cfg.hidden_act)                                                                 # :349
    return x + F.linear(h, w[f"{p}.mlp.fc2.weight"], w[f"{p}.mlp.fc2.bias"])                   # :350, :381-382


@torch.no_grad()
def clip_vision_forward(sd: Dict[str, torch.Tensor], cfg: ClipVisionConfig, pixel_values: torch.Tensor,
                        dtype: torch.dtype = torch.float32, sdpa: bool = False) -> Tuple[torch.Tensor, torch.Tensor]:
    """CLIPVisionModelWithProjection.forward (:1036-1075) -> CLIPVisionTransformer.forward (:667-690). Computes on the
    device of `pixel_values` in `dtype`; returns (image_embeds [N, projection_dim], last_hidden_state [N, P + 1, C])."""
    dev = pixel_values.device
    w = {k: v.to(dev, dtype) for k, v in sd.items() if k != "vision_model.embeddings.position_ids"}
    C = cfg.hidden_size
    x = embeddings(w, cfg, pixel_values.to(dtype))                                                   # :676
    x = F.layer_norm(x, (C,), w["vision_model.pre_layrnorm.weight"], w["vision_model.pre_layrnorm.bias"],
                     cfg.layer_norm_eps)                                                             # :677
    for i in range(cfg.num_hidden_layers):                                                           # CLIPEncoder :477-506
        x = encoder_layer(w, i, cfg, x, sdpa)
    last = x                                                                                         # :684 (not post-normalised)
    pooled = F.layer_norm(last[:, 0, :], (C,), w["vision_model.post_layernorm.weight"],
                          w["vision_model.post_layernorm.bias"], cfg.layer_norm_eps)                 # :685-686
    return F.linear(pooled, w["visual_projection.weight"]), last                                    # :1068-1069
