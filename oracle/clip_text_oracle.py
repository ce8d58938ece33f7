"""Plain-torch restatement of `transformers.CLIPTextModel.forward` (models/clip/modeling_clip.py; line numbers below are
transformers 5.5.0, whose arithmetic -- the causal mask, final_layer_norm and both pooling rules -- is the same as the 4.33.1
the reference pins, requirements.txt:15).

`clip_text_forward(sd, cfg, input_ids)` returns (last_hidden_state, pooler_output). By default it computes in fp32;
`dtype=torch.float16` runs it the way the reference runs the model (fp16 weights and activations, eager PyTorch), and
`sdpa=True` uses F.scaled_dot_product_attention with is_causal, transformers' default attention implementation.
"""
from __future__ import annotations

from typing import Dict, Tuple

import torch
import torch.nn.functional as F

from musev_b200.schema import ClipTextConfig
from oracle.clip_vision_oracle import _act


def embeddings(w: Dict[str, torch.Tensor], input_ids: torch.Tensor) -> torch.Tensor:
    """CLIPTextEmbeddings.forward (:234-257): token_embedding[ids] + position_embedding[0..L)."""
    L = input_ids.shape[1]
    tok = F.embedding(input_ids, w["text_model.embeddings.token_embedding.weight"])                # :253
    pos = w["text_model.embeddings.position_embedding.weight"][:L].unsqueeze(0)                    # :255 (position_ids = arange)
    return tok + pos                                                                                # :256


def attention(w: Dict[str, torch.Tensor], p: str, cfg: ClipTextConfig, x: torch.Tensor, sdpa: bool = False) -> torch.Tensor:
    """CLIPAttention.forward (:300-336) with the causal mask of CLIPTextTransformer.forward (:546-557): query q sees keys
    k <= q of its own sequence; softmax(q k^T * d^-0.5 + mask) v per head, out_proj."""
    N, L, C = x.shape
    H = cfg.num_attention_heads
    d = C // H

    def heads(n):
        return F.linear(x, w[f"{p}.{n}.weight"], w[f"{p}.{n}.bias"]).view(N, L, H, d).transpose(1, 2)
    q, k, v = heads("q_proj"), heads("k_proj"), heads("v_proj")
    if sdpa:
        o = F.scaled_dot_product_attention(q, k, v, is_causal=True, scale=d ** -0.5)
    else:
        s = torch.matmul(q, k.transpose(2, 3)) * d ** -0.5                                          # :271
        mask = torch.ones(L, L, dtype=torch.bool, device=x.device).triu(1)
        s = s.masked_fill(mask, torch.finfo(s.dtype).min)                                           # :272-273 (additive mask)
        s = torch.softmax(s, dim=-1, dtype=torch.float32).to(q.dtype)                               # :274
        o = torch.matmul(s, v)                                                                       # :277
    o = o.transpose(1, 2).reshape(N, L, C)
    return F.linear(o, w[f"{p}.out_proj.weight"], w[f"{p}.out_proj.bias"])                          # :334


def encoder_layer(w: Dict[str, torch.Tensor], i: int, cfg: ClipTextConfig, x: torch.Tensor, sdpa: bool = False) -> torch.Tensor:
    """CLIPEncoderLayer.forward (:363-386) with CLIPMLP (:347-351)."""
    p = f"text_model.encoder.layers.{i}"
    eps = cfg.layer_norm_eps
    C = x.shape[-1]
    h = F.layer_norm(x, (C,), w[f"{p}.layer_norm1.weight"], w[f"{p}.layer_norm1.bias"], eps)
    x = x + attention(w, f"{p}.self_attn", cfg, h, sdpa)
    h = F.layer_norm(x, (C,), w[f"{p}.layer_norm2.weight"], w[f"{p}.layer_norm2.bias"], eps)
    h = _act(F.linear(h, w[f"{p}.mlp.fc1.weight"], w[f"{p}.mlp.fc1.bias"]), cfg.hidden_act)
    return x + F.linear(h, w[f"{p}.mlp.fc2.weight"], w[f"{p}.mlp.fc2.bias"])


def pool_index(input_ids: torch.Tensor, eos_token_id: int) -> torch.Tensor:
    """The pooled position per sequence (:564-585): argmax of the ids (first occurrence) when eos_token_id == 2 (legacy
    configs), else the first position holding eos_token_id (0 if there is none)."""
    ids = input_ids.to(torch.int)
    if eos_token_id == 2:
        return ids.argmax(dim=-1)                                                                   # :573
    return (ids == eos_token_id).int().argmax(dim=-1)                                               # :581-583


@torch.no_grad()
def clip_text_forward(sd: Dict[str, torch.Tensor], cfg: ClipTextConfig, input_ids: torch.Tensor,
                      dtype: torch.dtype = torch.float32, sdpa: bool = False) -> Tuple[torch.Tensor, torch.Tensor]:
    """CLIPTextModel.forward -> CLIPTextTransformer.forward (:531-592). Computes on the device of `input_ids` in `dtype`;
    returns (last_hidden_state [N, L, C], pooler_output [N, C])."""
    dev = input_ids.device
    w = {k: v.to(dev, dtype) for k, v in sd.items() if k != "text_model.embeddings.position_ids"}
    x = embeddings(w, input_ids)
    for i in range(cfg.num_hidden_layers):                                                          # CLIPEncoder :477-506
        x = encoder_layer(w, i, cfg, x, sdpa)
    C = cfg.hidden_size
    last = F.layer_norm(x, (C,), w["text_model.final_layer_norm.weight"], w["text_model.final_layer_norm.bias"],
                        cfg.layer_norm_eps)                                                          # :562
    idx = pool_index(input_ids, cfg.eos_token_id).to(dev)
    return last, last[torch.arange(last.shape[0], device=dev), idx]                                 # :571-585
