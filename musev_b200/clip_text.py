"""The prompt encoder on the engine: `transformers.CLIPTextModel` (CLIP text tower, models/clip/modeling_clip.py), as MuseV
runs it through `encode_weighted_prompt` (musev/utils/text_emb_util.py:178-215,352-420): `pipe.text_encoder(ids)[0]` once
per 77-token chunk of the prompt and of the negative prompt. Tokenization stays with the caller: the engine takes
`input_ids`."""
from __future__ import annotations

from collections import OrderedDict
from dataclasses import asdict
from types import SimpleNamespace
from typing import Dict, Optional, Tuple, Union

import torch

from ._capi import EngineModel, MvbControlnetArgs, _is_f32, make_config
from .schema import CLIP_ACT_CODES, ClipTextConfig, clip_text_config, clip_text_param_shapes


class BaseModelOutputWithPooling(OrderedDict):
    """The fields of transformers' `BaseModelOutputWithPooling`: attribute access, and `[i]` / `to_tuple()` over the fields
    that are not None (last_hidden_state, pooler_output), like `ModelOutput`."""

    def __init__(self, last_hidden_state=None, pooler_output=None, hidden_states=None, attentions=None):
        super().__init__()
        for k, v in (("last_hidden_state", last_hidden_state), ("pooler_output", pooler_output),
                     ("hidden_states", hidden_states), ("attentions", attentions)):
            object.__setattr__(self, k, v)
            if v is not None:
                self[k] = v

    def __getitem__(self, k):
        if isinstance(k, str):
            return super().__getitem__(k)
        return self.to_tuple()[k]

    def to_tuple(self) -> Tuple:
        return tuple(self.values())


class CLIPTextModel(EngineModel):
    """CUDA engine behind the call surface of `transformers.CLIPTextModel`, a drop-in for `pipeline.text_encoder`:

        pipeline.text_encoder = CLIPTextModel.from_state_dict(old.state_dict(), config=old.config)

    Kept: `.config` (vocab_size, hidden_size, max_position_embeddings, eos_token_id, ...), `.dtype`, `.device`, `.eval()`,
    `.to()`, the state-dict names, and `forward(input_ids)` -> `last_hidden_state` [N, L, hidden_size] and `pooler_output`
    [N, hidden_size] in `.dtype` (ordinary tensors: `encode_weighted_prompt` scales `[0]` in place). Not kept: a padding
    `attention_mask` (anything but None or all ones), `position_ids`, `output_hidden_states` (clip_skip) and
    `output_attentions` raise NotImplementedError; MuseV's prompt path passes none of them. The residual stream is fp16, as
    in the reference's fp16 model; every matrix product accumulates in fp32."""

    _create, _workspace, _forward = "mvb_create_clip_text", "mvb_clip_text_workspace_bytes", "mvb_clip_text_forward"
    _ignored = ("text_model.embeddings.position_ids",)   # a persistent buffer in older transformers checkpoints

    def __init__(self, config: Union[ClipTextConfig, Dict, object] = ClipTextConfig(),
                 device: Union[str, torch.device] = "cuda", dtype: torch.dtype = torch.float16):
        self.cfg = clip_text_config(config)
        self.config = SimpleNamespace(**asdict(self.cfg))
        c = self.cfg
        mc = make_config(0, c.eos_token_id, (c.hidden_size, c.intermediate_size, c.max_position_embeddings, c.vocab_size),
                         layers_per_block=c.num_hidden_layers, heads=c.num_attention_heads,
                         norm_num_groups=CLIP_ACT_CODES[c.hidden_act], norm_eps=c.layer_norm_eps)
        super().__init__(mc, device, dtype, unsupported=f"unsupported geometry {self.cfg}")

    @classmethod
    def from_state_dict(cls, state_dict: Dict[str, torch.Tensor], config, device: Union[str, torch.device] = "cuda",
                        dtype: torch.dtype = torch.float16) -> "CLIPTextModel":
        """A loaded model from a `CLIPTextModel.state_dict()` and its config (a transformers `CLIPTextConfig`, a dict or a
        `ClipTextConfig`)."""
        m = cls(config, device=device, dtype=dtype)
        m.load_state_dict(state_dict)
        return m

    def _param_shapes(self):
        return clip_text_param_shapes(self.cfg)

    def load_state_dict(self, state_dict: Dict[str, torch.Tensor], strict: bool = True):
        """As the base class; a missing key raises KeyError naming it, whatever `strict` says (the engine has no
        initialiser for it)."""
        missing = [k for k in self._param_shapes() if k not in state_dict]
        if missing:
            more = f" (and {len(missing) - 1} more)" if len(missing) > 1 else ""
            raise KeyError(f"CLIP text state dict is missing {missing[0]!r}{more}")
        return super().load_state_dict(state_dict, strict)

    @torch.no_grad()
    def forward(self, input_ids: torch.Tensor, attention_mask: Optional[torch.Tensor] = None,
                position_ids: Optional[torch.Tensor] = None, output_attentions: Optional[bool] = None,
                output_hidden_states: Optional[bool] = None, return_dict: Optional[bool] = None):
        """CLIPTextModel.forward: input_ids [N, L], any integer dtype, L <= max_position_embeddings."""
        if output_hidden_states or output_attentions:
            raise NotImplementedError("output_hidden_states / output_attentions (clip_skip) are not available from the engine")
        if position_ids is not None:
            raise NotImplementedError("position_ids are not supported: positions are 0..L-1")
        if attention_mask is not None and not bool((attention_mask == 1).all()):
            raise NotImplementedError("a padding attention_mask is not supported (it changes the rows at padding "
                                      "positions, which the UNet reads); pass None or all ones")
        self._check_loaded()
        c = self.cfg
        if input_ids.dim() != 2 or input_ids.dtype.is_floating_point or input_ids.dtype.is_complex or input_ids.dtype == torch.bool:
            raise ValueError(f"input_ids must be a 2-D integer tensor, got {input_ids.dtype} {tuple(input_ids.shape)}")
        N, L = input_ids.shape
        if L > c.max_position_embeddings:
            raise ValueError(f"Sequence length must be less than max_position_embeddings (got `sequence length`: {L} and "
                             f"max_position_embeddings: {c.max_position_embeddings}")
        if L < 1 or N < 1 or N > 1024:
            raise ValueError(f"1..1024 sequences of at least one token per call, got {tuple(input_ids.shape)}")
        ids = input_ids.to(self.device, torch.int64).contiguous()
        lo, hi = int(ids.min()), int(ids.max())
        if lo < 0 or hi >= c.vocab_size:
            raise IndexError(f"index out of range in self: input_ids span [{lo}, {hi}], vocab_size is {c.vocab_size}")
        last = torch.empty((N, L, c.hidden_size), dtype=self.dtype, device=self.device)
        pooled = torch.empty((N, c.hidden_size), dtype=self.dtype, device=self.device)
        a = MvbControlnetArgs()
        a.sample, a.sample_is_f32 = ids.data_ptr(), 0
        a.NF, a.H, a.W = N, L, 1
        a.n_out = 2
        a.outs[0], a.outs[1] = last.data_ptr(), pooled.data_ptr()
        a.out_is_f32 = _is_f32(last)
        self._launch(a)
        self._keep = ids   # the input must outlive the asynchronous launch
        if return_dict is False:
            return (last, pooled)
        return BaseModelOutputWithPooling(last_hidden_state=last, pooler_output=pooled)

    __call__ = forward
