"""The IP-Adapter image encoder on the engine: `transformers.CLIPVisionModelWithProjection` (CLIP ViT vision tower + visual
projection, models/clip/modeling_clip.py), as MuseV runs it through MMCM's `ImageClipVisionFeatureExtractor`
(MMCM/mmcm/vision/feature_extractor/clip_vision_extractor.py:54-97; musev/models/ip_adapter_loader.py:52-68) in
`get_ip_adapter_image_emb` (musev/pipelines/pipeline_controlnet.py:686-780). Image preprocessing (`CLIPImageProcessor`)
stays with the caller: the engine takes `pixel_values`."""
from __future__ import annotations

from collections import OrderedDict
from dataclasses import asdict
from types import SimpleNamespace
from typing import Dict, Optional, Tuple, Union

import torch

from ._capi import EngineModel, MvbControlnetArgs, _is_f32, make_config
from .schema import CLIP_ACT_CODES, ClipVisionConfig, clip_vision_config, clip_vision_param_shapes


class CLIPVisionModelOutput(OrderedDict):
    """The fields of transformers' `CLIPVisionModelOutput`: attribute access, and `[i]` / `to_tuple()` over the fields that
    are not None (image_embeds, last_hidden_state), like `ModelOutput`."""

    def __init__(self, image_embeds=None, last_hidden_state=None, hidden_states=None, attentions=None):
        super().__init__()
        for k, v in (("image_embeds", image_embeds), ("last_hidden_state", last_hidden_state),
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


class CLIPVisionModelWithProjection(EngineModel):
    """CUDA engine behind the call surface of `transformers.CLIPVisionModelWithProjection`, a drop-in for the
    `image_encoder` attribute of MMCM's `ImageClipVisionFeatureExtractor`:

        extractor.image_encoder = CLIPVisionModelWithProjection.from_state_dict(old.state_dict(), config=old.config)

    Kept: `.config` (hidden_size, projection_dim, image_size, patch_size, ...), `.dtype`, `.device`, `.eval()`, `.to()`, the
    state-dict names, and `forward(pixel_values)` -> `image_embeds` [N, projection_dim] and `last_hidden_state`
    [N, patches + 1, hidden_size] in `.dtype`. Not kept: `output_hidden_states` / `output_attentions` (only IPAdapterPlus
    reads hidden states, and MuseV's pipeline does not support it) raise NotImplementedError; there is no
    position-embedding interpolation, so pixel_values must be image_size x image_size. The residual stream is fp16, as
    in the reference's fp16 model; every matrix product accumulates in fp32."""

    _create, _workspace, _forward = "mvb_create_clip_vision", "mvb_clip_vision_workspace_bytes", "mvb_clip_vision_forward"
    _ignored = ("vision_model.embeddings.position_ids",)   # a persistent buffer in older transformers checkpoints

    def __init__(self, config: Union[ClipVisionConfig, Dict, object] = ClipVisionConfig(),
                 device: Union[str, torch.device] = "cuda", dtype: torch.dtype = torch.float16):
        self.cfg = clip_vision_config(config)
        self.config = SimpleNamespace(**asdict(self.cfg), num_patches=self.cfg.num_patches)
        c = self.cfg
        mc = make_config(c.num_channels, c.projection_dim, (c.hidden_size, c.intermediate_size, c.patch_size, c.image_size),
                         layers_per_block=c.num_hidden_layers, heads=c.num_attention_heads,
                         norm_num_groups=CLIP_ACT_CODES[c.hidden_act], norm_eps=c.layer_norm_eps)
        super().__init__(mc, device, dtype, unsupported=f"unsupported geometry {self.cfg}")

    @classmethod
    def from_state_dict(cls, state_dict: Dict[str, torch.Tensor], config, device: Union[str, torch.device] = "cuda",
                        dtype: torch.dtype = torch.float16) -> "CLIPVisionModelWithProjection":
        """A loaded model from a `CLIPVisionModelWithProjection.state_dict()` and its config (a transformers
        `CLIPVisionConfig`, a dict or a `ClipVisionConfig`)."""
        m = cls(config, device=device, dtype=dtype)
        m.load_state_dict(state_dict)
        return m

    def _param_shapes(self):
        return clip_vision_param_shapes(self.cfg)

    def load_state_dict(self, state_dict: Dict[str, torch.Tensor], strict: bool = True):
        """As the base class; a missing key raises KeyError naming it, whatever `strict` says (the engine has no
        initialiser for it)."""
        missing = [k for k in self._param_shapes() if k not in state_dict]
        if missing:
            more = f" (and {len(missing) - 1} more)" if len(missing) > 1 else ""
            raise KeyError(f"CLIP vision state dict is missing {missing[0]!r}{more}")
        return super().load_state_dict(state_dict, strict)

    @torch.no_grad()
    def forward(self, pixel_values: torch.Tensor, output_attentions: Optional[bool] = None,
                output_hidden_states: Optional[bool] = None, return_dict: Optional[bool] = None,
                interpolate_pos_encoding: bool = False):
        """CLIPVisionModelWithProjection.forward: pixel_values [N, num_channels, image_size, image_size] fp16 / fp32."""
        if output_hidden_states or output_attentions:
            raise NotImplementedError("output_hidden_states / output_attentions are not available from the engine "
                                      "(only IPAdapterPlus reads hidden states; MuseV's pipeline does not support it)")
        if interpolate_pos_encoding:
            raise NotImplementedError("position-embedding interpolation is not supported")
        self._check_loaded()
        c = self.cfg
        if pixel_values.dim() != 4 or pixel_values.shape[1] != c.num_channels:
            raise ValueError(f"pixel_values must be [N, {c.num_channels}, H, W], got {tuple(pixel_values.shape)}")
        N, _, H, W = pixel_values.shape
        if H != c.image_size or W != c.image_size:
            raise ValueError(f"pixel_values must be {c.image_size} x {c.image_size} (no position-embedding interpolation), "
                             f"got {H} x {W}")
        if N < 1 or N > 1024:
            raise ValueError(f"1..1024 images per call, got {N}")
        x = pixel_values.to(self.device)
        if x.dtype not in (torch.float16, torch.float32):
            x = x.float()
        x = x.contiguous()
        emb = torch.empty((N, c.projection_dim), dtype=self.dtype, device=self.device)
        last = torch.empty((N, c.num_patches + 1, c.hidden_size), dtype=self.dtype, device=self.device)
        a = MvbControlnetArgs()
        a.sample, a.sample_is_f32 = x.data_ptr(), _is_f32(x)
        a.NF, a.H, a.W = N, H, W
        a.n_out = 2
        a.outs[0], a.outs[1] = emb.data_ptr(), last.data_ptr()
        a.out_is_f32 = _is_f32(emb)
        self._launch(a)
        self._keep = x   # the input must outlive the asynchronous launch
        if return_dict is False:
            return (emb, last)
        return CLIPVisionModelOutput(image_embeds=emb, last_hidden_state=last)

    __call__ = forward
