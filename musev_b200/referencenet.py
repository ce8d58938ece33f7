"""Host mirrors of the two one-shot side paths of the `musev_referencenet*` presets (SURVEY.md section 8(a15) / 8(f)-2).

  * `ReferenceNet2D`   musev/models/referencenet.py:86,640-1127, called once per pipeline call at step 0
                       (musev/pipelines/pipeline_controlnet.py:867-964,1883-1899). The SD-1.5 encoder half + mid block run
                       inside libmusevb200.so (`mvb_referencenet_forward`, the same engine graph as the ControlNet encoder
                       with the musev LayerNorm eps and without condition embedding / zero convolutions).
  * `ImageProjModel`   the IP-Adapter image projection (`ip_adapter.ip_adapter.ImageProjModel`, a pip dependency of the
                       reference: requirements.txt:2; built at musev/models/ip_adapter_loader.py:89-93, called at
                       musev/pipelines/pipeline_controlnet.py:725,745): Linear(1024 -> 4 x 768) + LayerNorm(768), as one
                       wgmma GEMM + one LayerNorm kernel through the op-level C ABI.
There is no CPU / PyTorch fallback.
"""
from __future__ import annotations

from dataclasses import asdict
from types import SimpleNamespace
from typing import Dict, List, Tuple, Union

import torch

from . import ops
from ._capi import EngineModel, MvbControlnetArgs, _is_f32, make_config
# Names callers imported from this module before the binding moved to _capi; they are the binding's own objects.
from ._capi import lib as _lib  # noqa: F401
from .schema import ImageProjConfig, ReferenceNetConfig, image_proj_param_shapes, referencenet_param_shapes


class ReferenceNet2D(EngineModel):
    """CUDA engine behind the call surface of `musev.models.referencenet.ReferenceNet2D` (need_block_embs=True,
    need_self_attn_block_embs=False -- the only configuration the released presets use, referencenet_loader.py:109-118)."""

    _create = "mvb_create_referencenet"
    _workspace, _forward = "mvb_referencenet_workspace_bytes", "mvb_referencenet_forward"

    def __init__(self, config: ReferenceNetConfig, device: Union[str, torch.device] = "cuda", dtype: torch.dtype = torch.float16):
        self.cfg = config
        self.config = SimpleNamespace(**asdict(config))
        self.need_block_embs, self.need_self_attn_block_embs = True, False
        c = make_config(config.in_channels, config.in_channels, config.block_out_channels, config.layers_per_block,
                        config.attention_head_dim, config.cross_attention_dim, config.norm_num_groups, config.norm_eps)
        super().__init__(c, device, dtype)
        self._maps: List[Tuple[int, int]] = [(config.block_out_channels[0], 1)]     # (channels, downscale) of the 12 + 1 maps
        ds, nb = 1, len(config.block_out_channels)
        for i, ch in enumerate(config.block_out_channels):
            for _ in range(config.layers_per_block):
                self._maps.append((ch, ds))
            if i != nb - 1:
                ds *= 2
                self._maps.append((ch, ds))
        self._maps.append((config.block_out_channels[-1], ds))

    @classmethod
    def from_state_dict(cls, state_dict: Dict[str, torch.Tensor], device="cuda", dtype=torch.float16, **config_overrides):
        m = cls(ReferenceNetConfig(**config_overrides), device=device, dtype=dtype)
        m.load_state_dict(state_dict)
        return m

    def _param_shapes(self):
        return referencenet_param_shapes(self.cfg)

    @torch.no_grad()
    def forward(self, sample: torch.Tensor, timestep, encoder_hidden_states: torch.Tensor, class_labels=None,
                timestep_cond=None, attention_mask=None, cross_attention_kwargs=None, added_cond_kwargs=None,
                down_block_additional_residuals=None, mid_block_additional_residual=None,
                down_intrablock_additional_residuals=None, encoder_attention_mask=None, return_dict: bool = True,
                num_frames: int = None, return_ndim: int = 5):
        """Reference: ReferenceNet2D.forward, musev/models/referencenet.py:640-1127. Returns
        (down_block_refer_embs [12 x (b, C, t, h, w)], mid_block_refer_emb, None)."""
        self._check_loaded()
        for name, v in (("class_labels", class_labels), ("timestep_cond", timestep_cond), ("attention_mask", attention_mask),
                        ("added_cond_kwargs", added_cond_kwargs), ("down_block_additional_residuals", down_block_additional_residuals),
                        ("mid_block_additional_residual", mid_block_additional_residual),
                        ("down_intrablock_additional_residuals", down_intrablock_additional_residuals),
                        ("encoder_attention_mask", encoder_attention_mask)):
            if v is not None:
                raise NotImplementedError(f"{name} is not used on MuseV's ReferenceNet path and is not supported")
        if sample.dim() != 4:
            raise ValueError(f"sample must be (b t) c h w, got {tuple(sample.shape)}")
        if return_ndim not in (4, 5):
            raise ValueError(f"reshape_emb only support 4, 5 but given {return_ndim}")     # referencenet.py:1046-1049
        NF, _, H, W = sample.shape
        frames = int(num_frames) if (return_ndim == 5 and num_frames) else 1
        if return_ndim == 5 and not num_frames:
            raise ValueError("num_frames is required for return_ndim=5")
        if encoder_hidden_states.dim() != 3 or encoder_hidden_states.shape[0] != NF:
            raise ValueError("encoder_hidden_states must be [(b t), n_tokens, dim]")
        dev = self.device
        sample = sample.to(dev).contiguous()
        ehs = encoder_hidden_states.to(dev).contiguous()
        t_val = float(timestep.reshape(-1)[0].item()) if torch.is_tensor(timestep) else float(timestep)
        n_out = len(self._maps)
        if return_ndim == 5:
            outs = [torch.empty((NF // frames, c, frames, H // ds, W // ds), device=dev, dtype=self.dtype) for c, ds in self._maps]
        else:
            outs = [torch.empty((NF, c, H // ds, W // ds), device=dev, dtype=self.dtype) for c, ds in self._maps]
        a = MvbControlnetArgs()
        a.sample, a.sample_is_f32 = sample.data_ptr(), _is_f32(sample)
        a.NF, a.H, a.W = NF, H, W
        a.timestep = t_val
        a.encoder_hidden_states, a.ehs_is_f32, a.n_text = ehs.data_ptr(), _is_f32(ehs), ehs.shape[1]
        a.n_out = n_out
        for k in range(n_out):
            a.scales[k] = 1.0
            a.outs[k] = outs[k].data_ptr()
        a.out_is_f32 = _is_f32(outs[0])
        a.out_frames = frames
        self._launch(a)
        self._keep = (sample, ehs)
        return outs[:-1], outs[-1], None          # referencenet.py:1116-1127 (self_attn_block_embs is None)

    __call__ = forward


class ImageProjModel:
    """IP-Adapter image projection on the engine: clip image embedding [N, clip_dim] (or [N, 1, clip_dim]) ->
    [N, tokens, cross_dim]. Weights by the package's state-dict names (`proj.*`, `norm.*`; the reference loads them from
    `ip_adapter_state_dict["image_proj"]`, ip_adapter_loader.py:126)."""

    def __init__(self, config: ImageProjConfig = ImageProjConfig(), device: Union[str, torch.device] = "cuda",
                 dtype: torch.dtype = torch.float16):
        if not torch.cuda.is_available():
            raise RuntimeError("musev_b200 needs a CUDA (sm_90a) device; there is no CPU path")
        if config.clip_embeddings_dim % 64 or config.cross_attention_dim % 8:
            raise ValueError("clip_embeddings_dim must be a multiple of 64 and cross_attention_dim a multiple of 8")
        self.cfg = config
        self.device = torch.device(device if str(device) != "cuda" else f"cuda:{torch.cuda.current_device()}")
        self.dtype = dtype
        self._w: Dict[str, torch.Tensor] = {}

    def load_state_dict(self, state_dict: Dict[str, torch.Tensor], strict: bool = True):
        expected = image_proj_param_shapes(self.cfg)
        missing = [k for k in expected if k not in state_dict]
        unexpected = [k for k in state_dict if k not in expected]
        if strict and (missing or unexpected):
            raise RuntimeError(f"Error(s) in loading state_dict: missing {missing} unexpected {unexpected}")
        for name, shape in expected.items():
            t = state_dict[name]
            if tuple(t.shape) != tuple(shape):
                raise RuntimeError(f"size mismatch for {name}: {tuple(t.shape)} vs {tuple(shape)}")
            # GEMM operand fp16; bias and LayerNorm affine fp32 (the kernels' parameter types)
            self._w[name] = t.to(self.device, torch.float16 if name == "proj.weight" else torch.float32).contiguous()
        return SimpleNamespace(missing_keys=missing, unexpected_keys=unexpected)

    def eval(self):
        return self

    @torch.no_grad()
    def forward(self, image_embeds: torch.Tensor) -> torch.Tensor:
        if not self._w:
            raise RuntimeError("weights not loaded: call load_state_dict first")
        c = self.cfg
        x = image_embeds.to(self.device).reshape(-1, c.clip_embeddings_dim).half().contiguous()
        n = x.shape[0]
        y = ops.conv_gemm(x.view(1, 1, n, c.clip_embeddings_dim), self._w["proj.weight"], bias=self._w["proj.bias"])
        y = ops.layernorm(y.view(n * c.clip_extra_context_tokens, c.cross_attention_dim), self._w["norm.weight"],
                          self._w["norm.bias"], 1e-5)
        return y.view(n, c.clip_extra_context_tokens, c.cross_attention_dim).to(self.dtype)

    __call__ = forward


def ip_adapter_image_emb(image_proj: ImageProjModel, clip_image_embeds: torch.Tensor, n_images: int, batch_size: int,
                         do_classifier_free_guidance: bool = True) -> torch.Tensor:
    """The projection part of `get_ip_adapter_image_emb` (musev/pipelines/pipeline_controlnet.py:719-770) after the CLIP
    vision encoder: project, regroup `(b t) n q -> b (t n) q`, repeat to the batch size and prepend the uncond branch
    `image_proj(zeros)` for CFG."""
    def group(e):
        bt, n, q = e.shape
        e = e.view(bt // n_images, n_images * n, q)
        rep = -(-batch_size // e.shape[0])
        return e.repeat_interleave(rep, dim=0)[:batch_size]                      # align_repeat_tensor_single_dim
    emb = group(image_proj(clip_image_embeds))
    if do_classifier_free_guidance:
        emb = torch.cat([group(image_proj(torch.zeros_like(clip_image_embeds))), emb])
    return emb
