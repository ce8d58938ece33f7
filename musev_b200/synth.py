"""Seeded synthetic weights / inputs (no checkpoints exist offline).

Every tensor is drawn from its own generator seeded by (seed, crc32(name)), on CPU in fp32, so the build
container and the GPU box produce bit-identical values irrespective of creation order. The zero-initialised
tensors of the reference (temporal `proj_out`, `conv4`, ReferEmbFuse `to_out`; SURVEY.md Q5) are drawn non-zero
and `temporal_weight` gets O(1) magnitudes with mixed signs, otherwise the temporal / reference paths would
contribute ~1e-5 and parity tests could not see bugs in them.
"""
from __future__ import annotations

import zlib
from collections import OrderedDict
from typing import Dict, List, Optional, Tuple

import torch

from .schema import (ClipTextConfig, ClipVisionConfig, ControlNetConfig, ImageProjConfig, PoseGuiderConfig, ReferenceNetConfig, UNetConfig,
                     VAEConfig, clip_text_param_shapes, clip_vision_param_shapes, controlnet_param_shapes, image_proj_param_shapes, pose_guider_param_shapes, refer_emb_shapes,
                     referencenet_param_shapes, unet_param_shapes, vae_decoder_param_shapes, vae_encoder_param_shapes)

_BRANCH_OUT = ("conv2.weight", "proj_out.weight", "to_out.0.weight", "ff.net.2.weight", "conv4.3.weight")
# the ControlNet's zero-initialised convolutions (controlnet.py:97-99,425-444) are drawn non-zero for the same reason
_ZERO_INIT = ("controlnet_cond_embedding.conv_out.weight", "controlnet_mid_block.weight")


def _gen(seed: int, name: str) -> torch.Generator:
    g = torch.Generator(device="cpu")
    g.manual_seed((seed * 1_000_003 + zlib.crc32(name.encode())) % (2 ** 63 - 1))
    return g


def make_state_dict(cfg, seed: int = 0, dtype: torch.dtype = torch.float32) -> "OrderedDict[str, torch.Tensor]":
    """Seeded weights for a `UNetConfig` (denoiser), a `ControlNetConfig` (ControlNet encoder), a `ReferenceNetConfig`, an
    `ImageProjConfig` or a `VAEConfig` (the full `AutoencoderKL`: encoder + quant_conv, decoder + post_quant_conv)."""
    sd: "OrderedDict[str, torch.Tensor]" = OrderedDict()
    if isinstance(cfg, ReferenceNetConfig):
        shapes = referencenet_param_shapes(cfg)
    elif isinstance(cfg, ControlNetConfig):
        shapes = controlnet_param_shapes(cfg)
    elif isinstance(cfg, ImageProjConfig):
        shapes = image_proj_param_shapes(cfg)
    elif isinstance(cfg, VAEConfig):
        shapes = OrderedDict(list(vae_encoder_param_shapes(cfg).items()) + list(vae_decoder_param_shapes(cfg).items()))
    else:
        shapes = unet_param_shapes(cfg)
    for name, shape in shapes.items():
        g = _gen(seed, name)
        if name.endswith("temporal_weight"):
            t = torch.empty(shape).uniform_(0.4, 0.9, generator=g)
            if zlib.crc32(name.encode()) & 1:
                t = -t  # the reference applies abs() (musev/models/resnet.py:128, temporal_transformer.py:299)
        elif len(shape) == 1:
            is_norm_w = name.endswith(".weight")
            t = torch.randn(shape, generator=g) * (0.1 if is_norm_w else 0.02)
            if is_norm_w:
                t = t + 1.0
        else:
            fan_in = 1
            for s in shape[1:]:
                fan_in *= s
            gain = 0.5 if (name.endswith(_BRANCH_OUT) or name.endswith(_ZERO_INIT) or name.startswith("controlnet_down_blocks")) else 1.0
            t = torch.randn(shape, generator=g) * (gain / fan_in ** 0.5)
        sd[name] = t.to(dtype)
    return sd


def make_inputs(cfg: UNetConfig, batch: int, frames: int, h: int, w: int, n_vis_cond: int = 1, seed: int = 1234,
                n_ref: int = 1) -> Dict[str, object]:
    """Synthetic call arguments of `UNet3DConditionModel.forward` for one window (SURVEY.md section 8d).

    `sample` already contains the vision-condition frame(s) at the front, as in the pipeline
    (musev/pipelines/pipeline_controlnet.py:1921-1946)."""
    def r(name, *shape, scale=1.0):
        return torch.randn(*shape, generator=_gen(seed, name)) * scale

    T = frames + n_vis_cond
    out: Dict[str, object] = {
        "sample": r("sample", batch, cfg.in_channels, T, h, w),
        "encoder_hidden_states": r("encoder_hidden_states", batch, 77, cfg.cross_attention_dim),
        "sample_index": torch.arange(n_vis_cond, T),
        "vision_conditon_frames_sample_index": torch.arange(n_vis_cond) if n_vis_cond > 0 else None,
    }
    if cfg.ip_adapter_cross_attn:
        out["vision_clip_emb"] = r("vision_clip_emb", batch, 4, cfg.cross_attention_dim)
    if cfg.need_refer_emb:
        shapes, mid = refer_emb_shapes(cfg, h, w)
        out["down_block_refer_embs"] = [r(f"refer{i}", batch, c, n_ref, hh, ww) for i, (c, hh, ww) in enumerate(shapes)]
        out["mid_block_refer_emb"] = r("refer_mid", batch, mid[0], n_ref, mid[1], mid[2])
    return out


def make_controlnet_inputs(cfg: ControlNetConfig, frames: int, h: int, w: int, seed: int = 4321) -> Dict[str, object]:
    """Synthetic call arguments of `ControlNetModel.forward` as `get_controlnet_emb` issues it
    (musev/pipelines/pipeline_controlnet.py:1238-1262): `sample` is `(b t) c h w`, the prompt embedding is repeated
    per frame, the condition image is 8x the latent size."""
    def r(name, *shape, scale=1.0):
        return torch.randn(*shape, generator=_gen(seed, name)) * scale

    return {
        "sample": r("cn_sample", frames, cfg.in_channels, h, w),
        "encoder_hidden_states": r("cn_text", frames, 77, cfg.cross_attention_dim),
        "controlnet_cond": torch.rand(frames, cfg.conditioning_channels, 8 * h, 8 * w, generator=_gen(seed, "cn_cond")),
    }


def make_referencenet_inputs(cfg: ReferenceNetConfig, batch: int, n_ref: int, h: int, w: int, n_tokens: int = 4,
                             seed: int = 2468) -> Dict[str, object]:
    """Synthetic call arguments of `ReferenceNet2D.forward` as `get_referencenet_emb` issues it
    (musev/pipelines/pipeline_controlnet.py:918-929): `sample` = reference-image VAE latents (b t) c h w, timestep 0,
    `encoder_hidden_states` = the IP-Adapter image tokens [(b t), 4 n_img, 768]."""
    def r(name, *shape, scale=1.0):
        return torch.randn(*shape, generator=_gen(seed, name)) * scale

    return {
        "sample": r("rn_sample", batch * n_ref, cfg.in_channels, h, w, scale=0.7),
        "encoder_hidden_states": r("rn_tokens", batch * n_ref, n_tokens, cfg.cross_attention_dim),
        "num_frames": n_ref,
    }


def make_lora_state_dict(cfg: UNetConfig, targets, rank: int = 4, seed: int = 0, amp: float = 0.5,
                         no_alpha=(), f32=(), text_targets=(), prefix: str = "lora_unet") -> "OrderedDict[str, torch.Tensor]":
    """A seeded kohya-style LoRA on the UNet weights `targets` (reference names; matrices, 1x1 and kxk convolutions).

    Every factor is drawn from its own generator (seed, kohya key), like `make_state_dict`. Factors are fp16 unless the
    target is in `f32`; `alpha` = rank / 2 except for targets in `no_alpha`, which get no `.alpha` key. kxk convolutions
    get the LoCon factorisation up [N, r, 1, 1], down [r, Cin, kh, kw]. `amp` sets |scale * up @ down| relative to the
    weight's own draw. `text_targets` is a list of (kohya name after `lora_te_`, out, in) linear layers of a text encoder."""
    shapes = unet_param_shapes(cfg)
    sd: "OrderedDict[str, torch.Tensor]" = OrderedDict()

    def add(mod, up_shape, down_shape, fan_in, dtype, alpha):
        g = _gen(seed, mod + ".lora_down.weight")
        down = torch.randn(down_shape, generator=g) / fan_in ** 0.5
        up = torch.randn(up_shape, generator=_gen(seed, mod + ".lora_up.weight")) * (amp / rank ** 0.5)
        if alpha:
            up = up * 2.0      # alpha / rank = 1 / 2
        sd[mod + ".lora_down.weight"] = down.to(dtype)
        sd[mod + ".lora_up.weight"] = up.to(dtype)
        if alpha:
            sd[mod + ".alpha"] = torch.tensor(rank / 2.0, dtype=dtype)

    for name in targets:
        shape = shapes[name]
        if len(shape) not in (2, 4):
            raise ValueError(f"{name}: LoRA factors exist for 2-D and 4-D weights only, not {shape}")
        mod = f"{prefix}_" + name[:-7].replace(".", "_")
        dtype = torch.float32 if name in f32 else torch.float16
        fan_in = 1
        for s in shape[1:]:
            fan_in *= s
        if len(shape) == 2:
            add(mod, (shape[0], rank), (rank, shape[1]), fan_in, dtype, name not in no_alpha)
        else:
            add(mod, (shape[0], rank, 1, 1), (rank,) + tuple(shape[1:]), fan_in, dtype, name not in no_alpha)
    for mod, n_out, n_in in text_targets:
        add("lora_te_" + mod, (n_out, rank), (rank, n_in), n_in, torch.float16, True)
    return sd


def make_text_encoder(width: int = 64, seed: int = 0) -> torch.nn.Module:
    """A stand-in for `pipeline.text_encoder` with CLIP's module path to one attention: `text_model.encoder.layers.0.
    self_attn.{q,k,v,out}_proj`, fp16 seeded linears. The LoRA key of its k_proj is `lora_te_text_model_encoder_layers_0_
    self_attn_k_proj`."""
    nn = torch.nn
    attn = nn.Module()
    for p in ("q_proj", "k_proj", "v_proj", "out_proj"):
        lin = nn.Linear(width, width, bias=False)
        lin.weight.data = torch.randn(width, width, generator=_gen(seed, "te." + p)).div(width ** 0.5).half()
        setattr(attn, p, lin)
    layer = nn.Module()
    layer.self_attn = attn
    enc = nn.Module()
    enc.layers = nn.ModuleList([layer])
    tm = nn.Module()
    tm.encoder = enc
    root = nn.Module()
    root.text_model = tm
    return root


def make_vae_images(frames: int, H: int, W: int, seed: int = 2469, channels: int = 3) -> torch.Tensor:
    """Seeded images in [-1, 1], what `prepare_image` hands to `vae.encode`: [frames, channels, H, W] fp32."""
    return torch.rand(frames, channels, H, W, generator=torch.Generator().manual_seed(seed)) * 2 - 1


def make_pose_guider_state_dict(cfg: PoseGuiderConfig, seed: int = 0, dtype: torch.dtype = torch.float32,
                                bias_scale: float = 0.05) -> "OrderedDict[str, torch.Tensor]":
    """Seeded weights for a `PoseGuider` (musev/models/controlnet.py:326-359), one generator per name as in `make_state_dict`.
    Every convolution is drawn with unit gain (std 1 / sqrt(fan_in)) and biases with std `bias_scale`. The reference
    zero-initialises `conv_out` (`zero_module`, :352-359); it is drawn non-zero here, otherwise every output is zero and a
    parity test could not see anything."""
    sd: "OrderedDict[str, torch.Tensor]" = OrderedDict()
    for name, shape in pose_guider_param_shapes(cfg).items():
        g = _gen(seed, "pose_guider." + name)
        if len(shape) == 1:
            t = torch.randn(shape, generator=g) * bias_scale
        else:
            t = torch.randn(shape, generator=g) / (shape[1] * 9) ** 0.5
        sd[name] = t.to(dtype)
    return sd


def make_pose_images(frames: int, H: int, W: int, seed: int = 1717, channels: int = 3) -> torch.Tensor:
    """Seeded condition images in [0, 1] (what the pipeline's control-image processor hands the pose guider): [frames,
    channels, H, W] fp32, smooth enough that the stride-2 layers see structure rather than white noise."""
    g = torch.Generator().manual_seed(seed)
    lo = torch.rand(frames, channels, max(1, H // 8), max(1, W // 8), generator=g)
    hi = torch.rand(frames, channels, H, W, generator=g)
    up = torch.nn.functional.interpolate(lo, size=(H, W), mode="bilinear", align_corners=False)
    return (0.75 * up + 0.25 * hi).clamp(0, 1)


def make_pose_guider_emb(frames: int, channels: int, h: int, w: int, seed: int = 5151, scale: float = 0.5) -> torch.Tensor:
    """A seeded stand-in for the UNet's `pose_guider_emb`: [(b t), channels, h, w] fp32."""
    return torch.randn(frames, channels, h, w, generator=torch.Generator().manual_seed(seed)) * scale


def make_clip_vision_state_dict(cfg: ClipVisionConfig, seed: int = 0, dtype: torch.dtype = torch.float32,
                                outlier_channels: int = 0, outlier_offset: float = 40.0) -> "OrderedDict[str, torch.Tensor]":
    """Seeded weights for `CLIPVisionModelWithProjection` (`clip_vision_param_shapes`), one generator per name as in
    `make_state_dict`. Matrices have std 1 / sqrt(fan_in); the two residual-branch outputs (`out_proj`, `fc2`) are scaled by
    1 / sqrt(2 num_hidden_layers), so a 32-layer residual stream stays O(1) and fits fp16 with room to spare. LayerNorm
    weights are 1 + 0.1 N(0, 1), biases 0.02 N(0, 1), the class embedding N(0, 1) and the position embedding 0.5 N(0, 1).

    `outlier_channels` > 0 picks that many channels (seeded) and adds `outlier_offset` to them in the position embedding
    (the input of pre_layrnorm) and in layer 0's fc2 bias, so every later LayerNorm sees a few residual channels with a large
    constant offset, as trained ViTs carry."""
    sd: "OrderedDict[str, torch.Tensor]" = OrderedDict()
    branch_gain = (2.0 * cfg.num_hidden_layers) ** -0.5
    for name, shape in clip_vision_param_shapes(cfg).items():
        g = _gen(seed, "clip_vision." + name)
        if name.endswith("class_embedding"):
            t = torch.randn(shape, generator=g)
        elif name.endswith("position_embedding.weight"):
            t = torch.randn(shape, generator=g) * 0.5
        elif len(shape) == 1:
            t = torch.randn(shape, generator=g) * (0.1 if name.endswith(".weight") else 0.02)
            if name.endswith(".weight"):
                t = t + 1.0
        else:
            fan_in = 1
            for d in shape[1:]:
                fan_in *= d
            gain = branch_gain if name.endswith(("out_proj.weight", "fc2.weight")) else 1.0
            t = torch.randn(shape, generator=g) * (gain / fan_in ** 0.5)
        sd[name] = t
    if outlier_channels > 0:
        ch = torch.randperm(cfg.hidden_size, generator=_gen(seed, "clip_vision.outliers"))[:outlier_channels]
        sd["vision_model.embeddings.position_embedding.weight"][:, ch] += outlier_offset
        sd["vision_model.encoder.layers.0.mlp.fc2.bias"][ch] += outlier_offset
    return OrderedDict((k, v.to(dtype)) for k, v in sd.items())


OPENAI_CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)   # CLIPImageProcessor image_mean / image_std
OPENAI_CLIP_STD = (0.26862954, 0.26130258, 0.27577711)


def make_clip_pixel_values(n: int, image_size: int = 224, seed: int = 3131, channels: int = 3) -> torch.Tensor:
    """Seeded `pixel_values` as `CLIPImageProcessor` returns them: smooth images in [0, 1] normalised with the OpenAI CLIP
    mean / std, [n, channels, image_size, image_size] fp32."""
    g = torch.Generator().manual_seed(seed)
    lo = torch.rand(n, channels, max(1, image_size // 16), max(1, image_size // 16), generator=g)
    hi = torch.rand(n, channels, image_size, image_size, generator=g)
    img = (0.8 * torch.nn.functional.interpolate(lo, size=(image_size, image_size), mode="bilinear", align_corners=False)
           + 0.2 * hi).clamp(0, 1)
    mean = torch.tensor((OPENAI_CLIP_MEAN * 2)[:channels]).view(1, -1, 1, 1)
    std = torch.tensor((OPENAI_CLIP_STD * 2)[:channels]).view(1, -1, 1, 1)
    return (img - mean) / std


def make_clip_text_state_dict(cfg: ClipTextConfig, seed: int = 0, dtype: torch.dtype = torch.float32,
                              outlier_channels: int = 0, outlier_offset: float = 40.0) -> "OrderedDict[str, torch.Tensor]":
    """Seeded weights for `CLIPTextModel` (`clip_text_param_shapes`), one generator per name as in `make_state_dict`.
    Matrices have std 1 / sqrt(fan_in); the residual-branch outputs (`out_proj`, `fc2`) are scaled by
    1 / sqrt(2 num_hidden_layers), so the residual stream stays O(1) over the layers. LayerNorm weights are 1 + 0.1 N(0, 1),
    biases 0.02 N(0, 1), the token embedding N(0, 1) and the position embedding 0.5 N(0, 1).

    `outlier_channels` > 0 picks that many channels (seeded) and adds `outlier_offset` to them in the position embedding and
    in layer 0's fc2 bias, so every LayerNorm sees a few residual channels with a large constant offset."""
    sd: "OrderedDict[str, torch.Tensor]" = OrderedDict()
    branch_gain = (2.0 * cfg.num_hidden_layers) ** -0.5
    for name, shape in clip_text_param_shapes(cfg).items():
        g = _gen(seed, "clip_text." + name)
        if name.endswith("token_embedding.weight"):
            t = torch.randn(shape, generator=g)
        elif name.endswith("position_embedding.weight"):
            t = torch.randn(shape, generator=g) * 0.5
        elif len(shape) == 1:
            t = torch.randn(shape, generator=g) * (0.1 if name.endswith(".weight") else 0.02)
            if name.endswith(".weight"):
                t = t + 1.0
        else:
            gain = branch_gain if name.endswith(("out_proj.weight", "fc2.weight")) else 1.0
            t = torch.randn(shape, generator=g) * (gain / shape[1] ** 0.5)
        sd[name] = t
    if outlier_channels > 0:
        ch = torch.randperm(cfg.hidden_size, generator=_gen(seed, "clip_text.outliers"))[:outlier_channels]
        sd["text_model.embeddings.position_embedding.weight"][:, ch] += outlier_offset
        sd["text_model.encoder.layers.0.mlp.fc2.bias"][ch] += outlier_offset
    return OrderedDict((k, v.to(dtype)) for k, v in sd.items())


def make_input_ids(n: int, L: int, cfg: ClipTextConfig, seed: int = 4747, lengths=None) -> torch.Tensor:
    """Tokenizer-like `input_ids` [n, L] int64, as `pad_tokens_and_weights` (musev/utils/text_emb_util.py:153-175) builds
    them with SD-1.5's tokenizer: bos, `lengths[i]` content ids, then eos up to the end (SD-1.5's pad token is its eos).
    With the legacy `eos_token_id == 2` the tokenizer's ids are used (bos = vocab - 2, eos = vocab - 1, content below them);
    otherwise bos / eos are the config's and content ids lie above both, so argmax and the eos rule pick different rows.
    `lengths` defaults to seeded values in [0, L - 2]."""
    g = torch.Generator().manual_seed(seed)
    V = cfg.vocab_size
    if cfg.eos_token_id == 2:
        bos, eos, lo, hi = V - 2, V - 1, 0, V - 2
    else:
        bos, eos = cfg.bos_token_id, cfg.eos_token_id
        lo, hi = max(bos, eos) + 1, V
    if lengths is None:
        lengths = torch.randint(0, max(1, L - 1), (n,), generator=g).tolist()
    ids = torch.full((n, L), eos, dtype=torch.int64)
    for i, k in enumerate(lengths):
        k = max(0, min(int(k), L - 2))
        ids[i, 0] = bos
        ids[i, 1:1 + k] = torch.randint(lo, hi, (k,), generator=g)
    return ids
