"""Configuration and state-dict schema of the denoiser (names/shapes of `UNet3DConditionModel.state_dict()`) and of
the per-window-step ControlNet encoder that feeds it (SURVEY.md section 8(f), rank 1).

Mirrors what the reference builds in musev/models/unet_3d_condition.py:213-610 for the two released presets
(musev/models/unet_loader.py:232-268); oracle/make_golden.py checks the generated schema against the
reference's own `state_dict()` key by key.
"""
from __future__ import annotations

from collections import OrderedDict
from dataclasses import asdict, dataclass, field, fields
from typing import Dict, Tuple


@dataclass
class UNetConfig:
    in_channels: int = 4
    out_channels: int = 4
    block_out_channels: Tuple[int, ...] = (320, 640, 1280, 1280)
    layers_per_block: int = 2
    attention_head_dim: int = 8          # number of heads in the reference (a diffusers naming accident)
    cross_attention_dim: int = 768
    norm_num_groups: int = 32
    norm_eps: float = 1e-5
    sample_size: int = 64
    # musev switches
    need_transformer_in: bool = True
    use_anivv1_cfg: bool = False
    resnet_2d_skip_time_act: bool = False
    keep_vision_condtion: bool = False
    need_refer_emb: bool = False
    ip_adapter_cross_attn: bool = False
    need_t2i_ip_adapter: bool = True      # reference-only self-attention toward the vision-condition frame
    preset: str = "musev"

    @property
    def heads(self) -> int:
        return self.attention_head_dim

    @property
    def temb_dim(self) -> int:
        return self.block_out_channels[0] * 4

    def to_dict(self):
        return asdict(self)


def preset_config(name: str, **overrides) -> UNetConfig:
    """The two released configurations (musev/models/unet_loader.py:232-268)."""
    if name == "musev":
        cfg = UNetConfig(preset="musev")
    elif name in ("musev_referencenet", "musev_referencenet_pose"):
        cfg = UNetConfig(
            preset="musev_referencenet", need_transformer_in=False, use_anivv1_cfg=True,
            resnet_2d_skip_time_act=True, keep_vision_condtion=True, need_refer_emb=True,
            ip_adapter_cross_attn=True)
    else:
        raise ValueError(
            f"unsupport model_name={name}, only support musev, musev_referencenet, musev_referencenet_pose")
    for k, v in overrides.items():
        if not hasattr(cfg, k):
            raise ValueError(f"unknown config field {k}")
        setattr(cfg, k, tuple(v) if k == "block_out_channels" else v)
    return cfg


def _attn(prefix: str, C: int, kv_dim: int, out: Dict, ip: bool = False):
    out[f"{prefix}.to_q.weight"] = (C, C)
    out[f"{prefix}.to_k.weight"] = (C, kv_dim)
    out[f"{prefix}.to_v.weight"] = (C, kv_dim)
    out[f"{prefix}.to_out.0.weight"] = (C, C)
    out[f"{prefix}.to_out.0.bias"] = (C,)
    if ip:
        out[f"{prefix}.to_k_ip.weight"] = (C, kv_dim)
        out[f"{prefix}.to_v_ip.weight"] = (C, kv_dim)


def _tblock(prefix: str, C: int, cross_dim, out: Dict, ip: bool):
    for n in ("norm1", "norm2", "norm3"):
        out[f"{prefix}.{n}.weight"] = (C,)
        out[f"{prefix}.{n}.bias"] = (C,)
    _attn(f"{prefix}.attn1", C, C, out)
    _attn(f"{prefix}.attn2", C, cross_dim if cross_dim else C, out, ip=ip)
    out[f"{prefix}.ff.net.0.proj.weight"] = (8 * C, C)
    out[f"{prefix}.ff.net.0.proj.bias"] = (8 * C,)
    out[f"{prefix}.ff.net.2.weight"] = (C, 4 * C)
    out[f"{prefix}.ff.net.2.bias"] = (C,)


def _resnet(prefix: str, cin: int, C: int, temb: int, out: Dict):
    out[f"{prefix}.norm1.weight"] = (cin,)
    out[f"{prefix}.norm1.bias"] = (cin,)
    out[f"{prefix}.conv1.weight"] = (C, cin, 3, 3)
    out[f"{prefix}.conv1.bias"] = (C,)
    out[f"{prefix}.time_emb_proj.weight"] = (C, temb)
    out[f"{prefix}.time_emb_proj.bias"] = (C,)
    out[f"{prefix}.norm2.weight"] = (C,)
    out[f"{prefix}.norm2.bias"] = (C,)
    out[f"{prefix}.conv2.weight"] = (C, C, 3, 3)
    out[f"{prefix}.conv2.bias"] = (C,)
    if cin != C:
        out[f"{prefix}.conv_shortcut.weight"] = (C, cin, 1, 1)
        out[f"{prefix}.conv_shortcut.bias"] = (C,)


def _temp_conv(prefix: str, C: int, out: Dict):
    for i, conv_idx in ((1, 2), (2, 3), (3, 3), (4, 3)):
        out[f"{prefix}.conv{i}.0.weight"] = (C,)
        out[f"{prefix}.conv{i}.0.bias"] = (C,)
        out[f"{prefix}.conv{i}.{conv_idx}.weight"] = (C, C, 3, 1, 1)
        out[f"{prefix}.conv{i}.{conv_idx}.bias"] = (C,)
    out[f"{prefix}.temporal_weight"] = (1,)


def _spatial_tfm(prefix: str, C: int, cfg: UNetConfig, out: Dict):
    out[f"{prefix}.norm.weight"] = (C,)
    out[f"{prefix}.norm.bias"] = (C,)
    out[f"{prefix}.proj_in.weight"] = (C, C, 1, 1)
    out[f"{prefix}.proj_in.bias"] = (C,)
    _tblock(f"{prefix}.transformer_blocks.0", C, cfg.cross_attention_dim, out, ip=cfg.ip_adapter_cross_attn)
    out[f"{prefix}.proj_out.weight"] = (C, C, 1, 1)
    out[f"{prefix}.proj_out.bias"] = (C,)


def _temporal_tfm(prefix: str, C: int, cfg: UNetConfig, out: Dict):
    out[f"{prefix}.temporal_weight"] = (1,)
    out[f"{prefix}.norm.weight"] = (C,)
    out[f"{prefix}.norm.bias"] = (C,)
    out[f"{prefix}.proj_in.weight"] = (C, C)
    out[f"{prefix}.proj_in.bias"] = (C,)
    out[f"{prefix}.frame_emb_proj.weight"] = (C, cfg.temb_dim)
    out[f"{prefix}.frame_emb_proj.bias"] = (C,)
    _tblock(f"{prefix}.transformer_blocks.0", C, None, out, ip=False)
    out[f"{prefix}.proj_out.weight"] = (C, C)
    out[f"{prefix}.proj_out.bias"] = (C,)


def _refer_attn(prefix: str, C: int, out: Dict):
    _attn(prefix, C, C, out)


def unet_param_shapes(cfg: UNetConfig) -> "OrderedDict[str, Tuple[int, ...]]":
    """name -> shape for every tensor of the reference `state_dict()` (order is not significant)."""
    out: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    boc = cfg.block_out_channels
    c0, temb = boc[0], cfg.temb_dim
    out["conv_in.weight"] = (c0, cfg.in_channels, 3, 3)
    out["conv_in.bias"] = (c0,)
    for emb in ("time_embedding", "frame_embedding"):
        out[f"{emb}.linear_1.weight"] = (temb, c0)
        out[f"{emb}.linear_1.bias"] = (temb,)
        out[f"{emb}.linear_2.weight"] = (temb, temb)
        out[f"{emb}.linear_2.bias"] = (temb,)
    if cfg.need_transformer_in:
        _temporal_tfm("transformer_in", c0, cfg, out)
    if cfg.need_refer_emb:
        _refer_attn("first_refer_emb_attns", c0, out)
        _refer_attn("mid_block_refer_emb_attns", boc[-1], out)
    nb = len(boc)
    # down
    ch = c0
    for i in range(nb):
        cin, ch = ch, boc[i]
        final = i == nb - 1
        has_attn = not final
        for j in range(cfg.layers_per_block):
            _resnet(f"down_blocks.{i}.resnets.{j}", cin if j == 0 else ch, ch, temb, out)
            _temp_conv(f"down_blocks.{i}.temp_convs.{j}", ch, out)
            if has_attn:
                _spatial_tfm(f"down_blocks.{i}.attentions.{j}", ch, cfg, out)
                _temporal_tfm(f"down_blocks.{i}.temp_attentions.{j}", ch, cfg, out)
        if not final:
            out[f"down_blocks.{i}.downsamplers.0.conv.weight"] = (ch, ch, 3, 3)
            out[f"down_blocks.{i}.downsamplers.0.conv.bias"] = (ch,)
        if cfg.need_refer_emb:
            for k in range(cfg.layers_per_block + (0 if final else 1)):
                _refer_attn(f"down_blocks.{i}.refer_emb_attns.{k}", ch, out)
    # mid
    cm = boc[-1]
    _resnet("mid_block.resnets.0", cm, cm, temb, out)
    _temp_conv("mid_block.temp_convs.0", cm, out)
    _spatial_tfm("mid_block.attentions.0", cm, cfg, out)
    _temporal_tfm("mid_block.temp_attentions.0", cm, cfg, out)
    _resnet("mid_block.resnets.1", cm, cm, temb, out)
    _temp_conv("mid_block.temp_convs.1", cm, out)
    # up
    rev = list(reversed(boc))
    ch = rev[0]
    for i in range(nb):
        prev, ch = ch, rev[i]
        cin_block = rev[min(i + 1, nb - 1)]
        has_attn = i > 0
        final = i == nb - 1
        for j in range(cfg.layers_per_block + 1):
            skip = cin_block if j == cfg.layers_per_block else ch
            rin = prev if j == 0 else ch
            _resnet(f"up_blocks.{i}.resnets.{j}", rin + skip, ch, temb, out)
            _temp_conv(f"up_blocks.{i}.temp_convs.{j}", ch, out)
            if has_attn:
                _spatial_tfm(f"up_blocks.{i}.attentions.{j}", ch, cfg, out)
                _temporal_tfm(f"up_blocks.{i}.temp_attentions.{j}", ch, cfg, out)
        if not final:
            out[f"up_blocks.{i}.upsamplers.0.conv.weight"] = (ch, ch, 3, 3)
            out[f"up_blocks.{i}.upsamplers.0.conv.bias"] = (ch,)
    out["conv_norm_out.weight"] = (c0,)
    out["conv_norm_out.bias"] = (c0,)
    out["conv_out.weight"] = (cfg.out_channels, c0, 3, 3)
    out["conv_out.bias"] = (cfg.out_channels,)
    return out


def refer_emb_shapes(cfg: UNetConfig, h: int, w: int):
    """Shapes [C, h, w] of the 12 down-block ReferenceNet maps + the mid map the UNet consumes
    (musev/models/referencenet.py:1116-1127; consumed at unet_3d_condition.py:1052-1095,1176-1187)."""
    boc = cfg.block_out_channels
    shapes = [(boc[0], h, w)]
    hh, ww = h, w
    for i, c in enumerate(boc):
        final = i == len(boc) - 1
        for _ in range(cfg.layers_per_block):
            shapes.append((c, hh, ww))
        if not final:
            hh, ww = hh // 2, ww // 2
            shapes.append((c, hh, ww))
    mid = (boc[-1], hh, ww)
    return shapes, mid


# ------------------------------------------------------------------------------------------------ ControlNet (8f-1)
@dataclass
class ControlNetConfig:
    """diffusers `ControlNetModel.__init__` defaults for SD-1.5 ControlNets (models/controlnet.py:181-262)."""
    in_channels: int = 4
    conditioning_channels: int = 3
    block_out_channels: Tuple[int, ...] = (320, 640, 1280, 1280)
    layers_per_block: int = 2
    attention_head_dim: int = 8          # number of heads, as in UNetConfig
    cross_attention_dim: int = 768
    norm_num_groups: int = 32
    norm_eps: float = 1e-5
    conditioning_embedding_out_channels: Tuple[int, ...] = (16, 32, 96, 256)
    resnet_2d_skip_time_act: bool = False   # lets the oracle reuse the UNet's ResnetBlock2D restatement

    @property
    def heads(self) -> int:
        return self.attention_head_dim

    @property
    def temb_dim(self) -> int:
        return self.block_out_channels[0] * 4


def _vanilla_tfm(prefix: str, C: int, cross_dim: int, out: Dict):
    out[f"{prefix}.norm.weight"] = (C,)
    out[f"{prefix}.norm.bias"] = (C,)
    out[f"{prefix}.proj_in.weight"] = (C, C, 1, 1)
    out[f"{prefix}.proj_in.bias"] = (C,)
    _tblock(f"{prefix}.transformer_blocks.0", C, cross_dim, out, ip=False)
    out[f"{prefix}.proj_out.weight"] = (C, C, 1, 1)
    out[f"{prefix}.proj_out.bias"] = (C,)


def controlnet_param_shapes(cfg: ControlNetConfig) -> "OrderedDict[str, Tuple[int, ...]]":
    """name -> shape of the reference `ControlNetModel.state_dict()` (diffusers models/controlnet.py:181-447):
    SD-1.5 encoder half (3 x CrossAttnDownBlock2D + DownBlock2D + UNetMidBlock2DCrossAttn), the conditioning
    embedding and the 12 + 1 zero convolutions."""
    out: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    boc = cfg.block_out_channels
    c0, temb = boc[0], cfg.temb_dim
    out["conv_in.weight"] = (c0, cfg.in_channels, 3, 3)
    out["conv_in.bias"] = (c0,)
    out["time_embedding.linear_1.weight"] = (temb, c0)
    out["time_embedding.linear_1.bias"] = (temb,)
    out["time_embedding.linear_2.weight"] = (temb, temb)
    out["time_embedding.linear_2.bias"] = (temb,)
    ce = cfg.conditioning_embedding_out_channels
    out["controlnet_cond_embedding.conv_in.weight"] = (ce[0], cfg.conditioning_channels, 3, 3)
    out["controlnet_cond_embedding.conv_in.bias"] = (ce[0],)
    for i in range(len(ce) - 1):
        out[f"controlnet_cond_embedding.blocks.{2 * i}.weight"] = (ce[i], ce[i], 3, 3)
        out[f"controlnet_cond_embedding.blocks.{2 * i}.bias"] = (ce[i],)
        out[f"controlnet_cond_embedding.blocks.{2 * i + 1}.weight"] = (ce[i + 1], ce[i], 3, 3)
        out[f"controlnet_cond_embedding.blocks.{2 * i + 1}.bias"] = (ce[i + 1],)
    out["controlnet_cond_embedding.conv_out.weight"] = (c0, ce[-1], 3, 3)
    out["controlnet_cond_embedding.conv_out.bias"] = (c0,)
    nb = len(boc)
    taps = [c0]                     # channels of the 12 residual taps (conv_in output first)
    ch = c0
    for i in range(nb):
        cin, ch = ch, boc[i]
        final = i == nb - 1
        for j in range(cfg.layers_per_block):
            _resnet(f"down_blocks.{i}.resnets.{j}", cin if j == 0 else ch, ch, temb, out)
            if not final:
                _vanilla_tfm(f"down_blocks.{i}.attentions.{j}", ch, cfg.cross_attention_dim, out)
            taps.append(ch)
        if not final:
            out[f"down_blocks.{i}.downsamplers.0.conv.weight"] = (ch, ch, 3, 3)
            out[f"down_blocks.{i}.downsamplers.0.conv.bias"] = (ch,)
            taps.append(ch)
    cm = boc[-1]
    _resnet("mid_block.resnets.0", cm, cm, temb, out)
    _vanilla_tfm("mid_block.attentions.0", cm, cfg.cross_attention_dim, out)
    _resnet("mid_block.resnets.1", cm, cm, temb, out)
    for k, c in enumerate(taps):
        out[f"controlnet_down_blocks.{k}.weight"] = (c, c, 1, 1)
        out[f"controlnet_down_blocks.{k}.bias"] = (c,)
    out["controlnet_mid_block.weight"] = (cm, cm, 1, 1)
    out["controlnet_mid_block.bias"] = (cm,)
    return out


# ------------------------------------------------------------------------------------------------ ReferenceNet (8f-2)
@dataclass
class ReferenceNetConfig(ControlNetConfig):
    """`ReferenceNet2D` as `load_referencenet_by_name("musev_referencenet")` builds it (musev/models/referencenet_loader.py
    :109-118: need_block_embs=True, need_self_attn_block_embs=False) from an SD-1.5 `unet/config.json`: the encoder half +
    mid block of the 2-D UNet; conv_norm_out / conv_out / up_blocks are set to None (referencenet.py:624-636)."""


def referencenet_param_shapes(cfg: ReferenceNetConfig) -> "OrderedDict[str, Tuple[int, ...]]":
    """name -> shape of the reference `ReferenceNet2D.state_dict()` (296 tensors at SD-1.5 size): conv_in, time_embedding,
    down_blocks (3 x CrossAttnDownBlock2D + DownBlock2D), mid_block (musev/models/referencenet.py:213-636)."""
    full = controlnet_param_shapes(cfg)
    return OrderedDict((k, v) for k, v in full.items()
                       if not (k.startswith("controlnet_cond_embedding.") or k.startswith("controlnet_down_blocks.")
                               or k.startswith("controlnet_mid_block.")))


@dataclass
class ImageProjConfig:
    """`ImageProjModel` of the IP-Adapter package (ip_adapter/ip_adapter.py, tencent-ailab/IP-Adapter@main -- a pip
    dependency of the reference, requirements.txt:2, not vendored) with the arguments the reference passes
    (musev/models/ip_adapter_loader.py:89-93)."""
    cross_attention_dim: int = 768
    clip_embeddings_dim: int = 1024
    clip_extra_context_tokens: int = 4


def image_proj_param_shapes(cfg: ImageProjConfig) -> "OrderedDict[str, Tuple[int, ...]]":
    out: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    out["proj.weight"] = (cfg.clip_extra_context_tokens * cfg.cross_attention_dim, cfg.clip_embeddings_dim)
    out["proj.bias"] = (cfg.clip_extra_context_tokens * cfg.cross_attention_dim,)
    out["norm.weight"] = (cfg.cross_attention_dim,)
    out["norm.bias"] = (cfg.cross_attention_dim,)
    return out


# ------------------------------------------------------------------------------------------------ VAE (8f-3)
@dataclass
class VAEConfig:
    """SD-1.5 `vae/config.json` as `AutoencoderKL.__init__` takes it (diffusers models/autoencoder_kl.py:65-118). Both halves
    are built: the encoder (+ quant_conv, `vae_encoder_param_shapes`) and the decoder (+ post_quant_conv,
    `vae_decoder_param_shapes`)."""
    in_channels: int = 3
    out_channels: int = 3
    latent_channels: int = 4
    block_out_channels: Tuple[int, ...] = (128, 256, 512, 512)
    layers_per_block: int = 2
    norm_num_groups: int = 32
    scaling_factor: float = 0.18215
    # SD-1.5's vae/config.json (diffusers' class default is 32): the tile size of tiled mode, in image pixels
    sample_size: int = 512


def _vae_resnet(out, p, cin, c):
    out[f"{p}.norm1.weight"] = (cin,)
    out[f"{p}.norm1.bias"] = (cin,)
    out[f"{p}.conv1.weight"] = (c, cin, 3, 3)
    out[f"{p}.conv1.bias"] = (c,)
    out[f"{p}.norm2.weight"] = (c,)
    out[f"{p}.norm2.bias"] = (c,)
    out[f"{p}.conv2.weight"] = (c, c, 3, 3)
    out[f"{p}.conv2.bias"] = (c,)
    if cin != c:
        out[f"{p}.conv_shortcut.weight"] = (c, cin, 1, 1)
        out[f"{p}.conv_shortcut.bias"] = (c,)


def _vae_mid(out, p, cm):
    """UNetMidBlock2D of either half: resnet, single-head Attention (GroupNorm, biased q/k/v/out), resnet."""
    _vae_resnet(out, f"{p}.mid_block.resnets.0", cm, cm)
    a = f"{p}.mid_block.attentions.0"
    out[f"{a}.group_norm.weight"] = (cm,)
    out[f"{a}.group_norm.bias"] = (cm,)
    for n in ("to_q", "to_k", "to_v", "to_out.0"):
        out[f"{a}.{n}.weight"] = (cm, cm)
        out[f"{a}.{n}.bias"] = (cm,)
    _vae_resnet(out, f"{p}.mid_block.resnets.1", cm, cm)


def vae_decoder_param_shapes(cfg: VAEConfig) -> "OrderedDict[str, Tuple[int, ...]]":
    """name -> shape of the `post_quant_conv.*` and `decoder.*` entries of the reference `AutoencoderKL.state_dict()`
    (diffusers models/vae.py:201-263; 138 tensors at SD-1.5 size)."""
    out: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    boc = cfg.block_out_channels
    zc, cm = cfg.latent_channels, boc[-1]
    out["post_quant_conv.weight"] = (zc, zc, 1, 1)
    out["post_quant_conv.bias"] = (zc,)
    out["decoder.conv_in.weight"] = (cm, zc, 3, 3)
    out["decoder.conv_in.bias"] = (cm,)
    _vae_mid(out, "decoder", cm)
    ch = cm
    nb = len(boc)
    for i in range(nb):
        prev, ch = ch, boc[nb - 1 - i]
        for j in range(cfg.layers_per_block + 1):
            _vae_resnet(out, f"decoder.up_blocks.{i}.resnets.{j}", prev if j == 0 else ch, ch)
        if i != nb - 1:
            out[f"decoder.up_blocks.{i}.upsamplers.0.conv.weight"] = (ch, ch, 3, 3)
            out[f"decoder.up_blocks.{i}.upsamplers.0.conv.bias"] = (ch,)
    out["decoder.conv_norm_out.weight"] = (boc[0],)
    out["decoder.conv_norm_out.bias"] = (boc[0],)
    out["decoder.conv_out.weight"] = (cfg.out_channels, boc[0], 3, 3)
    out["decoder.conv_out.bias"] = (cfg.out_channels,)
    return out


def vae_encoder_param_shapes(cfg: VAEConfig) -> "OrderedDict[str, Tuple[int, ...]]":
    """name -> shape of the `encoder.*` and `quant_conv.*` entries of the reference `AutoencoderKL.state_dict()`
    (diffusers models/vae.py:65-131, autoencoder_kl.py:101; 108 tensors at SD-1.5 size)."""
    out: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    boc = cfg.block_out_channels
    zc2, cm = 2 * cfg.latent_channels, boc[-1]
    out["encoder.conv_in.weight"] = (boc[0], cfg.in_channels, 3, 3)
    out["encoder.conv_in.bias"] = (boc[0],)
    ch = boc[0]
    nb = len(boc)
    for i in range(nb):
        prev, ch = ch, boc[i]
        for j in range(cfg.layers_per_block):
            _vae_resnet(out, f"encoder.down_blocks.{i}.resnets.{j}", prev if j == 0 else ch, ch)
        if i != nb - 1:
            out[f"encoder.down_blocks.{i}.downsamplers.0.conv.weight"] = (ch, ch, 3, 3)
            out[f"encoder.down_blocks.{i}.downsamplers.0.conv.bias"] = (ch,)
    _vae_mid(out, "encoder", cm)
    out["encoder.conv_norm_out.weight"] = (cm,)
    out["encoder.conv_norm_out.bias"] = (cm,)
    out["encoder.conv_out.weight"] = (zc2, cm, 3, 3)
    out["encoder.conv_out.bias"] = (zc2,)
    out["quant_conv.weight"] = (zc2, zc2, 1, 1)
    out["quant_conv.bias"] = (zc2,)
    return out


# ------------------------------------------------------------------------------------------------ PoseGuider
@dataclass
class PoseGuiderConfig:
    """Constructor arguments of `musev.models.controlnet.PoseGuider` (musev/models/controlnet.py:326-359). The class default
    is (16, 32, 64, 128); scripts/inference/video2video.py:1024-1030 builds (16, 32, 96, 256) -> 320."""
    conditioning_embedding_channels: int = 320
    conditioning_channels: int = 3
    block_out_channels: Tuple[int, ...] = (16, 32, 64, 128)


def pose_guider_layers(cfg: PoseGuiderConfig):
    """(name, cin, cout, stride) of the PoseGuider's 3x3 convolutions in forward order; SiLU follows all but conv_out."""
    boc = cfg.block_out_channels
    out = [("conv_in", cfg.conditioning_channels, boc[0], 1)]
    for i in range(len(boc) - 1):
        out.append((f"blocks.{2 * i}", boc[i], boc[i], 1))
        out.append((f"blocks.{2 * i + 1}", boc[i], boc[i + 1], 2))
    out.append(("conv_out", boc[-1], cfg.conditioning_embedding_channels, 1))
    return out


def pose_guider_param_shapes(cfg: PoseGuiderConfig) -> "OrderedDict[str, Tuple[int, ...]]":
    """name -> shape of the reference `PoseGuider.state_dict()`: a weight and a bias per convolution, 4 len(block_out_channels)
    tensors."""
    out: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    for name, cin, cout, _ in pose_guider_layers(cfg):
        out[f"{name}.weight"] = (cout, cin, 3, 3)
        out[f"{name}.bias"] = (cout,)
    return out


# ------------------------------------------------------------------------------------------------ CLIP vision tower
CLIP_ACT_CODES = {"gelu": 2, "quick_gelu": 3}   # transformers ACT2FN name -> conv_gemm epilogue act code


@dataclass
class ClipVisionConfig:
    """The `transformers.CLIPVisionConfig` fields `CLIPVisionModelWithProjection` computes with. The defaults are the
    IP-Adapter SD-1.5 image encoder (OpenCLIP ViT-H/14): 632 M parameters, 257 tokens per 224 x 224 image."""
    hidden_size: int = 1280
    intermediate_size: int = 5120
    num_hidden_layers: int = 32
    num_attention_heads: int = 16
    num_channels: int = 3
    image_size: int = 224
    patch_size: int = 14
    projection_dim: int = 1024
    hidden_act: str = "gelu"
    layer_norm_eps: float = 1e-5

    @property
    def num_patches(self) -> int:
        return (self.image_size // self.patch_size) ** 2


def _read_config(config, cls):
    """A `cls` dataclass from an instance of it, a transformers config object or a dict (other keys are ignored)."""
    if isinstance(config, cls):
        return cls(**asdict(config))
    get = config.get if isinstance(config, dict) else (lambda k, d=None: getattr(config, k, d))
    return cls(**{f.name: get(f.name, f.default) for f in fields(cls)})


def _check_clip_layers(cfg) -> None:
    """The encoder-layer geometry both CLIP towers share on the engine (conv_gemm K, the attention kernel's head dims)."""
    if cfg.hidden_act not in CLIP_ACT_CODES:
        raise ValueError(f"hidden_act {cfg.hidden_act!r} is not supported (the engine has {sorted(CLIP_ACT_CODES)})")
    C, H = cfg.hidden_size, cfg.num_attention_heads
    if C % 64 or not 64 <= C <= 2048 or H < 1 or C % H or (C // H) % 8 or C // H > 192:
        raise ValueError(f"hidden_size {C} / {H} heads: the hidden size must be a multiple of 64 (at most 2048) and the "
                         "head dim a multiple of 8, at most 192")
    if cfg.intermediate_size % 64 or cfg.intermediate_size < 64 or cfg.num_hidden_layers < 1:
        raise ValueError("intermediate_size must be a positive multiple of 64 and num_hidden_layers at least 1")


def clip_vision_config(config) -> ClipVisionConfig:
    """A `ClipVisionConfig` from a `ClipVisionConfig`, a `transformers.CLIPVisionConfig` or a dict (other keys are ignored).
    Raises ValueError for an activation other than gelu / quick_gelu and for geometry the engine's kernels do not take."""
    cfg = _read_config(config, ClipVisionConfig)
    _check_clip_layers(cfg)
    if cfg.intermediate_size % 64 or cfg.projection_dim % 8 or cfg.image_size % cfg.patch_size or cfg.num_hidden_layers < 1:
        raise ValueError("intermediate_size must be a multiple of 64, projection_dim of 8, image_size of patch_size")
    if not 1 <= cfg.num_channels <= 4:
        raise ValueError(f"num_channels must be 1..4, got {cfg.num_channels}")
    return cfg


def clip_vision_param_shapes(cfg: ClipVisionConfig) -> "OrderedDict[str, Tuple[int, ...]]":
    """name -> shape of `transformers.CLIPVisionModelWithProjection.state_dict()` (models/clip/modeling_clip.py; the
    non-persistent `position_ids` buffer is not part of it)."""
    out: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    C, I, p = cfg.hidden_size, cfg.intermediate_size, cfg.patch_size
    e = "vision_model.embeddings."
    out[e + "class_embedding"] = (C,)
    out[e + "patch_embedding.weight"] = (C, cfg.num_channels, p, p)
    out[e + "position_embedding.weight"] = (cfg.num_patches + 1, C)
    out["vision_model.pre_layrnorm.weight"] = (C,)
    out["vision_model.pre_layrnorm.bias"] = (C,)
    for i in range(cfg.num_hidden_layers):
        q = f"vision_model.encoder.layers.{i}."
        for n in ("k_proj", "v_proj", "q_proj", "out_proj"):
            out[f"{q}self_attn.{n}.weight"] = (C, C)
            out[f"{q}self_attn.{n}.bias"] = (C,)
        out[q + "layer_norm1.weight"] = (C,)
        out[q + "layer_norm1.bias"] = (C,)
        out[q + "mlp.fc1.weight"] = (I, C)
        out[q + "mlp.fc1.bias"] = (I,)
        out[q + "mlp.fc2.weight"] = (C, I)
        out[q + "mlp.fc2.bias"] = (C,)
        out[q + "layer_norm2.weight"] = (C,)
        out[q + "layer_norm2.bias"] = (C,)
    out["vision_model.post_layernorm.weight"] = (C,)
    out["vision_model.post_layernorm.bias"] = (C,)
    out["visual_projection.weight"] = (cfg.projection_dim, C)
    return out


# ------------------------------------------------------------------------------------------------ CLIP text encoder
@dataclass
class ClipTextConfig:
    """The `transformers.CLIPTextConfig` fields `CLIPTextModel` computes with. The defaults are SD-1.5's
    `text_encoder/config.json` (OpenAI CLIP ViT-L/14 text tower): 123 M parameters, 77 positions, and the legacy
    `eos_token_id = 2`, which makes the pooled row the argmax of the ids (the tokenizer's eos, 49407, is the largest id)."""
    vocab_size: int = 49408
    hidden_size: int = 768
    intermediate_size: int = 3072
    num_hidden_layers: int = 12
    num_attention_heads: int = 12
    max_position_embeddings: int = 77
    hidden_act: str = "quick_gelu"
    layer_norm_eps: float = 1e-5
    bos_token_id: int = 0
    eos_token_id: int = 2
    pad_token_id: int = 1


def clip_text_config(config) -> ClipTextConfig:
    """A `ClipTextConfig` from a `ClipTextConfig`, a `transformers.CLIPTextConfig` or a dict (other keys are ignored). Raises
    ValueError for an activation other than gelu / quick_gelu and for geometry the engine's kernels do not take."""
    cfg = _read_config(config, ClipTextConfig)
    _check_clip_layers(cfg)
    if not 1 <= cfg.max_position_embeddings <= 4096 or cfg.vocab_size < 1:
        raise ValueError(f"max_position_embeddings must be 1..4096 and vocab_size positive, got "
                         f"{cfg.max_position_embeddings} / {cfg.vocab_size}")
    if cfg.eos_token_id is None or cfg.eos_token_id < 0:
        raise ValueError(f"eos_token_id must be a non-negative id, got {cfg.eos_token_id}")
    return cfg


def clip_text_param_shapes(cfg: ClipTextConfig) -> "OrderedDict[str, Tuple[int, ...]]":
    """name -> shape of `transformers.CLIPTextModel.state_dict()` (models/clip/modeling_clip.py; the `position_ids` buffer is
    not part of it)."""
    out: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    C, I = cfg.hidden_size, cfg.intermediate_size
    out["text_model.embeddings.token_embedding.weight"] = (cfg.vocab_size, C)
    out["text_model.embeddings.position_embedding.weight"] = (cfg.max_position_embeddings, C)
    for i in range(cfg.num_hidden_layers):
        q = f"text_model.encoder.layers.{i}."
        for n in ("k_proj", "v_proj", "q_proj", "out_proj"):
            out[f"{q}self_attn.{n}.weight"] = (C, C)
            out[f"{q}self_attn.{n}.bias"] = (C,)
        out[q + "layer_norm1.weight"] = (C,)
        out[q + "layer_norm1.bias"] = (C,)
        out[q + "mlp.fc1.weight"] = (I, C)
        out[q + "mlp.fc1.bias"] = (I,)
        out[q + "mlp.fc2.weight"] = (C, I)
        out[q + "mlp.fc2.bias"] = (C,)
        out[q + "layer_norm2.weight"] = (C,)
        out[q + "layer_norm2.bias"] = (C,)
    out["text_model.final_layer_norm.weight"] = (C,)
    out["text_model.final_layer_norm.bias"] = (C,)
    return out


def kohya_text_name_map(cfg: ClipTextConfig) -> "OrderedDict[str, str]":
    """kohya module name (without the `lora_te_` prefix) -> reference weight name, for every linear-layer matrix of the text
    encoder (q / k / v / out_proj, fc1, fc2: the modules kohya's text-encoder LoRAs target): the inverse of
    `name[:-len(".weight")].replace(".", "_")`, which is injective over this schema (asserted)."""
    out: "OrderedDict[str, str]" = OrderedDict()
    for name, shape in clip_text_param_shapes(cfg).items():
        if name.endswith(".weight") and len(shape) == 2 and ".encoder.layers." in name:
            k = name[:-7].replace(".", "_")
            assert k not in out, f"kohya names collide: {out[k]} and {name}"
            out[k] = name
    return out
