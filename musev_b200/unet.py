"""Drop-in host mirror of `musev.models.unet_3d_condition.UNet3DConditionModel` (reference file:line below).

The forward runs entirely inside libmusevb200.so (musev_b200/csrc/engine_unet.cu) on the tensors' device pointers; this
class only marshals arguments. There is no PyTorch / CPU fallback: without the library or without a CUDA device it
raises.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from types import SimpleNamespace
from typing import Any, Dict, Optional, Sequence, Tuple, Union

import torch

from ._capi import MAX_REFER, EngineModel, MvbError, MvbNamedTensor, MvbUnetArgs, _is_f32, _named, lib, make_config
# Names callers imported from this module before the binding moved to _capi; they are the binding's own objects.
from ._capi import MvbConfig, lib as _lib  # noqa: F401
from .schema import UNetConfig, preset_config, unet_param_shapes


@dataclass
class UNet3DConditionOutput:
    """musev/models/unet_3d_condition.py:166-176."""
    sample: torch.Tensor

    def __getitem__(self, i):
        return (self.sample,)[i]


def check_pose_guider_emb(emb: torch.Tensor, B: int, T: int, c0: int, H: int, W: int) -> None:
    """`pose_guider_emb` is added to conv_in's output (unet_3d_condition.py:1011-1016): (b t) c h w over every frame of the
    sample, vision-condition frames included, fp16 or fp32. Raises ValueError otherwise."""
    want = (B * T, c0, H, W)
    if tuple(emb.shape) != want:
        raise ValueError(f"pose_guider_emb must be (b t) c h w = {want}, got {tuple(emb.shape)}")
    if emb.dtype not in (torch.float16, torch.float32):
        raise ValueError(f"pose_guider_emb must be float16 or float32, got {emb.dtype}")


def _contiguous_index_range(idx, name) -> Tuple[int, int]:
    """vision_conditon_frames_sample_index -> (first, count); the engine supports a contiguous range."""
    if idx is None:
        return 0, 0
    v = [int(i) for i in torch.as_tensor(idx).reshape(-1).tolist()]
    if not v:
        return 0, 0
    if v != list(range(v[0], v[0] + len(v))):
        raise NotImplementedError(f"{name} must be a contiguous ascending range, got {v}")
    return v[0], len(v)


class UNet3DConditionModel(EngineModel):
    """CUDA engine behind the call surface of the reference model (musev/models/unet_3d_condition.py:179).

    Kept: `forward` signature and return type (:773-803, :1277-1280), `.config`, `.dtype`, `.device`,
    `.ip_adapter_cross_attn`, `.set_skip_temporal_layers` (:1639), `.to()`, `.eval()`, reference state-dict names
    (load_state_dict: from_pretrained_2d / load_state_dict, unet_3d_condition.py:1284-1637).
    """

    _create, _workspace, _forward = "mvb_create", "mvb_workspace_bytes", "mvb_unet_forward"

    def __init__(self, config: UNetConfig, device: Union[str, torch.device] = "cuda", dtype: torch.dtype = torch.float16):
        self.cfg = config
        self.config = SimpleNamespace(**config.to_dict())
        self.ip_adapter_cross_attn = config.ip_adapter_cross_attn
        self.need_refer_emb = config.need_refer_emb
        self.skip_temporal_layers = False
        self.skip_refer_downblock_emb = False
        c = make_config(config.in_channels, config.out_channels, config.block_out_channels, config.layers_per_block,
                        config.attention_head_dim, config.cross_attention_dim, config.norm_num_groups, config.norm_eps,
                        need_transformer_in=config.need_transformer_in, use_anivv1_cfg=config.use_anivv1_cfg,
                        resnet_2d_skip_time_act=config.resnet_2d_skip_time_act,
                        keep_vision_condtion=config.keep_vision_condtion, need_refer_emb=config.need_refer_emb,
                        ip_adapter_cross_attn=config.ip_adapter_cross_attn, need_t2i_ip_adapter=config.need_t2i_ip_adapter)
        super().__init__(c, device, dtype)

    # ------------------------------------------------------------------ construction helpers
    @classmethod
    def from_state_dict(cls, state_dict: Dict[str, torch.Tensor], preset: str = "musev", device="cuda",
                        dtype=torch.float16, **config_overrides) -> "UNet3DConditionModel":
        m = cls(preset_config(preset, **config_overrides), device=device, dtype=dtype)
        m.load_state_dict(state_dict)
        return m

    def _param_shapes(self):
        return unet_param_shapes(self.cfg)

    def set_skip_temporal_layers(self, valid: bool, ignore_names=()):
        """musev/models/unet_3d_condition.py:1639-1661 (temporal layers + ReferenceNet down-block fusion)."""
        self.skip_temporal_layers = bool(valid)
        self.skip_refer_downblock_emb = bool(valid)

    # ------------------------------------------------------------------ forward
    @torch.no_grad()
    def forward(
        self,
        sample: torch.Tensor,
        timestep: Union[torch.Tensor, float, int],
        encoder_hidden_states: torch.Tensor,
        class_labels: Optional[torch.Tensor] = None,
        timestep_cond: Optional[torch.Tensor] = None,
        attention_mask: Optional[torch.Tensor] = None,
        cross_attention_kwargs: Optional[Dict[str, Any]] = None,
        down_block_additional_residuals: Optional[Tuple[torch.Tensor]] = None,
        mid_block_additional_residual: Optional[torch.Tensor] = None,
        return_dict: bool = True,
        sample_index: torch.LongTensor = None,
        vision_condition_frames_sample: torch.Tensor = None,
        vision_conditon_frames_sample_index: torch.LongTensor = None,
        sample_frame_rate: int = 10,
        skip_temporal_layers: bool = None,
        frame_index: torch.LongTensor = None,
        down_block_refer_embs: Optional[Tuple[torch.Tensor]] = None,
        mid_block_refer_emb: Optional[torch.Tensor] = None,
        refer_self_attn_emb=None,
        refer_self_attn_emb_mode: str = "read",
        vision_clip_emb: torch.Tensor = None,
        ip_adapter_scale: float = 1.0,
        face_emb: torch.Tensor = None,
        facein_scale: float = 1.0,
        ip_adapter_face_emb: torch.Tensor = None,
        ip_adapter_face_scale: float = 1.0,
        do_classifier_free_guidance: bool = False,
        pose_guider_emb: torch.Tensor = None,
        cfg_shared_sample: bool = False,
    ):
        """Reference: UNet3DConditionModel.forward, musev/models/unet_3d_condition.py:773-1280.

        `cfg_shared_sample` (not in the reference): the caller guarantees that the two halves of the batch of `sample` are
        equal, as in a CFG batch built from one latent. The engine then runs the layers before the first one that reads a
        per-half input (text tokens, reference maps, pose embedding) on the first half only. Nothing is checked: halves
        that differ give a wrong result. The library refuses the flag for an odd batch."""
        self._check_loaded()
        for name, v in (("class_labels", class_labels), ("timestep_cond", timestep_cond), ("attention_mask", attention_mask),
                        ("frame_index", frame_index), ("refer_self_attn_emb", refer_self_attn_emb),
                        ("face_emb", face_emb), ("ip_adapter_face_emb", ip_adapter_face_emb)):
            if v is not None:
                raise NotImplementedError(f"musev_b200: `{name}` is not used by the released presets and is not supported")
        if skip_temporal_layers is not None:
            self.set_skip_temporal_layers(skip_temporal_layers)
        if encoder_hidden_states.ndim != 3:
            raise ValueError(f"only support ndim in [3, 4], but given {encoder_hidden_states.ndim}")
        if vision_condition_frames_sample is not None:
            # batch_concat_two_tensor_with_index (musev/data/data_util.py:242-292; unet_3d_condition.py:875-882)
            total = sample.shape[2] + vision_condition_frames_sample.shape[2]
            merged = sample.new_zeros(sample.shape[0], sample.shape[1], total, *sample.shape[3:])
            merged[:, :, sample_index.to(sample.device)] = sample
            merged[:, :, vision_conditon_frames_sample_index.to(sample.device)] = vision_condition_frames_sample.to(sample.dtype)
            sample = merged
        dev = self.device
        sample = sample.to(dev).contiguous()
        enc = encoder_hidden_states.to(dev).contiguous()
        B, Cin, T, H, W = sample.shape
        if Cin != self.cfg.in_channels:
            raise ValueError(f"sample has {Cin} channels, model expects {self.cfg.in_channels}")
        keep = [sample, enc]
        a = MvbUnetArgs()
        a.sample, a.sample_is_f32 = sample.data_ptr(), _is_f32(sample)
        a.B, a.T, a.H, a.W = B, T, H, W
        a.timestep = float(timestep.reshape(-1)[0].item()) if torch.is_tensor(timestep) else float(timestep)
        a.encoder_hidden_states, a.ehs_is_f32, a.n_text = enc.data_ptr(), _is_f32(enc), enc.shape[1]
        if enc.shape[0] != B or enc.shape[2] != self.cfg.cross_attention_dim:
            raise ValueError(f"encoder_hidden_states {tuple(enc.shape)} does not match batch {B} / dim {self.cfg.cross_attention_dim}")
        a.has_sample_index = int(sample_index is not None)
        first, n = _contiguous_index_range(vision_conditon_frames_sample_index, "vision_conditon_frames_sample_index")
        a.vis_cond_first, a.n_vis_cond = first, n
        a.sample_frame_rate = float(sample_frame_rate)
        if self.cfg.ip_adapter_cross_attn and vision_clip_emb is not None:
            clip = vision_clip_emb.to(dev).contiguous()
            keep.append(clip)
            a.vision_clip_emb, a.clip_is_f32, a.n_clip = clip.data_ptr(), _is_f32(clip), clip.shape[1]
        a.ip_adapter_scale = float(ip_adapter_scale)
        use_ref = self.cfg.need_refer_emb and down_block_refer_embs is not None and not self.skip_refer_downblock_emb
        if use_ref:
            refs = [r.to(dev).contiguous() for r in down_block_refer_embs]
            keep += refs
            if len(refs) > MAX_REFER:
                raise ValueError("too many down_block_refer_embs")
            a.n_refer = len(refs)
            a.refer_is_f32 = _is_f32(refs[0])
            for i, r in enumerate(refs):
                if _is_f32(r) != a.refer_is_f32 or r.dim() != 5 or r.shape[0] != B:
                    raise ValueError("down_block_refer_embs must be [B, C, t, h, w] tensors of one dtype")
                a.refer_embs[i], a.refer_t[i], a.refer_h[i], a.refer_w[i] = r.data_ptr(), r.shape[2], r.shape[3], r.shape[4]
        if self.cfg.need_refer_emb and mid_block_refer_emb is not None and not self.skip_refer_downblock_emb:
            mr = mid_block_refer_emb.to(dev).contiguous()
            if use_ref and _is_f32(mr) != a.refer_is_f32:
                mr = mr.to(refs[0].dtype)
            keep.append(mr)
            a.refer_is_f32 = _is_f32(mr)
            a.mid_refer_emb, a.mid_refer_t, a.mid_refer_h, a.mid_refer_w = mr.data_ptr(), mr.shape[2], mr.shape[3], mr.shape[4]
        if down_block_additional_residuals is not None:
            res = [r.to(dev).contiguous() for r in down_block_additional_residuals]
            keep += res
            a.n_down_residuals = len(res)
            a.residual_is_f32 = _is_f32(res[0])
            for i, r in enumerate(res):
                a.down_residuals[i] = r.data_ptr()
        if mid_block_additional_residual is not None:
            mres = mid_block_additional_residual.to(dev).contiguous()
            if down_block_additional_residuals is not None:
                mres = mres.to(res[0].dtype)
            keep.append(mres)
            a.residual_is_f32 = _is_f32(mres)
            a.mid_residual = mres.data_ptr()
        if pose_guider_emb is not None:
            check_pose_guider_emb(pose_guider_emb, B, T, self.cfg.block_out_channels[0], H, W)
            pose = pose_guider_emb.to(dev).contiguous()
            keep.append(pose)
            a.pose_guider_emb, a.pose_is_f32 = pose.data_ptr(), _is_f32(pose)
        a.skip_temporal_layers = int(self.skip_temporal_layers)
        a.cfg_shared_sample = int(cfg_shared_sample)
        out = torch.empty((B, self.cfg.out_channels, T, H, W), dtype=sample.dtype, device=dev)
        a.out, a.out_is_f32 = out.data_ptr(), _is_f32(out)
        self._launch(a)
        self._keep = keep  # inputs must outlive the asynchronous launch sequence
        if skip_temporal_layers is not None:
            self.set_skip_temporal_layers(not skip_temporal_layers)   # unet_3d_condition.py:1275-1276
        if not return_dict:
            return (out,)
        return UNet3DConditionOutput(sample=out)

    __call__ = forward

    # ------------------------------------------------------------------ LoRA (musev_b200/lora.py is the public surface)
    # ------------------------------------------------------------------ debug
    def debug_taps(self) -> Dict[str, torch.Tensor]:
        """Layer outputs of the last forward as [(b t), C, h*w]-ordered channels-last copies (fp32, [rows, C])."""
        l = lib()
        out = {}
        torch.cuda.synchronize()
        base = self._ws.data_ptr()
        for i in range(l.mvb_debug_num_taps(self._h)):
            name = C.create_string_buffer(128)
            ptr, rows, ch = C.c_void_p(), C.c_longlong(), C.c_int()
            l.mvb_debug_tap(self._h, i, name, 128, C.byref(ptr), C.byref(rows), C.byref(ch))
            off = ptr.value - base
            n = rows.value * ch.value
            view = self._ws[off:off + 2 * n].view(torch.float16).view(rows.value, ch.value)
            out[name.value.decode()] = view.float().clone()
        return out
