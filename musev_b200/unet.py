"""Drop-in host mirror of `musev.models.unet_3d_condition.UNet3DConditionModel` (reference file:line below).

The forward runs entirely inside libmusevb200.so (musev_b200/csrc/engine.cu) on the tensors' device pointers; this
class only marshals arguments. There is no PyTorch / CPU fallback: without the library or without a CUDA device it
raises.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from types import SimpleNamespace
from typing import Any, Dict, Optional, Sequence, Tuple, Union

import torch

from . import _capi
from .schema import UNetConfig, preset_config, unet_param_shapes


class MvbConfig(C.Structure):
    _fields_ = [
        ("in_channels", C.c_int), ("out_channels", C.c_int), ("num_blocks", C.c_int),
        ("block_out_channels", C.c_int * 4), ("layers_per_block", C.c_int), ("heads", C.c_int),
        ("cross_attention_dim", C.c_int), ("norm_num_groups", C.c_int), ("norm_eps", C.c_float),
        ("need_transformer_in", C.c_int), ("use_anivv1_cfg", C.c_int), ("resnet_2d_skip_time_act", C.c_int),
        ("keep_vision_condtion", C.c_int), ("need_refer_emb", C.c_int), ("ip_adapter_cross_attn", C.c_int),
        ("need_t2i_ip_adapter", C.c_int),
    ]


MAX_REFER = 16


class MvbUnetArgs(C.Structure):
    _fields_ = [
        ("sample", C.c_void_p), ("sample_is_f32", C.c_int),
        ("B", C.c_int), ("T", C.c_int), ("H", C.c_int), ("W", C.c_int),
        ("timestep", C.c_float),
        ("encoder_hidden_states", C.c_void_p), ("ehs_is_f32", C.c_int), ("n_text", C.c_int),
        ("has_sample_index", C.c_int),
        ("n_vis_cond", C.c_int), ("vis_cond_first", C.c_int),
        ("sample_frame_rate", C.c_float),
        ("vision_clip_emb", C.c_void_p), ("clip_is_f32", C.c_int), ("n_clip", C.c_int), ("ip_adapter_scale", C.c_float),
        ("n_refer", C.c_int),
        ("refer_embs", C.c_void_p * MAX_REFER), ("refer_t", C.c_int * MAX_REFER), ("refer_h", C.c_int * MAX_REFER),
        ("refer_w", C.c_int * MAX_REFER),
        ("mid_refer_emb", C.c_void_p), ("mid_refer_t", C.c_int), ("mid_refer_h", C.c_int), ("mid_refer_w", C.c_int),
        ("refer_is_f32", C.c_int),
        ("n_down_residuals", C.c_int), ("down_residuals", C.c_void_p * MAX_REFER),
        ("mid_residual", C.c_void_p), ("residual_is_f32", C.c_int),
        ("skip_temporal_layers", C.c_int),
        ("out", C.c_void_p), ("out_is_f32", C.c_int),
        ("pose_guider_emb", C.c_void_p), ("pose_is_f32", C.c_int),
    ]


class MvbNamedTensor(C.Structure):
    _fields_ = [("name", C.c_char_p), ("device_ptr", C.c_void_p), ("is_f32", C.c_int), ("ndim", C.c_int),
                ("shape", C.c_longlong * 5)]


_declared = False
PACK_BATCH_BYTES = 512 << 20     # source bytes staged on the device per mvb_load_weights call


def load_weights_batched(handle, named_tensors, device) -> None:
    """Feeds (name, tensor) pairs to `mvb_load_weights` in batches of ~PACK_BATCH_BYTES: one host->device staging copy
    per tensor, ONE packing kernel per batch (the per-tensor entry point costs a launch + a sync per tensor)."""
    l = _lib()
    batch, keep, nbytes = [], [], 0

    def flush():
        nonlocal batch, keep, nbytes
        if not batch:
            return
        arr = (MvbNamedTensor * len(batch))(*batch)
        rc = l.mvb_load_weights(handle, arr, len(batch))
        if rc != 0:
            raise _capi.MvbError(f"mvb_load_weights: {l.mvb_handle_error(handle).decode()}")
        batch, keep, nbytes = [], [], 0

    for name, t in named_tensors:
        if t.dtype not in (torch.float16, torch.float32):
            t = t.float()
        t = t.to(device).contiguous()
        e = MvbNamedTensor()
        e.name, e.device_ptr, e.is_f32, e.ndim = name.encode(), t.data_ptr(), _is_f32(t), t.dim()
        for i, v in enumerate(t.shape):
            e.shape[i] = v
        batch.append(e)
        keep.append(t)
        nbytes += t.numel() * t.element_size()
        if nbytes >= PACK_BATCH_BYTES:
            torch.cuda.current_stream(device).synchronize()
            flush()
    torch.cuda.current_stream(device).synchronize()
    flush()


def _lib():
    global _declared
    l = _capi.lib()
    if not _declared:
        l.mvb_create.argtypes = [C.POINTER(MvbConfig), C.c_int, C.POINTER(C.c_void_p)]
        l.mvb_create.restype = C.c_int
        l.mvb_destroy.argtypes = [C.c_void_p]
        l.mvb_destroy.restype = None
        l.mvb_load_weight.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int, C.POINTER(C.c_longlong), C.c_int]
        l.mvb_load_weight.restype = C.c_int
        l.mvb_load_weights.argtypes = [C.c_void_p, C.POINTER(MvbNamedTensor), C.c_int]
        l.mvb_load_weights.restype = C.c_int
        l.mvb_finalize.argtypes = [C.c_void_p]
        l.mvb_finalize.restype = C.c_int
        l.mvb_num_params.argtypes = [C.c_void_p]
        l.mvb_num_params.restype = C.c_int
        l.mvb_workspace_bytes.argtypes = [C.c_void_p, C.POINTER(MvbUnetArgs)]
        l.mvb_workspace_bytes.restype = C.c_longlong
        l.mvb_unet_forward.argtypes = [C.c_void_p, C.POINTER(MvbUnetArgs), C.c_void_p, C.c_longlong, C.c_void_p]
        l.mvb_unet_forward.restype = C.c_int
        l.mvb_handle_error.argtypes = [C.c_void_p]
        l.mvb_handle_error.restype = C.c_char_p
        l.mvb_debug_num_taps.argtypes = [C.c_void_p]
        l.mvb_debug_num_taps.restype = C.c_int
        l.mvb_debug_tap.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_int, C.POINTER(C.c_void_p),
                                    C.POINTER(C.c_longlong), C.POINTER(C.c_int)]
        l.mvb_debug_tap.restype = C.c_int
        l.mvb_unet_merge_lora.argtypes = [C.c_void_p, C.POINTER(MvbNamedTensor), C.POINTER(MvbNamedTensor),
                                          C.POINTER(C.c_float), C.c_int, C.c_int]
        l.mvb_unet_merge_lora.restype = C.c_int
        l.mvb_debug_read_weight.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p]
        l.mvb_debug_read_weight.restype = C.c_int
        _declared = True
    return l


@dataclass
class UNet3DConditionOutput:
    """musev/models/unet_3d_condition.py:166-176."""
    sample: torch.Tensor

    def __getitem__(self, i):
        return (self.sample,)[i]


def _named(name: str, t: torch.Tensor) -> MvbNamedTensor:
    e = MvbNamedTensor()
    e.name, e.device_ptr, e.is_f32, e.ndim = name.encode(), t.data_ptr(), _is_f32(t), t.dim()
    for i, v in enumerate(t.shape):
        e.shape[i] = v
    return e


def _is_f32(t: torch.Tensor) -> int:
    if t.dtype == torch.float32:
        return 1
    if t.dtype == torch.float16:
        return 0
    raise ValueError(f"musev_b200 takes float16 or float32 tensors, got {t.dtype}")


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


class UNet3DConditionModel:
    """CUDA engine behind the call surface of the reference model (musev/models/unet_3d_condition.py:179).

    Kept: `forward` signature and return type (:773-803, :1277-1280), `.config`, `.dtype`, `.device`,
    `.ip_adapter_cross_attn`, `.set_skip_temporal_layers` (:1639), `.to()`, `.eval()`, reference state-dict names.
    """

    def __init__(self, config: UNetConfig, device: Union[str, torch.device] = "cuda", dtype: torch.dtype = torch.float16):
        if not torch.cuda.is_available():
            raise RuntimeError("musev_b200 needs a CUDA (sm_90a) device; there is no CPU path")
        self.cfg = config
        self.device = torch.device(device if str(device) != "cuda" else f"cuda:{torch.cuda.current_device()}")
        self.dtype = dtype
        self.config = SimpleNamespace(**config.to_dict())
        self.ip_adapter_cross_attn = config.ip_adapter_cross_attn
        self.need_refer_emb = config.need_refer_emb
        self.skip_temporal_layers = False
        self.skip_refer_downblock_emb = False
        self._ws: Optional[torch.Tensor] = None
        self._h = C.c_void_p()
        self._loaded = False
        c = MvbConfig()
        c.in_channels, c.out_channels = config.in_channels, config.out_channels
        c.num_blocks = len(config.block_out_channels)
        for i, v in enumerate(config.block_out_channels):
            c.block_out_channels[i] = v
        c.layers_per_block, c.heads = config.layers_per_block, config.attention_head_dim
        c.cross_attention_dim, c.norm_num_groups, c.norm_eps = config.cross_attention_dim, config.norm_num_groups, config.norm_eps
        c.need_transformer_in = int(config.need_transformer_in)
        c.use_anivv1_cfg = int(config.use_anivv1_cfg)
        c.resnet_2d_skip_time_act = int(config.resnet_2d_skip_time_act)
        c.keep_vision_condtion = int(config.keep_vision_condtion)
        c.need_refer_emb = int(config.need_refer_emb)
        c.ip_adapter_cross_attn = int(config.ip_adapter_cross_attn)
        c.need_t2i_ip_adapter = int(config.need_t2i_ip_adapter)
        rc = _lib().mvb_create(C.byref(c), self.device.index or 0, C.byref(self._h))
        if rc != 0:
            raise _capi.MvbError(f"mvb_create failed ({rc}): unsupported configuration or out of device memory")

    # ------------------------------------------------------------------ construction helpers
    @classmethod
    def from_state_dict(cls, state_dict: Dict[str, torch.Tensor], preset: str = "musev", device="cuda",
                        dtype=torch.float16, **config_overrides) -> "UNet3DConditionModel":
        m = cls(preset_config(preset, **config_overrides), device=device, dtype=dtype)
        m.load_state_dict(state_dict)
        return m

    def load_state_dict(self, state_dict: Dict[str, torch.Tensor], strict: bool = True):
        """Reference: from_pretrained_2d / load_state_dict (unet_3d_condition.py:1284-1637). Tensors are packed into
        the kernel layouts on the device in batches (peak extra memory = one ~512 MB staging batch)."""
        expected = unet_param_shapes(self.cfg)
        missing = [k for k in expected if k not in state_dict]
        unexpected = [k for k in state_dict if k not in expected]
        if strict and (missing or unexpected):
            raise RuntimeError(f"Error(s) in loading state_dict: missing {missing[:5]} unexpected {unexpected[:5]}")
        l = _lib()
        todo = []
        for name, shape in expected.items():
            if name not in state_dict:
                continue
            t = state_dict[name]
            if tuple(t.shape) != tuple(shape):
                raise RuntimeError(f"size mismatch for {name}: {tuple(t.shape)} vs {tuple(shape)}")
            todo.append((name, t))
        load_weights_batched(self._h, todo, self.device)
        rc = l.mvb_finalize(self._h)
        if rc != 0:
            raise _capi.MvbError(f"mvb_finalize: {l.mvb_handle_error(self._h).decode()}")
        self._loaded = True
        return SimpleNamespace(missing_keys=missing, unexpected_keys=unexpected)

    def __del__(self):
        try:
            if getattr(self, "_h", None) and self._h.value:
                _lib().mvb_destroy(self._h)
                self._h = C.c_void_p()
        except Exception:
            pass

    # ------------------------------------------------------------------ nn.Module-like surface
    def eval(self):
        return self

    def to(self, *args, **kwargs):
        for a in list(args) + list(kwargs.values()):
            if isinstance(a, torch.dtype):
                if a not in (torch.float16, torch.float32):
                    raise ValueError("musev_b200 computes in fp16 with fp32 accumulation; I/O dtype is fp16 or fp32")
                self.dtype = a
            elif isinstance(a, (str, torch.device)) and torch.device(a).type != "cuda":
                raise RuntimeError("musev_b200 has no CPU path")
        return self

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
    ):
        """Reference: UNet3DConditionModel.forward, musev/models/unet_3d_condition.py:773-1280."""
        if not self._loaded:
            raise RuntimeError("weights not loaded: call load_state_dict first")
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
        out = torch.empty((B, self.cfg.out_channels, T, H, W), dtype=sample.dtype, device=dev)
        a.out, a.out_is_f32 = out.data_ptr(), _is_f32(out)
        l = _lib()
        need = l.mvb_workspace_bytes(self._h, C.byref(a))
        if need < 0:
            raise _capi.MvbError(f"mvb_workspace_bytes: {l.mvb_handle_error(self._h).decode()}")
        if self._ws is None or self._ws.numel() < need:
            self._ws = None
            self._ws = torch.empty(int(need), dtype=torch.uint8, device=dev)
        rc = l.mvb_unet_forward(self._h, C.byref(a), self._ws.data_ptr(), self._ws.numel(),
                                torch.cuda.current_stream(dev).cuda_stream)
        if rc != 0:
            raise _capi.MvbError(f"mvb_unet_forward ({rc}): {l.mvb_handle_error(self._h).decode()}")
        self._keep = keep  # inputs must outlive the asynchronous launch sequence
        if skip_temporal_layers is not None:
            self.set_skip_temporal_layers(not skip_temporal_layers)   # unet_3d_condition.py:1275-1276
        if not return_dict:
            return (out,)
        return UNet3DConditionOutput(sample=out)

    __call__ = forward

    # ------------------------------------------------------------------ LoRA (musev_b200/lora.py is the public surface)
    def _merge_lora(self, targets: Sequence[str], ups: Sequence[torch.Tensor], downs: Sequence[torch.Tensor],
                    scales: Sequence[float], subtract: bool = False) -> None:
        """W16 = fp16(W16 +- fp16(scale * (up @ down))) for every target (reference weight names), one `mvb_unet_merge_lora`
        call. The factors must be contiguous fp16 / fp32 tensors on this model's device."""
        n = len(targets)
        if not (len(ups) == len(downs) == len(scales) == n):
            raise ValueError("targets, ups, downs and scales differ in length")
        for t in list(ups) + list(downs):
            if t.device != self.device or not t.is_contiguous():
                raise ValueError(f"LoRA factors must be contiguous tensors on {self.device}")
        up_arr = (MvbNamedTensor * max(n, 1))(*[_named(nm, u) for nm, u in zip(targets, ups)])
        down_arr = (MvbNamedTensor * max(n, 1))(*[_named(nm, d) for nm, d in zip(targets, downs)])
        sc = (C.c_float * max(n, 1))(*[float(s) for s in scales])
        torch.cuda.current_stream(self.device).synchronize()      # the factors may still be in flight
        l = _lib()
        rc = l.mvb_unet_merge_lora(self._h, up_arr, down_arr, sc, n, int(bool(subtract)))
        if rc != 0:
            raise _capi.MvbError(f"mvb_unet_merge_lora ({rc}): {l.mvb_handle_error(self._h).decode()}")

    def debug_weight(self, name: str) -> torch.Tensor:
        """The packed matrix / convolution weight `name` read back into its reference shape, fp16 on the device."""
        shape = unet_param_shapes(self.cfg).get(name)
        if shape is None or len(shape) < 2:
            raise ValueError(f"{name} is not a matrix or convolution weight of this UNet")
        out = torch.empty(shape, dtype=torch.float16, device=self.device)
        l = _lib()
        rc = l.mvb_debug_read_weight(self._h, name.encode(), out.data_ptr())
        if rc != 0:
            raise _capi.MvbError(f"mvb_debug_read_weight ({rc}): {l.mvb_handle_error(self._h).decode()}")
        return out

    # ------------------------------------------------------------------ debug
    def debug_taps(self) -> Dict[str, torch.Tensor]:
        """Layer outputs of the last forward as [(b t), C, h*w]-ordered channels-last copies (fp32, [rows, C])."""
        l = _lib()
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
