"""Host mirror of diffusers `ControlNetModel` as MuseV runs it per window-step (SURVEY.md section 8(f), rank 1).

Reference: diffusers/src/diffusers/models/controlnet.py:645-852, called from
musev/pipelines/pipeline_controlnet.py:1238-1262. The SD-1.5 encoder half, the 12 + 1 zero convolutions and the output
scaling run inside libmusevb200.so (`mvb_controlnet_forward`, musev_b200/csrc/engine_encoder.cu). The conditioning embedding
(controlnet.py:101-112) is a one-shot conv stack on the 8x larger condition image; the pipeline computes it once per
call and passes `controlnet_cond_latents` on every step (pipeline_controlnet.py:1258), so it stays a handful of torch
convolutions here, outside the per-step path.

`MultiControlNetModel` (diffusers pipelines/controlnet/multicontrolnet.py:15-72) runs several ControlNets on one input and
sums their maps: the second and later nets add into the first net's output tensors inside the engine
(`mvb_controlnet_args.accumulate`).

`PoseGuider` (musev/models/controlnet.py:326-399) is the pose-guided video2video encoder: eight 3x3 convolutions run once per
pipeline call on the pose images (`mvb_pose_guider_forward`, `Engine::run_pose_guider`); its output is the UNet's
`pose_guider_emb`.
"""
from __future__ import annotations

from dataclasses import asdict
from types import SimpleNamespace
from typing import Any, Dict, List, Optional, Sequence, Tuple, Union

import torch
import torch.nn.functional as F

from ._capi import EngineModel, MvbControlnetArgs, _is_f32, make_config
# Names callers imported from this module before the binding moved to _capi; they are the binding's own objects.
from ._capi import lib as _lib  # noqa: F401
from .schema import ControlNetConfig, PoseGuiderConfig, controlnet_param_shapes, pose_guider_param_shapes


class ControlNetOutput(SimpleNamespace):
    """diffusers models/controlnet.py:46-61."""


class ControlNetModel(EngineModel):
    """CUDA engine behind the call surface of diffusers `ControlNetModel` (models/controlnet.py:114)."""

    _create, _workspace, _forward = "mvb_create_controlnet", "mvb_controlnet_workspace_bytes", "mvb_controlnet_forward"
    _COND = "controlnet_cond_embedding."

    def __init__(self, config: ControlNetConfig, device: Union[str, torch.device] = "cuda", dtype: torch.dtype = torch.float16):
        self.cfg = config
        self.config = SimpleNamespace(**asdict(config), global_pool_conditions=False)
        self._cond_w: Dict[str, torch.Tensor] = {}
        c = make_config(config.in_channels, config.in_channels, config.block_out_channels, config.layers_per_block,
                        config.attention_head_dim, config.cross_attention_dim, config.norm_num_groups, config.norm_eps)
        super().__init__(c, device, dtype)
        # residual map geometry: (channels, downscale) of the 12 + 1 outputs (controlnet.py:788-823)
        self._maps: List[Tuple[int, int]] = [(config.block_out_channels[0], 1)]
        ds = 1
        nb = len(config.block_out_channels)
        for i, ch in enumerate(config.block_out_channels):
            for _ in range(config.layers_per_block):
                self._maps.append((ch, ds))
            if i != nb - 1:
                ds *= 2
                self._maps.append((ch, ds))
        self._maps.append((config.block_out_channels[-1], ds))

    @classmethod
    def from_state_dict(cls, state_dict: Dict[str, torch.Tensor], device="cuda", dtype=torch.float16,
                        **config_overrides) -> "ControlNetModel":
        m = cls(ControlNetConfig(**config_overrides), device=device, dtype=dtype)
        m.load_state_dict(state_dict)
        return m

    def _param_shapes(self):
        return controlnet_param_shapes(self.cfg)

    def _load(self, todo):
        # the conditioning embedding stays a torch conv stack (module docstring); the engine takes the rest
        self._cond_w.update({n: t.to(self.device, self.dtype).contiguous() for n, t in todo if n.startswith(self._COND)})
        super()._load([(n, t) for n, t in todo if not n.startswith(self._COND)])

    # ------------------------------------------------------------------ one-shot conditioning embedding
    @torch.no_grad()
    def controlnet_cond_embedding(self, conditioning: torch.Tensor) -> torch.Tensor:
        """ControlNetConditioningEmbedding.forward (models/controlnet.py:101-112); once per pipeline call."""
        p = "controlnet_cond_embedding"
        w = self._cond_w
        x = conditioning.to(self.device, self.dtype)
        e = F.silu(F.conv2d(x, w[p + ".conv_in.weight"], w[p + ".conv_in.bias"], padding=1))
        n_blocks = 2 * (len(self.cfg.conditioning_embedding_out_channels) - 1)
        for i in range(n_blocks):
            e = F.silu(F.conv2d(e, w[f"{p}.blocks.{i}.weight"], w[f"{p}.blocks.{i}.bias"], padding=1, stride=2 if i % 2 else 1))
        return F.conv2d(e, w[p + ".conv_out.weight"], w[p + ".conv_out.bias"], padding=1)

    # ------------------------------------------------------------------ forward
    @torch.no_grad()
    def forward(
        self,
        sample: torch.Tensor,
        timestep: Union[torch.Tensor, float, int],
        encoder_hidden_states: torch.Tensor,
        controlnet_cond: Optional[torch.Tensor] = None,
        conditioning_scale: float = 1.0,
        class_labels: Optional[torch.Tensor] = None,
        timestep_cond: Optional[torch.Tensor] = None,
        attention_mask: Optional[torch.Tensor] = None,
        added_cond_kwargs: Optional[Dict[str, torch.Tensor]] = None,
        cross_attention_kwargs: Optional[Dict[str, Any]] = None,
        guess_mode: bool = False,
        return_dict: bool = True,
        controlnet_cond_latents: Optional[torch.Tensor] = None,
        accumulate_into: Optional[Tuple[List[torch.Tensor], torch.Tensor]] = None,
    ):
        """Reference: ControlNetModel.forward, diffusers models/controlnet.py:645-852.

        accumulate_into: the `(down, mid)` an earlier call returned. This call's scaled maps are then added into those
        tensors on the device (fp32 sum, one rounding to their dtype) and they are returned: the Multi-ControlNet sum
        `samples_prev + samples_curr` of diffusers multicontrolnet.py:64-70, without a second set of maps."""
        self._check_loaded()
        for name, v in (("class_labels", class_labels), ("timestep_cond", timestep_cond), ("attention_mask", attention_mask),
                        ("added_cond_kwargs", added_cond_kwargs)):
            if v is not None:
                raise NotImplementedError(f"{name} is not used by the SD-1.5 ControlNets MuseV loads")
        if sample.dim() != 4:
            raise ValueError(f"sample must be (b t) c h w, got {tuple(sample.shape)}")
        if controlnet_cond_latents is None:
            if controlnet_cond is None:
                raise ValueError("controlnet_cond or controlnet_cond_latents is required")
            controlnet_cond_latents = self.controlnet_cond_embedding(controlnet_cond)
        NF, _, H, W = sample.shape
        if encoder_hidden_states.dim() != 3 or encoder_hidden_states.shape[0] != NF:
            raise ValueError("encoder_hidden_states must be [(b t), n_text, dim] (one row block per frame)")
        dev = self.device
        sample = sample.to(dev).contiguous()
        ehs = encoder_hidden_states.to(dev).contiguous()
        cond = controlnet_cond_latents.to(dev).contiguous()
        if tuple(cond.shape) != (NF, self.cfg.block_out_channels[0], H, W):
            raise ValueError(f"controlnet_cond_latents has shape {tuple(cond.shape)}")
        t_val = float(timestep.reshape(-1)[0].item()) if torch.is_tensor(timestep) else float(timestep)
        n_out = len(self._maps)
        scale = float(conditioning_scale)
        if guess_mode:   # :826-830
            scales = (torch.logspace(-1, 0, n_out) * scale).tolist()
        else:            # :831-833
            scales = [scale] * n_out
        if accumulate_into is None:
            outs = [torch.empty((NF, c, H // ds, W // ds), device=dev, dtype=self.dtype) for c, ds in self._maps]
        else:
            outs = list(accumulate_into[0]) + [accumulate_into[1]]
            if len(outs) != n_out:
                raise ValueError(f"accumulate_into holds {len(outs)} maps; this ControlNet has {n_out}")
            for o, (c, ds) in zip(outs, self._maps):
                if (tuple(o.shape) != (NF, c, H // ds, W // ds) or o.device != dev or o.dtype != outs[0].dtype
                        or o.dtype not in (torch.float16, torch.float32) or not o.is_contiguous()):
                    raise ValueError(f"accumulate_into: a map of shape {tuple(o.shape)} ({o.dtype}, {o.device}) is not the "
                                     f"contiguous {(NF, c, H // ds, W // ds)} map on {dev} this call adds into")
        a = MvbControlnetArgs()
        a.sample, a.sample_is_f32 = sample.data_ptr(), _is_f32(sample)
        a.NF, a.H, a.W = NF, H, W
        a.timestep = t_val
        a.encoder_hidden_states, a.ehs_is_f32, a.n_text = ehs.data_ptr(), _is_f32(ehs), ehs.shape[1]
        a.cond_latents, a.cond_is_f32 = cond.data_ptr(), _is_f32(cond)
        a.n_out = n_out
        for k in range(n_out):
            a.scales[k] = scales[k]
            a.outs[k] = outs[k].data_ptr()
        a.out_is_f32 = _is_f32(outs[0])
        a.accumulate = int(accumulate_into is not None)
        self._launch(a)
        down, mid = outs[:-1], outs[-1]
        if not return_dict:
            return (down, mid)
        return ControlNetOutput(down_block_res_samples=down, mid_block_res_sample=mid)

    __call__ = forward


def _geometry(net) -> Tuple:
    """What fixes the shapes of a ControlNet's 12 + 1 residual maps (controlnet.py:181-447)."""
    c = net.config
    return (tuple(c.block_out_channels), c.layers_per_block, c.cross_attention_dim)


class MultiControlNetModel:
    """Several ControlNets whose residual maps are summed, behind the call surface of diffusers `MultiControlNetModel`
    (diffusers/src/diffusers/pipelines/controlnet/multicontrolnet.py:15-72). The first net writes the 12 + 1 output
    tensors; every later net adds its maps into them on the device (`accumulate_into`), in net order, so the sum rounds
    as the reference's `samples_prev + samples_curr` does."""

    def __init__(self, controlnets: Sequence[Any]):
        nets = list(controlnets)
        if not nets:
            raise ValueError("For multiple controlnets: `controlnets` must hold at least one ControlNet")
        for k, n in enumerate(nets[1:], 1):
            if _geometry(n) != _geometry(nets[0]):
                raise ValueError(f"For multiple controlnets: ControlNet {k} has block_out_channels / layers_per_block / "
                                 f"cross_attention_dim {_geometry(n)}, ControlNet 0 has {_geometry(nets[0])}; their "
                                 "residuals cannot be summed")
            if torch.device(n.device) != torch.device(nets[0].device) or n.dtype != nets[0].dtype:
                raise ValueError(f"For multiple controlnets: ControlNet {k} is on {n.device} in {n.dtype}, ControlNet 0 on "
                                 f"{nets[0].device} in {nets[0].dtype}; every net must share one device and dtype")
        self.nets = nets

    @property
    def dtype(self) -> torch.dtype:
        return self.nets[0].dtype

    @property
    def device(self) -> torch.device:
        return self.nets[0].device

    def check_list(self, name: str, values) -> list:
        """diffusers check_inputs (pipelines/controlnet/pipeline_controlnet.py:570-615): one entry per ControlNet."""
        if not isinstance(values, (list, tuple)):
            raise ValueError(f"For multiple controlnets: `{name}` must be type `list`")
        if len(values) != len(self.nets):
            raise ValueError(f"For multiple controlnets: `{name}` must have the same length as the number of controlnets, "
                             f"but got {len(values)} entries and {len(self.nets)} ControlNets.")
        return list(values)

    @torch.no_grad()
    def forward(
        self,
        sample: torch.Tensor,
        timestep: Union[torch.Tensor, float, int],
        encoder_hidden_states: torch.Tensor,
        controlnet_cond: Optional[List[torch.Tensor]],
        conditioning_scale: List[float],
        class_labels: Optional[torch.Tensor] = None,
        timestep_cond: Optional[torch.Tensor] = None,
        attention_mask: Optional[torch.Tensor] = None,
        added_cond_kwargs: Optional[Dict[str, torch.Tensor]] = None,
        cross_attention_kwargs: Optional[Dict[str, Any]] = None,
        guess_mode: bool = False,
        return_dict: bool = True,
        controlnet_cond_latents: Optional[List[torch.Tensor]] = None,
    ):
        """multicontrolnet.py:31-72. Returns `(down, mid)` whatever `return_dict` says, as the reference does. Without a
        `controlnet_cond_latents` list each net embeds its own image (`controlnet_cond_embedding`); `controlnet_cond` may
        be None when the list is given."""
        n = len(self.nets)
        scales = self.check_list("controlnet_conditioning_scale", conditioning_scale)
        lats = self.check_list("controlnet_cond_latents", controlnet_cond_latents) \
            if isinstance(controlnet_cond_latents, (list, tuple)) else [None] * n
        images = self.check_list("image", controlnet_cond) if controlnet_cond is not None else [None] * n
        res = None
        for net, image, scale, lat in zip(self.nets, images, scales, lats):
            res = net(sample, timestep, encoder_hidden_states, controlnet_cond=image, conditioning_scale=scale,
                      class_labels=class_labels, timestep_cond=timestep_cond, attention_mask=attention_mask,
                      added_cond_kwargs=added_cond_kwargs, cross_attention_kwargs=cross_attention_kwargs,
                      guess_mode=guess_mode, return_dict=False, controlnet_cond_latents=lat, accumulate_into=res)
        return res

    __call__ = forward


def check_pose_guider_state_dict(cfg: PoseGuiderConfig, state_dict: Dict[str, torch.Tensor], strict: bool = True):
    """(name, tensor) pairs to load and the unexpected keys of a PoseGuider state dict. A missing key raises KeyError naming
    it, whatever `strict` says; a wrong shape raises RuntimeError; unexpected keys raise only when `strict`."""
    expected = pose_guider_param_shapes(cfg)
    missing = [k for k in expected if k not in state_dict]
    if missing:
        more = f" (and {len(missing) - 1} more)" if len(missing) > 1 else ""
        raise KeyError(f"PoseGuider state dict is missing {missing[0]!r}{more}; the engine has no initialiser for it")
    unexpected = [k for k in state_dict if k not in expected]
    if strict and unexpected:
        raise RuntimeError(f"Error(s) in loading state_dict: unexpected {unexpected[:5]}")
    todo = []
    for name, shape in expected.items():
        t = state_dict[name]
        if tuple(t.shape) != tuple(shape):
            raise RuntimeError(f"size mismatch for {name}: {tuple(t.shape)} vs {tuple(shape)}")
        todo.append((name, t))
    return todo, unexpected


class PoseGuider(EngineModel):
    """CUDA engine behind the call surface of `musev.models.controlnet.PoseGuider` (musev/models/controlnet.py:326-399).

    Kept: the constructor arguments, `from_pretrained(path, conditioning_embedding_channels, conditioning_channels,
    block_out_channels)`, `forward(conditioning [b, c, t, H, W]) -> [b, emb, t, H/8, W/8]`, `.to()`, `.eval()` and the
    reference state-dict names. Frames run in chunks of `frames_per_call` (bounds the activation workspace, like the VAE).
    Departure: the reference loads with `strict=False` and keeps its initialiser's values for a missing key; the engine
    has no initialiser, so a missing key raises, naming it. Unexpected keys are ignored when `strict=False`."""

    _create, _workspace, _forward = "mvb_create_pose_guider", "mvb_pose_guider_workspace_bytes", "mvb_pose_guider_forward"

    def __init__(self, conditioning_embedding_channels: int, conditioning_channels: int = 3,
                 block_out_channels: Tuple[int, ...] = (16, 32, 64, 128), device: Union[str, torch.device] = "cuda",
                 dtype: torch.dtype = torch.float16, frames_per_call: int = 8):
        self.cfg = PoseGuiderConfig(int(conditioning_embedding_channels), int(conditioning_channels), tuple(block_out_channels))
        self.config = SimpleNamespace(**asdict(self.cfg))
        self.frames_per_call = int(frames_per_call)
        if not 1 <= len(self.cfg.block_out_channels) <= 4:
            raise ValueError(f"block_out_channels must have 1..4 entries, got {self.cfg.block_out_channels}")
        c = make_config(self.cfg.conditioning_channels, self.cfg.conditioning_embedding_channels, self.cfg.block_out_channels)
        super().__init__(c, device, dtype, unsupported=f"unsupported channel counts {self.cfg}")

    @classmethod
    def from_pretrained(cls, pretrained_model_path, conditioning_embedding_channels: int, conditioning_channels: int = 3,
                        block_out_channels: Tuple[int, ...] = (16, 32, 64, 128), device="cuda", dtype=torch.float16):
        """controlnet.py:373-399: a `torch.load`-able state dict file; loaded with `strict=False` (see the class notes)."""
        state_dict = torch.load(pretrained_model_path, map_location="cpu")
        m = cls(conditioning_embedding_channels, conditioning_channels, block_out_channels, device=device, dtype=dtype)
        m.load_state_dict(state_dict, strict=False)
        return m

    def _param_shapes(self):
        return pose_guider_param_shapes(self.cfg)

    def load_state_dict(self, state_dict: Dict[str, torch.Tensor], strict: bool = True):
        todo, unexpected = check_pose_guider_state_dict(self.cfg, state_dict, strict)
        self._load(todo)
        return SimpleNamespace(missing_keys=[], unexpected_keys=unexpected)

    @torch.no_grad()
    def embed_frames(self, images: torch.Tensor, out_dtype: Optional[torch.dtype] = None,
                     process_group=None) -> torch.Tensor:
        """images [N, c, H, W] (fp16 / fp32, frames on the batch axis) -> [N, emb, H / 2^(nb-1), W / 2^(nb-1)].

        process_group: a `torch.distributed` group (or `group.WORLD`) shares the frames out over its ranks, in the chunks
        of `frames_per_call` frames one GPU would launch, and exchanges the rows on the device
        (`_capi.launch_frame_chunks`). Every rank must make the same call, with the same images, and every rank
        receives the full embedding, bit-identical to the single-GPU one. None (the default) embeds every frame here."""
        self._check_loaded()
        f = 2 ** (len(self.cfg.block_out_channels) - 1)
        if images.dim() != 4 or images.shape[1] != self.cfg.conditioning_channels:
            raise ValueError(f"conditioning must have {self.cfg.conditioning_channels} channels, got {tuple(images.shape)}")
        N, _, H, W = images.shape
        if N < 1 or H < f or W < f or H % f or W % f:
            raise ValueError(f"image size {H}x{W} must be a positive multiple of {f} (the pose guider downsamples {f}x)")
        x = images.to(self.device)
        if x.dtype not in (torch.float16, torch.float32):
            x = x.float()
        x = x.contiguous()
        h, w = H // f, W // f
        out = torch.empty((N, self.cfg.conditioning_embedding_channels, h, w), dtype=out_dtype or self.dtype, device=self.device)
        return self._launch_frames(x, out, h, w, 1.0, 0, process_group)

    @torch.no_grad()
    def forward(self, conditioning: torch.Tensor, process_group=None) -> torch.Tensor:
        """PoseGuider.forward (controlnet.py:361-371): conditioning [b, c, t, H, W] -> [b, emb, t, H/8, W/8] (four blocks).
        process_group: as in `embed_frames`."""
        if conditioning.dim() != 5:
            raise ValueError(f"conditioning must be [b, c, t, H, W], got {tuple(conditioning.shape)}")
        b, c, t, H, W = conditioning.shape
        x = conditioning.permute(0, 2, 1, 3, 4).reshape(b * t, c, H, W)                    # InflatedConv3d, :308-316
        e = self.embed_frames(x, process_group=process_group)
        return e.view(b, t, *e.shape[1:]).permute(0, 2, 1, 3, 4).contiguous()

    __call__ = forward
