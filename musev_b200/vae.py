"""Host mirror of the VAE decode that follows the denoise loop (SURVEY.md section 8(f)-3).

Reference: `MusevControlNetPipeline.decode_latents` (musev/pipelines/pipeline_controlnet.py:233-238; called per T-segment at
:2157-2171) -> `decode_latents` of the diffusers img2img pipeline (pipeline_stable_diffusion_img2img.py:486-495) ->
`AutoencoderKL.decode` (models/autoencoder_kl.py:275-302). post_quant_conv, the decoder's convolutions / GroupNorms /
single-head mid-block attention and the `image / 2 + 0.5, clamp(0, 1)` post-processing run inside libmusevb200.so
(`mvb_vae_decode`, musev_b200/csrc/engine.cu `Engine::run_vae`). Frames are decoded in chunks (the reference enables VAE
slicing = one frame at a time, pipeline_controlnet_predictor.py:284) to bound the activation arena. No CPU fallback.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import asdict, dataclass
from types import SimpleNamespace
from typing import Dict, Optional, Union

import torch

from . import _capi
from .schema import VAEConfig, vae_decoder_param_shapes
from .unet import MvbConfig, _is_f32, _lib as _unet_lib, load_weights_batched


class MvbVaeDecodeArgs(C.Structure):
    _fields_ = [("latents", C.c_void_p), ("latents_is_f32", C.c_int), ("N", C.c_int), ("h", C.c_int), ("w", C.c_int),
                ("latent_scale", C.c_float), ("out", C.c_void_p), ("out_is_f32", C.c_int), ("postprocess", C.c_int)]


_declared = False


def _lib():
    global _declared
    l = _unet_lib()
    if not _declared:
        l.mvb_create_vae_decoder.argtypes = [C.POINTER(MvbConfig), C.c_int, C.POINTER(C.c_void_p)]
        l.mvb_create_vae_decoder.restype = C.c_int
        l.mvb_vae_decode_workspace_bytes.argtypes = [C.c_void_p, C.POINTER(MvbVaeDecodeArgs)]
        l.mvb_vae_decode_workspace_bytes.restype = C.c_longlong
        l.mvb_vae_decode.argtypes = [C.c_void_p, C.POINTER(MvbVaeDecodeArgs), C.c_void_p, C.c_longlong, C.c_void_p]
        l.mvb_vae_decode.restype = C.c_int
        _declared = True
    return l


@dataclass
class DecoderOutput:
    """diffusers models/vae.py:29-38."""
    sample: torch.Tensor

    def __getitem__(self, i):
        return (self.sample,)[i]


class AutoencoderKLDecoder:
    """Decode half of `AutoencoderKL` on the CUDA engine: `.decode(z)` (autoencoder_kl.py:275-302) and the pipeline-level
    `.decode_latents(latents)`; `.config.scaling_factor`, `.dtype`, `.device`, reference state-dict names (`decoder.*`,
    `post_quant_conv.*`; encoder / quant_conv entries of a full VAE state dict are ignored)."""

    def __init__(self, config: VAEConfig = VAEConfig(), device: Union[str, torch.device] = "cuda", dtype: torch.dtype = torch.float16,
                 frames_per_call: int = 4):
        if not torch.cuda.is_available():
            raise RuntimeError("musev_b200 needs a CUDA (sm_90a) device; there is no CPU path")
        self.cfg = config
        self.device = torch.device(device if str(device) != "cuda" else f"cuda:{torch.cuda.current_device()}")
        self.dtype = dtype
        self.config = SimpleNamespace(**asdict(config))
        self.frames_per_call = int(frames_per_call)
        self._ws: Optional[torch.Tensor] = None
        self._h = C.c_void_p()
        self._loaded = False
        c = MvbConfig()
        c.in_channels, c.out_channels = config.latent_channels, config.out_channels
        c.num_blocks = len(config.block_out_channels)
        for i, v in enumerate(config.block_out_channels):
            c.block_out_channels[i] = v
        c.layers_per_block, c.heads = config.layers_per_block, 1
        c.cross_attention_dim, c.norm_num_groups, c.norm_eps = 64, config.norm_num_groups, 1e-6
        rc = _lib().mvb_create_vae_decoder(C.byref(c), self.device.index or 0, C.byref(self._h))
        if rc != 0:
            raise _capi.MvbError(f"mvb_create_vae_decoder failed ({rc}): unsupported configuration or out of device memory")

    def load_state_dict(self, state_dict: Dict[str, torch.Tensor], strict: bool = True):
        expected = vae_decoder_param_shapes(self.cfg)
        missing = [k for k in expected if k not in state_dict]
        unexpected = [k for k in state_dict if k not in expected and not k.startswith(("encoder.", "quant_conv."))]
        if strict and (missing or unexpected):
            raise RuntimeError(f"Error(s) in loading state_dict: missing {missing[:5]} unexpected {unexpected[:5]}")
        todo = []
        for name, shape in expected.items():
            if name not in state_dict:
                continue
            t = state_dict[name]
            if tuple(t.shape) != tuple(shape):
                raise RuntimeError(f"size mismatch for {name}: {tuple(t.shape)} vs {tuple(shape)}")
            todo.append((name, t))
        load_weights_batched(self._h, todo, self.device)
        l = _lib()
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

    def eval(self):
        return self

    def _run(self, z: torch.Tensor, latent_scale: float, postprocess: bool, out_dtype: torch.dtype) -> torch.Tensor:
        if not self._loaded:
            raise RuntimeError("weights not loaded: call load_state_dict first")
        if z.dim() != 4 or z.shape[1] != self.cfg.latent_channels:
            raise ValueError(f"latents must be [N, {self.cfg.latent_channels}, h, w], got {tuple(z.shape)}")
        dev = self.device
        z = z.to(dev)
        if z.dtype not in (torch.float16, torch.float32):
            z = z.float()
        z = z.contiguous()
        N, _, h, w = z.shape
        up = 2 ** (len(self.cfg.block_out_channels) - 1)
        out = torch.empty((N, self.cfg.out_channels, h * up, w * up), dtype=out_dtype, device=dev)
        l = _lib()
        step = max(1, self.frames_per_call)
        for n0 in range(0, N, step):
            n1 = min(N, n0 + step)
            a = MvbVaeDecodeArgs()
            zc, oc = z[n0:n1], out[n0:n1]
            a.latents, a.latents_is_f32 = zc.data_ptr(), _is_f32(zc)
            a.N, a.h, a.w = n1 - n0, h, w
            a.latent_scale = float(latent_scale)
            a.out, a.out_is_f32 = oc.data_ptr(), _is_f32(oc)
            a.postprocess = int(postprocess)
            need = l.mvb_vae_decode_workspace_bytes(self._h, C.byref(a))
            if need < 0:
                raise _capi.MvbError(f"mvb_vae_decode_workspace_bytes: {l.mvb_handle_error(self._h).decode()}")
            if self._ws is None or self._ws.numel() < need:
                self._ws = None
                self._ws = torch.empty(int(need), dtype=torch.uint8, device=dev)
            rc = l.mvb_vae_decode(self._h, C.byref(a), self._ws.data_ptr(), self._ws.numel(), torch.cuda.current_stream(dev).cuda_stream)
            if rc != 0:
                raise _capi.MvbError(f"mvb_vae_decode: {l.mvb_handle_error(self._h).decode()}")
        self._keep = z
        return out

    @torch.no_grad()
    def decode(self, z: torch.Tensor, return_dict: bool = True):
        """AutoencoderKL.decode (autoencoder_kl.py:275-302): z [N, 4, h, w] -> image [N, 3, 8h, 8w] (no scaling, no clamp)."""
        img = self._run(z, 1.0, False, self.dtype)
        if not return_dict:
            return (img,)
        return DecoderOutput(sample=img)

    @torch.no_grad()
    def decode_latents(self, latents: torch.Tensor) -> torch.Tensor:
        """MusevControlNetPipeline.decode_latents (pipeline_controlnet.py:233-238): latents [b, c, f, h, w] ->
        video [b, c, f, H, W] float32 in [0, 1]. The reference returns a CPU numpy array; this returns the device tensor
        (call `.cpu().numpy()` where the reference's `np.concatenate` of segments needs it)."""
        b, c, f, h, w = latents.shape
        z = latents.permute(0, 2, 1, 3, 4).reshape(b * f, c, h, w)
        img = self._run(z, 1.0 / self.cfg.scaling_factor, True, torch.float32)
        return img.view(b, f, *img.shape[1:]).permute(0, 2, 1, 3, 4).contiguous()
