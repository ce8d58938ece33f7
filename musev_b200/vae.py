"""Host mirror of the VAE: the decode that follows the denoise loop (SURVEY.md section 8(f)-3) and the encode before it.

Reference: `MusevControlNetPipeline.decode_latents` (musev/pipelines/pipeline_controlnet.py:233-238; called per T-segment at
:2157-2171) -> `decode_latents` of the diffusers img2img pipeline (pipeline_stable_diffusion_img2img.py:486-495) ->
`AutoencoderKL.decode` (models/autoencoder_kl.py:275-302). post_quant_conv, the decoder's convolutions / GroupNorms /
single-head mid-block attention and the `image / 2 + 0.5, clamp(0, 1)` post-processing run inside libmusevb200.so
(`mvb_vae_decode`, musev_b200/csrc/engine.cu `Engine::run_vae`). Frames are decoded in chunks (the reference enables VAE
slicing = one frame at a time, pipeline_controlnet_predictor.py:284) to bound the activation arena. No CPU fallback.

Encode: `AutoencoderKL.encode` (models/autoencoder_kl.py:256-297) = `Encoder.forward` (models/vae.py:133-175) + quant_conv run
inside the library (`mvb_vae_encode`, `Engine::run_vae_encode`); `DiagonalGaussianDistribution` (vae.py:741-785) is a few
torch ops on the small moments tensor here. The pipeline reads `vae.config.scaling_factor * vae.encode(x).latent_dist.mean`
at three call sites (musev/pipelines/pipeline_controlnet.py:348-368, 809-811, 978-981); `encode_video` computes exactly that
for a whole video in the library. `AutoencoderKL` holds both halves and stands in for `pipeline.vae`.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import asdict, dataclass
from types import SimpleNamespace
from typing import Dict, Optional, Union

import torch

from . import _capi
from .schema import VAEConfig, vae_decoder_param_shapes, vae_encoder_param_shapes
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
        l.mvb_create_vae_encoder.argtypes = [C.POINTER(MvbConfig), C.c_int, C.POINTER(C.c_void_p)]
        l.mvb_create_vae_encoder.restype = C.c_int
        l.mvb_vae_encode_workspace_bytes.argtypes = [C.c_void_p, C.POINTER(MvbVaeDecodeArgs)]
        l.mvb_vae_encode_workspace_bytes.restype = C.c_longlong
        l.mvb_vae_encode.argtypes = [C.c_void_p, C.POINTER(MvbVaeDecodeArgs), C.c_void_p, C.c_longlong, C.c_void_p]
        l.mvb_vae_encode.restype = C.c_int
        _declared = True
    return l


@dataclass
class DecoderOutput:
    """diffusers models/vae.py:29-38."""
    sample: torch.Tensor

    def __getitem__(self, i):
        return (self.sample,)[i]


class DiagonalGaussianDistribution:
    """Host mirror of diffusers models/vae.py:741-785 on the moments [N, 2 zc, h, w] the engine returns: mean, logvar
    clamped to [-30, 20], std, var, `sample(generator)`, `mode()`."""

    def __init__(self, parameters: torch.Tensor, deterministic: bool = False):
        self.parameters = parameters
        self.mean, self.logvar = torch.chunk(parameters, 2, dim=1)
        self.logvar = torch.clamp(self.logvar, -30.0, 20.0)
        self.deterministic = deterministic
        self.std = torch.exp(0.5 * self.logvar)
        self.var = torch.exp(self.logvar)
        if self.deterministic:
            self.var = self.std = torch.zeros_like(self.mean)

    def sample(self, generator: Optional[torch.Generator] = None) -> torch.Tensor:
        # diffusers randn_tensor: drawn on the generator's device, then moved to the parameters' device
        gen_dev = generator.device if generator is not None else self.parameters.device
        eps = torch.randn(self.mean.shape, generator=generator, device=gen_dev, dtype=self.parameters.dtype)
        return self.mean + self.std * eps.to(self.parameters.device)

    def mode(self) -> torch.Tensor:
        return self.mean


@dataclass
class AutoencoderKLOutput:
    """diffusers models/autoencoder_kl.py:29-38."""
    latent_dist: DiagonalGaussianDistribution

    def __getitem__(self, i):
        return (self.latent_dist,)[i]


class _EngineHalf:
    """One engine handle of a VAE half: creation from a `VAEConfig`, weight loading by reference names, chunked calls."""

    _kind = ""                      # "decoder" / "encoder": selects the C entry points
    _own: tuple = ()                # state-dict prefixes of this half
    _other: tuple = ()              # prefixes of the other half (ignored by load_state_dict)

    def __init__(self, config: VAEConfig, device, dtype, frames_per_call, in_channels, out_channels):
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
        c.in_channels, c.out_channels = in_channels, out_channels
        c.num_blocks = len(config.block_out_channels)
        for i, v in enumerate(config.block_out_channels):
            c.block_out_channels[i] = v
        c.layers_per_block, c.heads = config.layers_per_block, 1
        c.cross_attention_dim, c.norm_num_groups, c.norm_eps = 64, config.norm_num_groups, 1e-6
        create = getattr(_lib(), f"mvb_create_vae_{self._kind}")
        rc = create(C.byref(c), self.device.index or 0, C.byref(self._h))
        if rc != 0:
            raise _capi.MvbError(f"mvb_create_vae_{self._kind} failed ({rc}): unsupported configuration or out of device memory")

    def _param_shapes(self):
        raise NotImplementedError

    def load_state_dict(self, state_dict: Dict[str, torch.Tensor], strict: bool = True):
        expected = self._param_shapes()
        missing = [k for k in expected if k not in state_dict]
        unexpected = [k for k in state_dict if k not in expected and not k.startswith(self._other)]
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

    def _call(self, x: torch.Tensor, out: torch.Tensor, h: int, w: int, latent_scale: float, postprocess: int) -> torch.Tensor:
        """Runs the half on x [N, ...] -> out [N, ...] in chunks of `frames_per_call` frames; h, w = latent size."""
        l = _lib()
        ws_fn = getattr(l, "mvb_vae_decode_workspace_bytes" if self._kind == "decoder" else "mvb_vae_encode_workspace_bytes")
        run_fn = getattr(l, "mvb_vae_decode" if self._kind == "decoder" else "mvb_vae_encode")
        N = x.shape[0]
        step = max(1, self.frames_per_call)
        for n0 in range(0, N, step):
            n1 = min(N, n0 + step)
            a = MvbVaeDecodeArgs()
            xc, oc = x[n0:n1], out[n0:n1]
            a.latents, a.latents_is_f32 = xc.data_ptr(), _is_f32(xc)
            a.N, a.h, a.w = n1 - n0, h, w
            a.latent_scale = float(latent_scale)
            a.out, a.out_is_f32 = oc.data_ptr(), _is_f32(oc)
            a.postprocess = int(postprocess)
            need = ws_fn(self._h, C.byref(a))
            if need < 0:
                raise _capi.MvbError(f"{ws_fn.__name__}: {l.mvb_handle_error(self._h).decode()}")
            if self._ws is None or self._ws.numel() < need:
                self._ws = None
                self._ws = torch.empty(int(need), dtype=torch.uint8, device=self.device)
            rc = run_fn(self._h, C.byref(a), self._ws.data_ptr(), self._ws.numel(), torch.cuda.current_stream(self.device).cuda_stream)
            if rc != 0:
                raise _capi.MvbError(f"{run_fn.__name__}: {l.mvb_handle_error(self._h).decode()}")
        self._keep = x
        return out


class AutoencoderKLDecoder(_EngineHalf):
    """Decode half of `AutoencoderKL` on the CUDA engine: `.decode(z)` (autoencoder_kl.py:275-302) and the pipeline-level
    `.decode_latents(latents)`; `.config.scaling_factor`, `.dtype`, `.device`, reference state-dict names (`decoder.*`,
    `post_quant_conv.*`; encoder / quant_conv entries of a full VAE state dict are ignored)."""

    _kind = "decoder"
    _other = ("encoder.", "quant_conv.")

    def __init__(self, config: VAEConfig = VAEConfig(), device: Union[str, torch.device] = "cuda", dtype: torch.dtype = torch.float16,
                 frames_per_call: int = 4):
        super().__init__(config, device, dtype, frames_per_call, config.latent_channels, config.out_channels)

    def _param_shapes(self):
        return vae_decoder_param_shapes(self.cfg)

    def _run(self, z: torch.Tensor, latent_scale: float, postprocess: bool, out_dtype: torch.dtype) -> torch.Tensor:
        if not self._loaded:
            raise RuntimeError("weights not loaded: call load_state_dict first")
        if z.dim() != 4 or z.shape[1] != self.cfg.latent_channels:
            raise ValueError(f"latents must be [N, {self.cfg.latent_channels}, h, w], got {tuple(z.shape)}")
        z = z.to(self.device)
        if z.dtype not in (torch.float16, torch.float32):
            z = z.float()
        z = z.contiguous()
        N, _, h, w = z.shape
        up = 2 ** (len(self.cfg.block_out_channels) - 1)
        out = torch.empty((N, self.cfg.out_channels, h * up, w * up), dtype=out_dtype, device=self.device)
        return self._call(z, out, h, w, latent_scale, postprocess)

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


class AutoencoderKLEncoder(_EngineHalf):
    """Encode half of `AutoencoderKL` on the CUDA engine: `.encode(x)` (autoencoder_kl.py:256-297) and `.encode_video(video)`;
    reference state-dict names (`encoder.*`, `quant_conv.*`; decoder / post_quant_conv entries of a full VAE state dict are
    ignored). The engine computes in fp16 with fp32 accumulation and statistics; conv_out and quant_conv stay in fp32.
    The moments come back in the input's dtype, as the reference returns them (autoencoder_kl.py:286-290)."""

    _kind = "encoder"
    _other = ("decoder.", "post_quant_conv.")

    def __init__(self, config: VAEConfig = VAEConfig(), device: Union[str, torch.device] = "cuda", dtype: torch.dtype = torch.float16,
                 frames_per_call: int = 4):
        super().__init__(config, device, dtype, frames_per_call, config.in_channels, config.latent_channels)

    def _param_shapes(self):
        return vae_encoder_param_shapes(self.cfg)

    def _run(self, x: torch.Tensor, postprocess: int, out_dtype: torch.dtype) -> torch.Tensor:
        if not self._loaded:
            raise RuntimeError("weights not loaded: call load_state_dict first")
        f = 2 ** (len(self.cfg.block_out_channels) - 1)
        if x.dim() != 4 or x.shape[1] != self.cfg.in_channels:
            raise ValueError(f"images must have {self.cfg.in_channels} channels ([N, {self.cfg.in_channels}, H, W]), got {tuple(x.shape)}")
        N, _, H, W = x.shape
        if H % f or W % f:
            raise ValueError(f"image size {H}x{W} must be a multiple of {f} (the encoder downsamples {f}x)")
        h, w = H // f, W // f
        if (h * w) % 64 or h * w > 8192:
            raise ValueError(f"latent size {h}x{w}: h*w must be a multiple of 64 and at most 8192 (mid-block attention)")
        x = x.to(self.device)
        if x.dtype not in (torch.float16, torch.float32):
            x = x.float()
        x = x.contiguous()
        zc = self.cfg.latent_channels
        out = torch.empty((N, zc if postprocess else 2 * zc, h, w), dtype=out_dtype, device=self.device)
        return self._call(x, out, h, w, self.cfg.scaling_factor, postprocess)

    @torch.no_grad()
    def encode(self, x: torch.Tensor, return_dict: bool = True):
        """AutoencoderKL.encode (autoencoder_kl.py:256-297): images [N, 3, H, W] in [-1, 1] ->
        latent_dist = DiagonalGaussianDistribution(moments [N, 8, H/8, W/8])."""
        out_dtype = x.dtype if x.dtype in (torch.float16, torch.float32) else torch.float32
        posterior = DiagonalGaussianDistribution(self._run(x, 0, out_dtype))
        if not return_dict:
            return (posterior,)
        return AutoencoderKLOutput(latent_dist=posterior)

    @torch.no_grad()
    def encode_video(self, video: torch.Tensor, out_dtype: Optional[torch.dtype] = None) -> torch.Tensor:
        """`scaling_factor * encode(frames).latent_dist.mean` of every frame of video [b, 3, f, H, W] -> latents
        [b, 4, f, H/8, W/8] (the mirror of `decode_latents`): the `condition_latents` / video2video init latents of
        pipeline_controlnet.py:348-368,978-981. Scale and the mean are applied in the library (fp32)."""
        b, c, f, H, W = video.shape
        x = video.permute(0, 2, 1, 3, 4).reshape(b * f, c, H, W)
        lat = self._run(x, 1, out_dtype or self.dtype)
        return lat.view(b, f, *lat.shape[1:]).permute(0, 2, 1, 3, 4).contiguous()


class AutoencoderKL:
    """Drop-in for the pipeline's `vae` (diffusers `AutoencoderKL` as MuseV uses it): one encoder and one decoder handle
    loaded from one full `AutoencoderKL.state_dict()`. `encode`, `decode`, `decode_latents`, `encode_video`, `config`
    (`scaling_factor`, `block_out_channels`, ...), `dtype`, `device`, `eval`."""

    def __init__(self, config: VAEConfig = VAEConfig(), device: Union[str, torch.device] = "cuda", dtype: torch.dtype = torch.float16,
                 frames_per_call: int = 4):
        self.encoder = AutoencoderKLEncoder(config, device, dtype, frames_per_call)
        self.decoder = AutoencoderKLDecoder(config, device, dtype, frames_per_call)
        self.cfg, self.config, self.device, self.dtype = config, self.decoder.config, self.decoder.device, dtype

    @property
    def frames_per_call(self) -> int:
        return self.encoder.frames_per_call

    @frames_per_call.setter
    def frames_per_call(self, n: int):
        self.encoder.frames_per_call = self.decoder.frames_per_call = int(n)

    def load_state_dict(self, state_dict: Dict[str, torch.Tensor], strict: bool = True):
        e = self.encoder.load_state_dict(state_dict, strict)
        d = self.decoder.load_state_dict(state_dict, strict)
        return SimpleNamespace(missing_keys=e.missing_keys + d.missing_keys,
                               unexpected_keys=[k for k in e.unexpected_keys if k in d.unexpected_keys])

    def eval(self):
        return self

    def encode(self, x: torch.Tensor, return_dict: bool = True):
        return self.encoder.encode(x, return_dict)

    def decode(self, z: torch.Tensor, return_dict: bool = True):
        return self.decoder.decode(z, return_dict)

    def decode_latents(self, latents: torch.Tensor) -> torch.Tensor:
        return self.decoder.decode_latents(latents)

    def encode_video(self, video: torch.Tensor, out_dtype: Optional[torch.dtype] = None) -> torch.Tensor:
        return self.encoder.encode_video(video, out_dtype)
