"""Host mirror of the VAE: the decode that follows the denoise loop (SURVEY.md section 8(f)-3) and the encode before it.

Reference: `MusevControlNetPipeline.decode_latents` (musev/pipelines/pipeline_controlnet.py:233-238; called per T-segment at
:2157-2171) -> `decode_latents` of the diffusers img2img pipeline (pipeline_stable_diffusion_img2img.py:486-495) ->
`AutoencoderKL.decode` (models/autoencoder_kl.py:275-302). post_quant_conv, the decoder's convolutions / GroupNorms /
single-head mid-block attention and the `image / 2 + 0.5, clamp(0, 1)` post-processing run inside libmusevb200.so
(`mvb_vae_decode`, musev_b200/csrc/engine_vae.cu `Engine::run_vae`). Frames are decoded in chunks (the reference enables VAE
slicing = one frame at a time, pipeline_controlnet_predictor.py:284) to bound the activation arena. No CPU fallback.

Encode: `AutoencoderKL.encode` (models/autoencoder_kl.py:256-297) = `Encoder.forward` (models/vae.py:133-175) + quant_conv run
inside the library (`mvb_vae_encode`, `Engine::run_vae_encode`); `DiagonalGaussianDistribution` (vae.py:741-785) is a few
torch ops on the small moments tensor here. The pipeline reads `vae.config.scaling_factor * vae.encode(x).latent_dist.mean`
at three call sites (musev/pipelines/pipeline_controlnet.py:348-368, 809-811, 978-981); `encode_video` computes exactly that
for a whole video in the library. `AutoencoderKL` holds both halves and stands in for `pipeline.vae`.

Multi-GPU: every frame is encoded and decoded on its own, so `process_group=<torch.distributed group>` (or
`torch.distributed.group.WORLD`) shares a call's frames out over the group's ranks: the chunks of `frames_per_call` frames
a single GPU would launch go to the ranks in contiguous ranges, and the ranks then exchange their rows on the device
(`_capi.launch_frame_chunks`). Every rank must make the same call, with the same input, and every rank receives the full
result, bit-identical to the single-GPU one. `process_group=None` (the default) never looks at `torch.distributed`.
"""
from __future__ import annotations

from dataclasses import asdict, dataclass
from types import SimpleNamespace
from typing import Dict, Optional, Union

import torch

from ._capi import EngineModel, make_config
# Names callers imported from this module before the binding moved to _capi; they are the binding's own objects.
from ._capi import MvbVaeDecodeArgs, lib as _lib  # noqa: F401
from .schema import VAEConfig, vae_decoder_param_shapes, vae_encoder_param_shapes


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


class _VaeHalf(EngineModel):
    """One engine handle of a VAE half, created from a `VAEConfig`; entries of the other half in a full VAE state dict are
    ignored by load_state_dict."""

    def __init__(self, config: VAEConfig, device, dtype, frames_per_call, in_channels, out_channels):
        self.cfg = config
        self.config = SimpleNamespace(**asdict(config))
        self.frames_per_call = int(frames_per_call)
        c = make_config(in_channels, out_channels, config.block_out_channels, config.layers_per_block, 1, 64,
                        config.norm_num_groups, 1e-6)
        super().__init__(c, device, dtype)


class AutoencoderKLDecoder(_VaeHalf):
    """Decode half of `AutoencoderKL` on the CUDA engine: `.decode(z)` (autoencoder_kl.py:275-302) and the pipeline-level
    `.decode_latents(latents)`; `.config.scaling_factor`, `.dtype`, `.device`, reference state-dict names (`decoder.*`,
    `post_quant_conv.*`; encoder / quant_conv entries of a full VAE state dict are ignored)."""

    _create, _workspace, _forward = "mvb_create_vae_decoder", "mvb_vae_decode_workspace_bytes", "mvb_vae_decode"
    _ignored = ("encoder.", "quant_conv.")

    def __init__(self, config: VAEConfig = VAEConfig(), device: Union[str, torch.device] = "cuda", dtype: torch.dtype = torch.float16,
                 frames_per_call: int = 4):
        super().__init__(config, device, dtype, frames_per_call, config.latent_channels, config.out_channels)

    def _param_shapes(self):
        return vae_decoder_param_shapes(self.cfg)

    def _run(self, z: torch.Tensor, latent_scale: float, postprocess: bool, out_dtype: torch.dtype,
             process_group=None) -> torch.Tensor:
        self._check_loaded()
        if z.dim() != 4 or z.shape[1] != self.cfg.latent_channels:
            raise ValueError(f"latents must be [N, {self.cfg.latent_channels}, h, w], got {tuple(z.shape)}")
        z = z.to(self.device)
        if z.dtype not in (torch.float16, torch.float32):
            z = z.float()
        z = z.contiguous()
        N, _, h, w = z.shape
        up = 2 ** (len(self.cfg.block_out_channels) - 1)
        out = torch.empty((N, self.cfg.out_channels, h * up, w * up), dtype=out_dtype, device=self.device)
        return self._launch_frames(z, out, h, w, latent_scale, postprocess, process_group)

    @torch.no_grad()
    def decode(self, z: torch.Tensor, return_dict: bool = True, process_group=None):
        """AutoencoderKL.decode (autoencoder_kl.py:275-302): z [N, 4, h, w] -> image [N, 3, 8h, 8w] (no scaling, no clamp).
        process_group: a `torch.distributed` group (or `group.WORLD`) shares the frames out over its ranks; see the module
        notes. None (the default) decodes every frame here."""
        img = self._run(z, 1.0, False, self.dtype, process_group)
        if not return_dict:
            return (img,)
        return DecoderOutput(sample=img)

    @torch.no_grad()
    def decode_latents(self, latents: torch.Tensor, process_group=None) -> torch.Tensor:
        """MusevControlNetPipeline.decode_latents (pipeline_controlnet.py:233-238): latents [b, c, f, h, w] ->
        video [b, c, f, H, W] float32 in [0, 1]. The reference returns a CPU numpy array; this returns the device tensor
        (call `.cpu().numpy()` where the reference's `np.concatenate` of segments needs it). process_group: as in `decode`;
        every rank holds the whole video afterwards (a 512-frame 512x768 video is 2.4 GB of fp32 per rank)."""
        b, c, f, h, w = latents.shape
        z = latents.permute(0, 2, 1, 3, 4).reshape(b * f, c, h, w)
        img = self._run(z, 1.0 / self.cfg.scaling_factor, True, torch.float32, process_group)
        return img.view(b, f, *img.shape[1:]).permute(0, 2, 1, 3, 4).contiguous()


class AutoencoderKLEncoder(_VaeHalf):
    """Encode half of `AutoencoderKL` on the CUDA engine: `.encode(x)` (autoencoder_kl.py:256-297) and `.encode_video(video)`;
    reference state-dict names (`encoder.*`, `quant_conv.*`; decoder / post_quant_conv entries of a full VAE state dict are
    ignored). The engine computes in fp16 with fp32 accumulation and statistics; conv_out and quant_conv stay in fp32.
    The moments come back in the input's dtype, as the reference returns them (autoencoder_kl.py:286-290)."""

    _create, _workspace, _forward = "mvb_create_vae_encoder", "mvb_vae_encode_workspace_bytes", "mvb_vae_encode"
    _ignored = ("decoder.", "post_quant_conv.")

    def __init__(self, config: VAEConfig = VAEConfig(), device: Union[str, torch.device] = "cuda", dtype: torch.dtype = torch.float16,
                 frames_per_call: int = 4):
        super().__init__(config, device, dtype, frames_per_call, config.in_channels, config.latent_channels)

    def _param_shapes(self):
        return vae_encoder_param_shapes(self.cfg)

    def _run(self, x: torch.Tensor, postprocess: int, out_dtype: torch.dtype, process_group=None) -> torch.Tensor:
        self._check_loaded()
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
        return self._launch_frames(x, out, h, w, self.cfg.scaling_factor, postprocess, process_group)

    @torch.no_grad()
    def encode(self, x: torch.Tensor, return_dict: bool = True, process_group=None):
        """AutoencoderKL.encode (autoencoder_kl.py:256-297): images [N, 3, H, W] in [-1, 1] ->
        latent_dist = DiagonalGaussianDistribution(moments [N, 8, H/8, W/8]). process_group: a `torch.distributed` group
        (or `group.WORLD`) shares the frames out over its ranks; see the module notes. None (the default) encodes every
        frame here."""
        out_dtype = x.dtype if x.dtype in (torch.float16, torch.float32) else torch.float32
        posterior = DiagonalGaussianDistribution(self._run(x, 0, out_dtype, process_group))
        if not return_dict:
            return (posterior,)
        return AutoencoderKLOutput(latent_dist=posterior)

    @torch.no_grad()
    def encode_video(self, video: torch.Tensor, out_dtype: Optional[torch.dtype] = None,
                     process_group=None) -> torch.Tensor:
        """`scaling_factor * encode(frames).latent_dist.mean` of every frame of video [b, 3, f, H, W] -> latents
        [b, 4, f, H/8, W/8] (the mirror of `decode_latents`): the `condition_latents` / video2video init latents of
        pipeline_controlnet.py:348-368,978-981. Scale and the mean are applied in the library (fp32). process_group: as
        in `encode`."""
        b, c, f, H, W = video.shape
        x = video.permute(0, 2, 1, 3, 4).reshape(b * f, c, H, W)
        lat = self._run(x, 1, out_dtype or self.dtype, process_group)
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

    def encode(self, x: torch.Tensor, return_dict: bool = True, process_group=None):
        return self.encoder.encode(x, return_dict, process_group=process_group)

    def decode(self, z: torch.Tensor, return_dict: bool = True, process_group=None):
        return self.decoder.decode(z, return_dict, process_group=process_group)

    def decode_latents(self, latents: torch.Tensor, process_group=None) -> torch.Tensor:
        return self.decoder.decode_latents(latents, process_group=process_group)

    def encode_video(self, video: torch.Tensor, out_dtype: Optional[torch.dtype] = None,
                     process_group=None) -> torch.Tensor:
        return self.encoder.encode_video(video, out_dtype, process_group=process_group)
