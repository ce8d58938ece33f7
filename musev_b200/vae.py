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

from . import ops, vae_tiling
from ._capi import EngineModel, _is_f32, frame_chunks, launch_frame_chunks, make_config
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
    ignored by load_state_dict.

    Tiled mode (diffusers autoencoder_kl.py:127-171): `enable_tiling()` makes encode / decode split frames larger than
    `tile_sample_min_size` image pixels (`tile_latent_min_size` latent pixels) into overlapping tiles, run each tile on
    its own and blend them (`musev_b200.vae_tiling`, `mvb_op_vae_tile_blend`). `enable_slicing()` only records the flag:
    frames are always run in chunks of `frames_per_call`, with the same bits per frame as one at a time."""

    def __init__(self, config: VAEConfig, device, dtype, frames_per_call, in_channels, out_channels):
        self.cfg = config
        self.config = SimpleNamespace(**asdict(config))
        self.frames_per_call = int(frames_per_call)
        self.factor = 2 ** (len(config.block_out_channels) - 1)
        self.use_slicing = False
        self.use_tiling = False
        self.tile_sample_min_size = config.sample_size
        self.tile_latent_min_size = int(config.sample_size / self.factor)
        self.tile_overlap_factor = 0.25
        c = make_config(in_channels, out_channels, config.block_out_channels, config.layers_per_block, 1, 64,
                        config.norm_num_groups, 1e-6)
        super().__init__(c, device, dtype)

    def enable_tiling(self, use_tiling: bool = True):
        self.use_tiling = use_tiling

    def disable_tiling(self):
        self.enable_tiling(False)

    def enable_slicing(self):
        self.use_slicing = True

    def disable_slicing(self):
        self.use_slicing = False

    def _launch_tiles(self, x: torch.Tensor, out: torch.Tensor, plan: vae_tiling.TilePlan, latent_scale: float,
                      tile_dtype: torch.dtype, mode: int, scale: float, process_group=None) -> torch.Tensor:
        """x [N, c, H, W] -> out [N, c', H', W'] by the tile plan, per chunk of `frames_per_call` frames (shared out over
        the ranks of a process group as untiled calls are): each shape group's tiles are cut out of the chunk's frames
        with strided views and one copy, run as the N of engine calls of at most `frames_per_call` tiles (in
        `tile_dtype`, no post-processing), and one `mvb_op_vae_tile_blend` stitches the chunk into out."""
        step = max(1, self.frames_per_call)
        S = plan.overlap_size
        cout = self._tile_channels()

        def launch(n0: int, n1: int) -> None:
            xc = x[n0:n1]
            nf = n1 - n0
            bufs = {}
            for rc, cc in plan.groups:
                v = xc[:, :, rc.first * S:, cc.first * S:].unfold(2, rc.size_in, S)[:, :, :rc.count]
                v = v.unfold(3, cc.size_in, S)[:, :, :, :cc.count]                   # [nf, c, nr, nc, th, tw]
                tiles_in = v.permute(0, 2, 3, 1, 4, 5).contiguous().view(nf * rc.count * cc.count, xc.shape[1],
                                                                          rc.size_in, cc.size_in)
                tiles_out = torch.empty((tiles_in.shape[0], cout, rc.size_out, cc.size_out), dtype=tile_dtype,
                                        device=self.device)
                h, w = self._engine_hw(rc, cc)
                for k0, k1 in frame_chunks(tiles_in.shape[0], step):
                    ti, to = tiles_in[k0:k1], tiles_out[k0:k1]
                    a = MvbVaeDecodeArgs()
                    a.latents, a.latents_is_f32 = ti.data_ptr(), _is_f32(ti)
                    a.N, a.h, a.w = ti.shape[0], h, w
                    a.latent_scale = float(latent_scale)
                    a.out, a.out_is_f32 = to.data_ptr(), _is_f32(to)
                    a.postprocess = 0
                    self._launch(a)
                bufs[(rc, cc)] = tiles_out
            ops.vae_tile_blend([[bufs[(rc, cc)] for cc in plan.cols.classes] for rc in plan.rows.classes], plan,
                               out[n0:n1], mode, scale)

        # the tile buffers are freed to the caching allocator in stream order, so they need no keeping
        launch_frame_chunks(x, out, step, launch, process_group)
        self._keep = x   # the input must outlive the asynchronous launches
        return out


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

    def _tile_channels(self) -> int:
        return self.cfg.out_channels

    def _engine_hw(self, rc, cc):
        return rc.size_in, cc.size_in          # mvb_vae_decode takes the latent size

    def _tiled(self, z: torch.Tensor) -> bool:
        """autoencoder_kl.py:300: tiled when tiling is on and a latent side exceeds tile_latent_min_size."""
        return self.use_tiling and (z.shape[-1] > self.tile_latent_min_size or z.shape[-2] > self.tile_latent_min_size)

    def _run_tiled(self, z: torch.Tensor, latent_scale: float, postprocess: bool, out_dtype: torch.dtype,
                   process_group=None) -> torch.Tensor:
        """`tiled_decode` (autoencoder_kl.py:420-466): tiles decoded to fp32 (decode's fp32 up-cast, :329-335), blended in
        fp32 and rounded once to out_dtype by the blend kernel, which also applies decode_latents' post-processing after
        the blend."""
        self._check_loaded()
        if z.dim() != 4 or z.shape[1] != self.cfg.latent_channels:
            raise ValueError(f"latents must be [N, {self.cfg.latent_channels}, h, w], got {tuple(z.shape)}")
        N, _, h, w = z.shape
        plan = vae_tiling.plan_decode(h, w, self.tile_sample_min_size, self.tile_latent_min_size,
                                      self.tile_overlap_factor, self.factor)
        z = z.to(self.device)
        if z.dtype not in (torch.float16, torch.float32):
            z = z.float()
        z = z.contiguous()
        out = torch.empty((N, self.cfg.out_channels, plan.out_h, plan.out_w), dtype=out_dtype, device=self.device)
        return self._launch_tiles(z, out, plan, latent_scale, torch.float32, 1 if postprocess else 0, 1.0, process_group)

    @torch.no_grad()
    def tiled_decode(self, z: torch.Tensor, return_dict: bool = True, process_group=None):
        """AutoencoderKL.tiled_decode (autoencoder_kl.py:420-466) whatever the frame size: z [N, 4, h, w] -> image
        [N, 3, 8h, 8w] in the handle's dtype. Raises ValueError, before any launch, for tile attributes the engine cannot
        run (`musev_b200.vae_tiling.plan_decode`)."""
        img = self._run_tiled(z, 1.0, False, self.dtype, process_group)
        if not return_dict:
            return (img,)
        return DecoderOutput(sample=img)

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
        if self._tiled(z):
            return self.tiled_decode(z, return_dict, process_group=process_group)
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
        run = self._run_tiled if self._tiled(z) else self._run
        img = run(z, 1.0 / self.cfg.scaling_factor, True, torch.float32, process_group)
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

    def _tile_channels(self) -> int:
        return 2 * self.cfg.latent_channels

    def _engine_hw(self, rc, cc):
        return rc.size_out, cc.size_out        # mvb_vae_encode takes the latent size

    def _tiled(self, x: torch.Tensor) -> bool:
        """autoencoder_kl.py:267: tiled when tiling is on and an image side exceeds tile_sample_min_size."""
        return self.use_tiling and (x.shape[-1] > self.tile_sample_min_size or x.shape[-2] > self.tile_sample_min_size)

    def _run_tiled(self, x: torch.Tensor, postprocess: int, out_dtype: torch.dtype, process_group=None) -> torch.Tensor:
        """`tiled_encode` (autoencoder_kl.py:366-418): encode dispatches to it before its fp32 up-cast (:267-276), so the
        tiles' moments are blended in the image's dtype (fp16 / fp32; other dtypes run as fp32). postprocess 1 then
        takes `scaling_factor * mean` in fp32, as the untiled path does, and rounds once to out_dtype."""
        self._check_loaded()
        if x.dim() != 4 or x.shape[1] != self.cfg.in_channels:
            raise ValueError(f"images must have {self.cfg.in_channels} channels ([N, {self.cfg.in_channels}, H, W]), got {tuple(x.shape)}")
        N, _, H, W = x.shape
        plan = vae_tiling.plan_encode(H, W, self.tile_sample_min_size, self.tile_latent_min_size,
                                      self.tile_overlap_factor, self.factor)
        x = x.to(self.device)
        if x.dtype not in (torch.float16, torch.float32):
            x = x.float()
        x = x.contiguous()
        zc = self.cfg.latent_channels
        out = torch.empty((N, zc if postprocess else 2 * zc, plan.out_h, plan.out_w), dtype=out_dtype, device=self.device)
        return self._launch_tiles(x, out, plan, self.cfg.scaling_factor, x.dtype, 2 if postprocess else 0,
                                  self.cfg.scaling_factor, process_group)

    @torch.no_grad()
    def tiled_encode(self, x: torch.Tensor, return_dict: bool = True, process_group=None):
        """AutoencoderKL.tiled_encode (autoencoder_kl.py:366-418) whatever the image size: images [N, 3, H, W] ->
        latent_dist of the blended moments, in the images' dtype. Raises ValueError, before any launch, for geometries
        the engine cannot run (`musev_b200.vae_tiling.plan_encode`)."""
        out_dtype = x.dtype if x.dtype in (torch.float16, torch.float32) else torch.float32
        posterior = DiagonalGaussianDistribution(self._run_tiled(x, 0, out_dtype, process_group))
        if not return_dict:
            return (posterior,)
        return AutoencoderKLOutput(latent_dist=posterior)

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
        if self._tiled(x):
            return self.tiled_encode(x, return_dict, process_group=process_group)
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
        run = self._run_tiled if self._tiled(x) else self._run
        lat = run(x, 1, out_dtype or self.dtype, process_group)
        return lat.view(b, f, *lat.shape[1:]).permute(0, 2, 1, 3, 4).contiguous()


class AutoencoderKL:
    """Drop-in for the pipeline's `vae` (diffusers `AutoencoderKL` as MuseV uses it): one encoder and one decoder handle
    loaded from one full `AutoencoderKL.state_dict()`. `encode`, `decode`, `decode_latents`, `encode_video`, `config`
    (`scaling_factor`, `block_out_channels`, `sample_size`, ...), `dtype`, `device`, `eval`; tiled mode (`enable_tiling`,
    `tiled_encode`, `tiled_decode` and the `tile_*` attributes, shared by both halves) and `enable_slicing`."""

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

    def tiled_encode(self, x: torch.Tensor, return_dict: bool = True, process_group=None):
        return self.encoder.tiled_encode(x, return_dict, process_group=process_group)

    def tiled_decode(self, z: torch.Tensor, return_dict: bool = True, process_group=None):
        return self.decoder.tiled_decode(z, return_dict, process_group=process_group)

    def enable_tiling(self, use_tiling: bool = True):
        """diffusers autoencoder_kl.py:144-150; what `pipeline.enable_vae_tiling()` calls."""
        self.use_tiling = use_tiling

    def disable_tiling(self):
        self.enable_tiling(False)

    def enable_slicing(self):
        """autoencoder_kl.py:159-164 (pipeline_controlnet_predictor.py:284 calls it); records the flag only."""
        self.use_slicing = True

    def disable_slicing(self):
        self.use_slicing = False


def _both_halves(name: str) -> property:
    """A tiling attribute of `AutoencoderKL`: read from the decoder, written to both halves."""
    def get(self):
        return getattr(self.decoder, name)

    def set(self, value):
        setattr(self.encoder, name, value)
        setattr(self.decoder, name, value)
    return property(get, set)


for _name in ("use_slicing", "use_tiling", "tile_sample_min_size", "tile_latent_min_size", "tile_overlap_factor"):
    setattr(AutoencoderKL, _name, _both_halves(_name))
