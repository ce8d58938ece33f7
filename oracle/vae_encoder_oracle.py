"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the VAE encode that runs before the denoise loop.

`AutoencoderKL.encode` = `Encoder.forward` + quant_conv + `DiagonalGaussianDistribution` (diffusers models/autoencoder_kl.py:256-297,
models/vae.py:133-175, 741-785): conv_in -> 4 x DownEncoderBlock2D (2 resnets + `Downsample2D(padding=0)`, which pads
(0, 1, 0, 1) and runs a stride-2 3x3 conv with pad 0, resnet.py:213-278; no downsampler on the last block) ->
UNetMidBlock2D (the decoder's: resnet, single-head attention, resnet) -> GroupNorm(eps 1e-6) + SiLU + conv_out (2 x latent
channels) -> quant_conv (1x1) -> moments = [mean | logvar]. The pipeline reads `scaling_factor * latent_dist.mean`
(musev/pipelines/pipeline_controlnet.py:348-368, 809-811, 978-981). The resnet / attention restatements are the decoder
oracle's (oracle/vae_oracle.py). Pinned against the unmodified diffusers `AutoencoderKL` by oracle/make_golden_vae_encoder.py
-> tests/golden/vae_encoder_*.pt. Not imported by the product path.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle.vae_oracle import VAEDecoderOracle


class VAEEncoderOracle(VAEDecoderOracle):
    @torch.no_grad()
    def moments(self, x):
        """images [N, C, H, W] -> moments [N, 2 zc, H / 2^(nb-1), W / 2^(nb-1)] (autoencoder_kl.py:282-284)."""
        cfg = self.cfg
        x = x.to(self.device, self.dtype)
        x = F.conv2d(x, self.sd["encoder.conv_in.weight"], self.sd["encoder.conv_in.bias"], padding=1)     # vae.py:136
        nb = len(cfg.block_out_channels)
        for i in range(nb):
            for j in range(cfg.layers_per_block):
                x = self.resnet(x, f"encoder.down_blocks.{i}.resnets.{j}")
            if i != nb - 1:
                p = f"encoder.down_blocks.{i}.downsamplers.0.conv"
                x = F.conv2d(F.pad(x, (0, 1, 0, 1)), self.sd[p + ".weight"], self.sd[p + ".bias"], stride=2)
        x = self.resnet(x, "encoder.mid_block.resnets.0")
        x = self.attention(x, "encoder.mid_block.attentions.0")
        x = self.resnet(x, "encoder.mid_block.resnets.1")
        x = F.silu(self._gn(x, "encoder.conv_norm_out"))
        x = F.conv2d(x, self.sd["encoder.conv_out.weight"], self.sd["encoder.conv_out.bias"], padding=1)
        return F.conv2d(x, self.sd["quant_conv.weight"], self.sd["quant_conv.bias"])

    @torch.no_grad()
    def latent_dist(self, x):
        """DiagonalGaussianDistribution (vae.py:741-753): (mean, clamped logvar, std)."""
        mean, logvar = torch.chunk(self.moments(x), 2, dim=1)
        logvar = torch.clamp(logvar, -30.0, 20.0)
        return mean, logvar, torch.exp(0.5 * logvar)

    @torch.no_grad()
    def encode_video(self, video):
        """scaling_factor * encode(frames).latent_dist.mean of video [b, c, f, H, W] -> [b, zc, f, h, w]."""
        b, c, f, H, W = video.shape
        x = video.permute(0, 2, 1, 3, 4).reshape(b * f, c, H, W)
        lat = self.cfg.scaling_factor * self.latent_dist(x)[0]
        return lat.view(b, f, *lat.shape[1:]).permute(0, 2, 1, 3, 4).contiguous()
