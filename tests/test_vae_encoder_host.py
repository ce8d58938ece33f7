"""CPU tests of the VAE encoder's host side: the encoder oracle against the unmodified diffusers `AutoencoderKL.encode`
(tests/golden/vae_encoder_*.pt), the VAE FLOP counters against torch's FlopCounterMode on the oracles, the full-VAE
seeded state dict, and the DiagonalGaussianDistribution mirror."""
import os

import pytest
import torch
from torch.utils.flop_counter import FlopCounterMode

from conftest import GOLDEN


@pytest.mark.parametrize("tag", ["narrow", "full"])
def test_vae_encoder_oracle_matches_reference_golden(tag):
    from musev_b200.schema import VAEConfig
    from musev_b200.synth import make_state_dict, make_vae_images
    from oracle.vae_encoder_oracle import VAEEncoderOracle
    g = torch.load(os.path.join(GOLDEN, f"vae_encoder_{tag}.pt"))
    m = g["meta"]
    cfg = VAEConfig(block_out_channels=tuple(m["block_out_channels"]))
    oracle = VAEEncoderOracle(cfg, make_state_dict(cfg, seed=m["weight_seed"]))
    mom = oracle.moments(make_vae_images(m["frames"], m["H"], m["W"], m["input_seed"]))
    assert list(mom.shape) == m["shape"]
    idx = torch.randint(0, mom.numel(), (m["n_samples"],), generator=torch.Generator().manual_seed(m["sample_seed"]))
    assert (mom.reshape(-1)[idx] - g["moments"]).abs().max().item() < 1e-5 * max(1.0, g["moments"].abs().max().item())


def _meta_flops(fn):
    with FlopCounterMode(display=False) as fc:
        fn()
    return fc.get_total_flops()


def test_vae_flop_counters_match_flop_counter_mode():
    from musev_b200.flops import vae_decoder_flops, vae_encoder_flops
    from musev_b200.schema import VAEConfig, vae_decoder_param_shapes, vae_encoder_param_shapes
    from oracle.vae_encoder_oracle import VAEEncoderOracle
    from oracle.vae_oracle import VAEDecoderOracle
    for cfg, N, h, w in ((VAEConfig(), 1, 64, 64), (VAEConfig(block_out_channels=(64, 64, 128, 128)), 2, 8, 16)):
        f = 2 ** (len(cfg.block_out_channels) - 1)
        sd = {k: torch.empty(s, device="meta") for k, s in vae_encoder_param_shapes(cfg).items()}
        sd.update({k: torch.empty(s, device="meta") for k, s in vae_decoder_param_shapes(cfg).items()})
        enc = VAEEncoderOracle(cfg, sd, device="meta")
        dec = VAEDecoderOracle(cfg, sd, device="meta")
        x = torch.empty(N, cfg.in_channels, h * f, w * f, device="meta")
        z = torch.empty(N, cfg.latent_channels, h, w, device="meta")
        assert vae_encoder_flops(cfg, N, h, w)["total"] == _meta_flops(lambda: enc.moments(x))
        assert vae_decoder_flops(cfg, N, h, w)["total"] == _meta_flops(lambda: dec.decode(z))
    sd15 = VAEConfig()
    assert round(vae_encoder_flops(sd15, 1, 64, 64)["total"] / 1e12, 3) == 1.117
    assert round(vae_decoder_flops(sd15, 1, 64, 64)["total"] / 1e12, 3) == 2.515


def test_vae_state_dict_is_both_halves():
    from musev_b200.schema import VAEConfig, vae_decoder_param_shapes, vae_encoder_param_shapes
    from musev_b200.synth import make_state_dict
    cfg = VAEConfig(block_out_channels=(64, 64, 128, 128))
    sd = make_state_dict(cfg, seed=11)
    enc, dec = vae_encoder_param_shapes(cfg), vae_decoder_param_shapes(cfg)
    assert not set(enc) & set(dec)
    assert {k: tuple(v.shape) for k, v in sd.items()} == {**enc, **dec}
    assert len(vae_encoder_param_shapes(VAEConfig())) == 108


def test_diagonal_gaussian_mirror():
    from musev_b200.vae import DiagonalGaussianDistribution
    g = torch.Generator().manual_seed(0)
    moments = torch.randn(2, 8, 4, 4, generator=g) * 30
    d = DiagonalGaussianDistribution(moments)
    assert torch.equal(d.mean, moments[:, :4]) and torch.equal(d.mode(), d.mean)
    assert torch.equal(d.logvar, moments[:, 4:].clamp(-30.0, 20.0))
    assert torch.equal(d.std, torch.exp(0.5 * d.logvar)) and torch.equal(d.var, torch.exp(d.logvar))
    s = d.sample(torch.Generator().manual_seed(3))
    eps = torch.randn(2, 4, 4, 4, generator=torch.Generator().manual_seed(3))
    assert torch.equal(s, d.mean + d.std * eps)
