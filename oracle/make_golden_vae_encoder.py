"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/vae_encoder_{narrow,full}.pt by running the UNMODIFIED diffusers
`AutoencoderKL.encode` of the reference tree on CPU in fp32 (the companion of `golden_vae` in oracle/make_golden.py).

Run in the build container only:  python -m oracle.make_golden_vae_encoder
Weights and images are regenerated from the seeds in the fixture's meta (musev_b200.synth, bit-identical CPU RNG);
the fixture keeps 2048 seeded sample positions of the moments. The reference is never read at test time.
"""
from __future__ import annotations

import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from musev_b200.schema import VAEConfig, vae_encoder_param_shapes  # noqa: E402
from musev_b200.synth import make_state_dict, make_vae_images  # noqa: E402
from oracle import ref_shim  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")


def golden_vae_encoder(boc, tag, frames, H, W, wseed=11, iseed=2469):
    """The unmodified diffusers `AutoencoderKL.encode` (vendored fork; fp32 input, so its fp16 up-cast does not apply) on
    seeded weights: 2048 seeded sample positions of the moments [mean | logvar] before the logvar clamp."""
    ref_shim.load()
    from diffusers.models.autoencoder_kl import AutoencoderKL
    cfg = VAEConfig(block_out_channels=tuple(boc))
    kw = dict(in_channels=3, out_channels=3, down_block_types=("DownEncoderBlock2D",) * 4, up_block_types=("UpDecoderBlock2D",) * 4,
              block_out_channels=tuple(boc), layers_per_block=2, act_fn="silu", latent_channels=4, norm_num_groups=32,
              sample_size=512, scaling_factor=0.18215)
    t0 = time.time()
    m = AutoencoderKL(**kw).eval()
    ref_shapes = {k: tuple(v.shape) for k, v in m.state_dict().items() if k.startswith(("encoder.", "quant_conv."))}
    mine = {k: tuple(v) for k, v in vae_encoder_param_shapes(cfg).items()}
    assert ref_shapes == mine, "VAE encoder schema mismatch vs reference state_dict"
    res = m.load_state_dict(make_state_dict(cfg, seed=wseed), strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    x = make_vae_images(frames, H, W, iseed)
    with torch.no_grad():
        post = m.encode(x).latent_dist
    moments = post.parameters
    flat = moments.reshape(-1)
    idx = torch.randint(0, flat.numel(), (2048,), generator=torch.Generator().manual_seed(3001))
    meta = dict(block_out_channels=list(boc), frames=frames, H=H, W=W, weight_seed=wseed, input_seed=iseed,
                shape=list(moments.shape), sample_seed=3001, n_samples=2048,
                source="reference diffusers.models.autoencoder_kl.AutoencoderKL.encode (vendored fork), CPU fp32")
    path = os.path.join(GOLDEN, f"vae_encoder_{tag}.pt")
    torch.save({"meta": meta, "moments": flat[idx].clone(),
                "stats": [float(post.mean.mean()), float(post.mean.abs().mean()), float(post.logvar.mean())]}, path)
    print(f"{path}: mean abs-mean {float(post.mean.abs().mean()):.4f} logvar mean {float(post.logvar.mean()):.4f} "
          f"({time.time() - t0:.1f}s)", flush=True)


if __name__ == "__main__":
    os.makedirs(GOLDEN, exist_ok=True)
    torch.set_num_threads(os.cpu_count() or 1)
    golden_vae_encoder((64, 64, 128, 128), "narrow", frames=2, H=64, W=64)
    golden_vae_encoder((128, 256, 512, 512), "full", frames=1, H=64, W=64)
