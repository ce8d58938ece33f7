"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/vae_tiled_*.pt by running the UNMODIFIED diffusers `AutoencoderKL`
(tiled mode, models/autoencoder_kl.py:354-466) of the reference tree on CPU.

Run in the build container only:  python -m oracle.make_golden_vae_tiled

  vae_tiled_blend.pt   the stitch alone: `tiled_decode` / `tiled_encode` with the VAE halves replaced by stubs that hand
                       out seeded random tiles in call order (post_quant_conv / quant_conv by identities). Each case keeps
                       the tile seed, the tile shapes in call order and the reference's stitched output; the tiles
                       themselves are redrawn from the seed at test time (oracle/vae_tiled_oracle.py `blend_case_tiles`,
                       bit-identical CPU RNG).
                       Decode in fp32, encode in fp32 and fp16. Geometries with sliver edge tiles, one tile row and one
                       tile column.
  vae_tiled_narrow.pt  the narrow VAE (64, 64, 128, 128) with sample_size 256 (32-latent tiles, 8- and 16-latent
                       slivers): `decode` of a 56x40 latent and `encode` of a 448x320 image with `enable_tiling()`, fp32,
                       2048 seeded sample positions of each output (as oracle/make_golden_vae_encoder.py keeps them).
Weights and inputs are regenerated from the seeds in the meta (musev_b200.synth); the reference is never read at test time.
"""
from __future__ import annotations

import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from musev_b200.schema import VAEConfig  # noqa: E402
from musev_b200.synth import make_state_dict, make_vae_images  # noqa: E402
from oracle import ref_shim  # noqa: E402
from oracle.vae_tiled_oracle import blend_case_tiles  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")

# (kind, input H, W, tile_sample_min_size, tile_latent_min_size, dtype); the stubs scale sizes by FACTOR. Decode cases run
# one frame of 2 channels, encode cases 2 frames of 4 moment channels (2 mean + 2 logvar), so that the fixture stays small
FACTOR = 2
BLEND_CASES = [
    ("decode", 28, 28, 32, 16, torch.float32),     # 3 x 3 tiles, 8-pixel slivers (as long as the 8-pixel extent)
    ("decode", 30, 28, 32, 16, torch.float32),     # 12-pixel row sliver, 8-pixel column sliver
    ("decode", 12, 40, 32, 16, torch.float32),     # one tile row
    ("decode", 40, 12, 32, 16, torch.float32),     # one tile column
    ("encode", 56, 56, 32, 16, torch.float32),     # 3 x 3 tiles, 4-latent slivers
    ("encode", 56, 56, 32, 16, torch.float16),
    ("encode", 60, 56, 32, 16, torch.float16),     # 6-latent row sliver, 4-latent column sliver
    ("encode", 24, 80, 32, 16, torch.float32),     # one tile row
    ("encode", 80, 24, 32, 16, torch.float16),     # one tile column
]
BLEND_FRAMES = {"decode": 1, "encode": 2}
BLEND_CHANNELS = {"decode": 2, "encode": 4}


class _TileStub(torch.nn.Module):
    """Stands in for `decoder` / `encoder`: each call returns a fresh seeded random tile of the output shape, recorded."""

    def __init__(self, channels: int, scale_num: int, scale_den: int, seed: int):
        super().__init__()
        self.c, self.num, self.den = channels, scale_num, scale_den
        self.gen = torch.Generator().manual_seed(seed)
        self.drawn = []

    def forward(self, x):
        n, _, h, w = x.shape
        t = torch.randn(n, self.c, h * self.num // self.den, w * self.num // self.den, generator=self.gen).to(x.dtype)
        self.drawn.append(t.clone())
        return t


def _reference_vae(boc, sample_size):
    ref_shim.load()
    from diffusers.models.autoencoder_kl import AutoencoderKL
    return AutoencoderKL(in_channels=3, out_channels=3, down_block_types=("DownEncoderBlock2D",) * len(boc),
                         up_block_types=("UpDecoderBlock2D",) * len(boc), block_out_channels=tuple(boc),
                         layers_per_block=2, act_fn="silu", latent_channels=4, norm_num_groups=32,
                         sample_size=sample_size, scaling_factor=0.18215).eval()


def golden_blend():
    m = _reference_vae((32,), 32)
    cases = []
    for k, (kind, H, W, tsm, tlm, dtype) in enumerate(BLEND_CASES):
        m.tile_sample_min_size, m.tile_latent_min_size, m.tile_overlap_factor = tsm, tlm, 0.25
        x = torch.randn(BLEND_FRAMES[kind], 4 if kind == "decode" else 3, H, W,
                        generator=torch.Generator().manual_seed(100 + k)).to(dtype)
        with torch.no_grad():
            if kind == "decode":
                stub = _TileStub(BLEND_CHANNELS[kind], FACTOR, 1, 200 + k)
                m.decoder, m.post_quant_conv = stub, torch.nn.Identity()
                out = m.tiled_decode(x).sample
            else:
                stub = _TileStub(BLEND_CHANNELS[kind], 1, FACTOR, 200 + k)
                m.encoder, m.quant_conv = stub, torch.nn.Identity()
                out = m.tiled_encode(x).latent_dist.parameters
        assert out.dtype == dtype
        case = dict(kind=kind, H=H, W=W, tile_sample_min_size=tsm, tile_latent_min_size=tlm, tile_overlap_factor=0.25,
                    factor=FACTOR, dtype=str(dtype).split(".")[-1], tile_seed=200 + k,
                    tile_shapes=[tuple(t.shape) for t in stub.drawn], out=out.clone())
        assert all(torch.equal(a, b) for a, b in zip(blend_case_tiles(case), stub.drawn))
        cases.append(case)
        print(f"blend {kind} {H}x{W} {dtype}: {len(stub.drawn)} tiles -> {list(out.shape)}", flush=True)
    meta = dict(source="reference diffusers AutoencoderKL.tiled_decode / tiled_encode (vendored fork), CPU, tile stubs")
    torch.save({"meta": meta, "cases": cases}, os.path.join(GOLDEN, "vae_tiled_blend.pt"))


def golden_narrow(wseed=11):
    boc = (64, 64, 128, 128)
    cfg = VAEConfig(block_out_channels=boc, sample_size=256)
    m = _reference_vae(boc, 256)
    res = m.load_state_dict(make_state_dict(cfg, seed=wseed), strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    m.enable_tiling()
    assert m.tile_latent_min_size == 32 and m.tile_sample_min_size == 256
    t0 = time.time()
    z = torch.randn(2, 4, 56, 40, generator=torch.Generator().manual_seed(77)) * 1.2
    x = make_vae_images(2, 448, 320, seed=78)
    with torch.no_grad():
        raw = m.decode(z).sample
        moments = m.encode(x).latent_dist.parameters
    g = torch.Generator().manual_seed(3001)
    idx_d = torch.randint(0, raw.numel(), (2048,), generator=g)
    idx_e = torch.randint(0, moments.numel(), (2048,), generator=g)
    meta = dict(block_out_channels=list(boc), sample_size=256, weight_seed=wseed, latent_seed=77, latent_shape=list(z.shape),
                latent_std=1.2, image_seed=78, image_shape=list(x.shape), raw_shape=list(raw.shape),
                moments_shape=list(moments.shape), sample_seed=3001, n_samples=2048,
                source="reference diffusers AutoencoderKL.decode / encode with enable_tiling() (vendored fork), CPU fp32")
    torch.save({"meta": meta, "idx_raw": idx_d, "raw": raw.reshape(-1)[idx_d].clone(), "idx_moments": idx_e,
                "moments": moments.reshape(-1)[idx_e].clone()}, os.path.join(GOLDEN, "vae_tiled_narrow.pt"))
    print(f"narrow: raw {list(raw.shape)} moments {list(moments.shape)} ({time.time() - t0:.1f}s)", flush=True)


if __name__ == "__main__":
    os.makedirs(GOLDEN, exist_ok=True)
    torch.set_num_threads(os.cpu_count() or 1)
    golden_blend()
    golden_narrow()
