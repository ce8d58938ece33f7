"""TEST INFRASTRUCTURE ONLY -- plain-torch restatement of diffusers' tiled VAE (`AutoencoderKL.tiled_decode` /
`tiled_encode`, models/autoencoder_kl.py:354-466) around the decoder and encoder oracles, plus the closed form of the
stitch that the engine's blend kernel evaluates per pixel (musev_b200/csrc/vae_tiles.cu, DESIGN.md 4.9).

  * `stitch`: the reference's loop. Tiles are visited row-major; tile (i, j) is blended IN PLACE with the tile above
    (`blend_v`, :354-358) and then with the tile to its left (`blend_h`, :360-364), both already blended themselves, and
    its [:row_limit, :row_limit] crop is kept (:400-412, :449-462).
  * `stitch_closed_form`: the same result from the raw tiles only, vectorised; equal to `stitch` whenever
    `musev_b200.vae_tiling` accepts the geometry (tests/test_vae_tiled_host.py).
  * `tiled_decode` / `tiled_encode`: the tile loops of :385-398 and :434-448 with the oracles as the VAE halves.
Pinned against the unmodified diffusers `AutoencoderKL` by oracle/make_golden_vae_tiled.py -> tests/golden/vae_tiled_*.pt.
Not imported by the product path.
"""
from __future__ import annotations

from typing import List

import torch


def blend_v(a: torch.Tensor, b: torch.Tensor, extent: int) -> torch.Tensor:
    """Mixes the top rows of b with the bottom rows of a, in place on b: weight t/e for b at row t."""
    e = min(a.shape[2], b.shape[2], extent)
    for t in range(e):
        b[:, :, t, :] = a[:, :, t - e, :] * (1 - t / e) + b[:, :, t, :] * (t / e)
    return b


def blend_h(a: torch.Tensor, b: torch.Tensor, extent: int) -> torch.Tensor:
    """blend_v along the columns."""
    e = min(a.shape[3], b.shape[3], extent)
    for t in range(e):
        b[:, :, :, t] = a[:, :, :, t - e] * (1 - t / e) + b[:, :, :, t] * (t / e)
    return b


def stitch(grid: List[List[torch.Tensor]], extent: int, row_limit: int) -> torch.Tensor:
    """The reference's stitch of a grid of raw tile outputs (modified in place, as the reference does)."""
    out_rows = []
    for i, row in enumerate(grid):
        kept = []
        for j, tile in enumerate(row):
            if i > 0:
                tile = blend_v(grid[i - 1][j], tile, extent)
            if j > 0:
                tile = blend_h(row[j - 1], tile, extent)
            kept.append(tile[:, :, :row_limit, :row_limit])
        out_rows.append(torch.cat(kept, dim=3))
    return torch.cat(out_rows, dim=2)


def _weights(e: int, n: int, dtype, device):
    """fl32 weights (1 - t/e, t/e) of offsets t < n (zero-extent slots unused), as Python doubles rounded to the tensor's
    scalar type."""
    t = torch.arange(n, dtype=torch.float64)
    r = t / max(e, 1)
    return (1 - r).to(torch.float32), r.to(torch.float32)


def _blend(a, b, wa, wb):
    """fl(fl(a wa) + fl(b wb)) in a's dtype, the products and the sum each computed in fp32 and rounded (torch's op math
    for fp16 with a Python-scalar weight)."""
    dt = a.dtype
    pa = (a.float() * wa).to(dt)
    pb = (b.float() * wb).to(dt)
    return (pa.float() + pb.float()).to(dt)


def stitch_closed_form(grid: List[List[torch.Tensor]], extent: int, row_limit: int) -> torch.Tensor:
    """Every output pixel from the raw tiles of (i, j), (i-1, j), (i, j-1), (i-1, j-1) alone (vae_tiles.cu's form)."""
    L, E = row_limit, extent
    hs = [row[0].shape[2] for row in grid]
    ws = [t.shape[3] for t in grid[0]]
    out_rows = []
    for i, row in enumerate(grid):
        kept = []
        for j, C in enumerate(row):
            h, w = min(hs[i], L), min(ws[j], L)
            v = C[:, :, :h, :w].clone()
            ev = min(hs[i - 1], hs[i], E) if i > 0 else 0
            eh = min(ws[j - 1], ws[j], E) if j > 0 else 0
            wav, wbv = _weights(ev, h, v.dtype, v.device)
            wah, wbh = _weights(eh, w, v.dtype, v.device)
            wav, wbv = wav.view(-1, 1), wbv.view(-1, 1)
            yv, xh = torch.arange(h).view(-1, 1) < ev, torch.arange(w).view(1, -1) < eh
            if ev:
                U = grid[i - 1][j][:, :, hs[i - 1] - ev:hs[i - 1] - ev + h, :w]
                U = torch.nn.functional.pad(U, (0, 0, 0, h - U.shape[2]))
                if eh:
                    UL = grid[i - 1][j - 1][:, :, hs[i - 1] - ev:hs[i - 1] - ev + h, ws[j - 1] - eh:ws[j - 1] - eh + w]
                    UL = torch.nn.functional.pad(UL, (0, w - UL.shape[3], 0, h - UL.shape[2]))
                    U = torch.where(xh, _blend(UL, U, wah, wbh), U)
                v = torch.where(yv, _blend(U, v, wav, wbv), v)
            if eh:
                Lt = grid[i][j - 1][:, :, :h, ws[j - 1] - eh:ws[j - 1] - eh + w]
                Lt = torch.nn.functional.pad(Lt, (0, w - Lt.shape[3]))
                if ev:
                    UL = grid[i - 1][j - 1][:, :, hs[i - 1] - ev:hs[i - 1] - ev + h, ws[j - 1] - eh:ws[j - 1] - eh + w]
                    UL = torch.nn.functional.pad(UL, (0, w - UL.shape[3], 0, h - UL.shape[2]))
                    Lt = torch.where(yv, _blend(UL, Lt, wav, wbv), Lt)
                v = torch.where(xh, _blend(Lt, v, wah, wbh), v)
            kept.append(v)
        out_rows.append(torch.cat(kept, dim=3))
    return torch.cat(out_rows, dim=2)


def blend_case_tiles(case) -> List[torch.Tensor]:
    """The tiles the stub of a tests/golden/vae_tiled_blend.pt case handed out, in call order: torch.randn of every recorded
    shape from the case's seed, rounded to its dtype (oracle/make_golden_vae_tiled.py draws them the same way)."""
    gen = torch.Generator().manual_seed(case["tile_seed"])
    dtype = getattr(torch, case["dtype"])
    return [torch.randn(*shape, generator=gen).to(dtype) for shape in case["tile_shapes"]]


def tile_grid(x: torch.Tensor, tile: int, overlap: int, run) -> List[List[torch.Tensor]]:
    """run() of every tile x[:, :, i : i + tile, j : j + tile], i and j stepping by overlap (autoencoder_kl.py:390-398)."""
    return [[run(x[:, :, i:i + tile, j:j + tile]) for j in range(0, x.shape[3], overlap)]
            for i in range(0, x.shape[2], overlap)]


@torch.no_grad()
def tiled_decode(dec_oracle, z: torch.Tensor, tile_sample_min_size: int, tile_latent_min_size: int,
                 tile_overlap_factor: float = 0.25) -> torch.Tensor:
    """AutoencoderKL.tiled_decode (:420-466) with VAEDecoderOracle.decode as post_quant_conv + decoder."""
    overlap = int(tile_latent_min_size * (1 - tile_overlap_factor))
    extent = int(tile_sample_min_size * tile_overlap_factor)
    grid = tile_grid(z, tile_latent_min_size, overlap, dec_oracle.decode)
    return stitch(grid, extent, tile_sample_min_size - extent)


@torch.no_grad()
def tiled_encode(enc_oracle, x: torch.Tensor, tile_sample_min_size: int, tile_latent_min_size: int,
                 tile_overlap_factor: float = 0.25) -> torch.Tensor:
    """AutoencoderKL.tiled_encode (:366-418) with VAEEncoderOracle.moments as encoder + quant_conv: the moments."""
    overlap = int(tile_sample_min_size * (1 - tile_overlap_factor))
    extent = int(tile_latent_min_size * tile_overlap_factor)
    grid = tile_grid(x, tile_sample_min_size, overlap, enc_oracle.moments)
    return stitch(grid, extent, tile_latent_min_size - extent)
