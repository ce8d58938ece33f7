"""Tile plan of the engine's tiled VAE: diffusers `AutoencoderKL.tiled_decode` / `tiled_encode` (models/autoencoder_kl.py:
366-466), the geometry only. Pure Python, no device.

The reference splits a frame into tiles that start every `overlap_size` input pixels along each axis and are at most
`tile` input pixels long (:385-394, :434-444), runs the VAE half on each, blends every tile with its upper and left
neighbours over `blend_extent` output pixels and keeps its first `row_limit` output rows and columns. A tile's size
depends only on where it starts, so tiles of equal size form contiguous runs (classes) along each axis, and a shape
group (row class x column class) can be cut out of a batch of frames with two `unfold`s and one copy.

`plan_decode` / `plan_encode` return that geometry, or raise ValueError naming the first condition the engine cannot
meet: a tile the VAE kernels cannot run (latent area not a multiple of 64 or above 8192, image side not a multiple of
the downsampling factor), or tile attributes whose stitch the blend kernel cannot reproduce exactly (DESIGN.md 4.9).
MuseV's sizes (pixel sides multiples of 64) with the default attributes always pass.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Tuple

MAX_CLASSES = 4                    # MVB_VAE_TILE_CLASSES of include/musev_b200.h
MAX_LATENT_PIXELS = 8192           # the VAE's mid-block attention holds one frame's scores


@dataclass(frozen=True)
class TileClass:
    first: int                     # index of its first tile along the axis
    count: int
    size_in: int                   # tile extent in input pixels (latent for a decode, image for an encode)
    size_out: int                  # the same tile in output pixels


@dataclass(frozen=True)
class TileAxis:
    starts: Tuple[int, ...]        # input offset of every tile: range(0, n, overlap_size)
    sizes_in: Tuple[int, ...]
    sizes_out: Tuple[int, ...]
    classes: Tuple[TileClass, ...]

    def extents(self, blend_extent: int) -> Tuple[int, ...]:
        """min(previous tile, this tile, blend_extent) of every tile after the first (blend_v / blend_h, :354-364)."""
        s = self.sizes_out
        return tuple(min(s[i - 1], s[i], blend_extent) for i in range(1, len(s)))


@dataclass(frozen=True)
class TilePlan:
    rows: TileAxis
    cols: TileAxis
    overlap_size: int              # tile stride, input pixels
    tile_in: int                   # nominal tile size, input pixels
    blend_extent: int              # output pixels
    row_limit: int                 # output pixels kept per tile and axis
    out_h: int
    out_w: int

    @property
    def groups(self):
        """(row class, column class) of every shape group, row-major (the order of the blend kernel's `tiles`)."""
        return [(r, c) for r in self.rows.classes for c in self.cols.classes]

    @property
    def tiles_per_frame(self) -> int:
        return len(self.rows.starts) * len(self.cols.starts)

    def covered(self) -> int:
        """Output pixels the tiles of one frame hold (the work of tiling against one untiled frame)."""
        return sum(self.rows.sizes_out) * sum(self.cols.sizes_out)


def _axis(n: int, tile: int, overlap: int, to_out) -> TileAxis:
    starts = tuple(range(0, n, overlap))
    sizes_in = tuple(min(tile, n - s) for s in starts)     # x[..., s : s + tile] clips at the edge
    sizes_out = tuple(to_out(s) for s in sizes_in)
    classes, i = [], 0
    while i < len(starts):
        k = i
        while k + 1 < len(starts) and sizes_in[k + 1] == sizes_in[i]:
            k += 1
        classes.append(TileClass(i, k - i + 1, sizes_in[i], sizes_out[i]))
        i = k + 1
    return TileAxis(starts, sizes_in, sizes_out, tuple(classes))


def _check_blend(plan: TilePlan, what: str) -> None:
    L, E = plan.row_limit, plan.blend_extent
    for name, ax, n_out in (("row", plan.rows, plan.out_h), ("column", plan.cols, plan.out_w)):
        if len(ax.classes) > MAX_CLASSES:
            raise ValueError(f"{what}: {len(ax.classes)} tile sizes along a {name} axis; the blend kernel takes at most "
                             f"{MAX_CLASSES}")
        s = ax.sizes_out
        if any(h < L for h in s[:-1]):
            raise ValueError(f"{what}: a {name} tile other than the last is shorter than row_limit {L} (tile sizes {s}); "
                             "its crop would not tile the output")
        if sum(min(h, L) for h in s) != n_out:
            raise ValueError(f"{what}: the {name} crops add up to {sum(min(h, L) for h in s)} pixels, not the output's "
                             f"{n_out} (the tile stride {plan.overlap_size} must map to row_limit {L})")
        ev = (0,) + ax.extents(E)
        for i in range(1, len(s)):
            if s[i - 1] - ev[i] < ev[i - 1]:
                raise ValueError(f"{what}: {name} tile {i - 1} ({s[i - 1]} pixels) blends {ev[i - 1]} pixels with the tile "
                                 f"before it and {ev[i]} with the tile after it; the strips overlap, so the in-place "
                                 "blends have no closed form (needs size - extent_after >= extent_before)")


def _common(tile_sample_min_size, tile_latent_min_size, tile_overlap_factor):
    for name, v in (("tile_sample_min_size", tile_sample_min_size), ("tile_latent_min_size", tile_latent_min_size)):
        if isinstance(v, bool) or not isinstance(v, int) or v < 1:
            raise ValueError(f"{name} must be a positive int, got {v!r}")
    if not 0.0 <= float(tile_overlap_factor) < 1.0:
        raise ValueError(f"tile_overlap_factor must be in [0, 1), got {tile_overlap_factor!r}")


def plan_tiles(n_h: int, n_w: int, tile: int, overlap_size: int, to_out, blend_extent: int, row_limit: int, out_h: int,
               out_w: int, what: str = "tiled VAE") -> TilePlan:
    """The tile grid of an n_h x n_w input (tiles every overlap_size pixels, at most `tile` long; `to_out` maps a tile
    size to output pixels), refused with ValueError when the blend kernel cannot stitch it exactly."""
    rows = _axis(n_h, tile, overlap_size, to_out)
    cols = _axis(n_w, tile, overlap_size, to_out)
    plan = TilePlan(rows, cols, overlap_size, tile, blend_extent, row_limit, out_h, out_w)
    _check_blend(plan, what)
    return plan


def _check_latent_tiles(sizes_h, sizes_w, what: str) -> None:
    for h in sorted(set(sizes_h)):
        for w in sorted(set(sizes_w)):
            if (h * w) % 64 or h * w > MAX_LATENT_PIXELS:
                raise ValueError(f"{what}: a {h}x{w}-latent tile: the latent area h*w must be a multiple of 64 and at most "
                                 f"{MAX_LATENT_PIXELS} (latent tile sides multiples of 8 qualify)")


def plan_decode(h: int, w: int, tile_sample_min_size: int, tile_latent_min_size: int, tile_overlap_factor: float,
                factor: int) -> TilePlan:
    """`tiled_decode` (autoencoder_kl.py:434-462) of an h x w latent; the decoder upsamples `factor`x."""
    _common(tile_sample_min_size, tile_latent_min_size, tile_overlap_factor)
    overlap_size = int(tile_latent_min_size * (1 - tile_overlap_factor))
    blend_extent = int(tile_sample_min_size * tile_overlap_factor)
    row_limit = tile_sample_min_size - blend_extent
    if overlap_size < 1:
        raise ValueError(f"tiled decode: overlap_size = int(tile_latent_min_size * (1 - tile_overlap_factor)) = "
                         f"{overlap_size}; it must be >= 1")
    plan = plan_tiles(h, w, tile_latent_min_size, overlap_size, lambda s: s * factor, blend_extent, row_limit,
                      h * factor, w * factor, "tiled decode")
    _check_latent_tiles(plan.rows.sizes_in, plan.cols.sizes_in, "tiled decode")
    return plan


def plan_encode(H: int, W: int, tile_sample_min_size: int, tile_latent_min_size: int, tile_overlap_factor: float,
                factor: int) -> TilePlan:
    """`tiled_encode` (autoencoder_kl.py:385-412) of an H x W image; the encoder downsamples `factor`x."""
    _common(tile_sample_min_size, tile_latent_min_size, tile_overlap_factor)
    overlap_size = int(tile_sample_min_size * (1 - tile_overlap_factor))
    blend_extent = int(tile_latent_min_size * tile_overlap_factor)
    row_limit = tile_latent_min_size - blend_extent
    if overlap_size < 1:
        raise ValueError(f"tiled encode: overlap_size = int(tile_sample_min_size * (1 - tile_overlap_factor)) = "
                         f"{overlap_size}; it must be >= 1")
    if H % factor or W % factor:
        raise ValueError(f"image size {H}x{W} must be a multiple of {factor} (the encoder downsamples {factor}x)")
    for s in {min(tile_sample_min_size, n - s) for n in (H, W) for s in range(0, n, overlap_size)}:
        if s % factor:
            raise ValueError(f"tiled encode: a {s}-pixel tile side is not a multiple of {factor} (tile_sample_min_size "
                             f"{tile_sample_min_size}, overlap_size {overlap_size})")
    plan = plan_tiles(H, W, tile_sample_min_size, overlap_size, lambda s: s // factor, blend_extent, row_limit,
                      H // factor, W // factor, "tiled encode")
    _check_latent_tiles(plan.rows.sizes_out, plan.cols.sizes_out, "tiled encode")
    return plan
