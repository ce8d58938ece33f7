"""CPU tests of the tiled VAE: the tile plan (musev_b200.vae_tiling) against the reference's loop ranges, crops and blend
extents, for the blend fixtures' geometries and every task size of MuseV's configs/tasks/example.yaml; the refusal rules;
the closed form of the in-place stitch (oracle/vae_tiled_oracle.py, the blend kernel's form) against the fixture of the
unmodified diffusers `tiled_decode` / `tiled_encode` (tests/golden/vae_tiled_blend.pt); the C-ABI struct of the blend entry."""
import ctypes
import os
import random
import re
import subprocess

import pytest
import torch

from conftest import GOLDEN, ROOT
from musev_b200 import vae_tiling
from oracle import vae_tiled_oracle as O

# (name, height, width, img_length_ratio) of MuseV's configs/tasks/example.yaml; text2video.py:1054-1055 sizes them as
# int(side * ratio // 64 * 64)
EXAMPLE_TASKS = [
    ("yongen", 1308, 736, 0.957), ("jinkesi2", 714, 563, 1.25), ("seaside4", 317, 564, 2.221),
    ("seaside_girl", 736, 736, 0.957), ("boy_play_guitar", 846, 564, 1.248), ("girl_play_guitar2", 1002, 564, 1.248),
    ("boy_play_guitar2", 630, 420, 1.676), ("girl_play_guitar4", 846, 564, 1.248), ("dufu", 500, 471, 1.495),
    ("Mona_Lisa.", 894, 600, 1.173), ("Portrait-of-Dr.-Gachet", 985, 800, 0.88),
    ("Self-Portrait-with-Cropped-Hair", 565, 848, 1.246), ("The-Laughing-Cavalier", 1462, 1200, 0.587),
    ("waterfall4", 846, 564, 1.248), ("river", 736, 736, 0.957), ("seaside2", 1313, 736, 0.957),
    ("dance1", 960, 512, 1.0), ("dance2", 960, 512, 1.0), ("duffy", 1280, 704, 1.0),
]
TASK_SIZES = sorted({(int(h * r // 64 * 64), int(w * r // 64 * 64)) for _, h, w, r in EXAMPLE_TASKS})


def _blend_cases():
    return torch.load(os.path.join(GOLDEN, "vae_tiled_blend.pt"))["cases"]


def _reference_grid(n_h, n_w, tile, overlap, scale):
    """The reference's tile loops (autoencoder_kl.py:390-394, 441-444), run on a shape-only tensor: output tile shapes."""
    x = torch.empty(1, 1, n_h, n_w)
    return O.tile_grid(x, tile, overlap, lambda t: (int(t.shape[2] * scale), int(t.shape[3] * scale)))


def _check_plan_against_reference(plan, grid, extent, row_limit, out_h, out_w):
    assert plan.blend_extent == extent and plan.row_limit == row_limit
    assert (plan.out_h, plan.out_w) == (out_h, out_w)
    assert plan.rows.sizes_out == tuple(row[0][0] for row in grid)
    assert plan.cols.sizes_out == tuple(t[1] for t in grid[0])
    # the reference's output is the concatenation of the crops: exactly the frame
    assert sum(min(h, row_limit) for h in plan.rows.sizes_out) == out_h
    assert sum(min(w, row_limit) for w in plan.cols.sizes_out) == out_w
    # blend extents min(a, b, E) of blend_v / blend_h
    assert plan.rows.extents(extent) == tuple(min(grid[i - 1][0][0], grid[i][0][0], extent) for i in range(1, len(grid)))
    # classes: contiguous runs of equal size, covering every tile once
    for ax in (plan.rows, plan.cols):
        idx = [c.first + k for c in ax.classes for k in range(c.count)]
        assert idx == list(range(len(ax.starts)))
        assert all(ax.sizes_in[c.first + k] == c.size_in for c in ax.classes for k in range(c.count))


@pytest.mark.parametrize("H,W", TASK_SIZES)
def test_plan_matches_reference_loops_at_task_sizes(H, W):
    assert len(EXAMPLE_TASKS) == 19
    h, w = H // 8, W // 8
    dec = vae_tiling.plan_decode(h, w, 512, 64, 0.25, 8)
    _check_plan_against_reference(dec, _reference_grid(h, w, 64, 48, 8), 128, 384, H, W)
    enc = vae_tiling.plan_encode(H, W, 512, 64, 0.25, 8)
    _check_plan_against_reference(enc, _reference_grid(H, W, 512, 384, 1 / 8), 16, 48, h, w)
    for p in (dec, enc):
        assert len(p.groups) <= 16 and p.tiles_per_frame == len(p.rows.starts) * len(p.cols.starts)


def test_plan_of_the_1216x704_decode():
    """The issue's worked example: 8 tiles per frame in 6 shapes, 192 x 104 latents covered (1.49x the frame)."""
    p = vae_tiling.plan_decode(152, 88, 512, 64, 0.25, 8)
    assert p.rows.sizes_in == (64, 64, 56, 8) and p.cols.sizes_in == (64, 40)
    assert p.tiles_per_frame == 8 and len(p.groups) == 6
    assert p.covered() == 192 * 104 * 64


def fixture_plan(c):
    """The blend plan of a blend-fixture case (the stubs' tiles are not VAE-runnable, so only the stitch is planned)."""
    f, tof = c["factor"], c["tile_overlap_factor"]
    tsm, tlm = c["tile_sample_min_size"], c["tile_latent_min_size"]
    if c["kind"] == "decode":
        E = int(tsm * tof)
        return vae_tiling.plan_tiles(c["H"], c["W"], tlm, int(tlm * (1 - tof)), lambda s: s * f, E, tsm - E,
                                     c["H"] * f, c["W"] * f)
    E = int(tlm * tof)
    return vae_tiling.plan_tiles(c["H"], c["W"], tsm, int(tsm * (1 - tof)), lambda s: s // f, E, tlm - E,
                                 c["H"] // f, c["W"] // f)


@pytest.mark.parametrize("k", range(9))
def test_plan_matches_blend_fixture_geometries(k):
    c = _blend_cases()[k]
    p = fixture_plan(c)
    scale = c["factor"] if c["kind"] == "decode" else 1 / c["factor"]
    grid = _reference_grid(c["H"], c["W"], p.tile_in, p.overlap_size, scale)
    _check_plan_against_reference(p, grid, p.blend_extent, p.row_limit, c["out"].shape[2], c["out"].shape[3])
    assert [tuple(shape[2:]) for shape in c["tile_shapes"]] == [s for row in grid for s in row]


@pytest.mark.parametrize("k", range(9))
def test_closed_form_equals_reference_stitch(k):
    """The per-pixel closed form (and the restated loop) reproduce the unmodified reference's output bit for bit, in
    fp32 and fp16."""
    c = _blend_cases()[k]
    p = fixture_plan(c)
    nc = len(p.cols.starts)
    tiles = O.blend_case_tiles(c)
    grid = [tiles[i:i + nc] for i in range(0, len(tiles), nc)]
    E, L = p.blend_extent, p.row_limit
    closed = O.stitch_closed_form(grid, E, L)
    assert closed.dtype == c["out"].dtype and torch.equal(closed, c["out"])
    assert torch.equal(O.stitch([[t.clone() for t in row] for row in grid], E, L), c["out"])


def test_closed_form_on_random_accepted_geometries():
    """Any geometry the plan accepts stitches by the closed form exactly as by the in-place loop."""
    rng = random.Random(5)
    accepted = 0
    for _ in range(80):
        tile = rng.choice([8, 12, 16, 24])
        tof = rng.choice([0.0, 0.125, 0.25, 0.3])
        n_h, n_w = rng.randint(1, 60), rng.randint(1, 60)
        ov, E = int(tile * (1 - tof)), int(tile * tof)
        try:
            p = vae_tiling.plan_tiles(n_h, n_w, tile, ov, lambda s: s, E, tile - E, n_h, n_w)
        except ValueError:
            continue
        accepted += 1
        dtype = rng.choice([torch.float32, torch.float16])
        gen = torch.Generator().manual_seed(rng.randint(0, 1 << 30))
        grid = [[torch.randn(1, 2, h, w, generator=gen).to(dtype) for w in p.cols.sizes_out] for h in p.rows.sizes_out]
        ref = O.stitch([[t.clone() for t in row] for row in grid], p.blend_extent, p.row_limit)
        assert torch.equal(O.stitch_closed_form(grid, p.blend_extent, p.row_limit), ref), (n_h, n_w, tile, tof)
    assert accepted >= 40, accepted


def test_refusals_name_the_condition():
    # latent tiles the engine cannot run
    with pytest.raises(ValueError, match="multiple of 64"):
        vae_tiling.plan_decode(100, 60, 512, 64, 0.25, 8)        # 4-latent row sliver x 12: area 48
    with pytest.raises(ValueError, match="multiple of 8"):
        vae_tiling.plan_encode(1004, 704, 512, 64, 0.25, 8)       # image side not a multiple of 8
    with pytest.raises(ValueError, match="not a multiple of 8"):
        vae_tiling.plan_encode(1024, 704, 500, 64, 0.25, 8)       # tile side 500
    with pytest.raises(ValueError, match="8192"):
        vae_tiling.plan_decode(200, 200, 1024, 128, 0.25, 8)      # 128 x 128 latent tiles
    # attributes the blend cannot reproduce
    with pytest.raises(ValueError, match="crops add up"):
        vae_tiling.plan_decode(128, 128, 512, 64, 0.3, 8)         # stride 44 latents = 352 px, row_limit 359
    with pytest.raises(ValueError, match="overlap_size"):
        vae_tiling.plan_decode(152, 88, 512, 1, 0.25, 8)
    with pytest.raises(ValueError, match="strips overlap"):
        vae_tiling.plan_decode(20, 8, 8, 8, 0.625, 1)             # stride 3, extent 5: an 8-pixel tile blends 5 + 5
    with pytest.raises(ValueError, match="at most 4"):
        vae_tiling.plan_decode(64, 8, 16, 16, 0.875, 1)           # stride 2: sizes 16, 14, ..., 2 along the rows
    with pytest.raises(ValueError, match="tile_overlap_factor"):
        vae_tiling.plan_decode(152, 88, 512, 64, 1.0, 8)
    with pytest.raises(ValueError, match="positive int"):
        vae_tiling.plan_decode(152, 88, (512, 512), 64, 0.25, 8)
    # the closed form's condition is what the refusal guards: where the plan refuses, the closed form can differ
    gen = torch.Generator().manual_seed(0)
    grid = [[torch.randn(1, 1, h, 8, generator=gen)] for h in (10, 5, 5, 5, 5, 5, 5, 5)]
    ref = O.stitch([[t.clone() for t in row] for row in grid], 4, 5)
    assert not torch.equal(O.stitch_closed_form(grid, 4, 5), ref)


def test_blend_args_struct_matches_ctypes_mirror(tmp_path):
    from musev_b200 import _capi
    cls = _capi.MvbVaeTileBlendArgs
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "musev_b200.h"', "int main(void) {",
             '  printf(". %zu\\n", sizeof(mvb_vae_tile_blend_args));',
             '  printf("K %d\\n", MVB_VAE_TILE_CLASSES);']
    lines += [f'  printf("{f} %zu\\n", offsetof(mvb_vae_tile_blend_args, {f}));' for f, *_ in cls._fields_]
    lines += ["  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    r = subprocess.run(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.strip().splitlines():
        name, value = line.split()
        expect = {".": ctypes.sizeof(cls), "K": _capi.VAE_TILE_CLASSES}.get(name)
        if expect is None:
            expect = getattr(cls, name).offset
        assert int(value) == expect, (name, value, expect)
    assert vae_tiling.MAX_CLASSES == _capi.VAE_TILE_CLASSES


def test_blend_entry_refuses_before_launch(built_lib):
    """Bad arguments are refused by the host-side checks (nothing reaches the device; the pointers are never read)."""
    from musev_b200 import _capi
    l = _capi.lib()
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "musev_b200.h")).read(), flags=re.S)
    assert re.search(r"\bmvb_op_vae_tile_blend\s*\(([^()]*)\)", src).group(1).count(",") + 1 == 2
    assert len(l.mvb_op_vae_tile_blend.argtypes) == 2
    p = vae_tiling.plan_decode(152, 88, 512, 64, 0.25, 8)

    def args(**kw):
        a = _capi.MvbVaeTileBlendArgs()
        for k in range(16):
            a.tiles[k] = 1 << 32
        a.tiles_is_f32, a.N, a.C = 1, 1, 3
        a.n_row_classes, a.n_col_classes = len(p.rows.classes), len(p.cols.classes)
        for k, c in enumerate(p.rows.classes):
            a.row_count[k], a.row_size[k] = c.count, c.size_out
        for k, c in enumerate(p.cols.classes):
            a.col_count[k], a.col_size[k] = c.count, c.size_out
        a.extent, a.row_limit, a.H, a.W, a.mode, a.out, a.out_is_f32 = 128, 384, 1216, 704, 0, 1 << 33, 1
        for k, v in kw.items():
            if isinstance(v, tuple):
                getattr(a, k)[v[0]] = v[1]
            else:
                setattr(a, k, v)
        return a

    n0 = _capi.launch_count(-1)
    for kw, msg in ((dict(out=None), "null"), (dict(tiles=(5, None)), "null"), (dict(N=0), ">= 1"),
                    (dict(mode=3), "mode"), (dict(mode=2), "even"), (dict(n_row_classes=5), "classes"),
                    (dict(H=1215), "add up"), (dict(row_size=(2, 100)), "add up"),
                    (dict(row_limit=500), "shorter than row_limit"), (dict(extent=300), "overlap")):
        rc = l.mvb_op_vae_tile_blend(ctypes.byref(args(**kw)), None)
        err = l.mvb_last_error().decode()
        assert rc == -1 and msg in err, (kw, rc, err)
    assert _capi.launch_count(-1) == n0
