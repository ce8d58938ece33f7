"""CPU tests of histogram matching (`need_hist_match`): the numpy oracle against the fixture of the unmodified MMCM wrapper
and against hand-derived answers, the drop-in's argument checks, and the C entry point's surface and refusals. No
call here reaches a kernel launch."""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from oracle import hist_match_oracle as H
from oracle import ref_shim


def _golden():
    return torch.load(os.path.join(GOLDEN, "hist_match.pt"))


def _as_predictor(fn, video):
    """out_videos[:, :, 1:] = fn(out_videos[:, :, 1:], out_videos[:, :, :1], value=255.0) on a float32 array."""
    out = video.copy()
    out[:, :, 1:, :, :] = fn(out[:, :, 1:, :, :], out[:, :, :1, :, :], value=255.0)
    return out


def test_oracle_equals_fixture_bitwise():
    g = _golden()
    out = _as_predictor(H.hist_match_video_bcthw, g["video"].numpy())
    assert out.dtype == np.float32
    assert np.array_equal(out.view(np.uint32), g["out"].numpy().view(np.uint32))


@pytest.mark.skipif(not ref_shim.available(), reason="reference tree not present")
def test_restated_wrapper_equals_mmcm_wrapper():
    ref = H.mmcm_hist_match_video_bcthw()
    rng = np.random.default_rng(1)
    video = rng.random((2, 3, 5, 13, 17), dtype=np.float32)
    target = rng.random((2, 3, 1, 9, 6), dtype=np.float32)
    a, b = ref(video, target, value=255.0), H.hist_match_video_bcthw(video, target)
    assert a.dtype == b.dtype == np.float64 and np.array_equal(a, b)


def _q(x):
    return (np.float32(x) * 255.0).astype(np.uint8)


def _match(src, tmpl):
    """one-channel frames [h, w] through the video wrapper"""
    return H.hist_match_video_f32(src[None, None, None], tmpl[None, None, None])[0, 0, 0]


def test_constant_source_maps_to_template_max():
    rng = np.random.default_rng(2)
    tmpl = rng.random((9, 7), dtype=np.float32)
    out = _match(np.full((5, 6), 0.3, np.float32), tmpl)
    assert np.all(out == np.float32(_q(tmpl).max() / 255.0))


def test_source_equal_to_template_quantises():
    rng = np.random.default_rng(3)
    x = rng.random((11, 13), dtype=np.float32)
    x[0, :8] = (np.arange(8) * 30 / np.float32(255)).astype(np.float32)        # values at k / 255
    out = _match(x, x)
    assert np.array_equal(out, (np.floor(x * np.float32(255.0)) / 255.0).astype(np.float32))


def test_quantiles_below_and_between_template_quantiles():
    tmpl = np.array([[100] * 4 + [200] * 4], np.float32) / np.float32(255)      # quantiles 0.5 @ 100, 1.0 @ 200
    src = np.array([[5] * 2 + [60] * 4 + [250] * 2], np.float32) / np.float32(255)   # 0.25, 0.75, 1.0
    out = _match(src, tmpl)
    q = _q(src)
    exp = np.where(q == _q(5 / 255), 100.0, np.where(q == _q(60 / 255), 150.0, 200.0)) / 255.0
    assert np.array_equal(out, exp.astype(np.float32))


def test_quantisation_boundaries_at_k_over_255():
    """fl32(k / 255) quantises to k for every k; the float one ulp below it to k - 1 (truncation of fl32(x * 255))."""
    k = np.arange(256)
    x = (k / np.float32(255)).astype(np.float32)
    assert np.array_equal(_q(x), k)
    assert np.array_equal(_q(np.nextafter(x[1:], np.float32(0))), k[1:] - 1)


def test_drop_in_refuses_what_would_quantise_differently():
    from musev_b200.correct_color import hist_match_video_bcthw
    v = np.zeros((1, 3, 2, 4, 4), np.float32)
    t = np.zeros((1, 3, 1, 4, 4), np.float32)
    with pytest.raises(ValueError, match="255"):
        hist_match_video_bcthw(v, t, value=1.0)
    with pytest.raises(TypeError, match="float32"):
        hist_match_video_bcthw(v.astype(np.float64), t)
    with pytest.raises(TypeError, match="float32"):
        hist_match_video_bcthw(v, t.astype(np.float64))
    with pytest.raises(TypeError, match="CUDA"):
        hist_match_video_bcthw(torch.from_numpy(v), torch.from_numpy(t))
    with pytest.raises(TypeError, match="both"):
        hist_match_video_bcthw(v, torch.from_numpy(t))


def _proto_nparams(name):
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "musev_b200.h")).read(), flags=re.S)
    m = re.search(r"\b" + name + r"\s*\(([^()]*)\)\s*;", src)
    return m.group(1).count(",") + 1


def test_symbols_and_argtypes(built_lib):
    from musev_b200 import _capi
    lib = _capi.lib()
    assert lib.mvb_version() == 9
    for name, n in (("mvb_op_hist_match", 21), ("mvb_op_hist_match_workspace_bytes", 7)):
        assert _proto_nparams(name) == n
        assert len(getattr(lib, name).argtypes) == n


def test_lut_kernel_has_no_dfma(built_lib):
    """np.interp's slope * (x - xp) + fp is a separate multiply and add: the table kernel must not contract it."""
    sass = subprocess.run(["cuobjdump", "-sass", built_lib], capture_output=True, text=True, check=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)
    lut = [f for f in funcs if f.split("\n", 1)[0].find("hist_match_lut_kernel") >= 0]
    assert len(lut) == 1
    assert "DMUL" in lut[0] and "DADD" in lut[0]
    assert "DFMA" not in lut[0]
    for k in ("hist_match_count_kernel", "hist_match_apply_kernel"):
        assert any(f.split("\n", 1)[0].find(k) >= 0 for f in funcs), k


def test_workspace_query_and_refusals(built_lib):
    """Every call below is refused by argument checks before anything reaches the device."""
    from musev_b200 import _capi
    lib = _capi.lib()
    assert lib.mvb_op_hist_match_workspace_bytes(1, 3, 16, 512, 512, 512, 512) > 0
    assert lib.mvb_op_hist_match_workspace_bytes(1, 3, 0, 512, 512, 512, 512) < 0
    assert lib.mvb_op_hist_match_workspace_bytes(1, 3, 1, 65536, 65536, 8, 8) < 0
    hw = 8 * 8
    need = lib.mvb_op_hist_match_workspace_bytes(2, 3, 4, 8, 8, 8, 8)
    v, t, o, ws = 1 << 32, 1 << 33, 1 << 34, 1 << 35          # never dereferenced: every call is refused
    ok = dict(video=v, B=2, C=3, F=4, H=8, W=8, sb=12 * hw, sc=4 * hw, sf=hw, target=t, Ht=8, Wt=8, tsb=3 * hw, tsc=hw,
              out=o, osb=12 * hw, osc=4 * hw, osf=hw, ws=ws, ws_bytes=need)

    def call(**kw):
        a = dict(ok, **kw)
        return lib.mvb_op_hist_match(*a.values(), None), lib.mvb_last_error().decode()

    for kw, msg in ((dict(video=None), "null"), (dict(ws=None), "null"), (dict(F=0), "sizes"), (dict(Wt=0), "sizes"),
                    (dict(sf=-hw), "negative"), (dict(osf=0), "overlap"), (dict(osc=2 * hw), "overlap"),
                    (dict(out=v + 4 * hw), "overlaps video"), (dict(out=v, osb=24 * hw), "overlaps video"),
                    (dict(ws_bytes=need - 1), "workspace")):
        rc, err = call(**kw)
        assert rc == -1 and msg in err, (kw, rc, err)
