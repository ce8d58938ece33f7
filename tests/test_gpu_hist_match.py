"""Histogram matching on the engine (`musev_b200.ops.hist_match`, `musev_b200.correct_color`) against the numpy oracle
(oracle/hist_match_oracle.py) and the fixture of the unmodified MMCM wrapper (tests/golden/hist_match.pt): every output
bit equal to what the predictor stores, for the shapes, strides and value patterns the kernels treat differently."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle.hist_match_oracle import hist_match_video_f32

pytestmark = pytest.mark.gpu
dev = "cuda"


def _noise(rng, shape):
    return np.clip(rng.normal(0.45, 0.22, shape), 0, 1).astype(np.float32)


def _engine(video, target, out=None):
    from musev_b200 import ops
    return ops.hist_match(video, target, out=out)


def _check(video, target):
    got = _engine(torch.from_numpy(video).to(dev), torch.from_numpy(target).to(dev)).cpu().numpy()
    exp = hist_match_video_f32(video, target)
    bad = got.view(np.uint32) != exp.view(np.uint32)
    assert not bad.any(), (int(bad.sum()), got[bad][:5], exp[bad][:5])


@pytest.mark.parametrize("B,F,H,W,Ht,Wt", [
    (1, 1, 512, 512, 512, 512),
    (2, 16, 320, 576, 512, 512),       # template larger than the frames
    (1, 127, 512, 512, 512, 512),
    (2, 16, 37, 53, 29, 41),           # odd planes: unaligned heads and tails
    (2, 127, 37, 53, 37, 53),
    (1, 16, 512, 512, 37, 53),         # template smaller than the frames
])
def test_seeded_noise(built_lib, B, F, H, W, Ht, Wt):
    rng = np.random.default_rng(B * 1000 + F)
    _check(_noise(rng, (B, 3, F, H, W)), _noise(rng, (B, 3, 1, Ht, Wt)))


@pytest.mark.parametrize("levels", [1, 2, 3])
@pytest.mark.parametrize("H,W", [(37, 53), (320, 576)])
def test_few_distinct_values(built_lib, levels, H, W):
    """1-3 distinct values in the frames, in the template, and in both (flat images: one bin takes most pixels)."""
    rng = np.random.default_rng(levels)
    vals = np.array([0.2, 0.61, 0.97], np.float32)[:levels]
    flat = rng.choice(vals, size=(2, 3, 4, H, W)).astype(np.float32)
    flat_t = rng.choice(vals[::-1] * np.float32(0.9), size=(2, 3, 1, H, W)).astype(np.float32)
    _check(flat, _noise(rng, (2, 3, 1, H, W)))
    _check(_noise(rng, (2, 3, 4, H, W)), flat_t)
    _check(flat, flat_t)


def test_all_zero_and_all_one_frames(built_lib):
    rng = np.random.default_rng(9)
    v = _noise(rng, (2, 3, 6, 64, 96))
    v[:, :, 0] = 0.0
    v[:, :, 1] = 1.0
    t = _noise(rng, (2, 3, 1, 64, 96))
    _check(v, t)
    _check(v, np.zeros_like(t))
    _check(v, np.ones_like(t))


def test_values_at_k_over_255(built_lib):
    """fl32(k / 255) quantises to k, the float one ulp below to k - 1: both in frames and template."""
    rng = np.random.default_rng(11)
    k = rng.integers(0, 256, (2, 3, 8, 61, 67))
    v = (k / np.float32(255)).astype(np.float32)
    below = rng.random(v.shape) < 0.5
    v[below] = np.nextafter(v[below], np.float32(0))
    t = (rng.integers(30, 220, (2, 3, 1, 40, 40)) / np.float32(255)).astype(np.float32)
    _check(v, t)


def test_fixture_of_the_unmodified_wrapper(built_lib):
    g = torch.load(os.path.join(GOLDEN, "hist_match.pt"))
    video = g["video"].to(dev)
    _engine(video[:, :, 1:], video[:, :, :1], out=video[:, :, 1:])
    assert torch.equal(video.cpu().view(torch.int32), g["out"].view(torch.int32))


def test_narrow_vae_decode_output(built_lib):
    """The route the engine's text2video takes: decode_latents, then the frames after the first matched to it in place."""
    from musev_b200.schema import VAEConfig
    from musev_b200.synth import make_state_dict
    from musev_b200.vae import AutoencoderKLDecoder
    cfg = VAEConfig(block_out_channels=(64, 64, 128, 128))
    vae = AutoencoderKLDecoder(cfg, device=dev, dtype=torch.float32, frames_per_call=4)
    vae.load_state_dict({k: v.half() for k, v in make_state_dict(cfg, seed=3).items()})
    lat = torch.randn(2, 4, 5, 16, 16, generator=torch.Generator().manual_seed(5)) * 0.18215
    video = vae.decode_latents(lat.to(dev))                                   # [2, 3, 5, 128, 128] in [0, 1]
    host = video.cpu().numpy()
    exp = host.copy()
    exp[:, :, 1:] = hist_match_video_f32(host[:, :, 1:], host[:, :, :1])
    _engine(video[:, :, 1:], video[:, :, :1], out=video[:, :, 1:])
    assert np.array_equal(video.cpu().numpy().view(np.uint32), exp.view(np.uint32))


def test_in_place_equals_out_of_place_on_a_frame_slice(built_lib):
    rng = np.random.default_rng(13)
    for H, W in ((37, 53), (64, 64)):
        full = torch.from_numpy(_noise(rng, (2, 3, 9, H, W))).to(dev)
        src, tmpl = full[:, :, 1:], full[:, :, :1]
        assert not src.is_contiguous()
        fresh = _engine(src, tmpl)
        into = torch.full_like(src, float("nan"))
        _engine(src, tmpl, out=into)
        _engine(src, tmpl, out=src)
        assert torch.equal(fresh, into) and torch.equal(fresh.view(torch.int32), src.view(torch.int32))
        assert torch.equal(full[:, :, 1:].view(torch.int32), fresh.view(torch.int32))


def test_batch_items_are_independent(built_lib):
    rng = np.random.default_rng(17)
    v = torch.from_numpy(_noise(rng, (2, 3, 5, 45, 70))).to(dev)
    t = torch.from_numpy(_noise(rng, (2, 3, 1, 45, 70))).to(dev)
    a = _engine(v, t)
    v2, t2 = v.clone(), t.clone()
    v2[1] = torch.rand_like(v2[1])
    t2[1] = 1.0 - t2[1]
    b = _engine(v2, t2)
    assert torch.equal(a[0].view(torch.int32), b[0].view(torch.int32))
    assert not torch.equal(a[1], b[1])


def test_numpy_drop_in_as_the_predictor_calls_it(built_lib):
    from musev_b200.correct_color import hist_match_video_bcthw
    rng = np.random.default_rng(19)
    out_videos = _noise(rng, (1, 3, 17, 96, 128))
    exp = out_videos.copy()
    exp[:, :, 1:, :, :] = hist_match_video_f32(exp[:, :, 1:, :, :], exp[:, :, :1, :, :])
    out_videos[:, :, 1:, :, :] = hist_match_video_bcthw(out_videos[:, :, 1:, :, :], out_videos[:, :, :1, :, :], value=255.0)
    assert np.array_equal(out_videos.view(np.uint32), exp.view(np.uint32))
    dev_videos = torch.from_numpy(_noise(rng, (1, 3, 5, 40, 40))).to(dev)
    got = hist_match_video_bcthw(dev_videos[:, :, 1:], dev_videos[:, :, :1])
    assert got.is_cuda and got.dtype == torch.float32
    host = dev_videos.cpu().numpy()
    assert np.array_equal(got.cpu().numpy(), hist_match_video_f32(host[:, :, 1:], host[:, :, :1]))


def test_launch_count_does_not_grow_with_frames(built_lib):
    from musev_b200 import _capi
    rng = np.random.default_rng(23)
    t = torch.from_numpy(_noise(rng, (1, 3, 1, 64, 64))).to(dev)
    counts = []
    for F in (1, 127):
        v = torch.from_numpy(_noise(rng, (1, 3, F, 64, 64))).to(dev)
        n0 = _capi.launch_count()
        _engine(v, t)
        counts.append(_capi.launch_count() - n0)
    torch.cuda.synchronize()
    assert counts == [3, 3]
