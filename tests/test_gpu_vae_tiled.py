"""Tiled VAE on the engine (`enable_tiling`, `tiled_decode`, `tiled_encode`): the blend kernel against the stitch of the
unmodified diffusers `tiled_decode` / `tiled_encode` (tests/golden/vae_tiled_blend.pt, bit for bit in fp32 and fp16);
the narrow VAE with 256-pixel tiles against the tiled oracle and the reference samples (tests/golden/vae_tiled_narrow.pt);
SD-1.5 at 1216x704; the dispatch rules; refusals before any launch; two ranks sharing one GPU. With MVB_PARITY_LOG=<file>
set, every measured distance is appended to <file> next to its bound, one JSON object per line."""
import datetime
import json
import os
import socket

import pytest
import torch
import torch.multiprocessing as mp

from conftest import GOLDEN
from oracle.vae_tiled_oracle import blend_case_tiles
from test_vae_tiled_host import fixture_plan

pytestmark = pytest.mark.gpu
dev = "cuda"


def _record(name, err, bound):
    path = os.environ.get("MVB_PARITY_LOG")
    if path:
        try:
            with open(path, "a") as fh:
                fh.write(json.dumps({"test": name, "value": err, "bound": bound}) + "\n")
        except OSError:
            pass
    assert err < bound, (name, err, bound)


def _sd16(cfg, seed=11):
    from musev_b200.synth import make_state_dict
    return {k: v.half() for k, v in make_state_dict(cfg, seed=seed).items()}


def _pack(tiles, plan):
    """Tiles in call order (row-major, each [N, C, h, w]) -> the blend kernel's shape groups [N * nr * nc, C, h, w]."""
    nc = len(plan.cols.starts)
    groups = []
    for r in plan.rows.classes:
        row = []
        for c in plan.cols.classes:
            t = torch.stack([torch.stack([tiles[i * nc + j] for j in range(c.first, c.first + c.count)], 1)
                             for i in range(r.first, r.first + r.count)], 1)            # [N, nr, nc, C, h, w]
            row.append(t.reshape(-1, *t.shape[3:]).contiguous().to(dev))
        groups.append(row)
    return groups


@pytest.mark.parametrize("k", range(9))
def test_blend_op_matches_reference_stitch(built_lib, k):
    from musev_b200 import ops
    c = torch.load(os.path.join(GOLDEN, "vae_tiled_blend.pt"))["cases"][k]
    plan = fixture_plan(c)
    groups = _pack(blend_case_tiles(c), plan)
    ref = c["out"]
    out = torch.empty(ref.shape, dtype=ref.dtype, device=dev)
    ops.vae_tile_blend(groups, plan, out)
    assert torch.equal(out.cpu(), ref), (out.cpu().float() - ref.float()).abs().max().item()
    blended = out.float()
    if c["kind"] == "decode":         # decode_latents' post-processing after the blend, in fp32
        img = torch.empty(ref.shape, dtype=torch.float32, device=dev)
        ops.vae_tile_blend(groups, plan, img, mode=1)
        assert torch.equal(img, (blended / 2 + 0.5).clamp(0, 1))
        half = torch.empty(ref.shape, dtype=torch.float16, device=dev)
        ops.vae_tile_blend(groups, plan, half)
        assert torch.equal(half, blended.half())
    else:                             # encode_video's scaled mean in fp32, rounded once
        half_c = ref.shape[1] // 2
        lat = torch.empty((ref.shape[0], half_c, *ref.shape[2:]), dtype=torch.float32, device=dev)
        ops.vae_tile_blend(groups, plan, lat, mode=2, scale=0.18215)
        assert torch.equal(lat, 0.18215 * blended[:, :half_c])


def _narrow():
    from musev_b200.schema import VAEConfig
    g = torch.load(os.path.join(GOLDEN, "vae_tiled_narrow.pt"))
    m = g["meta"]
    cfg = VAEConfig(block_out_channels=tuple(m["block_out_channels"]), sample_size=m["sample_size"])
    return g, m, cfg, _sd16(cfg, m["weight_seed"])


def test_narrow_tiled_decode_vs_oracle_and_reference(built_lib):
    from musev_b200.vae import AutoencoderKLDecoder
    from oracle.vae_oracle import VAEDecoderOracle
    from oracle.vae_tiled_oracle import tiled_decode
    g, m, cfg, sd16 = _narrow()
    vae = AutoencoderKLDecoder(cfg, device=dev, dtype=torch.float32, frames_per_call=1)
    vae.load_state_dict(sd16)
    vae.enable_tiling()
    assert (vae.tile_sample_min_size, vae.tile_latent_min_size, vae.tile_overlap_factor) == (256, 32, 0.25)
    z = torch.randn(*m["latent_shape"], generator=torch.Generator().manual_seed(m["latent_seed"])) * m["latent_std"]
    raw = vae.decode(z.to(dev)).sample
    oracle = VAEDecoderOracle(cfg, {k: v.float() for k, v in sd16.items()}, device=dev)
    ref = tiled_decode(oracle, z, 256, 32)
    assert list(raw.shape) == m["raw_shape"] and torch.isfinite(raw).all()
    scale = max(1.0, ref.abs().max().item())
    _record("tiled_decode_narrow_vs_oracle", (raw - ref).abs().max().item(), 1.5e-2 * scale)   # measured 6.1e-3 at scale 4.2
    _record("tiled_decode_narrow_vs_reference", (raw.reshape(-1)[g["idx_raw"].to(dev)].cpu() - g["raw"]).abs().max().item(),
            2e-2 * scale)                                                         # measured 4.1e-3
    # decode_latents: the same latents as a [1, 4, f, h, w] video, post-processed after the blend
    lat = (z * cfg.scaling_factor).view(1, *z.shape).permute(0, 2, 1, 3, 4).contiguous()
    video = vae.decode_latents(lat.to(dev))
    exp = (tiled_decode(oracle, lat[0].permute(1, 0, 2, 3) / cfg.scaling_factor, 256, 32) / 2 + 0.5).clamp(0, 1)
    assert video.shape == (1, 3, z.shape[0], *m["raw_shape"][2:]) and video.min() >= 0 and video.max() <= 1
    _record("tiled_decode_latents_narrow_vs_oracle", (video[0].permute(1, 0, 2, 3) - exp).abs().max().item(), 1e-2 * scale)
    # measured 2.5e-3


def test_narrow_tiled_encode_vs_oracle_and_reference(built_lib):
    from musev_b200.synth import make_vae_images
    from musev_b200.vae import AutoencoderKLEncoder
    from oracle.vae_encoder_oracle import VAEEncoderOracle
    from oracle.vae_tiled_oracle import tiled_encode
    g, m, cfg, sd16 = _narrow()
    enc = AutoencoderKLEncoder(cfg, device=dev, dtype=torch.float32, frames_per_call=1)
    enc.load_state_dict(sd16)
    enc.enable_tiling()
    x = make_vae_images(m["image_shape"][0], *m["image_shape"][2:], seed=m["image_seed"])
    mom = enc.encode(x.to(dev)).latent_dist.parameters
    oracle = VAEEncoderOracle(cfg, {k: v.float() for k, v in sd16.items()}, device=dev)
    ref = tiled_encode(oracle, x, 256, 32)
    assert list(mom.shape) == m["moments_shape"] and mom.dtype == torch.float32 and torch.isfinite(mom).all()
    scale = max(1.0, ref.abs().max().item())
    _record("tiled_encode_narrow_vs_oracle", (mom - ref).abs().max().item(), 3e-3 * scale)   # measured 3.5e-3 at scale 2.7
    _record("tiled_encode_narrow_vs_reference",
            (mom.reshape(-1)[g["idx_moments"].to(dev)].cpu() - g["moments"]).abs().max().item(), 4e-3 * scale)   # measured 3.2e-3
    video = x.view(1, *x.shape).permute(0, 2, 1, 3, 4).contiguous()
    lat = enc.encode_video(video.to(dev), out_dtype=torch.float32)
    exp = cfg.scaling_factor * ref[:, :4]
    _record("tiled_encode_video_narrow_vs_oracle", (lat[0].permute(1, 0, 2, 3) - exp).abs().max().item(), 3e-3 * scale)   # measured 6.3e-4
    # the scaled mean of the blended moments: bit-identical to the host expression on encode's moments
    assert torch.equal(lat[0].permute(1, 0, 2, 3), cfg.scaling_factor * mom[:, :4])


def test_sd15_at_1216x704(built_lib):
    """SD-1.5 at a MuseV task size (1216x704 = 152x88 latents, 8 tiles in 6 shapes per frame), fp16 weights as the
    pipeline runs them, against the tiled oracle in fp32 on the GPU; frames_per_call 1 and 3 give the same frames."""
    from musev_b200.schema import VAEConfig
    from musev_b200.synth import make_vae_images
    from musev_b200.vae import AutoencoderKL
    from oracle.vae_encoder_oracle import VAEEncoderOracle
    from oracle.vae_tiled_oracle import tiled_decode, tiled_encode
    cfg = VAEConfig()
    sd16 = _sd16(cfg)
    vae = AutoencoderKL(cfg, device=dev, dtype=torch.float16, frames_per_call=3)
    vae.load_state_dict(sd16)
    vae.enable_tiling()
    oracle = VAEEncoderOracle(cfg, {k: v.float() for k, v in sd16.items()}, device=dev)
    lat = torch.randn(1, 4, 3, 152, 88, generator=torch.Generator().manual_seed(4)) * 0.18215
    video = vae.decode_latents(lat.to(dev))
    assert video.shape == (1, 3, 3, 1216, 704) and video.dtype == torch.float32
    z = lat[0].permute(1, 0, 2, 3) / cfg.scaling_factor
    exp = (tiled_decode(oracle, z, 512, 64) / 2 + 0.5).clamp(0, 1)
    _record("tiled_decode_latents_1216x704_vs_oracle", (video[0].permute(1, 0, 2, 3) - exp).abs().max().item(), 1.5e-2)   # measured 3.2e-3
    images = make_vae_images(3, 1216, 704, seed=5).half()
    vid = images.permute(1, 0, 2, 3)[None].contiguous()                                    # [1, 3, 3, 1216, 704] fp16
    latents = vae.encode_video(vid.to(dev), out_dtype=torch.float32)
    assert latents.shape == (1, 4, 3, 152, 88)
    ref = cfg.scaling_factor * tiled_encode(oracle, images.float(), 512, 64)[:, :4]
    _record("tiled_encode_video_1216x704_vs_oracle", (latents[0].permute(1, 0, 2, 3) - ref).abs().max().item(),
            3e-3 * max(1.0, ref.abs().max().item()))        # measured 7.2e-4 (moments blended in fp16, as the reference does)
    vae.frames_per_call = 1
    assert torch.equal(vae.decode_latents(lat.to(dev)), video)
    assert torch.equal(vae.encode_video(vid.to(dev), out_dtype=torch.float32), latents)


def test_dispatch(built_lib):
    """Tiling on at or under the tile size is the untiled path; disable_tiling() restores it (with its 8192 refusal);
    enable_tiling() on the drop-in object tiles both halves; enable_slicing() changes no bits."""
    from musev_b200.synth import make_vae_images
    from musev_b200.vae import AutoencoderKL
    g, m, cfg, sd16 = _narrow()
    vae = AutoencoderKL(cfg, device=dev, dtype=torch.float16, frames_per_call=2)
    vae.load_state_dict(sd16)
    small_z = torch.randn(2, 4, 32, 24, generator=torch.Generator().manual_seed(1)).half().to(dev)
    small_x = make_vae_images(2, 256, 192, seed=2).half().to(dev)
    big_z = torch.randn(2, 4, 56, 40, generator=torch.Generator().manual_seed(3)).half().to(dev)
    big_x = make_vae_images(2, 448, 320, seed=4).half().to(dev)
    base_dec = vae.decode(small_z).sample
    base_enc = vae.encode(small_x).latent_dist.parameters
    vae.enable_tiling()          # what pipeline.enable_vae_tiling() calls on pipeline.vae
    assert vae.use_tiling and vae.encoder.use_tiling and vae.decoder.use_tiling
    assert torch.equal(vae.decode(small_z).sample, base_dec)
    assert torch.equal(vae.encode(small_x).latent_dist.parameters, base_enc)
    tiled_dec = vae.decode(big_z).sample
    tiled_mom = vae.encode(big_x).latent_dist.parameters
    assert tiled_dec.dtype == torch.float16 and tiled_mom.dtype == torch.float16     # encode blends in the image dtype
    assert torch.equal(tiled_dec, vae.tiled_decode(big_z).sample)
    assert torch.equal(tiled_mom, vae.tiled_encode(big_x).latent_dist.parameters)
    assert not torch.equal(tiled_dec, vae.decoder._run(big_z, 1.0, False, torch.float16))   # a different computation
    # a latent side above tile_latent_min_size tiles even when the frame fits untiled (autoencoder_kl.py:300)
    wide = torch.randn(1, 4, 32, 48, generator=torch.Generator().manual_seed(5)).half().to(dev)
    assert torch.equal(vae.decode(wide).sample, vae.tiled_decode(wide).sample)
    vae.enable_slicing()
    assert vae.use_slicing and torch.equal(vae.decode(big_z).sample, tiled_dec)
    assert torch.equal(vae.encode(big_x).latent_dist.parameters, tiled_mom)
    vae.disable_slicing()
    vae.tile_overlap_factor = 0.25          # the drop-in's attributes reach both halves
    assert vae.encoder.tile_overlap_factor == vae.decoder.tile_overlap_factor == 0.25
    vae.disable_tiling()
    assert not vae.use_tiling
    assert torch.equal(vae.decode(small_z).sample, base_dec)
    with pytest.raises(ValueError, match="8192"):
        vae.encode(torch.zeros(1, 3, 1024, 768, device=dev, dtype=torch.float16))
    vae.enable_tiling()
    big = vae.encode(torch.zeros(1, 3, 1024, 768, device=dev, dtype=torch.float16)).latent_dist.mean
    assert big.shape == (1, 4, 128, 96) and torch.isfinite(big).all()


def test_refusals_before_launch(built_lib):
    from musev_b200 import _capi
    from musev_b200.vae import AutoencoderKL
    g, m, cfg, sd16 = _narrow()
    vae = AutoencoderKL(cfg, device=dev, dtype=torch.float16)
    vae.load_state_dict(sd16)
    vae.enable_tiling()
    torch.cuda.synchronize()
    n0 = _capi.launch_count(-1)
    z = torch.zeros(1, 4, 50, 40, device=dev, dtype=torch.float16)          # a 2 x 16-latent sliver tile
    with pytest.raises(ValueError, match="multiple of 64"):
        vae.decode(z)
    with pytest.raises(ValueError, match="multiple of 64"):
        vae.decode_latents(z.view(1, 4, 1, 50, 40))
    with pytest.raises(ValueError, match="multiple of 8"):
        vae.encode(torch.zeros(1, 3, 452, 320, device=dev, dtype=torch.float16))
    vae.tile_overlap_factor = 0.3           # a 22-latent stride is 176 pixels against a row_limit of 180
    with pytest.raises(ValueError, match="crops add up"):
        vae.decode(torch.zeros(1, 4, 56, 40, device=dev, dtype=torch.float16))
    with pytest.raises(ValueError, match="not a multiple of 8"):                # a 179-pixel stride
        vae.encode_video(torch.zeros(1, 3, 1, 448, 320, device=dev, dtype=torch.float16))
    vae.tile_overlap_factor = 0.25
    vae.tile_latent_min_size = 33
    with pytest.raises(ValueError):
        vae.decode(torch.zeros(1, 4, 56, 40, device=dev, dtype=torch.float16))
    assert _capi.launch_count(-1) == n0


def _run_sharded(rank, world, port):
    import torch.distributed as dist
    from musev_b200.synth import make_vae_images
    from musev_b200.vae import AutoencoderKL
    d = torch.device("cuda", 0)
    torch.cuda.set_device(d)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world,
                            timeout=datetime.timedelta(seconds=180))
    group = dist.group.WORLD
    g, m, cfg, sd16 = _narrow()
    vae = AutoencoderKL(cfg, device=d, dtype=torch.float16, frames_per_call=2)
    vae.load_state_dict(sd16)
    vae.enable_tiling()
    f = 5                                                                                 # 3 chunks: 2 + 1 per rank
    frames = make_vae_images(f, 448, 320, seed=9).to(d)
    video = frames.half().permute(1, 0, 2, 3)[None].contiguous()
    latents = (torch.randn(1, 4, f, 56, 40, generator=torch.Generator().manual_seed(9)) * 0.18215).to(d)
    z = latents[0].permute(1, 0, 2, 3).contiguous() / cfg.scaling_factor
    calls = {
        "decode_latents": lambda pg: vae.decode_latents(latents, process_group=pg),
        "decode": lambda pg: vae.decode(z, process_group=pg).sample,
        "encode_video": lambda pg: vae.encode_video(video, process_group=pg),
        "encode": lambda pg: vae.encode(frames, process_group=pg).latent_dist.parameters,
    }
    for name, call in calls.items():
        one = call(None)
        shard = call(group)
        torch.cuda.synchronize()
        assert shard.shape == one.shape and torch.isfinite(one).all(), (rank, name)
        assert torch.equal(shard, one), (rank, name, (shard.float() - one.float()).abs().max().item())
    dist.destroy_process_group()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_two_ranks_on_one_gpu_gloo_equal_unsharded(built_lib):
    mp.spawn(_run_sharded, args=(2, _free_port()), nprocs=2, join=True)
