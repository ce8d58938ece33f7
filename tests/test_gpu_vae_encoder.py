"""VAE encode on the engine: the pad-(0,1,0,1) stride-2 convolution, the encoder against the oracle and the reference golden
samples (tests/golden/vae_encoder_*.pt, produced by the unmodified diffusers AutoencoderKL.encode), SD-1.5 at 512x512,
the drop-in `AutoencoderKL` driven by the pipeline's own expressions, and shape validation. With MVB_PARITY_LOG=<file> set,
every measured distance is appended to <file> next to its bound (`_record`), one JSON object per line, so that the written
bounds can be audited against what was measured."""
import ctypes as C
import json
import os

import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN

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


# C = 128 / 256 / 512 (the encoder's downsamplers), a non-square image and frame counts that leave partial tiles
@pytest.mark.parametrize("NF,H,W,C", [(3, 16, 24, 128), (2, 32, 32, 256), (5, 8, 16, 512), (7, 64, 48, 128)])
def test_conv_stride2_pad_end(built_lib, NF, H, W, C):
    from musev_b200 import ops
    torch.manual_seed(3)
    x = torch.randn(NF, H, W, C, device=dev).half()
    wt = (torch.randn(C, C, 3, 3, device=dev) / (9 * C) ** 0.5).half()
    b = torch.randn(C, device=dev)
    out = ops.conv_gemm(x, wt.permute(0, 2, 3, 1).reshape(C, 9 * C).contiguous(), taps=ops.TAPS_3X3, bias=b, stride2=2)
    ref = F.conv2d(F.pad(x.float().permute(0, 3, 1, 2), (0, 1, 0, 1)), wt.float(), b, stride=2)
    ref = ref.permute(0, 2, 3, 1).reshape(-1, C)
    assert out.shape == ref.shape and not torch.isnan(out.float()).any()
    # the _close tolerance of test_gpu_ops.py::test_conv_stride2
    _record(f"conv_stride2_pad_end[{NF},{H},{W},{C}]", (out.float() - ref).abs().max().item(), 2e-3 + 3e-3 * ref.abs().max().item())


@pytest.mark.parametrize("tag", ["narrow", "full"])
def test_vae_encode_vs_oracle_and_reference_golden(built_lib, tag):
    from musev_b200.schema import VAEConfig
    from musev_b200.synth import make_vae_images
    from musev_b200.vae import AutoencoderKLEncoder
    from oracle.vae_encoder_oracle import VAEEncoderOracle
    g = torch.load(os.path.join(GOLDEN, f"vae_encoder_{tag}.pt"))
    m = g["meta"]
    cfg = VAEConfig(block_out_channels=tuple(m["block_out_channels"]))
    sd16 = _sd16(cfg, m["weight_seed"])
    enc = AutoencoderKLEncoder(cfg, device=dev, dtype=torch.float32, frames_per_call=1)
    enc.load_state_dict(sd16)
    x = make_vae_images(m["frames"], m["H"], m["W"], m["input_seed"])
    mom = enc.encode(x.to(dev)).latent_dist.parameters
    assert list(mom.shape) == m["shape"] and mom.dtype == torch.float32 and torch.isfinite(mom).all()
    ref = VAEEncoderOracle(cfg, {k: v.float() for k, v in sd16.items()}, device=dev).moments(x)
    scale = max(1.0, ref.abs().max().item())
    _record(f"vae_encode_{tag}_vs_oracle", (mom - ref).abs().max().item(), 3e-3 * scale)   # measured 2.6e-3 / 2.7e-3 at scale 2.3 / 2.5
    idx = torch.randint(0, mom.numel(), (m["n_samples"],), generator=torch.Generator().manual_seed(m["sample_seed"]))
    _record(f"vae_encode_{tag}_vs_reference", (mom.reshape(-1)[idx].cpu() - g["moments"]).abs().max().item(),
            4e-3 * scale)   # measured 3.3e-3 / 3.5e-3 at scale 2.3 / 2.5


def test_vae_encode_512(built_lib):
    """SD-1.5 encoder at the pipeline's size and dtype (512x512, fp16 images), 2 frames, against the oracle run as eager fp32
    on the GPU; chunking (frames_per_call 1 vs 2) gives the same latents; the in-library `scaling_factor * mean` equals the
    host expression on the moments bit for bit."""
    from musev_b200.schema import VAEConfig
    from musev_b200.synth import make_vae_images
    from musev_b200.vae import AutoencoderKLEncoder
    from oracle.vae_encoder_oracle import VAEEncoderOracle
    cfg = VAEConfig()
    sd16 = _sd16(cfg)
    enc = AutoencoderKLEncoder(cfg, device=dev, dtype=torch.float16, frames_per_call=2)
    enc.load_state_dict(sd16)
    video = make_vae_images(2, 512, 512, seed=5).half().permute(1, 0, 2, 3)[None].contiguous()     # [1, 3, 2, 512, 512]
    lat = enc.encode_video(video.to(dev), out_dtype=torch.float32)
    assert lat.shape == (1, 4, 2, 64, 64)
    ref = VAEEncoderOracle(cfg, {k: v.float() for k, v in sd16.items()}, device=dev).encode_video(video.float())
    _record("vae_encode_512_vs_oracle", (lat - ref).abs().max().item(), 1.5e-3 * max(1.0, ref.abs().max().item()))   # measured 6.0e-4
    enc.frames_per_call = 1
    assert torch.equal(enc.encode_video(video.to(dev), out_dtype=torch.float32), lat)
    x = video[0].permute(1, 0, 2, 3).contiguous().to(dev)
    mean = enc.encode(x.float()).latent_dist.mean
    assert torch.equal(cfg.scaling_factor * mean, lat[0].permute(1, 0, 2, 3))
    assert enc.encode(x).latent_dist.mean.dtype == torch.float16          # moments come back in the input dtype


def test_autoencoderkl_drop_in(built_lib):
    """One object for `pipeline.vae`: a full AutoencoderKL state dict, encode and decode, and the pipeline's expressions
    (musev/pipelines/pipeline_controlnet.py:348-368, 809-811, 978-981) run unmodified."""
    from einops import rearrange
    from musev_b200.schema import VAEConfig
    from musev_b200.synth import make_vae_images
    from musev_b200.vae import AutoencoderKL
    from oracle.vae_encoder_oracle import VAEEncoderOracle
    cfg = VAEConfig()
    sd16 = _sd16(cfg)
    vae = AutoencoderKL(cfg, device=dev, dtype=torch.float16)
    res = vae.load_state_dict(sd16)
    assert not res.missing_keys and not res.unexpected_keys
    assert vae.config.scaling_factor == 0.18215 and tuple(vae.config.block_out_channels) == (128, 256, 512, 512)
    assert vae.dtype == torch.float16 and vae.device.type == "cuda" and vae.eval() is vae
    oracle = VAEEncoderOracle(cfg, {k: v.float() for k, v in sd16.items()}, device=dev)
    images = make_vae_images(2, 256, 256, seed=8).half().to(dev)
    ref = cfg.scaling_factor * oracle.latent_dist(images.float())[0]
    bound = 1.5e-3 * max(1.0, ref.abs().max().item())          # measured 5.2e-4
    # prepare_condition_latents_and_index (:978-981) and get_referencenet_image_vae_emb (:809-811)
    condition_latents = vae.encode(images).latent_dist.mean
    condition_latents = vae.config.scaling_factor * condition_latents
    _record("drop_in_condition_latents", (condition_latents.float() - ref).abs().max().item(), bound)
    # prepare_latents, video2video (:348-368), with and without a list of generators
    image = rearrange(images[None].permute(0, 2, 1, 3, 4), "b c t h w->(b t) c h w")
    init_latents = vae.config.scaling_factor * vae.encode(image).latent_dist.mean
    per = torch.cat([vae.encode(image[i: i + 1]).latent_dist.mean for i in range(2)], dim=0)
    assert torch.equal(vae.config.scaling_factor * per, init_latents)
    assert torch.equal(init_latents, condition_latents)
    # the same object decodes
    img = vae.decode(init_latents / vae.config.scaling_factor).sample
    assert img.shape == (2, 3, 256, 256) and img.dtype == torch.float16 and torch.isfinite(img).all()
    video = vae.decode_latents(init_latents.permute(1, 0, 2, 3)[None])
    assert video.shape == (1, 3, 2, 256, 256) and video.min() >= 0 and video.max() <= 1
    # latent_dist.sample(generator): mean + std * N(0, 1)
    dist = vae.encode(images.float()).latent_dist
    s = dist.sample(torch.Generator().manual_seed(0))
    assert s.shape == (2, 4, 32, 32) and s.device == dist.mean.device
    z = (s - dist.mean) / dist.std
    assert abs(z.mean().item()) < 0.05 and abs(z.std().item() - 1.0) < 0.05
    assert torch.equal(dist.sample(torch.Generator().manual_seed(0)), s)


def test_vae_encode_rejects_bad_shapes_before_launch(built_lib):
    from musev_b200 import _capi
    from musev_b200.schema import VAEConfig
    from musev_b200._capi import MvbVaeDecodeArgs
    from musev_b200.vae import AutoencoderKLEncoder
    cfg = VAEConfig(block_out_channels=(64, 64, 128, 128))
    enc = AutoencoderKLEncoder(cfg, device=dev, dtype=torch.float16)
    enc.load_state_dict(_sd16(cfg))
    torch.cuda.synchronize()
    n0 = _capi.launch_count(-1)
    for shape, what in (((1, 4, 64, 64), "channels"), ((1, 3, 100, 96), "multiple of 8"), ((1, 3, 1024, 768), "8192")):
        with pytest.raises(ValueError, match=what):
            enc.encode(torch.zeros(shape, device=dev, dtype=torch.float16))
    assert _capi.launch_count(-1) == n0
    # the library checks the latent size itself, before any launch
    l = _capi.lib()
    x = torch.zeros(1, 3, 1024, 768, device=dev, dtype=torch.float16)
    out = torch.empty(1, 8, 128, 96, device=dev, dtype=torch.float16)
    a = MvbVaeDecodeArgs()
    a.latents, a.N, a.h, a.w, a.out, a.postprocess = x.data_ptr(), 1, 128, 96, out.data_ptr(), 0
    assert l.mvb_vae_encode_workspace_bytes(enc._h, C.byref(a)) == -1
    assert b"8192" in l.mvb_handle_error(enc._h)
    ws = torch.empty(1 << 20, dtype=torch.uint8, device=dev)
    assert l.mvb_vae_encode(enc._h, C.byref(a), ws.data_ptr(), ws.numel(), None) == -1          # MVB_ERR_INVALID
    a.h, a.w, a.postprocess = 8, 8, 3
    assert l.mvb_vae_encode(enc._h, C.byref(a), ws.data_ptr(), ws.numel(), None) == -1
    assert _capi.launch_count(-1) == n0
