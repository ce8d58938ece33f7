"""PoseGuider on the engine: the engine PoseGuider against the oracle and the reference fixtures
(tests/golden/pose_guider_*.pt), the UNet's `pose_guider_emb` against the oracle and the reference
(tests/golden/unet_pose_narrow.pt), a multi-window loop, and rejection of bad shapes before any launch. With
MVB_PARITY_LOG=<file> set, every measured distance is appended to <file> next to its bound."""
import ctypes as C
import json
import os

import pytest
import torch

from conftest import GOLDEN
from musev_b200.schema import PoseGuiderConfig, preset_config
from musev_b200.synth import (make_inputs, make_pose_guider_emb, make_pose_guider_state_dict, make_pose_images,
                              make_state_dict)

pytestmark = pytest.mark.gpu
dev = "cuda"
FWD_TOL = 1e-2
PG_TOL = 2.5e-4                  # engine PoseGuider vs fp32 oracle / reference, per max(1, max|ref|)
UNET_TOL = {"musev": 7e-3, "musev_referencenet": FWD_TOL}   # measured 3.2e-3 / 5.2e-3 on H100
CONFIGS = [PoseGuiderConfig(64, 3, (16, 32, 64, 128)), PoseGuiderConfig(320, 3, (16, 32, 96, 256))]


def _record(name, err, bound):
    path = os.environ.get("MVB_PARITY_LOG")
    if path:
        try:
            with open(path, "a") as fh:
                fh.write(json.dumps({"test": name, "value": err, "bound": bound}) + "\n")
        except OSError:
            pass
    assert err < bound, (name, err, bound)


def _pose_guider(cfg, seed, dtype=torch.float32, frames_per_call=8):
    from musev_b200.controlnet import PoseGuider
    sd = {k: v.half() for k, v in make_pose_guider_state_dict(cfg, seed=seed).items()}
    pg = PoseGuider(cfg.conditioning_embedding_channels, cfg.conditioning_channels, cfg.block_out_channels, device=dev,
                    dtype=dtype, frames_per_call=frames_per_call).eval()
    pg.load_state_dict(sd)
    return pg, {k: v.float() for k, v in sd.items()}


@pytest.mark.parametrize("tag", ["narrow", "full"])
def test_pose_guider_vs_oracle_and_reference_golden(built_lib, tag):
    from oracle.pose_guider_oracle import PoseGuiderOracle
    g = torch.load(os.path.join(GOLDEN, f"pose_guider_{tag}.pt"))
    m = g["meta"]
    cfg = PoseGuiderConfig(m["conditioning_embedding_channels"], m["conditioning_channels"], tuple(m["block_out_channels"]))
    pg, sd32 = _pose_guider(cfg, m["weight_seed"], frames_per_call=1)
    x = make_pose_images(m["b"] * m["t"], m["H"], m["W"], m["input_seed"])
    x = x.reshape(m["b"], m["t"], 3, m["H"], m["W"]).permute(0, 2, 1, 3, 4).contiguous()
    out = pg(x.to(dev))
    assert out.shape == g["out"].shape and out.dtype == torch.float32
    ref = PoseGuiderOracle(cfg, sd32, device=dev)(x.to(dev))
    scale = max(1.0, ref.abs().max().item())
    # measured 6.7e-5 .. 1.1e-4 on H100 (start: FWD_TOL)
    _record(f"pose_guider_{tag}_vs_oracle", (out - ref).abs().max().item(), PG_TOL * scale)
    _record(f"pose_guider_{tag}_vs_reference_golden", (out.cpu() - g["out"]).abs().max().item(), PG_TOL * scale)


def test_pose_guider_full_512_vs_oracle(built_lib):
    """The script's config at the size users run it: (16, 32, 96, 256) -> 320 on 512 x 512, fp16 input and output."""
    from oracle.pose_guider_oracle import PoseGuiderOracle
    cfg = CONFIGS[1]
    pg, sd32 = _pose_guider(cfg, 21, dtype=torch.float16)
    x = make_pose_images(3, 512, 512, 99).to(dev).half()
    out = pg(x.permute(1, 0, 2, 3).unsqueeze(0))
    assert out.shape == (1, 320, 3, 64, 64) and out.dtype == torch.float16
    ref = PoseGuiderOracle(cfg, sd32, device=dev).frames(x.float())
    got = out[0].permute(1, 0, 2, 3).float()
    scale = max(1.0, ref.abs().max().item())
    _record("pose_guider_full_512_vs_oracle", (got - ref).abs().max().item(), PG_TOL * scale)   # measured 8.2e-5
    # deterministic, and frames do not interact
    again = pg.embed_frames(x[1:2])
    assert torch.equal(again[0], out[0, :, 1])


@pytest.mark.parametrize("cfg", CONFIGS, ids=["narrow", "script"])
def test_packed_weights_read_back_bit_exact(built_lib, cfg):
    """Every weight reads back from its packed layout bit for bit. The layers alternate between the per-tensor and the
    batched load; the script config's blocks.4 / blocks.5 read 96 channels stored as 128 (zero padding columns)."""
    from musev_b200 import _capi
    from musev_b200.controlnet import PoseGuider
    sd = {k: v.half().to(dev).contiguous() for k, v in make_pose_guider_state_dict(cfg, seed=5).items()}
    pg = PoseGuider(cfg.conditioning_embedding_channels, cfg.conditioning_channels, cfg.block_out_channels, device=dev)
    layers = list(dict.fromkeys(n.rsplit(".", 1)[0] for n in sd))
    per_tensor = [n for n in sd if layers.index(n.rsplit(".", 1)[0]) % 2 == 0]
    l = _capi.lib()
    for name in per_tensor:
        t = sd[name]
        shape = (C.c_longlong * t.dim())(*t.shape)
        assert l.mvb_load_weight(pg._h, name.encode(), t.data_ptr(), 0, shape, t.dim()) == 0, pg._error()
    _capi.load_weights_batched(pg._h, [(n, t) for n, t in sd.items() if n not in per_tensor], pg.device)
    assert l.mvb_finalize(pg._h) == 0, pg._error()
    bad = [n for n, t in sd.items() if t.dim() > 1 and not torch.equal(pg.debug_weight(n).view(torch.int16), t.view(torch.int16))]
    assert not bad, bad


def _unet(preset):
    from musev_b200.unet import UNet3DConditionModel
    from oracle.pose_guider_oracle import UNet3DPoseOracle
    g = torch.load(os.path.join(GOLDEN, "unet_pose_narrow.pt"))
    m = g["meta"]
    cfg = preset_config(preset, block_out_channels=tuple(m["block_out_channels"]))
    sd16 = {k: v.half() for k, v in make_state_dict(cfg, seed=m["weight_seed"]).items()}
    model = UNet3DConditionModel(cfg, device=dev, dtype=torch.float32)
    model.load_state_dict({k: v.to(dev) for k, v in sd16.items()})
    oracle = UNet3DPoseOracle(cfg, {k: v.float() for k, v in sd16.items()}, device=dev)
    inp = make_inputs(cfg, batch=m["batch"], frames=m["frames"], h=m["h"], w=m["w"], n_vis_cond=1, seed=m["input_seed"])
    emb = make_pose_guider_emb(m["batch"] * (m["frames"] + 1), m["block_out_channels"][0], m["h"], m["w"], seed=m["pose_seed"])
    kw = dict(sample_index=inp["sample_index"], vision_conditon_frames_sample_index=inp["vision_conditon_frames_sample_index"],
              sample_frame_rate=m["sample_frame_rate"], ip_adapter_scale=m["ip_adapter_scale"])
    for k in ("down_block_refer_embs", "mid_block_refer_emb", "vision_clip_emb"):
        if k in inp:
            kw[k] = inp[k]
    return g, m, model, oracle, inp, emb, kw


def _dev(v):
    if torch.is_tensor(v) and v.is_floating_point():
        return v.to(dev)
    if isinstance(v, list):
        return [_dev(x) for x in v]
    return v


@pytest.mark.parametrize("preset", ["musev", "musev_referencenet"])
def test_unet_pose_guider_emb_vs_oracle_and_reference_golden(built_lib, preset):
    g, m, model, oracle, inp, emb, kw = _unet(preset)
    dkw = {k: _dev(v) for k, v in kw.items()}
    sample, enc = inp["sample"].to(dev), inp["encoder_hidden_states"].to(dev)
    out = model(sample, torch.tensor(m["timestep"]), enc, pose_guider_emb=emb.to(dev), do_classifier_free_guidance=True, **dkw).sample
    ref = oracle(inp["sample"], m["timestep"], inp["encoder_hidden_states"], pose_guider_emb=emb, **kw)
    e_or = (out - ref).abs().max().item()
    e_gold = (out.cpu() - g["out"][preset]).abs().max().item()
    _record(f"unet_pose_{preset}_vs_oracle", e_or, UNET_TOL[preset])
    _record(f"unet_pose_{preset}_vs_reference_golden", e_gold, UNET_TOL[preset])
    plain = model(sample, torch.tensor(m["timestep"]), enc, **dkw).sample
    moved = (out - plain).abs().max().item()
    assert moved > 10 * max(e_or, e_gold), (moved, e_or, e_gold)
    # fp16 emb, as the pipeline passes it with an fp16 UNet
    out16 = model(sample, torch.tensor(m["timestep"]), enc, pose_guider_emb=emb.to(dev).half(), **dkw).sample
    ref16 = oracle(inp["sample"], m["timestep"], inp["encoder_hidden_states"], pose_guider_emb=emb.half().float(), **kw)
    _record(f"unet_pose_{preset}_fp16_emb_vs_oracle", (out16 - ref16).abs().max().item(), UNET_TOL[preset])


def test_unet_zero_pose_emb_is_bit_identical_to_none(built_lib):
    g, m, model, oracle, inp, emb, kw = _unet("musev_referencenet")
    dkw = {k: _dev(v) for k, v in kw.items()}
    sample, enc = inp["sample"].to(dev), inp["encoder_hidden_states"].to(dev)
    a = model(sample, torch.tensor(m["timestep"]), enc, **dkw).sample.clone()
    b = model(sample, torch.tensor(m["timestep"]), enc, pose_guider_emb=torch.zeros_like(emb).to(dev), **dkw).sample
    assert torch.equal(a, b)


def test_parallel_denoise_loop_with_pose_emb_vs_oracle_loop(built_lib):
    """2 DDIM steps x 3 overlapping windows, pose_guider_emb sliced per window, engine vs the oracle loop."""
    from musev_b200.pipeline import ParallelDenoiser
    from musev_b200.scheduler import SD15_DDIM_CONFIG, DDIMScheduler
    from oracle.pipeline_oracle import SD15_DDIM, DDIMOracle
    from oracle.pose_guider_oracle import denoise_loop_with_pose
    g, m, model, oracle, inp, emb, kw = _unet("musev")
    T, h, w = 20, 8, 8
    gen = torch.Generator().manual_seed(77)
    latents = torch.randn(1, 4, T, h, w, generator=gen)
    cond = torch.randn(1, 4, 1, h, w, generator=gen) * 0.5
    prompt = torch.randn(2, 77, 768, generator=gen)
    pose = torch.randn(2, m["block_out_channels"][0], 1 + T, h, w, generator=gen) * 0.5
    den = ParallelDenoiser(model, DDIMScheduler(**SD15_DDIM_CONFIG))
    res = den(latents.to(dev), cond.to(dev), prompt.to(dev), num_inference_steps=2, guidance_scale=3.5, context_frames=12,
              context_overlap=4, motion_speed=8, pose_guider_emb=pose.to(dev))
    assert len(res.windows) >= 2

    def unet(sample, t, enc, **k):
        return oracle(sample.to(dev), t, enc.to(dev), **{kk: _dev(v) for kk, v in k.items()}).cpu()
    ref = denoise_loop_with_pose(unet, DDIMOracle(**SD15_DDIM), latents, cond, prompt, 2, 3.5, pose, context_frames=12,
                                 context_overlap=4, motion_speed=8)
    plain = den(latents.to(dev), cond.to(dev), prompt.to(dev), num_inference_steps=2, guidance_scale=3.5, context_frames=12,
                context_overlap=4, motion_speed=8)
    err = (res.latents.cpu() - ref).abs().max().item()
    _record("loop_pose_musev_narrow_2step_vs_oracle", err, 5e-2)   # measured 2.3e-2 (start: 6e-2, test_gpu_unet.py)
    assert (res.latents - plain.latents).abs().max().item() > 10 * err


def test_rejects_bad_shapes_before_any_launch(built_lib):
    from musev_b200 import _capi
    from musev_b200._capi import MvbVaeDecodeArgs
    from musev_b200.controlnet import PoseGuider
    with pytest.raises(_capi.MvbError, match="mvb_create_pose_guider"):
        PoseGuider(320, 3, (16, 256), device=dev)                     # a 16-channel layer cannot produce 256 channels
    pg, _ = _pose_guider(CONFIGS[0], 21)
    n0 = _capi.launch_count()
    for bad in (torch.zeros(1, 3, 2, 60, 64), torch.zeros(1, 4, 2, 64, 64), torch.zeros(3, 64, 64), torch.zeros(1, 3, 2, 4, 8)):
        with pytest.raises(ValueError):
            pg(bad.to(dev))
    l = _capi.lib()
    x = torch.zeros(1, 3, 64, 64, device=dev)
    out = torch.zeros(1, 64, 8, 8, device=dev)
    ws = torch.empty(1 << 20, dtype=torch.uint8, device=dev)
    for N, h, w, post in ((0, 8, 8, 0), (1, 0, 8, 0), (1, 8, 8, 1), (1, 2048, 2048, 0)):
        a = MvbVaeDecodeArgs()
        a.latents, a.latents_is_f32, a.N, a.h, a.w = x.data_ptr(), 1, N, h, w
        a.out, a.out_is_f32, a.postprocess = out.data_ptr(), 1, post
        assert l.mvb_pose_guider_workspace_bytes(pg._h, C.byref(a)) < 0
        assert l.mvb_pose_guider_forward(pg._h, C.byref(a), ws.data_ptr(), ws.numel(), None) < 0
        assert l.mvb_handle_error(pg._h).decode().startswith("pose guider:")
    assert _capi.launch_count() == n0
    g, m, model, oracle, inp, emb, kw = _unet("musev")
    dkw = {k: _dev(v) for k, v in kw.items()}
    n1 = _capi.launch_count()
    for bad in (emb[:3], emb[:, :32], emb.unsqueeze(0), emb.to(torch.bfloat16)):
        with pytest.raises(ValueError, match="pose_guider_emb"):
            model(inp["sample"].to(dev), 601, inp["encoder_hidden_states"].to(dev), pose_guider_emb=bad.to(dev), **dkw)
    assert _capi.launch_count() == n1
