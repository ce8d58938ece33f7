"""CPU tests of the PoseGuider feature: the oracle against the reference fixtures (tests/golden/pose_guider_*.pt and
unet_pose_narrow.pt, produced by oracle/make_golden_pose_guider.py from the unmodified reference), the FLOP counter, the
host-side rejections, the per-window slicing of `pose_guider_emb` in ParallelDenoiser (fake UNet, CPU ops double; one and
two gloo ranks) and the ctypes bindings of the new C entry points."""
import os

import pytest
import torch
import torch.multiprocessing as mp

from conftest import GOLDEN
from musev_b200.context import prepare_global_context
from musev_b200.schema import PoseGuiderConfig, pose_guider_param_shapes, preset_config
from musev_b200.synth import (make_inputs, make_pose_guider_emb, make_pose_guider_state_dict, make_pose_images,
                              make_state_dict)
from test_host_logic import OracleOpsDouble, _free_port


def _pg_cfg(m):
    return PoseGuiderConfig(m["conditioning_embedding_channels"], m["conditioning_channels"], tuple(m["block_out_channels"]))


@pytest.mark.parametrize("tag", ["narrow", "full"])
def test_oracle_reproduces_reference_pose_guider(tag):
    from oracle.pose_guider_oracle import PoseGuiderOracle
    g = torch.load(os.path.join(GOLDEN, f"pose_guider_{tag}.pt"))
    m = g["meta"]
    cfg = _pg_cfg(m)
    o = PoseGuiderOracle(cfg, make_pose_guider_state_dict(cfg, seed=m["weight_seed"]))
    x = make_pose_images(m["b"] * m["t"], m["H"], m["W"], m["input_seed"])
    x = x.reshape(m["b"], m["t"], cfg.conditioning_channels, m["H"], m["W"]).permute(0, 2, 1, 3, 4)
    out = o(x)
    assert out.shape == g["out"].shape
    assert g["out"].abs().max().item() > 0.1                       # conv_out is drawn non-zero: the output carries signal
    assert (out - g["out"]).abs().max().item() < 1e-5


def test_unet_oracle_adds_pose_guider_emb_like_reference():
    from oracle.pose_guider_oracle import UNet3DPoseOracle
    g = torch.load(os.path.join(GOLDEN, "unet_pose_narrow.pt"))
    m = g["meta"]
    torch.set_num_threads(max(1, min(8, os.cpu_count() or 1)))
    for preset, ref in g["out"].items():
        cfg = preset_config(preset, block_out_channels=tuple(m["block_out_channels"]))
        o = UNet3DPoseOracle(cfg, make_state_dict(cfg, seed=m["weight_seed"]))
        inp = make_inputs(cfg, batch=m["batch"], frames=m["frames"], h=m["h"], w=m["w"], n_vis_cond=1, seed=m["input_seed"])
        T = m["frames"] + 1
        emb = make_pose_guider_emb(m["batch"] * T, m["block_out_channels"][0], m["h"], m["w"], seed=m["pose_seed"])
        kw = dict(sample_index=inp["sample_index"], vision_conditon_frames_sample_index=inp["vision_conditon_frames_sample_index"],
                  sample_frame_rate=m["sample_frame_rate"], down_block_refer_embs=inp.get("down_block_refer_embs"),
                  mid_block_refer_emb=inp.get("mid_block_refer_emb"), vision_clip_emb=inp.get("vision_clip_emb"),
                  ip_adapter_scale=m["ip_adapter_scale"])
        out = o.forward(inp["sample"], m["timestep"], inp["encoder_hidden_states"], pose_guider_emb=emb, **kw)
        plain = o.forward(inp["sample"], m["timestep"], inp["encoder_hidden_states"], **kw)
        assert (out - ref).abs().max().item() < 1e-3, preset           # the pinned UNet oracle's own distance is ~1e-4
        assert (plain - ref).abs().max().item() > 0.1, preset          # and the emb is not silently dropped


@pytest.mark.parametrize("boc,H,W", [((16, 32, 96, 256), 512, 512), ((16, 32, 64, 128), 64, 48), ((16, 32), 40, 24)])
def test_pose_guider_flops_match_flop_counter(boc, H, W):
    from torch.utils.flop_counter import FlopCounterMode
    from musev_b200.flops import pose_guider_flops
    from oracle.pose_guider_oracle import PoseGuiderOracle
    cfg = PoseGuiderConfig(320, 3, boc)
    o = PoseGuiderOracle(cfg, make_pose_guider_state_dict(cfg), device="meta")
    with FlopCounterMode(display=False) as fc:
        o.frames(torch.empty(2, 3, H, W, device="meta"))
    assert pose_guider_flops(cfg, 2, H, W)["total"] == fc.get_total_flops()
    if boc == (16, 32, 96, 256):
        assert abs(pose_guider_flops(cfg, 1, 512, 512)["total"] / 1e9 - 14.722) < 1e-3


def test_state_dict_and_emb_rejections():
    from musev_b200.controlnet import check_pose_guider_state_dict
    from musev_b200.unet import check_pose_guider_emb
    cfg = PoseGuiderConfig(320, 3, (16, 32, 96, 256))
    sd = make_pose_guider_state_dict(cfg)
    todo, unexpected = check_pose_guider_state_dict(cfg, dict(sd, extra=torch.zeros(1)), strict=False)
    assert [n for n, _ in todo] == list(pose_guider_param_shapes(cfg)) and unexpected == ["extra"]
    with pytest.raises(RuntimeError, match="unexpected"):
        check_pose_guider_state_dict(cfg, dict(sd, extra=torch.zeros(1)), strict=True)
    for strict in (True, False):                      # the reference's strict=False would keep an initialiser value
        bad = dict(sd)
        bad.pop("blocks.3.bias")
        with pytest.raises(KeyError, match="blocks.3.bias"):
            check_pose_guider_state_dict(cfg, bad, strict=strict)
    bad = dict(sd, **{"conv_out.weight": torch.zeros(320, 128, 3, 3)})
    with pytest.raises(RuntimeError, match="size mismatch for conv_out.weight"):
        check_pose_guider_state_dict(cfg, bad)
    check_pose_guider_emb(torch.zeros(6, 320, 8, 8), 2, 3, 320, 8, 8)
    check_pose_guider_emb(torch.zeros(6, 320, 8, 8, dtype=torch.float16), 2, 3, 320, 8, 8)
    for t in (torch.zeros(2, 320, 3, 8, 8), torch.zeros(6, 64, 8, 8), torch.zeros(3, 320, 8, 8), torch.zeros(6, 320, 8, 4),
              torch.zeros(6, 320, 8, 8, dtype=torch.bfloat16)):
        with pytest.raises(ValueError, match="pose_guider_emb"):
            check_pose_guider_emb(t, 2, 3, 320, 8, 8)


# ------------------------------------------------------------------ ParallelDenoiser slicing
C0 = 6


def _fake_unet(sample, t, enc, pose_guider_emb=None, **k):
    """eps depends on the frame position, the prompt rows and -- through the emb -- on exactly which frames of
    pose_guider_emb ((b t) c h w) the window got."""
    b, c, tt, h, w = sample.shape
    pos = torch.arange(tt, dtype=sample.dtype).view(1, 1, -1, 1, 1)
    out = torch.sin(sample * 1.3 + 0.01 * float(t) + 0.37 * pos) + 0.1 * enc.mean((1, 2)).view(b, 1, 1, 1, 1)
    if pose_guider_emb is not None:
        assert tuple(pose_guider_emb.shape) == (b * tt, C0, h, w)
        p = pose_guider_emb.view(b, tt, C0, h, w)[:, :, :c].permute(0, 2, 1, 3, 4)
        out = out + 0.3 * torch.tanh(p)
    return out


def _inputs(T, h=4, w=4, seed=3):
    g = torch.Generator().manual_seed(seed)
    latents = torch.randn(1, 4, T, h, w, generator=g)
    cond = torch.randn(1, 4, 1, h, w, generator=g)
    prompt = torch.randn(2, 77, 8, generator=g)
    pose = torch.randn(2, C0, 1 + T, h, w, generator=g)
    return latents, cond, prompt, pose


def _denoiser(calls=None):
    from musev_b200.pipeline import ParallelDenoiser
    from musev_b200.scheduler import SD15_DDIM_CONFIG, DDIMScheduler

    def unet(s, t, e, return_dict=False, do_classifier_free_guidance=True, **k):
        if calls is not None:
            calls.append(k.get("pose_guider_emb"))
        return (_fake_unet(s, t, e, **k),)
    return ParallelDenoiser(unet, DDIMScheduler(**SD15_DDIM_CONFIG), device_ops=OracleOpsDouble)


@pytest.mark.parametrize("T,frames,overlap,schedule,stride", [(8, 12, 4, "uniform_v2", 1),     # one window
                                                              (20, 8, 4, "uniform_v2", 1),    # overlapping windows
                                                              (20, 12, 4, "uniform", 2)])     # repeated frames
def test_parallel_denoiser_slices_pose_emb_per_window(T, frames, overlap, schedule, stride):
    from oracle.pipeline_oracle import SD15_DDIM, DDIMOracle
    from oracle.pose_guider_oracle import denoise_loop_with_pose
    latents, cond, prompt, pose = _inputs(T)
    ctx = [c[0] for c in prepare_global_context(schedule, 2, T, frames, stride, overlap, 1)]
    if schedule == "uniform":
        assert any(len(set(c)) < len(c) for c in ctx)
    calls = []
    kw = dict(num_inference_steps=2, guidance_scale=2.5, context_frames=frames, context_overlap=overlap,
              context_schedule=schedule, context_stride=stride)
    res = _denoiser(calls)(latents, cond, prompt, pose_guider_emb=pose, **kw)
    ref = denoise_loop_with_pose(_fake_unet, DDIMOracle(**SD15_DDIM), latents, cond, prompt, 2, 2.5, pose,
                                 context_frames=frames, context_overlap=overlap, context_schedule=schedule,
                                 context_stride=stride)
    plain = _denoiser()(latents, cond, prompt, **kw)
    assert res.windows == ctx and len(calls) == 2 * len(ctx)
    assert (res.latents - ref).abs().max().item() < 1e-5
    assert (res.latents - plain.latents).abs().max().item() > 1e-2         # the emb reaches the UNet
    for wi, c in enumerate(ctx):                                             # vis-cond frames + the window's, duplicates kept
        exp = pose[:, :, [0] + [f + 1 for f in c]].permute(0, 2, 1, 3, 4).reshape(-1, C0, 4, 4)
        assert torch.equal(calls[wi], exp)
    if len(ctx) == 1:                                                        # one window: the reference's whole-video add
        assert torch.equal(calls[0], pose.permute(0, 2, 1, 3, 4).reshape(-1, C0, 4, 4))


def test_parallel_denoiser_rejects_bad_pose_emb():
    latents, cond, prompt, pose = _inputs(8)
    den = _denoiser()
    for bad in (pose[:1], pose[:, :, 1:], pose[..., :2], pose[0]):
        with pytest.raises(ValueError, match="pose_guider_emb"):
            den(latents, cond, prompt, num_inference_steps=1, guidance_scale=2.0, pose_guider_emb=bad)


def _split_worker(rank, world, port, out_path, cfg_split):
    import torch.distributed as dist
    if world > 1:
        dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    torch.set_num_threads(1)
    latents, cond, prompt, pose = _inputs(20)
    res = _denoiser()(latents, cond, prompt, num_inference_steps=2, guidance_scale=2.5, context_frames=8,
                      context_overlap=4, pose_guider_emb=pose, cfg_split=cfg_split)
    if rank == 0:
        torch.save(res.latents, out_path)
    if world > 1:
        dist.destroy_process_group()


def test_parallel_denoiser_pose_emb_under_cfg_split_two_ranks(tmp_path):
    p1, p2 = str(tmp_path / "one.pt"), str(tmp_path / "split.pt")
    _split_worker(0, 1, 0, p1, False)
    mp.spawn(_split_worker, args=(2, _free_port(), p2, True), nprocs=2, join=True)
    one, split = torch.load(p1), torch.load(p2)
    assert (split - one).abs().max().item() < 1e-5            # each rank got its own CFG half of the emb


def test_ctypes_argtypes_of_pose_guider_entry_points(built_lib):
    from test_capi_symbols import _prototypes
    from musev_b200 import _capi
    protos = _prototypes()
    lib = _capi.lib()
    for name in ("mvb_create_pose_guider", "mvb_pose_guider_workspace_bytes", "mvb_pose_guider_forward"):
        assert name in protos
        assert len(getattr(lib, name).argtypes) == protos[name], name
    # mvb_unet_args grew at the end only: every earlier field keeps its offset
    names = [f[0] for f in _capi.MvbUnetArgs._fields_]
    assert names[-2:] == ["pose_guider_emb", "pose_is_f32"] and names[-4:-2] == ["out", "out_is_f32"]
    assert lib.mvb_version() >= 2
