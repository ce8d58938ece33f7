"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/pose_guider_{narrow,full}.pt and tests/golden/unet_pose_narrow.pt by
running the UNMODIFIED reference `musev.models.controlnet.PoseGuider` and `UNet3DConditionModel.forward(...,
pose_guider_emb=...)` on CPU in fp32.

Run in the build container only:  python -m oracle.make_golden_pose_guider
Weights and inputs are regenerated from the seeds in each fixture's meta (musev_b200.synth, bit-identical CPU RNG). The
reference is never read at test time.
"""
from __future__ import annotations

import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from musev_b200.schema import PoseGuiderConfig, pose_guider_param_shapes, preset_config  # noqa: E402
from musev_b200.synth import (make_inputs, make_pose_guider_emb, make_pose_guider_state_dict, make_pose_images,  # noqa: E402
                              make_state_dict)
from oracle import ref_shim  # noqa: E402
from oracle.make_golden import NARROW, build_reference, run_reference_unet  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
CONFIGS = {"narrow": PoseGuiderConfig(64, 3, (16, 32, 64, 128)),      # the class default, narrow UNet width
           "full": PoseGuiderConfig(320, 3, (16, 32, 96, 256))}       # scripts/inference/video2video.py:1024-1030


def golden_pose_guider(tag, b, t, H, W, wseed=21, iseed=1717):
    ref_shim.load()
    from musev.models.controlnet import PoseGuider
    cfg = CONFIGS[tag]
    t0 = time.time()
    m = PoseGuider(cfg.conditioning_embedding_channels, cfg.conditioning_channels, cfg.block_out_channels).eval()
    ref_shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert ref_shapes == {k: tuple(v) for k, v in pose_guider_param_shapes(cfg).items()}, "PoseGuider schema mismatch"
    res = m.load_state_dict(make_pose_guider_state_dict(cfg, seed=wseed), strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    x = make_pose_images(b * t, H, W, iseed).reshape(b, t, cfg.conditioning_channels, H, W).permute(0, 2, 1, 3, 4)
    with torch.no_grad():
        out = m(x.contiguous())
    meta = dict(conditioning_embedding_channels=cfg.conditioning_embedding_channels,
                conditioning_channels=cfg.conditioning_channels, block_out_channels=list(cfg.block_out_channels),
                b=b, t=t, H=H, W=W, weight_seed=wseed, input_seed=iseed,
                source="reference musev.models.controlnet.PoseGuider, CPU fp32")
    path = os.path.join(GOLDEN, f"pose_guider_{tag}.pt")
    torch.save({"meta": meta, "out": out.clone()}, path)
    print(f"{path}: out {tuple(out.shape)} std {out.std().item():.4f} ({time.time() - t0:.1f}s)", flush=True)


def golden_unet_pose(batch=2, frames=2, h=8, w=8, t=601, wseed=0, iseed=1234, pseed=5151, frame_rate=8, ip_scale=0.7):
    outs = {}
    for preset in ("musev", "musev_referencenet"):
        t0 = time.time()
        cfg = preset_config(preset, block_out_channels=NARROW)
        m, cfg = build_reference(preset, NARROW, make_state_dict(cfg, seed=wseed))
        inp = make_inputs(cfg, batch=batch, frames=frames, h=h, w=w, n_vis_cond=1, seed=iseed)
        T = frames + 1
        emb = make_pose_guider_emb(batch * T, NARROW[0], h, w, seed=pseed)
        with torch.no_grad():
            out = m(inp["sample"], torch.tensor(t), inp["encoder_hidden_states"], sample_index=inp["sample_index"],
                    vision_conditon_frames_sample_index=inp["vision_conditon_frames_sample_index"],
                    sample_frame_rate=frame_rate, do_classifier_free_guidance=True,
                    down_block_refer_embs=inp.get("down_block_refer_embs"), mid_block_refer_emb=inp.get("mid_block_refer_emb"),
                    vision_clip_emb=inp.get("vision_clip_emb"), ip_adapter_scale=ip_scale, pose_guider_emb=emb)[0]
            plain = run_reference_unet(m, inp, t, frame_rate, ip_scale)
        outs[preset] = out.clone()
        print(f"{preset}: pose moves the output by {float((out - plain).abs().max()):.4f} ({time.time() - t0:.1f}s)", flush=True)
        del m
    meta = dict(block_out_channels=list(NARROW), batch=batch, frames=frames, h=h, w=w, timestep=t, weight_seed=wseed,
                input_seed=iseed, pose_seed=pseed, sample_frame_rate=frame_rate, ip_adapter_scale=ip_scale, n_vis_cond=1,
                source="reference musev.models.unet_3d_condition.UNet3DConditionModel with pose_guider_emb, CPU fp32")
    path = os.path.join(GOLDEN, "unet_pose_narrow.pt")
    torch.save({"meta": meta, "out": outs}, path)
    print(path, flush=True)


if __name__ == "__main__":
    os.makedirs(GOLDEN, exist_ok=True)
    torch.set_num_threads(os.cpu_count() or 1)
    golden_pose_guider("narrow", b=1, t=2, H=48, W=64)
    golden_pose_guider("full", b=1, t=1, H=64, W=48)
    golden_unet_pose()
