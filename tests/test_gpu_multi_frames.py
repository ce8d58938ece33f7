"""The per-frame stages sharded over two ranks (`process_group=`): VAE decode and encode and the PoseGuider return, on every
rank, exactly the bits of the same call without a group. b = 2 videos of f = 9 frames (18 frames, frames_per_call 4 ->
5 chunks, split 3 + 2) and of f = 1 (one chunk; rank 1 launches nothing and only receives). Two processes, one per GPU,
NCCL; and two processes sharing one GPU over gloo, which runs wherever the GPU tests run."""
import datetime
import os
import socket

import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu


def _run(rank, world, port, backend):
    import torch.distributed as dist
    from musev_b200.controlnet import PoseGuider
    from musev_b200.schema import PoseGuiderConfig, VAEConfig
    from musev_b200.synth import make_pose_guider_state_dict, make_pose_images, make_state_dict, make_vae_images
    from musev_b200.vae import AutoencoderKL
    dev = torch.device("cuda", rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    os.environ.setdefault("NCCL_DEBUG", "WARN")
    dist.init_process_group(backend, init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world,
                            timeout=datetime.timedelta(seconds=180), device_id=dev if backend == "nccl" else None)
    group = dist.group.WORLD
    cfg = VAEConfig(block_out_channels=(64, 64, 128, 128))
    vae = AutoencoderKL(cfg, device=dev, dtype=torch.float16, frames_per_call=4)
    vae.load_state_dict({k: v.half() for k, v in make_state_dict(cfg, seed=11).items()})
    pcfg = PoseGuiderConfig(64, 3, (16, 32, 64, 128))
    pose_guider = PoseGuider(64, 3, pcfg.block_out_channels, device=dev, dtype=torch.float16, frames_per_call=4)
    pose_guider.load_state_dict({k: v.half() for k, v in make_pose_guider_state_dict(pcfg, seed=21).items()})
    for f in (9, 1):
        frames = make_vae_images(2 * f, 64, 64, seed=f).to(dev)                                # [b f, 3, 64, 64] fp32
        video = frames.half().view(2, f, 3, 64, 64).permute(0, 2, 1, 3, 4).contiguous()        # [b, 3, f, 64, 64] fp16
        latents = (torch.randn(2, 4, f, 8, 8, generator=torch.Generator().manual_seed(f)) * 0.18215).to(dev)
        z = latents.permute(0, 2, 1, 3, 4).reshape(2 * f, 4, 8, 8) / cfg.scaling_factor
        pose = make_pose_images(2 * f, 64, 64, seed=f + 1).to(dev).view(2, f, 3, 64, 64).permute(0, 2, 1, 3, 4)
        calls = {
            "decode_latents": lambda pg: vae.decode_latents(latents, process_group=pg),
            "decode": lambda pg: vae.decode(z, process_group=pg).sample,
            "encode_video": lambda pg: vae.encode_video(video, process_group=pg),
            "encode_mean": lambda pg: vae.encode(frames, process_group=pg).latent_dist.mean,
            "pose_guider": lambda pg: pose_guider(pose, process_group=pg),
        }
        for name, call in calls.items():
            one = call(None)
            shard = call(group)
            torch.cuda.synchronize()
            assert shard.shape == one.shape and torch.isfinite(one).all(), (rank, f, name)
            assert torch.equal(shard, one), (rank, f, name, (shard.float() - one.float()).abs().max().item())
    dist.destroy_process_group()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_nccl_equal_one_gpu(built_lib):
    mp.spawn(_run, args=(2, _free_port(), "nccl"), nprocs=2, join=True)


def test_two_ranks_on_one_gpu_gloo_equal_unsharded(built_lib):
    mp.spawn(_run, args=(2, _free_port(), "gloo"), nprocs=2, join=True)
