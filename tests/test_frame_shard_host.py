"""CPU tests of the frame sharding behind `process_group=` of the VAE and the PoseGuider (`_capi.launch_frame_chunks`): on 2
and 3 gloo ranks the gathered output equals the unsharded call bit for bit, the ranks launch exactly the chunks the
single-GPU `_launch_frames` launches, and ranks that disagree on the call all raise ValueError instead of waiting on each
other. A stand-in launch replaces the library."""
import datetime
import os
import socket

import pytest
import torch
import torch.multiprocessing as mp

from musev_b200._capi import EngineModel, frame_chunks, launch_frame_chunks

NS = (1, 2, 4, 5, 13, 17)
STEPS = (1, 4)


def _inputs(n):
    return torch.randn(n, 3, 5, 7, generator=torch.Generator().manual_seed(n))


def _model_fn(x, out):
    """A launch whose result depends on the other frames of its chunk, so a chunk boundary that moved would show."""
    def launch(n0, n1):
        xc = x[n0:n1]
        out[n0:n1] = torch.sin(1.7 * xc) + 0.25 * xc.sum(0, keepdim=True)
    return launch


class _RecordingModel:
    """Stands in for an `EngineModel` in `EngineModel._launch_frames`: records the frame range of every launch."""

    def __init__(self, x, frames_per_call):
        self.x, self.frames_per_call, self.ranges = x, frames_per_call, []

    def _launch(self, a):
        row = self.x[0].numel() * self.x.element_size()
        n0 = (a.latents - self.x.data_ptr()) // row
        self.ranges.append((n0, n0 + a.N))


def _launch_frames_ranges(n, step, process_group=None):
    x = _inputs(n)
    m = _RecordingModel(x, step)
    EngineModel._launch_frames(m, x, torch.zeros(n, 2, 5, 7), 5, 7, 1.0, 0, process_group)
    return m.ranges


def test_single_gpu_chunks():
    assert frame_chunks(13, 4) == [(0, 4), (4, 8), (8, 12), (12, 13)]
    assert frame_chunks(2, 4) == [(0, 2)] and frame_chunks(0, 4) == []
    for n in NS:
        for step in STEPS:
            assert _launch_frames_ranges(n, step) == frame_chunks(n, step)


def _init(rank, world, port):
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world,
                            timeout=datetime.timedelta(seconds=60))     # a rank left waiting fails instead of hanging
    torch.set_num_threads(1)
    return dist


def _shard_worker(rank, world, port):
    dist = _init(rank, world, port)
    for n in NS:
        for step in STEPS:
            x = _inputs(n)
            want = torch.empty(n, 3, 5, 7)
            launch_frame_chunks(x, want, step, _model_fn(x, want))
            got = torch.full_like(want, float("nan"))
            launched = []

            def launch(n0, n1, fn=_model_fn(x, got)):
                launched.append((n0, n1))
                fn(n0, n1)
            assert launch_frame_chunks(x, got, step, launch, dist.group.WORLD) is got
            assert torch.equal(got, want), (n, step)
            # this rank's launches through the engine's own chunking loop, then every rank's list
            mine = _launch_frames_ranges(n, step, dist.group.WORLD)
            assert mine == launched
            every = [None] * world
            dist.all_gather_object(every, mine)
            assert [r for ranks in every for r in ranks] == frame_chunks(n, step), (n, step, every)
            sizes = [len(r) for r in every]
            assert max(sizes) - min(sizes) <= 1, (n, step, every)          # balanced by chunk count
    dist.destroy_process_group()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_equals_unsharded(world):
    mp.spawn(_shard_worker, args=(world, _free_port()), nprocs=world, join=True)


MISMATCHES = ("frame", "n", "step", "dtype")


def _mismatch_worker(rank, world, port, out_dir):
    dist = _init(rank, world, port)
    for what in MISMATCHES:     # the agreement check completes its collective, so the group stays usable
        n, step, frame, dtype = 9, 4, (3, 5, 7), torch.float32
        if rank == world - 1:
            if what == "frame":
                frame = (3, 5, 8)
            elif what == "n":
                n = 10
            elif what == "step":
                step = 2
            else:
                dtype = torch.float64
        x = torch.randn(n, *frame, dtype=dtype)
        out = torch.empty_like(x)
        try:
            launch_frame_chunks(x, out, step, _model_fn(x, out), dist.group.WORLD)
            res = "returned"
        except ValueError as e:
            res = f"ValueError: {e}"
        with open(os.path.join(out_dir, f"{what}{rank}.txt"), "w") as fh:
            fh.write(res)
    dist.destroy_process_group()


def test_ranks_that_disagree_all_raise(tmp_path):
    world = 3
    mp.spawn(_mismatch_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    for what in MISMATCHES:
        res = [open(tmp_path / f"{what}{r}.txt").read() for r in range(world)]
        assert all(r.startswith("ValueError: the ranks of the process group made different") for r in res), (what, res)
        named = {"n": "rank 2: N=10 frames_per_call=4", "step": "rank 2: N=9 frames_per_call=2"}.get(what)
        if named:
            assert all(named in r for r in res), res
        else:
            assert all("shapes / dtypes not equal" in r for r in res), res
