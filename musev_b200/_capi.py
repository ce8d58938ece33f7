"""ctypes binding of include/musev_b200.h. There is no fallback: if the library is missing, loading raises.

Also the host side every whole-model wrapper shares (`EngineModel`): one engine handle, its weights by reference names,
the workspace and the launch, and the frame chunking of the per-frame models (`launch_frame_chunks`), on one GPU or
shared out over the ranks of a process group."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
from types import SimpleNamespace
from typing import Callable, Dict, Iterable, Optional, Sequence, Tuple

import torch
import torch.distributed as dist

from .build import LIB_PATH
from .context import assign_windows

_lib = None


class MvbError(RuntimeError):
    pass


class ConvGemmDesc(C.Structure):
    _fields_ = [
        ("a0", C.c_void_p), ("c0", C.c_int),
        ("a0_stride_w", C.c_longlong), ("a0_stride_h", C.c_longlong), ("a0_stride_n", C.c_longlong),
        ("a1", C.c_void_p), ("c1", C.c_int),
        ("a1_stride_w", C.c_longlong), ("a1_stride_h", C.c_longlong), ("a1_stride_n", C.c_longlong),
        ("W", C.c_int), ("H", C.c_int), ("NF", C.c_int),
        ("ntaps", C.c_int), ("dy", C.c_int8 * 9), ("dx", C.c_int8 * 9),
        ("weight", C.c_void_p), ("N", C.c_int),
        ("out", C.c_void_p), ("ldc", C.c_longlong),
        ("bias", C.c_void_p),
        ("rowadd", C.c_void_p), ("rows_per_group", C.c_int), ("ld_rowadd", C.c_int),
        ("residual", C.c_void_p), ("ld_res", C.c_longlong),
        ("alpha", C.c_float), ("beta", C.c_float),
        ("geglu", C.c_int), ("act", C.c_int), ("out_f32", C.c_int), ("stride2", C.c_int),
    ]


class AttentionDesc(C.Structure):
    _fields_ = [
        ("q", C.c_void_p), ("ldq", C.c_longlong),
        ("NF", C.c_int), ("Nq", C.c_int), ("heads", C.c_int), ("d", C.c_int), ("dp", C.c_int),
        ("scale", C.c_float), ("nseg", C.c_int),
        ("k", C.c_void_p * 2), ("v", C.c_void_p * 2), ("ldkv", C.c_longlong * 2), ("kv_rows", C.c_longlong * 2),
        ("nk", C.c_int * 2), ("fdiv", C.c_int * 2), ("fmul", C.c_longlong * 2), ("fadd", C.c_longlong * 2),
        ("out", C.c_void_p), ("ldo", C.c_longlong),
        ("out_scale", C.c_float), ("accumulate", C.c_int), ("v_ones_col", C.c_int), ("variant", C.c_int),
    ]


class MvbConfig(C.Structure):
    _fields_ = [
        ("in_channels", C.c_int), ("out_channels", C.c_int), ("num_blocks", C.c_int),
        ("block_out_channels", C.c_int * 4), ("layers_per_block", C.c_int), ("heads", C.c_int),
        ("cross_attention_dim", C.c_int), ("norm_num_groups", C.c_int), ("norm_eps", C.c_float),
        ("need_transformer_in", C.c_int), ("use_anivv1_cfg", C.c_int), ("resnet_2d_skip_time_act", C.c_int),
        ("keep_vision_condtion", C.c_int), ("need_refer_emb", C.c_int), ("ip_adapter_cross_attn", C.c_int),
        ("need_t2i_ip_adapter", C.c_int),
    ]


MAX_REFER = 16


class MvbUnetArgs(C.Structure):
    _fields_ = [
        ("sample", C.c_void_p), ("sample_is_f32", C.c_int),
        ("B", C.c_int), ("T", C.c_int), ("H", C.c_int), ("W", C.c_int),
        ("timestep", C.c_float),
        ("encoder_hidden_states", C.c_void_p), ("ehs_is_f32", C.c_int), ("n_text", C.c_int),
        ("has_sample_index", C.c_int),
        ("n_vis_cond", C.c_int), ("vis_cond_first", C.c_int),
        ("sample_frame_rate", C.c_float),
        ("vision_clip_emb", C.c_void_p), ("clip_is_f32", C.c_int), ("n_clip", C.c_int), ("ip_adapter_scale", C.c_float),
        ("n_refer", C.c_int),
        ("refer_embs", C.c_void_p * MAX_REFER), ("refer_t", C.c_int * MAX_REFER), ("refer_h", C.c_int * MAX_REFER),
        ("refer_w", C.c_int * MAX_REFER),
        ("mid_refer_emb", C.c_void_p), ("mid_refer_t", C.c_int), ("mid_refer_h", C.c_int), ("mid_refer_w", C.c_int),
        ("refer_is_f32", C.c_int),
        ("n_down_residuals", C.c_int), ("cfg_shared_sample", C.c_int), ("down_residuals", C.c_void_p * MAX_REFER),
        ("mid_residual", C.c_void_p), ("residual_is_f32", C.c_int),
        ("skip_temporal_layers", C.c_int),
        ("out", C.c_void_p), ("out_is_f32", C.c_int),
        ("pose_guider_emb", C.c_void_p), ("pose_is_f32", C.c_int),
    ]


class MvbNamedTensor(C.Structure):
    _fields_ = [("name", C.c_char_p), ("device_ptr", C.c_void_p), ("is_f32", C.c_int), ("ndim", C.c_int),
                ("shape", C.c_longlong * 5)]


MAX_OUT = 13


class MvbControlnetArgs(C.Structure):
    _fields_ = [
        ("sample", C.c_void_p), ("sample_is_f32", C.c_int),
        ("NF", C.c_int), ("H", C.c_int), ("W", C.c_int),
        ("timestep", C.c_float),
        ("encoder_hidden_states", C.c_void_p), ("ehs_is_f32", C.c_int), ("n_text", C.c_int),
        ("cond_latents", C.c_void_p), ("cond_is_f32", C.c_int),
        ("n_out", C.c_int),
        ("scales", C.c_float * MAX_OUT),
        ("outs", C.c_void_p * MAX_OUT),
        ("out_is_f32", C.c_int),
        ("out_frames", C.c_int),
        ("accumulate", C.c_int),
    ]


class MvbVaeDecodeArgs(C.Structure):
    _fields_ = [("latents", C.c_void_p), ("latents_is_f32", C.c_int), ("N", C.c_int), ("h", C.c_int), ("w", C.c_int),
                ("latent_scale", C.c_float), ("out", C.c_void_p), ("out_is_f32", C.c_int), ("postprocess", C.c_int)]


VAE_TILE_CLASSES = 4


class MvbVaeTileBlendArgs(C.Structure):
    _fields_ = [
        ("tiles", C.c_void_p * (VAE_TILE_CLASSES * VAE_TILE_CLASSES)), ("tiles_is_f32", C.c_int), ("N", C.c_int),
        ("C", C.c_int),
        ("n_row_classes", C.c_int), ("row_count", C.c_int * VAE_TILE_CLASSES), ("row_size", C.c_int * VAE_TILE_CLASSES),
        ("n_col_classes", C.c_int), ("col_count", C.c_int * VAE_TILE_CLASSES), ("col_size", C.c_int * VAE_TILE_CLASSES),
        ("extent", C.c_int), ("row_limit", C.c_int), ("H", C.c_int), ("W", C.c_int), ("mode", C.c_int),
        ("scale", C.c_float), ("out", C.c_void_p), ("out_is_f32", C.c_int),
    ]


class MvbMultistepArgs(C.Structure):
    _fields_ = [
        ("eps_sum", C.c_void_p), ("counter", C.c_void_p), ("latents_in", C.c_void_p), ("latents_out", C.c_void_p),
        ("m1", C.c_void_p), ("m2", C.c_void_p), ("noise", C.c_void_p), ("m0_out", C.c_void_p),
        ("is_f32", C.c_int), ("B", C.c_int), ("C", C.c_int), ("T", C.c_int), ("HW", C.c_int), ("cfg", C.c_int),
        ("guidance_scale", C.c_float), ("a_x", C.c_float), ("a_e", C.c_float), ("clip", C.c_float),
        ("c_x", C.c_float), ("c0", C.c_float), ("c1", C.c_float), ("c2", C.c_float), ("c_n", C.c_float),
    ]


def lib() -> C.CDLL:
    """Load libmusevb200.so (built in-tree by musev_b200.build). Raises if it is not there."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise MvbError(
                f"{LIB_PATH} not found: build it with `python -m musev_b200.build` "
                "(musev_b200 has no CPU or PyTorch fallback)")
        l = C.CDLL(LIB_PATH)
        _declare(l)
        _lib = l
    return _lib


def _declare(l: C.CDLL) -> None:
    def fn(name, restype, *argtypes):
        f = getattr(l, name)
        f.restype, f.argtypes = restype, list(argtypes)

    l.mvb_last_error.restype = C.c_char_p
    l.mvb_version.restype = C.c_int
    l.mvb_op_conv_gemm.argtypes = [C.POINTER(ConvGemmDesc), C.c_void_p]
    l.mvb_op_conv_gemm.restype = C.c_int
    l.mvb_op_small_conv.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                    C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    l.mvb_op_small_conv.restype = C.c_int
    for att in ("mvb_op_attention", "mvb_op_attention_causal"):
        fn(att, C.c_int, C.POINTER(AttentionDesc), C.c_void_p)
    l.mvb_debug_attention_trace.argtypes = [C.c_void_p]
    l.mvb_debug_attention_trace.restype = C.c_int
    l.mvb_tensor_map_cache_stats.argtypes = [C.POINTER(C.c_ulonglong), C.POINTER(C.c_ulonglong)]
    l.mvb_tensor_map_cache_stats.restype = C.c_int
    l.mvb_op_temporal_attention.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                            C.c_float, C.c_void_p, C.c_int, C.c_void_p]
    l.mvb_op_temporal_attention.restype = C.c_int
    l.mvb_op_groupnorm.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                   C.c_float, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    l.mvb_op_groupnorm.restype = C.c_int
    l.mvb_op_groupnorm_fused.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                         C.c_float, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.POINTER(C.c_uint), C.c_void_p]
    l.mvb_op_groupnorm_fused.restype = C.c_int
    l.mvb_op_layernorm.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_void_p]
    l.mvb_op_layernorm.restype = C.c_int
    fn("mvb_op_softmax_rows", C.c_int, C.c_void_p, C.c_longlong, C.c_int, C.c_longlong, C.c_float, C.c_void_p)
    l.mvb_fuse_cfg_ddim.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                    C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_int, C.c_float, C.c_int,
                                    C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    l.mvb_fuse_cfg_ddim.restype = C.c_int
    l.mvb_fuse_cfg_affine.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                      C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, C.c_void_p, C.c_float,
                                      C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]
    l.mvb_fuse_cfg_affine.restype = C.c_int
    fn("mvb_fuse_cfg_multistep", C.c_int, C.POINTER(MvbMultistepArgs), C.c_void_p)
    l.mvb_accumulate_window.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                        C.c_int, C.c_void_p, C.c_int, C.c_void_p]
    l.mvb_accumulate_window.restype = C.c_int
    fn("mvb_op_hist_match_workspace_bytes", C.c_longlong, *[C.c_int] * 7)
    fn("mvb_op_hist_match", C.c_int, C.c_void_p, *[C.c_int] * 5, *[C.c_longlong] * 3, C.c_void_p, C.c_int, C.c_int,
       C.c_longlong, C.c_longlong, C.c_void_p, *[C.c_longlong] * 3, C.c_void_p, C.c_longlong, C.c_void_p)
    fn("mvb_op_vae_tile_blend", C.c_int, C.POINTER(MvbVaeTileBlendArgs), C.c_void_p)
    l.mvb_launch_count.argtypes = [C.c_int]
    l.mvb_launch_count.restype = C.c_longlong
    l.mvb_profile_enable.argtypes = [C.c_int]
    l.mvb_profile_enable.restype = None
    l.mvb_profile_collect.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_longlong)]
    l.mvb_profile_collect.restype = C.c_int
    # whole-model handles
    H, I, LL, P = C.c_void_p, C.c_int, C.c_longlong, C.POINTER
    for create in ("mvb_create", "mvb_create_controlnet", "mvb_create_referencenet", "mvb_create_vae_decoder",
                   "mvb_create_vae_encoder", "mvb_create_pose_guider", "mvb_create_clip_vision",
                   "mvb_create_clip_text"):
        fn(create, I, P(MvbConfig), I, P(C.c_void_p))
    fn("mvb_destroy", None, H)
    fn("mvb_load_weight", I, H, C.c_char_p, C.c_void_p, I, P(LL), I)
    fn("mvb_load_weights", I, H, P(MvbNamedTensor), I)
    fn("mvb_finalize", I, H)
    fn("mvb_num_params", I, H)
    fn("mvb_handle_error", C.c_char_p, H)
    fn("mvb_debug_num_taps", I, H)
    fn("mvb_debug_tap", I, H, I, C.c_char_p, I, P(C.c_void_p), P(LL), P(I))
    fn("mvb_unet_merge_lora", I, H, P(MvbNamedTensor), P(MvbNamedTensor), P(C.c_float), I, I)
    fn("mvb_debug_read_weight", I, H, C.c_char_p, C.c_void_p)
    for ws, run, args in (("mvb_workspace_bytes", "mvb_unet_forward", MvbUnetArgs),
                          ("mvb_controlnet_workspace_bytes", "mvb_controlnet_forward", MvbControlnetArgs),
                          ("mvb_referencenet_workspace_bytes", "mvb_referencenet_forward", MvbControlnetArgs),
                          ("mvb_vae_decode_workspace_bytes", "mvb_vae_decode", MvbVaeDecodeArgs),
                          ("mvb_vae_encode_workspace_bytes", "mvb_vae_encode", MvbVaeDecodeArgs),
                          ("mvb_pose_guider_workspace_bytes", "mvb_pose_guider_forward", MvbVaeDecodeArgs),
                          ("mvb_clip_vision_workspace_bytes", "mvb_clip_vision_forward", MvbControlnetArgs),
                          ("mvb_clip_text_workspace_bytes", "mvb_clip_text_forward", MvbControlnetArgs)):
        fn(ws, LL, H, P(args))
        fn(run, I, H, P(args), C.c_void_p, LL, C.c_void_p)


def check(rc: int) -> None:
    if rc != 0:
        raise MvbError(f"musev_b200 error {rc}: {lib().mvb_last_error().decode()}")


CATEGORIES = ("gemm", "attention", "temporal_attention", "groupnorm", "layernorm", "other")


def launch_count(category: int = -1) -> int:
    return int(lib().mvb_launch_count(category))


def profile_enable(on: bool) -> None:
    lib().mvb_profile_enable(int(on))


def tensor_map_cache_stats():
    """(hits, misses) of the process-wide memo of encoded TMA descriptors."""
    h, m = C.c_ulonglong(0), C.c_ulonglong(0)
    check(lib().mvb_tensor_map_cache_stats(C.byref(h), C.byref(m)))
    return int(h.value), int(m.value)


def profile_collect():
    ms = (C.c_double * 6)()
    n = (C.c_longlong * 6)()
    check(lib().mvb_profile_collect(ms, n))
    return {c: dict(ms=ms[i], launches=int(n[i])) for i, c in enumerate(CATEGORIES)}


def _is_f32(t: torch.Tensor) -> int:
    if t.dtype == torch.float32:
        return 1
    if t.dtype == torch.float16:
        return 0
    raise ValueError(f"musev_b200 takes float16 or float32 tensors, got {t.dtype}")


def _named(name: str, t: torch.Tensor) -> MvbNamedTensor:
    e = MvbNamedTensor()
    e.name, e.device_ptr, e.is_f32, e.ndim = name.encode(), t.data_ptr(), _is_f32(t), t.dim()
    for i, v in enumerate(t.shape):
        e.shape[i] = v
    return e


PACK_BATCH_BYTES = 512 << 20     # source bytes staged on the device per mvb_load_weights call


def load_weights_batched(handle, named_tensors: Iterable[Tuple[str, torch.Tensor]], device) -> None:
    """Feeds (name, tensor) pairs to `mvb_load_weights` in batches of ~PACK_BATCH_BYTES: one host->device staging copy
    per tensor, ONE packing kernel per batch."""
    l = lib()
    batch, keep, nbytes = [], [], 0

    def flush():
        nonlocal batch, keep, nbytes
        if not batch:
            return
        arr = (MvbNamedTensor * len(batch))(*batch)
        rc = l.mvb_load_weights(handle, arr, len(batch))
        if rc != 0:
            raise MvbError(f"mvb_load_weights: {l.mvb_handle_error(handle).decode()}")
        batch, keep, nbytes = [], [], 0

    for name, t in named_tensors:
        if t.dtype not in (torch.float16, torch.float32):
            t = t.float()
        t = t.to(device).contiguous()
        batch.append(_named(name, t))
        keep.append(t)
        nbytes += t.numel() * t.element_size()
        if nbytes >= PACK_BATCH_BYTES:
            torch.cuda.current_stream(device).synchronize()
            flush()
    torch.cuda.current_stream(device).synchronize()
    flush()


def make_config(in_channels: int, out_channels: int, block_out_channels: Sequence[int], layers_per_block: int = 0,
                heads: int = 0, cross_attention_dim: int = 0, norm_num_groups: int = 0, norm_eps: float = 0.0,
                **switches) -> MvbConfig:
    """An `mvb_config`; `switches` are the int flags of the UNet (`need_transformer_in`, ...)."""
    c = MvbConfig()
    c.in_channels, c.out_channels, c.num_blocks = in_channels, out_channels, len(block_out_channels)
    for i, v in enumerate(block_out_channels):
        c.block_out_channels[i] = v
    c.layers_per_block, c.heads = layers_per_block, heads
    c.cross_attention_dim, c.norm_num_groups, c.norm_eps = cross_attention_dim, norm_num_groups, norm_eps
    for k, v in switches.items():
        setattr(c, k, int(v))
    return c


def frame_chunks(n: int, step: int) -> list:
    """The launches of one frame-chunked call: [(0, step), (step, 2 step), ...], the last one possibly short."""
    return [(n0, min(n0 + step, n)) for n0 in range(0, n, step)]


def _check_same_call(x: torch.Tensor, out: torch.Tensor, step: int, group) -> None:
    """All-gathers (N, step, digest of the per-frame shapes and dtypes) over the group and raises ValueError on every rank
    when any rank's call differs, so that no rank enters a row exchange the others would never join."""
    desc = f"per-frame input {list(x.shape[1:])} {x.dtype} -> output {list(out.shape[1:])} {out.dtype}"
    digest = int.from_bytes(hashlib.blake2b(desc.encode(), digest_size=8).digest(), "little", signed=True)
    # NCCL exchanges device tensors only; the other backends take host tensors
    dev = out.device if dist.get_backend(group) == dist.Backend.NCCL else torch.device("cpu")
    mine = torch.tensor([x.shape[0], step, digest], dtype=torch.int64, device=dev)
    keys = [torch.empty_like(mine) for _ in range(dist.get_world_size(group))]
    dist.all_gather(keys, mine, group=group)
    keys = [tuple(k.tolist()) for k in keys]
    if len(set(keys)) > 1:
        per_rank = ", ".join(f"rank {r}: N={k[0]} frames_per_call={k[1]}" for r, k in enumerate(keys))
        same = "equal" if len({k[2] for k in keys}) == 1 else "not equal"
        raise ValueError(f"the ranks of the process group made different frame-sharded calls ({per_rank}; per-frame "
                         f"shapes / dtypes {same}); this rank: {desc}. Every rank must make the same call")


def launch_frame_chunks(x: torch.Tensor, out: torch.Tensor, step: int, launch: Callable[[int, int], None],
                        process_group=None) -> torch.Tensor:
    """Runs `launch(n0, n1)` over the `frame_chunks(N, step)` of a per-frame model call x [N, ...] -> out [N, ...];
    `launch` writes out[n0:n1].

    process_group None: every chunk, in order, on this device. With a `torch.distributed` group the same chunks are
    handed to its ranks as contiguous, balanced ranges (a rank may get none); each rank launches its own chunks exactly
    as a single GPU would, so every frame gets bit-identical arithmetic, and then each rank broadcasts its rows of `out`
    into the others' `out` on the device. Every rank returns the full `out`. Every rank must make the same call: the
    ranks first compare N, `step` and the per-frame shapes and dtypes, and all raise ValueError on a mismatch."""
    chunks = frame_chunks(x.shape[0], step)
    if process_group is None:
        for n0, n1 in chunks:
            launch(n0, n1)
        return out
    _check_same_call(x, out, step, process_group)
    per_rank = assign_windows([1] * len(chunks), dist.get_world_size(process_group))
    for i in per_rank[dist.get_rank(process_group)]:
        launch(*chunks[i])
    for r, mine in enumerate(per_rank):
        if mine:     # every rank knows the partition, so all skip an idle rank's empty range alike
            rows = out[chunks[mine[0]][0]:chunks[mine[-1]][1]]
            dist.broadcast(rows, src=dist.get_global_rank(process_group, r), group=process_group)
    return out


class EngineModel:
    """One engine handle behind a reference model's call surface: creation, weights by reference state-dict names,
    `.eval()`, `.to()`, and the grow-only workspace every call runs in. A subclass names its C entry points and
    gives the expected parameter shapes."""

    _create = ""              # mvb_create_* of the model kind
    _workspace = ""           # its *_workspace_bytes
    _forward = ""             # its forward
    _ignored: Tuple[str, ...] = ()   # state-dict prefixes of other models, skipped by load_state_dict

    def __init__(self, config: MvbConfig, device, dtype: torch.dtype, unsupported: str = "unsupported configuration"):
        if not torch.cuda.is_available():
            raise RuntimeError("musev_b200 needs a CUDA (sm_90a) device; there is no CPU path")
        self.device = torch.device(device if str(device) != "cuda" else f"cuda:{torch.cuda.current_device()}")
        self.dtype = dtype
        self._ws: Optional[torch.Tensor] = None
        self._h = C.c_void_p()
        self._loaded = False
        rc = getattr(lib(), self._create)(C.byref(config), self.device.index or 0, C.byref(self._h))
        if rc != 0:
            raise MvbError(f"{self._create} failed ({rc}): {unsupported} or out of device memory")

    def _error(self) -> str:
        return lib().mvb_handle_error(self._h).decode()

    def _param_shapes(self) -> Dict[str, Tuple[int, ...]]:
        raise NotImplementedError

    def load_state_dict(self, state_dict: Dict[str, torch.Tensor], strict: bool = True):
        """Checks names and shapes against the schema, then packs the tensors on the device in batches (peak extra memory
        = one ~512 MB staging batch)."""
        expected = self._param_shapes()
        missing = [k for k in expected if k not in state_dict]
        unexpected = [k for k in state_dict if k not in expected and not k.startswith(self._ignored)]
        if strict and (missing or unexpected):
            raise RuntimeError(f"Error(s) in loading state_dict: missing {missing[:5]} unexpected {unexpected[:5]}")
        todo = []
        for name, shape in expected.items():
            if name not in state_dict:
                continue
            t = state_dict[name]
            if tuple(t.shape) != tuple(shape):
                raise RuntimeError(f"size mismatch for {name}: {tuple(t.shape)} vs {tuple(shape)}")
            todo.append((name, t))
        self._load(todo)
        return SimpleNamespace(missing_keys=missing, unexpected_keys=unexpected)

    def _load(self, todo: Sequence[Tuple[str, torch.Tensor]]) -> None:
        load_weights_batched(self._h, todo, self.device)
        if lib().mvb_finalize(self._h) != 0:
            raise MvbError(f"mvb_finalize: {self._error()}")
        self._loaded = True

    def _check_loaded(self) -> None:
        if not self._loaded:
            raise RuntimeError("weights not loaded: call load_state_dict first")

    def __del__(self):
        try:
            if getattr(self, "_h", None) and self._h.value:
                lib().mvb_destroy(self._h)
                self._h = C.c_void_p()
        except Exception:
            pass

    def eval(self):
        return self

    def to(self, *args, **kwargs):
        for a in list(args) + list(kwargs.values()):
            if isinstance(a, torch.dtype):
                if a not in (torch.float16, torch.float32):
                    raise ValueError("musev_b200 computes in fp16 with fp32 accumulation; I/O dtype is fp16 or fp32")
                self.dtype = a
            elif isinstance(a, (str, torch.device)) and torch.device(a).type != "cuda":
                raise RuntimeError("musev_b200 has no CPU path")
        return self

    def _launch(self, args: C.Structure) -> None:
        """One forward on the current stream of the model's device, in the handle's workspace (grown when too small)."""
        l = lib()
        need = getattr(l, self._workspace)(self._h, C.byref(args))
        if need < 0:
            raise MvbError(f"{self._workspace}: {self._error()}")
        if self._ws is None or self._ws.numel() < need:
            self._ws = None
            self._ws = torch.empty(int(need), dtype=torch.uint8, device=self.device)
        rc = getattr(l, self._forward)(self._h, C.byref(args), self._ws.data_ptr(), self._ws.numel(),
                                       torch.cuda.current_stream(self.device).cuda_stream)
        if rc != 0:
            raise MvbError(f"{self._forward} ({rc}): {self._error()}")

    def _launch_frames(self, x: torch.Tensor, out: torch.Tensor, h: int, w: int, latent_scale: float,
                       postprocess: int, process_group=None) -> torch.Tensor:
        """Runs an `mvb_vae_decode_args` model on x [N, ...] -> out [N, ...] in chunks of `frames_per_call` frames (bounds
        the activation workspace); h, w = the size the model's entry point documents. With a process group the chunks
        are shared out over its ranks and every rank returns the full output (`launch_frame_chunks`)."""
        def launch(n0: int, n1: int) -> None:
            xc, oc = x[n0:n1], out[n0:n1]
            a = MvbVaeDecodeArgs()
            a.latents, a.latents_is_f32 = xc.data_ptr(), _is_f32(xc)
            a.N, a.h, a.w = xc.shape[0], h, w
            a.latent_scale = float(latent_scale)
            a.out, a.out_is_f32 = oc.data_ptr(), _is_f32(oc)
            a.postprocess = int(postprocess)
            self._launch(a)

        launch_frame_chunks(x, out, max(1, self.frames_per_call), launch, process_group)
        self._keep = x   # the input must outlive the asynchronous launches
        return out

    def _merge_lora(self, targets: Sequence[str], ups: Sequence[torch.Tensor], downs: Sequence[torch.Tensor],
                    scales: Sequence[float], subtract: bool = False) -> None:
        """W16 = fp16(W16 +- fp16(scale * (up @ down))) for every target (reference weight names), one `mvb_unet_merge_lora`
        call (UNet and CLIP text encoder handles). The factors must be contiguous fp16 / fp32 tensors on this model's device."""
        n = len(targets)
        if not (len(ups) == len(downs) == len(scales) == n):
            raise ValueError("targets, ups, downs and scales differ in length")
        for t in list(ups) + list(downs):
            if t.device != self.device or not t.is_contiguous():
                raise ValueError(f"LoRA factors must be contiguous tensors on {self.device}")
        up_arr = (MvbNamedTensor * max(n, 1))(*[_named(nm, u) for nm, u in zip(targets, ups)])
        down_arr = (MvbNamedTensor * max(n, 1))(*[_named(nm, d) for nm, d in zip(targets, downs)])
        sc = (C.c_float * max(n, 1))(*[float(s) for s in scales])
        torch.cuda.current_stream(self.device).synchronize()      # the factors may still be in flight
        rc = lib().mvb_unet_merge_lora(self._h, up_arr, down_arr, sc, n, int(bool(subtract)))
        if rc != 0:
            raise MvbError(f"mvb_unet_merge_lora ({rc}): {self._error()}")

    def debug_weight(self, name: str) -> torch.Tensor:
        """The packed matrix / convolution weight `name` read back into its reference shape, fp16 on the device."""
        shape = self._param_shapes().get(name)
        if shape is None or len(shape) < 2:
            raise ValueError(f"{name} is not a matrix or convolution weight of this model")
        out = torch.empty(shape, dtype=torch.float16, device=self.device)
        rc = lib().mvb_debug_read_weight(self._h, name.encode(), out.data_ptr())
        if rc != 0:
            raise MvbError(f"mvb_debug_read_weight ({rc}): {self._error()}")
        return out
