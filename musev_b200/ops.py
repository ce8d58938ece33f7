"""Torch-tensor front ends of the op-level C ABI (device pointers + strides are taken from the tensors).

These are thin argument marshalling helpers used by the per-op parity tests; the whole UNet forward runs
inside the library (musev_b200.engine) and does not go through Python per layer.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence, Tuple

import torch

from . import _capi


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


TAPS_1 = ((0, 0),)
TAPS_3X3 = tuple((dy, dx) for dy in (-1, 0, 1) for dx in (-1, 0, 1))
TAPS_T3 = ((-1, 0), (0, 0), (1, 0))


def conv_gemm(
    a0: torch.Tensor,                      # [NF, H, W, C0] fp16 (any strides with unit channel stride)
    weight: torch.Tensor,                  # [N, ntaps*(C0+C1)] fp16 contiguous
    taps: Sequence[Tuple[int, int]] = TAPS_1,
    a1: Optional[torch.Tensor] = None,
    bias: Optional[torch.Tensor] = None,   # fp32 [N]
    rowadd: Optional[torch.Tensor] = None, # fp32 [groups, N]
    rows_per_group: int = 1,
    residual: Optional[torch.Tensor] = None,  # fp16 [M, Nout]
    alpha: float = 1.0,
    beta: float = 1.0,
    geglu: bool = False,
    act: int = 0,
    out: Optional[torch.Tensor] = None,
    out_f32: bool = False,
    stride2: int = 0,                      # 3x3 stride-2 conv: 1 (or True) pad 1 on every side, 2 pad (0, 1, 0, 1)
) -> torch.Tensor:
    assert a0.dtype == torch.float16 and weight.dtype == torch.float16 and a0.dim() == 4
    assert a0.stride(3) == 1 and weight.is_contiguous()
    NF, H, W, C0 = a0.shape
    N = weight.shape[0]
    nout = N // 2 if geglu else N
    M = NF * H * W if not stride2 else NF * (H // 2) * (W // 2)
    if out is None:
        out = torch.empty((M, nout), dtype=torch.float32 if out_f32 else torch.float16, device=a0.device)
    d = _capi.ConvGemmDesc()
    d.a0, d.c0 = a0.data_ptr(), C0
    d.a0_stride_w, d.a0_stride_h, d.a0_stride_n = a0.stride(2), a0.stride(1), a0.stride(0)
    if a1 is not None:
        assert a1.shape[:3] == a0.shape[:3] and a1.stride(3) == 1 and a1.dtype == torch.float16
        d.a1, d.c1 = a1.data_ptr(), a1.shape[3]
        d.a1_stride_w, d.a1_stride_h, d.a1_stride_n = a1.stride(2), a1.stride(1), a1.stride(0)
    d.W, d.H, d.NF = W, H, NF
    d.ntaps = len(taps)
    for i, (dy, dx) in enumerate(taps):
        d.dy[i], d.dx[i] = dy, dx
    if stride2:
        assert weight.shape[1] == 9 * C0
    else:
        assert weight.shape[1] == len(taps) * (C0 + (a1.shape[3] if a1 is not None else 0))
    d.weight, d.N = weight.data_ptr(), N
    d.out, d.ldc = out.data_ptr(), out.stride(0)
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.numel() == N
        d.bias = bias.data_ptr()
    if rowadd is not None:
        assert rowadd.dtype == torch.float32 and rowadd.shape[1] == N
        d.rowadd, d.rows_per_group, d.ld_rowadd = rowadd.data_ptr(), rows_per_group, rowadd.stride(0)
    else:
        d.rows_per_group = 1
    if residual is not None:
        assert residual.dtype == torch.float16
        d.residual, d.ld_res = residual.data_ptr(), residual.stride(0)
    d.alpha, d.beta, d.geglu, d.act = alpha, beta, int(geglu), act
    d.out_f32, d.stride2 = int(out_f32), int(stride2)
    _capi.check(_capi.lib().mvb_op_conv_gemm(C.byref(d), _stream()))
    return out


def small_conv(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor], stride: int = 1, act: bool = True,
               nchw: bool = False) -> torch.Tensor:
    """3x3 conv (pad 1) + bias + SiLU on the small-channel kernel. x: channels-last fp16 [NF, H, W, cin] (cin 16 / 32) or,
    with nchw, an image [NF, cin <= 3, H, W] fp16 / fp32; weight: packed fp16 [cout, 9 cin] (nchw: [cout, 32]), column
    tap * cin + c. Returns channels-last fp16 [NF, H / stride, W / stride, cout]."""
    if nchw:
        NF, cin, H, W = x.shape
    else:
        NF, H, W, cin = x.shape
    cout = weight.shape[0]
    out = torch.empty(NF, (H - 1) // stride + 1, (W - 1) // stride + 1, cout, dtype=torch.float16, device=x.device)
    _capi.check(_capi.lib().mvb_op_small_conv(_ptr(x), int(x.dtype == torch.float32), int(nchw), cin, H, W, NF, stride,
                                              _ptr(weight), _ptr(bias), cout, int(act), _ptr(out), _stream()))
    return out


def attention(q, segs, NF, Nq, heads, d, dp, scale, out=None, out_scale=1.0, accumulate=False, v_ones_col=False, variant=0,
              causal=False):
    """q: [NF*Nq, >=heads*dp] fp16 (row stride taken from the tensor); segs: list of dicts
    {k, v, nk, fdiv, fmul, fadd} with k/v [rows, >=heads*dp] views sharing a row stride. causal=True masks key k of a
    sequence from query q unless k <= q (`mvb_op_attention_causal`; one segment of the queries' own sequence only)."""
    assert q.dtype == torch.float16 and q.stride(1) == 1
    if out is None:
        out = torch.zeros((NF * Nq, heads * d), dtype=torch.float16, device=q.device)
    a = _capi.AttentionDesc()
    a.q, a.ldq = q.data_ptr(), q.stride(0)
    a.NF, a.Nq, a.heads, a.d, a.dp, a.scale, a.nseg = NF, Nq, heads, d, dp, scale, len(segs)
    for i, s in enumerate(segs):
        k, v = s["k"], s["v"]
        assert k.dtype == torch.float16 and v.dtype == torch.float16 and k.stride(0) == v.stride(0)
        a.k[i], a.v[i], a.ldkv[i], a.kv_rows[i] = k.data_ptr(), v.data_ptr(), k.stride(0), k.shape[0]
        a.nk[i], a.fdiv[i], a.fmul[i], a.fadd[i] = s["nk"], s.get("fdiv", 1), s.get("fmul", s["nk"]), s.get("fadd", 0)
    a.out, a.ldo, a.out_scale, a.accumulate = out.data_ptr(), out.stride(0), out_scale, int(accumulate)
    a.v_ones_col = int(v_ones_col)
    a.variant = int(variant)
    op = _capi.lib().mvb_op_attention_causal if causal else _capi.lib().mvb_op_attention
    _capi.check(op(C.byref(a), _stream()))
    return out


def temporal_attention(qkv, B, T, HW, heads, d, dp, scale):
    assert qkv.dtype == torch.float16 and qkv.is_contiguous()
    out = torch.empty((B * T * HW, heads * d), dtype=torch.float16, device=qkv.device)
    _capi.check(_capi.lib().mvb_op_temporal_attention(qkv.data_ptr(), qkv.shape[-1], B, T, HW, heads, d, dp, scale,
                                                      out.data_ptr(), out.shape[-1], _stream()))
    return out


_gn_barrier = {}     # device -> (zeroed uint32 tensor, ctypes arrival counter) of the one-launch GroupNorm


def groupnorm(x0, gamma, beta, groups=32, frames_per_stat=1, eps=1e-5, silu=False, x1=None, fused=False):
    """x0 [NF, HW, C0] fp16 (+ x1 [NF, HW, C1]); gamma/beta fp32 [C0+C1]. fused=True: the one-launch kernel the engine uses."""
    assert x0.dtype == torch.float16 and x0.is_contiguous() and (x1 is None or (x1.dtype == torch.float16 and x1.is_contiguous()))
    assert gamma.dtype == torch.float32 and beta.dtype == torch.float32
    NF, HW, C0 = x0.shape
    C1 = 0 if x1 is None else x1.shape[2]
    y = torch.empty((NF, HW, C0 + C1), dtype=torch.float16, device=x0.device)
    scratch = torch.empty(NF * 65 * groups * 2, dtype=torch.float32, device=x0.device)
    if fused:
        key = x0.device.index or 0
        if key not in _gn_barrier:
            _gn_barrier[key] = (torch.zeros(1, dtype=torch.int32, device=x0.device), C.c_uint(0))
        word, arrivals = _gn_barrier[key]
        _capi.check(_capi.lib().mvb_op_groupnorm_fused(x0.data_ptr(), C0, _ptr(x1), C1, NF, HW, groups, frames_per_stat, eps,
                                                       gamma.data_ptr(), beta.data_ptr(), int(silu), y.data_ptr(),
                                                       scratch.data_ptr(), word.data_ptr(), C.byref(arrivals), _stream()))
        return y
    _capi.check(_capi.lib().mvb_op_groupnorm(x0.data_ptr(), C0, _ptr(x1), C1, NF, HW, groups, frames_per_stat, eps,
                                             gamma.data_ptr(), beta.data_ptr(), int(silu), y.data_ptr(),
                                             scratch.data_ptr(), _stream()))
    return y


def layernorm(x, gamma, beta, eps):
    assert x.dtype == torch.float16 and x.is_contiguous() and gamma.dtype == torch.float32 and beta.dtype == torch.float32
    M, Cc = x.shape
    y = torch.empty_like(x)
    _capi.check(_capi.lib().mvb_op_layernorm(x.data_ptr(), M, Cc, eps, gamma.data_ptr(), beta.data_ptr(), y.data_ptr(),
                                             _stream()))
    return y


def softmax_rows(x, scale=1.0, N=None):
    """In place: the first N columns (default all) of every row of x [M, ld] fp16 become softmax(scale * row); the
    columns past N are left as they are. Returns x."""
    assert x.dtype == torch.float16 and x.dim() == 2 and x.stride(1) == 1
    M, ld = x.shape[0], x.stride(0)
    N = x.shape[1] if N is None else N
    assert N <= x.shape[1]
    _capi.check(_capi.lib().mvb_op_softmax_rows(x.data_ptr(), M, N, ld, scale, _stream()))
    return x


def fuse_cfg_ddim(eps_sum, counter, latents, guidance, alpha_t, alpha_prev, prediction_type=0, clip_range=0.0,
                  out=None, eps_out=None, cfg=True, use_clipped=False, std_dev=0.0, noise=None, x0_out=None):
    """eps_sum fp32 [2B,C,T,H,W] (cfg) or [B,C,T,H,W]; counter fp32 [T] or None; latents fp32/fp16 [B,C,T,H,W]."""
    B, Cc, T = latents.shape[:3]
    HW = latents.shape[3] * latents.shape[4]
    assert eps_sum.dtype == torch.float32 and eps_sum.is_contiguous() and latents.is_contiguous()
    assert eps_sum.numel() == latents.numel() * (2 if cfg else 1), "eps_sum must be [2B,...] with cfg, [B,...] without"
    assert latents.dtype in (torch.float16, torch.float32), f"latents must be fp16 or fp32, got {latents.dtype}"
    assert counter is None or (counter.dtype == torch.float32 and counter.is_contiguous() and counter.numel() == T)
    for t_ in (noise, eps_out, x0_out):
        assert t_ is None or (t_.dtype == torch.float32 and t_.is_contiguous() and t_.numel() == latents.numel())
    if out is None:
        out = torch.empty_like(latents)
    _capi.check(_capi.lib().mvb_fuse_cfg_ddim(
        eps_sum.data_ptr(), _ptr(counter), latents.data_ptr(), out.data_ptr(), int(latents.dtype == torch.float32),
        B, Cc, T, HW, int(cfg), guidance, alpha_t, alpha_prev, prediction_type, clip_range, int(use_clipped),
        std_dev, _ptr(noise), _ptr(eps_out), _ptr(x0_out), _stream()))
    return out


def fuse_cfg_affine(eps_sum, counter, latents, guidance, c_x, c_e, c_n=0.0, noise=None, a_x=0.0, a_e=0.0, aux_out=None,
                    eps_out=None, cfg=True, out=None):
    """x_prev = c_x x + c_e eps + c_n noise (eps = overlap mean + CFG of eps_sum); aux_out = a_x x + a_e eps."""
    B, Cc, T = latents.shape[:3]
    HW = latents.shape[3] * latents.shape[4]
    assert eps_sum.dtype == torch.float32 and eps_sum.is_contiguous() and latents.is_contiguous()
    assert eps_sum.numel() == latents.numel() * (2 if cfg else 1), "eps_sum must be [2B,...] with cfg, [B,...] without"
    assert latents.dtype in (torch.float16, torch.float32), f"latents must be fp16 or fp32, got {latents.dtype}"
    assert counter is None or (counter.dtype == torch.float32 and counter.is_contiguous() and counter.numel() == T)
    for t_ in (noise, aux_out, eps_out):
        assert t_ is None or (t_.dtype == torch.float32 and t_.is_contiguous() and t_.numel() == latents.numel())
    if out is None:
        out = torch.empty_like(latents)
    _capi.check(_capi.lib().mvb_fuse_cfg_affine(
        eps_sum.data_ptr(), _ptr(counter), latents.data_ptr(), out.data_ptr(), int(latents.dtype == torch.float32),
        B, Cc, T, HW, int(cfg), guidance, c_x, c_e, c_n, _ptr(noise), a_x, a_e, _ptr(aux_out), _ptr(eps_out), _stream()))
    return out


def fuse_cfg_multistep(eps_sum, counter, latents, guidance, a_x, a_e, clip, c_x, c0, c1=0.0, c2=0.0, c_n=0.0, m1=None,
                       m2=None, noise=None, m0_out=None, cfg=True, out=None):
    """m0 = clamp(a_x x + a_e eps, +-clip) (clip <= 0: none) -> m0_out; x_prev = c_x x + c0 m0 + c1 m1 + c2 m2 + c_n noise
    (eps = overlap mean + CFG of eps_sum). m1 / m2 / noise / m0_out: fp32 like latents, or None; m0_out may be m2."""
    B, Cc, T = latents.shape[:3]
    HW = latents.shape[3] * latents.shape[4]
    assert eps_sum.dtype == torch.float32 and eps_sum.is_contiguous() and latents.is_contiguous()
    assert eps_sum.numel() == latents.numel() * (2 if cfg else 1), "eps_sum must be [2B,...] with cfg, [B,...] without"
    assert latents.dtype in (torch.float16, torch.float32), f"latents must be fp16 or fp32, got {latents.dtype}"
    assert counter is None or (counter.dtype == torch.float32 and counter.is_contiguous() and counter.numel() == T)
    for t_ in (m1, m2, noise, m0_out):
        assert t_ is None or (t_.dtype == torch.float32 and t_.is_contiguous() and t_.numel() == latents.numel())
    if out is None:
        out = torch.empty_like(latents)
    a = _capi.MvbMultistepArgs()
    a.eps_sum, a.counter, a.latents_in, a.latents_out = eps_sum.data_ptr(), _ptr(counter), latents.data_ptr(), out.data_ptr()
    a.m1, a.m2, a.noise, a.m0_out = _ptr(m1), _ptr(m2), _ptr(noise), _ptr(m0_out)
    a.is_f32, a.B, a.C, a.T, a.HW, a.cfg = int(latents.dtype == torch.float32), B, Cc, T, HW, int(cfg)
    a.guidance_scale, a.a_x, a.a_e, a.clip = guidance, a_x, a_e, clip
    a.c_x, a.c0, a.c1, a.c2, a.c_n = c_x, c0, c1, c2, c_n
    _capi.check(_capi.lib().mvb_fuse_cfg_multistep(C.byref(a), _stream()))
    return out


def accumulate_window(eps_sum, eps_win, src_t0, frames_dev):
    B2, Cc, T = eps_sum.shape[:3]
    HW = eps_sum.shape[3] * eps_sum.shape[4]
    assert eps_sum.dtype == torch.float32 and eps_sum.is_contiguous()
    assert eps_win.dtype in (torch.float16, torch.float32) and eps_win.is_contiguous(), "eps_win: contiguous fp16 / fp32"
    assert frames_dev.dtype == torch.int32 and frames_dev.is_contiguous()
    assert eps_win.shape[0] == B2 and eps_win.shape[1] == Cc and src_t0 + frames_dev.numel() <= eps_win.shape[2]
    _capi.check(_capi.lib().mvb_accumulate_window(eps_sum.data_ptr(), B2, Cc, T, HW, eps_win.data_ptr(),
                                                  int(eps_win.dtype == torch.float32), eps_win.shape[2], src_t0,
                                                  frames_dev.data_ptr(), frames_dev.numel(), _stream()))


def hist_match(video: torch.Tensor, target: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Histogram-matches every frame of video [B, C, F, H, W] to target [B, C, 1, Ht, Wt] per batch item and channel
    (`mvb_op_hist_match`): the float32 values MMCM's `hist_match_video_bcthw(video, target, 255.0)` stores, bit for bit.
    Both fp32 CUDA tensors with values in [0, 1]; any strides on the first three axes, each H x W plane contiguous, so
    a frame slice such as `x[:, :, 1:]` is taken as it is. out: a new tensor (None), or a tensor of video's shape that is
    video itself (in place) or overlaps neither video nor itself. Returns out."""
    for name, t in (("video", video), ("target", target)):
        if t.dtype != torch.float32 or not t.is_cuda or t.dim() != 5:
            raise TypeError(f"hist_match: {name} must be a 5-D float32 CUDA tensor, got {t.dim()}-D {t.dtype} on {t.device}")
        if t.stride(4) != 1 or (t.shape[3] > 1 and t.stride(3) != t.shape[4]):
            raise ValueError(f"hist_match: every H x W plane of {name} must be contiguous, strides {t.stride()}")
    B, Cc, F, H, W = video.shape
    if target.device != video.device or tuple(target.shape[:3]) != (B, Cc, 1):
        raise ValueError(f"hist_match: target must be [{B}, {Cc}, 1, H', W'] on {video.device}, got "
                         f"{list(target.shape)} on {target.device}")
    if out is None:
        out = torch.empty_like(video, memory_format=torch.contiguous_format)
    elif out.dtype != torch.float32 or out.device != video.device or out.shape != video.shape or out.stride(4) != 1 or \
            (H > 1 and out.stride(3) != W):
        raise ValueError(f"hist_match: out must be a float32 tensor of shape {list(video.shape)} on {video.device} with "
                         "contiguous H x W planes")
    Ht, Wt = target.shape[3:]
    l = _capi.lib()
    need = l.mvb_op_hist_match_workspace_bytes(B, Cc, F, H, W, Ht, Wt)
    if need < 0:
        _capi.check(int(need))
    ws = torch.empty(int(need), dtype=torch.uint8, device=video.device)
    _capi.check(l.mvb_op_hist_match(video.data_ptr(), B, Cc, F, H, W, *video.stride()[:3], target.data_ptr(), Ht, Wt,
                                    *target.stride()[:2], out.data_ptr(), *out.stride()[:3], ws.data_ptr(), ws.numel(),
                                    _stream()))
    return out


def vae_tile_blend(tiles, plan, out: torch.Tensor, mode: int = 0, scale: float = 1.0) -> torch.Tensor:
    """The stitch of a tiled VAE decode / encode (`mvb_op_vae_tile_blend`): tiles[r][c] holds the tiles of row class r
    and column class c of `plan` (a `musev_b200.vae_tiling.TilePlan`) as contiguous [N * count_r * count_c, C, h_r, w_c]
    tensors in the blend dtype (fp32 or fp16, frame-major, then tile row, then tile column); out [N, C (mode 0, 1) or
    C / 2 (mode 2), out_h, out_w], contiguous fp32 / fp16. mode 0: the blended tiles; 1: clamp(v / 2 + 0.5, 0, 1);
    2: scale * v of the first C / 2 channels. Bit-identical to diffusers' `blend_v` / `blend_h` in the tiles' dtype."""
    rows, cols = plan.rows.classes, plan.cols.classes
    t0 = tiles[0][0]
    if len(tiles) != len(rows) or any(len(t) != len(cols) for t in tiles):
        raise ValueError(f"vae_tile_blend: tiles must be a {len(rows)} x {len(cols)} grid of shape groups")
    ch = t0.shape[1]
    N = out.shape[0]
    for r, row in zip(rows, tiles):
        for c, t in zip(cols, row):
            want = (N * r.count * c.count, ch, r.size_out, c.size_out)
            if tuple(t.shape) != want or t.dtype != t0.dtype or not t.is_contiguous() or t.device != out.device:
                raise ValueError(f"vae_tile_blend: a tile group must be a contiguous {t0.dtype} tensor {list(want)} on "
                                 f"{out.device}, got {list(t.shape)} {t.dtype}")
    cout = ch // 2 if mode == 2 else ch
    if tuple(out.shape) != (N, cout, plan.out_h, plan.out_w) or not out.is_contiguous():
        raise ValueError(f"vae_tile_blend: out must be a contiguous [{N}, {cout}, {plan.out_h}, {plan.out_w}] tensor, "
                         f"got {list(out.shape)}")
    a = _capi.MvbVaeTileBlendArgs()
    K = _capi.VAE_TILE_CLASSES
    for i, row in enumerate(tiles):
        for j, t in enumerate(row):
            a.tiles[i * K + j] = t.data_ptr()
    a.tiles_is_f32, a.N, a.C = _capi._is_f32(t0), N, ch
    a.n_row_classes, a.n_col_classes = len(rows), len(cols)
    for k, r in enumerate(rows):
        a.row_count[k], a.row_size[k] = r.count, r.size_out
    for k, c in enumerate(cols):
        a.col_count[k], a.col_size[k] = c.count, c.size_out
    a.extent, a.row_limit, a.H, a.W = plan.blend_extent, plan.row_limit, plan.out_h, plan.out_w
    a.mode, a.scale = int(mode), float(scale)
    a.out, a.out_is_f32 = out.data_ptr(), _capi._is_f32(out)
    _capi.check(_capi.lib().mvb_op_vae_tile_blend(C.byref(a), _stream()))
    return out
