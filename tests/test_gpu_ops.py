"""GPU parity tests of the individual kernels, called through the C ABI, against torch fp32 on the same inputs.

Tolerances (written per test): operands are fp16, accumulation fp32, outputs rounded to fp16, so the bound is
~2^-10 relative to the output magnitude (plus fp16 rounding of softmax probabilities in attention)."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
dev = "cuda"


@pytest.fixture(scope="module")
def ops(built_lib):
    from musev_b200 import ops as o
    return o


def _close(got, ref, rel=3e-3, abs_=2e-3):
    err = (got.float() - ref).abs().max().item()
    lim = abs_ + rel * ref.abs().max().item()
    assert err <= lim, f"max_abs_err {err:.3e} > {lim:.3e}"
    assert not torch.isnan(got.float()).any()


def _pad_heads(x, heads, d, dp, ones=False):
    o = torch.zeros(x.shape[0], heads, dp, device=x.device, dtype=x.dtype)
    o[:, :, :d] = x.view(x.shape[0], heads, d)
    if ones:
        o[:, :, d] = 1.0
    return o.view(x.shape[0], heads * dp)


# the last two shapes fill more than one wave of tiles on the GPU, one with a ragged last tile
@pytest.mark.parametrize("M,K,N", [(128, 64, 64), (100, 64, 48), (1000, 320, 320), (4096, 1280, 640), (2, 320, 1280),
                                   (40000, 128, 320), (149 * 128 + 37, 192, 64)])
def test_linear(ops, M, K, N):
    torch.manual_seed(0)
    a = torch.randn(1, 1, M, K, device=dev).half()
    w = (torch.randn(N, K, device=dev) / K ** 0.5).half()
    b = torch.randn(N, device=dev)
    res = torch.randn(M, N, device=dev).half()
    out = ops.conv_gemm(a, w, bias=b, residual=res, alpha=0.5, beta=2.0)
    _close(out, (a.float().view(M, K) @ w.float().t() + b) * 0.5 + 2.0 * res.float())


@pytest.mark.parametrize("NF,H,W,C,N,C1", [(2, 16, 16, 64, 64, 0), (3, 8, 8, 128, 320, 0), (2, 32, 32, 640, 640, 320),
                                           (5, 4, 4, 64, 64, 0), (2, 24, 16, 64, 128, 0), (34, 32, 32, 64, 64, 0),
                                           (9, 32, 32, 64, 160, 64)])
def test_conv3x3(ops, NF, H, W, C, N, C1):
    torch.manual_seed(1)
    x = torch.randn(NF, H, W, C, device=dev).half()
    x1 = torch.randn(NF, H, W, C1, device=dev).half() if C1 else None
    Ct = C + C1
    wt = (torch.randn(N, Ct, 3, 3, device=dev) / (9 * Ct) ** 0.5).half()
    bias, temb = torch.randn(N, device=dev), torch.randn(NF, N, device=dev)
    packed = wt.permute(0, 2, 3, 1).reshape(N, 9 * Ct).contiguous()
    out = ops.conv_gemm(x, packed, taps=ops.TAPS_3X3, a1=x1, bias=bias, rowadd=temb, rows_per_group=H * W)
    xin = x if x1 is None else torch.cat([x, x1], 3)
    ref = F.conv2d(xin.float().permute(0, 3, 1, 2), wt.float(), bias, padding=1) + temb[:, :, None, None]
    _close(out, ref.permute(0, 2, 3, 1).reshape(-1, N))


@pytest.mark.parametrize("NF,H,W,C", [(3, 16, 16, 64), (4, 8, 8, 128)])
def test_conv_stride2(ops, NF, H, W, C):
    torch.manual_seed(2)
    x = torch.randn(NF, H, W, C, device=dev).half()
    wt = (torch.randn(C, C, 3, 3, device=dev) / (9 * C) ** 0.5).half()
    b = torch.randn(C, device=dev)
    out = ops.conv_gemm(x, wt.permute(0, 2, 3, 1).reshape(C, 9 * C).contiguous(), taps=ops.TAPS_3X3, bias=b, stride2=True)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), wt.float(), b, stride=2, padding=1)
    _close(out, ref.permute(0, 2, 3, 1).reshape(-1, C))


@pytest.mark.parametrize("B,T,HW,C", [(2, 5, 64, 320), (1, 3, 16, 64), (2, 9, 256, 128)])
def test_temporal_conv(ops, B, T, HW, C):
    torch.manual_seed(3)
    x = torch.randn(B, T, HW, C, device=dev).half()
    wt = (torch.randn(C, C, 3, device=dev) / (3 * C) ** 0.5).half()
    out = ops.conv_gemm(x, wt.permute(0, 2, 1).reshape(C, 3 * C).contiguous(), taps=ops.TAPS_T3)
    ref = F.conv1d(x.float().permute(0, 2, 3, 1).reshape(B * HW, C, T), wt.float(), padding=1)
    _close(out, ref.reshape(B, HW, C, T).permute(0, 3, 1, 2).reshape(-1, C))


def test_geglu_and_fp32_out(ops):
    torch.manual_seed(4)
    M, K, Nout = 512, 320, 1280
    a = torch.randn(1, 1, M, K, device=dev).half()
    w = (torch.randn(2 * Nout, K, device=dev) / K ** 0.5).half()
    b = torch.randn(2 * Nout, device=dev)
    packed = torch.cat([w[:Nout].view(-1, 16, K), w[Nout:].view(-1, 16, K)], 1).reshape(2 * Nout, K).contiguous()
    bp = torch.cat([b[:Nout].view(-1, 16), b[Nout:].view(-1, 16)], 1).reshape(-1).contiguous()
    out = ops.conv_gemm(a, packed, bias=bp, geglu=True)
    h = a.float().view(M, K) @ w.float().t() + b
    _close(out, h[:, :Nout] * F.gelu(h[:, Nout:]))
    o32 = ops.conv_gemm(a, w[:640].contiguous(), bias=b[:640].contiguous(), act=1, out_f32=True)
    assert o32.dtype == torch.float32
    _close(o32, F.silu(h[:, :640]), rel=1e-4, abs_=1e-4)


@pytest.mark.parametrize("NF,HW,C0,C1,fps,silu", [(4, 256, 320, 0, 1, True), (6, 64, 1280, 1280, 1, True),
                                                  (6, 1024, 640, 320, 3, False), (4, 64, 64, 0, 2, True),
                                                  (34, 4096, 320, 0, 17, True), (34, 4096, 320, 0, 1, False)])
@pytest.mark.parametrize("fused", [False, True])
def test_groupnorm(ops, NF, HW, C0, C1, fps, silu, fused):
    torch.manual_seed(5)
    x0 = (torch.randn(NF, HW, C0, device=dev) * 2 + 0.5).half()
    x1 = (torch.randn(NF, HW, C1, device=dev) - 1).half() if C1 else None
    C = C0 + C1
    g, b = torch.randn(C, device=dev), torch.randn(C, device=dev)
    y = ops.groupnorm(x0, g, b, 32, fps, 1e-5, silu, x1, fused=fused)
    if fused:      # one launch vs three launches: same partial layout; deterministic
        assert torch.equal(y, ops.groupnorm(x0, g, b, 32, fps, 1e-5, silu, x1, fused=True))
        y3 = ops.groupnorm(x0, g, b, 32, fps, 1e-5, silu, x1)
        if fps == 1:   # same reduction order -> bit-identical (the three-launch path merges 5-D statistics on 8 warps instead of 1)
            assert torch.equal(y, y3)
        else:
            assert (y.float() - y3.float()).abs().max().item() <= 4e-3
    x = x0 if x1 is None else torch.cat([x0, x1], 2)
    ref = F.group_norm(x.float().view(NF // fps, fps * HW, C).permute(0, 2, 1), 32, g, b, 1e-5)
    if silu:
        ref = F.silu(ref)
    _close(y, ref.permute(0, 2, 1).reshape(NF, HW, C), rel=2e-3, abs_=4e-3)


@pytest.mark.parametrize("M,C,eps", [(1000, 320, 0.0), (77, 1280, 1e-5), (513, 640, 0.0), (64, 64, 0.0)])
def test_layernorm(ops, M, C, eps):
    torch.manual_seed(6)
    x = (torch.randn(M, C, device=dev) * 3 + 1).half()
    g, b = torch.randn(C, device=dev), torch.randn(C, device=dev)
    _close(ops.layernorm(x, g, b, eps), F.layer_norm(x.float(), (C,), g, b, eps), rel=2e-3, abs_=4e-3)


@pytest.mark.parametrize("B,T,HW,d", [(2, 5, 64, 40), (2, 17, 256, 80), (1, 9, 16, 160), (2, 13, 64, 16), (1, 1, 32, 40)])
def test_temporal_attention(ops, B, T, HW, d):
    torch.manual_seed(7)
    heads, dp, M = 8, (d + 15) // 16 * 16, B * T * HW
    q, k, v = (torch.randn(M, heads * d, device=dev).half() for _ in range(3))
    qkv = torch.cat([_pad_heads(t, heads, d, dp) for t in (q, k, v)], 1).contiguous()
    out = ops.temporal_attention(qkv, B, T, HW, heads, d, dp, d ** -0.5)

    def r(x):
        return x.float().view(B, T, HW, heads, d).permute(0, 2, 3, 1, 4)
    ref = F.scaled_dot_product_attention(r(q), r(k), r(v)).permute(0, 3, 1, 2, 4).reshape(M, heads * d)
    _close(out, ref, rel=2e-3, abs_=1e-3)


@pytest.mark.parametrize("NF,T,Nq,d,viscond,ones", [(2, 1, 128, 64, False, False), (4, 2, 256, 40, True, False),
                                                    (4, 2, 256, 40, True, True), (4, 2, 256, 80, True, False),
                                                    (4, 2, 64, 160, True, False), (2, 1, 200, 40, False, True),
                                                    (2, 1, 16, 16, False, False), (6, 3, 1024, 40, True, True)])
@pytest.mark.parametrize("variant", [0, 1, 2, 4])
def test_spatial_attention(ops, NF, T, Nq, d, viscond, ones, variant):
    """Reference-only self attention: K/V = own frame (+) first frame of the batch (attention_processor.py:431-493).
    Every `variant` value is accepted by the op-level ABI and runs the same kernel; the result must not depend on it."""
    torch.manual_seed(8)
    heads, dp, M = 8, (d + 15) // 16 * 16, NF * Nq
    q, k, v = (torch.randn(M, heads * d, device=dev).half() for _ in range(3))
    qkv = torch.cat([_pad_heads(q, heads, d, dp), _pad_heads(k, heads, d, dp), _pad_heads(v, heads, d, dp, ones)], 1).contiguous()
    hd = heads * dp
    segs = [dict(k=qkv[:, hd:2 * hd], v=qkv[:, 2 * hd:], nk=Nq, fdiv=1, fmul=Nq, fadd=0)]
    if viscond:
        segs.append(dict(k=qkv[:, hd:2 * hd], v=qkv[:, 2 * hd:], nk=Nq, fdiv=T, fmul=T * Nq, fadd=0))
    out = ops.attention(qkv[:, :hd], segs, NF, Nq, heads, d, dp, d ** -0.5, v_ones_col=ones, variant=variant)
    qf, kf, vf = (t.float().view(NF, Nq, heads, d).permute(0, 2, 1, 3) for t in (q, k, v))
    if viscond:
        idx = (torch.arange(NF, device=dev) // T) * T
        kf, vf = torch.cat([kf, kf[idx]], 2), torch.cat([vf, vf[idx]], 2)
    ref = F.scaled_dot_product_attention(qf, kf, vf).permute(0, 2, 1, 3).reshape(M, heads * d)
    _close(out, ref, rel=3e-3, abs_=1e-3)


@pytest.mark.parametrize("d,Nq", [(40, 256), (160, 64), (80, 1024)])
def test_cross_attention_text_plus_ip(ops, d, Nq):
    """Text cross attention + ip_scale * image cross attention: two softmaxes (attention_processor.py:258-300)."""
    torch.manual_seed(9)
    NF, T, heads, nk = 6, 3, 8, 77
    B, dp, M = NF // T, (d + 15) // 16 * 16, NF * Nq
    hd = heads * dp
    q = torch.randn(M, heads * d, device=dev).half()
    k, v = (torch.randn(B * nk, heads * d, device=dev).half() for _ in range(2))
    k2, v2 = (torch.randn(B * 4, heads * d, device=dev).half() for _ in range(2))
    qp = _pad_heads(q, heads, d, dp)
    kv = torch.cat([_pad_heads(k, heads, d, dp), _pad_heads(v, heads, d, dp)], 1).contiguous()
    kv2 = torch.cat([_pad_heads(k2, heads, d, dp), _pad_heads(v2, heads, d, dp)], 1).contiguous()
    out = ops.attention(qp, [dict(k=kv[:, :hd], v=kv[:, hd:], nk=nk, fdiv=T, fmul=nk, fadd=0)], NF, Nq, heads, d, dp, d ** -0.5)
    ops.attention(qp, [dict(k=kv2[:, :hd], v=kv2[:, hd:], nk=4, fdiv=T, fmul=4, fadd=0)], NF, Nq, heads, d, dp, d ** -0.5,
                  out=out, out_scale=0.7, accumulate=True)
    idx = torch.arange(NF, device=dev) // T
    qf = q.float().view(NF, Nq, heads, d).permute(0, 2, 1, 3)

    def kvf(t, n):
        return t.float().view(B, n, heads, d).permute(0, 2, 1, 3)[idx]
    ref = F.scaled_dot_product_attention(qf, kvf(k, nk), kvf(v, nk)) + 0.7 * F.scaled_dot_product_attention(qf, kvf(k2, 4), kvf(v2, 4))
    _close(out, ref.permute(0, 2, 1, 3).reshape(M, heads * d), rel=3e-3, abs_=2e-3)


def test_fused_step_matches_oracle_scheduler(ops):
    """Overlap mean + CFG + DDIM in one kernel vs the oracle's DDIM (pinned to the reference scheduler)."""
    from oracle.pipeline_oracle import SD15_DDIM, DDIMOracle
    torch.manual_seed(10)
    B, C, T, H, W = 1, 4, 6, 8, 8
    eps_sum = torch.randn(2 * B, C, T, H, W, device=dev)
    counter = torch.tensor([1, 1, 2, 2, 1, 1.0], device=dev)
    lat = torch.randn(B, C, T, H, W, device=dev)
    s = DDIMOracle(**SD15_DDIM)
    s.set_timesteps(20)
    for t in (951, 501, 1):
        a_t = float(s.alphas_cumprod[t])
        a_p = float(s.alphas_cumprod[t - 50]) if t - 50 >= 0 else float(s.final_alpha_cumprod)
        out = ops.fuse_cfg_ddim(eps_sum, counter, lat, 3.5, a_t, a_p)
        e = (eps_sum / counter.view(1, 1, T, 1, 1)).cpu()
        e = e[:B] + 3.5 * (e[B:] - e[:B])
        ref, _ = s.step(e, t, lat.cpu())
        assert (out.cpu() - ref).abs().max().item() < 2e-5
    # window accumulation (pipeline_controlnet.py:2068-2078)
    win = torch.randn(2, C, 4, H, W, device=dev)
    es = torch.zeros(2, C, T, H, W, device=dev)
    ops.accumulate_window(es, win, 1, torch.tensor([2, 3, 4], device=dev, dtype=torch.int32))
    ref2 = torch.zeros_like(es)
    ref2[:, :, 2:5] = win[:, :, 1:4]
    assert torch.equal(es, ref2)


def test_scheduler_step_api(ops):
    """musev_b200.DDIMScheduler.step (cfg = 0 form of the fused kernel) vs the reference-scheduler fixture."""
    import os
    from conftest import GOLDEN
    from musev_b200.scheduler import SD15_DDIM_CONFIG, DDIMScheduler
    g = torch.load(os.path.join(GOLDEN, "ddim_sd15.pt"))
    s = DDIMScheduler(**SD15_DDIM_CONFIG)
    s.set_timesteps(20, device=dev)
    assert s.timesteps.tolist() == g["timesteps"].tolist()
    for t, ref in g["prev"].items():
        out = s.step(g["eps"].to(dev), int(t), g["x"].to(dev), eta=0.0)
        assert (out.prev_sample.cpu() - ref).abs().max().item() < 2e-6
        assert out.pred_original_sample.shape == ref.shape
    out16 = s.step(g["eps"].to(dev).half(), 501, g["x"].to(dev).half()).prev_sample
    assert out16.dtype == torch.float16 and (out16.float().cpu() - g["prev"]["501"]).abs().max().item() < 5e-3


def test_sampler_steps_match_oracle(ops):
    """EulerDiscreteScheduler.step / LCMScheduler.step on the fused affine kernel vs the reference-form oracle."""
    from musev_b200.samplers import EulerDiscreteScheduler, LCMScheduler
    from oracle.sampler_oracle import EulerOracle, LCMOracle
    kw = dict(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
              timestep_spacing="leading", steps_offset=1)
    g = torch.Generator().manual_seed(2)
    x, e = torch.randn(1, 4, 5, 8, 8, generator=g), torch.randn(1, 4, 5, 8, 8, generator=g)
    for pred in ("epsilon", "v_prediction"):
        s, o = EulerDiscreteScheduler(prediction_type=pred, **kw), EulerOracle(prediction_type=pred, **kw)
        s.set_timesteps(20)
        o.set_timesteps(20)
        xs, xo = x.to(dev) * float(s.init_noise_sigma), x * o.init_noise_sigma
        for t in s.timesteps[:4]:
            assert (s.scale_model_input(xs, t).cpu() - o.scale_model_input(xo, t)).abs().max().item() < 1e-5
            r = s.step(e.to(dev), t, xs)
            po, x0o = o.step(e, t, xo)
            assert (r.prev_sample.cpu() - po).abs().max().item() < 1e-4 and (r.pred_original_sample.cpu() - x0o).abs().max().item() < 1e-4
            xs, xo = r.prev_sample, po
    l, lo = LCMScheduler(), LCMOracle()
    l.set_timesteps(4)
    lo.set_timesteps(4)
    xs, xo = x.to(dev), x.clone()
    gd, gc = torch.Generator(device=dev).manual_seed(5), torch.Generator().manual_seed(5)
    for t in l.timesteps:
        # CPU and CUDA generators give different streams: compare through the noise-free part and the noise scale
        a_t_prev = l.step(e.to(dev), t, xs, generator=gd)
        po, deno, noise = lo.step(e, t, xo, gc)
        assert (a_t_prev.denoised.cpu() - deno).abs().max().item() < 1e-4
        if noise is None:
            assert (a_t_prev.prev_sample.cpu() - po).abs().max().item() < 1e-4
        xs, xo = po.to(dev), po


@pytest.mark.parametrize("fused", [False, True])
def test_groupnorm_large_mean(ops, fused):
    """|mean| >> std: sum / sum-of-squares statistics in fp32 lose the variance here (E[x^2] - E[x]^2 cancels to ~6 % at
    mean 2048, std 4); the (count, mean, M2) statistics do not."""
    torch.manual_seed(11)
    NF, HW, C = 4, 1024, 320
    x = (torch.randn(NF, HW, C, device=dev) * 4 + 2048).half()
    g, b = torch.randn(C, device=dev), torch.randn(C, device=dev)
    y = ops.groupnorm(x, g, b, 32, 1, 1e-5, False, None, fused=fused)
    ref = F.group_norm(x.float().permute(0, 2, 1), 32, g, b, 1e-5).permute(0, 2, 1)
    _close(y, ref, rel=2e-3, abs_=4e-3)
