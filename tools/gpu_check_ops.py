"""GPU check of attention / norm / step kernels against torch fp32."""
import sys, math
import torch
import torch.nn.functional as F
sys.path.insert(0, ".")
from musev_b200 import ops

torch.manual_seed(0)
dev = "cuda"
allok = True


def rep(name, got, ref, tol):
    global allok
    err = (got.float() - ref).abs()
    bad = err > tol
    ok = not bad.any().item()
    allok &= ok
    print(f"[{name}] max_abs_err={err.max().item():.4e} ref_absmax={ref.abs().max().item():.3f} bad={bad.sum().item()}/{bad.numel()}", flush=True)
    if not ok:
        idx = bad.nonzero()
        print("   first bad:", idx[:6].tolist())
        print("   got", got.float().flatten()[:8].tolist())
        print("   ref", ref.flatten()[:8].tolist())


def pad_heads(x, heads, d, dp):
    M = x.shape[0]
    o = torch.zeros(M, heads, dp, device=x.device, dtype=x.dtype)
    o[:, :, :d] = x.view(M, heads, d)
    return o.view(M, heads * dp)


def attn_case(NF, T, Nq, heads, d, nk1_mode, name, ones=False):
    """self attention with K/V = own frame (+) vis-cond frame (frame 0 of each batch of T frames)."""
    dp = (d + 15) // 16 * 16
    M = NF * Nq
    q = torch.randn(M, heads * d, device=dev).half()
    k = torch.randn(M, heads * d, device=dev).half()
    v = torch.randn(M, heads * d, device=dev).half()
    vp = pad_heads(v, heads, d, dp)
    if ones:
        vp.view(M, heads, dp)[:, :, d] = 1.0
    qkv = torch.cat([pad_heads(q, heads, d, dp), pad_heads(k, heads, d, dp), vp], dim=1).contiguous()
    hd = heads * dp
    qv, kv, vv = qkv[:, :hd], qkv[:, hd:2 * hd], qkv[:, 2 * hd:]
    segs = [dict(k=kv, v=vv, nk=Nq, fdiv=1, fmul=Nq, fadd=0)]
    if nk1_mode == "viscond":
        segs.append(dict(k=kv, v=vv, nk=Nq, fdiv=T, fmul=T * Nq, fadd=0))
    out = ops.attention(qv, segs, NF, Nq, heads, d, dp, d ** -0.5, v_ones_col=ones)
    torch.cuda.synchronize()
    qf = q.float().view(NF, Nq, heads, d).permute(0, 2, 1, 3)
    kf = k.float().view(NF, Nq, heads, d).permute(0, 2, 1, 3)
    vf = v.float().view(NF, Nq, heads, d).permute(0, 2, 1, 3)
    if nk1_mode == "viscond":
        idx = (torch.arange(NF, device=dev) // T) * T
        kf = torch.cat([kf, kf[idx]], dim=2)
        vf = torch.cat([vf, vf[idx]], dim=2)
    ref = F.scaled_dot_product_attention(qf, kf, vf).permute(0, 2, 1, 3).reshape(M, heads * d)
    rep(name, out, ref, 6e-3)


def cross_case(NF, T, Nq, heads, d, nk, name, ip=False):
    dp = (d + 15) // 16 * 16
    B = NF // T
    M = NF * Nq
    q = torch.randn(M, heads * d, device=dev).half()
    k = torch.randn(B * nk, heads * d, device=dev).half()
    v = torch.randn(B * nk, heads * d, device=dev).half()
    qp = pad_heads(q, heads, d, dp)
    kvp = torch.cat([pad_heads(k, heads, d, dp), pad_heads(v, heads, d, dp)], dim=1).contiguous()
    hd = heads * dp
    segs = [dict(k=kvp[:, :hd], v=kvp[:, hd:], nk=nk, fdiv=T, fmul=nk, fadd=0)]
    out = ops.attention(qp, segs, NF, Nq, heads, d, dp, d ** -0.5)
    qf = q.float().view(NF, Nq, heads, d).permute(0, 2, 1, 3)
    idx = torch.arange(NF, device=dev) // T
    kf = k.float().view(B, nk, heads, d).permute(0, 2, 1, 3)[idx]
    vf = v.float().view(B, nk, heads, d).permute(0, 2, 1, 3)[idx]
    ref = F.scaled_dot_product_attention(qf, kf, vf).permute(0, 2, 1, 3).reshape(M, heads * d)
    if ip:
        k2 = torch.randn(B * 4, heads * d, device=dev).half()
        v2 = torch.randn(B * 4, heads * d, device=dev).half()
        kv2 = torch.cat([pad_heads(k2, heads, d, dp), pad_heads(v2, heads, d, dp)], dim=1).contiguous()
        ops.attention(qp, [dict(k=kv2[:, :hd], v=kv2[:, hd:], nk=4, fdiv=T, fmul=4, fadd=0)], NF, Nq, heads, d, dp,
                      d ** -0.5, out=out, out_scale=0.7, accumulate=True)
        k2f = k2.float().view(B, 4, heads, d).permute(0, 2, 1, 3)[idx]
        v2f = v2.float().view(B, 4, heads, d).permute(0, 2, 1, 3)[idx]
        ref = ref + 0.7 * F.scaled_dot_product_attention(qf, k2f, v2f).permute(0, 2, 1, 3).reshape(M, heads * d)
    torch.cuda.synchronize()
    rep(name, out, ref, 6e-3)


def tattn_case(B, T, HW, heads, d):
    dp = (d + 15) // 16 * 16
    M = B * T * HW
    q, k, v = (torch.randn(M, heads * d, device=dev).half() for _ in range(3))
    qkv = torch.cat([pad_heads(q, heads, d, dp), pad_heads(k, heads, d, dp), pad_heads(v, heads, d, dp)], dim=1).contiguous()
    out = ops.temporal_attention(qkv, B, T, HW, heads, d, dp, d ** -0.5)
    torch.cuda.synchronize()
    def r(x):
        return x.float().view(B, T, HW, heads, d).permute(0, 2, 3, 1, 4)  # b hw h t d
    ref = F.scaled_dot_product_attention(r(q), r(k), r(v)).permute(0, 3, 1, 2, 4).reshape(M, heads * d)
    rep(f"temporal_attn B={B} T={T} HW={HW} d={d}", out, ref, 4e-3)


def gn_case(NF, HW, C0, C1, fps, silu):
    x0 = (torch.randn(NF, HW, C0, device=dev) * 2 + 0.5).half()
    x1 = (torch.randn(NF, HW, C1, device=dev) - 1).half() if C1 else None
    C = C0 + C1
    g = torch.randn(C, device=dev); b = torch.randn(C, device=dev)
    y = ops.groupnorm(x0, g, b, 32, fps, 1e-5, silu, x1)
    torch.cuda.synchronize()
    x = x0 if x1 is None else torch.cat([x0, x1], 2)
    xr = x.float().view(NF // fps, fps * HW, C).permute(0, 2, 1)
    ref = F.group_norm(xr, 32, g, b, 1e-5)
    if silu:
        ref = F.silu(ref)
    ref = ref.permute(0, 2, 1).reshape(NF, HW, C)
    rep(f"groupnorm NF={NF} HW={HW} C={C0}+{C1} fps={fps} silu={silu}", y, ref, 2e-2)


def ln_case(M, C, eps):
    x = (torch.randn(M, C, device=dev) * 3 + 1).half()
    g = torch.randn(C, device=dev); b = torch.randn(C, device=dev)
    y = ops.layernorm(x, g, b, eps)
    torch.cuda.synchronize()
    rep(f"layernorm M={M} C={C} eps={eps}", y, F.layer_norm(x.float(), (C,), g, b, eps), 2e-2)


def ddim_case():
    B, C, T, H, W = 1, 4, 6, 8, 8
    eps_sum = torch.randn(2 * B, C, T, H, W, device=dev)
    counter = torch.tensor([1, 1, 2, 2, 1, 1.0], device=dev)
    lat = torch.randn(B, C, T, H, W, device=dev)
    a_t, a_p, g = 0.35, 0.42, 3.5
    out = ops.fuse_cfg_ddim(eps_sum, counter, lat, g, a_t, a_p)
    e = eps_sum / counter.view(1, 1, T, 1, 1)
    e = e[:B] + g * (e[B:] - e[:B])
    x0 = (lat - (1 - a_t) ** 0.5 * e) / a_t ** 0.5
    ref = a_p ** 0.5 * x0 + (1 - a_p) ** 0.5 * e
    torch.cuda.synchronize()
    rep("fuse_cfg_ddim", out, ref, 1e-5)
    win = torch.randn(2, C, 4, H, W, device=dev)
    es = torch.zeros(2, C, T, H, W, device=dev)
    fr = torch.tensor([2, 3, 4], device=dev, dtype=torch.int32)
    ops.accumulate_window(es, win, 1, fr)
    torch.cuda.synchronize()
    ref2 = torch.zeros_like(es); ref2[:, :, 2:5] = win[:, :, 1:4]
    rep("accumulate_window", es, ref2, 1e-6)


def conv_s2_case(NF, H, W, C, N):
    x = torch.randn(NF, H, W, C, device=dev).half()
    wt = (torch.randn(N, C, 3, 3, device=dev) / (9 * C) ** 0.5).half()
    bias = torch.randn(N, device=dev)
    packed = wt.permute(0, 2, 3, 1).reshape(N, 9 * C).contiguous()
    out = ops.conv_gemm(x, packed, taps=ops.TAPS_3X3, bias=bias, stride2=True)
    torch.cuda.synchronize()
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), wt.float(), bias, stride=2, padding=1).permute(0, 2, 3, 1).reshape(-1, N)
    rep(f"conv3x3 stride2 NF={NF} {H}x{W} C={C} N={N}", out, ref, 2e-2)


def f32_case(M, K, N):
    a = torch.randn(1, 1, M, K, device=dev).half()
    w = (torch.randn(N, K, device=dev) / K ** 0.5).half()
    b = torch.randn(N, device=dev)
    out = ops.conv_gemm(a, w, bias=b, act=1, out_f32=True)
    torch.cuda.synchronize()
    rep(f"gemm fp32-out silu M={M} K={K} N={N}", out, F.silu(a.float().view(M, K) @ w.float().t() + b), 5e-3)


def guard(fn, *a, **k):
    global allok
    try:
        fn(*a, **k)
    except Exception as e:  # keep going: one GPU call must report on every kernel
        allok = False
        print(f"[EXC] {fn.__name__}{a}: {type(e).__name__}: {e}", flush=True)
        try:
            torch.cuda.synchronize()
        except Exception as e2:
            print("   device error is sticky:", e2, flush=True)
            raise SystemExit(3)


if __name__ == "__main__":
    guard(gn_case, 4, 256, 320, 0, 1, True)
    guard(gn_case, 6, 64, 1280, 1280, 1, True)
    guard(gn_case, 6, 1024, 640, 320, 3, False)
    guard(gn_case, 34, 4096, 320, 0, 17, True)
    guard(ln_case, 1000, 320, 0.0)
    guard(ln_case, 77, 1280, 1e-5)
    guard(ln_case, 513, 640, 0.0)
    guard(ddim_case)
    guard(conv_s2_case, 3, 16, 16, 64, 64)
    guard(conv_s2_case, 34, 64, 64, 320, 320)
    guard(conv_s2_case, 5, 4, 4, 128, 128)
    guard(f32_case, 2, 320, 1280)
    guard(f32_case, 34, 1280, 640)
    guard(tattn_case, 2, 5, 64, 8, 40)
    guard(tattn_case, 2, 17, 256, 8, 80)
    guard(tattn_case, 1, 9, 16, 8, 160)
    guard(tattn_case, 2, 13, 64, 8, 16)
    guard(attn_case, 2, 1, 128, 1, 64, "none", "attn 1 tile d=64 1 head")
    guard(attn_case, 2, 1, 256, 2, 64, "none", "attn 2x2 tiles d=64")
    guard(attn_case, 2, 1, 128, 8, 40, "none", "attn d=40 (dp=48)")
    guard(attn_case, 4, 2, 256, 8, 40, "viscond", "attn d=40 viscond 2 segs")
    guard(attn_case, 4, 2, 256, 8, 40, "viscond", "attn d=40 viscond 2 segs ONES", ones=True)
    guard(attn_case, 2, 1, 200, 8, 40, "none", "attn d=40 Nq=200 (masked tail) ONES", ones=True)
    guard(attn_case, 4, 2, 256, 8, 80, "viscond", "attn d=80 viscond")
    guard(attn_case, 4, 2, 64, 8, 160, "viscond", "attn d=160 Nq=64 viscond")
    guard(attn_case, 6, 3, 1024, 8, 40, "viscond", "attn d=40 Nq=1024 viscond")
    guard(attn_case, 2, 1, 16, 8, 16, "none", "attn d=16 Nq=16")
    guard(cross_case, 4, 2, 256, 8, 40, 77, "cross nk=77 d=40")
    guard(cross_case, 4, 2, 64, 8, 160, 77, "cross nk=77 d=160 + ip", ip=True)
    guard(cross_case, 6, 3, 1024, 8, 80, 77, "cross nk=77 d=80 + ip", ip=True)
    print("ALL OK" if allok else "SOME FAILED", flush=True)
    if allok:
        # level-0 benchmark: (272, 4096, 8192, 40)
        NF, T, Nq, heads, d, dp = 34, 17, 4096, 8, 40, 48
        M = NF * Nq
        qkv = torch.randn(M, 3 * heads * dp, device=dev).half()
        hd = heads * dp
        qkv[:, 2 * hd:].view(M, heads, dp)[:, :, d] = 1.0
        segs = [dict(k=qkv[:, hd:2 * hd], v=qkv[:, 2 * hd:], nk=Nq, fdiv=1, fmul=Nq, fadd=0),
                dict(k=qkv[:, hd:2 * hd], v=qkv[:, 2 * hd:], nk=Nq, fdiv=T, fmul=T * Nq, fadd=0)]
        out = torch.empty(M, heads * d, device=dev, dtype=torch.half)
        for _ in range(2):
            ops.attention(qkv[:, :hd], segs, NF, Nq, heads, d, dp, d ** -0.5, out=out, v_ones_col=True)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5):
            ops.attention(qkv[:, :hd], segs, NF, Nq, heads, d, dp, d ** -0.5, out=out, v_ones_col=True)
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 5
        fl = 4.0 * NF * heads * Nq * 2 * Nq * d
        print(f"[bench] attention (272,4096,8192,40): {ms:.3f} ms {fl / ms / 1e9:.1f} TFLOP/s", flush=True)
        x = torch.randn(34, 4096, 320, device=dev).half()
        g = torch.ones(320, device=dev); b = torch.zeros(320, device=dev)
        for fps in (1, 17):
            for _ in range(2): ops.groupnorm(x, g, b, 32, fps, 1e-5, True)
            e0.record()
            for _ in range(10): ops.groupnorm(x, g, b, 32, fps, 1e-5, True)
            e1.record(); torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 10
            print(f"[bench] groupnorm+silu 34x4096x320 fps={fps}: {ms:.3f} ms  {3 * x.numel() * 2 / ms / 1e6:.0f} GB/s (2R+1W)", flush=True)
        for (Ml, Cl) in ((139264, 320), (34816, 640)):
            xl = torch.randn(Ml, Cl, device=dev).half()
            gl = torch.ones(Cl, device=dev); bl = torch.zeros(Cl, device=dev)
            for _ in range(2): ops.layernorm(xl, gl, bl, 1e-5)
            e0.record()
            for _ in range(10): ops.layernorm(xl, gl, bl, 1e-5)
            e1.record(); torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 10
            print(f"[bench] layernorm {Ml}x{Cl}: {ms:.3f} ms  {2 * xl.numel() * 2 / ms / 1e6:.0f} GB/s (1R+1W)", flush=True)
        qkv_t = torch.randn(2 * 17 * 4096, 3 * 8 * 48, device=dev).half()
        for _ in range(2): ops.temporal_attention(qkv_t, 2, 17, 4096, 8, 40, 48, 40 ** -0.5)
        e0.record()
        for _ in range(5): ops.temporal_attention(qkv_t, 2, 17, 4096, 8, 40, 48, 40 ** -0.5)
        e1.record(); torch.cuda.synchronize()
        print(f"[bench] temporal attention level0: {e0.elapsed_time(e1) / 5:.3f} ms", flush=True)
