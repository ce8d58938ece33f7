"""GPU check of the wgmma implicit-GEMM kernel against torch fp32.

Prints, per case, max-abs error and -- on mismatch -- where the wrong elements are, so that descriptor /
swizzle / pipeline bugs can be told apart from a single run.
"""
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, ".")
from musev_b200 import ops  # noqa: E402

torch.manual_seed(0)
dev = "cuda"


def report(name, got, ref, tol=2e-2):
    got = got.float()
    err = (got - ref).abs()
    scale = ref.abs().max().item() + 1e-6
    bad = err > tol * max(1.0, scale)
    print(f"[{name}] max_abs_err={err.max().item():.4e} ref_max={scale:.3f} bad={bad.sum().item()}/{bad.numel()}",
          flush=True)
    if bad.any():
        idx = bad.nonzero()
        print("   first bad idx:", idx[:8].tolist())
        rows = idx[:, 0]
        cols = idx[:, 1]
        print("   bad rows%128 hist (8 bins):", torch.histc((rows % 128).float(), 8, 0, 128).tolist())
        print("   bad rows%8 hist:", torch.bincount(rows % 8, minlength=8).tolist())
        print("   bad cols%64 hist (8 bins):", torch.histc((cols % 64).float(), 8, 0, 64).tolist())
        print("   got[:2,:8]", got[:2, :8].tolist())
        print("   ref[:2,:8]", ref[:2, :8].tolist())
        return False
    return True


def case_plain(M, K, N, **kw):
    a = torch.randn(1, 1, M, K, device=dev).half()
    w = (torch.randn(N, K, device=dev) / K ** 0.5).half()
    bias = torch.randn(N, device=dev) if kw.get("bias") else None
    res = torch.randn(M, N, device=dev).half() if kw.get("res") else None
    out = ops.conv_gemm(a, w, bias=bias, residual=res, alpha=kw.get("alpha", 1.0), beta=kw.get("beta", 1.0))
    torch.cuda.synchronize()
    ref = a.float().view(M, K) @ w.float().t()
    if bias is not None:
        ref = ref + bias
    ref = ref * kw.get("alpha", 1.0)
    if res is not None:
        ref = ref + kw.get("beta", 1.0) * res.float()
    return report(f"plain M={M} K={K} N={N} {kw}", out, ref)


def case_conv3x3(NF, H, W, C, N, C1=0):
    x = torch.randn(NF, H, W, C, device=dev).half()
    x1 = torch.randn(NF, H, W, C1, device=dev).half() if C1 else None
    Ct = C + C1
    wt = (torch.randn(N, Ct, 3, 3, device=dev) / (9 * Ct) ** 0.5).half()
    bias = torch.randn(N, device=dev)
    temb = torch.randn(NF, N, device=dev)
    packed = wt.permute(0, 2, 3, 1).reshape(N, 9 * Ct).contiguous()
    out = ops.conv_gemm(x, packed, taps=ops.TAPS_3X3, a1=x1, bias=bias, rowadd=temb, rows_per_group=H * W)
    torch.cuda.synchronize()
    xin = x if x1 is None else torch.cat([x, x1], dim=3)
    ref = F.conv2d(xin.float().permute(0, 3, 1, 2), wt.float(), bias, padding=1) + temb[:, :, None, None]
    ref = ref.permute(0, 2, 3, 1).reshape(-1, N)
    return report(f"conv3x3 NF={NF} H={H} W={W} C={C}+{C1} N={N}", out, ref)


def case_tconv(B, T, HW, C, N):
    x = torch.randn(B, T, HW, C, device=dev).half()
    wt = (torch.randn(N, C, 3, device=dev) / (3 * C) ** 0.5).half()
    packed = wt.permute(0, 2, 1).reshape(N, 3 * C).contiguous()
    out = ops.conv_gemm(x, packed, taps=ops.TAPS_T3)
    torch.cuda.synchronize()
    ref = F.conv1d(x.float().permute(0, 2, 3, 1).reshape(B * HW, C, T), wt.float(), padding=1)
    ref = ref.reshape(B, HW, N, T).permute(0, 3, 1, 2).reshape(-1, N)
    return report(f"tconv B={B} T={T} HW={HW} C={C} N={N}", out, ref)


def case_geglu(M, K, Nout):
    a = torch.randn(1, 1, M, K, device=dev).half()
    w = (torch.randn(2 * Nout, K, device=dev) / K ** 0.5).half()
    b = torch.randn(2 * Nout, device=dev)
    # pack [16 value | 16 gate] chunks
    wv, wg = w[:Nout].view(Nout // 16, 16, K), w[Nout:].view(Nout // 16, 16, K)
    packed = torch.cat([wv, wg], dim=1).reshape(2 * Nout, K).contiguous()
    bp = torch.cat([b[:Nout].view(-1, 16), b[Nout:].view(-1, 16)], dim=1).reshape(-1).contiguous()
    out = ops.conv_gemm(a, packed, bias=bp, geglu=True)
    torch.cuda.synchronize()
    h = a.float().view(M, K) @ w.float().t() + b
    ref = h[:, :Nout] * F.gelu(h[:, Nout:])
    return report(f"geglu M={M} K={K} Nout={Nout}", out, ref)


def bench(NF, H, W, C, N, taps, iters=10):
    x = torch.randn(NF, H, W, C, device=dev).half()
    w = (torch.randn(N, len(taps) * C, device=dev) / (len(taps) * C) ** 0.5).half()
    out = torch.empty(NF * H * W, N, device=dev, dtype=torch.half)
    for _ in range(3):
        ops.conv_gemm(x, w, taps=taps, out=out)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        ops.conv_gemm(x, w, taps=taps, out=out)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    fl = 2.0 * NF * H * W * N * len(taps) * C
    print(f"[bench] NF={NF} {H}x{W} C={C} N={N} taps={len(taps)}: {ms:.3f} ms  {fl / ms / 1e9:.1f} TFLOP/s", flush=True)


def bench2(M, K, N, geglu=False, res=False, iters=10):
    a = torch.randn(1, 1, M, K, device=dev).half()
    w = (torch.randn(N, K, device=dev) / K ** 0.5).half()
    b = torch.randn(N, device=dev)
    r = torch.randn(M, N, device=dev).half() if res else None
    out = torch.empty(M, N // 2 if geglu else N, device=dev, dtype=torch.half)
    for _ in range(3):
        ops.conv_gemm(a, w, bias=b, geglu=geglu, residual=r, out=out)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        ops.conv_gemm(a, w, bias=b, geglu=geglu, residual=r, out=out)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    print(f"[bench] M={M} K={K} N={N} geglu={geglu} res={res}: {ms:.3f} ms  {2.0 * M * N * K / ms / 1e9:.1f} TFLOP/s", flush=True)


if __name__ == "__main__":
    print(torch.cuda.get_device_name(0), flush=True)
    ok = True
    ok &= case_plain(128, 64, 64)
    ok &= case_plain(128, 64, 16)
    ok &= case_plain(256, 128, 128)
    ok &= case_plain(1000, 320, 320, bias=True)
    ok &= case_plain(4096, 1280, 1280, bias=True, res=True, alpha=0.5, beta=2.0)
    ok &= case_plain(100, 64, 48)
    ok &= case_plain(4096, 1280, 1280, bias=True, res=True, alpha=0.5)        # fast residual epilogue
    ok &= case_plain(1000, 320, 320, bias=True, res=True, alpha=0.37)         # fast residual epilogue, ragged M
    ok &= case_plain(40000, 320, 1152)                                         # fast plain epilogue, no bias
    ok &= case_plain(777, 640, 96, bias=True)                                  # N % 32 == 0, N < block tile
    ok &= case_geglu(139264 // 8, 320, 1280)
    ok &= case_geglu(1000, 640, 2560)
    ok &= case_conv3x3(2, 16, 16, 64, 64)
    ok &= case_conv3x3(3, 8, 8, 128, 320)
    ok &= case_conv3x3(2, 64, 64, 320, 320)
    ok &= case_conv3x3(2, 32, 32, 640, 640, C1=320)
    ok &= case_conv3x3(5, 4, 4, 64, 64)
    ok &= case_tconv(2, 5, 64, 320, 320)
    ok &= case_tconv(2, 17, 256, 640, 640)
    ok &= case_tconv(1, 3, 16, 64, 64)
    ok &= case_geglu(512, 320, 1280)
    print("ALL OK" if ok else "SOME FAILED", flush=True)
    if ok:
        bench(34, 64, 64, 320, 320, ops.TAPS_3X3)
        bench(34, 32, 32, 640, 640, ops.TAPS_3X3)
        bench(34, 16, 16, 1280, 1280, ops.TAPS_3X3)
        bench(34, 8, 8, 1280, 1280, ops.TAPS_3X3)
        bench(1, 1, 139264, 320, 2560, ops.TAPS_1)
        bench(1, 1, 139264, 1280, 320, ops.TAPS_1)
        bench(1, 1, 8192, 8192, 8192, ops.TAPS_1)
        bench2(139264, 320, 2560, geglu=True)
        bench2(34816, 640, 5120, geglu=True)
        bench2(139264, 320, 320, res=True)
        bench2(34816, 640, 640, res=True)
        bench2(139264, 320, 1152)
