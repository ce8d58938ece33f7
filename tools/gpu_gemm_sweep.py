"""Per-tile time of the GEMM kernel against the bytes a tile pulls into the SM (A + B operands): is it ingest-bound?"""
import sys
import torch
sys.path.insert(0, ".")
from musev_b200 import ops
dev = "cuda"
M = 139264
for K in (320, 640, 1280, 2560):
    for N in (64, 128, 192, 256):
        a = torch.randn(1, 1, M, K, device=dev).half()
        w = (torch.randn(N, K, device=dev) / K ** 0.5).half()
        out = torch.empty(M, N, device=dev, dtype=torch.half)
        for _ in range(3):
            ops.conv_gemm(a, w, out=out)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            ops.conv_gemm(a, w, out=out)
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 10
        tiles = (M // 128)
        waves = -(-tiles // 132)
        t_tile = ms * 1e3 / waves
        ingest = (128 + N) * K * 2 / 1024
        print(f"[sweep] K={K} N={N}: {ms*1e3:.1f} us  {2.0*M*N*K/ms/1e9:.0f} TF/s  per-tile {t_tile:.2f} us  ingest {ingest:.0f} KB/tile -> {ingest/t_tile*1.024:.0f} MB/s-per-us = GB/s per SM", flush=True)
