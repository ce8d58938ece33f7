"""conv_gemm with the epilogue on its own warpgroup: the MMA warpgroups hand each finished tile over through one staging
buffer (acc_full / acc_empty), whose phases only wrap once a CTA has run more than two tiles. Every case here has at least
3 x 132 x 128 output rows, so every CTA of a 132-SM grid runs three tiles or more, and together the cases cover each
epilogue variant, each tile width the selector picks (256 with the epilogue in line), row-add, a concatenated second A source, the stride-2 and the
(3,1,1) temporal conv, and ragged last tiles in rows and in columns.

The cases run in one child process with MVB_TRACE set (the library reads it once per process), which reports for each
case the tile width and epilogue variant its launch took, and its error against an fp32 torch reference."""
import json
import os
import subprocess
import sys
import tempfile

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M_RAGGED = 406 * 128 + 37            # >= 3 x 132 tiles of 128 rows, the last one partly filled
EPI = {"generic": 0, "plain": 1, "residual": 2, "geglu": 3, "act": 4}


def _linear(ops, g, K, N):
    a = torch.randn(1, 1, M_RAGGED, K, generator=g).half().cuda()
    w = (torch.randn(N, K, generator=g) / K ** 0.5).half().cuda()
    return a, w, a.float().view(M_RAGGED, K) @ w.float().t()


def _packed_geglu(w, b):
    """[value | gate] rows -> the kernel's [16 value | 16 gate] chunk order."""
    nout = w.shape[0] // 2
    wp = torch.cat([w[:nout].view(-1, 16, w.shape[1]), w[nout:].view(-1, 16, w.shape[1])], 1).reshape(w.shape).contiguous()
    bp = torch.cat([b[:nout].view(-1, 16), b[nout:].view(-1, 16)], 1).reshape(-1).contiguous()
    return wp, bp


def case_plain_bn64(ops, g):
    a, w, h = _linear(ops, g, 128, 64)
    b = torch.randn(64, generator=g).cuda()
    return ops.conv_gemm(a, w, bias=b), h + b


def case_plain_rowadd_concat_3x3_bn160(ops, g):
    NF, H, W, C0, C1, N = 13, 64, 64, 64, 64, 160
    x0 = torch.randn(NF, H, W, C0, generator=g).half().cuda()
    x1 = torch.randn(NF, H, W, C1, generator=g).half().cuda()
    wt = (torch.randn(N, C0 + C1, 3, 3, generator=g) / (9 * (C0 + C1)) ** 0.5).half().cuda()
    bias, temb = torch.randn(N, generator=g).cuda(), torch.randn(NF, N, generator=g).cuda()
    out = ops.conv_gemm(x0, wt.permute(0, 2, 3, 1).reshape(N, -1).contiguous(), taps=ops.TAPS_3X3, a1=x1, bias=bias,
                        rowadd=temb, rows_per_group=H * W)
    ref = F.conv2d(torch.cat([x0, x1], 3).float().permute(0, 3, 1, 2), wt.float(), bias, padding=1) + temb[:, :, None, None]
    return out, ref.permute(0, 2, 3, 1).reshape(-1, N)


def case_residual_bn128(ops, g):
    a, w, h = _linear(ops, g, 320, 128)
    b = torch.randn(128, generator=g).cuda()
    res = torch.randn(M_RAGGED, 128, generator=g).half().cuda()
    return ops.conv_gemm(a, w, bias=b, residual=res, alpha=0.5), (h + b) * 0.5 + res.float()


def case_residual_temporal_bn160(ops, g):
    B, T, HW, C, N = 2, 8, 4096, 64, 160
    x = torch.randn(B, T, HW, C, generator=g).half().cuda()
    wt = (torch.randn(N, C, 3, generator=g) / (3 * C) ** 0.5).half().cuda()
    res = torch.randn(B * T * HW, N, generator=g).half().cuda()
    out = ops.conv_gemm(x, wt.permute(0, 2, 1).reshape(N, 3 * C).contiguous(), taps=ops.TAPS_T3, residual=res)
    ref = F.conv1d(x.float().permute(0, 2, 3, 1).reshape(B * HW, C, T), wt.float(), padding=1)
    return out, ref.reshape(B, HW, N, T).permute(0, 3, 1, 2).reshape(-1, N) + res.float()


def case_generic_residual_beta_bn160(ops, g):
    a, w, h = _linear(ops, g, 64, 320)
    b = torch.randn(320, generator=g).cuda()
    res = torch.randn(M_RAGGED, 320, generator=g).half().cuda()
    return ops.conv_gemm(a, w, bias=b, residual=res, beta=2.0), h + b + 2.0 * res.float()


def case_generic_ragged_n_bn128(ops, g):
    a, w, h = _linear(ops, g, 192, 72)
    b = torch.randn(72, generator=g).cuda()
    res = torch.randn(M_RAGGED, 72, generator=g).half().cuda()
    return ops.conv_gemm(a, w, bias=b, residual=res), h + b + res.float()


def case_generic_stride2_bn128(ops, g):
    NF, H, W, C, N = 13, 128, 128, 64, 128
    x = torch.randn(NF, H, W, C, generator=g).half().cuda()
    wt = (torch.randn(N, C, 3, 3, generator=g) / (9 * C) ** 0.5).half().cuda()
    b = torch.randn(N, generator=g).cuda()
    out = ops.conv_gemm(x, wt.permute(0, 2, 3, 1).reshape(N, 9 * C).contiguous(), taps=ops.TAPS_3X3, bias=b, alpha=0.5,
                        stride2=True)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), wt.float(), b, stride=2, padding=1) * 0.5
    return out, ref.permute(0, 2, 3, 1).reshape(-1, N)


def case_geglu_bn128(ops, g):
    a, w, h = _linear(ops, g, 320, 128)
    b = torch.randn(128, generator=g).cuda()
    wp, bp = _packed_geglu(w, b)
    h = h + b
    return ops.conv_gemm(a, wp, bias=bp, geglu=True), h[:, :64] * F.gelu(h[:, 64:])


def case_generic_geglu_ragged_n_bn128(ops, g):
    a, w, h = _linear(ops, g, 128, 96)          # N % 64 != 0: the generic epilogue's GEGLU branch, a ragged column tile
    b = torch.randn(96, generator=g).cuda()
    wp, bp = _packed_geglu(w, b)
    h = h + b
    return ops.conv_gemm(a, wp, bias=bp, geglu=True), h[:, :48] * F.gelu(h[:, 48:])


def case_gelu_bn160(ops, g):
    a, w, h = _linear(ops, g, 128, 160)
    b = torch.randn(160, generator=g).cuda()
    return ops.conv_gemm(a, w, bias=b, act=2), F.gelu(h + b)


def case_quick_gelu_bn64(ops, g):
    a, w, h = _linear(ops, g, 256, 64)
    b = torch.randn(64, generator=g).cuda()
    return ops.conv_gemm(a, w, bias=b, act=3), (h + b) * torch.sigmoid(1.702 * (h + b))


def case_residual_bn256_inline(ops, g):
    a, w, h = _linear(ops, g, 128, 1280)          # BN = 256 keeps the epilogue in the MMA warpgroups
    b = torch.randn(1280, generator=g).cuda()
    res = torch.randn(M_RAGGED, 1280, generator=g).half().cuda()
    return ops.conv_gemm(a, w, bias=b, residual=res), h + b + res.float()


def case_f32_silu_bn128(ops, g):
    a, w, h = _linear(ops, g, 320, 128)
    b = torch.randn(128, generator=g).cuda()
    return ops.conv_gemm(a, w, bias=b, act=1, out_f32=True), F.silu(h + b)


# name: (tile width, epilogue variant the launch must take)
CASES = {
    "plain_bn64": (64, "plain"),
    "plain_rowadd_concat_3x3_bn160": (160, "plain"),
    "residual_bn128": (128, "residual"),
    "residual_temporal_bn160": (160, "residual"),
    "generic_residual_beta_bn160": (160, "generic"),
    "generic_ragged_n_bn128": (128, "generic"),
    "generic_stride2_bn128": (128, "generic"),
    "geglu_bn128": (128, "geglu"),
    "generic_geglu_ragged_n_bn128": (128, "generic"),
    "gelu_bn160": (160, "act"),
    "quick_gelu_bn64": (64, "act"),
    "f32_silu_bn128": (128, "generic"),
    "residual_bn256_inline": (256, "residual"),
}


def _run_all():
    """Child process: every case, one JSON line each (tile width and variant from the MVB_TRACE line of its launch)."""
    sys.path.insert(0, ROOT)
    from musev_b200 import ops
    results = {}
    for name in CASES:
        g = torch.Generator().manual_seed(sum(map(ord, name)))
        sys.stderr.flush()
        saved = os.dup(2)
        with tempfile.TemporaryFile(mode="w+") as log:
            os.dup2(log.fileno(), 2)
            try:
                out, ref = globals()["case_" + name](ops, g)
                torch.cuda.synchronize()
            finally:
                os.dup2(saved, 2)
                os.close(saved)
            log.seek(0)
            trace = [dict(kv.split("=", 1) for kv in ln.split()[2:]) for ln in log.read().splitlines()
                     if ln.startswith("MVB_TRACE gemm")]
        f32 = out.dtype == torch.float32
        rel, abs_ = (1e-4, 1e-4) if f32 else (3e-3, 2e-3)
        results[name] = {
            "launches": len(trace), "block_n": int(trace[0]["block_n"]) if trace else None,
            "epi": int(trace[0]["epi"]) if trace else None, "tiles": int(trace[0]["tiles"]) if trace else None,
            "err": (out.float() - ref).abs().max().item(), "lim": abs_ + rel * ref.abs().max().item(),
            "nan": bool(torch.isnan(out.float()).any()), "shape_ok": list(out.shape) == list(ref.shape),
        }
    print(json.dumps(results))


@pytest.fixture(scope="module")
def results(built_lib):
    r = subprocess.run([sys.executable, os.path.abspath(__file__)], env=dict(os.environ, MVB_TRACE="1"),
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("name", list(CASES))
def test_overlapped_epilogue(results, name):
    bn, variant = CASES[name]
    res = results[name]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert res["launches"] == 1
    assert (res["block_n"], res["epi"]) == (bn, EPI[variant]), res
    assert res["tiles"] >= 3 * sms, res                       # every CTA runs at least three tiles
    assert res["shape_ok"] and not res["nan"], res
    assert res["err"] <= res["lim"], f"max_abs_err {res['err']:.3e} > {res['lim']:.3e}"


if __name__ == "__main__":
    _run_all()
