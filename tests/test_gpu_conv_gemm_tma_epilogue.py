"""conv_gemm's TMA epilogue: at tile widths up to 160 the plain, residual and GEGLU variants write each 32-column run of
fp16 outputs into shared memory and store it as one TMA box {32, bw, bh, bn} of a {columns, W, H, NF} view, and the
residual variant reads its residual runs through a ring that a second producer warp fills with TMA loads. Every case has
at least 3 x 132 tiles, so every CTA of a 132-SM grid runs three tiles or more and the ring and the staging wrap. The
cases cover residual linears at K 320 / 640 / 1 280 with a ragged last tile, an in-place residual (out is the
residual, as in the UNet's transformer blocks), a 3x3 conv whose pixel box is narrower than the image with ragged
H / W edges, the (3,1,1) temporal conv, GEGLU (N / 2 output columns), plain with row-add and a concatenated second
source, an output that is a column window of a wider tensor, and the generic epilogue, which keeps per-thread loads and
stores. A residual whose rows are not whole 16-byte vectors is refused before launch.

The cases run in one child process with MVB_TRACE set (the library reads it once per process), which reports for each
case the tile width, the epilogue variant and the epilogue I/O path its launch took, and its error against an fp32
torch reference."""
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


def _linear(g, K, N):
    a = torch.randn(1, 1, M_RAGGED, K, generator=g).half().cuda()
    w = (torch.randn(N, K, generator=g) / K ** 0.5).half().cuda()
    return a, w, a.float().view(M_RAGGED, K) @ w.float().t()


def _residual_linear(ops, g, K, N=320, alpha=1.0):
    a, w, h = _linear(g, K, N)
    b = torch.randn(N, generator=g).cuda()
    res = torch.randn(M_RAGGED, N, generator=g).half().cuda()
    return ops.conv_gemm(a, w, bias=b, residual=res, alpha=alpha), (h + b) * alpha + res.float()


def case_residual_k320(ops, g):
    return _residual_linear(ops, g, 320, alpha=0.5)


def case_residual_k640(ops, g):
    return _residual_linear(ops, g, 640)


def case_residual_k1280(ops, g):
    return _residual_linear(ops, g, 1280)


def case_residual_bn128(ops, g):
    return _residual_linear(ops, g, 320, N=128)


def case_residual_bn64(ops, g):
    return _residual_linear(ops, g, 320, N=64)


def case_residual_inplace_k640(ops, g):
    a, w, h = _linear(g, 640, 640)
    b = torch.randn(640, generator=g).cuda()
    x = torch.randn(M_RAGGED, 640, generator=g).half().cuda()
    ref = h + b + x.float()
    out = ops.conv_gemm(a, w, bias=b, residual=x, out=x)
    return out, ref


def case_plain_3x3_narrow_box(ops, g):
    NF, H, W, C, N = 11, 30, 46, 128, 640       # box 16 x 8 x 1: the last box column and row partly outside W and H
    x = torch.randn(NF, H, W, C, generator=g).half().cuda()
    wt = (torch.randn(N, C, 3, 3, generator=g) / (9 * C) ** 0.5).half().cuda()
    b = torch.randn(N, generator=g).cuda()
    out = ops.conv_gemm(x, wt.permute(0, 2, 3, 1).reshape(N, -1).contiguous(), taps=ops.TAPS_3X3, bias=b)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), wt.float(), b, padding=1)
    return out, ref.permute(0, 2, 3, 1).reshape(-1, N)


def case_residual_temporal(ops, g):
    B, T, HW, C, N = 2, 9, 2900, 320, 320       # W = 2900 pixels: a ragged last box
    x = torch.randn(B, T, HW, C, generator=g).half().cuda()
    wt = (torch.randn(N, C, 3, generator=g) / (3 * C) ** 0.5).half().cuda()
    res = torch.randn(B * T * HW, N, generator=g).half().cuda()
    out = ops.conv_gemm(x, wt.permute(0, 2, 1).reshape(N, 3 * C).contiguous(), taps=ops.TAPS_T3, residual=res, alpha=0.75)
    ref = F.conv1d(x.float().permute(0, 2, 3, 1).reshape(B * HW, C, T), wt.float(), padding=1)
    return out, ref.reshape(B, HW, N, T).permute(0, 3, 1, 2).reshape(-1, N) * 0.75 + res.float()


def case_geglu(ops, g):
    a, w, h = _linear(g, 640, 256)
    b = torch.randn(256, generator=g).cuda()
    nout = 128                                   # [value | gate] rows -> the kernel's [16 value | 16 gate] chunks
    wp = torch.cat([w[:nout].view(-1, 16, 640), w[nout:].view(-1, 16, 640)], 1).reshape(w.shape).contiguous()
    bp = torch.cat([b[:nout].view(-1, 16), b[nout:].view(-1, 16)], 1).reshape(-1).contiguous()
    h = h + b
    return ops.conv_gemm(a, wp, bias=bp, geglu=True), h[:, :nout] * F.gelu(h[:, nout:])


def case_plain_rowadd_concat(ops, g):
    NF, H, W, C0, C1, N = 13, 36, 20, 64, 128, 320
    x0 = torch.randn(NF, H, W, C0, generator=g).half().cuda()
    x1 = torch.randn(NF, H, W, C1, generator=g).half().cuda()
    wt = (torch.randn(N, C0 + C1, 3, 3, generator=g) / (9 * (C0 + C1)) ** 0.5).half().cuda()
    bias, temb = torch.randn(N, generator=g).cuda(), torch.randn(NF, N, generator=g).cuda()
    out = ops.conv_gemm(x0, wt.permute(0, 2, 3, 1).reshape(N, -1).contiguous(), taps=ops.TAPS_3X3, a1=x1, bias=bias,
                        rowadd=temb, rows_per_group=H * W)
    ref = F.conv2d(torch.cat([x0, x1], 3).float().permute(0, 3, 1, 2), wt.float(), bias, padding=1) + temb[:, :, None, None]
    return out, ref.permute(0, 2, 3, 1).reshape(-1, N)


def case_plain_out_window(ops, g):
    a, w, h = _linear(g, 320, 320)
    wide = torch.full((M_RAGGED, 576), 7.0, dtype=torch.float16, device="cuda")
    ops.conv_gemm(a, w, out=wide[:, 192:512])
    # the columns around the window must keep their contents
    untouched = bool((wide[:, :192] == 7).all() and (wide[:, 512:] == 7).all())
    return wide[:, 192:512], h if untouched else h + float("nan")


def case_generic_residual_beta(ops, g):
    a, w, h = _linear(g, 320, 320)
    res = torch.randn(M_RAGGED, 320, generator=g).half().cuda()
    return ops.conv_gemm(a, w, residual=res, beta=0.5), h + 0.5 * res.float()


# name: (tile width, epilogue variant, epilogue I/O path)
CASES = {
    "residual_k320": (160, "residual", "tma"),
    "residual_k640": (160, "residual", "tma"),
    "residual_k1280": (160, "residual", "tma"),
    "residual_bn128": (128, "residual", "tma"),
    "residual_bn64": (64, "residual", "tma"),
    "residual_inplace_k640": (160, "residual", "tma"),
    "plain_3x3_narrow_box": (160, "plain", "tma"),
    "residual_temporal": (160, "residual", "tma"),
    "geglu": (128, "geglu", "tma"),
    "plain_rowadd_concat": (64, "plain", "tma"),
    "plain_out_window": (160, "plain", "tma"),
    "generic_residual_beta": (160, "generic", "lsu"),
}


def _run_all():
    """Child process: every case, one JSON line each (launch fields from the MVB_TRACE line of its launch)."""
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
        t = trace[0] if trace else {}
        results[name] = {
            "launches": len(trace), "block_n": int(t.get("block_n", -1)), "epi": int(t.get("epi", -1)),
            "epi_io": t.get("epi_io"), "tiles": int(t.get("tiles", -1)),
            "err": (out.float() - ref).abs().max().item(), "lim": 2e-3 + 3e-3 * ref.abs().max().item(),
            "nan": bool(torch.isnan(out.float()).any() or torch.isnan(ref).any()),
            "shape_ok": list(out.shape) == list(ref.shape),
        }
    # a residual view 2 bytes off a 16-byte boundary, with a row stride of 321 elements: refused, nothing launched
    g = torch.Generator().manual_seed(1)
    a, w, _ = _linear(g, 320, 320)
    base = torch.zeros(M_RAGGED, 321, dtype=torch.float16, device="cuda")
    try:
        ops.conv_gemm(a, w, residual=base[:, 1:])
        results["unaligned_residual"] = None
    except Exception as e:  # noqa: BLE001 -- the library's error, whichever Python type carries it
        results["unaligned_residual"] = str(e)
    torch.cuda.synchronize()
    print(json.dumps(results))


@pytest.fixture(scope="module")
def results(built_lib):
    r = subprocess.run([sys.executable, os.path.abspath(__file__)], env=dict(os.environ, MVB_TRACE="1"),
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("name", list(CASES))
def test_tma_epilogue(results, name):
    bn, variant, io = CASES[name]
    res = results[name]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert res["launches"] == 1
    assert (res["block_n"], res["epi"], res["epi_io"]) == (bn, EPI[variant], io), res
    assert res["tiles"] >= 3 * sms, res                       # every CTA runs at least three tiles
    assert res["shape_ok"] and not res["nan"], res
    assert res["err"] <= res["lim"], f"max_abs_err {res['err']:.3e} > {res['lim']:.3e}"


def test_unaligned_residual_refused(results):
    assert results["unaligned_residual"] is not None and "residual must be 16-byte aligned" in results["unaligned_residual"]


if __name__ == "__main__":
    _run_all()
