"""conv_gemm's 256-column tiles: the MMA warpgroups finish the plain, residual and GEGLU variants on their accumulator
fragments, write the fp16 results into a 128 x 256 output tile in shared memory and warp 1 stores it with TMA boxes
{32, bw, bh, bn}; for the residual variant warp 1 first TMA-loads the tile's residual runs into the same tile, and the
fragments read each residual from the place they then write. Every case has at least 3 x 132 tiles, so every CTA of a
132-SM grid runs three tiles or more and the output tile and the residual reload wrap. The cases cover GEGLU at K 320
with a ragged last tile, an in-place residual linear (out is the residual, as in the UNet's transformer blocks), a
residual 3x3 conv at N 1 280 whose pixel box is narrower than the image with ragged H / W edges, a plain 3x3 conv with
a time-embedding row-add, an N that is not a multiple of 256 written into a column window of a wider tensor (the
columns around the window keep their contents), and a long-K (5 120) residual linear.

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
M_RAGGED = 406 * 128 + 37            # >= 3 x 132 tiles of 128 rows x 256 columns, the last row of tiles partly filled
EPI = {"generic": 0, "plain": 1, "residual": 2, "geglu": 3, "act": 4}


def _linear(g, K, N):
    a = torch.randn(1, 1, M_RAGGED, K, generator=g).half().cuda()
    w = (torch.randn(N, K, generator=g) / K ** 0.5).half().cuda()
    return a, w, a.float().view(M_RAGGED, K) @ w.float().t()


def _conv3x3(g, NF, H, W, C, N):
    x = torch.randn(NF, H, W, C, generator=g).half().cuda()
    wt = (torch.randn(N, C, 3, 3, generator=g) / (9 * C) ** 0.5).half().cuda()
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), wt.float(), padding=1)
    return x, wt.permute(0, 2, 3, 1).reshape(N, -1).contiguous(), ref


def case_geglu_k320(ops, g):
    a, w, h = _linear(g, 320, 2560)
    b = torch.randn(2560, generator=g).cuda()
    nout = 1280                                  # [value | gate] rows -> the kernel's [16 value | 16 gate] chunks
    wp = torch.cat([w[:nout].view(-1, 16, 320), w[nout:].view(-1, 16, 320)], 1).reshape(w.shape).contiguous()
    bp = torch.cat([b[:nout].view(-1, 16), b[nout:].view(-1, 16)], 1).reshape(-1).contiguous()
    h = h + b
    return ops.conv_gemm(a, wp, bias=bp, geglu=True), h[:, :nout] * F.gelu(h[:, nout:])


def case_residual_inplace_k640(ops, g):
    a, w, h = _linear(g, 640, 1280)
    b = torch.randn(1280, generator=g).cuda()
    x = torch.randn(M_RAGGED, 1280, generator=g).half().cuda()
    ref = h + b + x.float()
    out = ops.conv_gemm(a, w, bias=b, residual=x, out=x)
    return out, ref


def case_residual_3x3_narrow_box(ops, g):
    NF, H, W, C, N = 11, 30, 46, 128, 1280      # box 16 x 8 x 1: the last box column and row partly outside W and H
    x, wt, ref = _conv3x3(g, NF, H, W, C, N)
    b = torch.randn(N, generator=g).cuda()
    res = torch.randn(NF * H * W, N, generator=g).half().cuda()
    out = ops.conv_gemm(x, wt, taps=ops.TAPS_3X3, bias=b, residual=res, alpha=0.5)
    return out, (ref + b[None, :, None, None]).permute(0, 2, 3, 1).reshape(-1, N) * 0.5 + res.float()


def case_plain_3x3_rowadd(ops, g):
    NF, H, W, C, N = 11, 30, 46, 64, 1280
    x, wt, ref = _conv3x3(g, NF, H, W, C, N)
    bias, temb = torch.randn(N, generator=g).cuda(), torch.randn(NF, N, generator=g).cuda()
    out = ops.conv_gemm(x, wt, taps=ops.TAPS_3X3, bias=bias, rowadd=temb, rows_per_group=H * W)
    ref = ref + bias[None, :, None, None] + temb[:, :, None, None]
    return out, ref.permute(0, 2, 3, 1).reshape(-1, N)


def case_plain_n1216_window(ops, g):
    a, w, h = _linear(g, 320, 1216)             # the last column tile holds 6 of its 8 runs
    b = torch.randn(1216, generator=g).cuda()
    wide = torch.full((M_RAGGED, 1504), 7.0, dtype=torch.float16, device="cuda")
    ops.conv_gemm(a, w, bias=b, out=wide[:, 160:1376])
    # the columns around the window must keep their contents
    untouched = bool((wide[:, :160] == 7).all() and (wide[:, 1376:] == 7).all())
    return wide[:, 160:1376], (h + b) if untouched else h + float("nan")


def case_residual_k5120(ops, g):
    a, w, h = _linear(g, 5120, 1280)
    b = torch.randn(1280, generator=g).cuda()
    res = torch.randn(M_RAGGED, 1280, generator=g).half().cuda()
    return ops.conv_gemm(a, w, bias=b, residual=res), h + b + res.float()


# name: epilogue variant; every case runs 256-column tiles with TMA epilogue I/O
CASES = {
    "geglu_k320": "geglu",
    "residual_inplace_k640": "residual",
    "residual_3x3_narrow_box": "residual",
    "plain_3x3_rowadd": "plain",
    "plain_n1216_window": "plain",
    "residual_k5120": "residual",
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
    print(json.dumps(results))


@pytest.fixture(scope="module")
def results(built_lib):
    r = subprocess.run([sys.executable, os.path.abspath(__file__)], env=dict(os.environ, MVB_TRACE="1"),
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("name", list(CASES))
def test_wide_epilogue(results, name):
    res = results[name]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert res["launches"] == 1
    assert (res["block_n"], res["epi"], res["epi_io"]) == (256, EPI[CASES[name]], "tma"), res
    assert res["tiles"] >= 3 * sms, res                       # every CTA runs at least three tiles
    assert res["shape_ok"] and not res["nan"], res
    assert res["err"] <= res["lim"], f"max_abs_err {res['err']:.3e} > {res['lim']:.3e}"


if __name__ == "__main__":
    _run_all()
