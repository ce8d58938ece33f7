"""conv_gemm at every reachable (tile width, epilogue) instantiation, at the K depths that wrap its operand ring and at
the shapes and epilogue options where it goes wrong, against one float64 reference of the operation the header
documents:
    out[m, n] = act((sum_{tap, c} A[pixel(m) + tap, c] W[n, tap (C0 + C1) + c] + bias[n] + rowadd[m / rpg, n]) alpha
                    + beta res[m, n])
with GEGLU on the packed [16 value | 16 gate] chunks (bias only). The reference is computed on the device from per-tap
shifted views of the fp16 inputs upcast to float64 with explicit zero padding, one float64 matmul per tap; the same
code takes 1-tap, 3x3 and (3,1,1) taps, two concatenated sources, stride 2 with either pad mode and strided views.

Every element is held to its own bound, never one relative to the tensor's maximum:
    |out - ref| <= ulp16(ref) / 2 + C_ACC S_acc + 2^-23 S_epi (+ 1e-6 |pre-activation| with an activation)
where S_acc = |alpha| slope sum |a| |w| (a second float64 GEMM on absolute values), S_epi the magnitudes of the fp32
epilogue terms, slope 1.13 (the largest slope of GELU, SiLU and quick-GELU) with an activation and 1 without; for
GEGLU the two halves are weighted by |gelu(gate)| and |value| slope. fp32 outputs drop the ulp16 term. The bound
discriminates: on small host shapes of each group the test computes named wrong answers in float64 (a 64-channel K
block left out, also at the longest K; the last k16 step left out; the accumulator rounded to fp16 before the
epilogue; the residual added before alpha; the row-add group of the tile's first row; GELU in its tanh form;
quick-GELU's 1.702 replaced by exact GELU; a temporal tap reading the neighbouring video; stride-2 pad mode 1 for
mode 2; GEGLU value and gate swapped), rounds them as the kernel would and asserts that each breaks the bound
(`test_*_bounds_catch_wrong_answers`, no GPU).

A mirror of the host arithmetic of conv_gemm.cu (`pick_box`, `pick_block_n`, `ring_stages`, the epilogue selection of
`launch_common`) gives each case's plan: tile width, epilogue variant, epilogue I/O path, ring depth, tiles and K
blocks per tile. Each case states the plan it is meant to reach (checked on the host at 132 SMs), and on the GPU the
MVB_TRACE line of its launch must equal the mirror's plan at the device's SM count, so a case that drifts onto another
path fails. The matrix runs every reachable (BN, epilogue) at 1, nstages - 1, nstages and nstages + 1 K blocks per
tile and at a long K, each with at least 3 tiles per CTA and the ring wrapping at least twice (in the middle of a tile
for nstages +- 1), ragged last row tiles, bias on and off, plus ragged column tiles; then grid shapes, A operands,
epilogue options and the distinct launches of one full-width UNet forward per preset, replayed on seeded data.

All GPU cases run in one child process with MVB_TRACE set (the library reads it once per process); the file takes
about 35 s on the GPU. With MVB_PARITY_LOG=<file> set, the worst ratio |out - ref| / bound of every case is appended
to <file>. Measured on an H100 80GB HBM3 at 700 W, worst ratio per group: matrix plain 0.993, residual 0.997, generic
0.994, GEGLU 0.977, GELU 0.990; grid shapes 0.984; A operands 0.991 (t3_T1_B3); epilogue options 0.991; the earlier
per-feature rows 0.996; engine launches 0.989 (musev), 0.991 (musev_referencenet). Near 1 for fp16 outputs because a
correctly rounded result may sit half an ulp away. The fp32-output cases carry no rounding term and measure the wgmma
accumulation: 0.599 at K = 23 040, 0.366 at K = 5 120, 0.10 at K = 320 with C_ACC = 2.5e-6, i.e. an accumulation error
of at most 1.5e-6 sum |a| |w| at the longest K; C_ACC keeps 1.7x above that.
"""
import json
import math
import os
import subprocess
import sys
import tempfile
import zlib
from dataclasses import dataclass, field

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C_ACC = 2.5e-6
ACT_SLOPE = 1.13
EPS_EPI = 2.0 ** -23
HOST_SMS = 132

TAPS = {"1": ((0, 0),), "3x3": tuple((dy, dx) for dy in (-1, 0, 1) for dx in (-1, 0, 1)), "t3": ((-1, 0), (0, 0), (1, 0))}
EPI = {"generic": 0, "plain": 1, "residual": 2, "geglu": 3, "act": 4}
EPI_NAME = {v: k for k, v in EPI.items()}
# the shared-memory budget per (epilogue, tile width), as conv_gemm.cu's static_assert states it
NSTAGES = {(e, bn): n for bn, row in ((64, (8, 8, 6, 8, 8)), (128, (5, 5, 4, 5, 5)), (160, (4, 4, 3, 4, 4)),
                                      (256, (None, 3, 3, 3, None))) for e, n in enumerate(row) if n}
# the kernel table of launch_common: no generic / GELU epilogue at BN 256, no GEGLU at BN 160
REACHABLE = sorted(NSTAGES.keys() - {(3, 160)}, key=lambda k: (k[1], k[0]))


# ------------------------------------------------------------------------------------------------ plan mirror
def ceil_div(a, b):
    return -(-a // b)


def ring_stages(epi, bn):
    """ring_stages (conv_gemm.cu:71-82)."""
    inline = bn == 256
    epi_buf = 128 * bn * (2 if inline else 4)
    res_ring = 4 * 128 * 32 * 2 if (not inline and epi == EPI["residual"]) else 0
    bias_buf = 256 * 4 if inline else 160 * 4
    ring = 227 * 1024 - epi_buf - res_ring - bias_buf - 1024 - 256
    return min(ring // (16384 + ceil_div(bn * 64 * 2, 1024) * 1024), 8)


def pick_box(W, H, NF):
    """pick_box: the power-of-two pixel box of 128 rows that wastes the fewest padded rows (first found wins)."""
    best, box = None, None
    w = 128
    while w >= 1:
        h = 128 // w
        while h >= 1:
            n = 128 // (w * h)
            padded = ceil_div(W, w) * ceil_div(H, h) * ceil_div(NF, n)
            if best is None or padded < best:
                best, box = padded, (w, h, n)
            h //= 2
        w //= 2
    return box


def pick_block_n(N, geglu, wide_ok, tiles_m, sms):
    best, best_cost = 0, 1e30
    for bn in (256, 160, 128, 64):
        if (geglu and bn % 64) or (not wide_ok and bn == 256):
            continue
        waves = ceil_div(tiles_m * ceil_div(N, bn), sms)
        cost = waves * (bn + 24.0)
        if cost < best_cost - 1e-9:
            best, best_cost = bn, cost
    return best


def select_epi(N, geglu, res, alpha, beta, act, f32):
    epi = EPI["generic"]
    if not f32 and act == 0:
        if geglu:
            if N % 64 == 0:
                epi = EPI["geglu"]
        elif N % 32 == 0:
            if res and beta == 1.0:
                epi = EPI["residual"]
            elif not res and alpha == 1.0:
                epi = EPI["plain"]
    if act in (2, 3):
        epi = EPI["act"]
    return epi


def plan(W, H, NF, ntaps, kb_per_tap, N, geglu=False, res=False, alpha=1.0, beta=1.0, act=0, f32=False, sms=HOST_SMS):
    """What launch_common does with a launch of output image W x H x NF: the plan fields MVB_TRACE reports, and the
    per-CTA schedule (tiles of the least loaded CTA, ring wraps over them, whether a wrap falls inside a tile)."""
    bw, bh, bnf = pick_box(W, H, NF)
    tiles_m = ceil_div(W, bw) * ceil_div(H, bh) * ceil_div(NF, bnf)
    epi = select_epi(N, geglu, res, alpha, beta, act, f32)
    block_n = pick_block_n(N, geglu, epi in (1, 2, 3), tiles_m, sms)
    tiles = tiles_m * ceil_div(N, block_n)
    nstages = ring_stages(epi, block_n)
    kb = ntaps * kb_per_tap
    per_cta = tiles // min(tiles, sms)
    wraps = per_cta * kb // nstages
    return {"block_n": block_n, "epi": epi, "epi_io": "tma" if epi in (1, 2, 3) else "lsu", "nstages": nstages,
            "tiles": tiles, "kb": kb, "box": (bw, bh, bnf), "tiles_per_cta": per_cta, "wraps": wraps,
            "mid_tile_wrap": any((j * nstages) % kb for j in range(1, wraps + 1)),
            "ragged_rows": W * H * NF % 128 != 0 or (W % bw, H % bh, NF % bnf) != (0, 0, 0),
            "ragged_cols": N % block_n != 0}


# ------------------------------------------------------------------------------------------------ cases
@dataclass(frozen=True)
class Case:
    id: str
    NF: int
    H: int
    W: int            # input image; a linear layer is NF = H = 1, W = M
    C0: int
    N: int
    C1: int = 0
    taps: str = "1"
    s2: int = 0       # stride-2 pad mode
    a0_view: str = "dense"   # "chwin": channels [64, 64 + C0) of a wider tensor; "fstride": every other frame
    bias: bool = True
    rpg: int = 0      # rows per row-add group (0: no row-add)
    ld_rowadd_pad: int = 0
    res: str = ""     # "dense", "window" (a column window of a wider tensor), "inplace" (out = res, inside a window)
    alpha: float = 1.0
    beta: float = 1.0
    geglu: bool = False
    act: int = 0
    f32: bool = False
    out_pad: tuple = (0, 0)   # columns kept around the output window, left and right
    expect: dict = field(default_factory=dict, hash=False, compare=False)
    per_cta3: bool = False    # every CTA runs at least three tiles

    @property
    def ntaps(self):
        return 9 if self.s2 else len(TAPS[self.taps])

    @property
    def out_hw(self):
        return (self.H // 2, self.W // 2) if self.s2 else (self.H, self.W)

    @property
    def M(self):
        return self.NF * self.out_hw[0] * self.out_hw[1]

    @property
    def nout(self):
        return self.N // 2 if self.geglu else self.N

    def plan(self, sms=HOST_SMS):
        Ho, Wo = self.out_hw
        return plan(Wo, Ho, self.NF, self.ntaps, (self.C0 + self.C1) // 64, self.N, self.geglu, bool(self.res),
                    self.alpha, self.beta, self.act, self.f32, sms)


def _pair_options(bn, epi):
    """Epilogue options and N that select (bn, epi); their ragged-column N (None where the path has none)."""
    name = EPI_NAME[epi]
    if name == "generic":
        return dict(res="dense", beta=0.5), bn, {64: 40, 128: 96, 160: 288}[bn]
    if name == "plain":
        return {}, bn, {64: 32, 128: 96, 160: 288, 256: 1216}[bn]
    if name == "residual":
        return dict(res="dense", alpha=0.5), bn, {64: 32, 128: 96, 160: 288, 256: 1216}[bn]
    if name == "geglu":
        return dict(geglu=True), bn, {256: 1216}.get(bn)
    return dict(act=2 if bn != 128 else 3), bn, {64: 40, 128: 104, 160: 288}[bn]


def _linear_rows(tiles_m):
    return (tiles_m - 1) * 128 + 37          # a ragged last row tile


def matrix_cases(sms):
    cs = []
    for epi, bn in REACHABLE:
        opts, N, n_ragged = _pair_options(bn, epi)
        ns = NSTAGES[(epi, bn)]
        exp = dict(block_n=bn, epi=epi, nstages=ns)
        for tag, kb in (("kb1", 1), ("kbns-1", ns - 1), ("kbns", ns), ("kbns+1", ns + 1), ("kblong", 36)):
            # tiles per CTA: at least 3 and two ring wraps. With one extra row tile, 256-wide tiles win over two
            # 128-wide ones only from 6 waves on (pick_block_n's cost per wave)
            t = max(8 if bn == 256 else 3, ceil_div(2 * ns, kb))
            cs.append(Case(f"m_{EPI_NAME[epi]}_bn{bn}_{tag}", 1, 1, _linear_rows(t * sms + 1), 64 * kb, N,
                           bias=tag in ("kb1", "kbns", "kblong"), expect=dict(exp, kb=kb), per_cta3=True, **opts))
        if n_ragged:
            kb = ns + 1
            cs.append(Case(f"m_{EPI_NAME[epi]}_bn{bn}_ragged_n{n_ragged}", 1, 1, _linear_rows(3 * sms + 1), 64 * kb,
                           n_ragged, expect=dict(exp, kb=kb), per_cta3=True, **opts))
    return cs


M_OLD = 406 * 128 + 37       # the earlier per-feature cases: >= 3 x 132 tiles, the last row tile partly filled


def special_cases(sms):
    def lin(id, K, N, rows=None, **kw):
        return Case(id, 1, 1, rows or _linear_rows(3 * sms + 1), K, N, **kw)

    def e(bn, epi, **kw):
        return dict(block_n=bn, epi=EPI[epi], **kw)

    cs = [
        # grid shapes
        lin("grid_k_sms_plus_1", 640, 160, rows=2 * sms * 128 + 1, expect=e(160, "plain", tiles=2 * sms + 1)),
        lin("grid_tiles_lt_sms", 320, 128, rows=40 * 128 + 5, expect=e(64, "plain", tiles=82)),
        lin("grid_single_tile_m100", 128, 64, rows=100, res="dense", expect=e(64, "residual", tiles=1)),
        # 3x3 at the lowest UNet levels: images smaller than the pixel box, NF ragged against it
        Case("a_3x3_1x1_nf130_rowadd", 130, 1, 1, 1280, 1280, taps="3x3", rpg=1, expect=e(64, "plain", box=(1, 1, 128))),
        Case("a_3x3_2x2_nf70_res", 70, 2, 2, 640, 640, taps="3x3", res="dense", alpha=0.5, expect=e(64, "residual", box=(2, 2, 32))),
        Case("a_3x3_4x4_nf20_silu", 20, 4, 4, 640, 1280, taps="3x3", act=1, expect=e(64, "generic", box=(4, 4, 8))),
        Case("a_3x3_8x8_nf10", 10, 8, 8, 320, 640, taps="3x3", rpg=64, expect=e(64, "plain", box=(8, 8, 2))),
        Case("a_3x3_30x46_nf11", 11, 30, 46, 128, 640, taps="3x3", expect=e(160, "plain", box=(16, 8, 1))),
        # concatenated sources, C0 != C1, both orders
        Case("a_concat_64_128", 13, 36, 20, 64, 320, C1=128, taps="3x3", rpg=36 * 20, expect=e(64, "plain")),
        Case("a_concat_128_64", 13, 36, 20, 128, 320, C1=64, taps="3x3", rpg=36 * 20, expect=e(64, "plain")),
        # temporal taps over several videos: NF = videos, H = frames
        Case("a_t3_T1_B3", 3, 1, 1000, 320, 320, taps="t3", res="dense", expect=e(64, "residual")),
        Case("a_t3_T2_B3", 3, 2, 700, 320, 320, taps="t3", expect=e(128, "plain")),
        Case("a_t3_T9_B2", 2, 9, 2900, 320, 320, taps="t3", res="dense", alpha=0.75, expect=e(160, "residual")),
        # stride 2, both pad modes, smallest even sizes and H != W
        Case("a_s2_pad1_2x2", 5, 2, 2, 64, 64, s2=1, expect=e(64, "plain")),
        Case("a_s2_pad2_2x2", 5, 2, 2, 64, 64, s2=2, expect=e(64, "plain")),
        Case("a_s2_pad1_8x12", 3, 8, 12, 128, 128, s2=1, res="dense", expect=e(64, "residual", tiles=2)),
        Case("a_s2_pad2_12x8", 3, 12, 8, 128, 128, s2=2, alpha=0.5, expect=e(64, "generic", tiles=2)),
        # strided A views
        Case("a_chwin_3x3", 3, 16, 24, 64, 128, taps="3x3", a0_view="chwin", expect=e(64, "plain")),
        Case("a_fstride_t3", 4, 3, 200, 128, 128, taps="t3", a0_view="fstride", expect=e(64, "plain")),
        Case("a_fstride_3x3_concat", 3, 8, 8, 64, 64, C1=64, taps="3x3", a0_view="fstride", expect=e(64, "plain")),
        # the longest K the UNet runs: 3x3 over 1280 + 1280 channels, K = 23 040
        Case("a_k23040_3x3_concat", 10, 4, 4, 1280, 1280, C1=1280, taps="3x3", expect=e(64, "plain", kb=360)),
        Case("a_k23040_res", 10, 8, 8, 1280, 1280, C1=1280, taps="3x3", res="dense", expect=e(64, "residual", kb=360)),
        # fp32 outputs carry no fp16 rounding: these measure the accumulation against C_ACC, also at the longest K
        Case("a_k23040_f32", 10, 4, 4, 1280, 1280, C1=1280, taps="3x3", f32=True, expect=e(64, "generic", kb=360)),
        lin("e_k5120_f32", 5120, 256, f32=True, expect=e(128, "generic", kb=80)),
        # row-add groups: one row, a size not dividing 128, 4 096; a row-add wider than N
        lin("e_rowadd_rpg1", 128, 128, rpg=1, expect=e(128, "plain")),
        lin("e_rowadd_rpg100_ld", 320, 320, rpg=100, ld_rowadd_pad=24, expect=e(160, "plain")),
        lin("e_rowadd_rpg4096", 320, 1280, rpg=4096, expect=e(256, "plain")),
        lin("e_rowadd_rpg100_generic", 128, 200, rpg=100, ld_rowadd_pad=8, expect=e(128, "generic")),
        # residual layouts
        lin("e_res_window", 320, 320, res="window", expect=e(160, "residual", epi_io="tma")),
        lin("e_res_inplace_window_tma", 640, 640, res="inplace", out_pad=(32, 64), expect=e(160, "residual", epi_io="tma")),
        lin("e_res_inplace_window_lsu", 640, 640, res="inplace", beta=0.5, out_pad=(32, 64), expect=e(160, "generic", epi_io="lsu")),
        lin("e_res_inplace_window_bn256", 640, 1280, res="inplace", out_pad=(64, 32), expect=e(256, "residual", epi_io="tma")),
        # output windows whose surrounding columns must stay untouched
        lin("e_out_window_lsu", 320, 200, out_pad=(8, 16), expect=e(128, "generic")),
        lin("e_out_window_f32", 320, 128, act=1, f32=True, out_pad=(4, 12), expect=e(128, "generic")),
        # GEGLU with N % 64 != 0 (generic epilogue)
        lin("e_geglu_n96", 128, 96, geglu=True, expect=e(128, "generic")),
        lin("e_geglu_n160", 320, 160, geglu=True, expect=e(64, "generic")),
    ]
    for N, exp in ((8, e(64, "generic")), (24, e(64, "generic")), (40, e(64, "generic")), (72, e(128, "generic")),
                   (200, e(128, "generic")), (1216, e(256, "plain"))):
        cs.append(lin(f"e_n{N}", 192, N, expect=exp))
    for act, f32 in ((1, False), (1, True), (2, False), (2, True), (3, False), (3, True)):
        cs.append(lin(f"e_act{act}_{'f32' if f32 else 'f16'}", 320, 128, act=act, f32=f32,
                      expect=e(128, "generic" if act == 1 else "act")))
    return cs


def old_cases(sms):
    """The cases of the earlier per-feature conv_gemm files, same shapes and options, with >= 3 tiles per CTA."""
    def lin(id, K, N, **kw):
        return Case(id, 1, 1, M_OLD, K, N, per_cta3=True, **kw)

    def e(bn, epi, io=None):
        return dict(block_n=bn, epi=EPI[epi], **({"epi_io": io} if io else {}))

    return [
        # overlapped epilogue
        lin("ov_plain_bn64", 128, 64, expect=e(64, "plain")),
        Case("ov_plain_rowadd_concat_3x3_bn160", 13, 64, 64, 64, 160, C1=64, taps="3x3", rpg=64 * 64, per_cta3=True,
             expect=e(160, "plain")),
        lin("ov_residual_bn128", 320, 128, res="dense", alpha=0.5, expect=e(128, "residual")),
        Case("ov_residual_temporal_bn160", 2, 8, 4096, 64, 160, taps="t3", bias=False, res="dense", per_cta3=True,
             expect=e(160, "residual")),
        lin("ov_generic_residual_beta_bn160", 64, 320, res="dense", beta=2.0, expect=e(160, "generic")),
        lin("ov_generic_ragged_n_bn128", 192, 72, res="dense", expect=e(128, "generic")),
        Case("ov_generic_stride2_bn128", 13, 128, 128, 64, 128, s2=1, alpha=0.5, per_cta3=True, expect=e(128, "generic")),
        lin("ov_geglu_bn128", 320, 128, geglu=True, expect=e(128, "geglu")),
        lin("ov_generic_geglu_ragged_n_bn128", 128, 96, geglu=True, expect=e(128, "generic")),
        lin("ov_gelu_bn160", 128, 160, act=2, expect=e(160, "act")),
        lin("ov_quick_gelu_bn64", 256, 64, act=3, expect=e(64, "act")),
        lin("ov_f32_silu_bn128", 320, 128, act=1, f32=True, expect=e(128, "generic")),
        lin("ov_residual_bn256_inline", 128, 1280, res="dense", expect=e(256, "residual")),
        # TMA epilogue
        lin("tma_residual_k320", 320, 320, res="dense", alpha=0.5, expect=e(160, "residual", "tma")),
        lin("tma_residual_k640", 640, 320, res="dense", expect=e(160, "residual", "tma")),
        lin("tma_residual_k1280", 1280, 320, res="dense", expect=e(160, "residual", "tma")),
        lin("tma_residual_bn128", 320, 128, res="dense", expect=e(128, "residual", "tma")),
        lin("tma_residual_bn64", 320, 64, res="dense", expect=e(64, "residual", "tma")),
        lin("tma_residual_inplace_k640", 640, 640, res="inplace", expect=e(160, "residual", "tma")),
        Case("tma_plain_3x3_narrow_box", 11, 30, 46, 128, 640, taps="3x3", per_cta3=True, expect=e(160, "plain", "tma")),
        Case("tma_residual_temporal", 2, 9, 2900, 320, 320, taps="t3", bias=False, res="dense", alpha=0.75,
             per_cta3=True, expect=e(160, "residual", "tma")),
        lin("tma_geglu", 640, 256, geglu=True, expect=e(128, "geglu", "tma")),
        Case("tma_plain_rowadd_concat", 13, 36, 20, 64, 320, C1=128, taps="3x3", rpg=36 * 20, per_cta3=True,
             expect=e(64, "plain", "tma")),
        lin("tma_plain_out_window", 320, 320, bias=False, out_pad=(192, 64), expect=e(160, "plain", "tma")),
        lin("tma_generic_residual_beta", 320, 320, bias=False, res="dense", beta=0.5, expect=e(160, "generic", "lsu")),
        # 256-wide tiles
        lin("wide_geglu_k320", 320, 2560, geglu=True, expect=e(256, "geglu", "tma")),
        lin("wide_residual_inplace_k640", 640, 1280, res="inplace", expect=e(256, "residual", "tma")),
        Case("wide_residual_3x3_narrow_box", 11, 30, 46, 128, 1280, taps="3x3", res="dense", alpha=0.5, per_cta3=True,
             expect=e(256, "residual", "tma")),
        Case("wide_plain_3x3_rowadd", 11, 30, 46, 64, 1280, taps="3x3", rpg=30 * 46, per_cta3=True,
             expect=e(256, "plain", "tma")),
        lin("wide_plain_n1216_window", 320, 1216, out_pad=(160, 128), expect=e(256, "plain", "tma")),
        lin("wide_residual_k5120", 5120, 1280, res="dense", expect=e(256, "residual", "tma")),
    ]


def all_cases(sms=HOST_SMS):
    return matrix_cases(sms) + special_cases(sms) + old_cases(sms)


CASES = all_cases()
CASE_IDS = [c.id for c in CASES]
assert len(set(CASE_IDS)) == len(CASE_IDS)


# ------------------------------------------------------------------------------------------------ inputs
def make_inputs(case, device):
    """The ops.conv_gemm keyword arguments of a case on seeded data, and the wide output buffer (or None) whose columns
    around the output window must stay untouched."""
    g = torch.Generator(device=device).manual_seed(zlib.crc32(case.id.encode()))

    def rnd(*shape, scale=1.0, dtype=torch.float16):
        return (torch.randn(*shape, generator=g, device=device) * scale).to(dtype)

    NF, H, W = case.NF, case.H, case.W
    if case.a0_view == "chwin":
        a0 = rnd(NF, H, W, case.C0 + 128)[..., 64:64 + case.C0]
    elif case.a0_view == "fstride":
        a0 = rnd(2 * NF, H, W, case.C0)[::2]
    else:
        a0 = rnd(NF, H, W, case.C0)
    K = case.ntaps * (case.C0 + case.C1)
    kw = dict(a0=a0, weight=rnd(case.N, K, scale=K ** -0.5))
    if case.s2:
        kw["stride2"] = case.s2
    else:
        kw["taps"] = TAPS[case.taps]
    if case.C1:
        kw["a1"] = rnd(NF, H, W, case.C1)
    if case.bias:
        kw["bias"] = rnd(case.N, scale=0.5, dtype=torch.float32)
    M, nout = case.M, case.nout
    if case.rpg:
        kw["rowadd"] = rnd(ceil_div(M, case.rpg), case.N + case.ld_rowadd_pad, scale=0.5, dtype=torch.float32)[:, :case.N]
        kw["rows_per_group"] = case.rpg
    lo, hi = case.out_pad
    wide = None
    if case.res == "dense":
        kw["residual"] = rnd(M, nout)
    elif case.res == "window":
        kw["residual"] = rnd(M, nout + 96)[:, 64:64 + nout]
    elif case.res == "inplace":
        wide = rnd(M, lo + nout + hi)
        kw["residual"] = kw["out"] = wide[:, lo:lo + nout]
    if wide is None and (lo or hi):
        wide = torch.full((M, lo + nout + hi), 7.0, dtype=torch.float32 if case.f32 else torch.float16, device=device)
        kw["out"] = wide[:, lo:lo + nout]
    kw.update(alpha=case.alpha, beta=case.beta, geglu=case.geglu, act=case.act, out_f32=case.f32)
    return kw, wide


# ------------------------------------------------------------------------------------------------ float64 reference
def _ulp16(r):
    """Spacing of fp16 at |r| (float64 tensor): 2^(e - 11) for |r| in [2^(e-1), 2^e), 2^-24 in the subnormal range."""
    _, e = torch.frexp(r.abs())
    return torch.where(r.abs() < 2.0 ** -14, torch.full_like(r, 2.0 ** -24), torch.ldexp(torch.ones_like(r), e - 11))


def _gelu(x, tanh=False):
    if tanh:
        return 0.5 * x * (1 + torch.tanh(math.sqrt(2 / math.pi) * (x + 0.044715 * x ** 3)))
    return 0.5 * x * (1 + torch.erf(x / math.sqrt(2)))


def _act(x, act, wrong):
    if act == 1:
        return x * torch.sigmoid(x)
    if act == 2:
        return _gelu(x, "gelu tanh form" in wrong)
    if act == 3:
        return _gelu(x) if "quick-gelu as exact gelu" in wrong else x * torch.sigmoid(1.702 * x)
    return x


def conv_ref(a0, weight, taps=TAPS["1"], a1=None, bias=None, rowadd=None, rows_per_group=1, residual=None, alpha=1.0,
             beta=1.0, geglu=False, act=0, out_f32=False, stride2=0, out=None, wrong=()):
    """float64 reference of one ops.conv_gemm call and the per-element bound: (ref [M, nout], bound [M, nout]).
    `wrong` names the deliberate errors of the host checks. Computed on the tensors' device; call it before the
    launch when the output is the residual."""
    x = (a0 if a1 is None else torch.cat([a0, a1], 3)).double()
    NF, H, W, Ct = x.shape
    s = 2 if stride2 else 1
    if stride2:
        mode = stride2 if "stride-2 pad mode 1 for 2" not in wrong else 1
        offs = (-1, 0, 1) if mode == 1 else (0, 1, 2)
        taps = tuple((dy, dx) for dy in offs for dx in offs)
    Ho, Wo = (H // 2, W // 2) if stride2 else (H, W)
    if "temporal tap reads the neighbouring video" in wrong:
        x = x.reshape(1, NF * H, W, Ct)             # frames of consecutive videos become neighbours
    n_, H_ = x.shape[0], x.shape[1]
    Ho_ = Ho * NF // n_
    lo = max(0, -min(min(t) for t in taps))
    hi_h = max(0, max(t[0] for t in taps) + s * (Ho_ - 1) - (H_ - 1))
    hi_w = max(0, max(t[1] for t in taps) + s * (Wo - 1) - (W - 1))
    xp = F.pad(x, (0, 0, lo, hi_w, lo, hi_h))
    M, N = NF * Ho * Wo, weight.shape[0]
    wd = weight.double()
    if "k block left out" in wrong:
        wd = wd.clone()
        wd[:, (wd.shape[1] // 64 // 2) * 64:][:, :64] = 0      # the middle 64-channel block of K
    if "last k16 left out" in wrong:
        wd = wd.clone()
        wd[:, -16:] = 0
    acc = torch.zeros(M, N, dtype=torch.float64, device=x.device)
    sab = torch.zeros_like(acc)
    for t, (dy, dx) in enumerate(taps):
        v = xp[:, lo + dy:lo + dy + s * (Ho_ - 1) + 1:s, lo + dx:lo + dx + s * (Wo - 1) + 1:s].reshape(M, Ct)
        wt = wd[:, t * Ct:(t + 1) * Ct]
        acc += v @ wt.t()
        sab += v.abs() @ wt.abs().t()
        del v
    if "accumulator rounded to fp16" in wrong:
        acc = acc.half().double()
    b = bias.double() if bias is not None else torch.zeros(N, dtype=torch.float64, device=x.device)
    if geglu:
        pre = (acc + b).view(M, N // 32, 2, 16)
        val, gate = (pre[:, :, 1], pre[:, :, 0]) if "geglu value and gate swapped" in wrong else (pre[:, :, 0], pre[:, :, 1])
        gl = _gelu(gate, "gelu tanh form" in wrong)
        ref = (val * gl).reshape(M, N // 2)
        a4 = (acc.abs() + b.abs()).view(M, N // 32, 2, 16)
        s4 = sab.view(M, N // 32, 2, 16)
        s_acc = (gl.abs() * s4[:, :, 0] + val.abs() * ACT_SLOPE * s4[:, :, 1]).reshape(M, N // 2)
        s_epi = (gl.abs() * a4[:, :, 0] + val.abs() * ACT_SLOPE * a4[:, :, 1]).reshape(M, N // 2) + ref.abs()
        extra = 1e-6 * (val.abs() * (1 + gate.abs())).reshape(M, N // 2)
    else:
        r = torch.zeros_like(acc)
        if rowadd is not None:
            rows = torch.arange(M, device=x.device)
            if "row-add group of the tile's first row" in wrong:
                bw, bh, bnf = pick_box(Wo, Ho, NF)
                w_, h_, n_i = rows % Wo, (rows // Wo) % Ho, rows // (Wo * Ho)
                rows = ((n_i // bnf * bnf) * Ho + h_ // bh * bh) * Wo + w_ // bw * bw
            r = rowadd.double()[rows // rows_per_group]
        pre = acc + b + r
        res = residual.double() if residual is not None else torch.zeros_like(acc)
        v = (pre + beta * res) * alpha if "residual added before alpha" in wrong else pre * alpha + beta * res
        ref = _act(v, act, wrong)
        slope = ACT_SLOPE if act else 1.0
        s_acc = abs(alpha) * slope * sab
        s_epi = slope * (abs(alpha) * (acc.abs() + b.abs() + r.abs()) + (beta * res).abs() + v.abs())
        extra = 1e-6 * v.abs() if act else 0.0
    bound = C_ACC * s_acc + EPS_EPI * s_epi + extra
    if not out_f32:
        bound = bound + 0.5 * _ulp16(ref)
    return ref, bound


def _ratio(got, ref, bound, f32=False):
    """max |got - ref| / bound (got rounded to fp16, or fp32, as a kernel would return it), its flat index; inf if got
    is not finite."""
    got = got.float().double() if f32 else got.half().double()
    if not torch.isfinite(got).all():
        return math.inf, -1
    r = ((got - ref).abs() / bound).flatten()
    i = int(r.argmax())
    return r[i].item(), i


def _record(name, err, bound, where=""):
    path = os.environ.get("MVB_PARITY_LOG")
    if path:
        try:
            with open(path, "a") as fh:
                fh.write(json.dumps({"test": name, "value": err, "bound": bound}) + "\n")
        except OSError:
            pass
    assert err <= bound, (name, where, err, bound)


# ------------------------------------------------------------------------------------------------ host checks
def test_plan_mirror_matches_the_kernel_table():
    """The ring depths the mirror computes are the static_assert's, and 17 (BN, epilogue) pairs are reachable."""
    for (epi, bn), n in NSTAGES.items():
        assert ring_stages(epi, bn) == n, (epi, bn)
    assert len(REACHABLE) == 17


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_case_plans(case):
    """Each case reaches the plan it states at 132 SMs; the per-feature rows keep >= 3 tiles per CTA."""
    p = case.plan()
    got = {k: p[k] for k in case.expect}
    assert got == case.expect, (case.id, got, case.expect)
    if case.per_cta3:
        assert p["tiles"] >= 3 * HOST_SMS and p["tiles_per_cta"] >= 3, p


def test_matrix_covers_every_pair_and_the_ring_wraps():
    """Every reachable pair runs at 1, nstages - 1, nstages, nstages + 1 and 36 K blocks per tile, every such case
    with >= 3 tiles per CTA and >= 2 ring wraps on the least loaded CTA, ragged rows, and each pair with a wrap inside
    a tile, bias on and off."""
    by_pair = {}
    for c in matrix_cases(HOST_SMS):
        p = c.plan()
        assert p["tiles_per_cta"] >= 3 and p["wraps"] >= 2 and p["ragged_rows"], (c.id, p)
        by_pair.setdefault((p["epi"], p["block_n"]), []).append((c, p))
    assert sorted(by_pair) == sorted(REACHABLE)
    for pair, cps in by_pair.items():
        ns = NSTAGES[pair]
        assert {1, ns - 1, ns, ns + 1, 36} <= {p["kb"] for _, p in cps}, pair
        assert any(p["mid_tile_wrap"] for _, p in cps), pair
        assert {c.bias for c, _ in cps} == {True, False}, pair
        if pair != (EPI["geglu"], 64) and pair != (EPI["geglu"], 128):
            assert any(p["ragged_cols"] for _, p in cps), pair


# host shapes of each group and the wrong answers that apply to it
HOST_GROUPS = {
    "plain": (Case("h_plain", 1, 1, 300, 128, 64), ("k block left out", "last k16 left out", "accumulator rounded to fp16")),
    "residual_alpha": (Case("h_res", 1, 1, 300, 192, 64, res="dense", alpha=0.5),
                       ("k block left out", "last k16 left out", "accumulator rounded to fp16", "residual added before alpha")),
    "generic_beta": (Case("h_beta", 1, 1, 300, 128, 40, res="dense", beta=0.5),
                     ("k block left out", "accumulator rounded to fp16")),
    "rowadd": (Case("h_rowadd", 1, 1, 300, 128, 64, rpg=100), ("k block left out", "row-add group of the tile's first row")),
    "rowadd_3x3": (Case("h_rowadd_3x3", 2, 6, 10, 64, 32, taps="3x3", rpg=50),
                   ("k block left out", "row-add group of the tile's first row")),
    "gelu": (Case("h_gelu", 1, 1, 300, 128, 64, act=2), ("k block left out", "last k16 left out", "gelu tanh form")),
    "quick_gelu": (Case("h_qgelu", 1, 1, 300, 128, 64, act=3), ("k block left out", "quick-gelu as exact gelu")),
    "silu_f32": (Case("h_silu_f32", 1, 1, 300, 128, 64, act=1, f32=True),
                 ("k block left out", "last k16 left out", "accumulator rounded to fp16")),
    "temporal": (Case("h_t3", 3, 2, 40, 64, 64, taps="t3"), ("k block left out", "temporal tap reads the neighbouring video")),
    "stride2": (Case("h_s2", 2, 4, 6, 64, 64, s2=2), ("k block left out", "stride-2 pad mode 1 for 2")),
    "geglu": (Case("h_geglu", 1, 1, 300, 128, 128, geglu=True),
              ("k block left out", "last k16 left out", "geglu value and gate swapped", "gelu tanh form")),
    "longest_k": (Case("h_k23040", 2, 2, 2, 1280, 16, C1=1280, taps="3x3"), ("k block left out",)),
}


@pytest.mark.parametrize("group", list(HOST_GROUPS))
def test_conv_gemm_bounds_catch_wrong_answers(group):
    """Host only: on each group's small shape the reference passes its own bound and every named wrong answer,
    rounded as the kernel would return it, breaks it."""
    case, wrongs = HOST_GROUPS[group]
    kw, _ = make_inputs(case, "cpu")
    kw.pop("out", None)
    ref, bound = conv_ref(**kw)
    assert _ratio(ref, ref, bound, case.f32)[0] <= 1.0
    for w in wrongs:
        y, _ = conv_ref(**kw, wrong=(w,))
        r = _ratio(y, ref, bound, case.f32)[0]
        assert r > 1.0, f"{group}: the wrong answer '{w}' stays inside the bound (worst ratio {r:.3g})"


# ------------------------------------------------------------------------------------------------ GPU: child process
def _traced(fn):
    """Run fn with fd 2 captured; returns (fn's result, the parsed MVB_TRACE gemm lines)."""
    from tools.gpu_gemm_census import _parse
    sys.stderr.flush()
    saved = os.dup(2)
    with tempfile.TemporaryFile(mode="w+") as log:
        os.dup2(log.fileno(), 2)
        try:
            out = fn()
            torch.cuda.synchronize()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        log.seek(0)
        lines = log.read().splitlines()
    return out, [kv for kv in map(_parse, lines) if kv is not None]


def _trace_fields(t):
    return {"block_n": int(t["block_n"]), "epi": int(t["epi"]), "epi_io": t["epi_io"], "nstages": int(t["nstages"]),
            "tiles": int(t["tiles"]), "kb": int(t["K"]) // 64}


def _run_case(ops, kw, wide, out_cols, f32):
    ref, bound = conv_ref(**kw)
    out, trace = _traced(lambda: ops.conv_gemm(**kw))
    r, i = _ratio(out, ref, bound, f32)
    untouched = True
    if wide is not None:
        lo, nout = out_cols
        untouched = bool((wide[:, :lo] == 7).all() and (wide[:, lo + nout:] == 7).all())
    res = {"launches": len(trace), "trace": _trace_fields(trace[0]) if trace else None, "ratio": r,
           "where": [i // max(ref.shape[1], 1), i % max(ref.shape[1], 1)] if i >= 0 else None,
           "shape_ok": list(out.shape) == list(ref.shape), "untouched": untouched}
    del ref, bound, out
    return res


def _inplace_untouched(case, wide, before):
    lo, hi = case.out_pad
    return bool(torch.equal(wide[:, :lo], before[:, :lo]) and torch.equal(wide[:, lo + case.nout:], before[:, lo + case.nout:]))


def _run_all():
    sys.path.insert(0, ROOT)
    from musev_b200 import ops
    from tools import gpu_gemm_census as census
    dev = torch.device("cuda", 0)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    results = {"sms": sms, "cases": {}, "engine": {}}
    for case in all_cases(sms):
        kw, wide = make_inputs(case, dev)
        before = wide.clone() if case.res == "inplace" else None
        rr = _run_case(ops, kw, wide if case.res != "inplace" else None, (case.out_pad[0], case.nout), case.f32)
        if before is not None:
            rr["untouched"] = _inplace_untouched(case, wide, before)
        rr["plan"] = {k: v for k, v in case.plan(sms).items() if k in ("block_n", "epi", "epi_io", "nstages", "tiles", "kb")}
        results["cases"][case.id] = rr
        del kw, wide, before
    torch.cuda.empty_cache()
    for preset in ("musev", "musev_referencenet"):
        entries, _ = census.capture_forward(preset, batch=2, frames=4, h=16, w=16, warmup=0, profile=False)
        g = torch.Generator().manual_seed(zlib.crc32(preset.encode()))
        rows = []
        for e in entries:
            kw, _, _, _ = census.make_case(e, dev, g)
            kw["out"] = census.make_out(e, kw, dev)
            rr = _run_case(ops, kw, None, None, bool(int(e["f32"])))
            ntaps = len(e["offsets"].split(",")) if not int(e["s2"]) else 9
            p = plan(int(e["W"]), int(e["H"]), int(e["NF"]), ntaps, (int(e["c0"]) + int(e["c1"])) // 64, int(e["N"]),
                     bool(int(e["geglu"])), bool(int(e["res"])), float(e["alpha"]), float(e["beta"]), int(e["act"]),
                     bool(int(e["f32"])), sms)
            rr["plan"] = {k: p[k] for k in ("block_n", "epi", "epi_io", "nstages", "tiles", "kb")}
            rr["key"] = {k: e[k] for k in census.KEY_FIELDS}
            rows.append(rr)
        results["engine"][preset] = rows
    print(json.dumps(results))


@pytest.fixture(scope="module")
def results(built_lib):
    r = subprocess.run([sys.executable, os.path.abspath(__file__)], env=dict(os.environ, MVB_TRACE="1"),
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-4000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def _check_row(name, rr):
    assert rr["launches"] == 1, (name, rr)
    assert rr["trace"] == rr["plan"], (name, rr["trace"], rr["plan"])
    assert rr["shape_ok"] and rr["untouched"], (name, rr)
    _record(f"conv_gemm_{name}_vs_fp64", rr["ratio"], 1.0, rr["where"])


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_conv_gemm_edges(results, case):
    rr = results["cases"][case.id]
    assert rr["launches"] == 1, rr
    if results["sms"] == HOST_SMS:
        assert {k: rr["trace"][k] for k in case.expect if k in rr["trace"]} == \
            {k: v for k, v in case.expect.items() if k in rr["trace"]}, (case.id, rr["trace"])
    if case.per_cta3:
        assert rr["trace"]["tiles"] >= 3 * results["sms"], rr
    _check_row(case.id, rr)


@pytest.mark.gpu
def test_conv_gemm_covers_every_instantiation(results):
    """The union of the traced (BN, epilogue, I/O path) is every reachable instantiation."""
    seen = {(r["trace"]["block_n"], r["trace"]["epi"], r["trace"]["epi_io"]) for r in results["cases"].values()}
    want = {(bn, epi, "tma" if epi in (1, 2, 3) else "lsu") for epi, bn in REACHABLE}
    assert seen == want, (sorted(want - seen), sorted(seen - want))
    assert len(seen) == 17


@pytest.mark.gpu
@pytest.mark.parametrize("preset", ["musev", "musev_referencenet"])
def test_conv_gemm_engine_launches(results, preset):
    """Every distinct conv_gemm launch of one full-width UNet forward (2 x (4 + 1) frames, 16 x 16 latents), replayed
    with the engine's output and residual strides on seeded data."""
    rows = results["engine"][preset]
    assert len(rows) >= 20, len(rows)
    assert any(int(r["key"]["res_is_out"]) for r in rows)
    for i, rr in enumerate(rows):
        _check_row(f"engine_{preset}_{i}_" + "_".join(f"{k}{rr['key'][k]}" for k in ("N", "K", "W", "H", "NF")), rr)


@pytest.mark.gpu
def test_conv_gemm_refuses_before_launch(built_lib):
    """Option combinations the kernel would drop or misread are refused before anything is launched: GEGLU with a
    row-add, residual, alpha != 1 or an activation; an act code outside 0..3; stride 2 with a second source or a strided
    first one; channels not a multiple of 64, N not a multiple of 8, odd H or W at stride 2; a misaligned output, output
    row stride or residual; fp32 output with a residual or GEGLU."""
    from musev_b200 import _capi, ops
    from musev_b200._capi import MvbError
    dev = "cuda"
    z = lambda *s, dt=torch.float16: torch.zeros(*s, dtype=dt, device=dev)   # noqa: E731
    M = 256
    a, w, w128 = z(1, 1, M, 64), z(64, 64), z(128, 64)
    b128 = z(128, dt=torch.float32)
    x = z(2, 8, 8, 64)
    ws2 = z(64, 9 * 64)
    geglu_only = "geglu takes a bias only"
    s2_contig = "stride2 takes one contiguous"
    calls = {
        "geglu + row-add": (lambda: ops.conv_gemm(a, w128, bias=b128, geglu=True, rowadd=z(M, 128, dt=torch.float32)), geglu_only),
        "geglu + residual": (lambda: ops.conv_gemm(a, w128, bias=b128, geglu=True, residual=z(M, 64)), geglu_only),
        "geglu + alpha": (lambda: ops.conv_gemm(a, w128, bias=b128, geglu=True, alpha=0.5), geglu_only),
        "geglu + silu": (lambda: ops.conv_gemm(a, w128, geglu=True, act=1), geglu_only),
        "geglu + gelu": (lambda: ops.conv_gemm(a, w128, geglu=True, act=2), geglu_only),
        "act 4": (lambda: ops.conv_gemm(a, w, act=4), "act must be"),
        "act -1": (lambda: ops.conv_gemm(a, w, act=-1), "act must be"),
        "stride2 + a1": (lambda: ops.conv_gemm(x, ws2, a1=z(2, 8, 8, 64), stride2=1), s2_contig),
        "stride2 channel window": (lambda: ops.conv_gemm(z(2, 8, 8, 128)[..., 64:], ws2, stride2=1), s2_contig),
        "stride2 frame-strided": (lambda: ops.conv_gemm(z(4, 8, 8, 64)[::2], ws2, stride2=2), s2_contig),
        "C % 64": (lambda: ops.conv_gemm(z(1, 1, M, 96), z(64, 96)), "channels must be multiples of 64"),
        "N % 8": (lambda: ops.conv_gemm(a, z(60, 64)), "N a multiple of 8"),
        "odd H stride2": (lambda: ops.conv_gemm(z(2, 7, 8, 64), ws2, stride2=1), "even H and W"),
        "odd W stride2": (lambda: ops.conv_gemm(z(2, 8, 7, 64), ws2, stride2=2), "even H and W"),
        "misaligned out": (lambda: ops.conv_gemm(a, w, out=z(M, 72)[:, 1:65]), "output must be 16-byte aligned"),
        "out row stride": (lambda: ops.conv_gemm(a, w, out=z(M, 68)[:, :64]), "output must be 16-byte aligned"),
        "misaligned residual": (lambda: ops.conv_gemm(a, w, residual=z(M, 65)[:, 1:]), "residual must be 16-byte aligned"),
        "residual row stride": (lambda: ops.conv_gemm(a, w, residual=z(M, 68)[:, :64]), "residual must be 16-byte aligned"),
        "f32 + residual": (lambda: ops.conv_gemm(a, w, residual=z(M, 64), out_f32=True), "fp32 output excludes"),
        "f32 + geglu": (lambda: ops.conv_gemm(a, w128, geglu=True, out_f32=True), "fp32 output excludes"),
    }
    torch.cuda.synchronize()
    n0 = _capi.launch_count()
    for what, (call, msg) in calls.items():
        with pytest.raises(MvbError, match=msg):
            call()
            pytest.fail(f"{what}: not refused")
    torch.cuda.synchronize()
    assert _capi.launch_count() == n0


if __name__ == "__main__":
    _run_all()
