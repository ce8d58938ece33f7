"""GroupNorm, LayerNorm and the row softmax at every launch path and at the data where normalisations go wrong, against
one float64 reference each.

Each reference upcasts the fp16 inputs the kernel saw to float64. Every element is held to its own bound,
    |y - ref| <= ulp16(ref) / 2 + 1e-5 |ref| + C_NORM * slope * |gamma| * (1 + |xhat|)    (GroupNorm, LayerNorm)
    |y - ref| <= 1.5 ulp16(ref) + 1e-4 ref                                                (softmax)
where xhat is the float64 normalised input, slope = 1.1 (the largest slope of SiLU) with SiLU and 1 without, ulp16 the
spacing of fp16 at |ref| (2^-24 below the normal range) and C_NORM = 1e-4. For the normalisations that is the rounding to
fp16 plus fp32-level slack: statistics off by 1e-4 of a standard deviation break it. The softmax rounds twice (the
unnormalised exponentials, then the probabilities). Never a bound relative to the tensor's maximum.

Each case first asserts which launch path its shape takes, from a mirror of the host arithmetic of ops.cu (`gn_plan`,
`ln_plan`), so that a case that drifts onto another path fails instead of silently testing something else. Each case
also shows that its bound discriminates: on the same data the test computes named wrong answers in float64 (variance
with N - 1, eps x 10, per-frame statistics where frames share statistics, the group edge one channel off, the last pixel
chunk left out; for the softmax the last 8 columns left unnormalised and the scale ignored), rounds them to fp16 as a
kernel would, and asserts that each applicable one breaks the bound. Those checks need no GPU and run on the host as
well (`test_*_bounds_catch_wrong_answers`). N - 1 moves xhat by 1 / (2N), which fp16 resolves only for N <= 512; eps
x 10 needs a group or row whose variance is near eps, so the random data carries one group (row) with variance ~eps.

With MVB_PARITY_LOG=<file> set, the worst ratio |y - ref| / bound of every test is appended to <file>. Measured on an
H100 80GB HBM3 at 700 W, worst ratio per group: GroupNorm 0.977 (fps8_wide), LayerNorm 0.979 (C 1024), the layernorm40
grid-stride cases 0.978, softmax 0.855 (N 8192, sigma 1). Near 1 for the normalisations because a correctly rounded
result may sit half an ulp away and the slack above that is small.
"""
import json
import math
import os
import zlib
from dataclasses import dataclass, field

import pytest
import torch

dev = "cuda"
C_NORM = 1e-4
SILU_SLOPE = 1.1


def _record(name, err, bound, where=""):
    path = os.environ.get("MVB_PARITY_LOG")
    if path:
        try:
            with open(path, "a") as fh:
                fh.write(json.dumps({"test": name, "value": err, "bound": bound}) + "\n")
        except OSError:
            pass
    assert err <= bound, (name, where, err, bound)


def _ulp16(r):
    """Spacing of fp16 at |r| (float64 tensor): 2^(e - 11) for |r| in [2^(e-1), 2^e), 2^-24 in the subnormal range."""
    _, e = torch.frexp(r.abs())
    return torch.where(r.abs() < 2.0 ** -14, torch.full_like(r, 2.0 ** -24), torch.ldexp(torch.ones_like(r), e - 11))


def _norm_bound(ref, gamma, xhat, silu):
    slope = SILU_SLOPE if silu else 1.0
    return 0.5 * _ulp16(ref) + 1e-5 * ref.abs() + C_NORM * slope * gamma.double().abs() * (1 + xhat.abs())


def _ratio(got, ref, bound):
    """max |got - ref| / bound (got rounded to fp16 as a kernel would return it); inf if got is not finite."""
    got = got.half().double() if got.dtype != torch.float16 else got.double()
    if not torch.isfinite(got).all():
        return math.inf
    return ((got - ref).abs() / bound).max().item()


def _assert_catches(wrong, ref, bound, what):
    for name, y in wrong.items():
        r = _ratio(y, ref, bound)
        assert r > 1.0, f"{what}: the wrong answer '{name}' stays inside the bound (worst ratio {r:.3g})"


@pytest.fixture(scope="module")
def ops(built_lib):
    from musev_b200 import ops as o
    return o


# ------------------------------------------------------------------------------------------------ launch-path mirrors
def gn_plan(C, NF, HW, fps, G=32):
    """The work decomposition of a GroupNorm op call, mirroring ops.cu: gn_chunks (the chunk count, ops.cu:147-154),
    gn_stats and gn_stats_unit (channel-vector passes and rows of the statistics block, :156-169 and :54-64), gn_apply
    (finalize choice and apply block size, :391-397), the fixed_col rule of gn_apply_unit (:252) and gn_fused (the same
    block size rule, :421-425). The op entries take chunk_nf = NF."""
    vecs, cpg = C // 8, C // G
    terms = {"nf": (8 * 132) // NF, "hw": max(HW // 32, 1), "cap": 64}
    chunks = max(min(terms.values()), 1)
    limit = min(terms, key=lambda k: (terms[k], list(terms).index(k)))
    threads = 256
    if vecs <= 256 and 256 % vecs:
        threads = (256 // vecs) * vecs
    if threads < 64:
        threads = 256
    return {"chunks": chunks, "limit": limit, "ragged": HW % chunks != 0,
            "stats_passes": -(-vecs // 256),
            "apply": "fixed_col" if threads % vecs == 0 and cpg >= 8 else "per_element",
            "finalize": "wide" if fps * chunks > 64 else "narrow",
            "idle_rows": HW // chunks < 256 // min(vecs, 256)}     # statistics threads (gn_stats) that own no sample


def ln_plan(C, M):
    """The LayerNorm instantiation and grid of an op call, mirroring ops.cu layernorm() (ops.cu:589-609)."""
    if C in (320, 640, 1280):
        L = C // 40
        groups = -(-M // (32 // L))
        blocks = min(-(-groups // 8), 132 * 8)
        return {"kernel": f"layernorm40<{L}>", "grid_stride": groups > blocks * 8}
    vecs = C // 8
    for lim, name in ((32, "<1,4>"), (64, "<2,4>"), (160, "<5,2>"), (320, "<10,1>")):
        if vecs <= lim:
            return {"kernel": "layernorm_kernel" + name, "grid_stride": False}
    raise AssertionError(C)


# ------------------------------------------------------------------------------------------------ GroupNorm
@dataclass(frozen=True)
class GN:
    id: str
    C0: int
    C1: int
    NF: int
    HW: int
    fps: int = 1
    eps: float = 1e-5
    silu: bool = True
    data: str = "randn"
    expect: dict = field(default_factory=dict, hash=False, compare=False)

    @property
    def C(self):
        return self.C0 + self.C1


def _gn_cases():
    cs = []
    # channels per group at G = 32, NF 3, HW 200 (6 chunks limited by HW / 32, 200 not a multiple of 6)
    for cpg in (2, 4, 8, 10, 16, 20, 30, 40, 60, 80):
        apply = "fixed_col" if 8 <= cpg <= 60 else "per_element"
        cs.append(GN(f"cpg{cpg}", 32 * cpg, 0, 3, 200, expect=dict(apply=apply, chunks=6, limit="hw", ragged=True,
                                                                  stats_passes=2 if cpg == 80 else 1)))
    # concatenated inputs whose boundary falls inside a group
    for c0, c1 in ((320, 640), (1280, 640), (640, 320)):
        cs.append(GN(f"cat{c0}+{c1}", c0, c1, 2, 256, silu=False, expect=dict(apply="fixed_col", chunks=8, ragged=False)))
    # finalize kernel: one warp (fps * chunks <= 64) or eight
    cs += [GN("fps1_narrow", 320, 0, 4, 256, 1, expect=dict(finalize="narrow", chunks=8)),
           GN("fps8_narrow64", 320, 0, 8, 256, 8, expect=dict(finalize="narrow", chunks=8)),
           GN("fps8_wide", 320, 0, 8, 512, 8, expect=dict(finalize="wide", chunks=16)),
           GN("fps16_narrow", 640, 0, 16, 64, 16, expect=dict(finalize="narrow", chunks=2, limit="hw")),
           GN("fps16_wide", 640, 0, 16, 256, 16, silu=False, expect=dict(finalize="wide", chunks=8)),
           GN("fps17_narrow", 1280, 0, 17, 64, 17, expect=dict(finalize="narrow", chunks=2)),
           GN("fps17_wide_nf34", 320, 0, 34, 4096, 17, expect=dict(finalize="wide", chunks=31, limit="nf", ragged=True))]
    # chunk count limited by the frame count, by HW / 32, by the cap of 64 (the VAE's shapes, eps 1e-6)
    cs += [GN("nf34_ragged", 640, 0, 34, 1024, expect=dict(chunks=31, limit="nf", ragged=True)),
           GN("hw16", 320, 0, 2, 16, silu=False, expect=dict(chunks=1, limit="hw")),
           GN("vae_c128_cap", 128, 0, 1, 64 * 96 * 64, eps=1e-6, expect=dict(chunks=64, limit="cap", apply="per_element")),
           GN("vae_c256_cap", 256, 0, 1, 96 * 1024, eps=1e-6, expect=dict(chunks=64, limit="cap", apply="fixed_col")),
           GN("vae_c512_cap", 512, 0, 1, 24 * 1024, eps=1e-6, silu=False, expect=dict(chunks=64, limit="cap")),
           GN("cap_ragged", 128, 0, 1, 100000, eps=1e-6, expect=dict(chunks=64, limit="cap", ragged=True))]
    # tiny HW: most statistics threads own no sample
    cs += [GN("hw1_c64", 64, 0, 2, 1, silu=False, expect=dict(chunks=1, idle_rows=True, apply="per_element")),
           GN("hw1_c320", 320, 0, 2, 1, expect=dict(chunks=1, idle_rows=True)),
           GN("hw4_c128", 128, 0, 3, 4, expect=dict(chunks=1, idle_rows=True)),
           GN("hw4_c2560", 2560, 0, 2, 4, silu=False, expect=dict(chunks=1, stats_passes=2, apply="per_element"))]
    # data: channels of one group 2048 apart, a group spanning +-33000, all zeros
    for c, tag in ((320, "c320"), (128, "c128"), (2560, "c2560")):
        cs.append(GN(f"mean2048_{tag}", c, 0, 2, 1024, data="mean2048"))
        cs.append(GN(f"wide_{tag}", c, 0, 2, 1024, silu=False, data="wide"))
    cs += [GN("wide_fps2_wide_finalize", 640, 0, 4, 4096, 2, data="wide", expect=dict(finalize="wide")),
           GN("zero_c320", 320, 0, 2, 1024, silu=False, data="zero"),
           GN("zero_c128_hw1", 128, 0, 2, 1, silu=False, data="zero")]
    return cs


GN_CASES = _gn_cases()


def gn_inputs(case, device):
    """x [NF, HW, C] fp16, gamma, beta fp32. 'randn': N(0, 1) plus a ramp over the pixels (so that a missing chunk shows)
    and an offset per frame (so that per-frame statistics show), with group 1 scaled to variance ~eps (so that eps
    shows). 'mean2048': the randn data with the odd channels of group 2 shifted by 2048 (each channel pair straddles
    its pilot). 'wide': the randn data with group 3's even channels around -33000 and odd ones around +33000."""
    g = torch.Generator().manual_seed(zlib.crc32(case.id.encode()))
    NF, HW, C, G = case.NF, case.HW, case.C, 32
    cpg = C // G
    gamma = torch.randn(C, generator=g)
    beta = torch.randn(C, generator=g) * 0.5
    if case.data == "zero":
        x = torch.zeros(NF, HW, C)
    else:
        x = torch.randn(NF, HW, C, generator=g)
        x += 0.5 * (torch.arange(HW) / HW - 0.5)[None, :, None]
        x += 0.3 * (torch.arange(NF) % 3)[:, None, None]
        x[..., cpg:2 * cpg] *= math.sqrt(case.eps)
        if case.data == "mean2048":
            x[..., 2 * cpg + 1:3 * cpg:2] += 2048
        elif case.data == "wide":
            x[..., 3 * cpg:4 * cpg:2] = x[..., 3 * cpg:4 * cpg:2] * 500 - 33000
            x[..., 3 * cpg + 1:4 * cpg:2] = x[..., 3 * cpg + 1:4 * cpg:2] * 500 + 33000
    x = x.half()
    x0, x1 = x[..., :case.C0].contiguous(), (x[..., case.C0:].contiguous() if case.C1 else None)
    return x0.to(device), (x1.to(device) if x1 is not None else None), gamma.to(device), beta.to(device)


def gn_ref(x, gamma, beta, G, fps, eps, silu, ddof=0, per_frame=False, edge_shift=False, keep_pixels=None):
    """float64 GroupNorm (+SiLU) of x [NF, HW, C] with statistics over (fps frames, HW, C / G channels); the keyword
    arguments produce the wrong answers. Returns (y, xhat)."""
    NF, HW, C = x.shape
    xs = torch.cat([x[..., 1:], x[..., -1:]], -1) if edge_shift else x
    if keep_pixels is not None:
        xs = xs[:, :keep_pixels]
    f = 1 if per_frame else fps
    xg = xs.reshape(NF // f, f, xs.shape[1], G, C // G)
    mean = xg.mean((1, 2, 4))
    var = xg.var((1, 2, 4), correction=ddof)
    mean = mean.repeat_interleave(C // G, 1).repeat_interleave(f, 0)[:, None]
    var = var.repeat_interleave(C // G, 1).repeat_interleave(f, 0)[:, None]
    xhat = (x - mean) / torch.sqrt(var + eps)
    z = xhat * gamma.double() + beta.double()
    return (z * torch.sigmoid(z) if silu else z), xhat


def _gn_check_and_wrong(case, x0, x1, gamma, beta):
    x = (x0 if x1 is None else torch.cat([x0, x1], 2)).double()
    kw = dict(G=32, fps=case.fps, eps=case.eps, silu=case.silu)
    ref, xhat = gn_ref(x, gamma, beta, **kw)
    bound = _norm_bound(ref, gamma, xhat, case.silu)
    plan = gn_plan(case.C, case.NF, case.HW, case.fps)
    wrong = {}
    if case.data != "zero":
        if case.C // 32 * case.HW * case.fps <= 512:
            wrong["variance with N-1"] = lambda: gn_ref(x, gamma, beta, ddof=1, **kw)[0]
        wrong["eps x 10"] = lambda: gn_ref(x, gamma, beta, **{**kw, "eps": 10 * case.eps})[0]
        if case.fps > 1:
            wrong["per-frame statistics"] = lambda: gn_ref(x, gamma, beta, per_frame=True, **kw)[0]
        wrong["group edge one channel off"] = lambda: gn_ref(x, gamma, beta, edge_shift=True, **kw)[0]
        if plan["chunks"] > 1:
            keep = case.HW * (plan["chunks"] - 1) // plan["chunks"]
            wrong["last pixel chunk left out"] = lambda: gn_ref(x, gamma, beta, keep_pixels=keep, **kw)[0]
    return ref, bound, wrong


def _gn_assert_plan(case):
    plan = gn_plan(case.C, case.NF, case.HW, case.fps)
    got = {k: plan[k] for k in case.expect}
    assert got == case.expect, (case.id, got, case.expect)


@pytest.mark.parametrize("case", [c for c in GN_CASES if c.NF * c.HW * c.C <= 4 << 20], ids=lambda c: c.id)
def test_groupnorm_bounds_catch_wrong_answers(case):
    """Host only: the launch path each case is meant to reach, and every applicable wrong answer breaking the bound on
    the case's own data (the larger cases run the same check on the GPU in test_groupnorm_edges)."""
    _gn_assert_plan(case)
    x0, x1, gamma, beta = gn_inputs(case, "cpu")
    ref, bound, wrong = _gn_check_and_wrong(case, x0, x1, gamma, beta)
    assert case.data == "zero" or wrong
    _assert_catches({k: f() for k, f in wrong.items()}, ref, bound, case.id)


@pytest.mark.gpu
@pytest.mark.parametrize("fused", [False, True], ids=["three_launch", "fused"])
@pytest.mark.parametrize("case", GN_CASES, ids=lambda c: c.id)
def test_groupnorm_edges(ops, case, fused):
    _gn_assert_plan(case)
    x0, x1, gamma, beta = gn_inputs(case, dev)
    y = ops.groupnorm(x0, gamma, beta, 32, case.fps, case.eps, case.silu, x1, fused=fused)
    if fused and case.fps == 1:   # same partial layout and reduction order as the three launches
        assert torch.equal(y, ops.groupnorm(x0, gamma, beta, 32, case.fps, case.eps, case.silu, x1))
    ref, bound, wrong = _gn_check_and_wrong(case, x0, x1, gamma, beta)
    if case.data == "zero":       # zero variance: (0 - 0) * rsqrt(eps) * gamma + beta is beta, bit for bit
        assert torch.equal(y, beta.half().expand_as(y)), case.id
    if not fused and case.NF * case.HW * case.C > 4 << 20:
        _assert_catches({k: f() for k, f in wrong.items()}, ref, bound, case.id)
    _record(f"groupnorm_{case.id}_{'fused' if fused else 'three_launch'}_vs_fp64", _ratio(y, ref, bound), 1.0)


@pytest.mark.gpu
@pytest.mark.parametrize("fused", [False, True], ids=["three_launch", "fused"])
def test_groupnorm_refuses_before_launch(ops, fused):
    """Odd channels per group, a first input whose width breaks the 8-channel vectors, more than 64 groups and a frame
    count that is not a multiple of frames_per_stat are refused before anything is launched."""
    from musev_b200 import _capi
    from musev_b200._capi import MvbError
    g = torch.ones(640, device=dev)
    n0 = _capi.launch_count()
    for C0, C1, NF, G, fps in ((96, 0, 2, 32, 1),        # 3 channels per group
                               (324, 316, 2, 32, 1),     # C0 % 8 != 0
                               (640, 0, 2, 80, 1),       # 80 groups
                               (640, 0, 5, 32, 2)):      # NF % frames_per_stat != 0
        x0 = torch.zeros(NF, 16, C0, dtype=torch.float16, device=dev)
        x1 = torch.zeros(NF, 16, C1, dtype=torch.float16, device=dev) if C1 else None
        with pytest.raises(MvbError, match="mvb_op_groupnorm"):
            ops.groupnorm(x0, g[:C0 + C1], g[:C0 + C1], G, fps, 1e-5, False, x1, fused=fused)
    torch.cuda.synchronize()
    assert _capi.launch_count() == n0


# ------------------------------------------------------------------------------------------------ LayerNorm
LN_CS = (64, 256, 264, 512, 520, 768, 1024, 320, 640, 1280, 1288, 2560)
LN_MS = (1, 7, 9, 77, 257)
LN_KERNEL = {64: "layernorm_kernel<1,4>", 256: "layernorm_kernel<1,4>", 264: "layernorm_kernel<2,4>",
             512: "layernorm_kernel<2,4>", 520: "layernorm_kernel<5,2>", 768: "layernorm_kernel<5,2>",
             1024: "layernorm_kernel<5,2>", 320: "layernorm40<8>", 640: "layernorm40<16>", 1280: "layernorm40<32>",
             1288: "layernorm_kernel<10,1>", 2560: "layernorm_kernel<10,1>"}
# rows past the grid-stride cap (132 * 8 blocks of 8 warps, 32 / L rows per warp), with a ragged last warp
LN_STRIDE_M = {320: 1056 * 8 * 4 + 23, 640: 1056 * 8 * 2 + 13, 1280: 1056 * 8 + 7}


def ln_inputs(M, C, eps, seed, device):
    """x [M, C] fp16: rows cycle through N(0, 3^2) + 1, mean 300 / std 1, variance ~9 eps (N(0, 1e-4) when eps = 0)
    and, with eps > 0, the constant 0.5."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, C, generator=g) * 3 + 1
    x[1::4] = torch.randn(x[1::4].shape, generator=g) + 300
    x[2::4] = torch.randn(x[2::4].shape, generator=g) * (3 * math.sqrt(eps) if eps > 0 else 1e-2)
    if eps > 0:
        x[3::4] = 0.5
    gamma, beta = torch.randn(C, generator=g), torch.randn(C, generator=g) * 0.5
    return x.half().to(device), gamma.to(device), beta.to(device)


def ln_ref(x, gamma, beta, eps, ddof=0):
    xd = x.double()
    xhat = (xd - xd.mean(1, keepdim=True)) / torch.sqrt(xd.var(1, correction=ddof, keepdim=True) + eps)
    return xhat * gamma.double() + beta.double(), xhat


def _ln_check_and_wrong(x, gamma, beta, eps):
    M, C = x.shape
    ref, xhat = ln_ref(x, gamma, beta, eps)
    bound = _norm_bound(ref, gamma, xhat, False)
    wrong = {}
    if C <= 512:
        wrong["variance with N-1"] = lambda: ln_ref(x, gamma, beta, eps, ddof=1)[0]
    if eps > 0 and M >= 3:
        wrong["eps x 10"] = lambda: ln_ref(x, gamma, beta, 10 * eps)[0]
    return ref, bound, wrong


@pytest.mark.parametrize("eps", [0.0, 1e-5])
@pytest.mark.parametrize("C", LN_CS)
def test_layernorm_bounds_catch_wrong_answers(C, eps):
    """Host only: the instantiation each width dispatches to, and the wrong answers breaking the bound."""
    for M in LN_MS:
        assert ln_plan(C, M) == {"kernel": LN_KERNEL[C], "grid_stride": False}
        x, gamma, beta = ln_inputs(M, C, eps, C * 10 + M, "cpu")
        ref, bound, wrong = _ln_check_and_wrong(x, gamma, beta, eps)
        _assert_catches({k: f() for k, f in wrong.items()}, ref, bound, f"C={C} M={M} eps={eps}")
    if C in LN_STRIDE_M:
        assert ln_plan(C, LN_STRIDE_M[C]) == {"kernel": LN_KERNEL[C], "grid_stride": True}


@pytest.mark.gpu
@pytest.mark.parametrize("eps", [0.0, 1e-5])
@pytest.mark.parametrize("C", LN_CS)
def test_layernorm_edges(ops, C, eps):
    """Every width the engine runs, at row counts around the per-warp row groups. The constant rows (eps > 0) give beta
    within the bound; the mean-300 rows test the centred variance."""
    worst, where = 0.0, ""
    for M in LN_MS:
        assert ln_plan(C, M)["kernel"] == LN_KERNEL[C]
        x, gamma, beta = ln_inputs(M, C, eps, C * 10 + M, dev)
        y = ops.layernorm(x, gamma, beta, eps)
        ref, bound, _ = _ln_check_and_wrong(x, gamma, beta, eps)
        r = _ratio(y, ref, bound)
        if r > worst:
            worst, where = r, f"M={M}"
    _record(f"layernorm_C{C}_eps{eps:g}_vs_fp64", worst, 1.0, where)


@pytest.mark.gpu
@pytest.mark.parametrize("C", sorted(LN_STRIDE_M))
def test_layernorm40_grid_stride(ops, C):
    """More row groups than the capped grid has warps: every warp goes round its grid-stride loop, the last pass ragged."""
    M = LN_STRIDE_M[C]
    plan = ln_plan(C, M)
    assert plan == {"kernel": LN_KERNEL[C], "grid_stride": True}
    x, gamma, beta = ln_inputs(M, C, 1e-5, C + 1, dev)
    y = ops.layernorm(x, gamma, beta, 1e-5)
    ref, bound, _ = _ln_check_and_wrong(x, gamma, beta, 1e-5)
    _record(f"layernorm40_C{C}_grid_stride_M{M}_vs_fp64", _ratio(y, ref, bound), 1.0)


@pytest.mark.gpu
def test_layernorm_refuses_before_launch(ops):
    """Widths past 2560 and widths that break the 8-channel vectors are refused before anything is launched."""
    from musev_b200 import _capi
    from musev_b200._capi import MvbError
    n0 = _capi.launch_count()
    for C in (2568, 100):
        x = torch.zeros(4, C, dtype=torch.float16, device=dev)
        g = torch.ones(C, device=dev)
        with pytest.raises(MvbError, match="mvb_op_layernorm"):
            ops.layernorm(x, g, g, 1e-5)
    torch.cuda.synchronize()
    assert _capi.launch_count() == n0


# ------------------------------------------------------------------------------------------------ row softmax
SM_NS = (8, 64, 4096, 6144, 8184, 8192)
SM_DATA = ("sigma1", "sigma30", "one_hot", "near_fp16_max")
SM_SCALES = (1.0, 512 ** -0.5)
SM_LAYOUTS = ((37, 24), (8, 0))       # (rows, spare columns past N): 37 rows end in a partly idle block


def sm_inputs(N, data, scale, M, spare, seed, device):
    """Scores [M, N + spare] fp16; the spare columns hold a sentinel."""
    g = torch.Generator().manual_seed(seed)
    if data in ("sigma1", "sigma30"):
        s = torch.randn(M, N, generator=g) * (1.0 if data == "sigma1" else 30.0)
    elif data == "one_hot":     # one score 40 units (after the scale) above zeros; row 0's in the last column
        s = torch.zeros(M, N)
        s[torch.arange(M), (torch.arange(M) * 7919 + N - 1) % N] = 40.0 / scale
    else:                       # half the columns within 8 fp16 steps below 65504, half around -6e4
        hi = torch.rand(M, N, generator=g) < 0.5
        s = torch.where(hi, 65504.0 - 32.0 * torch.randint(0, 8, (M, N), generator=g),
                        -60000.0 - 32.0 * torch.randint(0, 8, (M, N), generator=g))
    x = torch.full((M, N + spare), -1234.0)
    x[:, :N] = s
    return x.half().to(device)


def sm_ref(s, scale):
    return torch.softmax(scale * s.double(), -1)


def _sm_check_and_wrong(s, N, scale, data):
    ref = sm_ref(s, scale)
    bound = 1.5 * _ulp16(ref) + 1e-4 * ref
    drop = s.double().clone()
    if N > 8:
        drop[:, :N - 8] = sm_ref(s[:, :N - 8], scale)
    wrong = {"last 8 columns dropped": lambda: drop}
    if scale != 1.0 and data != "one_hot":
        wrong["scale ignored"] = lambda: sm_ref(s, 1.0)
    return ref, bound, wrong


@pytest.mark.parametrize("data", SM_DATA)
@pytest.mark.parametrize("N", SM_NS)
def test_softmax_rows_bounds_catch_wrong_answers(N, data):
    for scale in SM_SCALES:
        s = sm_inputs(N, data, scale, 37, 0, N + SM_DATA.index(data), "cpu")
        ref, bound, wrong = _sm_check_and_wrong(s, N, scale, data)
        _assert_catches({k: f() for k, f in wrong.items()}, ref, bound, f"N={N} {data} scale={scale:g}")


@pytest.mark.gpu
@pytest.mark.parametrize("data", SM_DATA)
@pytest.mark.parametrize("N", SM_NS)
def test_softmax_rows_edges(ops, N, data):
    """In place on [M, N] inside a wider row (ld = N + 24, whose spare columns must come back untouched) and on a dense
    [8, N]; scales 1 and 1/sqrt(512)."""
    worst, where = 0.0, ""
    for scale in SM_SCALES:
        for M, spare in SM_LAYOUTS:
            x = sm_inputs(N, data, scale, M, spare, N + SM_DATA.index(data), dev)
            s = x[:, :N].clone()
            ops.softmax_rows(x, scale, N)
            assert (x[:, N:] == -1234.0).all(), f"scale={scale:g} M={M}: columns past N were written"
            ref, bound, _ = _sm_check_and_wrong(s, N, scale, data)
            r = _ratio(x[:, :N], ref, bound)
            if r > worst:
                worst, where = r, f"scale={scale:g} M={M} ld={N + spare}"
    _record(f"softmax_rows_N{N}_{data}_vs_fp64", worst, 1.0, where)


@pytest.mark.gpu
def test_softmax_rows_refuses_before_launch(ops):
    """A row length that breaks the 8-column vectors, rows past 8192 columns and a row stride that breaks the 16-byte
    alignment are refused before anything is launched."""
    from musev_b200 import _capi
    from musev_b200._capi import MvbError
    x = torch.zeros(4, 8208, dtype=torch.float16, device=dev)
    n0 = _capi.launch_count()
    for N, ld in ((12, 16), (8200, 8208), (64, 68)):
        with pytest.raises(MvbError, match="mvb_op_softmax_rows"):
            _capi.check(_capi.lib().mvb_op_softmax_rows(x.data_ptr(), 4, N, ld, 1.0, torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    assert _capi.launch_count() == n0
