"""The step epilogues that run on every denoise step: `mvb_fuse_cfg_ddim`, `mvb_fuse_cfg_affine` and
`mvb_accumulate_window`, at every branch, against float64 restatements of the header's formulas:
    eps  = eps_sum[b] / counter[t]; cfg: eps = u + g (x_text - u), u the uncond half, x_text the half n = B C T HW
           elements further on (eps_sum is [2B, C, T, HW], uncond first)
    DDIM x0 / eps from eps (prediction_type 0), v (1) or sample (2); x0 clamped to +-clip when clip > 0; with
         use_clipped_model_output eps = (x - sqrt(a_t) x0) / sqrt(1 - a_t); x_prev = sqrt(a_prev) x0
         + sqrt(1 - a_prev - std^2) eps (+ std noise); eps_out holds the guided model output `eps` above, before any
         v / sample conversion; x0_out the clamped x0
    affine x_prev = c_x x + c_e eps (+ c_n noise); aux_out = a_x x + a_e eps; eps_out as above
    window eps_sum[:, :, frames[k]] += win[:, :, src_t0 + k], one fp32 add per element.
The DDIM kernel is also compared with `oracle.pipeline_oracle.DDIMOracle.step` run in float64 with the same a_t / a_prev
and eta (the oracle has no use_clipped_model_output; those cases use the restatement only).

Each fp32 output is held to C_STEP fp32 half-ulps (2^-24) of the sum of the magnitudes of its terms, propagated
through every operation of the formula (|a - b| -> |a| + |b|, constants by their absolute values); fp16 latents add
one rounding, ulp16(ref) / 2. The window accumulation must be bit-identical to
`eps_sum[:, :, frames] += win[:, :, src_t0:src_t0 + nframes].float()` in torch, and every frame not listed must keep
its bits. The bounds discriminate: `test_step_bounds_catch_wrong_answers` (no GPU) computes named wrong answers in
float64 (CFG halves swapped; the text half taken per batch item; the counter indexed by channel; v-prediction with
sqrt(a_t) and sqrt(1 - a_t) swapped; the clip applied to eps; use_clipped_model_output ignored; the noise scaled by
the direction coefficient; fp16 latents rounded before the update as well as after it; window frame k read at
src_t0 + frames[k]; `=` in place of `+=`), rounds them as the kernel would and asserts that each breaks its bound.

DDIM runs the full product of prediction type x clip (off / on where it clamps) x use_clipped x std (0 / > 0 with
noise / > 0 with NULL noise) x fp32 / fp16 latents x cfg x counter (NULL / 1..3 per frame) x eps_out / x0_out given
or NULL at (B, C, T, HW) = (3, 4, 5, 37), and a seeded pairwise cover of the same options plus the timestep at
(1, 4, 16, 4096), the headline step, and at (2, 4, 33, 4096), where n > 132 x 8 x 256 so the grid-stride loop runs.
An empty extent of any of the four step entry points (multistep included) returns MVB_OK, launches nothing and
touches no buffer; a negative extent, or a window outside [0, Tw), is refused before any launch.

With MVB_PARITY_LOG=<file> set, the worst ratio |out - ref| / bound of every case is appended to <file>. Measured on
an H100 80GB HBM3 at 700 W, worst ratio per group: DDIM x_prev with fp32 latents 0.222 (product and pairwise), with
fp16 latents 0.998; DDIM against the oracle 0.998 (fp16 latents); eps_out / x0_out 0.198; affine x_prev 0.998 (fp16
latents), aux_out / eps_out 0.189. The fp32 outputs therefore stay within 3.6 half-ulps of the sum of their terms'
magnitudes, and C_STEP = 16 keeps 4.5x above that; the fp16 ratios sit near 1 because a correctly rounded result may
lie half an ulp away.
"""
import ctypes as C
import itertools
import json
import os
import random
import zlib

import numpy as np
import pytest
import torch

from oracle.pipeline_oracle import SD15_DDIM, DDIMOracle

C_STEP = 16.0                # bound on fp32 outputs, in units of 2^-24 x (sum of the magnitudes of the terms)
U32 = 2.0 ** -24
GRID_STRIDE_N = 132 * 8 * 256
dev = "cuda"

DDIM_OPTS = {"pred": (0, 1, 2), "clip": (False, True), "use_clipped": (0, 1), "std": ("0", "noise", "null_noise"),
             "f16": (False, True), "cfg": (1, 0), "counter": (False, True), "outs": ("none", "eps", "x0", "both")}
AFFINE_OPTS = {"cfg": (1, 0), "f16": (False, True), "counter": (False, True), "noise": (False, True),
               "outs": ("none", "aux", "eps", "both")}
SMALL = (3, 4, 5, 37)                          # B > 1, odd HW
LARGE = ((1, 4, 16, 4096), (2, 4, 33, 4096))   # the headline step; n past one grid of 132 x 8 x 256 threads
TIMESTEPS = (951, 501, 1)
AFFINE_COEF = dict(c_x=0.97, c_e=-0.31, c_n=0.2, a_x=1.3, a_e=-0.7)
G = 3.5
CLIP = 1.0
ETA = 0.8


def f32(v):
    return float(np.float32(v))


def pairwise(factors, seed):
    """A seeded covering array of strength 2: a list of {name: value} rows in which every pair of values of every two
    factors occurs."""
    names = list(factors)
    sizes = [len(factors[n]) for n in names]
    todo = {(i, a, j, b) for i, j in itertools.combinations(range(len(names)), 2) for a in range(sizes[i])
            for b in range(sizes[j])}
    rng = random.Random(seed)
    rows = []
    while todo:
        i, a, j, b = min(todo)
        best, best_n = None, -1
        for _ in range(64):
            r = [rng.randrange(s) for s in sizes]
            r[i], r[j] = a, b
            n = sum((p, r[p], q, r[q]) in todo for p, q in itertools.combinations(range(len(names)), 2))
            if n > best_n:
                best, best_n = r, n
        todo -= {(p, best[p], q, best[q]) for p, q in itertools.combinations(range(len(names)), 2)}
        rows.append({n: factors[n][v] for n, v in zip(names, best)})
    return rows


def _product(opts):
    return [dict(zip(opts, vals)) for vals in itertools.product(*opts.values())]


def _ulp16(r):
    _, e = torch.frexp(r.abs())
    return torch.where(r.abs() < 2.0 ** -14, torch.full_like(r, 2.0 ** -24), torch.ldexp(torch.ones_like(r), e - 11))


def _schedule(t):
    """(a_t, a_prev, std at ETA) of SD-1.5's DDIM at timestep t of a 20-step run, as the kernel receives them."""
    o = DDIMOracle(**SD15_DDIM)
    o.set_timesteps(20)
    prev_t = t - 1000 // 20
    a_t = float(o.alphas_cumprod[t])
    a_p = float(o.alphas_cumprod[prev_t]) if prev_t >= 0 else float(o.final_alpha_cumprod)
    return a_t, a_p, float(ETA * o._get_variance(t, prev_t) ** 0.5)


# ------------------------------------------------------------------------------------------------ float64 references
def guided_eps(es, counter, B, cfg, g, wrong=()):
    """(eps, |terms| of eps) in float64, [B, C, T, HW]."""
    es = es.double()
    _, Cc, T, _ = es.shape
    cnt = counter.double() if counter is not None else torch.ones(T, dtype=torch.float64, device=es.device)
    cnt = cnt[:Cc].view(Cc, 1, 1) if "counter indexed by channel" in wrong else cnt.view(1, T, 1)
    if cfg:
        if "text half taken per batch item" in wrong:
            u, tx = es[0::2] / cnt, es[1::2] / cnt
        else:
            u, tx = es[:B] / cnt, es[B:] / cnt
        if "cfg halves swapped" in wrong:
            u, tx = tx, u
        return u + g * (tx - u), u.abs() + abs(g) * (tx.abs() + u.abs())
    return es / cnt, (es / cnt).abs()


def ddim_ref(es, counter, x, g, a_t, a_p, pred, clip, use_clipped, std, noise, cfg, wrong=()):
    """float64 restatement of mvb_fuse_cfg_ddim: {name: (value, magnitude)} for prev, eps, x0, and the count of x0
    elements the clip changed."""
    B = x.shape[0]
    e, me = guided_eps(es, counter, B, cfg, f32(g), wrong)
    xd = x.double()
    mx = xd.abs()
    a_t, a_p, std, clip = f32(a_t), f32(a_p), f32(std), f32(clip)
    sa, sb, sap = a_t ** 0.5, (1 - a_t) ** 0.5, a_p ** 0.5
    sdir = max(1 - a_p - std * std, 0.0) ** 0.5
    if pred == 0:
        x0, mx0, eps, meps = (xd - sb * e) / sa, (mx + sb * me) / sa, e, me
    elif pred == 1:
        if "v-prediction with sqrt(a_t) and sqrt(1 - a_t) swapped" in wrong:
            sa, sb = sb, sa
        x0, mx0 = sa * xd - sb * e, sa * mx + sb * me
        eps, meps = sa * e + sb * xd, sa * me + sb * mx
        sa, sb = a_t ** 0.5, (1 - a_t) ** 0.5
    else:
        x0, mx0 = e, me
        eps, meps = (xd - sa * x0) / sb, (mx + sa * mx0) / sb
    clamped = 0
    if clip > 0:
        if "clip applied to eps" in wrong:
            eps = eps.clamp(-clip, clip)
            x0 = (xd - sb * eps) / sa if pred == 0 else x0
        else:
            clamped = int((x0.abs() > clip).sum())
            x0 = x0.clamp(-clip, clip)
    if use_clipped and "use_clipped ignored" not in wrong:
        eps, meps = (xd - sa * x0) / sb, (mx + sa * mx0) / sb
    if "fp16 latents rounded before the update as well as after it" in wrong:
        prev = (sap * x0).half().double() + sdir * eps
    else:
        prev = sap * x0 + sdir * eps
    mprev = sap * mx0 + sdir * meps
    if noise is not None:
        nz = noise.double()
        prev = prev + (sdir if "noise scaled by the direction coefficient" in wrong else std) * nz
        mprev = mprev + std * nz.abs()
    return {"prev": (prev, mprev), "eps": (e, me), "x0": (x0, mx0)}, clamped


def affine_ref(es, counter, x, g, c_x, c_e, c_n, noise, a_x, a_e, cfg, wrong=()):
    B = x.shape[0]
    e, me = guided_eps(es, counter, B, cfg, f32(g), wrong)
    xd = x.double()
    c_x, c_e, c_n, a_x, a_e = map(f32, (c_x, c_e, c_n, a_x, a_e))
    prev, mprev = c_x * xd + c_e * e, abs(c_x) * xd.abs() + abs(c_e) * me
    if noise is not None:
        prev, mprev = prev + c_n * noise.double(), mprev + abs(c_n) * noise.double().abs()
    return {"prev": (prev, mprev), "aux": (a_x * xd + a_e * e, abs(a_x) * xd.abs() + abs(a_e) * me), "eps": (e, me)}


def window_ref(es, win, src_t0, frames, wrong=()):
    out = es.clone()
    n = len(frames)
    idx = torch.as_tensor(frames, dtype=torch.long, device=es.device)
    if "window frame k read at src_t0 + frames[k]" in wrong:
        src = win[:, :, (idx + src_t0)].float()
    else:
        src = win[:, :, src_t0:src_t0 + n].float()
    if "= in place of +=" in wrong:
        out[:, :, idx] = src
    else:
        out[:, :, idx] += src
    return out


def _ratio(got, ref, mag, f16):
    """max |got - ref| / bound over the elements; got as the kernel returns it (fp16 latents or fp32)."""
    got = got.double()
    if not torch.isfinite(got).all():
        return float("inf")
    bound = C_STEP * U32 * mag + (0.5 * _ulp16(ref) if f16 else 0.0)
    return ((got - ref).abs() / bound.clamp_min(1e-300)).max().item()


def _record(name, err, bound=1.0):
    path = os.environ.get("MVB_PARITY_LOG")
    if path:
        try:
            with open(path, "a") as fh:
                fh.write(json.dumps({"test": name, "value": err, "bound": bound}) + "\n")
        except OSError:
            pass
    assert err <= bound, (name, err, bound)


# ------------------------------------------------------------------------------------------------ inputs
def ddim_inputs(shape, o, seed, device):
    B, Cc, T, HW = shape
    g = torch.Generator(device=device).manual_seed(seed)
    es = torch.randn((2 * B if o["cfg"] else B, Cc, T, HW), generator=g, device=device) * 2.0
    counter = torch.randint(1, 4, (T,), generator=g, device=device).float() if o["counter"] else None
    x = torch.randn((B, Cc, T, HW), generator=g, device=device)
    x = x.half() if o["f16"] else x
    noise = torch.randn((B, Cc, T, HW), generator=g, device=device)
    return es, counter, x, noise


def _name(o):
    return "_".join(f"{k}{v}" for k, v in o.items())


# ------------------------------------------------------------------------------------------------ host checks
def test_pairwise_covers_every_pair():
    for opts in (dict(DDIM_OPTS, t=TIMESTEPS), AFFINE_OPTS):
        rows = pairwise(opts, 1)
        for a, b in itertools.combinations(opts, 2):
            assert {(r[a], r[b]) for r in rows} == set(itertools.product(opts[a], opts[b])), (a, b)
    assert np.prod(LARGE[1]) > GRID_STRIDE_N
    assert len(_product(DDIM_OPTS)) == 1152


def _host_ddim(o, wrong, t=501, shape=(2, 4, 5, 7)):
    es, counter, x, noise = ddim_inputs(shape, o, zlib.crc32(_name(o).encode()), "cpu")
    a_t, a_p, std = _schedule(t)
    std = std if o["std"] != "0" else 0.0
    nz = noise if o["std"] == "noise" else None
    clip = CLIP if o["clip"] else 0.0
    args = (es, counter, x, G, a_t, a_p, o["pred"], clip, o["use_clipped"], std, nz, o["cfg"])
    ref, _ = ddim_ref(*args)
    bad, _ = ddim_ref(*args, wrong=(wrong,))
    y = bad["prev"][0]
    y = y.half() if o["f16"] else y.float()
    return _ratio(y, *ref["prev"], o["f16"])


DDIM_BASE = dict(pred=0, clip=False, use_clipped=0, std="0", f16=False, cfg=1, counter=True, outs="none")
HOST_WRONG = {
    "cfg halves swapped": {},
    "text half taken per batch item": {},
    "counter indexed by channel": {},
    "v-prediction with sqrt(a_t) and sqrt(1 - a_t) swapped": dict(pred=1),
    "clip applied to eps": dict(clip=True),
    "use_clipped ignored": dict(clip=True, use_clipped=1),
    "noise scaled by the direction coefficient": dict(std="noise"),
    "fp16 latents rounded before the update as well as after it": dict(f16=True),
}


@pytest.mark.parametrize("wrong", list(HOST_WRONG) + ["window frame k read at src_t0 + frames[k]", "= in place of +="])
def test_step_bounds_catch_wrong_answers(wrong):
    """Host only: every named wrong answer, rounded as the kernel would return it, breaks its bound; the correct
    answer rounded the same way keeps it."""
    if wrong in HOST_WRONG:
        o = dict(DDIM_BASE, **HOST_WRONG[wrong])
        assert _host_ddim(o, None) <= 1.0
        r = _host_ddim(o, wrong)
        assert r > 1.0, f"the wrong answer '{wrong}' stays inside the bound (worst ratio {r:.3g})"
        if wrong in ("cfg halves swapped", "counter indexed by channel", "text half taken per batch item"):
            es, counter, x, noise = ddim_inputs((2, 4, 5, 7), DDIM_BASE, 3, "cpu")
            k = AFFINE_COEF
            args = (es, counter, x, G, k["c_x"], k["c_e"], k["c_n"], noise, k["a_x"], k["a_e"], 1)
            ref, bad = affine_ref(*args), affine_ref(*args, wrong=(wrong,))
            assert _ratio(bad["prev"][0].float(), *ref["prev"], False) > 1.0
    else:
        g = torch.Generator().manual_seed(5)
        es = torch.randn(2, 4, 20, 37, generator=g)
        win = torch.randn(2, 4, 9, 37, generator=g).half()
        frames = [3, 4, 0, 1]          # wrapped, and inside the window when read at src_t0 + frames[k]
        assert not torch.equal(window_ref(es, win, 2, frames, wrong=(wrong,)), window_ref(es, win, 2, frames))


# ------------------------------------------------------------------------------------------------ GPU: DDIM
def _ddim_case(shape, o, t, seed):
    """Runs one combination; returns {output: worst ratio} against the restatement (and the oracle), and the clamp
    count."""
    from musev_b200 import ops
    es, counter, x, noise = ddim_inputs(shape, o, seed, dev)
    a_t, a_p, std_eta = _schedule(t)
    std = 0.0 if o["std"] == "0" else std_eta
    nz = noise if o["std"] == "noise" else None
    clip = CLIP if o["clip"] else 0.0
    n = x.numel()
    eps_out = torch.full(x.shape, float("nan"), device=dev) if o["outs"] in ("eps", "both") else None
    x0_out = torch.full(x.shape, float("nan"), device=dev) if o["outs"] in ("x0", "both") else None
    out = ops.fuse_cfg_ddim(es.view(*es.shape, 1), counter, x.view(*x.shape, 1), G, a_t, a_p,
                            o["pred"], clip, cfg=bool(o["cfg"]), use_clipped=bool(o["use_clipped"]), std_dev=std, noise=nz,
                            eps_out=None if eps_out is None else eps_out.view(*x.shape, 1),
                            x0_out=None if x0_out is None else x0_out.view(*x.shape, 1)).view(x.shape)
    torch.cuda.synchronize()
    assert out.dtype == x.dtype and out.numel() == n
    ref, clamped = ddim_ref(es, counter, x, G, a_t, a_p, o["pred"], clip, o["use_clipped"], std, nz, o["cfg"])
    r = {"prev": _ratio(out, *ref["prev"], o["f16"])}
    if eps_out is not None:
        r["eps_out"] = _ratio(eps_out, *ref["eps"], False)
    if x0_out is not None:
        r["x0_out"] = _ratio(x0_out, *ref["x0"], False)
    if not o["use_clipped"]:
        orc = DDIMOracle(**dict(SD15_DDIM, prediction_type=("epsilon", "v_prediction", "sample")[o["pred"]],
                                clip_sample=o["clip"], clip_sample_range=CLIP))
        orc.set_timesteps(20)
        e = ref["eps"][0]
        prev_o, x0_o = orc.step(e, t, x.double(), eta=ETA if std > 0 else 0.0,
                                variance_noise=(nz.double() if nz is not None else torch.zeros_like(e)) if std > 0 else None)
        r["prev_vs_oracle"] = _ratio(out, prev_o, ref["prev"][1], o["f16"])
        if x0_out is not None:
            r["x0_vs_oracle"] = _ratio(x0_out, x0_o, ref["x0"][1], False)
    return r, clamped


def _check_ddim(name, o, r, clamped):
    if o["clip"]:
        assert clamped > 0, (name, "the clip changed nothing")
    for k, v in r.items():
        _record(f"{name}_{k}", v)


@pytest.mark.gpu
@pytest.mark.parametrize("pred", DDIM_OPTS["pred"])
@pytest.mark.parametrize("f16", DDIM_OPTS["f16"], ids=["f32", "f16"])
def test_fuse_cfg_ddim_product(built_lib, pred, f16):
    """Every combination of the other options at (3, 4, 5, 37)."""
    rest = {k: v for k, v in DDIM_OPTS.items() if k not in ("pred", "f16")}
    for o in _product(rest):
        o = dict(o, pred=pred, f16=f16)
        r, clamped = _ddim_case(SMALL, o, 501, zlib.crc32(_name(o).encode()))
        _check_ddim(f"fuse_cfg_ddim_small_{_name(o)}", o, r, clamped)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", LARGE, ids=["headline", "grid_stride"])
def test_fuse_cfg_ddim_pairwise(built_lib, shape):
    """A seeded pairwise cover of the options and three timesteps at the headline step and past one grid."""
    for o in pairwise(dict(DDIM_OPTS, t=TIMESTEPS), zlib.crc32(str(shape).encode())):
        t = o.pop("t")
        r, clamped = _ddim_case(shape, o, t, zlib.crc32((_name(o) + str(t)).encode()))
        _check_ddim(f"fuse_cfg_ddim_{'x'.join(map(str, shape))}_t{t}_{_name(o)}", o, r, clamped)


# ------------------------------------------------------------------------------------------------ GPU: affine
def _affine_case(shape, o, seed):
    from musev_b200 import ops
    es, counter, x, noise = ddim_inputs(shape, o, seed, dev)
    nz = noise if o["noise"] else None
    aux = torch.full(x.shape, float("nan"), device=dev) if o["outs"] in ("aux", "both") else None
    eps_out = torch.full(x.shape, float("nan"), device=dev) if o["outs"] in ("eps", "both") else None
    k = AFFINE_COEF
    out = ops.fuse_cfg_affine(es.view(*es.shape, 1), counter, x.view(*x.shape, 1), G, k["c_x"], k["c_e"], k["c_n"],
                              None if nz is None else nz.view(*x.shape, 1), k["a_x"], k["a_e"],
                              None if aux is None else aux.view(*x.shape, 1),
                              None if eps_out is None else eps_out.view(*x.shape, 1), cfg=bool(o["cfg"])).view(x.shape)
    torch.cuda.synchronize()
    ref = affine_ref(es, counter, x, G, k["c_x"], k["c_e"], k["c_n"], nz, k["a_x"], k["a_e"], o["cfg"])
    r = {"prev": _ratio(out, *ref["prev"], o["f16"])}
    if aux is not None:
        r["aux_out"] = _ratio(aux, *ref["aux"], False)
    if eps_out is not None:
        r["eps_out"] = _ratio(eps_out, *ref["eps"], False)
    return r


@pytest.mark.gpu
def test_fuse_cfg_affine_product(built_lib):
    for o in _product(AFFINE_OPTS):
        for k, v in _affine_case(SMALL, o, zlib.crc32(_name(o).encode())).items():
            _record(f"fuse_cfg_affine_small_{_name(o)}_{k}", v)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", LARGE, ids=["headline", "grid_stride"])
def test_fuse_cfg_affine_pairwise(built_lib, shape):
    for o in pairwise(AFFINE_OPTS, zlib.crc32(str(shape).encode())):
        for k, v in _affine_case(shape, o, zlib.crc32(_name(o).encode())).items():
            _record(f"fuse_cfg_affine_{'x'.join(map(str, shape))}_{_name(o)}_{k}", v)


# ------------------------------------------------------------------------------------------------ GPU: window
WINDOW_CASES = {
    #                   dtype  B2 C  T   HW    Tw  src_t0 frames
    "f32_b1":          ("f32", 1, 4, 12, 37, 6, 0, [3, 4, 5, 6, 7, 8]),
    "f16_b2_t0":       ("f16", 2, 4, 12, 37, 9, 2, [0, 1, 2, 3, 4]),
    "f32_b4_wrapped":  ("f32", 4, 4, 20, 37, 7, 1, [18, 19, 0, 1]),
    "f16_b4_wrapped":  ("f16", 4, 3, 20, 64, 6, 1, [18, 19, 0, 1]),
    "f32_b2_stride":   ("f32", 2, 4, 24, 4096, 20, 3, list(range(5, 21))),
    "f16_b2_stride":   ("f16", 2, 4, 40, 4095, 18, 1, [(35 + i) % 40 for i in range(16)]),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(WINDOW_CASES))
def test_accumulate_window_bit_exact(built_lib, case):
    from musev_b200 import ops
    dt, B2, Cc, T, HW, Tw, src_t0, frames = WINDOW_CASES[case]
    assert src_t0 + len(frames) <= Tw
    g = torch.Generator(device=dev).manual_seed(zlib.crc32(case.encode()))
    es = torch.randn(B2, Cc, T, HW, generator=g, device=dev)
    win = torch.randn(B2, Cc, Tw, HW, generator=g, device=dev).to(torch.float16 if dt == "f16" else torch.float32)
    ref = window_ref(es, win, src_t0, frames)
    ops.accumulate_window(es.view(B2, Cc, T, HW, 1), win.view(B2, Cc, Tw, HW, 1), src_t0,
                          torch.tensor(frames, dtype=torch.int32, device=dev))
    torch.cuda.synchronize()
    assert torch.equal(es.view(torch.int32), ref.view(torch.int32))
    rest = [f for f in range(T) if f not in frames]
    assert torch.equal(es[:, :, rest].view(torch.int32), ref[:, :, rest].view(torch.int32))


# ------------------------------------------------------------------------------------------------ GPU: extents
def _bufs(n=2 * 4 * 4 * 8):
    """Non-empty buffers, so that a zero extent (not a NULL pointer) is what the call sees; every output starts at 7."""
    full = lambda v=7.0: torch.full((n,), v, device=dev)   # noqa: E731
    return dict(es=full(1.0), cnt=full(1.0)[:8], lat=full(1.0), out=full(), noise=full(1.0), o1=full(), o2=full(),
                win=full(1.0), frames=torch.arange(8, dtype=torch.int32, device=dev))


def _calls(b, B, Cc, T, HW, nframes=4, Tw=8, src_t0=0):
    """The four step entry points on the buffers b with the given extents; each returns the C return code."""
    from musev_b200 import _capi
    l = _capi.lib()
    st = torch.cuda.current_stream().cuda_stream
    p = {k: v.data_ptr() for k, v in b.items()}

    def multistep():
        a = _capi.MvbMultistepArgs()
        a.eps_sum, a.counter, a.latents_in, a.latents_out = p["es"], p["cnt"], p["lat"], p["out"]
        a.m1, a.noise, a.m0_out = p["noise"], p["win"], p["o1"]
        a.is_f32, a.B, a.C, a.T, a.HW, a.cfg = 1, B, Cc, T, HW, 1
        a.guidance_scale, a.a_x, a.a_e, a.c_x, a.c0, a.c1, a.c_n = 2.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0
        return l.mvb_fuse_cfg_multistep(C.byref(a), st)

    return {
        "ddim": lambda: l.mvb_fuse_cfg_ddim(p["es"], p["cnt"], p["lat"], p["out"], 1, B, Cc, T, HW, 1, 2.0, 0.5, 0.6, 0, 0.0,
                                            0, 0.1, p["noise"], p["o1"], p["o2"], st),
        "affine": lambda: l.mvb_fuse_cfg_affine(p["es"], p["cnt"], p["lat"], p["out"], 1, B, Cc, T, HW, 1, 2.0, 1.0, 1.0,
                                                1.0, p["noise"], 1.0, 1.0, p["o1"], p["o2"], st),
        "multistep": multistep,
        "window": lambda: l.mvb_accumulate_window(p["o1"], B, Cc, T, HW, p["win"], 1, Tw, src_t0, p["frames"], nframes, st),
    }


@pytest.mark.gpu
def test_empty_extents_launch_nothing(built_lib):
    """B, C, T, HW (or nframes) = 0: MVB_OK, no launch, every buffer keeps its bits."""
    from musev_b200 import _capi
    b = _bufs()
    before = {k: v.clone() for k, v in b.items()}
    full = dict(B=1, Cc=4, T=4, HW=8)
    torch.cuda.synchronize()
    n0 = _capi.launch_count()
    for zero in ("B", "Cc", "T", "HW", "nframes"):
        ext = dict(full, **{zero: 0}) if zero != "nframes" else dict(full, nframes=0)
        for name, call in _calls(b, **ext).items():
            if zero == "nframes" and name != "window":
                continue
            rc = call()
            assert rc == 0, (name, zero, _capi.lib().mvb_last_error().decode())
    torch.cuda.synchronize()
    assert _capi.launch_count() == n0
    for k, v in b.items():
        assert torch.equal(v, before[k]), k
    # the same calls with every extent set do launch (the buffers are large enough for them)
    for name, call in _calls(b, **full).items():
        assert call() == 0, name
    torch.cuda.synchronize()
    assert _capi.launch_count() == n0 + 4


@pytest.mark.gpu
def test_negative_extents_refused_before_launch(built_lib):
    from musev_b200 import _capi
    l = _capi.lib()
    b = _bufs()
    full = dict(B=1, Cc=4, T=4, HW=8)
    torch.cuda.synchronize()
    n0 = _capi.launch_count()
    for neg in ("B", "Cc", "T", "HW"):
        for name, call in _calls(b, **dict(full, **{neg: -1})).items():
            assert call() != 0, (name, neg)
            assert "negative extent" in l.mvb_last_error().decode(), (name, neg)
    for kw, msg in ((dict(nframes=-1), "negative extent"), (dict(Tw=-1), "negative extent"),
                    (dict(src_t0=-1), "src_t0"), (dict(src_t0=5, nframes=4, Tw=8), "src_t0"),
                    (dict(src_t0=0, nframes=9, Tw=8), "src_t0")):
        assert _calls(b, **full, **kw)["window"]() != 0, kw
        assert msg in l.mvb_last_error().decode(), kw
    torch.cuda.synchronize()
    assert _capi.launch_count() == n0
