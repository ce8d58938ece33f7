"""The small-channel 3x3 conv (`mvb_op_small_conv`, cond_embed.cu) at every one of its 24 instantiations (input NCHW
image / NHWC 16 / NHWC 32 channels x stride 1 / 2 x cout 16 / 32 / 64 / 128), against one float64 reference of the
operation the header documents:
    out[n, oy, ox, o] = act(sum_{ky, kx, c} x[n, s oy + ky - 1, s ox + kx - 1, c] W[o, (3 ky + kx) cin + c] + bias[o])
with zero padding 1 on every side, stride s, act none or SiLU. The reference is computed on the device from the fp16
inputs upcast to float64; an fp32 NCHW image is first rounded to fp16, as the kernel does when it builds its halo.

Every element is held to its own bound, never one relative to the tensor's maximum:
    |out - ref| <= ulp16(ref) / 2 + C_ACC slope sum |x| |w| + 2^-23 slope (|acc| + |bias|) (+ 1e-6 |pre-activation| with SiLU)
where slope is 1.1 (the largest slope of SiLU) with SiLU and 1 without, and the last term covers `__expf`. The bound
discriminates: on small host shapes the test computes named wrong answers in float64 (weight columns read
channel-major, dy and dx swapped, stride-2 padding (0, 1, 0, 1), the next frame's top row as the bottom padding, the last
k16 step left out, bias added after SiLU, two 8-channel halves of an output block swapped), rounds them to fp16 as the
kernel would and asserts that each breaks the bound (`test_small_conv_bounds_catch_wrong_answers`, no GPU).

The matrix runs each instantiation with SiLU and bias on and off, NCHW images of 1, 2 and 3 channels in fp16 and fp32,
images smaller than one 8 x 16 output tile, ragged last tiles on both axes, one tall-narrow and one wide-short image,
and one persistent case with at least 3 x (SM count) x 8 output tiles. Eight 256-thread CTAs per SM is the most
`__launch_bounds__(256, 1)` allows, so at any occupancy every CTA runs at least three tiles and the NHWC kernels reuse
both halo buffers. The cout-128 kernels also run the PoseGuider's padded layout (96 real channels, zero weight rows and
zero bias), whose pad channels must be exactly 0, and the PoseGuider's own (cin, cout, stride) layers run at 40 x 72.
Repeating a call gives the same bits, and frame i of an NF-frame call equals a 1-frame call on frame i. A second case
runs every instantiation on cuda:0 and then cuda:1 in a fresh process (skipped with fewer than 2 GPUs): the
shared-memory opt-in belongs to each device, and 15 of the 24 kernels need more than 48 KB of it.

With MVB_PARITY_LOG=<file> set, the worst ratio |out - ref| / bound of every case is appended to <file>, together
with the smallest C_ACC the case would pass with. Measured on an H100 80GB HBM3 at 700 W, worst ratio per group: NCHW
0.998 (persistent 0.995), NHWC 16 channels 0.995 (persistent 0.994), NHWC 32 channels 0.993 (persistent 0.993),
PoseGuider layers 0.993. Near 1 because a correctly rounded fp16 result may sit half an ulp away. The largest C_ACC
any case needed was 1.1e-7 (NHWC 32 channels, stride 2, cout 32), an accumulation error of at most 1.1e-7 sum |x| |w|
over K <= 288; C_ACC = 1e-6 keeps 9x above that. The two-device case has not been run yet: it needs two GPUs.
"""
import json
import math
import os
import subprocess
import sys
import zlib
from dataclasses import dataclass

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C_ACC = 1e-6
SILU_SLOPE = 1.1
SILU_REL = 1e-6
EPS_EPI = 2.0 ** -23
HOST_SMS = 132
TH, TW = 8, 16               # output tile of one CTA iteration
CTAS_PER_SM = 8              # the most __launch_bounds__(256, 1) allows

# (input kind, stride, cout): kind 0 is the NCHW image path, 16 / 32 the NHWC channel counts
INSTANTIATIONS = [(k, s, co) for k in (0, 16, 32) for s in (1, 2) for co in (16, 32, 64, 128)]


def inst_id(kind, s, cout):
    return f"{'nchw' if kind == 0 else f'nhwc{kind}'}_s{s}_co{cout}"


def ceil_div(a, b):
    return -(-a // b)


def tiles(H, W, NF, s):
    Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
    return ceil_div(Ho, TH) * ceil_div(Wo, TW) * NF


# ------------------------------------------------------------------------------------------------ cases
@dataclass(frozen=True)
class Case:
    id: str
    kind: int         # 0: NCHW image, 16 / 32: NHWC channels
    s: int
    cout: int         # kernel cout (16 / 32 / 64 / 128)
    NF: int
    H: int
    W: int
    cin: int = 0      # NCHW image channels (1..3)
    f32: bool = False # NCHW: fp32 image
    act: bool = True
    bias: bool = True
    real: int = 0     # real output channels (0: all); the rest have zero weight rows and zero bias
    persist: bool = False

    @property
    def ch(self):
        return self.cin if self.kind == 0 else self.kind


def matrix_cases(sms):
    cs = []
    # NCHW (cin, fp32 image) per case slot: every instantiation sees cin 1, 2, 3 in fp16 and fp32
    img = [(3, True), (1, False), (2, True), (3, False), (1, True), (2, False), (3, True), (1, False)]
    for kind, s, co in INSTANTIATIONS:
        iid = inst_id(kind, s, co)
        # ragged last tiles on both axes, at least 3 tiles per CTA at 8 CTAs per SM
        H, W = (324, 328) if s == 1 else (648, 656)
        NF = ceil_div(3 * sms * CTAS_PER_SM, tiles(H, W, 1, s))
        small = ((1, 1), (3, 5)) if s == 1 else ((2, 2), (6, 10))
        shapes = [("persist", NF, H, W, True, True),
                  ("noact_nobias", 2, 24 * s, 40 * s, False, False),
                  ("act_nobias", 2, 20 * s, 36 * s, True, False),
                  ("noact_bias", 3, 17 * s, 33 * s, False, True),
                  (f"tiny{small[0][0]}x{small[0][1]}", 5, *small[0], True, True),
                  (f"tiny{small[1][0]}x{small[1][1]}", 3, *small[1], False, True),
                  ("tall", 2, 70 * s, 18 * s, True, True),
                  ("wide", 2, 10 * s, 150 * s, True, True)]
        if s == 1:   # odd sizes are stride-1 only: ragged against both the tile and the pixel pairs
            shapes[1:4] = [("noact_nobias", 2, 23, 41, False, False), ("act_nobias", 2, 21, 35, True, False),
                           ("noact_bias", 3, 17, 33, False, True)]
        for (tag, nf, h, w, act, bias), (cin, f32) in zip(shapes, img):
            cs.append(Case(f"{iid}_{tag}", kind, s, co, nf, h, w, cin=cin if kind == 0 else 0,
                           f32=f32 if kind == 0 else False, act=act, bias=bias, persist=tag == "persist"))
        if co == 128:   # the PoseGuider's 96-channel layers run on the 128-channel kernel
            cs.append(Case(f"{iid}_pad96", kind, s, co, 3, 16 * s, 40 * s, cin=3 if kind == 0 else 0, real=96))
            cs.append(Case(f"{iid}_pad96_noact", kind, s, co, 2, 16 * s, 24 * s, cin=3 if kind == 0 else 0, act=False,
                           real=96))
    return cs


def pose_guider_cases():
    """The (cin, cout, stride) of every PoseGuider layer that runs on this kernel, at 3 frames of 40 x 72."""
    sys.path.insert(0, ROOT)
    from musev_b200.schema import PoseGuiderConfig, pose_guider_layers
    seen = []
    for cfg in (PoseGuiderConfig(64, 3, (16, 32, 64, 128)), PoseGuiderConfig(320, 3, (16, 32, 96, 256))):
        for _, cin, cout, s in pose_guider_layers(cfg):
            if cin in (3, 16, 32) and (cin, cout, s) not in seen:
                seen.append((cin, cout, s))
    cs = []
    for cin, cout, s in seen:
        co = next(c for c in (16, 32, 64, 128) if c >= cout)
        cs.append(Case(f"pg_{cin}_{cout}_s{s}", 0 if cin == 3 else cin, s, co, 3, 40, 72, cin=3 if cin == 3 else 0,
                       f32=cin == 3, real=cout if cout != co else 0))
    return cs


def all_cases(sms=HOST_SMS):
    return matrix_cases(sms) + pose_guider_cases()


CASES = all_cases()
CASE_IDS = [c.id for c in CASES]
assert len(set(CASE_IDS)) == len(CASE_IDS)


# ------------------------------------------------------------------------------------------------ inputs
def make_inputs(case, device):
    """(x, packed weight, bias or None) of a case on seeded data."""
    g = torch.Generator(device=device).manual_seed(zlib.crc32(case.id.encode()))

    def rnd(*shape, scale=1.0):
        return torch.randn(*shape, generator=g, device=device) * scale

    cin, co = case.ch, case.cout
    if case.kind == 0:
        x = rnd(case.NF, cin, case.H, case.W)
        x = x if case.f32 else x.half()
        wp = torch.zeros(co, 32, dtype=torch.float16, device=device)
    else:
        x = rnd(case.NF, case.H, case.W, cin).half()
        wp = torch.zeros(co, 9 * cin, dtype=torch.float16, device=device)
    real = case.real or co
    wp[:real, :9 * cin] = rnd(real, 9 * cin, scale=(9 * cin) ** -0.5).half()
    b = None
    if case.bias:
        b = torch.zeros(co, device=device)
        b[:real] = rnd(real, scale=0.5)
    return x, wp, b


# ------------------------------------------------------------------------------------------------ float64 reference
def _ulp16(r):
    """Spacing of fp16 at |r| (float64 tensor): 2^(e - 11) for |r| in [2^(e-1), 2^e), 2^-24 in the subnormal range."""
    _, e = torch.frexp(r.abs())
    return torch.where(r.abs() < 2.0 ** -14, torch.full_like(r, 2.0 ** -24), torch.ldexp(torch.ones_like(r), e - 11))


def conv_ref(x, wp, bias, stride, act, nchw, wrong=()):
    """float64 reference of one ops.small_conv call and the per-element bound: (ref, bound), [NF, Ho, Wo, cout].
    `wrong` names the deliberate errors of the host check."""
    xd = x.half().double().permute(0, 2, 3, 1) if nchw else x.double()   # an fp32 image is read as fp16
    NF, H, W, cin = xd.shape
    cout = wp.shape[0]
    wd = wp.double()
    if "last k16 left out" in wrong:
        wd = wd.clone()
        wd[:, -16:] = 0
    w = wd[:, :9 * cin]
    w9 = w.view(cout, cin, 9).transpose(1, 2) if "weight columns read channel-major" in wrong else w.view(cout, 9, cin)
    if "dy and dx swapped" in wrong:
        w9 = w9.reshape(cout, 3, 3, cin).transpose(1, 2).reshape(cout, 9, cin)
    s = stride
    Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
    xp = F.pad(xd, (0, 0, 1, 2, 1, 2))      # pad 1 on top / left; the extra bottom / right one serves the pad-mode check
    if "next frame's top row as the bottom padding" in wrong:
        xp[:-1, H + 1, 1:W + 1] = xd[1:, 0]
    off = 1 if "stride-2 padding (0, 1, 0, 1)" in wrong else 0
    acc = torch.zeros(NF, Ho, Wo, cout, dtype=torch.float64, device=xd.device)
    sab = torch.zeros_like(acc)
    for ky in range(3):
        for kx in range(3):
            v = xp[:, off + ky:off + ky + s * (Ho - 1) + 1:s, off + kx:off + kx + s * (Wo - 1) + 1:s]
            wt = w9[:, 3 * ky + kx]
            acc += v @ wt.t()
            sab += v.abs() @ wt.abs().t()
    b = bias.double() if bias is not None else torch.zeros(cout, dtype=torch.float64, device=xd.device)
    pre = acc + b
    if act:
        ref = acc * torch.sigmoid(acc) + b if "bias added after SiLU" in wrong else pre * torch.sigmoid(pre)
    else:
        ref = pre
    if "two 8-channel halves of an output block swapped" in wrong:
        ref = ref[..., torch.arange(cout, device=ref.device).view(-1, 2, 8).flip(1).reshape(-1)]
    slope = SILU_SLOPE if act else 1.0
    acc_term = slope * sab
    bound = 0.5 * _ulp16(ref) + EPS_EPI * slope * (acc.abs() + b.abs()) + (SILU_REL * pre.abs() if act else 0.0)
    return ref, bound, acc_term


def _ratio(got, ref, bound, acc_term):
    """(max |got - ref| / (bound + C_ACC acc_term), its flat index, the smallest C_ACC that passes); got is rounded to
    fp16 as the kernel returns it."""
    got = got.half().double()
    if not torch.isfinite(got).all():
        return math.inf, -1, math.inf
    d = (got - ref).abs()
    r = (d / (bound + C_ACC * acc_term)).flatten()
    i = int(r.argmax())
    need = ((d - bound).clamp_min(0) / acc_term.clamp_min(1e-30)).max().item()
    return r[i].item(), i, need


def _record(name, err, bound, where="", need=None):
    path = os.environ.get("MVB_PARITY_LOG")
    if path:
        try:
            with open(path, "a") as fh:
                row = {"test": name, "value": err, "bound": bound}
                if need is not None:
                    row["c_acc_needed"] = need
                fh.write(json.dumps(row) + "\n")
        except OSError:
            pass
    assert err <= bound, (name, where, err, bound)


# ------------------------------------------------------------------------------------------------ host checks
def test_matrix_covers_every_instantiation():
    """24 instantiations, each with a persistent case of at least 3 x SMs x 8 tiles (so >= 3 tiles per CTA), ragged last
    tiles on both axes, SiLU and bias on and off, an image smaller than one tile; NCHW sees cin 1..3 in fp16 and fp32."""
    by = {}
    for c in matrix_cases(HOST_SMS):
        by.setdefault((c.kind, c.s, c.cout), []).append(c)
    assert sorted(by) == sorted(INSTANTIATIONS) and len(by) == 24
    for key, cs in by.items():
        p = [c for c in cs if c.persist]
        assert len(p) == 1 and tiles(p[0].H, p[0].W, p[0].NF, p[0].s) >= 3 * HOST_SMS * CTAS_PER_SM, key
        Ho, Wo = p[0].H // p[0].s, p[0].W // p[0].s
        assert Ho % TH and Wo % TW, key
        assert {(c.act, c.bias) for c in cs} >= {(True, True), (True, False), (False, True), (False, False)}, key
        assert any(c.H // c.s < TH and c.W // c.s < TW for c in cs), key
        assert any(c.H // c.s > 3 * c.W // c.s for c in cs) and any(c.W // c.s > 10 * c.H // c.s for c in cs), key
        if key[0] == 0:
            assert {(c.cin, c.f32) for c in cs} == {(ci, f) for ci in (1, 2, 3) for f in (False, True)}, key
        if key[2] == 128:
            assert any(c.real == 96 for c in cs), key


# host shapes and the wrong answers that apply to each
HOST_GROUPS = {
    "nhwc16_s1": (Case("h_nhwc16_s1", 16, 1, 32, 2, 9, 18),
                  ("weight columns read channel-major", "dy and dx swapped", "next frame's top row as the bottom padding",
                   "last k16 left out", "bias added after SiLU", "two 8-channel halves of an output block swapped")),
    "nhwc32_s2": (Case("h_nhwc32_s2", 32, 2, 16, 2, 10, 18),
                  ("weight columns read channel-major", "dy and dx swapped", "stride-2 padding (0, 1, 0, 1)",
                   "last k16 left out", "bias added after SiLU", "two 8-channel halves of an output block swapped")),
    "nchw3_s1": (Case("h_nchw3_s1", 0, 1, 16, 2, 9, 18, cin=3, f32=True),
                 ("weight columns read channel-major", "dy and dx swapped", "next frame's top row as the bottom padding",
                  "last k16 left out", "bias added after SiLU", "two 8-channel halves of an output block swapped")),
    "nchw2_s2": (Case("h_nchw2_s2", 0, 2, 32, 2, 10, 18, cin=2),
                 ("weight columns read channel-major", "dy and dx swapped", "stride-2 padding (0, 1, 0, 1)",
                  "last k16 left out", "bias added after SiLU", "two 8-channel halves of an output block swapped")),
}


@pytest.mark.parametrize("group", list(HOST_GROUPS))
def test_small_conv_bounds_catch_wrong_answers(group):
    """Host only: on each group's small shape the reference passes its own bound and every named wrong answer,
    rounded to fp16 as the kernel would return it, breaks it."""
    case, wrongs = HOST_GROUPS[group]
    x, wp, b = make_inputs(case, "cpu")
    ref, bound, acc_term = conv_ref(x, wp, b, case.s, case.act, case.kind == 0)
    assert _ratio(ref, ref, bound, acc_term)[0] <= 1.0
    for w in wrongs:
        y, _, _ = conv_ref(x, wp, b, case.s, case.act, case.kind == 0, wrong=(w,))
        r = _ratio(y, ref, bound, acc_term)[0]
        assert r > 1.0, f"{group}: the wrong answer '{w}' stays inside the bound (worst ratio {r:.3g})"


# ------------------------------------------------------------------------------------------------ GPU
def _run(ops, x, wp, b, case):
    return ops.small_conv(x, wp, b, case.s, case.act, nchw=case.kind == 0)


def _run_case(ops, case, dev):
    x, wp, b = make_inputs(case, dev)
    out = _run(ops, x, wp, b, case)
    ref, bound, acc_term = conv_ref(x, wp, b, case.s, case.act, case.kind == 0)
    real = case.real or case.cout
    r, i, need = _ratio(out[..., :real], ref[..., :real], bound[..., :real], acc_term[..., :real])
    res = {"ratio": r, "need": need, "where": i, "shape_ok": list(out.shape) == list(ref.shape),
           "pad_zero": bool((out[..., real:] == 0).all()) if case.real else True}
    if case.persist:
        again = _run(ops, x, wp, b, case)
        res["repeat_equal"] = bool(torch.equal(out.view(torch.int16), again.view(torch.int16)))
        res["frames_equal"] = all(torch.equal(out[f].view(torch.int16), _run(ops, x[f:f + 1], wp, b, case)[0].view(torch.int16))
                                  for f in range(case.NF))
    return res


@pytest.fixture(scope="module")
def results(built_lib):
    from musev_b200 import ops
    from musev_b200._capi import MvbError
    dev = torch.device("cuda", 0)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    out = {"sms": sms, "cases": {}}
    for case in all_cases(sms):
        try:
            out["cases"][case.id] = _run_case(ops, case, dev)
        except MvbError as e:
            out["cases"][case.id] = {"error": str(e)}
        torch.cuda.empty_cache()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_small_conv_edges(results, case):
    rr = results["cases"][case.id]
    assert "error" not in rr, rr
    assert rr["shape_ok"] and rr["pad_zero"], rr
    if case.persist:
        sms = results["sms"]
        c = next(c for c in all_cases(sms) if c.id == case.id)
        assert tiles(c.H, c.W, c.NF, c.s) >= 3 * sms * CTAS_PER_SM
        assert rr["repeat_equal"], "a repeated call changed bits"
        assert rr["frames_equal"], "an NF-frame call differs from 1-frame calls"
    _record(f"small_conv_{case.id}_vs_fp64", rr["ratio"], 1.0, rr["where"], rr["need"])


@pytest.mark.gpu
def test_small_conv_refuses_before_launch(built_lib):
    """A bad cin or cout, stride 3, odd H or W at stride 2, an empty image, fp32 NHWC input or a null pointer is refused
    with MvbError before anything is launched."""
    from musev_b200 import _capi
    from musev_b200._capi import MvbError
    dev = "cuda"
    x = torch.zeros(2, 8, 8, 32, dtype=torch.float16, device=dev)
    w = torch.zeros(128, 9 * 32, dtype=torch.float16, device=dev)
    b = torch.zeros(128, device=dev)
    out = torch.zeros(2 * 8 * 8 * 128, dtype=torch.float16, device=dev)
    xp, wp, bp, op = x.data_ptr(), w.data_ptr(), b.data_ptr(), out.data_ptr()
    st = torch.cuda.current_stream().cuda_stream
    #        x,  f32, nchw, cin, H, W, NF, s, w,  b,  cout, act, out
    ok = dict(x=xp, f32=0, nchw=0, cin=16, H=8, W=8, NF=2, s=1, w=wp, b=bp, cout=16, act=1, out=op)
    bad = {
        "nhwc cin 8": dict(cin=8), "nhwc cin 24": dict(cin=24), "nhwc cin 3": dict(cin=3),
        "nchw cin 0": dict(nchw=1, cin=0), "nchw cin 4": dict(nchw=1, cin=4), "nchw cin 16": dict(nchw=1, cin=16),
        "cout 48": dict(cout=48), "cout 256": dict(cout=256), "cout 0": dict(cout=0),
        "stride 3": dict(s=3), "stride 0": dict(s=0), "odd H stride 2": dict(s=2, H=7), "odd W stride 2": dict(s=2, W=7),
        "H 0": dict(H=0), "W 0": dict(W=0), "NF 0": dict(NF=0),
        "fp32 NHWC": dict(f32=1), "null x": dict(x=None), "null weight": dict(w=None), "null out": dict(out=None),
    }
    l = _capi.lib()
    torch.cuda.synchronize()
    n0 = _capi.launch_count()
    for what, kw in bad.items():
        a = dict(ok, **kw)
        with pytest.raises(MvbError, match="small_conv"):
            _capi.check(l.mvb_op_small_conv(a["x"], a["f32"], a["nchw"], a["cin"], a["H"], a["W"], a["NF"], a["s"], a["w"],
                                            a["b"], a["cout"], a["act"], a["out"], st))
            pytest.fail(f"{what}: not refused")
    torch.cuda.synchronize()
    assert _capi.launch_count() == n0


def _multi_device():
    """Every instantiation on cuda:0, then on cuda:1, in this (fresh) process; prints per instantiation whether each
    device ran it and whether the two outputs have the same bits."""
    sys.path.insert(0, ROOT)
    from musev_b200 import ops
    from musev_b200._capi import MvbError
    rows = {}
    for kind, s, co in INSTANTIATIONS:
        case = Case("multi_" + inst_id(kind, s, co), kind, s, co, 2, 24 * s, 40 * s, cin=3 if kind == 0 else 0)
        host = make_inputs(case, "cpu")
        outs, errs = [], []
        for d in (0, 1):
            dev = torch.device("cuda", d)
            with torch.cuda.device(dev):
                x, wp, b = (t.to(dev) for t in host)
                try:
                    outs.append(_run(ops, x, wp, b, case).cpu())
                    errs.append(None)
                except MvbError as e:
                    outs.append(None)
                    errs.append(str(e))
                torch.cuda.synchronize()
        rows[inst_id(kind, s, co)] = {"errors": errs, "equal": None not in outs and
                                      torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16))}
    print(json.dumps(rows))


@pytest.mark.gpu
def test_small_conv_runs_on_a_second_device(built_lib):
    """The shared-memory opt-in is set per device: a process that ran a kernel on cuda:0 runs it on cuda:1 too, with the
    same bits."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "multi"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    rows = json.loads(r.stdout.strip().splitlines()[-1])
    assert len(rows) == 24
    bad = {k: v for k, v in rows.items() if v["errors"] != [None, None] or not v["equal"]}
    assert not bad, bad


if __name__ == "__main__":
    if sys.argv[1:] == ["multi"]:
        _multi_device()
