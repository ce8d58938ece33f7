"""Multi-ControlNet on the engine: several ControlNets per window-step with their residual maps summed on the device
(`mvb_controlnet_args.accumulate`, `musev_b200.controlnet.MultiControlNetModel`, the multi-net `make_controlnet_fn`).

Bounds: the single-net ones (2e-2 of max|ref| against the fp32 oracle, 3e-2 against the reference fixture) tightened to about
twice the measured distances (1.5e-3 .. 1.8e-3 narrow, 1.4e-3 at SD-1.5 width, H100); the 2-step loop keeps the loop
bound 5e-2 (measured 2.5e-2 / 2.0e-2). Every measured distance is recorded with the UNet tests' `_record`."""
import os

import pytest
import torch

from conftest import GOLDEN
from test_gpu_unet import _record

pytestmark = pytest.mark.gpu
dev = "cuda"
NARROW = (64, 128, 128, 128)
FULL = (320, 640, 1280, 1280)


def _nets(seeds, boc=NARROW, dtype=torch.float32):
    """Engine ControlNets and fp32 oracles on the same fp16 weights."""
    from musev_b200.controlnet import ControlNetModel
    from musev_b200.schema import ControlNetConfig
    from musev_b200.synth import make_state_dict
    from oracle.controlnet_oracle import ControlNetOracle
    cfg = ControlNetConfig(block_out_channels=tuple(boc))
    nets, oracles = [], []
    for s in seeds:
        sd16 = {k: v.half() for k, v in make_state_dict(cfg, seed=s).items()}
        n = ControlNetModel(cfg, device=dev, dtype=dtype)
        n.load_state_dict(sd16)
        nets.append(n)
        oracles.append(ControlNetOracle(cfg, {k: v.float() for k, v in sd16.items()}, device=dev))
    return cfg, nets, oracles


def _images(n, h, w, seed):
    from musev_b200.schema import ControlNetConfig
    from musev_b200.synth import make_controlnet_inputs
    return make_controlnet_inputs(ControlNetConfig(block_out_channels=NARROW), frames=n, h=h, w=w, seed=seed)["controlnet_cond"]


def _inputs(cfg, frames, h, w, seed=4321):
    from musev_b200.synth import make_controlnet_inputs
    inp = make_controlnet_inputs(cfg, frames=frames, h=h, w=w, seed=seed)
    return inp["sample"].to(dev), inp["encoder_hidden_states"].to(dev)


# ---------------------------------------------------------------------------------------- 1. accumulate is the torch sum
@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("n_nets", [2, 3])
@pytest.mark.parametrize("guess_mode", [False, True])
def test_accumulate_is_the_reference_sum_bit_for_bit(built_lib, dtype, n_nets, guess_mode):
    """`samples_prev + samples_curr` in net order (multicontrolnet.py:64-70) in the output dtype, against accumulate = 0 calls
    summed by torch. 16x16 latents give maps with 256 .. 4 pixels: both the 16-byte and the scalar kernel run."""
    from musev_b200.controlnet import MultiControlNetModel
    cfg, nets, _ = _nets([3, 13, 23][:n_nets], dtype=dtype)
    x, enc = _inputs(cfg, 3, 16, 16)
    lats = [n.controlnet_cond_embedding(_images(3, 16, 16, 4401 + k).to(dev)) for k, n in enumerate(nets)]
    scales = [0.7, 1.3, 0.45][:n_nets]
    sep = [n(x, 601, enc, controlnet_cond_latents=l, conditioning_scale=s, guess_mode=guess_mode, return_dict=False)
           for n, l, s in zip(nets, lats, scales)]
    want = [m.clone() for m in list(sep[0][0]) + [sep[0][1]]]
    for d, m in sep[1:]:
        want = [a + b for a, b in zip(want, list(d) + [m])]
    down, mid = MultiControlNetModel(nets)(x, 601, enc, None, scales, guess_mode=guess_mode, controlnet_cond_latents=lats)
    assert all(a.dtype == dtype for a in list(down) + [mid])
    for k, (a, b) in enumerate(zip(list(down) + [mid], want)):
        assert torch.equal(a, b), f"map {k}: max diff {(a.float() - b.float()).abs().max().item()}"


def test_accumulate_rejects_referencenet_and_null_outputs(built_lib):
    from musev_b200 import _capi
    from musev_b200._capi import MvbControlnetArgs, MvbError
    from musev_b200.referencenet import ReferenceNet2D
    from musev_b200.schema import ReferenceNetConfig
    from musev_b200.synth import make_state_dict
    cfg, nets, _ = _nets([3])
    x, enc = _inputs(cfg, 2, 8, 8)
    lat = torch.zeros(2, NARROW[0], 8, 8, device=dev)
    down, mid = nets[0](x, 1, enc, controlnet_cond_latents=lat, return_dict=False)

    def args(outs):
        a = MvbControlnetArgs()
        a.sample, a.NF, a.H, a.W, a.sample_is_f32 = x.data_ptr(), 2, 8, 8, 1
        a.encoder_hidden_states, a.ehs_is_f32, a.n_text = enc.data_ptr(), 1, enc.shape[1]
        a.cond_latents, a.cond_is_f32 = lat.data_ptr(), 1
        a.n_out = len(outs)
        for k, o in enumerate(outs):
            a.scales[k] = 1.0
            a.outs[k] = o.data_ptr() if o is not None else None
        a.out_is_f32, a.accumulate = 1, 1
        return a

    outs = list(down) + [mid]
    torch.cuda.synchronize()
    n0 = _capi.launch_count()
    with pytest.raises(MvbError, match="NULL"):
        nets[0]._launch(args(outs[:5] + [None] + outs[6:]))
    torch.cuda.synchronize()
    assert _capi.launch_count() == n0
    rcfg = ReferenceNetConfig(block_out_channels=NARROW)
    ref = ReferenceNet2D(rcfg, device=dev, dtype=torch.float32)
    ref.load_state_dict({k: v.half() for k, v in make_state_dict(rcfg, seed=5).items()})
    torch.cuda.synchronize()
    n1 = _capi.launch_count()
    with pytest.raises(MvbError, match="ReferenceNet"):
        ref._launch(args(outs))
    torch.cuda.synchronize()
    assert _capi.launch_count() == n1
    with pytest.raises(ValueError, match="accumulate_into"):
        nets[0](x, 1, enc, controlnet_cond_latents=lat, return_dict=False, accumulate_into=(down[:-1], mid))


# ---------------------------------------------------------------------------------------- 2. one net is today's ControlNet
def test_one_net_through_the_multi_path_is_the_single_net(built_lib):
    from musev_b200.controlnet import MultiControlNetModel
    from musev_b200.pipeline import make_controlnet_fn
    cfg, nets, _ = _nets([3])
    net = nets[0]
    x, enc = _inputs(cfg, 3, 16, 16)
    lat = net.controlnet_cond_embedding(_images(3, 16, 16, 4401).to(dev))
    d1, m1 = net(x, 601, enc, controlnet_cond_latents=lat, conditioning_scale=0.8, return_dict=False)
    d2, m2 = MultiControlNetModel([net])(x, 601, enc, None, [0.8], controlnet_cond_latents=[lat])
    assert torch.equal(m1, m2) and all(torch.equal(a, b) for a, b in zip(d1, d2))
    g = torch.Generator().manual_seed(5)
    n_vc, T = 1, 6
    cn_lat = (torch.randn(2, NARROW[0], n_vc + T, 8, 8, generator=g) * 0.3).to(dev)
    prompt = torch.randn(2, 77, 768, generator=g).to(dev)
    xin = torch.randn(2, 4, n_vc + 4, 8, 8, generator=g).to(dev)
    for keep in (None, [0.5]):
        single = make_controlnet_fn(net, cn_lat, prompt, n_vc, controlnet_conditioning_scale=0.9, controlnet_keep=keep)
        multi = make_controlnet_fn([net], [cn_lat], prompt, n_vc, controlnet_conditioning_scale=0.9,
                                   controlnet_keep=None if keep is None else [[0.5]])
        (ds, ms), (dm, mm) = single([1, 2, 3, 4], xin, 500, 0), multi([1, 2, 3, 4], xin, 500, 0)
        assert torch.equal(ms, mm) and all(torch.equal(a, b) for a, b in zip(ds, dm))


# ---------------------------------------------------------------------------------------- 3. oracle and reference fixture
@pytest.mark.parametrize("tag", ["two", "three_guess"])
def test_multi_vs_oracle_and_reference_fixture(built_lib, tag):
    from musev_b200.controlnet import MultiControlNetModel
    from oracle.multicontrolnet_oracle import multi_controlnet_forward
    g = torch.load(os.path.join(GOLDEN, "multicontrolnet_narrow.pt"))[tag]
    m = g["meta"]
    cfg, nets, oracles = _nets(m["weight_seeds"], tuple(m["block_out_channels"]))
    x, enc = _inputs(cfg, m["frames"], m["h"], m["w"], seed=m["input_seed"])
    images = [_images(m["frames"], m["h"], m["w"], s).to(dev) for s in m["image_seeds"]]
    kw = dict(guess_mode=m["guess_mode"])
    # the diffusers call: a list of images, every net embeds its own
    down, mid = MultiControlNetModel(nets)(x, m["timestep"], enc, images, m["scales"], **kw)
    rdown, rmid = multi_controlnet_forward(oracles, x, m["timestep"], enc, images, m["scales"], **kw)
    worst_o, worst_g = 0.0, 0.0
    for k, (a, b) in enumerate(zip(list(down) + [mid], list(rdown) + [rmid])):
        rel = (a.float() - b.float()).abs().max().item() / max(1.0, b.abs().max().item())
        worst_o = max(worst_o, rel)
        flat = a.float().reshape(-1).cpu()
        idx = torch.randint(0, flat.numel(), (m["n_samples"],), generator=torch.Generator().manual_seed(m["sample_seed_base"] + k))
        ref = g["samples"][k]
        worst_g = max(worst_g, (flat[idx] - ref).abs().max().item() / max(1.0, ref.abs().max().item()))
    _record(f"multicontrolnet_{tag}_vs_oracle_rel", worst_o)
    _record(f"multicontrolnet_{tag}_vs_reference_fixture_rel", worst_g)
    assert worst_o < 4e-3, worst_o
    assert worst_g < 4e-3, worst_g


# ---------------------------------------------------------------------------------------- 4. / 5. the denoise loop
def _loop_setup():
    from musev_b200.schema import preset_config
    from musev_b200.synth import make_inputs, make_state_dict
    from musev_b200.unet import UNet3DConditionModel
    from oracle.unet3d_oracle import UNet3DOracle
    g = torch.load(os.path.join(GOLDEN, "multicontrolnet_narrow.pt"))["loop"]
    m = g["meta"]
    cfg = preset_config(m["preset"], block_out_channels=tuple(m["block_out_channels"]))
    sd = {k: v.half() for k, v in make_state_dict(cfg, seed=m["weight_seed"]).items()}
    unet = UNet3DConditionModel(cfg, device=dev, dtype=torch.float32)
    unet.load_state_dict(sd)
    uo = UNet3DOracle(cfg, {k: v.float() for k, v in sd.items()}, device=dev)
    _, nets, oracles = _nets(m["cn_weight_seeds"], tuple(m["block_out_channels"]))
    T, h, w = m["T"], m["h"], m["w"]
    gen = torch.Generator().manual_seed(m["input_seed"])
    latents = torch.randn(1, 4, T, h, w, generator=gen)
    cond = torch.randn(1, 4, 1, h, w, generator=gen) * 0.5
    prompt = torch.randn(2, 77, cfg.cross_attention_dim, generator=gen)
    extra = make_inputs(cfg, batch=2, frames=1, h=h, w=w, seed=m["input_seed"])
    kw = {k: (extra[k].to(dev) if torch.is_tensor(extra[k]) else [t.to(dev) for t in extra[k]])
          for k in ("down_block_refer_embs", "mid_block_refer_emb", "vision_clip_emb") if k in extra}
    kw["ip_adapter_scale"] = 1.0
    # each net's condition embedding of every frame, computed once per call, duplicated for CFG
    cn_lat = []
    for k, n in enumerate(nets):
        e = n.controlnet_cond_embedding(_images(1 + T, h, w, m["image_seed"] + k).to(dev))
        cn_lat.append(torch.cat([e.permute(1, 0, 2, 3).unsqueeze(0)] * 2).contiguous())
    return g, m, unet, uo, nets, oracles, latents, cond, prompt, kw, cn_lat


def test_two_controlnets_in_the_denoise_loop(built_lib):
    from musev_b200.pipeline import ParallelDenoiser, make_controlnet_fn
    from musev_b200.scheduler import SD15_DDIM_CONFIG, DDIMScheduler
    from oracle.multicontrolnet_oracle import denoise_loop_multi
    from oracle.pipeline_oracle import SD15_DDIM, DDIMOracle, denoise_loop
    g, m, unet, uo, nets, oracles, latents, cond, prompt, kw, cn_lat = _loop_setup()
    loop = dict(context_frames=m["context_frames"], context_overlap=m["context_overlap"])
    den = ParallelDenoiser(unet, DDIMScheduler(**SD15_DDIM_CONFIG))
    fn = make_controlnet_fn(nets, cn_lat, prompt.to(dev), 1, controlnet_conditioning_scale=m["scales"])
    res = den(latents.to(dev), cond.to(dev), prompt.to(dev), num_inference_steps=m["steps"],
              guidance_scale=m["guidance_scale"], motion_speed=8, unet_kwargs=kw, controlnet_fn=fn, **loop)
    assert res.windows == m["contexts"]
    out = res.latents.cpu()

    def unet_oracle(s, t, e, **k):
        return uo(s, t, e, **k).cpu()
    common = (DDIMOracle(**SD15_DDIM), latents, cond, prompt, m["steps"], m["guidance_scale"])
    ref = denoise_loop_multi(unet_oracle, *common, oracles, cn_lat, m["scales"], motion_speed=8, unet_kwargs=kw, **loop)
    first_only = denoise_loop(unet_oracle, *common, motion_speed=8, unet_kwargs=kw, controlnet=oracles[0],
                              controlnet_latents=cn_lat[0], controlnet_conditioning_scale=m["scales"][0], **loop)
    err = (out - ref).abs().max().item()
    err_g = (out - g["latents"]).abs().max().item()
    _record("multicontrolnet_loop_vs_oracle", err)
    _record("multicontrolnet_loop_vs_reference_fixture", err_g)
    assert (ref - first_only).abs().max().item() > 10 * err, "the second ControlNet must matter in this test"
    assert err < 5e-2, err
    assert err_g < 5e-2, err_g


def test_a_net_switched_off_is_not_run(built_lib):
    """control_guidance_end = [1.0, 0.5] switches net 1 off after step 0. Skipping it gives the bits of running it with
    scale 0: its maps are then +-0 and adding them changes nothing. (Where a map is not finite the reference's 0 * map
    is NaN and the skipped net contributes nothing; the engine follows the guidance window, not the NaN.)"""
    from musev_b200.pipeline import ParallelDenoiser, controlnet_keep_schedule, make_controlnet_fn
    from musev_b200.scheduler import SD15_DDIM_CONFIG, DDIMScheduler
    g, m, unet, uo, nets, oracles, latents, cond, prompt, kw, cn_lat = _loop_setup()
    loop = dict(num_inference_steps=m["steps"], guidance_scale=m["guidance_scale"], motion_speed=8, unet_kwargs=kw,
                context_frames=m["context_frames"], context_overlap=m["context_overlap"])
    keep = controlnet_keep_schedule(m["steps"], 0.0, [1.0, 0.5], 2)
    assert keep == [[1.0, 1.0], [1.0, 0.0]]
    p = prompt.to(dev)
    calls = []
    n1_launch = nets[1]._launch

    def counting(a):
        calls.append(a.accumulate)
        return n1_launch(a)
    nets[1]._launch = counting
    skip = make_controlnet_fn(nets, cn_lat, p, 1, controlnet_conditioning_scale=m["scales"], controlnet_keep=keep)
    out = ParallelDenoiser(unet, DDIMScheduler(**SD15_DDIM_CONFIG))(latents.to(dev), cond.to(dev), p, controlnet_fn=skip,
                                                                     **loop).latents
    assert len(calls) == len(m["contexts"])            # step 0 only
    full = make_controlnet_fn(nets, cn_lat, p, 1, controlnet_conditioning_scale=m["scales"])
    zero = make_controlnet_fn(nets, cn_lat, p, 1, controlnet_conditioning_scale=[m["scales"][0], 0.0])

    def run_with_scale_zero(c, x, t, i, rows=None):
        return (full if i == 0 else zero)(c, x, t, i)
    ref = ParallelDenoiser(unet, DDIMScheduler(**SD15_DDIM_CONFIG))(latents.to(dev), cond.to(dev), p,
                                                                     controlnet_fn=run_with_scale_zero, **loop).latents
    assert len(calls) == 3 * len(m["contexts"])
    assert torch.equal(out, ref)


# ---------------------------------------------------------------------------------------- 6. SD-1.5 width
def test_two_full_width_controlnets_vs_oracle(built_lib):
    """Two SD-1.5 ControlNets on the config-4 window's 34 frames (2B x (1 + 16)) of 16x16 latents."""
    from musev_b200.controlnet import MultiControlNetModel
    from oracle.multicontrolnet_oracle import multi_controlnet_forward
    cfg, nets, oracles = _nets([31, 41], FULL)
    x, enc = _inputs(cfg, 34, 16, 16, seed=99)
    lats = [(torch.randn(34, FULL[0], 16, 16, generator=torch.Generator().manual_seed(500 + k)) * 0.3).to(dev)
            for k in range(2)]
    down, mid = MultiControlNetModel(nets)(x, 401, enc, None, [1.0, 0.6], controlnet_cond_latents=lats)
    rdown, rmid = multi_controlnet_forward(oracles, x, 401, enc, None, [1.0, 0.6], controlnet_cond_latents=lats)
    worst = max((a.float() - b.float()).abs().max().item() / max(1.0, b.abs().max().item())
                for a, b in zip(list(down) + [mid], list(rdown) + [rmid]))
    _record("multicontrolnet_full_34x16x16_vs_oracle_rel", worst)
    assert worst < 3e-3, worst
