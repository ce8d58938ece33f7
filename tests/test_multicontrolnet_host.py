"""CPU tests of the Multi-ControlNet feature: the `controlnet_keep` schedule, scale broadcasting, input checks, per-net window
slicing in `make_controlnet_fn` (with a fake ControlNet that records its inputs), and the oracle against the reference
fixture tests/golden/multicontrolnet_narrow.pt (oracle/make_golden_multicontrolnet.py)."""
import os
from types import SimpleNamespace

import pytest
import torch

from conftest import GOLDEN

NARROW = (64, 128, 128, 128)


class FakeControlNet:
    """The call surface `make_controlnet_fn` uses. Its 'maps' are the condition latents' frame means times the scale, so
    a test can see which frames and which rows a net was given; `accumulate_into` adds into the earlier maps."""

    def __init__(self, boc=(4, 8), device="cpu", dtype=torch.float32):
        self.config = SimpleNamespace(block_out_channels=boc, layers_per_block=1, cross_attention_dim=16,
                                      global_pool_conditions=False)
        self.device, self.dtype = torch.device(device), dtype
        self.calls = []

    def __call__(self, sample, timestep, encoder_hidden_states, controlnet_cond=None, conditioning_scale=1.0,
                 guess_mode=False, return_dict=True, controlnet_cond_latents=None, accumulate_into=None, **kw):
        self.calls.append(dict(sample=sample, timestep=timestep, enc=encoder_hidden_states, lat=controlnet_cond_latents,
                               scale=conditioning_scale, guess_mode=guess_mode, accumulate=accumulate_into is not None))
        v = controlnet_cond_latents.mean(dim=(1, 2, 3)).view(-1, 1, 1, 1) * conditioning_scale
        down = [v.expand(-1, 2, 2, 2).clone()]
        mid = v.expand(-1, 2, 1, 1).clone()
        if accumulate_into is not None:
            d0, m0 = accumulate_into
            d0[0] += down[0]
            m0 += mid
            return d0, m0
        return down, mid


def _lat(B2, n_vc, T, h, w, offset):
    """Condition latents whose value is (offset + 100 * row + frame), so slices can be read back from the fake's maps."""
    f = torch.arange(n_vc + T, dtype=torch.float32).view(1, 1, -1, 1, 1)
    r = torch.arange(B2, dtype=torch.float32).view(-1, 1, 1, 1, 1) * 100
    return (offset + r + f).expand(B2, 3, n_vc + T, h, w).contiguous()


# ---------------------------------------------------------------------------------------- controlnet_keep
@pytest.mark.parametrize("steps,start,end,n", [
    (20, 0.0, 1.0, None), (20, 0.0, 1.0, 2), (10, [0.0, 0.2], [1.0, 0.6], 2), (7, 0.1, [0.5, 0.9, 1.0], 3),
    (5, [0.0, 0.4], 1.0, 2), (3, [0.0, 0.0], [1.0, 1.0 / 3.0], 2), (30, 0.25, 0.75, None),
])
def test_keep_schedule_is_the_reference_expression(steps, start, end, n):
    from musev_b200.pipeline import controlnet_keep_schedule
    got = controlnet_keep_schedule(steps, start, end, n)
    nn = 1 if n is None else n
    s = start if isinstance(start, list) else [start] * nn
    e = end if isinstance(end, list) else [end] * nn
    for i in range(steps):   # musev/pipelines/pipeline_controlnet.py:1700-1711
        keeps = [1.0 - float(i / steps < a or (i + 1) / steps > b) for a, b in zip(s, e)]
        assert got[i] == (keeps[0] if n is None else keeps)


@pytest.mark.parametrize("start,end,n,msg", [
    ([0.0, 0.1], [1.0], 2, "same number of elements"),
    ([0.0, 0.1], [1.0, 1.0], 3, "controlnets available"),
    (0.5, 0.5, 2, "cannot be larger or equal"),
    (-0.1, 1.0, None, "smaller than 0"),
    (0.0, 1.5, None, "larger than 1.0"),
])
def test_keep_schedule_rejects_bad_windows(start, end, n, msg):
    from musev_b200.pipeline import controlnet_keep_schedule
    with pytest.raises(ValueError, match=msg):
        controlnet_keep_schedule(4, start, end, n)


# ---------------------------------------------------------------------------------------- input checks
def test_multi_rejects_nets_that_cannot_be_summed():
    from musev_b200.controlnet import MultiControlNetModel
    with pytest.raises(ValueError, match="at least one"):
        MultiControlNetModel([])
    with pytest.raises(ValueError, match="block_out_channels"):
        MultiControlNetModel([FakeControlNet((4, 8)), FakeControlNet((4, 16))])
    odd = FakeControlNet()
    odd.config.cross_attention_dim = 32
    with pytest.raises(ValueError, match="cross_attention_dim"):
        MultiControlNetModel([FakeControlNet(), odd])
    odd = FakeControlNet()
    odd.config.layers_per_block = 2
    with pytest.raises(ValueError, match="layers_per_block"):
        MultiControlNetModel([FakeControlNet(), odd])
    with pytest.raises(ValueError, match="one device and dtype"):
        MultiControlNetModel([FakeControlNet(), FakeControlNet(dtype=torch.float16)])
    with pytest.raises(ValueError, match="one device and dtype"):
        MultiControlNetModel([FakeControlNet(), FakeControlNet(device="meta")])
    m = MultiControlNetModel([FakeControlNet(), FakeControlNet()])
    assert m.dtype == torch.float32 and m.device == torch.device("cpu") and len(m.nets) == 2
    assert m.nets[0].config.global_pool_conditions is False      # read by prepare_controlnet_guess_mode (:1083-1090)


def test_multi_forward_rejects_lists_of_the_wrong_length():
    from musev_b200.controlnet import MultiControlNetModel
    m = MultiControlNetModel([FakeControlNet(), FakeControlNet()])
    x, enc = torch.zeros(2, 4, 2, 2), torch.zeros(2, 3, 16)
    lat = [torch.ones(2, 4, 2, 2)] * 2
    with pytest.raises(ValueError, match="controlnet_conditioning_scale"):
        m(x, 1, enc, None, [1.0], controlnet_cond_latents=lat)
    with pytest.raises(ValueError, match="controlnet_conditioning_scale"):
        m(x, 1, enc, None, 1.0, controlnet_cond_latents=lat)
    with pytest.raises(ValueError, match="controlnet_cond_latents"):
        m(x, 1, enc, None, [1.0, 1.0], controlnet_cond_latents=lat[:1])
    with pytest.raises(ValueError, match="image"):
        m(x, 1, enc, [torch.zeros(2, 3, 16, 16)] * 3, [1.0, 1.0], controlnet_cond_latents=lat)
    down, mid = m(x, 1, enc, None, [1.0, 2.0], controlnet_cond_latents=lat, return_dict=True)   # a tuple regardless
    assert torch.equal(mid, torch.full_like(mid, 3.0))
    assert [c["accumulate"] for c in m.nets[0].calls + m.nets[1].calls] == [False, True]


def test_make_controlnet_fn_rejects_lists_of_the_wrong_length():
    from musev_b200.pipeline import make_controlnet_fn
    nets = [FakeControlNet(), FakeControlNet()]
    lat = [_lat(2, 1, 4, 2, 2, 0)] * 2
    prompt = torch.zeros(2, 3, 16)
    with pytest.raises(ValueError, match="controlnet_latents"):
        make_controlnet_fn(nets, lat[:1], prompt, 1)
    with pytest.raises(ValueError, match="controlnet_latents"):
        make_controlnet_fn(nets, lat[0], prompt, 1)
    with pytest.raises(ValueError, match="controlnet_conditioning_scale"):
        make_controlnet_fn(nets, lat, prompt, 1, controlnet_conditioning_scale=[1.0, 1.0, 1.0])
    fn = make_controlnet_fn(nets, lat, prompt, 1, controlnet_keep=[[1.0, 1.0, 1.0]])
    with pytest.raises(ValueError, match="controlnet_keep"):
        fn([0, 1], torch.zeros(2, 4, 3, 2, 2), 500, 0)


# ---------------------------------------------------------------------------------------- scales, keep, slicing
def test_scale_broadcast_keep_and_skipping():
    from musev_b200.pipeline import make_controlnet_fn
    prompt = torch.zeros(2, 3, 16)
    lat = [_lat(2, 1, 4, 2, 2, 0), _lat(2, 1, 4, 2, 2, 1000)]
    x = torch.zeros(2, 4, 3, 2, 2)
    nets = [FakeControlNet(), FakeControlNet()]
    fn = make_controlnet_fn(nets, lat, prompt, 1, controlnet_conditioning_scale=0.5,
                            controlnet_keep=[[1.0, 1.0], [1.0, 0.0], [0.0, 0.0], 1.0])
    fn([0, 1], x, 900, 0)
    assert [c["scale"] for c in nets[0].calls] == [0.5] and [c["scale"] for c in nets[1].calls] == [0.5]
    assert nets[1].calls[0]["accumulate"] and not nets[0].calls[0]["accumulate"]
    down, mid = fn([0, 1], x, 800, 1)                              # net 1 is off: not run, net 0's maps alone
    assert len(nets[0].calls) == 2 and len(nets[1].calls) == 1
    assert fn([0, 1], x, 700, 2) == (None, None)                   # every net off: no residuals
    assert len(nets[0].calls) == 2 and len(nets[1].calls) == 1
    fn([0, 1], x, 600, 3)                                          # a float keep applies to every net
    assert len(nets[0].calls) == 3 and len(nets[1].calls) == 2
    nets = [FakeControlNet(), FakeControlNet()]
    fn = make_controlnet_fn(nets, lat, prompt, 1, controlnet_conditioning_scale=[0.7, 1.3], controlnet_keep=[[1.0, 0.5]])
    fn([0, 1], x, 900, 0)
    assert nets[0].calls[0]["scale"] == 0.7 and nets[1].calls[0]["scale"] == 1.3 * 0.5
    # with the first net off, the next net that runs writes the maps instead of adding into them
    nets = [FakeControlNet(), FakeControlNet()]
    fn = make_controlnet_fn(nets, lat, prompt, 1, controlnet_keep=[[0.0, 1.0]])
    down, mid = fn([0, 1], x, 900, 0)
    assert not nets[0].calls and not nets[1].calls[0]["accumulate"]


@pytest.mark.parametrize("cfg_split", [False, True])
def test_per_net_slicing_under_cfg_split(cfg_split):
    """Each net gets its own latents at the window's frames (vision-condition frames first) and, under cfg_split, only the
    rows of the CFG half this rank runs; prompts are sliced the same way. One net gives today's single-net calls."""
    from musev_b200.pipeline import make_controlnet_fn
    B, n_vc, T, h, w = 1, 1, 6, 2, 2
    prompt = torch.arange(2, dtype=torch.float32).view(2, 1, 1).expand(2, 3, 16).contiguous()
    lats = [_lat(2 * B, n_vc, T, h, w, 0), _lat(2 * B, n_vc, T, h, w, 1000)]
    c = [2, 3, 4]
    rows = slice(B, 2 * B) if cfg_split else None
    x = torch.zeros(B if cfg_split else 2 * B, 4, n_vc + len(c), h, w)
    nets = [FakeControlNet(), FakeControlNet()]
    fn = make_controlnet_fn(nets, lats, prompt, n_vc, controlnet_conditioning_scale=[1.0, 2.0])
    down, mid = fn(c, x, 500, 0, rows) if cfg_split else fn(c, x, 500, 0)
    single = FakeControlNet()
    sfn = make_controlnet_fn(single, lats[1], prompt, n_vc)
    sfn(c, x, 500, 0, rows) if cfg_split else sfn(c, x, 500, 0)
    frames = [0] + [ci + n_vc for ci in c]
    row_ids = [1] if cfg_split else [0, 1]
    for k, (net, off) in enumerate(zip(nets, (0, 1000))):
        call = net.calls[0]
        assert call["lat"].shape == (len(row_ids) * len(frames), 3, h, w)
        want = torch.tensor([off + 100 * r + f for r in row_ids for f in frames], dtype=torch.float32)
        assert torch.equal(call["lat"][:, 0, 0, 0], want), k
        assert torch.equal(call["enc"][:, 0, 0], torch.tensor([float(r) for r in row_ids for _ in frames]))
        assert call["sample"].shape == (len(row_ids) * len(frames), 4, h, w)
    assert torch.equal(single.calls[0]["lat"], nets[1].calls[0]["lat"])
    assert torch.equal(single.calls[0]["enc"], nets[1].calls[0]["enc"])
    want_mid = nets[0].calls[0]["lat"].mean(dim=(1, 2, 3)) + 2.0 * nets[1].calls[0]["lat"].mean(dim=(1, 2, 3))
    assert torch.equal(mid[:, 0, 0, 0], want_mid)


def test_guess_mode_pads_the_summed_conditional_half_once():
    from musev_b200.pipeline import make_controlnet_fn
    B, n_vc, T, h, w = 1, 1, 4, 2, 2
    prompt = torch.zeros(2, 3, 16)
    lats = [_lat(B, n_vc, T, h, w, 0), _lat(B, n_vc, T, h, w, 1000)]      # [B, ...] in guess mode
    nets = [FakeControlNet(), FakeControlNet()]
    fn = make_controlnet_fn(nets, lats, prompt, n_vc, guess_mode=True)
    x = torch.zeros(2 * B, 4, n_vc + 2, h, w)
    down, mid = fn([0, 1], x, 500, 0)
    tc = n_vc + 2
    assert mid.shape[0] == 2 * B * tc and nets[0].calls[0]["sample"].shape[0] == B * tc
    assert torch.equal(mid[:B * tc], torch.zeros_like(mid[:B * tc]))
    want = nets[0].calls[0]["lat"].mean(dim=(1, 2, 3)) + nets[1].calls[0]["lat"].mean(dim=(1, 2, 3))
    assert torch.equal(mid[B * tc:, 0, 0, 0], want)
    assert all(c["guess_mode"] for n in nets for c in n.calls)


# ---------------------------------------------------------------------------------------- oracle vs the reference
def _oracle_nets(seeds, boc):
    from musev_b200.schema import ControlNetConfig
    from musev_b200.synth import make_state_dict
    from oracle.controlnet_oracle import ControlNetOracle
    cfg = ControlNetConfig(block_out_channels=tuple(boc))
    return [ControlNetOracle(cfg, make_state_dict(cfg, seed=s)) for s in seeds]


def _images(n, h, w, seed):
    from musev_b200.schema import ControlNetConfig
    from musev_b200.synth import make_controlnet_inputs
    return make_controlnet_inputs(ControlNetConfig(block_out_channels=NARROW), frames=n, h=h, w=w, seed=seed)["controlnet_cond"]


@pytest.mark.parametrize("tag", ["two", "three_guess"])
def test_multi_oracle_matches_reference_fixture(tag):
    from musev_b200.schema import ControlNetConfig
    from musev_b200.synth import make_controlnet_inputs
    from oracle.multicontrolnet_oracle import multi_controlnet_forward
    g = torch.load(os.path.join(GOLDEN, "multicontrolnet_narrow.pt"))[tag]
    m = g["meta"]
    nets = _oracle_nets(m["weight_seeds"], m["block_out_channels"])
    inp = make_controlnet_inputs(ControlNetConfig(block_out_channels=tuple(m["block_out_channels"])), frames=m["frames"],
                                 h=m["h"], w=m["w"], seed=m["input_seed"])
    images = [_images(m["frames"], m["h"], m["w"], s) for s in m["image_seeds"]]
    down, mid = multi_controlnet_forward(nets, inp["sample"], m["timestep"], inp["encoder_hidden_states"], images,
                                         m["scales"], guess_mode=m["guess_mode"])
    maps = list(down) + [mid]
    assert [list(t.shape) for t in maps] == m["shapes"]
    for k, mp in enumerate(maps):
        flat = mp.reshape(-1)
        idx = torch.randint(0, flat.numel(), (m["n_samples"],), generator=torch.Generator().manual_seed(m["sample_seed_base"] + k))
        ref = g["samples"][k]
        assert (flat[idx] - ref).abs().max().item() < 1e-5 * max(1.0, ref.abs().max().item()), f"map {k}"
    # embedding once and passing latents gives the same sum as embedding inside every net
    lat = [n.cond_embedding(im) for n, im in zip(nets, images)]
    down2, mid2 = multi_controlnet_forward(nets, inp["sample"], m["timestep"], inp["encoder_hidden_states"], None,
                                           m["scales"], guess_mode=m["guess_mode"], controlnet_cond_latents=lat)
    assert torch.equal(mid, mid2) and all(torch.equal(a, b) for a, b in zip(down, down2))


def test_multi_oracle_loop_matches_reference_fixture():
    """The oracle loop with per-net latents embedded once per call and sliced per window against the reference loop, whose
    nets embed their sliced images on every window-step."""
    from musev_b200.schema import preset_config
    from musev_b200.synth import make_inputs, make_state_dict
    from oracle.multicontrolnet_oracle import denoise_loop_multi
    from oracle.pipeline_oracle import SD15_DDIM, DDIMOracle
    from oracle.unet3d_oracle import UNet3DOracle
    g = torch.load(os.path.join(GOLDEN, "multicontrolnet_narrow.pt"))["loop"]
    m = g["meta"]
    cfg = preset_config(m["preset"], block_out_channels=tuple(m["block_out_channels"]))
    uo = UNet3DOracle(cfg, make_state_dict(cfg, seed=m["weight_seed"]))
    nets = _oracle_nets(m["cn_weight_seeds"], m["block_out_channels"])
    T, h, w = m["T"], m["h"], m["w"]
    gen = torch.Generator().manual_seed(m["input_seed"])
    latents = torch.randn(1, 4, T, h, w, generator=gen)
    cond = torch.randn(1, 4, 1, h, w, generator=gen) * 0.5
    prompt = torch.randn(2, 77, cfg.cross_attention_dim, generator=gen)
    extra = make_inputs(cfg, batch=2, frames=1, h=h, w=w, seed=m["input_seed"])
    kw = {k: extra[k] for k in ("down_block_refer_embs", "mid_block_refer_emb", "vision_clip_emb") if k in extra}
    cn_lat = []
    for k, net in enumerate(nets):
        e = net.cond_embedding(_images(1 + T, h, w, m["image_seed"] + k))                   # [(1 + T), C0, h, w]
        cn_lat.append(torch.cat([e.permute(1, 0, 2, 3).unsqueeze(0)] * 2))               # [2, C0, 1 + T, h, w]
    out = denoise_loop_multi(lambda *a, **k: uo(*a, **k), DDIMOracle(**SD15_DDIM), latents, cond, prompt, m["steps"],
                             m["guidance_scale"], nets, cn_lat, m["scales"], context_frames=m["context_frames"],
                             context_overlap=m["context_overlap"], motion_speed=8,
                             unet_kwargs=dict(kw, ip_adapter_scale=1.0))
    assert len(m["contexts"]) == 3
    err = (out - g["latents"]).abs().max().item()
    assert err < 2e-4, err
