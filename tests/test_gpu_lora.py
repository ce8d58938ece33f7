"""LoRA merged into the engine UNet on the device (`mvb_unet_merge_lora`, musev_b200/csrc/lora.cu): read-back bits against
the plain-torch oracle (oracle/lora_oracle.py, itself pinned to the unmodified reference by tests/golden/lora_narrow.pt),
the merged forward and a 4-step LCM loop against the fp32 oracle, atomicity of rejected calls, the drop-in
`update_pipeline_lora_models` / `unload_lora`, and a rank-64 LoRA on every matrix and convolution of the SD-1.5 UNet.
With MVB_PARITY_LOG=<file> set, every measured distance is appended to <file> next to its bound (`_record`).

Bits rule: the engine sums the rank in a fixed order with fp32 FMA, torch.mm in its own order, so a delta that lands
next to an fp16 rounding boundary may round the other way. At most 1e-3 of the elements may differ, each by one ulp."""
import json
import os
from types import SimpleNamespace

import pytest
import torch

from conftest import GOLDEN
from musev_b200.schema import preset_config, unet_param_shapes
from musev_b200.synth import make_inputs, make_lora_state_dict, make_state_dict, make_text_encoder

pytestmark = pytest.mark.gpu
dev = "cuda"
NARROW = (64, 128, 128, 128)
FULL = (320, 640, 1280, 1280)
FWD_TOL = 1e-2
EXTRA = ["down_blocks.0.attentions.0.transformer_blocks.0.attn2.to_k_ip.weight",
         "up_blocks.2.attentions.1.transformer_blocks.0.attn2.to_v_ip.weight",
         "mid_block_refer_emb_attns.to_v.weight", "down_blocks.1.temp_attentions.0.frame_emb_proj.weight"]


def _record(name, err, bound):
    path = os.environ.get("MVB_PARITY_LOG")
    if path:
        try:
            with open(path, "a") as fh:
                fh.write(json.dumps({"test": name, "value": err, "bound": bound}) + "\n")
        except OSError:
            pass
    assert err < bound, (name, err, bound)


def _ordered(t):
    i = t.contiguous().view(torch.int16).to(torch.int32)
    return torch.where(i < 0, -(i + 32768), i)      # fp16 bits -> integers ordered like the values (+0 == -0)


def _bits_rule(name, got, want):
    """(fraction of elements that differ, largest difference in ulps)"""
    assert got.shape == want.shape and got.dtype == want.dtype == torch.float16, name
    d = (_ordered(got) - _ordered(want.to(got.device))).abs()
    return (d > 0).float().mean().item(), int(d.max().item())


def _check_bits(tag, names, model, want):
    worst_frac, worst_ulp = 0.0, 0
    for n in names:
        frac, ulp = _bits_rule(n, model.debug_weight(n), want[n])
        worst_frac, worst_ulp = max(worst_frac, frac), max(worst_ulp, ulp)
        assert ulp <= 1, (n, ulp)
    _record(f"lora_{tag}_frac_differing", worst_frac, 1e-3)


def _spec():
    return torch.load(os.path.join(GOLDEN, "lora_narrow.pt"))


def _lora(cfg, meta, extra=()):
    shapes = unet_param_shapes(cfg)
    targets = [t for t in list(meta["targets"]) + list(extra) if t in shapes]
    return make_lora_state_dict(cfg, targets, rank=meta["rank"], seed=meta["lora_seed"], amp=meta["amp"],
                                no_alpha=meta["no_alpha"], f32=meta["f32"], text_targets=[tuple(t) for t in meta["text_targets"]])


def _model(cfg, sd16):
    from musev_b200.unet import UNet3DConditionModel
    m = UNet3DConditionModel(cfg, device=dev, dtype=torch.float32)
    m.load_state_dict(sd16)
    return m


def _unet_part(sd):
    return {k: v for k, v in sd.items() if not k.startswith("lora_te")}


def test_merge_and_unload_bits_narrow(built_lib):
    from musev_b200 import lora
    from oracle.lora_oracle import deltas, merged
    meta = _spec()["meta"]
    cfg = preset_config("musev_referencenet", block_out_channels=NARROW)
    sd16 = {k: v.half() for k, v in make_state_dict(cfg, seed=0).items()}
    model = _model(cfg, sd16)
    lsd = _unet_part(_lora(cfg, meta, EXTRA))
    ds = deltas(cfg, lsd, meta["strength"], "ALL")
    want = merged(sd16, ds)
    pipe = SimpleNamespace(unet=model, text_encoder=None)
    _, undo = lora.update_pipeline_lora_model(pipe, lsd, alpha=meta["strength"], need_unload=True)
    targets = list(ds)
    assert len(targets) == len(meta["targets"]) + len(EXTRA) and len(undo) == len(targets)
    _check_bits("apply_narrow", targets, model, want)
    untouched = [n for n, s in unet_param_shapes(cfg).items() if len(s) >= 2 and n not in ds]
    for n in untouched:
        assert torch.equal(model.debug_weight(n).cpu(), sd16[n]), n
    lora.unload_lora(undo)
    _check_bits("unload_narrow", targets, model, merged(want, ds, subtract=True))
    for n in untouched:
        assert torch.equal(model.debug_weight(n).cpu(), sd16[n]), n


@pytest.mark.parametrize("preset", ["musev", "musev_referencenet"])
def test_merged_forward_vs_oracle_and_reference(built_lib, preset):
    from oracle.lora_oracle import deltas, merged
    from oracle.unet3d_oracle import UNet3DOracle
    g = _spec()
    meta, fw = g["meta"], g["forward"]
    cfg = preset_config(preset, block_out_channels=NARROW)
    sd16 = {k: v.half() for k, v in make_state_dict(cfg, seed=0).items()}
    lsd = _unet_part(_lora(cfg, meta))
    model = _model(cfg, sd16)
    model._merge_lora(*_engine_args(cfg, lsd, meta["strength"]), subtract=False)
    m16 = merged(sd16, deltas(cfg, lsd, meta["strength"], "ALL"))
    inp = make_inputs(cfg, batch=fw["batch"], frames=fw["frames"], h=fw["h"], w=fw["w"], n_vis_cond=1, seed=fw["input_seed"])
    kw = dict(sample_index=inp["sample_index"], vision_conditon_frames_sample_index=inp["vision_conditon_frames_sample_index"],
              sample_frame_rate=fw["sample_frame_rate"], down_block_refer_embs=inp.get("down_block_refer_embs"),
              mid_block_refer_emb=inp.get("mid_block_refer_emb"), vision_clip_emb=inp.get("vision_clip_emb"),
              ip_adapter_scale=fw["ip_adapter_scale"])
    t = fw["timestep"]
    ref = UNet3DOracle(cfg, {k: v.float() for k, v in m16.items()}, device=dev)(inp["sample"], t, inp["encoder_hidden_states"], **kw)
    base = UNet3DOracle(cfg, {k: v.float() for k, v in sd16.items()}, device=dev)(inp["sample"], t, inp["encoder_hidden_states"], **kw)
    dk = {k: ([x.to(dev) for x in v] if isinstance(v, list) else (v.to(dev) if torch.is_tensor(v) and v.is_floating_point() else v))
          for k, v in kw.items()}
    out = model(inp["sample"].to(dev), torch.tensor(t), inp["encoder_hidden_states"].to(dev), do_classifier_free_guidance=True, **dk).sample
    err = (out - ref).abs().max().item()
    moved = (ref - base).abs().max().item()
    _record(f"lora_fwd_{preset}_vs_oracle", err, FWD_TOL)
    _record(f"lora_fwd_{preset}_moved_by_lora_over_10x_err", -moved, -10 * err)
    if preset == "musev_referencenet":
        _record(f"lora_fwd_{preset}_vs_reference_golden", (out.cpu() - g["out"]).abs().max().item(), FWD_TOL)


def _engine_args(cfg, lsd, strength):
    """(targets, ups, downs, scales) of a kohya UNet LoRA with block weights ALL, for UNet3DConditionModel._merge_lora."""
    from musev_b200 import lora
    names = lora.kohya_name_map(cfg)
    out = ([], [], [], [])
    for t in lora.pair_keys(lsd):
        up, down, r = lora.factors(lsd, t)
        out[0].append(names[t.module[len("lora_unet_"):]])
        out[1].append(up.to(dev).contiguous())
        out[2].append(down.to(dev).contiguous())
        out[3].append(lora.target_scale(lsd, t, strength, r))
    return out


def test_lcm_loop_with_merged_lora(built_lib):
    """ParallelDenoiser(engine + merged LCM-style LoRA, LCMScheduler), 4 steps, against the oracle loop around LCMOracle with
    the merged fp32 weights. Both sides draw the per-step noise from CUDA generators with the same seed."""
    from musev_b200.pipeline import ParallelDenoiser
    from musev_b200.samplers import LCMScheduler
    from oracle.lora_oracle import deltas, merged
    from oracle.pipeline_oracle import denoise_loop
    from oracle.sampler_oracle import LCMOracle
    from oracle.unet3d_oracle import UNet3DOracle
    meta = _spec()["meta"]
    cfg = preset_config("musev", block_out_channels=NARROW)
    sd16 = {k: v.half() for k, v in make_state_dict(cfg, seed=0).items()}
    lsd = _unet_part(_lora(cfg, meta))
    model = _model(cfg, sd16)
    model._merge_lora(*_engine_args(cfg, lsd, meta["strength"]), subtract=False)
    m16 = merged(sd16, deltas(cfg, lsd, meta["strength"], "ALL"))
    gen = torch.Generator().manual_seed(29)
    T, h, w = 12, 16, 16
    latents = torch.randn(1, 4, T, h, w, generator=gen)
    cond = torch.randn(1, 4, 1, h, w, generator=gen) * 0.5
    prompt = torch.randn(2, 77, cfg.cross_attention_dim, generator=gen)
    out = ParallelDenoiser(model, LCMScheduler())(latents.to(dev), cond.to(dev), prompt.to(dev), num_inference_steps=4,
                                                  guidance_scale=1.5, context_frames=8, context_overlap=4,
                                                  generator=torch.Generator(device=dev).manual_seed(5)).latents.cpu()

    class _Lcm(LCMOracle):
        """LCMOracle whose per-step noise comes from a CUDA generator seeded like the engine run's."""

        def __init__(self):
            super().__init__()
            self.g = torch.Generator(device=dev).manual_seed(5)

        def step(self, model_output, t, sample, generator=None):
            real = torch.randn

            def cuda_randn(shape, generator=None, dtype=torch.float32):
                return real(shape, generator=self.g, device=dev, dtype=torch.float32).cpu().to(dtype)

            torch.randn = cuda_randn
            try:
                return super().step(model_output, t, sample)
            finally:
                torch.randn = real

    def loop(sd):
        o = UNet3DOracle(cfg, {k: v.float() for k, v in sd.items()}, device=dev)
        return denoise_loop(lambda s, t, e, **k: o(s, t, e, **k).cpu(), _Lcm(), latents, cond, prompt, 4, 1.5,
                            context_frames=8, context_overlap=4)

    ref = loop(m16)
    # relative to the result's magnitude, as the Euler loop test is relative to its latents' scale: LCM's x0 prediction at
    # t = 999 multiplies the eps error by 1 / sqrt(alpha_bar) ~ 15, so the absolute error scales with the denoised latents
    scale = ref.abs().max().item()
    err = (out - ref).abs().max().item()
    _record("lora_lcm_loop_4step_rel", err / scale, 2e-2)
    moved = (ref - loop(sd16)).abs().max().item()
    _record("lora_lcm_moved_by_lora_over_10x_err", -moved, -10 * err)


def test_rejected_calls_change_no_weight(built_lib):
    from musev_b200._capi import MvbError
    from musev_b200.controlnet import ControlNetModel
    from musev_b200.schema import ControlNetConfig
    from musev_b200._capi import MvbNamedTensor, _named, lib
    from musev_b200.unet import UNet3DConditionModel
    cfg = preset_config("musev", block_out_channels=NARROW)
    sd16 = {k: v.half() for k, v in make_state_dict(cfg, seed=0).items()}
    model = _model(cfg, sd16)
    mats = [n for n, s in unet_param_shapes(cfg).items() if len(s) >= 2]
    before = {n: model.debug_weight(n).clone() for n in mats}
    a, b = "conv_in.weight", "down_blocks.0.attentions.0.proj_in.weight"
    up_a, down_a = torch.randn(64, 4, 1, 1, device=dev).half(), torch.randn(4, 4, 3, 3, device=dev).half()
    up_b, down_b = torch.randn(64, 4, 1, 1, device=dev).half(), torch.randn(4, 64, 1, 1, device=dev).half()
    with pytest.raises(MvbError, match="twice"):
        model._merge_lora([a, b, a], [up_a, up_b, up_a], [down_a, down_b, down_a], [1.0, 1.0, 1.0])
    with pytest.raises(MvbError, match="do not fit"):
        model._merge_lora([a, b], [up_a, up_b], [down_a, torch.randn(4, 63, 1, 1, device=dev).half()], [1.0, 1.0])
    with pytest.raises(MvbError, match="exceeds 256"):
        model._merge_lora([a], [torch.zeros(64, 257, 1, 1, device=dev).half()], [torch.zeros(257, 4, 3, 3, device=dev).half()], [1.0])
    with pytest.raises(MvbError, match="not a mergeable"):
        model._merge_lora(["down_blocks.0.resnets.0.norm1.weight"], [up_a], [down_a], [1.0])
    fresh = UNet3DConditionModel(cfg, device=dev)
    with pytest.raises(MvbError, match="finalize"):
        fresh._merge_lora([a], [up_a], [down_a], [1.0])
    cn = ControlNetModel(ControlNetConfig(block_out_channels=NARROW), device=dev)
    arr_u, arr_d = (MvbNamedTensor * 1)(_named(a, up_a)), (MvbNamedTensor * 1)(_named(a, down_a))
    import ctypes as C
    assert lib().mvb_unet_merge_lora(cn._h, arr_u, arr_d, (C.c_float * 1)(1.0), 1, 0) == -3
    for n in mats:
        assert torch.equal(model.debug_weight(n), before[n]), n


def test_drop_in_two_loras_and_unload(built_lib, tmp_path):
    from safetensors.torch import save_file
    from musev_b200 import lora
    from oracle.lora_oracle import deltas, merged
    meta = _spec()["meta"]
    cfg = preset_config("musev_referencenet", block_out_channels=NARROW)
    sd16 = {k: v.half() for k, v in make_state_dict(cfg, seed=0).items()}
    model = _model(cfg, sd16)
    te = make_text_encoder(meta["text_width"], meta["text_seed"])
    k_proj = te.text_model.encoder.layers[0].self_attn.k_proj
    te_w0 = k_proj.weight.data.clone()
    l1 = _lora(cfg, meta, EXTRA)
    l2 = make_lora_state_dict(cfg, ["conv_in.weight", "down_blocks.0.attentions.0.proj_in.weight", "conv_out.weight"],
                              rank=16, seed=77, f32=["conv_out.weight"])
    p1, p2 = str(tmp_path / "style.safetensors"), str(tmp_path / "lcm.safetensors")
    save_file(dict(l1), p1)
    save_file(dict(l2), p2)
    pipe = SimpleNamespace(unet=model, text_encoder=te)
    _, undo = lora.update_pipeline_lora_models(pipe, {p1: {"strength": 0.7, "lora_block_weight": "FACE"},
                                                      p2: {"strength": 1.0, "strength_offset": 0.25}})
    d1 = deltas(cfg, l1, 0.7, "FACE")
    d2 = deltas(cfg, l2, 1.25, "ALL")
    te_want = te_w0.clone()
    te_want += d1.pop("lora_te_" + meta["text_targets"][0][0])
    assert torch.equal(k_proj.weight.data, te_want)
    w1 = merged(sd16, d1)
    w2 = merged(w1, d2)
    _check_bits("dropin_two", list(dict.fromkeys(list(d1) + list(d2))), model, w2)
    lora.unload_lora(undo)        # the reference's unload list holds the last LoRA only (model_util.py:464)
    _check_bits("dropin_unload", list(dict.fromkeys(list(d1) + list(d2))), model, merged(w2, d2, subtract=True))


def test_full_width_rank64_every_matrix_and_conv(built_lib):
    from musev_b200 import lora
    from oracle.lora_oracle import deltas
    cfg = preset_config("musev_referencenet", block_out_channels=FULL)
    sd16 = {k: v.half() for k, v in make_state_dict(cfg, seed=0).items()}
    targets = [n for n, s in unet_param_shapes(cfg).items() if len(s) in (2, 4)]
    lsd = make_lora_state_dict(cfg, targets, rank=64, seed=9)
    model = _model(cfg, sd16)
    pipe = SimpleNamespace(unet=model, text_encoder=None)
    lora.update_pipeline_lora_model(pipe, lsd, alpha=1.0)
    ds = deltas(cfg, {k: v.to(dev) for k, v in lsd.items()}, 1.0, "ALL", device=dev)   # torch fp32 on the GPU
    groups = {}
    for n in targets:
        kind = n.split(".")[-2] if not n.split(".")[-2].isdigit() else n.split(".")[-3]
        groups.setdefault((kind, len(unet_param_shapes(cfg)[n])), []).append(n)
    sample = [n for g in groups.values() for n in (g[:2] + g[-1:])]
    assert len(groups) >= 15 and len(sample) >= 40
    want = {}
    for n in sample:
        w = sd16[n].to(dev).clone()
        w += ds[n]
        want[n] = w
    _check_bits("apply_full_rank64", sample, model, want)
