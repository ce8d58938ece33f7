"""`cfg_shared_sample`: with equal sample halves the UNet runs the layers before the first per-half input (text tokens,
IP-Adapter tokens, reference maps, pose embedding) on the first half only and copies their outputs over the second half.
Every layer of that prefix computes an output row from its own frame, so the flagged forward must give the same bits as
the unflagged one, in its output and in every debug tap. It launches the same kernels, each on half the frames, so the
launch count does not change.

Everything but the sample (text tokens, IP-Adapter tokens, reference maps, pose embedding, ControlNet residuals) differs
between the halves. A flagged forward on a sample whose second half differs shows that the prefix really ran on the first
half only: it gives the unflagged result of the sample with its first half in both places. The narrow cases use 16 + 1
frames at 32 x 32, where the half batch alone would pick a different GroupNorm chunk count than the full batch."""
import pytest
import torch

from musev_b200.schema import preset_config
from musev_b200.synth import make_inputs, make_state_dict

pytestmark = pytest.mark.gpu
dev = "cuda"
NARROW = (64, 128, 128, 128)


def _model(preset, boc, dtype=torch.float32):
    from musev_b200.unet import UNet3DConditionModel
    cfg = preset_config(preset, block_out_channels=boc)
    model = UNet3DConditionModel(cfg, device=dev, dtype=dtype)
    model.load_state_dict({k: v.to(dev) for k, v in make_state_dict(cfg, seed=0, dtype=torch.float16).items()})
    return cfg, model


def _inputs(cfg, frames, h, w, dtype, refer=True, seed=11):
    inp = make_inputs(cfg, batch=2, frames=frames, h=h, w=w, n_vis_cond=1, seed=seed)
    s = inp["sample"]
    sample = torch.cat([s[:1], s[:1]]).to(dev, dtype)                  # equal halves, as ParallelDenoiser builds them
    assert not torch.equal(s[0], s[1])
    kw = dict(sample_index=inp["sample_index"], vision_conditon_frames_sample_index=inp["vision_conditon_frames_sample_index"],
              sample_frame_rate=8)
    if "vision_clip_emb" in inp:
        kw["vision_clip_emb"], kw["ip_adapter_scale"] = inp["vision_clip_emb"].to(dev, dtype), 0.7
    if refer and "down_block_refer_embs" in inp:
        kw["down_block_refer_embs"] = [r.to(dev, dtype) for r in inp["down_block_refer_embs"]]
        kw["mid_block_refer_emb"] = inp["mid_block_refer_emb"].to(dev, dtype)
    return sample, s.to(dev, dtype), inp["encoder_hidden_states"].to(dev, dtype), kw


def _run(model, sample, enc, kw, shared):
    from musev_b200 import _capi
    torch.cuda.synchronize()
    n0 = _capi.launch_count()
    out = model(sample, 601, enc, cfg_shared_sample=shared, **kw).sample.clone()
    torch.cuda.synchronize()
    return out, _capi.launch_count() - n0, model.debug_taps()


def _check(model, sample, unequal, enc, kw, prefix_runs):
    ref, n_ref, taps_ref = _run(model, sample, enc, kw, False)
    out, n_out, taps = _run(model, sample, enc, kw, True)
    assert torch.isfinite(ref).all()
    assert torch.equal(out, ref)
    assert taps.keys() == taps_ref.keys() and len(taps) > 0
    for name, t in taps.items():
        assert torch.equal(t, taps_ref[name]), name
    assert n_out == n_ref, (n_out, n_ref)
    del taps, taps_ref
    # a sample with unequal halves: the flagged forward reads only the first half when the prefix runs
    got = _run(model, unequal, enc, kw, True)[0]
    want = ref if prefix_runs else _run(model, unequal, enc, kw, False)[0]
    assert torch.equal(got, want)


def test_musev_text_cut(built_lib):
    """musev: the prefix runs up to and including the q projection of down_blocks.0.attentions.0's attn2."""
    cfg, model = _model("musev", NARROW)
    sample, unequal, enc, kw = _inputs(cfg, 16, 32, 32, torch.float32)
    _check(model, sample, unequal, enc, kw, True)


def test_musev_controlnet_residuals(built_lib):
    cfg, model = _model("musev", NARROW)
    sample, unequal, enc, kw = _inputs(cfg, 16, 32, 32, torch.float32)
    g = torch.Generator().manual_seed(3)
    NF, h = sample.shape[0] * sample.shape[2], 32
    shapes = ([(64, h, h)] * 3 + [(64, h // 2, h // 2)] + [(128, h // 2, h // 2)] * 2 + [(128, h // 4, h // 4)] * 3
              + [(128, h // 8, h // 8)] * 3)
    kw["down_block_additional_residuals"] = [(torch.randn(NF, c, a, b, generator=g) * 0.1).to(dev) for (c, a, b) in shapes]
    kw["mid_block_additional_residual"] = (torch.randn(NF, 128, h // 8, h // 8, generator=g) * 0.1).to(dev)
    _check(model, sample, unequal, enc, kw, True)


def test_musev_pose_guider_emb_empties_the_prefix(built_lib):
    cfg, model = _model("musev", NARROW)
    sample, unequal, enc, kw = _inputs(cfg, 16, 32, 32, torch.float32)
    g = torch.Generator().manual_seed(4)
    kw["pose_guider_emb"] = (torch.randn(sample.shape[0] * sample.shape[2], 64, 32, 32, generator=g) * 0.3).to(dev)
    _check(model, sample, unequal, enc, kw, False)


@pytest.mark.parametrize("refer", [True, False])
def test_referencenet_refer_maps_and_ip_adapter(built_lib, refer):
    """musev_referencenet (no transformer_in, IP-Adapter tokens in attn2): with reference maps the prefix is conv_in
    only; without them it runs up to attn2's q projection, before the IP-Adapter tokens are read."""
    cfg, model = _model("musev_referencenet", NARROW)
    sample, unequal, enc, kw = _inputs(cfg, 16, 32, 32, torch.float32, refer=refer)
    assert "vision_clip_emb" in kw and ("down_block_refer_embs" in kw) == refer
    _check(model, sample, unequal, enc, kw, True)


def test_full_size_musev_config2(built_lib):
    """The config-2 shape: CFG batch 2, 16 + 1 frames, 64 x 64 latents, full width, fp16 I/O."""
    cfg, model = _model("musev", (320, 640, 1280, 1280), dtype=torch.float16)
    sample, unequal, enc, kw = _inputs(cfg, 16, 64, 64, torch.float16)
    _check(model, sample, unequal, enc, kw, True)


def test_odd_batch_is_refused(built_lib):
    from musev_b200._capi import MvbError
    cfg, model = _model("musev", NARROW)
    inp = make_inputs(cfg, batch=3, frames=2, h=8, w=8, n_vis_cond=1, seed=2)
    x, enc = inp["sample"].to(dev), inp["encoder_hidden_states"].to(dev)
    kw = dict(sample_index=inp["sample_index"], vision_conditon_frames_sample_index=inp["vision_conditon_frames_sample_index"])
    with pytest.raises(MvbError, match="even batch"):
        model(x, 1, enc, cfg_shared_sample=True, **kw)
    assert torch.isfinite(model(x, 1, enc, **kw).sample).all()      # the handle stays usable
