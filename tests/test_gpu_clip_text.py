"""CLIP text encoder (the prompt encoder) on the engine: the causal attention op against an fp32 masked softmax, the engine
against the fp32 oracle and the transformers fixtures (tests/golden/clip_text_*.pt), causality and sequence independence
bit for bit, the fp16 yardstick, the encode_weighted_prompt -> UNet chain, text-encoder LoRA merged on the device, and
rejections before any launch. With MVB_PARITY_LOG=<file> set, every measured distance is appended to <file> next to its
bound."""
import ctypes as C
import json
import os
from types import SimpleNamespace

import pytest
import torch

from conftest import GOLDEN
from musev_b200.schema import ClipTextConfig, preset_config
from musev_b200.synth import make_clip_text_state_dict, make_input_ids, make_lora_state_dict, make_state_dict, make_text_encoder

pytestmark = pytest.mark.gpu
dev = "cuda"
# per max(1, max|ref|); measured at most 1.4e-3 (narrow) and 2.3e-3 (SD-1.5) on an H100 80GB HBM3 at 700 W over the oracle,
# fixture and chain comparisons (start: 1e-2 / 2e-2); the causal op at most 1.13e-3 absolute (start: 5e-3)
TOL = {"narrow": 3e-3, "full": 5e-3}
OP_TOL = 2.5e-3
CHAIN_UNET_TOL = 4e-3   # measured 1.7e-3 (start: 2e-2)


def _record(name, err, bound):
    path = os.environ.get("MVB_PARITY_LOG")
    if path:
        try:
            with open(path, "a") as fh:
                fh.write(json.dumps({"test": name, "value": err, "bound": bound}) + "\n")
        except OSError:
            pass
    assert err < bound, (name, err, bound)


def _rel(got, ref):
    return (got.float() - ref.float()).abs().max().item() / max(1.0, ref.abs().max().item())


def _rms(got, ref):
    return (got.float() - ref.float()).pow(2).mean().sqrt().item()


def _fixture(tag):
    g = torch.load(os.path.join(GOLDEN, f"clip_text_{tag}.pt"))
    return g["meta"], g["configs"]


def _model(cfg, seed, outlier_channels=0, dtype=torch.float32):
    from musev_b200.clip_text import CLIPTextModel
    sd = {k: v.half() for k, v in make_clip_text_state_dict(cfg, seed=seed, outlier_channels=outlier_channels).items()}
    m = CLIPTextModel.from_state_dict(sd, cfg, device=dev, dtype=dtype)
    return m, {k: v.float() for k, v in sd.items()}


# ------------------------------------------------------------------------------------------------ causal attention op
def _causal_ref(qkv, NF, Nq, heads, d, dp, scale):
    hd = heads * dp
    x = qkv.float().view(NF, Nq, 3, heads, dp)[..., :d]
    q, k, v = (x[:, :, i].transpose(1, 2) for i in range(3))          # [NF, heads, Nq, d]
    s = (q @ k.transpose(-1, -2)) * scale
    s = s.masked_fill(torch.ones(Nq, Nq, dtype=torch.bool, device=qkv.device).triu(1), float("-inf"))
    o = torch.softmax(s, dim=-1) @ v
    assert hd == qkv.shape[1] // 3
    return o.transpose(1, 2).reshape(NF * Nq, heads * d)


@pytest.mark.parametrize("dp", [48, 64, 128])
@pytest.mark.parametrize("NF", [1, 3])
def test_causal_attention_op(built_lib, dp, NF):
    from musev_b200 import ops
    d = {48: 40, 64: 64, 128: 128}[dp]
    heads = 2
    hd = heads * dp
    worst = 0.0
    for Nq in (1, 77, 128, 129, 300):
        g = torch.Generator(device="cpu").manual_seed(dp * 1000 + NF * 10 + Nq)
        qkv = torch.zeros(NF * Nq, 3 * hd)
        for i in range(3):
            for h in range(heads):
                qkv[:, i * hd + h * dp: i * hd + h * dp + d] = torch.randn(NF * Nq, d, generator=g) * (1.5 if i < 2 else 1.0)
        qkv = qkv.half().to(dev)
        scale = d ** -0.5
        out = ops.attention(qkv[:, :hd], [dict(k=qkv[:, hd:2 * hd], v=qkv[:, 2 * hd:], nk=Nq)], NF, Nq, heads, d, dp, scale,
                            causal=True)
        ref = _causal_ref(qkv, NF, Nq, heads, d, dp, scale)
        assert torch.isfinite(out).all()
        worst = max(worst, (out.float() - ref).abs().max().item())
        if Nq == 1:   # one key: the output is v itself
            assert torch.allclose(out.float(), ref, atol=1e-3)
    _record(f"causal_attention_dp{dp}_NF{NF}_vs_fp32", worst, OP_TOL)


def test_causal_attention_rejects_other_layouts(built_lib):
    from musev_b200 import _capi, ops
    from musev_b200._capi import MvbError
    NF, Nq, heads, d, dp = 2, 77, 2, 64, 64
    hd = heads * dp
    qkv = torch.randn(NF * Nq, 3 * hd, device=dev).half()
    q, k, v = qkv[:, :hd], qkv[:, hd:2 * hd], qkv[:, 2 * hd:]
    n0 = _capi.launch_count()
    for seg in ([dict(k=k, v=v, nk=Nq), dict(k=k, v=v, nk=Nq)],        # two segments
                [dict(k=k, v=v, nk=Nq - 1)],                           # nk != Nq
                [dict(k=k, v=v, nk=Nq, fmul=Nq - 1)],                  # rows of another sequence
                [dict(k=k, v=v, nk=Nq, fadd=1)],
                [dict(k=k, v=v, nk=Nq, fdiv=2)]):
        with pytest.raises(MvbError, match="causal"):
            ops.attention(q, seg, NF, Nq, heads, d, dp, d ** -0.5, causal=True)
    assert _capi.launch_count() == n0


# ------------------------------------------------------------------------------------------------ engine
def _check_against(tag, name, m, sd32, cfg, ids, e=None, bound=None):
    from oracle.clip_text_oracle import clip_text_forward
    bound = bound or TOL[tag]
    out = m(ids.to(dev))
    last, pooled = out.last_hidden_state, out.pooler_output
    N, L = ids.shape
    assert last.shape == (N, L, cfg.hidden_size) and pooled.shape == (N, cfg.hidden_size) and last.dtype == m.dtype
    assert out[0] is last and out.to_tuple()[1] is pooled and out.hidden_states is None and out.attentions is None
    ref_last, ref_pooled = clip_text_forward(sd32, cfg, ids.to(dev))
    _record(f"clip_text_{name}_last_hidden_state_vs_oracle", _rel(last, ref_last), bound)
    _record(f"clip_text_{name}_pooler_output_vs_oracle", _rel(pooled, ref_pooled), bound)
    if e is not None:
        _record(f"clip_text_{name}_last_hidden_state_vs_transformers", _rel(last.cpu()[:, e["rows"]], e["last_hidden_state"]), bound)
        _record(f"clip_text_{name}_pooler_output_vs_transformers", _rel(pooled.cpu(), e["pooler_output"]), bound)
    return last, pooled


@pytest.mark.parametrize("out_dtype", [torch.float16, torch.float32], ids=["out16", "out32"])
@pytest.mark.parametrize("tag", ["narrow", "full"])
def test_engine_vs_oracle_and_transformers_fixture(built_lib, tag, out_dtype):
    meta, configs = _fixture(tag)
    for name, e in configs.items():
        cfg = ClipTextConfig(**e["config"])
        m, sd32 = _model(cfg, meta["weight_seed"], dtype=out_dtype)
        ids = make_input_ids(len(e["lengths"]), e["L"], cfg, seed=meta["input_seed"], lengths=e["lengths"])
        _check_against(tag, f"{name}_{'out16' if out_dtype == torch.float16 else 'out32'}", m, sd32, cfg, ids, e)


@pytest.mark.parametrize("name", ["a_quick_gelu_d64", "b_gelu_d40"])
def test_causality_bit_exact(built_lib, name):
    """Changing token j leaves rows < j of last_hidden_state bitwise unchanged (and changes row j)."""
    _, configs = _fixture("narrow")
    e = configs[name]
    cfg = ClipTextConfig(**e["config"])
    m, _ = _model(cfg, 3, dtype=torch.float16)
    ids = make_input_ids(2, e["L"], cfg, seed=8, lengths=[e["L"] - 2, e["L"] // 2])
    a = m(ids.to(dev)).last_hidden_state.clone()
    for j in (1, e["L"] // 2, e["L"] - 1):
        y = ids.clone()
        y[:, j] = (y[:, j] + 1) % cfg.vocab_size
        b = m(y.to(dev)).last_hidden_state
        assert torch.equal(a[:, :j], b[:, :j]), j
        assert not torch.equal(a[:, j], b[:, j]), j


def test_sequences_are_independent(built_lib):
    """Perturbing sequence 1 of 3 leaves sequences 0 and 2 bitwise unchanged; one sequence alone equals itself in a batch
    (SD-1.5, 77 tokens: the 128-row query / key tiles straddle sequences)."""
    cfg = ClipTextConfig()
    m, _ = _model(cfg, 3, dtype=torch.float16)
    ids = make_input_ids(3, 77, cfg, seed=9, lengths=[10, 60, 75]).to(dev)
    a = m(ids)
    a = (a.last_hidden_state.clone(), a.pooler_output.clone())
    y = ids.clone()
    y[1, 1:40] = torch.flip(y[1, 1:40], dims=(0,))
    b = m(y)
    for k in (0, 2):
        assert torch.equal(a[0][k], b.last_hidden_state[k]) and torch.equal(a[1][k], b.pooler_output[k]), k
    assert not torch.equal(a[0][1], b.last_hidden_state[1])
    one = m(ids[2:3])
    assert torch.equal(one.last_hidden_state[0], a[0][2]) and torch.equal(one.pooler_output[0], a[1][2])


@pytest.mark.parametrize("outliers", [0, 4])
def test_fp16_yardstick_full(built_lib, outliers):
    """The engine's rms distance to the fp32 oracle is no larger than that of the oracle run as eager fp16 ("ref16", the way
    the reference runs this model) on the same GPU, with and without residual outlier channels. 24 sequences, so that the
    pooled rows (one per sequence) are enough samples for an rms."""
    from oracle.clip_text_oracle import clip_text_forward
    cfg = ClipTextConfig()
    m, sd32 = _model(cfg, 7, outlier_channels=outliers, dtype=torch.float32)
    ids = make_input_ids(24, 77, cfg, seed=77).to(dev)
    out = m(ids)
    ref_last, ref_pooled = clip_text_forward(sd32, cfg, ids)
    r16_last, r16_pooled = clip_text_forward(sd32, cfg, ids, dtype=torch.float16)
    if outliers:
        assert out.last_hidden_state.abs().max().item() > 2.0
    for what, got, r16, ref in (("last_hidden_state", out.last_hidden_state, r16_last, ref_last),
                                ("pooler_output", out.pooler_output, r16_pooled, ref_pooled)):
        e, e16 = _rms(got, ref), _rms(r16, ref)
        _record(f"clip_text_full_outliers{outliers}_{what}_rms_engine_over_ref16", e / e16, 1.0 + 1e-9)


def test_prompt_chunks_to_unet_chain(built_lib):
    """encode_weighted_prompt's shape of work (musev/utils/text_emb_util.py:352-420): 3 chunks x 77 tokens for the prompt
    and for the negative prompt -> engine text encoder -> [2, 231, C] encoder_hidden_states -> engine UNet (narrow), against
    the same chain on the oracles."""
    from musev_b200.unet import UNet3DConditionModel
    from musev_b200.synth import make_inputs
    from oracle.unet3d_oracle import UNet3DOracle
    from oracle.clip_text_oracle import clip_text_forward
    _, configs = _fixture("narrow")
    tcfg = ClipTextConfig(**configs["a_quick_gelu_d64"]["config"])
    text, tsd32 = _model(tcfg, 5, dtype=torch.float16)
    ids = make_input_ids(6, 77, tcfg, seed=31, lengths=[75, 75, 20, 30, 0, 0]).to(dev)   # cond chunks, then uncond chunks
    C_ = tcfg.hidden_size

    def chain_emb(last):
        # chunks of one prompt are concatenated along the tokens (text_emb_util.py:396-410); weights all 1 here
        return last.reshape(2, 3 * 77, C_)
    emb = chain_emb(text(ids)[0])
    ref_emb = chain_emb(clip_text_forward(tsd32, tcfg, ids)[0])
    _record("clip_text_chain_encoder_hidden_states_vs_oracle", _rel(emb, ref_emb), TOL["narrow"])
    cfg = preset_config("musev", block_out_channels=(64, 128, 128, 128), cross_attention_dim=C_)
    sd16 = {k: v.half() for k, v in make_state_dict(cfg, seed=0).items()}
    unet = UNet3DConditionModel(cfg, device=dev, dtype=torch.float32)
    unet.load_state_dict({k: v.to(dev) for k, v in sd16.items()})
    oracle = UNet3DOracle(cfg, {k: v.float() for k, v in sd16.items()}, device=dev)
    inp = make_inputs(cfg, batch=2, frames=4, h=16, w=16, n_vis_cond=1, seed=12)
    kw = dict(sample_index=inp["sample_index"], vision_conditon_frames_sample_index=inp["vision_conditon_frames_sample_index"],
              sample_frame_rate=10)
    dkw = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in kw.items()}
    out = unet(inp["sample"].to(dev), torch.tensor(601), emb, **dkw).sample
    ref = oracle(inp["sample"], 601, ref_emb.float().cpu(), **kw)
    _record("clip_text_chain_unet_out_vs_oracle", _rel(out, ref), CHAIN_UNET_TOL)


# ------------------------------------------------------------------------------------------------ LoRA
def _ordered(t):
    i = t.contiguous().view(torch.int16).to(torch.int32)
    return torch.where(i < 0, -(i + 32768), i)


def _bits_rule(got, want):
    d = (_ordered(got) - _ordered(want.to(got.device))).abs()
    return (d > 0).float().mean().item(), int(d.max().item())


class _NoUnet:
    """Stands in for pipeline.unet when only text-encoder keys are merged."""

    def __init__(self):
        self.cfg, self.device = preset_config("musev", block_out_channels=(64, 128, 128, 128)), torch.device(dev)

    def _merge_lora(self, *a, **k):
        pass


def test_text_lora_merge_unload_vs_arithmetic(built_lib):
    from musev_b200 import lora
    from musev_b200.schema import kohya_text_name_map
    cfg = ClipTextConfig(vocab_size=1000, hidden_size=128, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2)
    m, sd32 = _model(cfg, 4, dtype=torch.float16)
    names = kohya_text_name_map(cfg)
    tt = [("text_model_encoder_layers_0_self_attn_q_proj", 128, 128), ("text_model_encoder_layers_0_self_attn_v_proj", 128, 128),
          ("text_model_encoder_layers_1_mlp_fc1", 512, 128), ("text_model_encoder_layers_1_mlp_fc2", 128, 512),
          ("text_model_encoder_layers_1_self_attn_out_proj", 128, 128)]
    mods = [t[0] for t in tt]
    lsd = make_lora_state_dict(preset_config("musev", block_out_channels=(64, 128, 128, 128)), [], rank=8, seed=3,
                               text_targets=tt)
    pipe = SimpleNamespace(unet=_NoUnet(), text_encoder=m)
    before = {names[k]: m.debug_weight(names[k]).clone() for k in mods}
    _, undo = lora.update_pipeline_lora_model(pipe, lsd, alpha=0.7, lora_block_weight_str="FACE", need_unload=True)
    assert len(undo) == len(mods)
    worst, applied, deltas = 0.0, {}, {}
    for t in lora.pair_keys(lsd):
        name = names[t.module[len("lora_te_"):]]
        up, down, r = lora.factors(lsd, t)
        delta = lora.text_delta(up, down, lora.target_scale(lsd, t, 0.7, r), 1.0)
        want = (before[name].cpu() + delta).half()
        applied[name], deltas[name] = want, delta
        frac, ulp = _bits_rule(m.debug_weight(name), want)
        assert ulp <= 1, (name, ulp)
        worst = max(worst, frac)
    _record("clip_text_lora_apply_frac_differing", worst, 1e-3)
    lora.unload_lora(undo)
    for n in before:   # the reference's unload subtracts the same delta16; it does not promise the original bits
        frac, ulp = _bits_rule(m.debug_weight(n), (applied[n] - deltas[n]).half())
        assert ulp <= 1, (n, ulp)
        worst = max(worst, frac)
    _record("clip_text_lora_unload_frac_differing", worst, 1e-3)
    untouched = [n for n in kohya_text_name_map(cfg).values() if n not in before]
    sd16 = {k: v.half() for k, v in make_clip_text_state_dict(cfg, seed=4).items()}
    for n in untouched:
        assert torch.equal(m.debug_weight(n).cpu(), sd16[n]), n


def test_text_lora_matches_reference_sha256(built_lib):
    """The reference's own merge (tests/golden/lora_narrow.pt, musev.utils.model_util on a torch text encoder) reproduced
    bit for bit on an engine text encoder holding the same k_proj weight: apply (ALL, FACE) and apply + unload."""
    from musev_b200 import lora
    from musev_b200.clip_text import CLIPTextModel
    g = torch.load(os.path.join(GOLDEN, "lora_narrow.pt"))
    meta = g["meta"]
    W = meta["text_width"]
    kproj = make_text_encoder(W, meta["text_seed"]).text_model.encoder.layers[0].self_attn.k_proj.weight.data
    cfg = ClipTextConfig(vocab_size=64, hidden_size=W, intermediate_size=64, num_hidden_layers=1, num_attention_heads=1)
    sd = {k: v.half() for k, v in make_clip_text_state_dict(cfg, seed=0).items()}
    sd[meta["text_weight"]] = kproj
    ucfg = preset_config(meta["preset"], block_out_channels=tuple(meta["block_out_channels"]))
    lsd = make_lora_state_dict(ucfg, [], rank=meta["rank"], seed=meta["lora_seed"], amp=meta["amp"],
                               no_alpha=meta["no_alpha"], f32=meta["f32"], text_targets=[tuple(t) for t in meta["text_targets"]])
    from oracle.lora_oracle import sha256
    for case, block, unload in (("all", "ALL", False), ("face", "FACE", False), ("unload", "ALL", True)):
        m = CLIPTextModel.from_state_dict(sd, cfg, device=dev)
        pipe = SimpleNamespace(unet=_NoUnet(), text_encoder=m)
        _, undo = lora.update_pipeline_lora_model(pipe, lsd, alpha=meta["strength"], lora_block_weight_str=block,
                                                  need_unload=True)
        if unload:
            lora.unload_lora(undo)
        got = m.debug_weight(meta["text_weight"]).cpu()
        assert sha256(got) == g[f"sha256_{case}"][meta["text_weight"]], (case, _bits_rule(got, kproj))


def test_lora_still_rejects_other_kinds(built_lib):
    from musev_b200._capi import MvbNamedTensor, _named, lib
    from musev_b200.controlnet import ControlNetModel
    from musev_b200.schema import ControlNetConfig
    cn = ControlNetModel(ControlNetConfig(block_out_channels=(64, 128, 128, 128)), device=dev)
    up, down = torch.zeros(64, 4, device=dev).half(), torch.zeros(4, 64, device=dev).half()
    a = "down_blocks.0.attentions.0.proj_out.weight"
    arr_u, arr_d = (MvbNamedTensor * 1)(_named(a, up)), (MvbNamedTensor * 1)(_named(a, down))
    assert lib().mvb_unet_merge_lora(cn._h, arr_u, arr_d, (C.c_float * 1)(1.0), 1, 0) == -3


# ------------------------------------------------------------------------------------------------ rejections
def test_rejections_before_any_launch(built_lib):
    from musev_b200 import _capi
    from musev_b200._capi import MvbControlnetArgs
    from musev_b200.clip_text import CLIPTextModel
    _, configs = _fixture("narrow")
    cfg = ClipTextConfig(**configs["a_quick_gelu_d64"]["config"])
    sd = {k: v.half() for k, v in make_clip_text_state_dict(cfg, seed=1).items()}
    empty = CLIPTextModel(cfg, device=dev)
    with pytest.raises(RuntimeError, match="weights not loaded"):
        empty(torch.zeros(1, 77, dtype=torch.long, device=dev))
    missing = dict(sd)
    del missing["text_model.encoder.layers.1.mlp.fc1.bias"]
    with pytest.raises(KeyError, match="layers.1.mlp.fc1.bias"):
        CLIPTextModel.from_state_dict(missing, cfg, device=dev)
    m = CLIPTextModel.from_state_dict({**sd, "text_model.embeddings.position_ids": torch.arange(77).unsqueeze(0)}, cfg,
                                      device=dev)
    ids = make_input_ids(2, 77, cfg, seed=3).to(dev)
    n0 = _capi.launch_count()
    bad_ids = ids.clone()
    bad_ids[1, 5] = cfg.vocab_size
    with pytest.raises(IndexError):
        m(bad_ids)
    bad_ids[1, 5] = -1
    with pytest.raises(IndexError):
        m(bad_ids)
    with pytest.raises(ValueError, match="max_position_embeddings"):
        m(torch.zeros(1, 78, dtype=torch.long, device=dev))
    mask = torch.ones_like(ids)
    mask[0, 50:] = 0
    with pytest.raises(NotImplementedError):
        m(ids, attention_mask=mask)
    with pytest.raises(NotImplementedError):
        m(ids, output_hidden_states=True)
    with pytest.raises(NotImplementedError):
        m(ids, position_ids=torch.arange(77, device=dev).unsqueeze(0))
    for bad in (ids.float(), ids[0]):
        with pytest.raises(ValueError):
            m(bad)
    assert _capi.launch_count() == n0
    # the C entry point: float ids, n_out, no output -- negative return and the handle's message, no launch
    l = _capi.lib()
    last = torch.zeros(2, 77, cfg.hidden_size, device=dev)
    ws = torch.empty(64 << 20, dtype=torch.uint8, device=dev)
    for f32, n_out, out0, H in ((1, 2, last, 77), (0, 1, last, 77), (0, 2, None, 77), (0, 2, last, 78)):
        a = MvbControlnetArgs()
        a.sample, a.sample_is_f32, a.NF, a.H, a.W, a.n_out, a.out_is_f32 = ids.data_ptr(), f32, 2, H, 1, n_out, 1
        a.outs[0] = out0.data_ptr() if out0 is not None else None
        assert l.mvb_clip_text_workspace_bytes(m._h, C.byref(a)) < 0
        assert l.mvb_clip_text_forward(m._h, C.byref(a), ws.data_ptr(), ws.numel(), None) < 0
        assert l.mvb_handle_error(m._h).decode().startswith("clip text:")
    assert _capi.launch_count() == n0
    cfg_bad = _capi.make_config(0, 2, (128, 512, 77, 1000), layers_per_block=2, heads=2, norm_num_groups=4, norm_eps=1e-5)
    h = C.c_void_p()
    assert l.mvb_create_clip_text(C.byref(cfg_bad), 0, C.byref(h)) < 0           # unknown activation code
    # all-ones mask and any integer dtype are accepted; return_dict=False gives the tuple
    out = m(ids.int(), attention_mask=torch.ones_like(ids), return_dict=False)
    assert isinstance(out, tuple) and len(out) == 2 and out[0].dtype == torch.float16
    assert torch.equal(out[0], m(ids)[0])
