"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/multicontrolnet_narrow.pt by running the UNMODIFIED reference on CPU in
fp32: diffusers `MultiControlNetModel` (diffusers/src/diffusers/pipelines/controlnet/multicontrolnet.py:15-72) over
`ControlNetModel`s of the vendored fork, and a denoise loop with two of them around the imported UNet.

Needs the reference tree (oracle/ref_shim.py):  python -m oracle.make_golden_multicontrolnet
Weights and inputs are regenerated from the seeds in the fixture's meta (musev_b200.synth, bit-identical CPU RNG). The
reference is never read at test time.

  * "two", "three_guess": one MultiControlNetModel call each, the way `get_controlnet_emb` issues it
    (musev/pipelines/pipeline_controlnet.py:1253-1262) in the multi-net branch: a list of control images and a list of
    scales, `controlnet_cond_latents` None, so every net embeds its own image. 128 seeded sample positions per map.
  * "loop": the window loop of make_golden.golden_loop (pipeline_controlnet.py:1846-2117, restated) with two imported
    ControlNets. The control images are sliced per window (:1969-1982) and every net embeds its slice on every
    window-step, which is what the engine's "embed once per call, slice per window" must reproduce. Final latents.
"""
from __future__ import annotations

import importlib.util
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from musev_b200.schema import ControlNetConfig, controlnet_param_shapes, preset_config  # noqa: E402
from musev_b200.synth import make_controlnet_inputs, make_inputs, make_state_dict  # noqa: E402
from oracle import ref_shim  # noqa: E402
from oracle.make_golden import NARROW, build_reference  # noqa: E402
from oracle.pipeline_oracle import SD15_DDIM  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
CASES = {
    "two": dict(weight_seeds=[3, 13], image_seeds=[4401, 4402], scales=[0.7, 1.3], guess_mode=False, frames=3, h=8, w=8,
                timestep=601, input_seed=4321),
    "three_guess": dict(weight_seeds=[3, 13, 23], image_seeds=[4411, 4412, 4413], scales=[1.0, 0.8, 0.5], guess_mode=True,
                        frames=2, h=8, w=8, timestep=301, input_seed=4322),
}
LOOP = dict(weight_seed=0, cn_weight_seeds=[3, 13], image_seed=5511, scales=[0.9, 0.6], T=16, h=8, w=8, steps=2,
            input_seed=77, context_frames=8, context_overlap=2, guidance_scale=3.5)
N_SAMPLES, SAMPLE_SEED_BASE = 128, 1000


def reference_controlnet(boc, seed):
    """The vendored diffusers ControlNetModel with SD-1.5's layout (as make_golden.golden_controlnet builds it)."""
    from diffusers.models.controlnet import ControlNetModel
    cfg = ControlNetConfig(block_out_channels=tuple(boc))
    kw = dict(in_channels=4, conditioning_channels=3, block_out_channels=tuple(boc), layers_per_block=2,
              cross_attention_dim=768, attention_head_dim=8, norm_num_groups=32,
              down_block_types=("CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "DownBlock2D"))
    with torch.device("meta"):
        m = ControlNetModel(**kw)
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == \
        {k: tuple(v) for k, v in controlnet_param_shapes(cfg).items()}, "ControlNet schema mismatch vs reference state_dict"
    m = m.to_empty(device="cpu")
    res = m.load_state_dict(make_state_dict(cfg, seed=seed), strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    return m.eval()


def control_images(n, h, w, seed):
    """n control images of 8x the latent size, values in [0, 1) (the prepared control image's range)."""
    return make_controlnet_inputs(ControlNetConfig(block_out_channels=NARROW), frames=n, h=h, w=w, seed=seed)["controlnet_cond"]


def golden_case(tag):
    from diffusers.pipelines.controlnet.multicontrolnet import MultiControlNetModel
    c = CASES[tag]
    t0 = time.time()
    multi = MultiControlNetModel([reference_controlnet(NARROW, s) for s in c["weight_seeds"]])
    inp = make_controlnet_inputs(ControlNetConfig(block_out_channels=NARROW), frames=c["frames"], h=c["h"], w=c["w"],
                                 seed=c["input_seed"])
    images = [control_images(c["frames"], c["h"], c["w"], s) for s in c["image_seeds"]]
    with torch.no_grad():
        down, mid = multi(inp["sample"], torch.tensor(c["timestep"]), inp["encoder_hidden_states"], controlnet_cond=images,
                          conditioning_scale=list(c["scales"]), guess_mode=c["guess_mode"], return_dict=False)
    maps = list(down) + [mid]
    samples, stats = [], []
    for k, mp in enumerate(maps):
        flat = mp.reshape(-1)
        idx = torch.randint(0, flat.numel(), (N_SAMPLES,), generator=torch.Generator().manual_seed(SAMPLE_SEED_BASE + k))
        samples.append(flat[idx].clone())
        stats.append([float(flat.mean()), float(flat.abs().mean())])
    print(f"{tag}: mid abs-mean {stats[-1][1]:.4f} ({time.time() - t0:.1f}s)", flush=True)
    return dict(meta=dict(c, block_out_channels=list(NARROW), shapes=[list(mp.shape) for mp in maps], n_samples=N_SAMPLES,
                          sample_seed_base=SAMPLE_SEED_BASE),
                samples=samples, stats=stats)


def golden_loop():
    """make_golden.golden_loop with the reference's Multi-ControlNet branch in every window-step."""
    from diffusers.pipelines.controlnet.multicontrolnet import MultiControlNetModel
    L = LOOP
    _, DDIM = ref_shim.load()
    spec = importlib.util.spec_from_file_location(
        "mmcm.utils.itertools_util", os.path.join(ref_shim.REFERENCE_ROOT, "MMCM/mmcm/utils/itertools_util.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    sys.modules["mmcm.utils.itertools_util"] = mod
    from musev.pipelines.context import prepare_global_context
    t0 = time.time()
    cfg = preset_config("musev", block_out_channels=NARROW)
    unet, cfg = build_reference("musev", NARROW, make_state_dict(cfg, seed=L["weight_seed"]))
    multi = MultiControlNetModel([reference_controlnet(NARROW, s) for s in L["cn_weight_seeds"]])
    T, h, w, steps = L["T"], L["h"], L["w"], L["steps"]
    sched = DDIM(**SD15_DDIM)
    sched.set_timesteps(steps)
    g = torch.Generator().manual_seed(L["input_seed"])
    latents = torch.randn(1, 4, T, h, w, generator=g)
    cond = torch.randn(1, 4, 1, h, w, generator=g) * 0.5
    prompt = torch.randn(2, 77, cfg.cross_attention_dim, generator=g)
    extra = make_inputs(cfg, batch=2, frames=1, h=h, w=w, seed=L["input_seed"])
    kw = {k: extra[k] for k in ("down_block_refer_embs", "mid_block_refer_emb", "vision_clip_emb") if k in extra}
    # one image per net and frame (vision-condition frame first), duplicated for CFG like prepare_control_image
    images = []
    for k in range(len(L["cn_weight_seeds"])):
        im = control_images(1 + T, h, w, L["image_seed"] + k)                               # [(1 + T), 3, 8h, 8w]
        im = im.permute(1, 0, 2, 3).unsqueeze(0)                                              # [1, 3, 1 + T, 8h, 8w]
        images.append(torch.cat([im] * 2))
    ctx = prepare_global_context("uniform_v2", steps, T, L["context_frames"], 1, L["context_overlap"], 1)
    vis_idx = torch.arange(1)
    with torch.no_grad():
        for t in sched.timesteps:
            noise_pred = torch.zeros(2, 4, T, h, w)
            counter = torch.zeros(1, 1, T, 1, 1)
            for context in ctx:
                c = context[0]
                sub = torch.arange(len(c)) + 1
                full = torch.zeros(2, 4, 1 + len(c), h, w)
                full[:, :, vis_idx] = torch.cat([cond] * 2)
                full[:, :, sub] = torch.cat([latents[:, :, c]] * 2)
                cctx = [0] + [ci + 1 for ci in c]                                             # :1955-1962
                imgs = [im[:, :, cctx].permute(0, 2, 1, 3, 4).reshape(-1, *im.shape[1:2], *im.shape[3:])
                        for im in images]                                                     # :1969-1982
                tc = full.shape[2]
                x2 = full.permute(0, 2, 1, 3, 4).reshape(2 * tc, 4, h, w)
                enc2 = prompt.repeat_interleave(tc, dim=0)
                down, mid = multi(x2, t, enc2, controlnet_cond=imgs, conditioning_scale=list(L["scales"]),
                                  guess_mode=False, return_dict=False)                       # :1253-1262
                eps = unet(full, t, prompt, sample_index=sub, vision_conditon_frames_sample_index=vis_idx,
                           sample_frame_rate=8, do_classifier_free_guidance=True, ip_adapter_scale=1.0,
                           down_block_additional_residuals=down, mid_block_additional_residual=mid, **kw)[0]
                noise_pred[:, :, c] += eps[:, :, sub]
                counter[:, :, c] += 1
            noise_pred = noise_pred / counter
            u, tx = noise_pred.chunk(2)
            noise_pred = u + L["guidance_scale"] * (tx - u)
            latents = sched.step(noise_pred, t, latents, eta=0.0).prev_sample
    print(f"loop: {len(ctx)} windows, final latents std {latents.std().item():.4f} ({time.time() - t0:.1f}s)", flush=True)
    return dict(meta=dict(L, block_out_channels=list(NARROW), preset="musev", contexts=[c[0] for c in ctx]),
                latents=latents.clone())


if __name__ == "__main__":
    os.makedirs(GOLDEN, exist_ok=True)
    torch.set_num_threads(os.cpu_count() or 1)
    ref_shim.load()
    out = {tag: golden_case(tag) for tag in CASES}
    out["loop"] = golden_loop()
    out["source"] = ("reference diffusers MultiControlNetModel over diffusers ControlNetModel (vendored fork) and the "
                     "imported musev UNet3DConditionModel + DDIMScheduler + prepare_global_context, CPU fp32")
    path = os.path.join(GOLDEN, "multicontrolnet_narrow.pt")
    torch.save(out, path)
    print(path, os.path.getsize(path), "bytes", flush=True)
