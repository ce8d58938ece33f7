#!/usr/bin/env python
"""Runs every model kind of the engine on seeded weights and inputs (musev_b200.synth) with the library given by --lib,
and saves, per call, the outputs, the workspace bytes the call asked for and the number of kernel launches it made
(`mvb_launch_count`). Two libraries that compute the same thing give bit-identical files; `--compare A B` reports, for
two such output directories, every output that differs, every launch count that differs and every workspace that grew.

  python tools/gpu_compare_builds.py --lib musev_b200/_lib/libmusevb200.so --out /tmp/new
  python tools/gpu_compare_builds.py --compare /tmp/old /tmp/new

The calls: the UNet (both presets, narrow and full width, with ControlNet residuals, reference embeddings and
`pose_guider_emb`), the ControlNet, the ReferenceNet, VAE decode and encode, the PoseGuider (both configurations), a
LoRA merge, forward and unload on the UNet, the CLIP vision tower (two narrow configurations and ViT-H/14) and, with a
library that has it, the CLIP text encoder (two narrow configurations and SD-1.5)."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

dev = "cuda"
NARROW, FULL = (64, 128, 128, 128), (320, 640, 1280, 1280)


def _dev(v):
    if torch.is_tensor(v):
        return v.to(dev) if v.is_floating_point() else v
    if isinstance(v, list):
        return [_dev(x) for x in v]
    return v


class Recorder:
    def __init__(self):
        from musev_b200 import _capi
        self.capi, self.results = _capi, {}

    def __call__(self, name, model, fn):
        torch.cuda.synchronize()
        n0 = self.capi.launch_count()
        out = fn()
        torch.cuda.synchronize()
        outs = [t.detach().cpu().clone() for t in (out if isinstance(out, (list, tuple)) else [out])]
        self.results[name] = {"outputs": outs, "launches": self.capi.launch_count() - n0,
                              "workspace": model._ws.numel() if model is not None and model._ws is not None else 0}
        print(name, self.results[name]["launches"], self.results[name]["workspace"], flush=True)


def _unet_calls(rec):
    from musev_b200.schema import preset_config
    from musev_b200.synth import make_inputs, make_pose_guider_emb, make_state_dict
    from musev_b200.unet import UNet3DConditionModel
    B, frames, h, w = 2, 3, 16, 16
    for preset in ("musev", "musev_referencenet"):
        for tag, boc in (("narrow", NARROW), ("full", FULL)):
            cfg = preset_config(preset, block_out_channels=boc)
            model = UNet3DConditionModel(cfg, device=dev, dtype=torch.float32)
            model.load_state_dict({k: v.to(dev) for k, v in make_state_dict(cfg, seed=0, dtype=torch.float16).items()})
            inp = make_inputs(cfg, batch=B, frames=frames, h=h, w=w, n_vis_cond=1, seed=7)
            NF = B * (frames + 1)
            g = torch.Generator().manual_seed(3)
            maps, ds = [(boc[0], 1)], 1
            for i, ch in enumerate(boc):
                maps += [(ch, ds)] * cfg.layers_per_block
                if i != len(boc) - 1:
                    ds *= 2
                    maps.append((ch, ds))
            down = [torch.randn(NF, c, h // s, w // s, generator=g) * 0.1 for c, s in maps]
            mid = torch.randn(NF, boc[-1], h // ds, w // ds, generator=g) * 0.1
            kw = dict(sample_index=inp["sample_index"], vision_conditon_frames_sample_index=inp["vision_conditon_frames_sample_index"],
                      sample_frame_rate=8, down_block_refer_embs=inp.get("down_block_refer_embs"),
                      mid_block_refer_emb=inp.get("mid_block_refer_emb"), vision_clip_emb=inp.get("vision_clip_emb"),
                      down_block_additional_residuals=down, mid_block_additional_residual=mid,
                      pose_guider_emb=make_pose_guider_emb(NF, boc[0], h, w, seed=11))
            kw = {k: _dev(v) for k, v in kw.items()}
            rec(f"unet_{preset}_{tag}", model,
                lambda: model(inp["sample"].to(dev), 601, inp["encoder_hidden_states"].to(dev), **kw).sample)


def _encoder_calls(rec):
    from musev_b200.controlnet import ControlNetModel
    from musev_b200.referencenet import ReferenceNet2D
    from musev_b200.schema import ControlNetConfig, ReferenceNetConfig
    from musev_b200.synth import make_controlnet_inputs, make_referencenet_inputs, make_state_dict
    for tag, boc in (("narrow", NARROW), ("full", FULL)):
        cfg = ControlNetConfig(block_out_channels=boc)
        cn = ControlNetModel(cfg, device=dev, dtype=torch.float32)
        cn.load_state_dict({k: v.to(dev) for k, v in make_state_dict(cfg, seed=1, dtype=torch.float16).items()})
        inp = make_controlnet_inputs(cfg, frames=4, h=16, w=16)
        cond = torch.randn(4, boc[0], 16, 16, generator=torch.Generator().manual_seed(5)).to(dev)
        rec(f"controlnet_{tag}", cn, lambda: (lambda down, mid: down + [mid])(
            *cn(inp["sample"].to(dev), 601, inp["encoder_hidden_states"].to(dev), controlnet_cond_latents=cond, return_dict=False)))
        rcfg = ReferenceNetConfig(block_out_channels=boc)
        rn = ReferenceNet2D(rcfg, device=dev, dtype=torch.float32)
        rn.load_state_dict({k: v.to(dev) for k, v in make_state_dict(rcfg, seed=2, dtype=torch.float16).items()})
        rinp = make_referencenet_inputs(rcfg, batch=2, n_ref=1, h=16, w=16)
        rec(f"referencenet_{tag}", rn, lambda: (lambda r: r[0] + [r[1]])(
            rn(rinp["sample"].to(dev), 0, rinp["encoder_hidden_states"].to(dev), num_frames=rinp["num_frames"])))


def _vae_calls(rec):
    from musev_b200.schema import VAEConfig
    from musev_b200.synth import make_state_dict, make_vae_images
    from musev_b200.vae import AutoencoderKLDecoder, AutoencoderKLEncoder
    for tag, boc in (("narrow", (64, 64, 128, 128)), ("full", (128, 256, 512, 512))):
        cfg = VAEConfig(block_out_channels=boc)
        sd = {k: v.to(dev) for k, v in make_state_dict(cfg, seed=3, dtype=torch.float16).items()}
        dec = AutoencoderKLDecoder(cfg, device=dev, dtype=torch.float32, frames_per_call=2)
        dec.load_state_dict(sd)
        z = torch.randn(1, 4, 3, 32, 32, generator=torch.Generator().manual_seed(9)).to(dev)
        rec(f"vae_decode_{tag}", dec, lambda: dec.decode_latents(z))
        enc = AutoencoderKLEncoder(cfg, device=dev, dtype=torch.float32, frames_per_call=2)
        enc.load_state_dict(sd)
        x = make_vae_images(3, 256, 256).to(dev)
        rec(f"vae_encode_{tag}", enc, lambda: enc.encode(x).latent_dist.parameters)


def _pose_guider_calls(rec):
    from musev_b200.controlnet import PoseGuider
    from musev_b200.schema import PoseGuiderConfig
    from musev_b200.synth import make_pose_guider_state_dict, make_pose_images
    for cfg in (PoseGuiderConfig(64, 3, (16, 32, 64, 128)), PoseGuiderConfig(320, 3, (16, 32, 96, 256))):
        pg = PoseGuider(cfg.conditioning_embedding_channels, cfg.conditioning_channels, cfg.block_out_channels, device=dev,
                        dtype=torch.float32, frames_per_call=2)
        pg.load_state_dict({k: v.to(dev) for k, v in make_pose_guider_state_dict(cfg, seed=4, dtype=torch.float16).items()})
        x = make_pose_images(3, 256, 256).to(dev)
        rec(f"pose_guider_{cfg.block_out_channels[2]}", pg, lambda: pg.embed_frames(x))


def _lora_calls(rec):
    from musev_b200.schema import preset_config, unet_param_shapes
    from musev_b200.synth import make_inputs, make_lora_state_dict, make_state_dict
    from musev_b200.unet import UNet3DConditionModel
    cfg = preset_config("musev_referencenet", block_out_channels=NARROW)
    model = UNet3DConditionModel(cfg, device=dev, dtype=torch.float32)
    model.load_state_dict({k: v.to(dev) for k, v in make_state_dict(cfg, seed=0, dtype=torch.float16).items()})
    targets = [n for n, s in unet_param_shapes(cfg).items() if len(s) in (2, 4)]
    lsd = make_lora_state_dict(cfg, targets, rank=8, seed=9)
    ups, downs, scales = [], [], []
    for n in targets:
        mod = "lora_unet_" + n[:-7].replace(".", "_")
        ups.append(lsd[mod + ".lora_up.weight"].to(dev).contiguous())
        downs.append(lsd[mod + ".lora_down.weight"].to(dev).contiguous())
        scales.append(0.5)
    probe = targets[::7]
    rec("lora_merge", None, lambda: (model._merge_lora(targets, ups, downs, scales), [model.debug_weight(n) for n in probe])[1])
    inp = make_inputs(cfg, batch=2, frames=3, h=8, w=8, n_vis_cond=1, seed=8)
    kw = {k: _dev(inp.get(k)) for k in ("down_block_refer_embs", "mid_block_refer_emb", "vision_clip_emb")}
    rec("lora_forward", model, lambda: model(inp["sample"].to(dev), 301, inp["encoder_hidden_states"].to(dev),
                                             sample_index=inp["sample_index"],
                                             vision_conditon_frames_sample_index=inp["vision_conditon_frames_sample_index"],
                                             **kw).sample)
    rec("lora_unload", None,
        lambda: (model._merge_lora(targets, ups, downs, scales, subtract=True), [model.debug_weight(n) for n in probe])[1])


def _clip_vision_calls(rec):
    from musev_b200.clip_vision import CLIPVisionModelWithProjection
    from musev_b200.schema import ClipVisionConfig
    from musev_b200.synth import make_clip_pixel_values, make_clip_vision_state_dict
    for tag, cfg, n in (("d64", ClipVisionConfig(hidden_size=128, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2,
                                                 image_size=56, patch_size=14, projection_dim=64), 3),
                        ("d40", ClipVisionConfig(hidden_size=320, intermediate_size=640, num_hidden_layers=2, num_attention_heads=8,
                                                 image_size=56, patch_size=14, projection_dim=64, hidden_act="quick_gelu"), 2),
                        ("vit_h14", ClipVisionConfig(), 2)):
        sd = {k: v.half() for k, v in make_clip_vision_state_dict(cfg, seed=6).items()}
        m = CLIPVisionModelWithProjection.from_state_dict(sd, cfg, device=dev, dtype=torch.float16)
        x = make_clip_pixel_values(n, cfg.image_size, seed=6).to(dev)
        rec(f"clip_vision_{tag}", m, lambda: m(x).to_tuple())


def _clip_text_calls(rec):
    from musev_b200.clip_text import CLIPTextModel
    from musev_b200.schema import ClipTextConfig
    from musev_b200.synth import make_clip_text_state_dict, make_input_ids
    for tag, cfg, n, L in (("d64", ClipTextConfig(vocab_size=1000, hidden_size=128, intermediate_size=512, num_hidden_layers=2,
                                                  num_attention_heads=2), 3, 77),
                           ("d40", ClipTextConfig(vocab_size=1000, hidden_size=320, intermediate_size=640, num_hidden_layers=2,
                                                  num_attention_heads=8, max_position_embeddings=160, hidden_act="gelu",
                                                  bos_token_id=6, eos_token_id=7), 2, 150),
                           ("sd15", ClipTextConfig(), 6, 77)):
        sd = {k: v.half() for k, v in make_clip_text_state_dict(cfg, seed=6).items()}
        m = CLIPTextModel.from_state_dict(sd, cfg, device=dev, dtype=torch.float16)
        ids = make_input_ids(n, L, cfg, seed=6).to(dev)
        rec(f"clip_text_{tag}", m, lambda: m(ids).to_tuple())


class _Missing:
    def __init__(self, name):
        self.name = name

    def __call__(self, *args):
        raise AttributeError(f"{self.name} is not exported by this library")


class _TolerantLib:
    """A library handle on which entry points a build does not export can still be declared (they raise when called), so
    that an older library runs the calls it has."""

    def __init__(self, path):
        import ctypes
        self._l = ctypes.CDLL(path)

    def __getattr__(self, name):
        try:
            return getattr(self._l, name)
        except AttributeError:
            setattr(self, name, _Missing(name))
            return getattr(self, name)


def run(lib_path: str, out_dir: str) -> None:
    from musev_b200 import _capi
    _capi.LIB_PATH = os.path.abspath(lib_path)
    tl = _TolerantLib(_capi.LIB_PATH)
    _capi._declare(tl)
    _capi._lib = tl
    rec = Recorder()
    calls = [_unet_calls, _encoder_calls, _vae_calls, _pose_guider_calls, _lora_calls, _clip_vision_calls]
    if hasattr(tl._l, "mvb_create_clip_text"):      # libraries before mvb_version 4 have no CLIP text handle
        calls.append(_clip_text_calls)
    for c in calls:
        c(rec)
    os.makedirs(out_dir, exist_ok=True)
    torch.save(rec.results, os.path.join(out_dir, "results.pt"))


def compare(a_dir: str, b_dir: str) -> dict:
    a = torch.load(os.path.join(a_dir, "results.pt"))
    b = torch.load(os.path.join(b_dir, "results.pt"))
    report = {"calls": len(a), "missing": sorted(set(a) ^ set(b)), "outputs_differ": {}, "launches_differ": {},
              "workspace_grew": {}, "workspace_shrank": {}}
    for name in sorted(set(a) & set(b)):
        ra, rb = a[name], b[name]
        diff = [i for i, (x, y) in enumerate(zip(ra["outputs"], rb["outputs"]))
                if x.shape != y.shape or x.dtype != y.dtype or not torch.equal(x.view(torch.uint8), y.view(torch.uint8))]
        if diff or len(ra["outputs"]) != len(rb["outputs"]):
            report["outputs_differ"][name] = {str(i): (ra["outputs"][i].float() - rb["outputs"][i].float()).abs().max().item()
                                              for i in diff}
        if ra["launches"] != rb["launches"]:
            report["launches_differ"][name] = [ra["launches"], rb["launches"]]
        if rb["workspace"] > ra["workspace"]:
            report["workspace_grew"][name] = [ra["workspace"], rb["workspace"]]
        elif rb["workspace"] < ra["workspace"]:
            report["workspace_shrank"][name] = [ra["workspace"], rb["workspace"]]
    return report


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", help="libmusevb200.so to run")
    ap.add_argument("--out", help="directory for results.pt")
    ap.add_argument("--compare", nargs=2, metavar=("A", "B"), help="compare two output directories")
    args = ap.parse_args()
    if args.compare:
        print(json.dumps(compare(*args.compare)), flush=True)
    elif args.lib and args.out:
        run(args.lib, args.out)
    else:
        ap.error("give --lib and --out, or --compare A B")


if __name__ == "__main__":
    main()
