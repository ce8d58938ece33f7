"""musev_b200 -- H100 (sm_90a) denoising engine behind MuseV's UNet3DConditionModel / DDIMScheduler / pipeline API.

The compute path is the in-tree CUDA library (musev_b200/_lib/libmusevb200.so, built by musev_b200.build);
importing this package does not load it, using any op does -- and fails loudly if it is missing.
"""
from .schema import UNetConfig, preset_config, unet_param_shapes  # noqa: F401

__all__ = ["UNetConfig", "preset_config", "unet_param_shapes", "UNet3DConditionModel", "DDIMScheduler",
           "ParallelDenoiser", "CLIPVisionModelWithProjection", "CLIPTextModel"]


def __getattr__(name):
    if name == "UNet3DConditionModel":
        from .unet import UNet3DConditionModel
        return UNet3DConditionModel
    if name == "DDIMScheduler":
        from .scheduler import DDIMScheduler
        return DDIMScheduler
    if name == "ParallelDenoiser":
        from .pipeline import ParallelDenoiser
        return ParallelDenoiser
    if name == "CLIPVisionModelWithProjection":
        from .clip_vision import CLIPVisionModelWithProjection
        return CLIPVisionModelWithProjection
    if name == "CLIPTextModel":
        from .clip_text import CLIPTextModel
        return CLIPTextModel
    raise AttributeError(name)
