"""uav_b200 — H100-native (sm_90a) implementation of the Upscale-A-Video diffusion sampling path.

Public surface mirrors the reference (`/root/reference/models_video/`): `VideoUpscalePipeline`,
`UNetVideoModel`, `AutoencoderKLVideo`, `DDIMScheduler`, `Propagation`, `RAFT_bi` (models_video/RAFT/raft_bi.py) and the
`CLIPTextModel` the pipeline holds as `text_encoder`, plus `LLavaAgent` (llava/llava_agent.py), the LLaVA-1.5 captioner.  The arithmetic runs in
hand-written CUDA kernels behind a C ABI (`include/uav_b200.h`, `csrc/`); there is no CPU path.
"""
__version__ = "0.1.0"

_LAZY = {
    "VideoUpscalePipeline": "pipeline_upscale_a_video",
    "UNetVideoModel": "unet_video",
    "AutoencoderKLVideo": "autoencoder_kl_cond_video",
    "DDIMScheduler": "scheduling_ddim",
    "DDPMScheduler": "scheduling_ddim",
    "Propagation": "propagation_module",
    "RAFT": "raft",
    "RAFT_bi": "raft",
    "initialize_RAFT": "raft",
    "CLIPTextModel": "clip_text",
    "CLIPTextConfig": "clip_text",
    "LLavaAgent": "llava",
}


def __getattr__(name):
    if name in _LAZY:
        import importlib
        return getattr(importlib.import_module(f"{__name__}.{_LAZY[name]}"), name)
    raise AttributeError(name)
