"""Colour fix after the decode — the uav_b200 mirror of the reference's `models_video/color_correction.py`
(same function names and argument meaning, reference lines cited per function) plus the two steps the CLI wraps
around it (`inference_upscale_a_video.py:323-357`): bicubic x4 of the low-resolution frames and uint8 packing.

Everything runs in `csrc/postprocess.cu` on the reference's planar fp32 "t c h w" frames; there is no CPU path."""
from typing import Optional

import torch

from . import _lib, ops

__all__ = ["calc_mean_std", "adaptive_instance_normalization", "adain_color_fix", "wavelet_blur", "wavelet_decomposition",
           "wavelet_reconstruction", "wavelet_color_fix", "upsample_lr_frames", "color_fix_frames", "pack_video_uint8",
           "pack_frames_png"]


def _check(x: torch.Tensor, name: str):
    if x.dim() != 4:
        raise AssertionError("The input feature should be 4D tensor.")  # color_correction.py:53
    _lib.require_cuda(x, name)


def calc_mean_std(feat: torch.Tensor, eps: float = 1e-5):
    """color_correction.py:45-58: per (b, c) mean and sqrt(unbiased var + eps), shaped (b, c, 1, 1)"""
    _check(feat, "calc_mean_std")
    return ops.plane_stats(feat, eps)


def adaptive_instance_normalization(content_feat: torch.Tensor, style_feat: torch.Tensor) -> torch.Tensor:
    """color_correction.py:60-73"""
    _check(content_feat, "adaptive_instance_normalization")
    _check(style_feat, "adaptive_instance_normalization")
    style_mean, style_std = calc_mean_std(style_feat)
    content_mean, content_std = calc_mean_std(content_feat)
    return ops.adain_apply(content_feat, content_mean, content_std, style_mean, style_std)


def adain_color_fix(target_tensor: torch.Tensor, source_tensor: torch.Tensor) -> torch.Tensor:
    """color_correction.py:14-27"""
    return adaptive_instance_normalization(target_tensor, source_tensor)


def wavelet_blur(image: torch.Tensor, radius: int) -> torch.Tensor:
    """color_correction.py:75-93 (any plane count; the reference hard-codes 3 channels)"""
    _check(image, "wavelet_blur")
    image = image.float().contiguous()
    low = torch.empty_like(image)
    ops.wavelet_level(image, radius, low=low)
    return low


def wavelet_decomposition(image: torch.Tensor, levels: int = 5):
    """color_correction.py:95-103: returns (high_freq, low_freq)"""
    _check(image, "wavelet_decomposition")
    image = image.float().contiguous()
    high = torch.empty_like(image)
    bufs = [torch.empty_like(image), torch.empty_like(image)]
    cur = image
    for i in range(levels):
        low = bufs[i & 1]
        ops.wavelet_level(cur, 2 ** i, low=low, high=high, high_first=(i == 0))
        cur = low
    return high, cur


def wavelet_reconstruction(content_feat: torch.Tensor, style_feat: torch.Tensor, levels: int = 5) -> torch.Tensor:
    """color_correction.py:105-118: content high frequencies + style low frequencies"""
    _check(content_feat, "wavelet_reconstruction")
    _check(style_feat, "wavelet_reconstruction")
    content_high, _ = wavelet_decomposition(content_feat, levels)
    style = style_feat.float().contiguous()
    bufs = [torch.empty_like(style), torch.empty_like(style)]
    cur = style
    for i in range(levels):
        low = bufs[i & 1]
        # the last level writes content_high + style_low directly
        ops.wavelet_level(cur, 2 ** i, low=low, add=content_high if i == levels - 1 else None)
        cur = low
    return cur


def wavelet_color_fix(target_tensor: torch.Tensor, source_tensor: torch.Tensor) -> torch.Tensor:
    """color_correction.py:29-43"""
    return wavelet_reconstruction(target_tensor, source_tensor)


def upsample_lr_frames(vframes: torch.Tensor, scale: int = 4) -> torch.Tensor:
    """inference_upscale_a_video.py:325-327: (1, c, t, h, w) or (t, c, h, w) low-resolution frames -> (t, c, 4h, 4w)"""
    if vframes.dim() == 5:
        vframes = vframes.squeeze(0).permute(1, 0, 2, 3)
    return ops.bicubic_upsample(vframes, scale)


def color_fix_frames(output: torch.Tensor, vframes: torch.Tensor, color_fix: Optional[str]) -> torch.Tensor:
    """inference_upscale_a_video.py:323-333: `output` (1, c, t, H, W) from the pipeline, `vframes` (1, c, t, h, w) the
    low-resolution input; returns (t, c, H, W)."""
    out = output.squeeze(0).permute(1, 0, 2, 3).contiguous() if output.dim() == 5 else output
    if color_fix in ("AdaIn", "Wavelet"):
        lr = upsample_lr_frames(vframes, out.shape[-1] // vframes.shape[-1])
        out = adaptive_instance_normalization(out, lr) if color_fix == "AdaIn" else wavelet_reconstruction(out, lr)
    elif color_fix not in (None, "None"):
        raise ValueError(f"color_fix must be one of None, 'AdaIn', 'Wavelet' (got {color_fix!r})")
    return out


def pack_video_uint8(frames: torch.Tensor) -> torch.Tensor:
    """inference_upscale_a_video.py:354-356: (t, c, h, w) in [-1, 1] -> (t, h, w, c) uint8 on the device"""
    return ops.pack_video_uint8(frames)


def pack_frames_png(frames: torch.Tensor) -> torch.Tensor:
    """inference_upscale_a_video.py:350 (save_image(normalize=True, value_range=(-1, 1))): (t, c, h, w) -> (t, h, w, c)
    uint8 on the device"""
    _lib.require_cuda(frames, "pack_frames_png")
    return ops.pack_frames_png(frames)
