"""AutoencoderKLVideo — drop-in for /root/reference/models_video/autoencoder_kl_cond_video.py:41-226 and
vae_video.py (Encoder / Decoder / DiagonalGaussianDistribution).

Same config keys (`configs/vae_3d_config.json`, `configs/vae_video_config.json`), same state-dict keys, same
`.decode(z, img, w_lr).sample` / `.encode(x).latent_dist` / `.config.scaling_factor` surface.  The decoder is the
hot part (SURVEY.md §8a a18-a20): 3x3 convolutions up to 128 channels at 4x resolution and a single-head d=512
attention over all h*w positions per frame — all on the same sm_90a kernels as the UNet (fp16 operands, fp32
accumulate; the reference runs this module in fp32/TF32, see DESIGN.md for the measured drift)."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional, Tuple

import torch
from torch import nn

from . import ops
from ._config import ConfigMixin
from . import _lib
from .layers import (Ctx, DownEncoderBlock3D, Fuse_sft_block, InflatedConv3d, PackedModule, ResnetBlock3D_plus,
                     UNetMidBlock3D, UNetMidBlock3D_plus, UpDecoderBlock3D, UpDecoderBlock3D_plus, _gn)


# The reference decodes in fp32 because the SD-x4-upscaler VAE "overflows in float16" (pipeline_upscale_a_video.py:667-669):
# the decoder's RESIDUAL STREAM grows past 65504 in the up blocks.  Every consumer of that stream is either linear
# (shortcut / upsampler convs, residual adds) or a GroupNorm — scale invariant once its eps is scaled too — so the decoder
# keeps the stream at 2^-k of the reference's values (fp16 range x 2^k, power-of-two scale = no rounding change) and every
# branch output (post-GroupNorm, O(1)) is multiplied by 2^-k in the GEMM epilogue that adds it to the stream.  All fp16
# stores also saturate instead of producing inf.
VAE_STREAM_SCALE = 2.0 ** -7


@dataclass
class DecoderOutput:
    sample: torch.Tensor


@dataclass
class AutoencoderKLOutput:
    latent_dist: "DiagonalGaussianDistribution"


class DiagonalGaussianDistribution:
    """vae_video.py:408-451 (tiny elementwise math on the 8-channel moments; not on the sampling path)"""

    def __init__(self, parameters, deterministic=False):
        self.parameters = parameters
        self.mean, self.logvar = torch.chunk(parameters, 2, dim=1)
        self.logvar = torch.clamp(self.logvar, -30.0, 20.0)
        self.deterministic = deterministic
        self.std = torch.exp(0.5 * self.logvar)
        self.var = torch.exp(self.logvar)
        if deterministic:
            self.var = self.std = torch.zeros_like(self.mean)

    def sample(self, generator: Optional[torch.Generator] = None):
        gdev = generator.device if generator is not None else self.parameters.device
        noise = torch.randn(self.mean.shape, generator=generator, device=gdev, dtype=self.parameters.dtype)
        return self.mean + self.std * noise.to(self.parameters.device)

    def kl(self, other=None):
        if self.deterministic:
            return torch.Tensor([0.0])
        if other is None:
            return 0.5 * torch.sum(torch.pow(self.mean, 2) + self.var - 1.0 - self.logvar, dim=[1, 2, 3])
        return 0.5 * torch.sum(torch.pow(self.mean - other.mean, 2) / other.var + self.var / other.var - 1.0
                               - self.logvar + other.logvar, dim=[1, 2, 3])

    def mode(self):
        return self.mean


class Encoder(nn.Module):
    """vae_video.py:55-156"""

    def __init__(self, in_channels=3, out_channels=3, down_block_types=("DownEncoderBlock3D",), block_out_channels=(64,),
                 layers_per_block=2, norm_num_groups=32, act_fn="silu", double_z=True):
        super().__init__()
        self.conv_in = InflatedConv3d(in_channels, block_out_channels[0], kernel_size=3, stride=1, padding=1)
        self.down_blocks = nn.ModuleList([])
        out_ch = block_out_channels[0]
        for i, t in enumerate(down_block_types):
            if t != "DownEncoderBlock3D":
                raise ValueError(f"{t} does not exist.")
            in_ch, out_ch = out_ch, block_out_channels[i]
            self.down_blocks.append(DownEncoderBlock3D(in_ch, out_ch, num_layers=layers_per_block, resnet_eps=1e-6,
                                                       resnet_groups=norm_num_groups,
                                                       add_downsample=i != len(block_out_channels) - 1,
                                                       downsample_padding=0))
        self.mid_block = UNetMidBlock3D(block_out_channels[-1], resnet_eps=1e-6, resnet_groups=norm_num_groups)
        self.conv_norm_out = nn.GroupNorm(num_channels=block_out_channels[-1], num_groups=norm_num_groups, eps=1e-6)
        self.conv_out = InflatedConv3d(block_out_channels[-1], 2 * out_channels if double_z else out_channels, 3, padding=1)

    def forward(self, c: Ctx, x):
        x = self.conv_in.run(c, x)
        for blk in self.down_blocks:
            x = blk(c, x)
        x = self.mid_block(c, x)
        x = _gn(c, self.conv_norm_out, x, True, x.shape[0])
        return self.conv_out.run(c, x)


class Decoder(nn.Module):
    """vae_video.py:242-405"""

    def __init__(self, in_channels=3, out_channels=3, up_block_types=("UpDecoderBlock3D",), block_out_channels=(64,),
                 layers_per_block=2, norm_num_groups=32, act_fn="silu", condition_img=False, condition_channels=128,
                 use_temporal_block=False):
        super().__init__()
        self.condition_img = condition_img
        plus = up_block_types[0] != "UpDecoderBlock3D"
        self.conv_in = InflatedConv3d(in_channels, block_out_channels[-1], kernel_size=3, stride=1, padding=1)
        if condition_img:
            self.condition_in = nn.Sequential(
                ResnetBlock3D_plus(in_channels=3, out_channels=condition_channels, temb_channels=None, groups=3, groups_out=32),
                ResnetBlock3D_plus(in_channels=condition_channels, out_channels=condition_channels, temb_channels=None))
            self.condition_fuse = Fuse_sft_block(condition_channels, block_out_channels[-1])
        self.mid_block = (UNetMidBlock3D_plus if plus else UNetMidBlock3D)(block_out_channels[-1], resnet_eps=1e-6,
                                                                            resnet_groups=norm_num_groups)
        self.up_blocks = nn.ModuleList([])
        rev = list(reversed(block_out_channels))
        out_ch = rev[0]
        for i, t in enumerate(up_block_types):
            if t not in ("UpDecoderBlock3D", "UpDecoderBlock3D_plus"):
                raise ValueError(f"{t} does not exist.")
            prev, out_ch = out_ch, rev[i]
            cls = UpDecoderBlock3D_plus if t.endswith("_plus") else UpDecoderBlock3D
            self.up_blocks.append(cls(prev, out_ch, num_layers=layers_per_block + 1, resnet_eps=1e-6,
                                      resnet_groups=norm_num_groups, add_upsample=i != len(block_out_channels) - 1))
        self.conv_norm_out = nn.GroupNorm(num_channels=block_out_channels[0], num_groups=norm_num_groups, eps=1e-6)
        self.conv_out = InflatedConv3d(block_out_channels[0], out_channels, 3, padding=1)

    def forward(self, c: Ctx, z, img=None, w_lr=1.0):
        s = VAE_STREAM_SCALE
        if self.condition_img:
            assert img is not None, "input img condition when condition_img is True."
            x = self.conv_in.run(c, z)
            cond = self.condition_in[0](c, img)
            cond = self.condition_in[1](c, cond)
            x = self.condition_fuse(c, cond, x, w=w_lr, out_scale=s)  # the scaled stream starts after the SFT fusion
        else:
            x = self.conv_in.run(c, z, out_scale=s)
        x = self.mid_block(c, x, s)
        for blk in self.up_blocks:
            x = blk(c, x, s)
        x = _gn(c, self.conv_norm_out, x, True, x.shape[0], s)
        return self.conv_out.run(c, x, out_dtype=torch.float32)


class AutoencoderKLVideo(PackedModule, ConfigMixin):
    def __init__(self, in_channels: int = 3, out_channels: int = 3, down_block_types: Tuple[str] = ("DownEncoderBlock3D",),
                 up_block_types: Tuple[str] = ("UpDecoderBlock3D",), block_out_channels: Tuple[int] = (64,),
                 layers_per_block: int = 1, act_fn: str = "silu", latent_channels: int = 4, norm_num_groups: int = 32,
                 sample_size: int = 32, scaling_factor: float = 0.18215, condition_img: bool = False,
                 condition_channels: int = 128, use_temporal_block: bool = False):
        super().__init__()
        self._init_config(locals())
        self.encoder = Encoder(in_channels, latent_channels, down_block_types, block_out_channels, layers_per_block,
                               norm_num_groups, act_fn, True)
        self.decoder = Decoder(latent_channels, out_channels, up_block_types, block_out_channels, layers_per_block,
                               norm_num_groups, act_fn, condition_img, condition_channels, use_temporal_block)
        self.quant_conv = InflatedConv3d(2 * latent_channels, 2 * latent_channels, 1)
        self.post_quant_conv = InflatedConv3d(latent_channels, latent_channels, 1)
        self.use_slicing = False
        self.use_tiling = False

    @property
    def dtype(self):
        return next(self.parameters()).dtype

    @property
    def device(self):
        return next(self.parameters()).device

    def enable_slicing(self):
        self.use_slicing = True

    def disable_slicing(self):
        self.use_slicing = False

    def enable_tiling(self, use_tiling: bool = True):
        if use_tiling:
            raise NotImplementedError("tiled_encode/tiled_decode are unused by the pipeline (SURVEY.md §5) and out of scope")

    def _to_cl(self, x, pad_to=8, scale=1.0):
        """(b, c, t, h, w) fp16/fp32 -> zero-padded channels-last fp16 (b, t, h, w, 8)"""
        _lib.require_cuda(x, "AutoencoderKLVideo")
        B, C, T, H, W = x.shape
        buf = torch.zeros(B, T, H, W, (C + pad_to - 1) // pad_to * pad_to, dtype=torch.float16, device=x.device)
        src = x if x.dtype in (torch.float16, torch.float32) else x.float()
        ops.planar_to_channels_last(src.contiguous(), buf, 0, scale=scale)
        return buf

    @torch.no_grad()
    def encode(self, x, return_dict: bool = True):
        """autoencoder_kl_cond_video.py:174-185"""
        c = Ctx(self._packed())
        h = self.encoder(c, self._to_cl(x))
        m = self.quant_conv.run(c, h, out_dtype=torch.float32)
        moments = ops.channels_last_to_planar(m, 2 * self.config.latent_channels, torch.float32)
        posterior = DiagonalGaussianDistribution(moments.to(x.dtype if x.dtype.is_floating_point else torch.float32))
        if not return_dict:
            return (posterior,)
        return AutoencoderKLOutput(latent_dist=posterior)

    def _decode_one(self, z, img, w_lr, latent_scale=1.0, clamp=False):
        c = Ctx(self._packed())
        zc = self.post_quant_conv.run(c, self._to_cl(z, scale=latent_scale))
        ic = self._to_cl(img) if (img is not None and self.decoder.condition_img) else None
        y = self.decoder(c, zc, ic, w_lr)  # (b, t, 4h, 4w, 3) fp32
        return ops.channels_last_to_planar(y, self.config.out_channels, torch.float32, clamp=clamp).to(z.dtype)

    @torch.no_grad()
    def decode(self, z, img=None, w_lr=1, return_dict: bool = True, *, latent_scale: float = 1.0, clamp: bool = False):
        """autoencoder_kl_cond_video.py:209-226.  `latent_scale` / `clamp` (keyword-only extensions) fold the pipeline's
        `1 / scaling_factor * latents` and `.clamp(-1, 1)` (pipeline...:351-353) into the layout-conversion kernels."""
        if self.use_slicing and z.shape[0] > 1:
            imgs = img.split(1) if img is not None else [None] * z.shape[0]
            decoded = torch.cat([self._decode_one(zs, im, w_lr, latent_scale, clamp) for zs, im in zip(z.split(1), imgs)])
        else:
            decoded = self._decode_one(z, img, w_lr, latent_scale, clamp)
        if not return_dict:
            return (decoded,)
        return DecoderOutput(sample=decoded)

    def forward(self, sample, sample_posterior: bool = False, return_dict: bool = True, generator=None):
        posterior = self.encode(sample).latent_dist
        z = posterior.sample(generator=generator) if sample_posterior else posterior.mode()
        dec = self.decode(z).sample
        if not return_dict:
            return (dec,)
        return DecoderOutput(sample=dec)
