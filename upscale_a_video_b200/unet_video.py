"""UNetVideoModel — drop-in for /root/reference/models_video/unet_video.py:103-601.

Same constructor / config keys (`from_config(configs/unet_video_config.json)`), same state-dict keys and shapes
(1158 tensors, 691 M parameters), same `forward(sample, timestep, low_res, encoder_hidden_states, class_labels)`
returning `.sample` in the reference's "b c t h w" layout.  Inside, activations are fp16 channels-last and every
operator is a hand-written sm_90a kernel behind the C ABI (include/uav_b200.h); there is no PyTorch compute
fallback: CPU tensors raise.

Work the reference repeats but that is exact to remove (SURVEY.md §7.2):
  * the 40 `time_emb_proj(silu(emb))` Linears run as ONE GEMM per forward;
  * the prompt's K/V projections of all 26 cross-attention sites run as ONE GEMM and are cached across DDIM
    steps (they depend on the prompt only; the reference recomputes them per frame and step, attention.py:364);
  * layout copies `b c t h w <-> (b t) c h w` and `(b f) d c <-> (b d) f c` do not exist in channels-last.
"""
from __future__ import annotations

import json
import os
from dataclasses import dataclass
from typing import Optional, Tuple, Union

import torch
from torch import nn

from . import ops
from ._config import ConfigMixin
from . import _lib
from .layers import (CrossAttention, CrossAttnDownBlock3D, CrossAttnUpBlock3D, Ctx, DownBlock3D, EmptyTemporalModule3D,
                     InflatedConv3d, PackedModule, ResnetBlock3D, RotaryEmbedding, TemporalModule3D,
                     UNetMidBlock3DCrossAttn, UpBlock3D, _gn, new_cat_slot)


@dataclass
class UNet3DConditionOutput:
    sample: torch.Tensor

    def __getitem__(self, i):
        return (self.sample,)[i]


@dataclass
class UNetCfgStepOutput:
    """forward(..., cfg_step=...): the guidance combine and DDIMScheduler.step_v0 ran in conv_out's epilogue"""
    noise_pred: torch.Tensor            # (1, c, t, h, w): u + g (c - u)
    pred_original_sample: torch.Tensor  # (1, c, t, h, w): step_v0(noise_pred, t, sample)


class TimestepEmbedding(nn.Module):
    """diffusers TimestepEmbedding parameter holder (unet_video.py:176)"""

    def __init__(self, in_channels, time_embed_dim):
        super().__init__()
        self.linear_1 = nn.Linear(in_channels, time_embed_dim)
        self.linear_2 = nn.Linear(time_embed_dim, time_embed_dim)


_DOWN = {"DownBlock3D": DownBlock3D, "CrossAttnDownBlock3D": CrossAttnDownBlock3D}
_UP = {"UpBlock3D": UpBlock3D, "CrossAttnUpBlock3D": CrossAttnUpBlock3D}


class UNetVideoModel(PackedModule, ConfigMixin):
    _supports_gradient_checkpointing = False

    def __init__(self, down_temporal_idx=(0, 1, 2), mid_temporal=False, up_temporal_idx=(1, 2, 3),
                 temporal_module_config=None, sample_size: Optional[int] = None, in_channels: int = 7,
                 out_channels: int = 4, center_input_sample: bool = False, max_noise_level: int = 350,
                 flip_sin_to_cos: bool = True, freq_shift: int = 0, attention_head_dim: Union[int, Tuple[int]] = 8,
                 block_out_channels: Tuple[int] = (256, 512, 512, 1024),
                 down_block_types: Tuple[str] = ("DownBlock3D", "CrossAttnDownBlock3D", "CrossAttnDownBlock3D",
                                                 "CrossAttnDownBlock3D"),
                 mid_block_type: str = "UNetMidBlock3DCrossAttn",
                 up_block_types: Tuple[str] = ("CrossAttnUpBlock3D", "CrossAttnUpBlock3D", "CrossAttnUpBlock3D",
                                               "UpBlock3D"),
                 only_cross_attention: Union[bool, Tuple[bool]] = (True, True, True, False), layers_per_block: int = 2,
                 downsample_padding: int = 1, mid_block_scale_factor: float = 1, act_fn: str = "silu",
                 norm_num_groups: int = 32, norm_eps: float = 1e-5, cross_attention_dim: int = 1024,
                 dual_cross_attention: bool = False, use_linear_projection: bool = True,
                 class_embed_type: Optional[str] = None, num_class_embeds: Optional[int] = 1000,
                 upcast_attention: bool = False, resnet_time_scale_shift: str = "default", use_first_frame: bool = False,
                 use_relative_position: bool = False):
        super().__init__()
        self._init_config(locals())
        if (dual_cross_attention or not use_linear_projection or class_embed_type is not None or upcast_attention or
                resnet_time_scale_shift != "default" or use_first_frame or use_relative_position or
                mid_block_scale_factor != 1 or act_fn not in ("silu", "swish") or center_input_sample):
            raise NotImplementedError("only the option set of configs/unet_video_config.json is implemented "
                                      "(SURVEY.md §3.3); the other branches are dead in the shipped pipeline")
        temporal_module_config = temporal_module_config or {}
        self.sample_size = sample_size
        time_embed_dim = block_out_channels[0] * 4
        n = len(down_block_types)
        self.conv_in = InflatedConv3d(in_channels, block_out_channels[0], kernel_size=3, padding=1)
        self.time_embedding = TimestepEmbedding(block_out_channels[0], time_embed_dim)
        self.class_embedding = nn.Embedding(num_class_embeds, time_embed_dim) if num_class_embeds is not None else None
        oca = [only_cross_attention] * n if isinstance(only_cross_attention, bool) else list(only_cross_attention)
        heads = (attention_head_dim,) * n if isinstance(attention_head_dim, int) else tuple(attention_head_dim)
        self.temporal_rotary_emb = RotaryEmbedding(32)

        self.down_blocks = nn.ModuleList([])
        self.down_temp_blocks = nn.ModuleList([])
        out_ch = block_out_channels[0]
        for i, bt in enumerate(down_block_types):
            in_ch, out_ch = out_ch, block_out_channels[i]
            final = i == n - 1
            self.down_blocks.append(_DOWN[bt](in_channels=in_ch, out_channels=out_ch, temb_channels=time_embed_dim,
                                              num_layers=layers_per_block, resnet_eps=norm_eps,
                                              resnet_groups=norm_num_groups, add_downsample=not final,
                                              downsample_padding=downsample_padding, attn_num_head_channels=heads[i],
                                              cross_attention_dim=cross_attention_dim, only_cross_attention=oca[i],
                                              rotary_emb=self.temporal_rotary_emb))
            self.down_temp_blocks.append(TemporalModule3D(in_channels=out_ch, out_channels=out_ch,
                                                          temb_channels=time_embed_dim, **temporal_module_config)
                                         if i in down_temporal_idx else EmptyTemporalModule3D())
        if mid_block_type != "UNetMidBlock3DCrossAttn":
            raise ValueError(f"unknown mid_block_type : {mid_block_type}")
        self.mid_block = UNetMidBlock3DCrossAttn(in_channels=block_out_channels[-1], temb_channels=time_embed_dim,
                                                 resnet_eps=norm_eps, resnet_groups=norm_num_groups,
                                                 attn_num_head_channels=heads[-1], cross_attention_dim=cross_attention_dim,
                                                 rotary_emb=self.temporal_rotary_emb)
        self.mid_temp_block = (TemporalModule3D(in_channels=block_out_channels[-1], out_channels=block_out_channels[-1],
                                                temb_channels=time_embed_dim, **temporal_module_config)
                               if mid_temporal else EmptyTemporalModule3D())
        self.num_upsamplers = 0
        self.up_blocks = nn.ModuleList([])
        self.up_temp_blocks = nn.ModuleList([])
        rev = list(reversed(block_out_channels))
        rheads, roca = list(reversed(heads)), list(reversed(oca))
        out_ch = rev[0]
        for i, bt in enumerate(up_block_types):
            final = i == n - 1
            prev, out_ch = out_ch, rev[i]
            in_ch = rev[min(i + 1, n - 1)]
            if not final:
                self.num_upsamplers += 1
            self.up_blocks.append(_UP[bt](in_channels=in_ch, out_channels=out_ch, prev_output_channel=prev,
                                          temb_channels=time_embed_dim, num_layers=layers_per_block + 1,
                                          resnet_eps=norm_eps, resnet_groups=norm_num_groups, add_upsample=not final,
                                          attn_num_head_channels=rheads[i], cross_attention_dim=cross_attention_dim,
                                          only_cross_attention=roca[i], rotary_emb=self.temporal_rotary_emb))
            self.up_temp_blocks.append(TemporalModule3D(in_channels=out_ch, out_channels=out_ch,
                                                        temb_channels=time_embed_dim, **temporal_module_config)
                                       if i in up_temporal_idx else EmptyTemporalModule3D())
        self.conv_norm_out = nn.GroupNorm(num_channels=block_out_channels[0], num_groups=norm_num_groups, eps=norm_eps)
        self.conv_out = InflatedConv3d(block_out_channels[0], out_channels, kernel_size=3, padding=1)

    # ------------------------------------------------------------------ diffusers-ish conveniences
    @property
    def dtype(self):
        return next(self.parameters()).dtype

    @property
    def device(self):
        return next(self.parameters()).device

    @classmethod
    def from_pretrained_2d(cls, config_path, pretrained_model_path):
        """unet_video.py:577-601 (load a checkpoint, keeping freshly initialised temporal layers)"""
        if not os.path.isfile(config_path):
            raise RuntimeError(f"{config_path} does not exist")
        with open(config_path) as f:
            config = json.load(f)
        model = cls.from_config(config)
        if not os.path.isfile(pretrained_model_path):
            raise RuntimeError(f"{pretrained_model_path} does not exist")
        state_dict = torch.load(pretrained_model_path, map_location="cpu")
        for k, v in model.state_dict().items():
            if "temporal" in k:
                state_dict.update({k: v})
        model.load_state_dict(state_dict, strict=True)
        return model

    # ------------------------------------------------------------------ per-forward batched projections
    def _temb_modules(self):
        mods = self.__dict__.get("_temb_mods")
        if mods is None:
            mods = [m for m in self.modules() if isinstance(m, ResnetBlock3D) and m.time_emb_proj is not None]
            self.__dict__["_temb_mods"] = mods
        return mods

    def _cross_modules(self):
        mods = self.__dict__.get("_cross_mods")
        if mods is None:
            mods = [m for m in self.modules() if isinstance(m, CrossAttention) and m.is_cross]
            self.__dict__["_cross_mods"] = mods
        return mods

    def _prepare_ctx(self, c: Ctx, emb, encoder_hidden_states, T):
        pk = c.pk
        mods = self._temb_modules()
        w, b = pk.fused_linear("temb_all", [m.time_emb_proj for m in mods])
        c.temb_all = ops.linear(ops.silu(emb), w, b)
        col = 0
        for m in mods:
            c.temb_slices[id(m)] = (col, col + m.out_channels)
            col += m.out_channels
        cross = self._cross_modules()
        col = 0
        for m in cross:
            cc = m.to_k.weight.shape[0]
            c.ctx_slices[id(m)] = (col, cc)
            col += 2 * cc
        ehs = encoder_hidden_states
        # cache hit only for the SAME tensor object, unmodified: the cache keeps a reference to it, so its storage
        # cannot be recycled for a different prompt while the entry is alive (a data_ptr key would go stale)
        hit = pk.cache.get("ctx_kv_src")
        if hit is None or hit[0] is not ehs or hit[1] != ehs._version:
            w, b = pk.fused_linear("ctx_kv_w", [x for m in cross for x in (m.to_k, m.to_v)])
            pk.cache["ctx_kv"] = ops.linear(ehs.to(torch.float16).contiguous(), w, b)
            pk.cache["ctx_kv_src"] = (ehs, ehs._version)
        c.ctx_kv = pk.cache["ctx_kv"]
        c.ctx_len = ehs.shape[1]
        c.rot = pk.tensor(f"rot{T}", lambda: self.temporal_rotary_emb.table(T))

    # ------------------------------------------------------------------ forward (unet_video.py:404-574)
    @torch.no_grad()
    def forward(self, sample, timestep, low_res, encoder_hidden_states=None, class_labels=20, attention_mask=None,
                return_dict: bool = True, *, cfg_shared_input: bool = False, cfg_step: Optional[dict] = None):
        """`cfg_shared_input` (keyword-only extension, set by VideoUpscalePipeline): the two batch items are the
        classifier-free-guidance halves of the SAME latents / LR frames / noise level (pipeline...:614,551), so everything
        before the first text-conditioned layer (conv_in, down block 0, its temporal module, the first resnet of down
        block 1) is identical for both and is computed once (SURVEY.md §7.2 iii: exact work removal, ~3.6 % of the FLOPs).
        `cfg_step` (keyword-only extension, set by VideoUpscalePipeline for the single-window case): dict(guidance_scale,
        pred_type, sqrt_alpha, sqrt_beta, clip, clip_range, sample) — classifier-free guidance and DDIMScheduler.step_v0
        (pipeline...:644-649) run in conv_out's epilogue and a UNetCfgStepOutput is returned; ignored (plain output) when
        the fused tail does not apply (batch != 2, fp32 working dtype)."""
        _lib.require_cuda(sample, "UNetVideoModel.forward")
        if attention_mask is not None:
            raise NotImplementedError("attention_mask is never passed by VideoUpscalePipeline")
        if encoder_hidden_states is None:
            raise ValueError("encoder_hidden_states is required (cross-attention blocks)")
        B, _, T, H, W = sample.shape
        dev = sample.device
        c = Ctx(self._packed())
        cfg = self.config

        # sample = torch.cat([sample, low_res], dim=1) -> channels-last, padded 7 -> 8 channels
        cin = sample.shape[1] + low_res.shape[1]
        if cin != cfg.in_channels:
            raise ValueError(f"expected {cfg.in_channels} input channels, got {cin}")
        share = (cfg_shared_input and B == 2 and len(self.down_blocks) > 1 and not self.down_blocks[0].has_cross_attention
                 and self.down_blocks[1].has_cross_attention)
        Bp = 1 if share else B
        x = torch.zeros(Bp, T, H, W, (cin + 7) // 8 * 8, dtype=torch.float16, device=dev)
        ops.planar_to_channels_last(sample[:Bp].contiguous(), x, 0)
        ops.planar_to_channels_last(low_res[:Bp].contiguous(), x, sample.shape[1])
        forward_upsample_size = any(s % (2 ** self.num_upsamplers) != 0 for s in (H, W))

        # time + class embedding (unet_video.py:457-491)
        if not torch.is_tensor(timestep):
            t = torch.full((B,), float(timestep), dtype=torch.float32, device=dev)
        else:
            t = timestep.to(device=dev, dtype=torch.float32).reshape(-1).expand(B).contiguous()
        t_emb = ops.timestep_embedding(t, cfg.block_out_channels[0], cfg.flip_sin_to_cos, float(cfg.freq_shift))
        w1, b1 = c.pk.linear(self.time_embedding.linear_1)
        w2, b2 = c.pk.linear(self.time_embedding.linear_2)
        e1 = ops.linear(t_emb, w1, b1, act=ops.ACT_SILU)
        cls_rows = None
        if self.class_embedding is not None:
            if class_labels is None:
                raise ValueError("class_labels should be provided when num_class_embeds > 0")
            cl = torch.as_tensor(class_labels, device=dev).reshape(-1).long()
            self._check_noise_level(class_labels, cl)
            tbl = c.pk.tensor("class_emb_f16", lambda: self.class_embedding.weight.detach().to(torch.float16))
            cls_rows = tbl.index_select(0, cl).expand(B, -1).contiguous()
        emb = ops.linear(e1, w2, b2, residual=cls_rows)
        self._prepare_ctx(c, emb, encoder_hidden_states, T)

        # pre-process / down / mid / up
        taps = self.__dict__.get("_debug_taps")  # tests/debug: dict receiving every stage output (channels-last)

        def _tap(name, v):
            if taps is not None:
                taps[name] = v

        x = self.conv_in.run(c, x)
        _tap("conv_in", x)
        skips = [x]
        for i, (blk, tmod) in enumerate(zip(self.down_blocks, self.down_temp_blocks)):
            if share and i == 1:
                x, outs = blk(c, x, expand_batch_to=B)
            else:
                x, outs = blk(c, x)
            skips += outs
            _tap(f"down{i}", x)
            x = tmod(c, x)
            _tap(f"down_temp{i}", x)
        # every up-block resnet consumes torch.cat([x, skip]): the layer that produces x stores straight into the head of the
        # concat buffer (layers.new_cat_slot), so only the skip half is ever copied
        def first_slot(i, cx, size_hw=None, producer_has_stats=False):
            """head slice of the concat buffer of up block i's first resnet (None: plain allocation by the producer)"""
            skip = skips[-1]
            if size_hw is not None and tuple(skip.shape[2:4]) != tuple(size_hw):
                return None
            return new_cat_slot(skip, cx, B, producer_has_stats)

        mid_empty = isinstance(self.mid_temp_block, EmptyTemporalModule3D)
        c_mid = cfg.block_out_channels[-1]
        slot = first_slot(0, c_mid, x.shape[2:4], True)
        x = self.mid_block(c, x, out=slot if mid_empty else None)
        _tap("mid", x)
        x = self.mid_temp_block(c, x, out=None if mid_empty else slot)
        _tap("mid_temp", x)
        for i, (blk, tmod) in enumerate(zip(self.up_blocks, self.up_temp_blocks)):
            nres = len(blk.resnets)
            res, skips = skips[-nres:], skips[:-nres]
            final = i == len(self.up_blocks) - 1
            up_size = tuple(skips[-1].shape[1:4]) if (not final and forward_upsample_size) else None
            t_empty = isinstance(tmod, EmptyTemporalModule3D)
            slot = None
            if not final:
                hw = tuple(up_size[1:]) if up_size is not None else (2 * x.shape[2], 2 * x.shape[3])
                # producer of the next block's main branch: the temporal module's shift_conv (emits statistics) or,
                # without a temporal module, the upsampler conv (its four phase launches emit none)
                slot = first_slot(i + 1, blk.resnets[-1].out_channels, hw, not t_empty)
            x = blk(c, x, res, up_size, out=slot if t_empty else None)
            _tap(f"up{i}", x)
            x = tmod(c, x, out=None if t_empty else slot)
            _tap(f"up_temp{i}", x)
        out_dtype = sample.dtype if sample.dtype in (torch.float16, torch.float32) else torch.float16
        if x.shape[-1] == 256 and cfg.out_channels <= 5 and x.shape[0] == B:
            # GroupNorm apply + SiLU + conv_out + the rearrange to "b c t h w" in ONE pass over the 256-channel tensor
            g, bt = c.pk.affine(self.conv_norm_out)
            w, bias = c.pk.conv(self.conv_out)
            if cfg_step is not None and B == 2 and out_dtype == torch.float16 and cfg_step["sample"].dtype == torch.float16:
                npred, x0 = ops.conv_out_fused(x, g, bt, self.conv_norm_out.num_groups, self.conv_norm_out.eps, w, bias,
                                               cfg.out_channels, out_dtype, cfg_step=cfg_step)
                return UNetCfgStepOutput(noise_pred=npred, pred_original_sample=x0)
            out = ops.conv_out_fused(x, g, bt, self.conv_norm_out.num_groups, self.conv_norm_out.eps, w, bias,
                                     cfg.out_channels, out_dtype)
        else:
            x = _gn(c, self.conv_norm_out, x, True, B)
            x = self.conv_out.run(c, x)
            out = ops.channels_last_to_planar(x, cfg.out_channels, out_dtype)
        if not return_dict:
            return (out,)
        return UNet3DConditionOutput(sample=out)

    def _check_noise_level(self, orig, cl):
        """`if torch.any(class_labels > max_noise_level): raise` (unet_video.py:484) without a per-step device sync:
        host values are checked directly, a device tensor once per distinct (pointer, version)."""
        mx = self.config.max_noise_level
        if not torch.is_tensor(orig) or not orig.is_cuda:
            if int(torch.as_tensor(orig).max()) > mx:
                raise ValueError(f"`noise_level` has to be <= {mx} but is {orig}")
            return
        # memo keyed on the tensor OBJECT (held alive by the entry, so its storage cannot be recycled for other labels while the
        # entry exists — a data_ptr key would go stale) and its version counter; a handful of entries at most
        seen = self.__dict__.setdefault("_nl_checked", [])
        for ref, ver in seen:
            if ref is orig and ver == orig._version:
                return
        if bool(torch.any(cl > mx)):
            raise ValueError(f"`noise_level` has to be <= {mx} but is {orig}")
        seen.append((orig, orig._version))
        del seen[:-4]
