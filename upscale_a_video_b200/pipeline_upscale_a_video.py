"""VideoUpscalePipeline — drop-in for /root/reference/models_video/pipeline_upscale_a_video.py:62-717.

Same constructor, attribute surface (`pipeline.vae/unet/scheduler/propagator = ...`, `.to(device)`) and `__call__`
signature / return types, so `inference_upscale_a_video.py` drives it unchanged.  What differs is below the API:

  * every tensor op of the denoising loop is a uav_b200 CUDA kernel (UNet, CFG, window blend, step_v0,
    propagation, step_vt) — no per-step `torch.cuda.empty_cache()` and no device->host syncs (the reference has
    both: pipeline...:612,622 and scheduling_ddim.py:404,459);
  * an exactly duplicated last window (pipeline...:624-625, e.g. T = 14, 32, 50) is computed once and blended twice
    in reference order (bit-identical, SURVEY.md §7.2 iv);
  * with torch.distributed initialised (one process per GPU) the UNet windows of a step and the VAE decode chunks
    are sharded over ranks with one NCCL all_gather per step (`sharding.py`, SURVEY.md §8e).
"""
from __future__ import annotations

import inspect
from dataclasses import dataclass
from typing import Any, Iterator, List, Optional, Tuple, Union

import torch

from . import _lib, ops, sharding
from .scheduling_ddim import _PRED
from ._config import ConfigMixin
from ._lib import UavError


@dataclass
class StableDiffusionPipelineOutput:
    images: Any
    nsfw_content_detected: Any = None


def randn_tensor(shape, generator=None, device=None, dtype=None):
    """diffusers.utils.randn_tensor: draw on the generator's device, then move (pipeline...:424,547)"""
    gdev = generator.device if generator is not None else torch.device(device)
    return torch.randn(shape, generator=generator, device=gdev, dtype=dtype).to(device)


class VideoUpscalePipeline(ConfigMixin):
    def __init__(self, text_encoder=None, tokenizer=None, low_res_scheduler=None, scheduler=None, vae=None, unet=None,
                 propagator=None, max_noise_level: int = 350):
        if vae is not None and hasattr(vae, "config") and getattr(vae.config, "scaling_factor", None) != 0.08333:
            vae.register_to_config(scaling_factor=0.08333)  # pipeline...:76-93
        self.vae, self.text_encoder, self.tokenizer, self.unet = vae, text_encoder, tokenizer, unet
        self.low_res_scheduler, self.scheduler, self.propagator = low_res_scheduler, scheduler, propagator
        self.register_to_config(max_noise_level=max_noise_level)
        self.process_group = None  # torch.distributed group used for window / chunk sharding (None = default)

    # ------------------------------------------------------------------ loading (inference_upscale_a_video.py:101)
    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path: str, torch_dtype=None, **_):
        """`DiffusionPipeline.from_pretrained(local_dir, torch_dtype=...)` for the layout the reference ships
        (README.md:78-101): `text_encoder/` (CLIP text model: config.json + weights) -> the uav_b200 `CLIPTextModel`,
        `tokenizer/` -> `transformers.CLIPTokenizer` (host-side string processing, not on the GPU path),
        `low_res_scheduler/scheduler_config.json` -> `DDPMScheduler`, and — when present — `scheduler/`, `vae/`, `unet/`
        (the reference CLI overwrites these three right after, lines 104-121).  Components that are absent stay None."""
        import json
        import os
        from .clip_text import CLIPTextModel
        from .scheduling_ddim import DDIMScheduler, DDPMScheduler
        root = pretrained_model_name_or_path
        if not os.path.isdir(root):
            raise EnvironmentError(f"{root} is not a local directory (there is no hub access: pass the downloaded folder)")

        def sub(*names):
            q = os.path.join(root, *names)
            return q if os.path.exists(q) else None

        text_encoder = tokenizer = low_res = sched = None
        if sub("text_encoder", "config.json"):
            text_encoder = CLIPTextModel.from_pretrained(sub("text_encoder"), torch_dtype=torch_dtype)
        if sub("tokenizer"):
            try:
                from transformers import CLIPTokenizer
            except ImportError as e:  # pragma: no cover
                raise ImportError("the tokenizer of the text prompt needs `transformers` (CLIPTokenizer)") from e
            tokenizer = CLIPTokenizer.from_pretrained(sub("tokenizer"))
        if sub("low_res_scheduler", "scheduler_config.json"):
            low_res = DDPMScheduler.from_config(json.load(open(sub("low_res_scheduler", "scheduler_config.json"))))
        if sub("scheduler", "scheduler_config.json"):
            sched = DDIMScheduler.from_config(json.load(open(sub("scheduler", "scheduler_config.json"))))
        max_noise_level = 350
        if sub("model_index.json"):
            max_noise_level = json.load(open(sub("model_index.json"))).get("max_noise_level", 350)
        return cls(text_encoder=text_encoder, tokenizer=tokenizer, low_res_scheduler=low_res, scheduler=sched, vae=None,
                   unet=None, propagator=None, max_noise_level=max_noise_level)

    # ------------------------------------------------------------------ plumbing
    def to(self, device):
        for name in ("vae", "text_encoder", "unet", "propagator"):
            m = getattr(self, name)
            if m is not None and hasattr(m, "to"):
                setattr(self, name, m.to(device))
        return self

    @property
    def device(self):
        for m in (self.unet, self.vae):
            if isinstance(m, torch.nn.Module):
                return next(m.parameters()).device
        return torch.device("cpu")

    @property
    def _execution_device(self):
        return self.device

    # ------------------------------------------------------------------ prompt (pipeline...:177-321)
    def _encode_prompt(self, prompt, device, num_images_per_prompt, do_classifier_free_guidance, negative_prompt=None,
                       prompt_embeds=None, negative_prompt_embeds=None):
        if prompt is not None and isinstance(prompt, str):
            batch_size = 1
        elif prompt is not None and isinstance(prompt, list):
            batch_size = len(prompt)
        else:
            batch_size = prompt_embeds.shape[0]
        te_dtype = getattr(self.text_encoder, "dtype", None) or (prompt_embeds.dtype if prompt_embeds is not None else torch.float16)
        if prompt_embeds is None:
            text_inputs = self.tokenizer(prompt, padding="max_length", max_length=self.tokenizer.model_max_length,
                                         truncation=True, return_tensors="pt")
            cfg = getattr(self.text_encoder, "config", None)
            mask = text_inputs.attention_mask.to(device) if getattr(cfg, "use_attention_mask", False) else None
            prompt_embeds = self.text_encoder(text_inputs.input_ids.to(device), attention_mask=mask)[0]
        prompt_embeds = prompt_embeds.to(dtype=te_dtype, device=device)
        bs, seq_len, _ = prompt_embeds.shape
        prompt_embeds = prompt_embeds.repeat(1, num_images_per_prompt, 1).view(bs * num_images_per_prompt, seq_len, -1)
        if do_classifier_free_guidance and negative_prompt_embeds is None:
            if negative_prompt is None:
                uncond_tokens = [""] * batch_size
            elif type(prompt) is not type(negative_prompt):
                raise TypeError(f"`negative_prompt` should be the same type to `prompt`, but got {type(negative_prompt)} !="
                                f" {type(prompt)}.")
            elif isinstance(negative_prompt, str):
                uncond_tokens = [negative_prompt]
            elif batch_size != len(negative_prompt):
                raise ValueError(f"`negative_prompt`: {negative_prompt} has batch size {len(negative_prompt)}, but `prompt`:"
                                 f" {prompt} has batch size {batch_size}. Please make sure that passed `negative_prompt` matches"
                                 " the batch size of `prompt`.")
            else:
                uncond_tokens = negative_prompt
            uncond_input = self.tokenizer(uncond_tokens, padding="max_length", max_length=prompt_embeds.shape[1],
                                          truncation=True, return_tensors="pt")
            cfg = getattr(self.text_encoder, "config", None)
            mask = uncond_input.attention_mask.to(device) if getattr(cfg, "use_attention_mask", False) else None
            negative_prompt_embeds = self.text_encoder(uncond_input.input_ids.to(device), attention_mask=mask)[0]
        if do_classifier_free_guidance:
            seq_len = negative_prompt_embeds.shape[1]
            negative_prompt_embeds = negative_prompt_embeds.to(dtype=te_dtype, device=device)
            negative_prompt_embeds = negative_prompt_embeds.repeat(1, num_images_per_prompt, 1).view(
                batch_size * num_images_per_prompt, seq_len, -1)
            prompt_embeds = torch.cat([negative_prompt_embeds, prompt_embeds])
        return prompt_embeds

    def prepare_extra_step_kwargs(self, generator, eta):
        keys = set(inspect.signature(self.scheduler.step).parameters.keys())
        out = {}
        if "eta" in keys:
            out["eta"] = eta
        if "generator" in keys:
            out["generator"] = generator
        return out

    def check_inputs(self, prompt, image, noise_level, negative_prompt=None, prompt_embeds=None, negative_prompt_embeds=None):
        """pipeline...:356-418"""
        if prompt is not None and prompt_embeds is not None:
            raise ValueError(f"Cannot forward both `prompt`: {prompt} and `prompt_embeds`: {prompt_embeds}. Please make sure to"
                             " only forward one of the two.")
        elif prompt is None and prompt_embeds is None:
            raise ValueError("Provide either `prompt` or `prompt_embeds`. Cannot leave both `prompt` and `prompt_embeds` undefined.")
        elif prompt is not None and (not isinstance(prompt, str) and not isinstance(prompt, list)):
            raise ValueError(f"`prompt` has to be of type `str` or `list` but is {type(prompt)}")
        if negative_prompt is not None and negative_prompt_embeds is not None:
            raise ValueError(f"Cannot forward both `negative_prompt`: {negative_prompt} and `negative_prompt_embeds`:"
                             f" {negative_prompt_embeds}. Please make sure to only forward one of the two.")
        if prompt_embeds is not None and negative_prompt_embeds is not None:
            if prompt_embeds.shape != negative_prompt_embeds.shape:
                raise ValueError("`prompt_embeds` and `negative_prompt_embeds` must have the same shape when passed directly, but"
                                 f" got: `prompt_embeds` {prompt_embeds.shape} != `negative_prompt_embeds`"
                                 f" {negative_prompt_embeds.shape}.")
        if not isinstance(image, torch.Tensor):
            raise ValueError(f"`image` has to be of type `torch.Tensor` but is {type(image)} (PIL inputs are not supported "
                             "by the video pipeline: it indexes image.shape[2:] as (t, h, w))")
        # the reference derives the batch size from `prompt` here and therefore cannot run with prompt=None
        # (len(None), SURVEY.md §3.2); with prompt_embeds the batch size is prompt_embeds.shape[0]
        batch_size = 1 if isinstance(prompt, str) else (len(prompt) if prompt is not None else prompt_embeds.shape[0])
        if batch_size != image.shape[0]:
            raise ValueError(f"`prompt` has batch size {batch_size} and `image` has batch size {image.shape[0]}."
                             " Please make sure that passed `prompt` matches the batch size of `image`.")
        if noise_level > self.config.max_noise_level:
            raise ValueError(f"`noise_level` has to be <= {self.config.max_noise_level} but is {noise_level}")

    def prepare_latents_3d(self, batch_size, num_channels_latents, seq_len, height, width, dtype, device, generator, latents=None):
        shape = (batch_size, num_channels_latents, seq_len, height, width)
        if latents is None:
            latents = randn_tensor(shape, generator=generator, device=device, dtype=dtype)
        else:
            if latents.shape != shape:
                raise ValueError(f"Unexpected latents shape, got {latents.shape}, expected {shape}")
            latents = latents.to(device=device, dtype=dtype)
        if self.scheduler.init_noise_sigma != 1.0:
            latents = latents * self.scheduler.init_noise_sigma
        return latents

    def decode_latents_vsr(self, latents, img, w_lr):
        """pipeline...:350-354: decode(latents / scaling_factor).clamp(-1, 1).float()"""
        return self.vae.decode(latents, img, w_lr, latent_scale=1.0 / self.vae.config.scaling_factor, clamp=True).sample.float()

    # ------------------------------------------------------------------ __call__ (pipeline...:436-717)
    @torch.no_grad()
    def __call__(self, prompt: Union[str, List[str]] = None, image: torch.Tensor = None, flows_bi: Optional[list] = None,
                 num_inference_steps: int = 75, guidance_scale: float = 9.0, noise_level: int = 20,
                 denoise_level: Optional[int] = None, negative_prompt: Optional[Union[str, List[str]]] = None,
                 num_images_per_prompt: Optional[int] = 1, eta: float = 0.0, generator=None,
                 latents: Optional[torch.Tensor] = None, prompt_embeds: Optional[torch.Tensor] = None,
                 negative_prompt_embeds: Optional[torch.Tensor] = None, propagation_steps: list = [], w_lr: float = 1,
                 return_dict: bool = True, *, noise: Optional[torch.Tensor] = None):
        """`noise` (keyword-only extension): the LR-noise draw of pipeline...:547, for generator-independent tests.
        The whole clip: `sample_latents`, then every chunk of `decode_chunks` concatenated along time."""
        sampled = self.sample_latents(prompt, image, flows_bi, num_inference_steps, guidance_scale, noise_level,
                                      denoise_level, negative_prompt, num_images_per_prompt, eta, generator, latents,
                                      prompt_embeds, negative_prompt_embeds, propagation_steps, w_lr, noise=noise)
        frames = [f for _, _, f in self.decode_chunks(sampled)]
        images = torch.cat(frames, dim=2) if len(frames) > 1 else frames[0]
        if not return_dict:
            return (images, sampled.latents)
        return StableDiffusionPipelineOutput(images=images, nsfw_content_detected=None)

    @torch.no_grad()
    def sample_latents(self, prompt: Union[str, List[str]] = None, image: torch.Tensor = None,
                       flows_bi: Optional[list] = None, num_inference_steps: int = 75, guidance_scale: float = 9.0,
                       noise_level: int = 20, denoise_level: Optional[int] = None,
                       negative_prompt: Optional[Union[str, List[str]]] = None, num_images_per_prompt: Optional[int] = 1,
                       eta: float = 0.0, generator=None, latents: Optional[torch.Tensor] = None,
                       prompt_embeds: Optional[torch.Tensor] = None, negative_prompt_embeds: Optional[torch.Tensor] = None,
                       propagation_steps: list = [], w_lr: float = 1, *,
                       noise: Optional[torch.Tensor] = None) -> "SampledLatents":
        """`__call__` up to the decode (same arguments but `return_dict`): the denoised latents of the whole clip and
        what the decoder needs with them.  `decode_chunks` turns the record into output frames a few at a time, so a
        caller that consumes them chunk by chunk never holds the whole clip at output resolution."""
        self.check_inputs(prompt, image, noise_level, negative_prompt, prompt_embeds, negative_prompt_embeds)
        if image is None:
            raise ValueError("`image` input cannot be undefined.")
        if prompt is not None and isinstance(prompt, str):
            batch_size = 1
        elif prompt is not None and isinstance(prompt, list):
            batch_size = len(prompt)
        else:
            batch_size = prompt_embeds.shape[0]
        device = self._execution_device
        _lib.require_cuda(torch.empty(0, device=device), "VideoUpscalePipeline (models must be on a CUDA device)")
        do_cfg = guidance_scale > 1.0
        prompt_embeds = self._encode_prompt(prompt, device, num_images_per_prompt, do_cfg, negative_prompt,
                                            prompt_embeds=prompt_embeds, negative_prompt_embeds=negative_prompt_embeds)
        dtype = prompt_embeds.dtype
        if dtype not in (torch.float16, torch.float32):
            raise UavError(f"unsupported working dtype {dtype} (fp16 like the reference, or fp32)")
        rank, world = sharding.world_info(self.process_group)

        # LR image: fp32 copy for the decoder, noised working copy (pipeline...:542-551)
        image_dec = image.clone().to(dtype=torch.float32, device=device)
        image = image.to(dtype=dtype, device=device)
        noise_level_t = torch.tensor([noise_level], dtype=torch.long, device=device)
        if noise is None:
            noise = randn_tensor(image.shape, generator=generator, device=device, dtype=dtype)
        image = self.low_res_scheduler.add_noise(image, noise.to(device=device, dtype=dtype),
                                                 torch.tensor([int(noise_level)], dtype=torch.long))
        mult = (2 if do_cfg else 1) * num_images_per_prompt
        image = torch.cat([image] * mult) if mult > 1 else image
        if denoise_level is None:
            denoise_level_t = torch.cat([noise_level_t] * image.shape[0])
        else:
            denoise_level_t = torch.cat([torch.tensor([denoise_level], dtype=torch.long, device=device)] * image.shape[0])

        self.scheduler.set_timesteps(num_inference_steps, device=device)
        timesteps = getattr(self.scheduler, "timesteps_host", None) or [int(t) for t in self.scheduler.timesteps]
        C_lat = self.vae.config.latent_channels
        T, H, W = image.shape[2:]
        latents = self.prepare_latents_3d(batch_size * num_images_per_prompt, C_lat, T, H, W, dtype, device, generator, latents)
        if C_lat + image.shape[1] != self.unet.config.in_channels:
            raise ValueError(f"Incorrect configuration settings! The config of `pipeline.unet`: {self.unet.config} expects"
                             f" {self.unet.config.in_channels} but received `num_channels_latents`: {C_lat} +"
                             f" `num_channels_image`: {image.shape[1]}  = {C_lat + image.shape[1]}. Please verify the config of"
                             " `pipeline.unet` or your `image` input.")
        extra = self.prepare_extra_step_kwargs(generator, eta)
        use_prop = flows_bi is not None and self.propagator is not None
        if use_prop:
            ff, fb = flows_bi[0].to(latents).contiguous(), flows_bi[1].to(latents).contiguous()

        # both CFG halves see the same latents / LR frames / noise level: our UNet computes the text-independent prefix once
        shared = {}
        if do_cfg and num_images_per_prompt == 1 and batch_size == 1 and \
                "cfg_shared_input" in inspect.signature(self.unet.forward).parameters:
            shared = {"cfg_shared_input": True}
        windows = sharding.unet_windows(T)
        uniq = sharding.unique(windows)
        # work units of a step: whole windows, or single CFG halves of windows when that balances the ranks better
        units = sharding.window_units(len(uniq), world, can_split=do_cfg and image.shape[0] == 2)
        split = bool(units) and units[0][1] >= 0
        pe_half = [prompt_embeds[0:1], prompt_embeds[1:2]] if split else None
        fuse_step = (do_cfg and dtype == torch.float16 and batch_size * num_images_per_prompt == 1 and
                     "cfg_step" in inspect.signature(self.unet.forward).parameters and hasattr(self.scheduler, "_coefs")
                     and getattr(self.scheduler.config, "prediction_type", None) in _PRED)
        for i, t in enumerate(timesteps):
            x0_fused = None
            lat_in = torch.cat([latents] * 2) if do_cfg else latents
            if T > sharding.SHORT_SEQ:
                local = {}
                for k, (ui, half) in enumerate(units):
                    if k % world != rank:
                        continue
                    s, e = uniq[ui]
                    if half < 0:
                        local[k] = self.unet(lat_in[:, :, s:e], t, image[:, :, s:e], encoder_hidden_states=prompt_embeds,
                                             class_labels=denoise_level_t, **shared).sample
                    else:
                        local[k] = self.unet(lat_in[half:half + 1, :, s:e], t, image[half:half + 1, :, s:e],
                                             encoder_hidden_states=pe_half[half],
                                             class_labels=denoise_level_t[half:half + 1]).sample
                nb = 1 if split else lat_in.shape[0]
                got = sharding.all_gather_units(local, len(units), (nb, C_lat, sharding.SHORT_SEQ, H, W), dtype, device,
                                                self.process_group)
                outs = [torch.cat([got[2 * w], got[2 * w + 1]]) for w in range(len(uniq))] if split else got
                noise_pred = torch.empty(lat_in.shape[0], C_lat, T, H, W, dtype=dtype, device=device)
                covered = [False] * T
                for (s, e) in windows:  # reference loop order (the blend is order dependent)
                    mask = 0
                    for k in range(e - s):
                        mask |= int(covered[s + k]) << k
                        covered[s + k] = True
                    ops.window_blend(noise_pred, outs[uniq.index((s, e))].contiguous(), s, mask)
            else:
                # single window: guidance combine + step_v0 ride the UNet's last kernel (conv_out epilogue) when both the
                # UNet and the scheduler are ours; bit-identical to the three separate kernels below
                fused = None
                if fuse_step:
                    cf = self.scheduler._coefs(t)
                    fused = dict(guidance_scale=float(guidance_scale), pred_type=_PRED[self.scheduler.config.prediction_type],
                                 sqrt_alpha=cf["sa"], sqrt_beta=cf["sb"], clip=bool(self.scheduler.config.clip_sample),
                                 clip_range=float(self.scheduler.config.clip_sample_range), sample=latents.contiguous())
                r = self.unet(lat_in, t, image, encoder_hidden_states=prompt_embeds, class_labels=noise_level_t,
                              **shared, **({"cfg_step": fused} if fused is not None else {}))
                if hasattr(r, "pred_original_sample"):
                    noise_pred, x0_fused = r.noise_pred, r.pred_original_sample
                else:
                    noise_pred = r.sample
            if x0_fused is not None:
                x0 = x0_fused
            else:
                if do_cfg:
                    noise_pred = ops.cfg_combine(noise_pred.contiguous(), float(guidance_scale))
                x0 = self.scheduler.step_v0(noise_pred, t, latents, **extra).pred_original_sample
            if use_prop and i in propagation_steps:
                x0 = self.propagator(x0, ff, fb, interpolation="nearest", mode="fuse", fuse_scale=0.5, alpha1=0.001, alpha2=0.05)
            latents = self.scheduler.step_vt(x0, noise_pred, t, latents, **extra).prev_sample

        return SampledLatents(latents=latents.float(), image_dec=image_dec, w_lr=w_lr)

    @torch.no_grad()
    def decode_chunks(self, sampled: "SampledLatents") -> Iterator[Tuple[int, int, torch.Tensor]]:
        """Decode `sample_latents`' record in the reference's independent 3-frame chunks (pipeline...:668-702): yields
        `(s, e, frames)` in time order, `frames` the clamped fp32 (b, 3, e - s, 4H, 4W) output of frames [s, e).
        With several ranks, chunk k is decoded by rank k % world and each run of `world` consecutive chunks is
        exchanged in one all_gather, so every rank yields every chunk and holds at most `world` of them at a time."""
        latents, image_dec, w_lr = sampled.latents, sampled.image_dec, sampled.w_lr
        rank, world = sharding.world_info(self.process_group)
        b, _, T, H, W = latents.shape
        chunks = sharding.decode_chunks(T)
        shape = (b, self.vae.config.out_channels, sharding.DECODE_SEQ, 4 * H, 4 * W)
        for g0 in range(0, len(chunks), world):
            group = chunks[g0:g0 + world]  # chunk g0 + k belongs to rank k: g0 is a multiple of world
            local = {}
            if rank < len(group):
                s, e = group[rank]
                d = self.decode_latents_vsr(latents[:, :, s:e], image_dec[:, :, s:e], w_lr)
                if e - s < sharding.DECODE_SEQ and world > 1:  # pad the ragged last chunk for the fixed-size gather
                    pad = torch.zeros(shape, dtype=d.dtype, device=d.device)
                    pad[:, :, : e - s] = d
                    d = pad
                local[rank] = d
            outs = sharding.all_gather_units(local, len(group), shape, torch.float32, latents.device, self.process_group)
            for (s, e), o in zip(group, outs):
                yield s, e, o[:, :, : e - s]


@dataclass
class SampledLatents:
    """What `VideoUpscalePipeline.sample_latents` hands to `decode_chunks`."""
    latents: torch.Tensor    # (b, 4, T, H, W) fp32 denoised latents
    image_dec: torch.Tensor  # (b, 3, T, H, W) fp32 LR frames that condition the decoder
    w_lr: float
