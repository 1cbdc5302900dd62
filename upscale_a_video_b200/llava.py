"""LLaVA-1.5 image captioner on the uav_b200 kernels — a drop-in for the reference's `llava.llava_agent.LLavaAgent`
(same constructor and `gen_image_caption`), which the reference CLI calls once per clip on frame 0.

The model folder is a LLaVA-1.5 release (`config.json`, `pytorch_model-*.bin` or `*.safetensors` shards with their index,
the Llama sentencepiece `tokenizer.model`); the vision tower is a CLIP folder (`vision_model.*` of `pytorch_model.bin`
or `model.safetensors`, and `preprocessor_config.json`).  Every weight is held once on the GPU, in fp16: the fused
q|k|v and gate|up matrices are filled shard by shard as the checkpoint is read.

Path of one caption:
- frame preprocessing on the host (`frame0_image`, `clip_preprocess`): the reference CLI's 512 bicubic resize, then
  CLIPImageProcessor's resize / centre crop / rescale / normalise;
- vision tower: patch embedding as one GEMM (K = 588 zero-padded to 592), class and position embeddings,
  pre-LayerNorm, then the CLIP encoder layers (`clip_text.encoder_layer`, bidirectional) up to `mm_vision_select_layer`;
  the CLS token is dropped;
- projector `mlp2x_gelu`: two GEMMs, the second writing straight into the image rows of the prompt's embeddings;
- Llama prefill: GEMMs for q|k|v, o (+ residual), gate|up and down (+ residual), RMSNorm, RoPE with the KV-cache
  append, causal attention; only the last row goes through lm_head;
- decode, one token at a time: the same layers on one row with the GEMV weight stream and attention against the
  KV cache; the sampler picks the token on the device from one uniform drawn from `generator` on the host.
Up to CAPTION_BATCH images go through this path together: one vision-tower batch, one prefill of B x n rows and one
decode step for all B rows, so each decoded token streams the weights once for the whole batch.  Every kernel on the
path gives each row the arithmetic of the one-row path, so a row's tokens do not depend on the rest of its batch.
There is no CPU path."""
from __future__ import annotations

import json
import os
from types import SimpleNamespace
from typing import List, Optional

import numpy as np
import torch
import torch.nn.functional as F

from . import _lib, ops
from .clip_text import encoder_layer

__all__ = ["LLavaAgent", "IMAGE_TOKEN_INDEX", "conversation_prompt", "tokenize_prompt", "postprocess_caption",
           "frame0_image", "clip_preprocess", "llava_key_map", "CAPTION_BATCH", "caption_groups"]

IMAGE_TOKEN_INDEX = -200  # llava/constants.py
DEFAULT_IMAGE_TOKEN = "<image>"
DEFAULT_QS = "Describe this image and its style in a very detailed manner."
VICUNA_V1_SYSTEM = ("A chat between a curious user and an artificial intelligence assistant. "
                    "The assistant gives helpful, detailed, and polite answers to the user's questions.")
STOP_STR = "</s>"           # vicuna_v1's sep2
MAX_NEW_TOKENS = 64         # llava_agent.py: generate(max_new_tokens=64)
FRAME_SHORT_SIDE = 512      # inference_upscale_a_video.py: fix_resize
PATCH_K_PADDED = 592        # 3 * 14 * 14 = 588 patch values, padded to a multiple of 16 for the GEMM
CAPTION_BATCH = 8           # images per weight pass: the batched GEMV and sampler take up to 8 rows


# ---------------------------------------------------------------------------------------------------------------
# prompt, tokens, caption text
# ---------------------------------------------------------------------------------------------------------------
def conversation_prompt(qs: str = DEFAULT_QS) -> str:
    """the `vicuna_v1` conversation with the image placeholder and the question, ending at the assistant's turn"""
    return f"{VICUNA_V1_SYSTEM} USER: {DEFAULT_IMAGE_TOKEN}\n{qs} ASSISTANT:"


def tokenize_prompt(prompt: str, encode, bos_id: int) -> List[int]:
    """LLaVA's `tokenizer_image_token`: each `<image>`-separated chunk is tokenised on its own as the Llama tokenizer
    does (`[bos] + encode(chunk)`), the chunks are joined without their bos, one `IMAGE_TOKEN_INDEX` between them, and
    the prompt starts with one bos"""
    ids = [bos_id]
    for i, chunk in enumerate(prompt.split(DEFAULT_IMAGE_TOKEN)):
        if i:
            ids.append(IMAGE_TOKEN_INDEX)
        ids.extend(encode(chunk))
    return ids


def postprocess_caption(text: str) -> str:
    """llava_agent.py: strip, drop a trailing `</s>`, strip again, newlines become spaces"""
    out = text.strip()
    if out.endswith(STOP_STR):
        out = out[:-len(STOP_STR)]
    return out.strip().replace("\n", " ").replace("\r", " ")


# ---------------------------------------------------------------------------------------------------------------
# image preprocessing (host)
# ---------------------------------------------------------------------------------------------------------------
def frame0_image(frame_rgb: np.ndarray):
    """inference_upscale_a_video.py's caption input: a (h, w, 3) uint8 RGB frame, bicubically resized (torch, fp32, on
    the CPU) so that its short side is 512, clipped, truncated to uint8, as a PIL image"""
    from PIL import Image
    h, w = frame_rgb.shape[:2]
    scale = FRAME_SHORT_SIDE / min(w, h)
    w0, h0 = round(w * scale), round(h * scale)
    x = torch.from_numpy(np.ascontiguousarray(frame_rgb)).permute(2, 0, 1)[None].float()
    x = F.interpolate(x, size=(h0, w0), mode="bicubic")
    return Image.fromarray(x[0].permute(1, 2, 0).numpy().clip(0, 255).astype(np.uint8))


def clip_preprocess(image, cfg: dict) -> torch.Tensor:
    """CLIPImageProcessor as configured by a `preprocessor_config.json`: short side to `size` with PIL (bicubic by
    default), centre crop, rescale, normalise -> (3, crop, crop) fp16, as LLaVA feeds the vision tower"""
    from PIL import Image
    size = cfg.get("size", 336)
    short = size["shortest_edge"] if isinstance(size, dict) else int(size)
    crop = cfg.get("crop_size", short)
    ch, cw = (crop["height"], crop["width"]) if isinstance(crop, dict) else (int(crop), int(crop))
    image = image.convert("RGB")
    w, h = image.size
    if cfg.get("do_resize", True):
        if w <= h:
            nw, nh = short, int(short * h / w)
        else:
            nw, nh = int(short * w / h), short
        image = image.resize((nw, nh), resample=Image.Resampling(cfg.get("resample", 3)))
    a = np.asarray(image)
    if cfg.get("do_center_crop", True):
        top, left = (a.shape[0] - ch) // 2, (a.shape[1] - cw) // 2
        a = a[top:top + ch, left:left + cw]
    a = (a.astype(np.float64) * cfg.get("rescale_factor", 1 / 255)).astype(np.float32)
    if cfg.get("do_normalize", True):
        a = (a - np.array(cfg["image_mean"], dtype=np.float32)) / np.array(cfg["image_std"], dtype=np.float32)
    return torch.from_numpy(np.ascontiguousarray(a.transpose(2, 0, 1))).half()


# ---------------------------------------------------------------------------------------------------------------
# checkpoints
# ---------------------------------------------------------------------------------------------------------------
def _shard_files(folder: str) -> List[str]:
    for index in ("model.safetensors.index.json", "pytorch_model.bin.index.json"):
        p = os.path.join(folder, index)
        if os.path.exists(p):
            return [os.path.join(folder, f) for f in sorted(set(json.load(open(p))["weight_map"].values()))]
    for single in ("model.safetensors", "pytorch_model.bin"):
        p = os.path.join(folder, single)
        if os.path.exists(p):
            return [p]
    raise FileNotFoundError(f"no model.safetensors / pytorch_model.bin (or their shard index) in {folder}")


def _iter_tensors(files: List[str]):
    """(key, CPU tensor) of every tensor of the shards, one shard held at a time (memory-mapped)"""
    for f in files:
        if f.endswith(".safetensors"):
            from safetensors import safe_open
            with safe_open(f, framework="pt") as st:
                for k in st.keys():
                    yield k, st.get_tensor(k)
        else:
            sd = torch.load(f, map_location="cpu", mmap=True, weights_only=True)
            yield from sd.items()
            del sd


def llava_key_map(cfg: SimpleNamespace) -> dict:
    """released key -> (destination name, row offset) of the decoder and projector: q, k, v land in row blocks of one
    q|k|v matrix and gate, up in one gate|up matrix"""
    H, I = cfg.hidden_size, cfg.intermediate_size
    m = {"model.embed_tokens.weight": ("embed", 0), "model.norm.weight": ("norm", 0), "lm_head.weight": ("lm_head", 0),
         "model.mm_projector.0.weight": ("proj0_w", 0), "model.mm_projector.0.bias": ("proj0_b", 0),
         "model.mm_projector.2.weight": ("proj2_w", 0), "model.mm_projector.2.bias": ("proj2_b", 0)}
    for i in range(cfg.num_hidden_layers):
        p = f"model.layers.{i}."
        m.update({p + "self_attn.q_proj.weight": (f"qkv{i}", 0), p + "self_attn.k_proj.weight": (f"qkv{i}", H),
                  p + "self_attn.v_proj.weight": (f"qkv{i}", 2 * H), p + "self_attn.o_proj.weight": (f"o{i}", 0),
                  p + "mlp.gate_proj.weight": (f"gu{i}", 0), p + "mlp.up_proj.weight": (f"gu{i}", I),
                  p + "mlp.down_proj.weight": (f"down{i}", 0), p + "input_layernorm.weight": (f"ln1_{i}", 0),
                  p + "post_attention_layernorm.weight": (f"ln2_{i}", 0)})
    return m


def _decoder_shapes(cfg: SimpleNamespace) -> dict:
    H, I, V, Hv = cfg.hidden_size, cfg.intermediate_size, cfg.vocab_size, cfg.mm_hidden_size
    s = {"embed": ((V, H), torch.float16), "norm": ((H,), torch.float16), "lm_head": ((V, H), torch.float16),
         "proj0_w": ((H, Hv), torch.float16), "proj0_b": ((H,), torch.float32),
         "proj2_w": ((H, H), torch.float16), "proj2_b": ((H,), torch.float32)}
    for i in range(cfg.num_hidden_layers):
        s.update({f"qkv{i}": ((3 * H, H), torch.float16), f"o{i}": ((H, H), torch.float16),
                  f"gu{i}": ((2 * I, H), torch.float16), f"down{i}": ((H, I), torch.float16),
                  f"ln1_{i}": ((H,), torch.float16), f"ln2_{i}": ((H,), torch.float16)})
    return s


def load_decoder(folder: str, cfg: SimpleNamespace, device) -> dict:
    """the decoder and projector weights of a released LLaVA-1.5 folder, each held once on `device`.  Keys other than
    the expected ones (`rotary_emb.inv_freq` buffers aside) and missing keys are errors."""
    keymap, shapes = llava_key_map(cfg), _decoder_shapes(cfg)
    out = {name: torch.empty(shape, dtype=dt, device=device) for name, (shape, dt) in shapes.items()}
    filled = set()
    unexpected = []
    for k, t in _iter_tensors(_shard_files(folder)):
        if k not in keymap:
            if not k.endswith("rotary_emb.inv_freq"):
                unexpected.append(k)
            continue
        name, row = keymap[k]
        dst = out[name]
        if dst.dim() == 2:
            dst = dst[row:row + t.shape[0]]
        if tuple(dst.shape) != tuple(t.shape):
            raise RuntimeError(f"{k}: shape {tuple(t.shape)} does not fit {tuple(dst.shape)}")
        dst.copy_(t)
        filled.add(k)
    if unexpected:
        raise RuntimeError(f"unexpected keys in the LLaVA checkpoint: {unexpected[:5]}")
    missing = sorted(set(keymap) - filled)
    if missing:
        raise RuntimeError(f"missing keys in the LLaVA checkpoint: {missing[:5]}")
    return out


def load_vision_tower(folder: str, vcfg: SimpleNamespace, layers: int, device) -> SimpleNamespace:
    """the first `layers` encoder layers, embeddings and pre-LayerNorm of a CLIP vision checkpoint, kernel-ready on
    `device` (fused q|k|v, fp16 weights, fp32 biases and LayerNorm affines)"""
    want = {"vision_model.embeddings.class_embedding", "vision_model.embeddings.patch_embedding.weight",
            "vision_model.embeddings.position_embedding.weight", "vision_model.pre_layrnorm.weight",
            "vision_model.pre_layrnorm.bias"}
    parts = ("self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.out_proj", "layer_norm1",
             "layer_norm2", "mlp.fc1", "mlp.fc2")
    for i in range(layers):
        for p in parts:
            want |= {f"vision_model.encoder.layers.{i}.{p}.weight", f"vision_model.encoder.layers.{i}.{p}.bias"}
    sd = {}
    for k, t in _iter_tensors(_shard_files(folder)):
        if k in want:
            sd[k] = t.to(device)
    missing = sorted(want - set(sd))
    if missing:
        raise RuntimeError(f"missing keys in the CLIP vision checkpoint {folder}: {missing[:5]}")
    h16 = lambda k: sd.pop(k).to(torch.float16).contiguous()
    f32 = lambda k: sd.pop(k).float().contiguous()
    e = "vision_model.embeddings."
    pw = h16(e + "patch_embedding.weight").reshape(vcfg.hidden_size, -1)
    tower = SimpleNamespace(patch_w=F.pad(pw, (0, PATCH_K_PADDED - pw.shape[1])).contiguous(),
                            cls=h16(e + "class_embedding"), pos=h16(e + "position_embedding.weight"),
                            pre_ln=(f32("vision_model.pre_layrnorm.weight"), f32("vision_model.pre_layrnorm.bias")),
                            layers=[])
    for i in range(layers):
        p = f"vision_model.encoder.layers.{i}."
        lin = lambda n: (h16(p + n + ".weight"), f32(p + n + ".bias"))
        q, k, v = lin("self_attn.q_proj"), lin("self_attn.k_proj"), lin("self_attn.v_proj")
        tower.layers.append(SimpleNamespace(
            ln1=(f32(p + "layer_norm1.weight"), f32(p + "layer_norm1.bias")),
            qkv=(torch.cat([q[0], k[0], v[0]]).contiguous(), torch.cat([q[1], k[1], v[1]]).contiguous()),
            out=lin("self_attn.out_proj"), ln2=(f32(p + "layer_norm2.weight"), f32(p + "layer_norm2.bias")),
            fc1=lin("mlp.fc1"), fc2=lin("mlp.fc2")))
        del q, k, v
    return tower


def caption_groups(n: int) -> List[range]:
    """indices [0, n) in consecutive groups of at most CAPTION_BATCH, the batches `gen_image_caption` runs"""
    return [range(i, min(i + CAPTION_BATCH, n)) for i in range(0, n, CAPTION_BATCH)]


def _caption_generators(n: int, temperature: float, generator):
    """(one generator per image, whether the images may share a batch).  A list of distinct generators gives each
    image its own uniforms, drawn as a one-image call draws them, so batching cannot change them; greedy decoding
    draws none.  A generator shared by several images (a single generator, None for the global RNG, or one object
    listed twice) at temperature > 0 is drawn across those images in the one-at-a-time loop's order, which only that
    loop reproduces."""
    if isinstance(generator, (list, tuple)):
        if len(generator) != n:
            raise ValueError(f"generator: a list of {len(generator)} generators for {n} images; pass one per image")
        gens = list(generator)
        distinct = None not in gens and len({id(g) for g in gens}) == n
        return gens, temperature == 0 or distinct
    return [generator] * n, temperature == 0


# ---------------------------------------------------------------------------------------------------------------
# the agent
# ---------------------------------------------------------------------------------------------------------------
class LLavaAgent:
    """`llava.llava_agent.LLavaAgent` on the uav_b200 kernels: fp16 weights, greedy decoding at temperature 0, top-p
    sampling otherwise, with the uniforms drawn from `generator` (the global RNG when None)"""

    def __init__(self, model_path, device="cuda", conv_mode="vicuna_v1", load_8bit=False, load_4bit=False, *,
                 vision_tower_path=None):
        if load_8bit or load_4bit:
            raise NotImplementedError("LLavaAgent runs in fp16: 8-bit and 4-bit loading are not supported")
        if conv_mode != "vicuna_v1":
            raise NotImplementedError(f"conv_mode {conv_mode!r}: only 'vicuna_v1' (LLaVA-1.5) is supported")
        model_path = os.path.expanduser(model_path)
        if not os.path.isdir(model_path):
            raise EnvironmentError(f"{model_path} is not a local LLaVA-1.5 folder (config.json, weight shards, "
                                   f"tokenizer.model)")
        raw = json.load(open(os.path.join(model_path, "config.json")))
        cfg = SimpleNamespace(hidden_size=raw["hidden_size"], intermediate_size=raw["intermediate_size"],
                              num_hidden_layers=raw["num_hidden_layers"], num_attention_heads=raw["num_attention_heads"],
                              num_key_value_heads=raw.get("num_key_value_heads", raw["num_attention_heads"]),
                              rms_norm_eps=raw.get("rms_norm_eps", 1e-6), rope_theta=raw.get("rope_theta", 10000.0),
                              vocab_size=raw["vocab_size"], mm_hidden_size=raw.get("mm_hidden_size", 1024),
                              mm_projector_type=raw.get("mm_projector_type", "linear"),
                              mm_vision_select_layer=raw.get("mm_vision_select_layer", -2),
                              mm_vision_select_feature=raw.get("mm_vision_select_feature", "patch"),
                              mm_use_im_start_end=raw.get("mm_use_im_start_end", False),
                              rope_scaling=raw.get("rope_scaling"))
        if cfg.hidden_size // cfg.num_attention_heads != 128 or cfg.hidden_size % cfg.num_attention_heads:
            raise NotImplementedError(f"head_dim {cfg.hidden_size / cfg.num_attention_heads:g}: the kernels take 128")
        if cfg.num_key_value_heads != cfg.num_attention_heads:
            raise NotImplementedError("grouped-query attention (num_key_value_heads != num_attention_heads)")
        if cfg.mm_projector_type != "mlp2x_gelu":
            raise NotImplementedError(f"mm_projector_type {cfg.mm_projector_type!r}: only 'mlp2x_gelu' (LLaVA-1.5)")
        if cfg.mm_vision_select_feature != "patch" or cfg.mm_use_im_start_end or cfg.rope_scaling:
            raise NotImplementedError("only LLaVA-1.5's patch features, without image start/end tokens or RoPE scaling")
        vt = vision_tower_path
        if vt is None:
            cand = raw.get("mm_vision_tower")
            vt = cand if cand and os.path.isdir(cand) else None
        if vt is None or not os.path.isdir(vt):
            raise EnvironmentError(f"no CLIP vision tower folder: vision_tower_path={vision_tower_path!r}, config "
                                   f"mm_vision_tower={raw.get('mm_vision_tower')!r}; pass an existing folder")
        import sentencepiece as spm
        self.sp = spm.SentencePieceProcessor(model_file=os.path.join(model_path, "tokenizer.model"))
        self.bos_id, self.eos_id = self.sp.bos_id(), self.sp.eos_id()
        self.special_ids = {i for i in (self.sp.unk_id(), self.bos_id, self.eos_id) if i >= 0}

        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _lib.UavError("LLavaAgent: CUDA device required — uav_b200 has no CPU path")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.config = cfg
        vraw = json.load(open(os.path.join(vt, "config.json")))
        vraw = vraw.get("vision_config", vraw)
        self.vision_config = SimpleNamespace(hidden_size=vraw.get("hidden_size", 1024),
                                             num_hidden_layers=vraw.get("num_hidden_layers", 24),
                                             num_attention_heads=vraw.get("num_attention_heads", 16),
                                             image_size=vraw.get("image_size", 336), patch_size=vraw.get("patch_size", 14),
                                             hidden_act=vraw.get("hidden_act", "quick_gelu"),
                                             layer_norm_eps=vraw.get("layer_norm_eps", 1e-5))
        vc = self.vision_config
        if vc.patch_size * vc.patch_size * 3 > PATCH_K_PADDED or vc.hidden_size != cfg.mm_hidden_size:
            raise NotImplementedError("the vision tower must have 14-pixel patches (or smaller) and mm_hidden_size columns")
        if vc.hidden_act not in ("gelu", "quick_gelu"):
            raise NotImplementedError(f"vision hidden_act {vc.hidden_act!r}")
        self.image_processor = json.load(open(os.path.join(vt, "preprocessor_config.json")))
        sel = cfg.mm_vision_select_layer
        self.vision_layers = sel + vc.num_hidden_layers + 1 if sel < 0 else sel
        if not 0 <= self.vision_layers <= vc.num_hidden_layers:
            raise ValueError(f"mm_vision_select_layer {sel} out of range for {vc.num_hidden_layers} layers")
        with torch.cuda.device(self.device):
            self.tower = load_vision_tower(vt, vc, self.vision_layers, self.device)
            self.w = load_decoder(model_path, cfg, self.device)
        self.qs = DEFAULT_QS
        self.conv_mode = conv_mode
        self.max_new_tokens = MAX_NEW_TOKENS

    # ---- model pieces ----
    def _rope_table(self, positions: int) -> torch.Tensor:
        """fp32 (positions, 64, 2) cos, sin of position * inv_freq, as transformers' LlamaRotaryEmbedding computes them"""
        inv_freq = 1.0 / (self.config.rope_theta ** (torch.arange(0, 128, 2, dtype=torch.int64).float() / 128))
        freqs = torch.arange(positions, dtype=torch.int64).float()[:, None] * inv_freq[None]
        return torch.stack([freqs.cos(), freqs.sin()], dim=-1).to(self.device).contiguous()

    @torch.no_grad()
    def vision_features(self, pixel_values: torch.Tensor) -> torch.Tensor:
        """(3, S, S) preprocessed image (host or device) -> (patches, mm_hidden_size) fp16 features of the selected layer,
        CLS dropped; (B, 3, S, S) images -> (B, patches, mm_hidden_size), the encoder layers run on all B at once"""
        vc, t = self.vision_config, self.tower
        ps = vc.patch_size
        g = vc.image_size // ps
        px = pixel_values.to(torch.float16).cpu()
        one = px.dim() == 3
        px = px[None] if one else px
        B = px.shape[0]
        assert px.shape[1:] == (3, vc.image_size, vc.image_size), px.shape
        patches = px.view(B, 3, g, ps, g, ps).permute(0, 2, 4, 1, 3, 5).reshape(B * g * g, 3 * ps * ps)
        patches = F.pad(patches, (0, PATCH_K_PADDED - patches.shape[1])).to(self.device)
        emb = ops.linear(patches, t.patch_w).view(B, g * g, -1)
        cls = t.cls[None, None].expand(B, 1, -1)
        x = (torch.cat([cls, emb], 1).float() + t.pos.float()).to(torch.float16)  # one rounding
        x = ops.layer_norm(x, *t.pre_ln, vc.layer_norm_eps)
        act = ops.ACT_GELU if vc.hidden_act == "gelu" else ops.ACT_QUICK_GELU
        for w in t.layers:
            x = encoder_layer(x, w, vc.num_attention_heads, vc.layer_norm_eps, act, causal=False)
        return x[0, 1:] if one else x[:, 1:]

    # The layers take B sequences: x holds B x n prefill rows (sequence-major) or B decode rows, and the caches are
    # (B, L_max, hidden) (or (L_max, hidden) for B = 1).  The prefill GEMMs run on all B x n rows: uav_linear picks its
    # tile width from N alone for a single-tap GEMM without GEGLU, so each output element's k-order does not depend on
    # M, and a sequence's rows come out as they do in a prefill of that sequence alone.
    def _layer_prefill(self, i, x, kc, vc_, rope):
        cfg, w = self.config, self.w
        H, heads, eps = cfg.hidden_size, cfg.num_attention_heads, cfg.rms_norm_eps
        if kc.dim() == 2:
            kc, vc_ = kc[None], vc_[None]
        B = kc.shape[0]
        n = x.shape[0] // B
        qkv = ops.linear(ops.rms_norm(x, w[f"ln1_{i}"], eps), w[f"qkv{i}"])
        ops.rope_kv_append_batched(qkv.view(B, n, -1), heads, 0, rope, kc, vc_)
        o = torch.empty(B * n, H, dtype=torch.float16, device=x.device)
        for b in range(B):  # the causal kernel reads a batch's keys n rows apart; each cache is L_max rows long
            ops.attention_causal(qkv[b * n:(b + 1) * n, :H].unsqueeze(0), kc[b, :n].unsqueeze(0),
                                 vc_[b, :n].unsqueeze(0), heads, out=o[b * n:(b + 1) * n].unsqueeze(0))
        x = ops.linear(o, w[f"o{i}"], residual=x)
        gu = ops.linear(ops.rms_norm(x, w[f"ln2_{i}"], eps), w[f"gu{i}"])
        return ops.linear(ops.swiglu(gu), w[f"down{i}"], residual=x)

    def _layer_decode(self, i, x, pos, kc, vc_, rope):
        cfg, w = self.config, self.w
        H, heads, eps = cfg.hidden_size, cfg.num_attention_heads, cfg.rms_norm_eps
        if kc.dim() == 2:
            kc, vc_ = kc[None], vc_[None]
        B = x.shape[0]
        qkv = ops.gemv_rows(w[f"qkv{i}"], ops.rms_norm(x, w[f"ln1_{i}"], eps))
        ops.rope_kv_append_batched(qkv.view(B, 1, -1), heads, pos, rope, kc, vc_)
        o = ops.attention_decode_batched(qkv[:, :H], kc, vc_, pos + 1, heads)
        x = ops.gemv_rows(w[f"o{i}"], o, residual=x)
        gu = ops.gemv_rows(w[f"gu{i}"], ops.rms_norm(x, w[f"ln2_{i}"], eps))
        return ops.gemv_rows(w[f"down{i}"], ops.swiglu(gu), residual=x)

    def _logits(self, x_rows):
        """fp32 (B, vocab) logits of the rows x_rows (B, hidden) (a strided row view allowed)"""
        h = ops.rms_norm(x_rows, self.w["norm"], self.config.rms_norm_eps)
        return ops.gemv_rows(self.w["lm_head"], h, out_dtype=torch.float32)

    def prompt_ids(self, qs: Optional[str] = None) -> List[int]:
        prompt = conversation_prompt(self.qs if qs is None else qs)
        return tokenize_prompt(prompt, self.sp.encode, self.bos_id)

    @torch.no_grad()
    def embed_prompt(self, ids: List[int], features: torch.Tensor) -> torch.Tensor:
        """(n, hidden) fp16 prefill rows: token embeddings, with the `IMAGE_TOKEN_INDEX` placeholder replaced by the
        projected image features (the projector's second GEMM writes into those rows).  Features of B images
        (B, patches, mm_hidden_size) give (B, n, hidden)."""
        w, H = self.w, self.config.hidden_size
        one = features.dim() == 2
        feats = features[None] if one else features
        B, n_img = feats.shape[:2]
        at = ids.index(IMAGE_TOKEN_INDEX)
        text = torch.tensor(ids[:at] + ids[at + 1:], dtype=torch.int64, device=self.device)
        tok = w["embed"].index_select(0, text)
        x = torch.empty(B, len(ids) - 1 + n_img, H, dtype=torch.float16, device=self.device)
        x[:, :at] = tok[:at]
        x[:, at + n_img:] = tok[at:]
        h = ops.linear(feats.reshape(B * n_img, -1), w["proj0_w"], w["proj0_b"], act=ops.ACT_GELU)
        for b in range(B):
            ops.linear(h[b * n_img:(b + 1) * n_img], w["proj2_w"], w["proj2_b"], out=x[b, at:at + n_img])
        return x[0] if one else x

    @torch.no_grad()
    def forward_logits(self, x: torch.Tensor, forced: List[int]) -> List[torch.Tensor]:
        """fp32 logits (vocab,) of the last prefill row of `x` (n, hidden), then of each decode step fed the tokens
        `forced` (teacher forcing): `forward_logits_batch` of one sequence"""
        return [logits[0] for logits in self.forward_logits_batch(x[None], [forced])]

    @torch.no_grad()
    def forward_logits_batch(self, x: torch.Tensor, forced: List[List[int]]) -> List[torch.Tensor]:
        """fp32 logits (B, vocab) of the last prefill row of each sequence of `x` (B, n, hidden), then of each decode
        step, row b fed the tokens forced[b] (teacher forcing; every row forces the same number of tokens)"""
        B = x.shape[0]
        steps = len(forced[0])
        assert len(forced) == B and all(len(f) == steps for f in forced), "one list of forced tokens per row, equal lengths"

        def pick(step, logits):
            if step >= steps:
                return None
            return torch.tensor([f[step] for f in forced], dtype=torch.int64, device=self.device)

        with torch.cuda.device(self.device):
            return list(self._run(x, steps + 1, pick))

    def _run(self, x, max_new, pick):
        """prefill x (B, n, hidden), then decode the B sequences together; pick(step, logits) -> device int64 (B,)
        token ids or None to stop; yields the fp32 (B, vocab) logits of every step"""
        cfg = self.config
        B, n, H = x.shape
        L = n + max_new
        cache = torch.empty(cfg.num_hidden_layers, 2, B, L, H, dtype=torch.float16, device=self.device)
        rope = self._rope_table(L)
        x = x.reshape(B * n, H)
        for i in range(cfg.num_hidden_layers):
            x = self._layer_prefill(i, x, cache[i, 0], cache[i, 1], rope)
        logits = self._logits(x.view(B, n, H)[:, n - 1])
        for step in range(max_new):
            yield logits
            tok = pick(step, logits)
            if tok is None or step == max_new - 1:
                return
            xr = self.w["embed"].index_select(0, tok.view(B))
            for i in range(cfg.num_hidden_layers):
                xr = self._layer_decode(i, xr, n + step, cache[i, 0], cache[i, 1], rope)
            logits = self._logits(xr)

    @torch.no_grad()
    def generate_ids(self, pixel_values: torch.Tensor, temperature=0.2, top_p=0.7, qs=None, generator=None,
                     max_new_tokens: Optional[int] = None) -> List[int]:
        """the new token ids (EOS included when reached) for one preprocessed image"""
        return self.generate_ids_batch(pixel_values[None], temperature, top_p, qs, [generator], max_new_tokens)[0]

    @torch.no_grad()
    def generate_ids_batch(self, pixel_values: torch.Tensor, temperature=0.2, top_p=0.7, qs=None, generators=None,
                           max_new_tokens: Optional[int] = None) -> List[List[int]]:
        """the new token ids (EOS included when reached) of each of B <= CAPTION_BATCH preprocessed images
        (B, 3, S, S), decoded together.  Row b draws one uniform per token from generators[b] (None: the global RNG)
        until it emits EOS, as `generate_ids` of that image alone does; a finished row is fed EOS and its outputs are
        ignored.  Decoding ends when every row has finished or after max_new_tokens."""
        B = pixel_values.shape[0]
        assert 1 <= B <= CAPTION_BATCH, B
        generators = [None] * B if generators is None else list(generators)
        assert len(generators) == B
        ids = self.prompt_ids(qs)
        out: List[List[int]] = [[] for _ in range(B)]
        done = [False] * B
        with torch.cuda.device(self.device):
            x = self.embed_prompt(ids, self.vision_features(pixel_values))
            tok_buf = torch.empty(B, dtype=torch.int64, device=self.device)

            def pick(step, logits):
                us = []
                for b, g in enumerate(generators):
                    u = 0.0
                    if temperature > 0 and not done[b]:
                        gdev = g.device if g is not None else "cpu"
                        u = float(torch.rand((), generator=g, device=gdev, dtype=torch.float64).item())
                    us.append(min(u, 1.0 - 2 ** -24))
                tok = ops.sample_top_p_batched(logits, float(temperature), float(top_p), us, out=tok_buf)
                toks = tok.tolist()  # the host reads the B tokens back once per step, to stop at EOS
                for b, t in enumerate(toks):
                    if not done[b]:
                        out[b].append(t)
                        done[b] = t == self.eos_id
                if all(done):
                    return None
                if any(done):
                    return torch.tensor([self.eos_id if d else t for d, t in zip(done, toks)], dtype=torch.int64,
                                        device=self.device)
                return tok

            for _ in self._run(x, max_new_tokens or self.max_new_tokens, pick):
                pass
        return out

    def decode(self, ids: List[int]) -> str:
        """`batch_decode(skip_special_tokens=True)` of one sequence"""
        return self.sp.decode([i for i in ids if i not in self.special_ids])

    def gen_image_caption(self, imgs, temperature=0.2, top_p=0.7, num_beams=1, qs=None, *, generator=None):
        """one caption per PIL image, as the reference's agent returns them.  `generator` is one torch.Generator for
        all images, or a list of one per image; None draws from the global RNG.  The images are decoded in batches of
        up to CAPTION_BATCH when that gives the captions of one-image calls: greedily (temperature 0) or with a
        list of distinct generators.  A generator shared between images (a single one, None, or one object listed
        twice) at temperature > 0 captions the images one at a time."""
        if num_beams != 1:
            raise NotImplementedError("beam search (num_beams > 1) is not supported")
        if temperature < 0:
            raise ValueError("temperature must be >= 0")
        gens, batched = _caption_generators(len(imgs), temperature, generator)
        groups = caption_groups(len(imgs)) if batched else [range(i, i + 1) for i in range(len(imgs))]
        caps = []
        for group in groups:
            px = torch.stack([clip_preprocess(imgs[i], self.image_processor) for i in group])
            for ids in self.generate_ids_batch(px, temperature, top_p, qs, [gens[i] for i in group]):
                caps.append(postprocess_caption(self.decode(ids)))
        return caps
