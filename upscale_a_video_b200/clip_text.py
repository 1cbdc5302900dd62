"""CLIP text encoder on the uav_b200 kernels — a drop-in for the `transformers.CLIPTextModel` that the reference pipeline holds
as `pipeline.text_encoder` (pipeline_upscale_a_video.py:239-245; SURVEY.md §8f rank 3): same state-dict keys
(`text_model.*`), same call (`model(input_ids, attention_mask=None)[0]` = last hidden state), `.config`, `.dtype`.

Per layer: LayerNorm -> fused q|k|v GEMM -> causal attention over the (<= 128 token) prompt -> out-proj GEMM with the
residual in its epilogue -> LayerNorm -> fc1 GEMM with GELU / quick-GELU in its epilogue -> fc2 GEMM with the residual.
The embedding lookup is an index_select on the fp16 tables.  There is no CPU path.  Padding masks are not supported
(`use_attention_mask` is false for the x4-upscaler's encoder: the reference passes `attention_mask=None`)."""
from __future__ import annotations

from types import SimpleNamespace
from typing import Optional

import torch
from torch import nn

from . import _lib, ops
from .layers import PackedModule

__all__ = ["CLIPTextConfig", "CLIPTextModel", "encoder_layer"]


def encoder_layer(x: torch.Tensor, w, heads: int, eps: float, act: int, causal: bool) -> torch.Tensor:
    """one pre-LayerNorm CLIP encoder layer on x (b, n, hidden) fp16, shared by the text encoder (causal) and LLaVA's
    vision tower (llava.py, bidirectional).  `w` holds the kernel-ready weights: ln1 / ln2 (fp32 gamma, beta), qkv, out,
    fc1, fc2 (fp16 weight, fp32 bias or None), the q|k|v projections row-concatenated."""
    hidden = x.shape[-1]
    h = ops.layer_norm(x, *w.ln1, eps)
    qkv = ops.linear(h, *w.qkv)
    attn = ops.attention_causal if causal else ops.attention
    o = attn(qkv[..., :hidden], qkv[..., hidden:2 * hidden], qkv[..., 2 * hidden:], heads)
    x = ops.linear(o, *w.out, residual=x)
    h = ops.layer_norm(x, *w.ln2, eps)
    return ops.linear(ops.linear(h, *w.fc1, act=act), *w.fc2, residual=x)


class CLIPTextConfig(SimpleNamespace):
    def __init__(self, vocab_size=49408, hidden_size=1024, intermediate_size=4096, num_hidden_layers=23, num_attention_heads=16,
                 max_position_embeddings=77, hidden_act="gelu", layer_norm_eps=1e-5, **extra):
        super().__init__(vocab_size=vocab_size, hidden_size=hidden_size, intermediate_size=intermediate_size,
                         num_hidden_layers=num_hidden_layers, num_attention_heads=num_attention_heads,
                         max_position_embeddings=max_position_embeddings, hidden_act=hidden_act, layer_norm_eps=layer_norm_eps,
                         use_attention_mask=False, **extra)


class _Attn(nn.Module):
    def __init__(self, h):
        super().__init__()
        self.k_proj, self.v_proj, self.q_proj, self.out_proj = (nn.Linear(h, h) for _ in range(4))


class _MLP(nn.Module):
    def __init__(self, h, inter):
        super().__init__()
        self.fc1, self.fc2 = nn.Linear(h, inter), nn.Linear(inter, h)


class _Layer(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.self_attn = _Attn(cfg.hidden_size)
        self.layer_norm1 = nn.LayerNorm(cfg.hidden_size, eps=cfg.layer_norm_eps)
        self.mlp = _MLP(cfg.hidden_size, cfg.intermediate_size)
        self.layer_norm2 = nn.LayerNorm(cfg.hidden_size, eps=cfg.layer_norm_eps)


class _Embeddings(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.token_embedding = nn.Embedding(cfg.vocab_size, cfg.hidden_size)
        self.position_embedding = nn.Embedding(cfg.max_position_embeddings, cfg.hidden_size)


class _Encoder(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.layers = nn.ModuleList([_Layer(cfg) for _ in range(cfg.num_hidden_layers)])


class _TextTransformer(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.embeddings = _Embeddings(cfg)
        self.encoder = _Encoder(cfg)
        self.final_layer_norm = nn.LayerNorm(cfg.hidden_size, eps=cfg.layer_norm_eps)


class CLIPTextModel(PackedModule):
    def __init__(self, config: CLIPTextConfig):
        super().__init__()
        if config.hidden_act not in ("gelu", "quick_gelu"):
            raise NotImplementedError(f"hidden_act={config.hidden_act!r}")
        if config.hidden_size % config.num_attention_heads or (config.hidden_size // config.num_attention_heads) % 2:
            raise ValueError("hidden_size must be a multiple of num_attention_heads with an even head_dim")
        self.config = config
        self.text_model = _TextTransformer(config)

    @property
    def dtype(self):
        return next(self.parameters()).dtype

    @property
    def device(self):
        return next(self.parameters()).device

    @classmethod
    def from_pretrained(cls, path: str, torch_dtype=None, **_):
        """`transformers.CLIPTextModel.from_pretrained(dir)` for a local directory: `config.json` (a `text_config` block is
        unwrapped) + `model.safetensors` or `pytorch_model.bin` with transformers' own key names"""
        import json
        import os
        cfg = json.load(open(os.path.join(path, "config.json")))
        cfg = cfg.get("text_config", cfg)
        keys = ("vocab_size", "hidden_size", "intermediate_size", "num_hidden_layers", "num_attention_heads",
                "max_position_embeddings", "hidden_act", "layer_norm_eps")
        model = cls(CLIPTextConfig(**{k: cfg[k] for k in keys if k in cfg}))
        st = os.path.join(path, "model.safetensors")
        if os.path.exists(st):
            from safetensors.torch import load_file
            sd = load_file(st)
        else:
            sd = torch.load(os.path.join(path, "pytorch_model.bin"), map_location="cpu")
        own = model.state_dict()
        # checkpoints written by other transformers versions carry buffers we do not hold (position_ids) — drop those only
        extra = [k for k in sd if k not in own]
        if any(not k.endswith("position_ids") for k in extra):
            raise RuntimeError(f"unexpected keys in the text-encoder checkpoint: {[k for k in extra if not k.endswith('position_ids')][:5]}")
        model.load_state_dict({k: v for k, v in sd.items() if k in own}, strict=True)
        if torch_dtype is not None:
            model = model.to(torch_dtype)
        return model.eval()

    @torch.no_grad()
    def forward(self, input_ids: torch.Tensor, attention_mask: Optional[torch.Tensor] = None, **_):
        """returns (last_hidden_state (b, n, hidden) in the model dtype, None): index [0] like the reference does"""
        if attention_mask is not None:
            raise NotImplementedError("padding masks are not used by the x4-upscaler text encoder (use_attention_mask=False)")
        cfg, pk, tm = self.config, self._packed(), self.text_model
        _lib.require_cuda(tm.final_layer_norm.weight, "CLIPTextModel")
        b, n = input_ids.shape
        if n > cfg.max_position_embeddings or n > 128:
            raise ValueError(f"sequence of {n} tokens exceeds max_position_embeddings / 128")
        dev = tm.final_layer_norm.weight.device
        tok = pk.tensor("tok16", lambda: tm.embeddings.token_embedding.weight.detach().to(torch.float16))
        pos = pk.tensor("pos16", lambda: tm.embeddings.position_embedding.weight.detach().to(torch.float16))
        # embeddings: fp32 sum of the two fp16 table rows, one rounding
        x = (tok.index_select(0, input_ids.reshape(-1).to(dev)).float().view(b, n, -1) + pos[:n].float()[None]).to(torch.float16)
        heads = cfg.num_attention_heads
        act = ops.ACT_GELU if cfg.hidden_act == "gelu" else ops.ACT_QUICK_GELU
        for i, layer in enumerate(tm.encoder.layers):
            a = layer.self_attn
            w = SimpleNamespace(ln1=pk.affine(layer.layer_norm1), qkv=pk.fused_linear(f"qkv{i}", [a.q_proj, a.k_proj, a.v_proj]),
                                out=pk.linear(a.out_proj), ln2=pk.affine(layer.layer_norm2), fc1=pk.linear(layer.mlp.fc1),
                                fc2=pk.linear(layer.mlp.fc2))
            x = encoder_layer(x, w, heads, cfg.layer_norm_eps, act, causal=True)
        gf, bf = pk.affine(tm.final_layer_norm)
        out = ops.layer_norm(x, gf, bf, cfg.layer_norm_eps)
        return out.to(self.dtype), None
