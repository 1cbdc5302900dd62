"""Synthetic LLaVA-1.5 folders in the released format, with seeded weights, for the captioner's tests: a decoder
folder (config.json, two `pytorch_model-*.bin` shards with their index, the golden sentencepiece tokenizer) and a CLIP
vision folder (config.json, model.safetensors, preprocessor_config.json)."""
import json
import os
import shutil

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")


def text_config(hidden=512, heads=4, layers=2, inter=1024, vocab=32000):
    return dict(hidden_size=hidden, intermediate_size=inter, num_hidden_layers=layers, num_attention_heads=heads,
                num_key_value_heads=heads, rms_norm_eps=1e-5, rope_theta=10000.0, vocab_size=vocab,
                max_position_embeddings=4096, hidden_act="silu", bos_token_id=1, eos_token_id=2)


def vision_config(hidden=1024, heads=16, layers=2, inter=4096, image_size=336):
    return dict(hidden_size=hidden, intermediate_size=inter, num_hidden_layers=layers, num_attention_heads=heads,
                image_size=image_size, patch_size=14, hidden_act="quick_gelu", layer_norm_eps=1e-5, projection_dim=768)


def released_state_dict(tc: dict, mm_hidden: int, seed: int, lm_scale: float = 3.0) -> dict:
    """fp16 decoder + projector weights under the released LLaVA-1.5 keys"""
    g = torch.Generator().manual_seed(seed)
    H, I, V = tc["hidden_size"], tc["intermediate_size"], tc["vocab_size"]
    lin = lambda n, k, s=1.0: (torch.randn(n, k, generator=g) * (s / k ** 0.5)).half()
    norm = lambda n: (1 + 0.1 * torch.randn(n, generator=g)).half()
    sd = {"model.embed_tokens.weight": (torch.randn(V, H, generator=g) * 0.5).half(), "model.norm.weight": norm(H),
          "lm_head.weight": lin(V, H, lm_scale),
          "model.mm_projector.0.weight": lin(H, mm_hidden), "model.mm_projector.0.bias": (0.02 * torch.randn(H, generator=g)).half(),
          "model.mm_projector.2.weight": lin(H, H), "model.mm_projector.2.bias": (0.02 * torch.randn(H, generator=g)).half()}
    for i in range(tc["num_hidden_layers"]):
        p = f"model.layers.{i}."
        for n in ("q", "k", "v", "o"):
            sd[p + f"self_attn.{n}_proj.weight"] = lin(H, H, 2.0 if n in "qk" else 1.0)
        sd[p + "self_attn.rotary_emb.inv_freq"] = 1.0 / (10000 ** (torch.arange(0, 128, 2).float() / 128))
        sd[p + "mlp.gate_proj.weight"] = lin(I, H)
        sd[p + "mlp.up_proj.weight"] = lin(I, H)
        sd[p + "mlp.down_proj.weight"] = lin(H, I)
        sd[p + "input_layernorm.weight"] = norm(H)
        sd[p + "post_attention_layernorm.weight"] = norm(H)
    return sd


def vision_state_dict(vc: dict, seed: int) -> dict:
    """fp16 `vision_model.*` weights of a CLIP vision tower"""
    g = torch.Generator().manual_seed(seed)
    D, I = vc["hidden_size"], vc["intermediate_size"]
    n_pos = (vc["image_size"] // vc["patch_size"]) ** 2 + 1
    lin = lambda n, k: (torch.randn(n, k, generator=g) / k ** 0.5).half()
    vec = lambda n, s=0.02, c=0.0: (c + s * torch.randn(n, generator=g)).half()
    e = "vision_model.embeddings."
    sd = {e + "class_embedding": vec(D, 1.0), e + "position_embedding.weight": (0.5 * torch.randn(n_pos, D, generator=g)).half(),
          e + "patch_embedding.weight": (torch.randn(D, 3, 14, 14, generator=g) / 588 ** 0.5).half(),
          "vision_model.pre_layrnorm.weight": vec(D, 0.1, 1.0), "vision_model.pre_layrnorm.bias": vec(D),
          "vision_model.post_layernorm.weight": vec(D, 0.1, 1.0), "vision_model.post_layernorm.bias": vec(D)}
    for i in range(vc["num_hidden_layers"]):
        p = f"vision_model.encoder.layers.{i}."
        for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
            sd[p + f"self_attn.{n}.weight"] = lin(D, D)
            sd[p + f"self_attn.{n}.bias"] = vec(D)
        sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"] = lin(I, D), vec(I)
        sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"] = lin(D, I), vec(D)
        for n in ("layer_norm1", "layer_norm2"):
            sd[p + n + ".weight"], sd[p + n + ".bias"] = vec(D, 0.1, 1.0), vec(D)
    return sd


def write_llava_folders(root: str, tc: dict, vc: dict, seed: int = 5):
    """(llava folder, CLIP folder, released state dict, vision state dict) under root"""
    from safetensors.torch import save_file
    llava, clip = os.path.join(root, "llava-v1.5"), os.path.join(root, "clip-vit")
    os.makedirs(llava)
    os.makedirs(clip)
    sd = released_state_dict(tc, vc["hidden_size"], seed)
    vsd = vision_state_dict(vc, seed + 1)
    cfg = dict(tc, architectures=["LlavaLlamaForCausalLM"], model_type="llava", mm_projector_type="mlp2x_gelu",
               mm_vision_select_layer=-2, mm_vision_select_feature="patch", mm_hidden_size=vc["hidden_size"],
               mm_vision_tower="openai/clip-vit-large-patch14-336", mm_use_im_start_end=False,
               mm_use_im_patch_token=False, image_aspect_ratio="pad", torch_dtype="float16")
    json.dump(cfg, open(os.path.join(llava, "config.json"), "w"))
    keys = list(sd)
    # the second shard starts between layer 1's q and k projections, so a fused matrix straddles two shards
    cut = keys.index("model.layers.1.self_attn.k_proj.weight") if "model.layers.1.self_attn.k_proj.weight" in keys else len(keys) // 2
    shards = [keys[:cut], keys[cut:]]
    weight_map = {}
    for j, ks in enumerate(shards):
        name = f"pytorch_model-{j + 1:05d}-of-{len(shards):05d}.bin"
        torch.save({k: sd[k] for k in ks}, os.path.join(llava, name))
        weight_map.update({k: name for k in ks})
    json.dump({"metadata": {}, "weight_map": weight_map}, open(os.path.join(llava, "pytorch_model.bin.index.json"), "w"))
    shutil.copy(os.path.join(GOLDEN, "llava_tokenizer.model"), os.path.join(llava, "tokenizer.model"))
    json.dump({"model_type": "clip", "vision_config": dict(vc, model_type="clip_vision_model")},
              open(os.path.join(clip, "config.json"), "w"))
    save_file({**vsd, "text_model.final_layer_norm.weight": torch.ones(8, dtype=torch.float16)},
              os.path.join(clip, "model.safetensors"))
    prompt = json.load(open(os.path.join(GOLDEN, "llava_prompt.json")))
    json.dump(prompt["preprocessor_config"], open(os.path.join(clip, "preprocessor_config.json"), "w"))
    return llava, clip, sd, vsd
