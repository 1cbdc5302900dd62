"""transformers' own `LlavaForConditionalGeneration`, built from a LLaVA-1.5 state dict in the released key layout
plus the `vision_model.*` keys of a CLIP vision checkpoint: the independent model the captioner (llava.py) is checked
against.  It is configured as LLaVA-1.5 runs: features of the second-to-last vision layer (`vision_feature_layer=-2`),
CLS dropped (`default` selection), `mlp2x_gelu` projector (`projector_hidden_act="gelu"`)."""
import torch


def remap_llava_keys(released: dict, vision: dict) -> dict:
    """released LLaVA-1.5 keys (`model.layers.N...`, `model.mm_projector.{0,2}`, `lm_head`) and CLIP `vision_model.*`
    keys -> transformers' LlavaForConditionalGeneration keys"""
    out = {}
    for k, v in released.items():
        if k.endswith("rotary_emb.inv_freq"):
            continue
        if k.startswith("model.mm_projector."):
            idx, rest = k[len("model.mm_projector."):].split(".", 1)
            out[f"model.multi_modal_projector.linear_{1 if idx == '0' else 2}.{rest}"] = v
        elif k.startswith("model."):
            out["model.language_model." + k[len("model."):]] = v
        elif k.startswith("lm_head."):
            out[k] = v
        else:
            raise KeyError(k)
    for k, v in vision.items():
        if k.startswith("vision_model."):
            out["model.vision_tower." + k] = v
    return out


def build_llava(text_cfg: dict, vision_cfg: dict, released: dict, vision: dict, image_token_index: int,
                dtype=torch.float32):
    """the transformers model with the given weights; `image_token_index` is the id that stands for an image patch"""
    from transformers import CLIPVisionConfig, LlamaConfig, LlavaConfig, LlavaForConditionalGeneration
    vc = CLIPVisionConfig(**vision_cfg)
    tc = LlamaConfig(**text_cfg)
    n_patches = (vc.image_size // vc.patch_size) ** 2
    cfg = LlavaConfig(vision_config=vc, text_config=tc, image_token_index=image_token_index, vision_feature_layer=-2,
                      vision_feature_select_strategy="default", projector_hidden_act="gelu",
                      image_seq_length=n_patches)
    model = LlavaForConditionalGeneration(cfg)
    sd = remap_llava_keys(released, vision)
    own = model.state_dict()
    # the unused post_layernorm of the vision tower is not part of LLaVA's path; it keeps its initial values
    missing = [k for k in own if k not in sd and "post_layernorm" not in k]
    assert not missing, missing[:5]
    model.load_state_dict({k: v for k, v in sd.items() if k in own}, strict=False)
    return model.to(dtype).eval()


def expand_image_ids(ids, image_token_index: int, n_patches: int, placeholder: int = -200):
    """prompt ids with the `placeholder` replaced by n_patches copies of the model's image token"""
    out = []
    for t in ids:
        out.extend([image_token_index] * n_patches if t == placeholder else [t])
    return torch.tensor([out], dtype=torch.long)
