"""Write tests/golden/llava_prompt.json, llava_tokenizer.model and llava_pixels.pt from the reference's own LLaVA code.

    python oracle/make_golden_llava.py <reference checkout>

The reference's `llava/__init__.py` cannot be imported with current transformers (its `AutoConfig.register("llava")`
clashes with transformers' own LLaVA, and its MPT code imports a removed bloom helper), so `llava/constants.py`,
`llava/conversation.py` and `llava/mm_utils.py` are loaded by file path under a stub `llava` package.

The golden holds:
- the vicuna_v1 prompt built by the reference's conversation template;
- `tokenizer_image_token` ids of that prompt for a small sentencepiece tokenizer trained here and stored beside the
  golden, driven through a Llama-tokenizer stand-in (`[bos] + encode(text)`, as LlamaTokenizer with add_bos_token);
- the reference agent's caption post-processing on a few raw outputs;
- `pixel_values` of a seeded frame through the reference CLI's preprocessing sequence: the 512 bicubic resize of
  inference_upscale_a_video.py (restated), then transformers' PIL CLIPImageProcessor configured as CLIP ViT-L/14-336's
  preprocessor_config.json (tests/golden/llava_pixels.pt).
"""
import hashlib
import importlib.util
import io
import json
import os
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "..", "tests", "golden")

# CLIP ViT-L/14-336's preprocessor_config.json (openai/clip-vit-large-patch14-336)
CLIP_L336_PREPROCESSOR = {
    "crop_size": 336, "do_center_crop": True, "do_normalize": True, "do_resize": True,
    "feature_extractor_type": "CLIPFeatureExtractor",
    "image_mean": [0.48145466, 0.4578275, 0.40821073], "image_std": [0.26862954, 0.26130258, 0.27577711],
    "resample": 3, "size": 336,
}

CORPUS = ["A chat between a curious user and an artificial intelligence assistant.",
          "The assistant gives helpful, detailed, and polite answers to the user's questions.",
          "USER: Describe this image and its style in a very detailed manner. ASSISTANT:",
          "The image shows a city street at night with bright lights, wet asphalt and a red car.",
          "A painting of a quiet lake surrounded by mountains, in an impressionist style with soft colours.",
          "\n"]


def load_reference_llava(ref: str):
    pkg = types.ModuleType("llava")
    pkg.__path__ = [os.path.join(ref, "llava")]
    sys.modules["llava"] = pkg
    mods = {}
    for name in ("constants", "conversation", "mm_utils"):
        spec = importlib.util.spec_from_file_location(f"llava.{name}", os.path.join(ref, "llava", f"{name}.py"))
        m = importlib.util.module_from_spec(spec)
        sys.modules[f"llava.{name}"] = m
        spec.loader.exec_module(m)
        mods[name] = m
    return mods


def train_tokenizer(path: str):
    import sentencepiece as spm
    buf = io.BytesIO()
    spm.SentencePieceTrainer.train(sentence_iterator=iter(CORPUS * 20), model_writer=buf, vocab_size=400,
                                   model_type="bpe", byte_fallback=True, unk_id=0, bos_id=1, eos_id=2, pad_id=-1,
                                   character_coverage=1.0, add_dummy_prefix=True, normalization_rule_name="identity")
    open(path, "wb").write(buf.getvalue())
    return spm.SentencePieceProcessor(model_file=path)


class LlamaLikeTokenizer:
    """the part of LlamaTokenizer (add_bos_token=True) that tokenizer_image_token uses"""

    def __init__(self, sp):
        self.sp, self.bos_token_id = sp, sp.bos_id()

    def __call__(self, text):
        return types.SimpleNamespace(input_ids=[self.bos_token_id] + self.sp.encode(text))


def seeded_frame(h=120, w=200, seed=7):
    g = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    base = np.stack([xx * 255 / w, yy * 255 / h, (xx + yy) * 255 / (w + h)], axis=-1)
    return np.clip(base + g.normal(0, 25, (h, w, 3)), 0, 255).astype(np.uint8)


def reference_pixel_values(frame_rgb: np.ndarray) -> torch.Tensor:
    """inference_upscale_a_video.py:161-170 on a (h, w, 3) uint8 RGB frame, then the CLIP processor"""
    from PIL import Image
    from transformers.models.clip.image_processing_pil_clip import CLIPImageProcessorPil
    # the CLI's resize, restated: scale both sides by 512 / short side (floats, rounded with Python's round), bicubic
    # torch interpolation of the fp32 CHW frame on the CPU, clip to [0, 255] and truncate to uint8
    h, w = frame_rgb.shape[:2]
    s = 512 / min(w, h)
    size = (round(h * s), round(w * s))
    x = F.interpolate(torch.from_numpy(frame_rgb).permute(2, 0, 1)[None].float(), size=size, mode="bicubic")
    img = Image.fromarray(x[0].permute(1, 2, 0).numpy().clip(0, 255).astype(np.uint8))
    proc = CLIPImageProcessorPil(**{k: v for k, v in CLIP_L336_PREPROCESSOR.items() if k != "feature_extractor_type"})
    return proc.preprocess(img, return_tensors="pt")["pixel_values"][0].half()


def main(ref: str):
    mods = load_reference_llava(ref)
    C, conv_mod, mm = mods["constants"], mods["conversation"], mods["mm_utils"]
    qs = C.DEFAULT_IMAGE_TOKEN + "\n" + "Describe this image and its style in a very detailed manner."
    conv = conv_mod.conv_templates["vicuna_v1"].copy()
    conv.append_message(conv.roles[0], qs)
    conv.append_message(conv.roles[1], None)
    prompt = conv.get_prompt()
    sp = train_tokenizer(os.path.join(GOLDEN, "llava_tokenizer.model"))
    ids = mm.tokenizer_image_token(prompt, LlamaLikeTokenizer(sp), C.IMAGE_TOKEN_INDEX)
    stop_str = conv.sep if conv.sep_style != conv_mod.SeparatorStyle.TWO else conv.sep2
    raw = ["  The image shows a street.</s>", "A lake\nwith mountains.\r\n", "</s>", " plain caption ",
           "two lines\n\nand a stop </s>  "]
    # the agent's post-processing, restated: strip, drop the trailing stop string, strip, newlines to spaces
    post = []
    for text in raw:
        t = text.strip()
        t = t[:-len(stop_str)] if t.endswith(stop_str) else t
        post.append(t.strip().replace("\n", " ").replace("\r", " "))
    frame = seeded_frame()
    px = reference_pixel_values(frame)
    # the pixel values are pinned by the sha256 of their fp16 bytes (a corner is kept to show a mismatch)
    torch.save({"frame_rgb": torch.from_numpy(frame), "pixel_values_sha256": hashlib.sha256(px.numpy().tobytes()).hexdigest(),
                "pixel_values_corner": px[:, :8, :8].clone()}, os.path.join(GOLDEN, "llava_pixels.pt"))
    json.dump({"prompt": prompt, "input_ids": ids, "image_token_index": C.IMAGE_TOKEN_INDEX,
               "stop_str": stop_str, "postprocess": [[r, p] for r, p in zip(raw, post)],
               "preprocessor_config": CLIP_L336_PREPROCESSOR},
              open(os.path.join(GOLDEN, "llava_prompt.json"), "w"), indent=1)
    print(prompt)
    print(ids)


if __name__ == "__main__":
    main(sys.argv[1])
