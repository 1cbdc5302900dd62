"""The LLaVA captioner's host logic, without a GPU: prompt, tokens and preprocessing against goldens made from the
reference's own code (oracle/make_golden_llava.py), the released-format key mapping against transformers' LLaVA,
caption post-processing, the command's flags, and the top-p keep rule against transformers' TopPLogitsWarper."""
import hashlib
import json
import os
import types

import numpy as np
import pytest
import torch

from llava_cases import GOLDEN, text_config, vision_config, write_llava_folders

PROMPT = json.load(open(os.path.join(GOLDEN, "llava_prompt.json")))


def _sp():
    import sentencepiece as spm
    return spm.SentencePieceProcessor(model_file=os.path.join(GOLDEN, "llava_tokenizer.model"))


def test_prompt_and_tokens_golden():
    from upscale_a_video_b200.llava import IMAGE_TOKEN_INDEX, conversation_prompt, tokenize_prompt
    assert conversation_prompt() == PROMPT["prompt"]
    sp = _sp()
    ids = tokenize_prompt(PROMPT["prompt"], sp.encode, sp.bos_id())
    assert ids == PROMPT["input_ids"]
    assert IMAGE_TOKEN_INDEX == PROMPT["image_token_index"] and ids.count(IMAGE_TOKEN_INDEX) == 1


def test_postprocess_golden():
    from upscale_a_video_b200.llava import STOP_STR, postprocess_caption
    assert STOP_STR == PROMPT["stop_str"]
    for raw, want in PROMPT["postprocess"]:
        assert postprocess_caption(raw) == want, raw


def test_preprocessing_golden_bit_exact():
    from upscale_a_video_b200.llava import clip_preprocess, frame0_image
    g = torch.load(os.path.join(GOLDEN, "llava_pixels.pt"))
    px = clip_preprocess(frame0_image(g["frame_rgb"].numpy()), PROMPT["preprocessor_config"])
    assert px.dtype == torch.float16 and px.shape == (3, 336, 336)
    assert torch.equal(px[:, :8, :8], g["pixel_values_corner"])
    assert hashlib.sha256(px.numpy().tobytes()).hexdigest() == g["pixel_values_sha256"]


@pytest.fixture(scope="module")
def tiny(tmp_path_factory):
    tc = text_config(hidden=256, heads=2, layers=2, inter=512, vocab=400)
    vc = vision_config(hidden=64, heads=4, layers=2, inter=128, image_size=28)
    root = str(tmp_path_factory.mktemp("llava"))
    return (tc, vc) + write_llava_folders(root, tc, vc)


def _cfg(tc, vc):
    from types import SimpleNamespace
    return SimpleNamespace(**tc, mm_hidden_size=vc["hidden_size"])


def test_key_mapping_matches_transformers(tiny):
    """every weight lands where transformers' LlavaForConditionalGeneration puts it (fused q|k|v and gate|up rows in
    order), read from two shards with a fused matrix straddling them"""
    from oracle.llava_oracle import build_llava
    from upscale_a_video_b200.llava import load_decoder
    tc, vc, folder, _clip, sd, vsd = tiny
    ours = load_decoder(folder, _cfg(tc, vc), "cpu")
    ref = build_llava(tc, vc, sd, vsd, image_token_index=tc["vocab_size"] - 1).state_dict()
    lm = "model.language_model."
    assert torch.equal(ours["embed"], ref[lm + "embed_tokens.weight"].half())
    assert torch.equal(ours["lm_head"], ref["lm_head.weight"].half())
    assert torch.equal(ours["norm"], ref[lm + "norm.weight"].half())
    for i in range(tc["num_hidden_layers"]):
        p = f"{lm}layers.{i}."
        qkv = torch.cat([ref[p + f"self_attn.{n}_proj.weight"] for n in "qkv"]).half()
        gu = torch.cat([ref[p + f"mlp.{n}_proj.weight"] for n in ("gate", "up")]).half()
        assert torch.equal(ours[f"qkv{i}"], qkv) and torch.equal(ours[f"gu{i}"], gu)
        assert torch.equal(ours[f"o{i}"], ref[p + "self_attn.o_proj.weight"].half())
        assert torch.equal(ours[f"down{i}"], ref[p + "mlp.down_proj.weight"].half())
        assert torch.equal(ours[f"ln1_{i}"], ref[p + "input_layernorm.weight"].half())
        assert torch.equal(ours[f"ln2_{i}"], ref[p + "post_attention_layernorm.weight"].half())
    mp = "model.multi_modal_projector."
    assert torch.equal(ours["proj0_w"], ref[mp + "linear_1.weight"].half())
    assert torch.equal(ours["proj2_b"], ref[mp + "linear_2.bias"].float())


def test_image_splice_matches_transformers():
    """the 576 image rows replace the placeholder at the position where transformers' model puts its image tokens"""
    from oracle.llava_oracle import expand_image_ids
    ids = PROMPT["input_ids"]
    at = ids.index(-200)
    expanded = expand_image_ids(ids, 31999, 576)[0]
    rows = (expanded == 31999).nonzero().flatten()
    assert rows[0].item() == at and rows[-1].item() == at + 575 and len(rows) == 576
    assert expanded.numel() == len(ids) - 1 + 576
    assert expanded[:at].tolist() == ids[:at] and expanded[at + 576:].tolist() == ids[at + 1:]


def _rewrite_shard(folder, fn):
    idx = json.load(open(os.path.join(folder, "pytorch_model.bin.index.json")))
    name = sorted(set(idx["weight_map"].values()))[-1]
    sd = torch.load(os.path.join(folder, name))
    fn(sd)
    torch.save(sd, os.path.join(folder, name))


def test_unexpected_and_missing_keys_rejected(tiny, tmp_path):
    import shutil
    from upscale_a_video_b200.llava import load_decoder
    tc, vc, folder, *_ = tiny
    for case, fn, msg in (("extra", lambda sd: sd.__setitem__("model.layers.1.self_attn.q_norm.weight", torch.ones(4)),
                           "unexpected"),
                          ("missing", lambda sd: sd.pop("model.layers.1.mlp.up_proj.weight"), "missing")):
        d = str(tmp_path / case)
        shutil.copytree(folder, d)
        _rewrite_shard(d, fn)
        with pytest.raises(RuntimeError, match=msg):
            load_decoder(d, _cfg(tc, vc), "cpu")


def test_agent_rejects_unsupported(tiny, tmp_path):
    from upscale_a_video_b200 import LLavaAgent
    tc, vc, folder, clip, *_ = tiny
    with pytest.raises(NotImplementedError):
        LLavaAgent(folder, load_8bit=True)
    with pytest.raises(NotImplementedError):
        LLavaAgent(folder, load_4bit=True)
    with pytest.raises(EnvironmentError):
        LLavaAgent(str(tmp_path / "liuhaotian" / "llava-v1.5-13b"))
    with pytest.raises(EnvironmentError, match="mm_vision_tower"):
        LLavaAgent(folder)  # the config's mm_vision_tower is a hub name, and no vision_tower_path was given
    import shutil
    for change, what in (({"num_key_value_heads": 1}, "grouped"), ({"mm_projector_type": "linear"}, "mlp2x_gelu"),
                         ({"num_attention_heads": 4}, "head_dim")):
        d = str(tmp_path / what)
        shutil.copytree(folder, d)
        cfg = json.load(open(os.path.join(d, "config.json")))
        cfg.update(change)
        json.dump(cfg, open(os.path.join(d, "config.json"), "w"))
        with pytest.raises(NotImplementedError, match=what):
            LLavaAgent(d, vision_tower_path=clip)


def test_cli_flags():
    from upscale_a_video_b200 import cli
    a = cli.parse_args([])
    assert a.llava_path is None and a.llava_vision_path is None and not cli.use_llava(a) and a.caption == ""
    a = cli.parse_args(["--llava_path", "L", "--llava_vision_path", "V"])
    assert cli.use_llava(a) and a.llava_vision_path == "V"
    assert not cli.use_llava(cli.parse_args(["--llava_path", "L", "--no_llava"]))
    assert cli.parse_args(["--llava_path", "L", "--no_llava", "--caption", "x"]).caption == "x"
    with pytest.raises(SystemExit):
        cli.parse_args(["--llava_path", "L", "--caption", "a cat"])


def test_load_8bit_still_rejected(capsys):
    from upscale_a_video_b200 import cli
    with pytest.raises(SystemExit):
        cli.parse_args(["--llava_path", "L", "--load_8bit_llava"])
    assert "no LLaVA captioner" in capsys.readouterr().err


# ---------------------------------------------------------------- the top-p keep rule
def keep_rule(logits: torch.Tensor, temperature: float, top_p: float) -> torch.Tensor:
    """the sampler kernel's nucleus, restated in fp64: a token is kept when the tokens strictly more probable than it
    have mass < top_p"""
    p = torch.softmax(logits.double() / temperature, -1)
    order = torch.sort(p, descending=True).values
    above = torch.cumsum(order, 0) - order  # mass strictly before each sorted position (distinct values)
    t = order[(above < top_p).nonzero().max()]
    return p >= t


def hf_kept(logits: torch.Tensor, temperature: float, top_p: float) -> torch.Tensor:
    from transformers.generation.logits_process import TemperatureLogitsWarper, TopPLogitsWarper
    s = TemperatureLogitsWarper(temperature)(None, logits[None].float())
    s = TopPLogitsWarper(top_p)(None, s)
    return torch.isfinite(s[0])


def _margin(logits, temperature, top_p):
    """distance of the nucleus boundary from 1 - top_p (HF's sums are fp32)"""
    p = torch.sort(torch.softmax(logits.double() / temperature, -1)).values
    return (torch.cumsum(p, 0) - (1 - top_p)).abs().min().item()


@pytest.mark.parametrize("kind", ["random", "peaked", "flat", "near_boundary"])
def test_top_p_keep_rule_matches_transformers(kind):
    g = torch.Generator().manual_seed(3)
    checked = 0
    for trial in range(40):
        V = 32000
        if kind == "random":
            x = torch.randn(V, generator=g) * 3
        elif kind == "peaked":
            x = torch.randn(V, generator=g)
            x[torch.randint(V, (3,), generator=g)] += 12
        elif kind == "flat":
            x = torch.randn(V, generator=g) * 1e-3
        else:
            x = torch.full((V,), -30.0)
            k = 2 + trial % 5
            x[:k] = torch.log(torch.tensor([0.7 / (k - 1)] * (k - 1) + [0.3])) * 0.2  # mass near 1 - top_p
            x[:k] += torch.randn(k, generator=g) * 1e-3
        for temperature, top_p in ((0.2, 0.7), (1.0, 0.9), (0.7, 0.5)):
            if _margin(x, temperature, top_p) < 1e-5:
                continue  # within rounding of the boundary, fp32 and fp64 may disagree
            assert torch.equal(keep_rule(x, temperature, top_p), hf_kept(x, temperature, top_p)), (kind, trial)
            checked += 1
    assert checked >= 40
