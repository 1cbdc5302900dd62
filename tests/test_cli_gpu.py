"""`python -m upscale_a_video_b200` on the GPU: the two new kernels bit-exact against the reference's op sequences, and
the whole command on a synthetic checkpoint folder against the public API called in the reference CLI's order
(inference_upscale_a_video.py:101-351)."""
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

cv2 = pytest.importorskip("cv2")

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG_CONFIGS = os.path.join(ROOT, "upscale_a_video_b200", "configs")


@pytest.fixture(autouse=True)
def _setup(uav_lib):
    torch.manual_seed(0)


def _bgr(t, h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, size=(t, h, w, 3), dtype=np.uint8)


def _reference_frames(bgr, from_video):
    """the reference's (t, c, h, w) frames: utils.read_frame_from_videos makes an image folder's frames contiguous,
    while torchvision.io.read_video returns a video's as a channels-last view; then inference_upscale_a_video.py:180-181"""
    v = torch.from_numpy(bgr[..., ::-1].copy()).permute(0, 3, 1, 2)
    if not from_video:
        v = v.contiguous()
    return ((v.float() / 255. - 0.5) * 2).cuda()


def _reference_ingest(bgr, from_video=False):
    """inference_upscale_a_video.py:180-188"""
    v = _reference_frames(bgr, from_video)
    h, w = v.shape[-2:]
    if h >= 1280 and w >= 1280:
        v = F.interpolate(v, (int(h // 4), int(w // 4)), mode="area")
    return v.permute(1, 0, 2, 3).unsqueeze(0).contiguous()


@pytest.mark.parametrize("from_video", [True, False])
@pytest.mark.parametrize("t,h,w", [(3, 45, 61), (2, 1280, 1280), (2, 1283, 1297), (1, 1280, 2560)])
def test_ingest_bit_exact(t, h, w, from_video):
    from upscale_a_video_b200 import cli
    bgr = _bgr(t, h, w, h + w)
    got = cli.ingest_frames(bgr, torch.device("cuda"), from_video)
    ref = _reference_ingest(bgr, from_video)
    assert got.shape == ref.shape and got.dtype == torch.float32 and got.is_contiguous()
    assert torch.equal(got, ref)


@pytest.mark.parametrize("from_video", [True, False])
def test_ingest_area_resize_any_size(from_video):
    """sizes the CLI never asks for, with overlapping windows in both directions"""
    from upscale_a_video_b200 import _lib, ops
    bgr = _bgr(2, 45, 61, 7)
    full = _reference_frames(bgr, from_video)
    for size in ((11, 15), (44, 60), (45, 7), (1, 2), (3, 1)):
        got = ops.unpack_video_uint8(torch.from_numpy(bgr).cuda(), size, channels_last=from_video)
        ref = F.interpolate(full, size, mode="area").permute(1, 0, 2, 3)[None]
        assert torch.equal(got, ref), size
    with pytest.raises(_lib.UavError, match="1x1"):
        ops.unpack_video_uint8(torch.from_numpy(bgr).cuda(), (1, 1))


def _save_image_quantise(frames):
    """torchvision save_image(frame, normalize=True, value_range=(-1, 1)) per frame, up to the uint8 array it writes"""
    from torchvision.utils import make_grid
    out = []
    for f in frames.cpu():
        grid = make_grid(f, normalize=True, value_range=(-1, 1))
        out.append(grid.mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to("cpu", torch.uint8))
    return torch.stack(out)


def test_png_quantisation_bit_exact():
    from upscale_a_video_b200 import color_correction as cc
    k = torch.arange(256, dtype=torch.float32)
    # inputs whose (x + 1) / 2 * 255 + 0.5 lands on or next to an integer, out-of-range values, and the ends
    half = (k + 0.5) / 255 * 2 - 1
    edges = torch.cat([half, torch.nextafter(half, torch.full_like(half, 2.0)), torch.nextafter(half, -torch.full_like(half, 2.0)),
                       k / 255 * 2 - 1, torch.tensor([-1.0, 1.0, -1.5, 2.0, -100.0, 1e9, 0.0, -0.0, 1 - 2 ** -24])])
    x = edges[: (edges.numel() // 4) * 4].view(1, 3, -1, 4).repeat(2, 1, 1, 1)
    x[1] = -x[1]
    assert torch.equal(cc.pack_frames_png(x.cuda()).cpu(), _save_image_quantise(x))
    dense = torch.linspace(-1.02, 1.02, 3 * 3 * 301 * 197).view(3, 3, 301, 197)
    assert torch.equal(cc.pack_frames_png(dense.cuda()).cpu(), _save_image_quantise(dense))


# ------------------------------------------------------------------------------------------------- end to end
SCHED = dict(beta_schedule="scaled_linear", clip_sample=False, steps_offset=1, prediction_type="v_prediction",
             set_alpha_to_one=False)


def _write_tokenizer(folder):
    from transformers import CLIPTokenizer
    chars = list("abcdefghijklmnopqrstuvwxyz,.")
    vocab = {c: i for i, c in enumerate(chars)}
    vocab.update({c + "</w>": len(chars) + i for i, c in enumerate(chars)})
    vocab.update({"<|startoftext|>": len(vocab), "<|endoftext|>": len(vocab) + 1})
    src = os.path.join(folder, "src")
    os.makedirs(src)
    json.dump(vocab, open(os.path.join(src, "vocab.json"), "w"))
    open(os.path.join(src, "merges.txt"), "w").write("#version: 0.2\n")
    tok = CLIPTokenizer(os.path.join(src, "vocab.json"), os.path.join(src, "merges.txt"), model_max_length=77)
    tok.save_pretrained(os.path.join(folder, "tokenizer"))
    shutil.rmtree(src)
    return len(vocab)


@pytest.fixture(scope="session")
def model_dir(tmp_path_factory):
    """the released folder layout with seeded weights: text encoder (hidden 1024, 1 layer), tokenizer, schedulers,
    vae_3d, the full fp16 UNet and RAFT"""
    from upscale_a_video_b200 import AutoencoderKLVideo, CLIPTextConfig, CLIPTextModel, UNetVideoModel
    from upscale_a_video_b200.raft import RAFT
    from upscale_a_video_b200.synthetic import seeded_state_dict
    d = str(tmp_path_factory.mktemp("upscale_a_video"))
    for sub in ("text_encoder", "low_res_scheduler", "scheduler", "vae", "unet", "propagator"):
        os.makedirs(os.path.join(d, sub))
    n_vocab = _write_tokenizer(d)
    cfg = dict(vocab_size=n_vocab, hidden_size=1024, intermediate_size=256, num_hidden_layers=1, num_attention_heads=16,
               max_position_embeddings=77, hidden_act="gelu", layer_norm_eps=1e-5)
    json.dump(dict(cfg, model_type="clip_text_model"), open(os.path.join(d, "text_encoder", "config.json"), "w"))
    te = CLIPTextModel(CLIPTextConfig(**cfg))
    torch.save(seeded_state_dict(te, 77), os.path.join(d, "text_encoder", "pytorch_model.bin"))
    json.dump({"beta_schedule": "scaled_linear", "_class_name": "DDPMScheduler"},
              open(os.path.join(d, "low_res_scheduler", "scheduler_config.json"), "w"))
    json.dump(SCHED, open(os.path.join(d, "scheduler", "scheduler_config.json"), "w"))
    json.dump({"max_noise_level": 350}, open(os.path.join(d, "model_index.json"), "w"))
    for kind, sub, cls, seed, dtype in (("vae_3d", "vae", AutoencoderKLVideo, 4321, torch.float32),
                                        ("unet_video", "unet", UNetVideoModel, 1234, torch.float16)):
        shutil.copy(os.path.join(PKG_CONFIGS, f"{kind}_config.json"), os.path.join(d, sub, f"{kind}_config.json"))
        m = cls.from_config(os.path.join(PKG_CONFIGS, f"{kind}_config.json"))
        torch.save(seeded_state_dict(m, seed, dtype), os.path.join(d, sub, f"{kind}.bin"))
        del m
    sd = seeded_state_dict(RAFT(), 99)
    torch.save({"module." + k: v for k, v in sd.items()}, os.path.join(d, "propagator", "raft-things.pth"))
    return d


@pytest.fixture(scope="module")
def reference_models(model_dir):
    """inference_upscale_a_video.py:101-131 through the public API"""
    from upscale_a_video_b200 import (AutoencoderKLVideo, DDIMScheduler, Propagation, RAFT_bi, UNetVideoModel,
                                      VideoUpscalePipeline)
    pipeline = VideoUpscalePipeline.from_pretrained(model_dir, torch_dtype=torch.float16)
    pipeline.vae = AutoencoderKLVideo.from_config(os.path.join(model_dir, "vae", "vae_3d_config.json"))
    pipeline.vae.load_state_dict(torch.load(os.path.join(model_dir, "vae", "vae_3d.bin"), map_location="cpu"))
    pipeline.unet = UNetVideoModel.from_config(os.path.join(model_dir, "unet", "unet_video_config.json"))
    pipeline.unet.load_state_dict(torch.load(os.path.join(model_dir, "unet", "unet_video.bin"), map_location="cpu"),
                                  strict=True)
    pipeline.unet = pipeline.unet.half()
    pipeline.unet.eval()
    pipeline.scheduler = DDIMScheduler.from_config(os.path.join(model_dir, "scheduler", "scheduler_config.json"))
    raft = RAFT_bi(os.path.join(model_dir, "propagator", "raft-things.pth"))
    pipeline.propagator = Propagation(4, learnable=False)
    return pipeline.to("cuda"), raft


def _reference_pngs(pipeline, raft, bgr, steps, tile_size=None):
    """inference_upscale_a_video.py:180-351 with --color_fix Wavelet --save_image, frames as save_image writes them"""
    from upscale_a_video_b200 import color_correction, tiling
    vframes = _reference_ingest(bgr)
    flows_bi = list(raft.forward_slicing(vframes))
    generator = torch.Generator(device="cuda").manual_seed(10)
    kw = dict(num_inference_steps=steps, guidance_scale=6, noise_level=120, negative_prompt="blur, worst quality",
              propagation_steps=[0, 1])
    prompt = "best quality, extremely detailed"
    if tile_size is None:
        output = pipeline(prompt, image=vframes, flows_bi=flows_bi, generator=generator, **kw).images
    else:
        output = tiling.upscale_tiled(pipeline, vframes, flows_bi, generator, tile_size=tile_size, overlap=64,
                                      prompt=prompt, **kw)
    output = color_correction.color_fix_frames(output, vframes, "Wavelet")
    return _save_image_quantise(output).numpy()


def _run_and_check(tmp_path, model_dir, reference_models, t, h, w, extra, tile_size=None):
    from upscale_a_video_b200 import cli, video_io
    rgb = _bgr(t, h, w, 5)
    clip = tmp_path / "clip"
    video_io.write_frames(str(clip), rgb)
    bgr, _, _ = video_io.read_frames(str(clip))
    out = tmp_path / "out"
    written = cli.main(["-i", str(clip), "-o", str(out), "--model_dir", str(model_dir), "-s", "2", "-p", "0,1",
                        "--color_fix", "Wavelet", "--save_image", *extra])
    name = "clip_n120_g6_s2_p0_1"
    assert written == [str(out / "video" / f"{name}.mp4")]
    mp4, fps, _ = video_io.read_frames(written[0])
    assert mp4.shape == (t, 4 * h, 4 * w, 3) and fps == pytest.approx(10.0)
    pngs = sorted(os.listdir(out / "frame" / name))
    assert pngs == [f"{i:04d}.png" for i in range(t)]
    got = np.stack([cv2.imread(str(out / "frame" / name / p))[..., ::-1] for p in pngs])
    ref = _reference_pngs(*reference_models, bgr, 2, tile_size)
    assert got.shape == ref.shape and np.array_equal(got, ref)
    return got


def test_cli_end_to_end(tmp_path, model_dir, reference_models):
    _run_and_check(tmp_path, model_dir, reference_models, 4, 64, 64, [])


def test_cli_end_to_end_tiled(tmp_path, model_dir, reference_models):
    _run_and_check(tmp_path, model_dir, reference_models, 4, 80, 96, ["--perform_tile", "--tile_size", "32"], 32)


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_cli_torchrun_two_gpus(tmp_path, model_dir):
    """tiles dealt over two ranks give the single-GPU PNGs, written by rank 0 only"""
    from upscale_a_video_b200 import cli, video_io
    clip = tmp_path / "clip"
    video_io.write_frames(str(clip), _bgr(4, 80, 96, 5))
    args = ["-i", str(clip), "--model_dir", str(model_dir), "-s", "2", "-p", "0,1", "--color_fix", "Wavelet",
            "--save_image", "--perform_tile", "--tile_size", "32"]
    cli.main(args + ["-o", str(tmp_path / "one")])
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nproc-per-node", "2", "--master-port", "29531",
                        "-m", "upscale_a_video_b200", *args, "-o", str(tmp_path / "two")],
                       cwd=ROOT, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.count("Saving upscaled video") == 1
    name = "clip_n120_g6_s2_p0_1"
    for i in range(4):
        a = cv2.imread(str(tmp_path / "one" / "frame" / name / f"{i:04d}.png"))
        b = cv2.imread(str(tmp_path / "two" / "frame" / name / f"{i:04d}.png"))
        assert np.array_equal(a, b), i
