"""`python -m upscale_a_video_b200` streams its output 3 frames at a time: on the GPU, the command's PNGs stay byte-identical
to the whole-clip library path, and the memory of the output phase does not grow with the clip's length."""
import json
import os
import shutil

import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

from test_cli_gpu import SCHED, _bgr, _reference_ingest, _save_image_quantise, _write_tokenizer  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG_CONFIGS = os.path.join(ROOT, "upscale_a_video_b200", "configs")
NAME = "clip_n120_g6_s2_p0_1"


@pytest.fixture(autouse=True)
def _setup(uav_lib):
    torch.manual_seed(0)


@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    """the released folder layout with seeded weights: text encoder (hidden 1024, 1 layer), tokenizer, schedulers,
    both VAEs, the full fp16 UNet and RAFT"""
    from upscale_a_video_b200 import AutoencoderKLVideo, CLIPTextConfig, CLIPTextModel, UNetVideoModel
    from upscale_a_video_b200.raft import RAFT
    from upscale_a_video_b200.synthetic import seeded_state_dict
    d = str(tmp_path_factory.mktemp("upscale_a_video_stream"))
    for sub in ("text_encoder", "low_res_scheduler", "scheduler", "vae", "unet", "propagator"):
        os.makedirs(os.path.join(d, sub))
    n_vocab = _write_tokenizer(d)
    cfg = dict(vocab_size=n_vocab, hidden_size=1024, intermediate_size=256, num_hidden_layers=1, num_attention_heads=16,
               max_position_embeddings=77, hidden_act="gelu", layer_norm_eps=1e-5)
    json.dump(dict(cfg, model_type="clip_text_model"), open(os.path.join(d, "text_encoder", "config.json"), "w"))
    torch.save(seeded_state_dict(CLIPTextModel(CLIPTextConfig(**cfg)), 78), os.path.join(d, "text_encoder",
                                                                                         "pytorch_model.bin"))
    json.dump({"beta_schedule": "scaled_linear", "_class_name": "DDPMScheduler"},
              open(os.path.join(d, "low_res_scheduler", "scheduler_config.json"), "w"))
    json.dump(SCHED, open(os.path.join(d, "scheduler", "scheduler_config.json"), "w"))
    json.dump({"max_noise_level": 350}, open(os.path.join(d, "model_index.json"), "w"))
    for kind, sub, cls, seed, dtype in (("vae_3d", "vae", AutoencoderKLVideo, 4322, torch.float32),
                                        ("vae_video", "vae", AutoencoderKLVideo, 4323, torch.float32),
                                        ("unet_video", "unet", UNetVideoModel, 1235, torch.float16)):
        shutil.copy(os.path.join(PKG_CONFIGS, f"{kind}_config.json"), os.path.join(d, sub, f"{kind}_config.json"))
        m = cls.from_config(os.path.join(PKG_CONFIGS, f"{kind}_config.json"))
        torch.save(seeded_state_dict(m, seed, dtype), os.path.join(d, sub, f"{kind}.bin"))
        del m
    sd = seeded_state_dict(RAFT(), 98)
    torch.save({"module." + k: v for k, v in sd.items()}, os.path.join(d, "propagator", "raft-things.pth"))
    return d


_MODELS = {}


def library_models(model_dir, vae_kind):
    """inference_upscale_a_video.py:101-131 through the public API"""
    if vae_kind not in _MODELS:
        from upscale_a_video_b200 import (AutoencoderKLVideo, DDIMScheduler, Propagation, RAFT_bi, UNetVideoModel,
                                          VideoUpscalePipeline)
        _MODELS.clear()
        pipeline = VideoUpscalePipeline.from_pretrained(model_dir, torch_dtype=torch.float16)
        pipeline.vae = AutoencoderKLVideo.from_config(os.path.join(model_dir, "vae", f"{vae_kind}_config.json"))
        pipeline.vae.load_state_dict(torch.load(os.path.join(model_dir, "vae", f"{vae_kind}.bin"), map_location="cpu"))
        pipeline.unet = UNetVideoModel.from_config(os.path.join(model_dir, "unet", "unet_video_config.json"))
        pipeline.unet.load_state_dict(torch.load(os.path.join(model_dir, "unet", "unet_video.bin"), map_location="cpu"),
                                      strict=True)
        pipeline.unet = pipeline.unet.half().eval()
        pipeline.scheduler = DDIMScheduler.from_config(os.path.join(model_dir, "scheduler", "scheduler_config.json"))
        raft = RAFT_bi(os.path.join(model_dir, "propagator", "raft-things.pth"))
        pipeline.propagator = Propagation(4, learnable=False)
        _MODELS[vae_kind] = (pipeline.to("cuda"), raft)
    return _MODELS[vae_kind]


KW = dict(num_inference_steps=2, guidance_scale=6, noise_level=120, negative_prompt="blur, worst quality",
          propagation_steps=[0, 1])
PROMPT = "best quality, extremely detailed"


def library_output(pipeline, raft, vframes, tile_size):
    """the whole clip through the library, as the command computed it before it streamed"""
    from upscale_a_video_b200 import tiling
    flows_bi = list(raft.forward_slicing(vframes))
    generator = torch.Generator(device="cuda").manual_seed(10)
    if tile_size is None:
        return pipeline(PROMPT, image=vframes, flows_bi=flows_bi, generator=generator, **KW).images
    return tiling.upscale_tiled(pipeline, vframes, flows_bi, generator, tile_size=tile_size, overlap=64, prompt=PROMPT,
                                **KW)


def run_command(tmp_path, model_dir, t, h, w, extra):
    from upscale_a_video_b200 import cli, video_io
    clip = tmp_path / "clip"
    video_io.write_frames(str(clip), _bgr(t, h, w, 5))
    out = tmp_path / "out"
    written = cli.main(["-i", str(clip), "-o", str(out), "--model_dir", str(model_dir), "-s", "2", "-p", "0,1",
                        "--save_image", *extra])
    assert written == [str(out / "video" / f"{NAME}.mp4")]
    return clip, out


CASES = {  # (h, w, color fix, vae, tile size)
    "untiled-adain": (64, 64, "AdaIn", "vae_3d", None),
    "untiled-wavelet-video_vae": (64, 64, "Wavelet", "vae_video", None),
    "tiled-wavelet": (80, 96, "Wavelet", "vae_3d", 32),
    "tiled-adain-video_vae": (80, 96, "AdaIn", "vae_video", 32),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_streamed_command_matches_whole_clip(tmp_path, model_dir, case):
    """14 frames (chunks 3 + 3 + 3 + 3 + 2): PNGs byte-identical to pipeline / upscale_tiled -> color_fix_frames ->
    save_image's rounding, and an mp4 of 14 frames"""
    from upscale_a_video_b200 import color_correction, video_io
    h, w, fix, vae, tile = CASES[case]
    t = 14
    extra = ["--color_fix", fix] + (["--use_video_vae"] if vae == "vae_video" else [])
    extra += ["--perform_tile", "--tile_size", str(tile)] if tile else []
    clip, out = run_command(tmp_path, model_dir, t, h, w, extra)
    mp4, _, _ = video_io.read_frames(str(out / "video" / f"{NAME}.mp4"))
    assert mp4.shape == (t, 4 * h, 4 * w, 3)
    pngs = sorted(os.listdir(out / "frame" / NAME))
    assert pngs == [f"{i:04d}.png" for i in range(t)]
    got = np.stack([cv2.imread(str(out / "frame" / NAME / p))[..., ::-1] for p in pngs])
    bgr, _, _ = video_io.read_frames(str(clip))
    vframes = _reference_ingest(bgr)
    output = library_output(*library_models(model_dir, vae), vframes, tile)
    ref = _save_image_quantise(color_correction.color_fix_frames(output, vframes, fix)).numpy()
    assert got.shape == ref.shape and np.array_equal(got, ref)


def _requested(kind):
    """bytes the program asked the caching allocator for ("current" or "peak").  `max_memory_allocated()` counts a
    reused cached block with its whole size, up to 1 MiB more than was asked for; at 64x64, where 0.1 x 24 output
    frames are 1.8 MiB, that slack changes from run to run by as much as the bound."""
    return torch.cuda.memory_stats()[f"requested_bytes.all.{kind}"]


def _phase_start(state):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    state["base"] = _requested("current")
    assert _requested("peak") == state["base"]  # the reset covers the requested-bytes peak


def _phase_bytes(state):
    torch.cuda.synchronize()
    return _requested("peak") - state["base"]


def streamed_output_phase(tmp_path, model_dir, monkeypatch, t, h, w, tile):
    """output-phase memory of the command: from the end of sampling (untiled: `sample_latents` returned; tiled: the
    first chunk left `iter_upscale_tiled`) to the end of the clip"""
    from upscale_a_video_b200 import VideoUpscalePipeline, tiling
    state = {}
    with monkeypatch.context() as m:
        if tile is None:
            real = VideoUpscalePipeline.sample_latents

            def hooked(self, *a, **k):
                r = real(self, *a, **k)
                _phase_start(state)
                return r
            m.setattr(VideoUpscalePipeline, "sample_latents", hooked)
        else:
            real = tiling.iter_upscale_tiled

            def hooked(*a, **k):
                for i, item in enumerate(real(*a, **k)):
                    if i == 0:
                        _phase_start(state)
                    yield item
            m.setattr(tiling, "iter_upscale_tiled", hooked)
        extra = ["--color_fix", "Wavelet"] + (["--perform_tile", "--tile_size", str(tile)] if tile else [])
        run_command(tmp_path / f"t{t}", model_dir, t, h, w, extra)
    return _phase_bytes(state)


def whole_clip_output_phase(model_dir, t, h, w):
    """the same phase for the whole clip: decode every chunk, concatenate, colour-fix, pack for the mp4 and the PNGs,
    copy.  Returns (bytes from the end of sampling, bytes from the end of the decode)."""
    from upscale_a_video_b200 import color_correction
    pipeline, raft = library_models(model_dir, "vae_3d")
    vframes = _reference_ingest(_bgr(t, h, w, 5))
    flows_bi = list(raft.forward_slicing(vframes))
    sampled = pipeline.sample_latents(PROMPT, image=vframes, flows_bi=flows_bi,
                                      generator=torch.Generator(device="cuda").manual_seed(10), **KW)
    del flows_bi
    from_sampling, from_decode = {}, {}
    _phase_start(from_sampling)
    chunks = [f for _, _, f in pipeline.decode_chunks(sampled)]
    torch.cuda.synchronize()
    decode_peak = _requested("peak")
    _phase_start(from_decode)
    output = torch.cat(chunks, dim=2)
    del chunks
    frames = color_correction.color_fix_frames(output, vframes, "Wavelet")
    del output
    video = color_correction.pack_video_uint8(frames).cpu()
    png = color_correction.pack_frames_png(frames).cpu()
    assert video.shape[0] == png.shape[0] == t
    after_decode = _phase_bytes(from_decode)
    return max(decode_peak, from_decode["base"] + after_decode) - from_sampling["base"], after_decode


@pytest.mark.parametrize("tiled", [False, True])
def test_output_phase_memory_does_not_grow_with_clip_length(tmp_path, model_dir, monkeypatch, tiled):
    """Wavelet and propagation at 14 and 38 frames (both end in a 2-frame chunk): the command's output phase grows by
    less than 0.1 x 24 fp32 output frames; the whole clip's concatenation, colour fix and packing by at least 4 x 24"""
    h, w, tile = (80, 96, 32) if tiled else (64, 64, None)
    frame = 4 * h * 4 * w * 3 * 4
    streamed = {t: streamed_output_phase(tmp_path, model_dir, monkeypatch, t, h, w, tile) for t in (14, 38)}
    growth = streamed[38] - streamed[14]
    print(f"\n[{'tiled' if tiled else 'untiled'} {h}x{w}] streamed output phase: T=14 {streamed[14] / 2**20:.2f} MiB, "
          f"T=38 {streamed[38] / 2**20:.2f} MiB, growth {growth / 2**20:.3f} MiB = {growth / frame:.3f} fp32 frames "
          f"({frame / 2**20:.3f} MiB each)")
    assert growth < 0.1 * 24 * frame
    if not tiled:
        # At 64x64 the decoder's activations for one 3-frame chunk take about as much as 360 fp32 output frames, so
        # a window that includes the decode shows the whole clip's growth only from about 70 frames on.  The
        # positive control therefore asserts on the window that starts after the decode (the chunks are then
        # already held, so it undercounts the growth by one clip) and prints both.
        whole_clip_output_phase(model_dir, 3, h, w)  # packs this pipeline's decoder weights outside the windows
        whole = {t: whole_clip_output_phase(model_dir, t, h, w) for t in (14, 38)}
        for k, label in ((0, "from the end of sampling"), (1, "from the end of the decode")):
            g = whole[38][k] - whole[14][k]
            print(f"[untiled {h}x{w}] whole-clip output phase {label}: T=14 {whole[14][k] / 2**20:.2f} MiB, T=38 "
                  f"{whole[38][k] / 2**20:.2f} MiB, growth {g / 2**20:.2f} MiB = {g / frame / 24:.2f} x 24 frames")
        assert whole[38][1] - whole[14][1] >= 4 * 24 * frame
