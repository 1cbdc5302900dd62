"""Host logic of `python -m upscale_a_video_b200` (upscale_a_video_b200/cli.py, video_io.py): flags and defaults of the
reference CLI, output names, input discovery, OpenCV round trips, and the errors raised before any GPU work."""
import os

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

from upscale_a_video_b200 import cli, video_io  # noqa: E402


def _frames(t, h, w, seed=0):
    return np.random.default_rng(seed).integers(0, 256, size=(t, h, w, 3), dtype=np.uint8)


def test_parse_defaults_match_the_reference():
    a = cli.parse_args([])
    assert (a.input_path, a.output_path) == ("./inputs", "./results")
    assert (a.noise_level, a.guidance_scale, a.inference_steps, a.propagation_steps) == (120, 6, 30, [])
    assert a.a_prompt == "best quality, extremely detailed" and a.n_prompt == "blur, worst quality"
    assert a.color_fix == "None" and a.tile_size == 256 and a.save_suffix == ""
    assert not (a.use_video_vae or a.perform_tile or a.save_image or a.no_llava or a.load_8bit_llava)
    assert a.model_dir == "./pretrained_models/upscale_a_video" and a.caption == ""
    a = cli.parse_args(["-i", "x.mp4", "-o", "out", "-n", "50", "-g", "9", "-s", "20", "-p", "24,26,28", "--color_fix",
                        "Wavelet", "--perform_tile", "--tile_size", "128", "--save_image", "--save_suffix", "v1",
                        "--no_llava", "--use_video_vae"])
    assert a.propagation_steps == [24, 26, 28] and a.color_fix == "Wavelet" and a.tile_size == 128
    assert a.perform_tile and a.save_image and a.no_llava and a.use_video_vae


def test_rejected_flags(capsys):
    with pytest.raises(SystemExit):
        cli.parse_args(["--load_8bit_llava"])
    assert "no LLaVA captioner" in capsys.readouterr().err
    with pytest.raises(SystemExit):
        cli.parse_args(["--color_fix", "Histogram"])


def test_output_names():
    a = cli.parse_args(["-o", "res"])
    assert cli.output_paths(a, "clip") == (os.path.join("res", "video", "clip_n120_g6_s30.mp4"),
                                           os.path.join("res", "frame", "clip_n120_g6_s30"))
    a = cli.parse_args(["-o", "res", "-p", "24,26,28", "--save_suffix", "x", "-n", "80", "-g", "7", "-s", "45"])
    assert cli.save_name("clip", a) == "clip_n80_g7_s45_p24_26_28_x"
    assert cli.output_paths(a, "clip")[1] == os.path.join("res", "frame", "clip_n80_g7_s45_p24_26_28_x")


def test_lr_size_rule():
    assert cli.lr_size(1280, 1280) == (320, 320)
    assert cli.lr_size(1283, 1297) == (320, 324)
    assert cli.lr_size(1279, 2560) == (1279, 2560)
    assert cli.lr_size(720, 1280) == (720, 1280)


def test_input_discovery(tmp_path):
    video = tmp_path / "a.MP4"
    video.write_bytes(b"")
    assert video_io.find_inputs(str(video)) == [str(video)]
    # image folder: classified by its first entry in sorted order, whatever order listdir returns
    frames = tmp_path / "frames"
    frames.mkdir()
    for name in ("0000.png", "0001.PNG", "zz_notes.txt", "~backup"):
        (frames / name).write_bytes(b"")
    assert video_io.find_inputs(str(frames)) == [str(frames)]
    # folder of videos, walked recursively and sorted
    vids = tmp_path / "videos"
    (vids / "sub").mkdir(parents=True)
    for p in ("b.mp4", "a.avi", "sub/c.mov", "sub/readme.md"):
        (vids / p).write_bytes(b"")
    assert video_io.find_inputs(str(vids)) == [str(vids / "a.avi"), str(vids / "b.mp4"), str(vids / "sub" / "c.mov")]
    with pytest.raises(FileNotFoundError):
        video_io.find_inputs(str(tmp_path / "missing.mp4"))
    other = tmp_path / "other"
    other.mkdir()
    (other / "a.txt").write_bytes(b"")
    with pytest.raises(ValueError, match="Invalid input"):
        video_io.find_inputs(str(other))


def test_png_folder_round_trip(tmp_path):
    rgb = _frames(3, 17, 23)
    folder = tmp_path / "clip"
    paths = video_io.write_frames(str(folder), rgb)
    assert [os.path.basename(p) for p in paths] == ["0000.png", "0001.png", "0002.png"]
    (folder / "notes.txt").write_text("not a frame")
    bgr, fps, name = video_io.read_frames(str(folder) + os.sep)
    assert fps is None and name == "clip"
    assert np.array_equal(bgr[..., ::-1], rgb)  # PNG is lossless; frames come back in OpenCV's BGR order


def test_mp4_round_trip(tmp_path):
    rgb = _frames(5, 48, 64)
    for fps, expect in ((24, 24.0), (None, float(video_io.DEFAULT_FPS))):
        path = str(tmp_path / f"v{fps}.mp4")
        video_io.write_video(path, rgb, fps)
        bgr, got_fps, name = video_io.read_frames(path)
        assert bgr.shape == (5, 48, 64, 3) and bgr.dtype == np.uint8
        assert got_fps == pytest.approx(expect) and name == f"v{fps}"


def test_missing_checkpoint_file_is_named(tmp_path):
    frames = tmp_path / "in"
    video_io.write_frames(str(frames), _frames(2, 8, 8))
    d = tmp_path / "models"
    with pytest.raises(FileNotFoundError, match="text_encoder"):
        cli.main(["-i", str(frames), "-o", str(tmp_path / "out"), "--model_dir", str(d)])
    for rel in ("text_encoder/config.json", "tokenizer/vocab.json", "low_res_scheduler/scheduler_config.json",
                "vae/vae_3d_config.json", "vae/vae_3d.bin", "unet/unet_video_config.json", "unet/unet_video.bin",
                "scheduler/scheduler_config.json"):
        (d / rel).parent.mkdir(parents=True, exist_ok=True)
        (d / rel).write_bytes(b"")
    assert cli.checkpoint_paths(cli.parse_args(["--model_dir", str(d)]))["unet"] == str(d / "unet" / "unet_video.bin")
    missing = str(d / "propagator" / "raft-things.pth")
    with pytest.raises(FileNotFoundError, match=missing.replace("\\", "\\\\")):
        cli.main(["-i", str(frames), "--model_dir", str(d), "-p", "24,26"])
    with pytest.raises(FileNotFoundError, match="vae_video_config.json"):
        cli.main(["-i", str(frames), "--model_dir", str(d), "--use_video_vae"])
    assert not (tmp_path / "out").exists()


def test_new_entry_points_reject_bad_arguments(uav_lib):
    """argument checks come before any CUDA call, so they hold on a machine without a GPU"""
    from upscale_a_video_b200 import _lib
    assert uav_lib.uav_unpack_video_uint8(None, 1, 8, 8, 8, 8, 0, None, None) != 0
    p = 1 << 20  # never dereferenced: the shape check fails first
    for bad in ((1, 8, 8, 9, 8), (1, 8, 8, 8, 0), (0, 8, 8, 8, 8), (1, 8, 8, 2, 9), (1, 8, 8, 1, 1)):
        assert uav_lib.uav_unpack_video_uint8(p, *bad, 1, p, None) != 0, bad
    assert b"uav_unpack_video_uint8" in uav_lib.uav_last_error_string()
    assert uav_lib.uav_pack_frames_png(p, 1, 5, 8, 8, p, None) != 0  # C > 4
    with pytest.raises(_lib.UavError, match="uav_pack_frames_png"):
        _lib.check(uav_lib.uav_pack_frames_png(None, 1, 3, 8, 8, None, None), "uav_pack_frames_png")
    assert uav_lib.uav_launch_count() == 0
