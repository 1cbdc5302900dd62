"""Batched captions on the host: generator-list validation, grouping into batches of at most CAPTION_BATCH, the
batched entry points of the C ABI, and `video_io.read_first_frame`."""
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_caption_groups():
    from upscale_a_video_b200.llava import CAPTION_BATCH, caption_groups
    assert CAPTION_BATCH == 8
    assert caption_groups(0) == []
    assert [list(g) for g in caption_groups(3)] == [[0, 1, 2]]
    assert [list(g) for g in caption_groups(8)] == [list(range(8))]
    assert [list(g) for g in caption_groups(17)] == [list(range(8)), list(range(8, 16)), [16]]


def test_generator_list_validation():
    from upscale_a_video_b200.llava import LLavaAgent, _caption_generators
    gens = [torch.Generator().manual_seed(i) for i in range(3)]
    assert _caption_generators(3, 0.2, gens) == (gens, True)
    g = torch.Generator()
    assert _caption_generators(3, 0.2, g) == ([g] * 3, False)   # one generator, sampled: one image at a time
    assert _caption_generators(3, 0.0, g) == ([g] * 3, True)    # greedy: no uniforms drawn
    assert _caption_generators(2, 0.2, None) == ([None] * 2, False)
    # one generator listed twice, or the global RNG in a list, is shared: its draws follow the one-at-a-time order
    assert _caption_generators(3, 0.2, [gens[0], gens[1], gens[0]]) == ([gens[0], gens[1], gens[0]], False)
    assert _caption_generators(2, 0.2, [gens[0], None]) == ([gens[0], None], False)
    assert _caption_generators(2, 0.0, [gens[0], gens[0]]) == ([gens[0], gens[0]], True)
    agent = LLavaAgent.__new__(LLavaAgent)  # the check runs before any model work
    with pytest.raises(ValueError, match="one per image"):
        agent.gen_image_caption([object()] * 3, generator=gens[:2])
    with pytest.raises(ValueError):
        agent.gen_image_caption([object()] * 2, generator=tuple(gens))


def test_batched_entry_points_declared():
    from upscale_a_video_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "uav_b200.h")).read()
    declared = set(re.findall(r"\b(uav_[a-z0-9_]+)\s*\(", hdr))
    new = {"uav_gemv_rows", "uav_attention_decode_batched", "uav_attention_decode_batched_workspace_bytes",
           "uav_rope_kv_append_batched", "uav_sample_top_p_batched"}
    assert new <= declared and new <= set(_lib.declared_symbols())
    assert len(declared) == 64


def _frames(t, h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, size=(t, h, w, 3), dtype=np.uint8)


def test_read_first_frame_video_and_folder(tmp_path):
    pytest.importorskip("cv2")
    from upscale_a_video_b200 import video_io
    path = str(tmp_path / "clip.mp4")
    video_io.write_video(path, _frames(4, 48, 64, 1), 10)
    assert np.array_equal(video_io.read_first_frame(path), video_io.read_frames(path)[0][0])
    folder = str(tmp_path / "frames")
    video_io.write_frames(folder, _frames(3, 40, 56, 2))
    open(os.path.join(folder, "notes.txt"), "w").write("not a frame")
    first = video_io.read_first_frame(folder)
    assert first.shape == (40, 56, 3) and np.array_equal(first, video_io.read_frames(folder)[0][0])
    with pytest.raises(RuntimeError):
        video_io.read_first_frame(str(tmp_path / "missing.mp4"))
    empty = tmp_path / "empty"
    empty.mkdir()
    with pytest.raises(RuntimeError):
        video_io.read_first_frame(str(empty))
