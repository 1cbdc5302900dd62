"""Batched captions on the GPU: every batched kernel against its one-row counterpart on each row, one 13B-shaped
decoder layer on four prompts at once, the reduced model's batched logits and captions against one-image runs, and
the command's group captioning.  Every comparison is bitwise: a row's result must not depend on the rest of its batch.

The name sorts after test_long_clip_gpu.py for the reason given in test_multimodal_llava_gpu.py: the kernel-selection
test there reads a torch.profiler trace that other GPU work run between the two files has been seen to disturb."""
import os
import textwrap

import numpy as np
import pytest
import torch

from llava_cases import text_config, vision_config, write_llava_folders

pytestmark = pytest.mark.gpu
SENTINEL = 1234.0
SHAPES_13B = [(15360, 5120), (5120, 5120), (27648, 5120), (5120, 13824), (32000, 5120)]


@pytest.fixture(autouse=True)
def _setup(uav_lib):
    yield


def _agent_stub(H, heads):
    from types import SimpleNamespace
    from upscale_a_video_b200.llava import LLavaAgent
    agent = LLavaAgent.__new__(LLavaAgent)
    agent.config = SimpleNamespace(hidden_size=H, num_attention_heads=heads, rms_norm_eps=1e-5, rope_theta=10000.0)
    agent.device = torch.device("cuda")
    return agent


# ---------------------------------------------------------------- kernels
@pytest.mark.parametrize("rows", [2, 3, 8])
@pytest.mark.parametrize("N,K", SHAPES_13B)
def test_gemv_rows_equals_gemv(N, K, rows):
    from upscale_a_video_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(N + K + rows)
    w = (torch.randn(N, K, generator=g, device="cuda") / K ** 0.5).half()
    x = torch.randn(rows, K, generator=g, device="cuda").half()
    res = torch.randn(rows, N, generator=g, device="cuda").half()
    for residual, dt in ((res, torch.float16), (None, torch.float16), (None, torch.float32)):
        pad = 64
        buf = torch.full((rows * N + 2 * pad,), float("nan"), dtype=dt, device="cuda")
        out = buf[pad:pad + rows * N].view(rows, N)
        ops.gemv_rows(w, x, residual=residual, out=out)
        assert bool(torch.isnan(buf[:pad]).all() and torch.isnan(buf[pad + rows * N:]).all()), "wrote outside out"
        for r in range(rows):
            want = ops.gemv(w, x[r].contiguous(), residual=None if residual is None else residual[r].contiguous(),
                            out_dtype=dt)
            assert torch.equal(out[r], want), (N, K, rows, r, residual is not None, dt)


def test_gemv_rows_rejects_bad_rows():
    from upscale_a_video_b200 import _lib
    w = torch.zeros(64, 64, dtype=torch.float16, device="cuda")
    x = torch.zeros(9, 64, dtype=torch.float16, device="cuda")
    out = torch.zeros(9, 64, dtype=torch.float16, device="cuda")
    lib = _lib.load()
    for rows in (0, 9):
        assert lib.uav_gemv_rows(w.data_ptr(), 64, 64, x.data_ptr(), rows, 0, out.data_ptr(), 0, 0) != 0
    big = torch.zeros(8, 14336, dtype=torch.float16, device="cuda")  # 8 x 14336 exceeds the shared-memory x
    wb = torch.zeros(64, 14336, dtype=torch.float16, device="cuda")
    assert lib.uav_gemv_rows(wb.data_ptr(), 64, 14336, big.data_ptr(), 8, 0, out.data_ptr(), 0, 0) != 0


@pytest.mark.parametrize("L", [1, 64, 129, 700])
def test_attention_decode_batched_equals_per_row(L):
    from upscale_a_video_b200 import ops
    B, heads, H = 3, 40, 5120
    Lmax = L + 37
    g = torch.Generator(device="cuda").manual_seed(L)
    cache = torch.full((2, B, Lmax, H), float("nan"), dtype=torch.float16, device="cuda")
    cache[:, :, :L] = torch.randn(2, B, L, H, generator=g, device="cuda").half()
    qkv = torch.randn(B, 3 * H, generator=g, device="cuda").half()
    for b in range(B):  # a needle per sequence, at a different key
        cache[0, b, (b * 53) % L, :128] = (qkv[b, :128].float() * 0.6).half()
    buf = torch.full((B, H + 64), SENTINEL, dtype=torch.float16, device="cuda")
    out = buf[:, 32:32 + H]
    ops.attention_decode_batched(qkv[:, :H], cache[0], cache[1], L, heads, out=out)
    assert bool((buf[:, :32] == SENTINEL).all() and (buf[:, 32 + H:] == SENTINEL).all()), "wrote outside out"
    for b in range(B):
        want = ops.attention_decode(qkv[b, :H].contiguous(), cache[0, b], cache[1, b], L, heads)
        assert torch.equal(out[b], want), (L, b)


@pytest.mark.parametrize("n,p0", [(630, 0), (1, 700)])
def test_rope_kv_append_batched_equals_per_sequence(n, p0):
    from upscale_a_video_b200 import ops
    B, heads, H = 3, 40, 5120
    L = p0 + n + 5
    g = torch.Generator(device="cuda").manual_seed(n)
    qkv = torch.randn(B, n, 3 * H, generator=g, device="cuda").half()
    rope = _agent_stub(H, heads)._rope_table(L)
    ours_qkv = qkv.clone()
    ours = torch.full((2, B, L, H), SENTINEL, dtype=torch.float16, device="cuda")
    ops.rope_kv_append_batched(ours_qkv, heads, p0, rope, ours[0], ours[1])
    want_qkv = qkv.clone()
    want = torch.full((2, B, L, H), SENTINEL, dtype=torch.float16, device="cuda")
    for b in range(B):
        ops.rope_kv_append(want_qkv[b], heads, p0, rope, want[0, b], want[1, b])
    assert torch.equal(ours_qkv, want_qkv)
    assert torch.equal(ours, want)


def test_sample_top_p_batched_equals_per_row():
    from upscale_a_video_b200 import ops
    g = torch.Generator().manual_seed(21)
    B, V = 6, 32000
    x = torch.randn(B, V, generator=g) * 2
    x[0, [5, 17, 31999]] = x[0].max() + 1  # argmax ties
    x[1, [31998, 31999]] = x[1].max() + 1
    x[2, torch.randint(V, (4,), generator=g)] += 6
    x = x.cuda()
    for temperature, top_p in ((0.0, 0.7), (0.2, 0.7), (1.0, 0.9)):
        for trial in range(4):
            u = torch.rand(B, generator=g).tolist()
            got = ops.sample_top_p_batched(x, temperature, top_p, u)
            for b in range(B):
                want = ops.sample_top_p(x[b].contiguous(), temperature, top_p, u[b])
                assert int(got[b]) == int(want), (temperature, trial, b)
    assert int(ops.sample_top_p_batched(x[:1], 0.0, 0.7, [0.0])[0]) == 5


# ---------------------------------------------------------------- one 13B-shaped layer, four prompts
def test_decoder_layer_13b_batch_of_four():
    H, heads, I, n, B = 5120, 40, 13824, 630, 4
    g = torch.Generator(device="cuda").manual_seed(9)
    lin = lambda a, b, s=1.0: (torch.randn(a, b, generator=g, device="cuda") * (s / b ** 0.5)).half()
    agent = _agent_stub(H, heads)
    agent.w = {"qkv0": torch.cat([lin(H, H, 2.0), lin(H, H, 2.0), lin(H, H)]), "o0": lin(H, H), "gu0": lin(2 * I, H),
               "down0": lin(H, I), "ln1_0": (1 + 0.1 * torch.randn(H, generator=g, device="cuda")).half(),
               "ln2_0": (1 + 0.1 * torch.randn(H, generator=g, device="cuda")).half()}
    x = torch.randn(B, n + 1, H, generator=g, device="cuda").half()
    L = n + 3
    rope = agent._rope_table(L)
    with torch.no_grad():
        cache = torch.zeros(2, B, L, H, dtype=torch.float16, device="cuda")
        pre = agent._layer_prefill(0, x[:, :n].reshape(B * n, H).clone(), cache[0], cache[1], rope).view(B, n, H)
        dec = agent._layer_decode(0, x[:, n].clone(), n, cache[0], cache[1], rope)
        for b in range(B):
            c1 = torch.zeros(2, L, H, dtype=torch.float16, device="cuda")
            p1 = agent._layer_prefill(0, x[b, :n].clone(), c1[0], c1[1], rope)
            d1 = agent._layer_decode(0, x[b, n:n + 1].clone(), n, c1[0], c1[1], rope)
            assert torch.equal(pre[b], p1), b
            assert torch.equal(dec[b], d1[0]), b
            assert torch.equal(cache[:, b], c1), b


# ---------------------------------------------------------------- the reduced model
@pytest.fixture(scope="module")
def small_llava(tmp_path_factory):
    """a tiny LLaVA whose vocabulary is the golden tokenizer's, with the EOS row of lm_head scaled so that greedy
    captions of different images end at different steps"""
    from upscale_a_video_b200 import LLavaAgent
    from upscale_a_video_b200.llava import clip_preprocess, frame0_image
    tc = text_config(hidden=256, heads=2, layers=2, inter=512, vocab=400)
    vc = vision_config(hidden=128, heads=2, layers=2, inter=256)
    folder, clip, _, _ = write_llava_folders(str(tmp_path_factory.mktemp("batch_llava")), tc, vc)
    agent = LLavaAgent(folder, vision_tower_path=clip)
    rng = np.random.default_rng(7)
    imgs = [frame0_image(rng.integers(0, 256, (90, 160, 3), dtype=np.uint8)) for _ in range(9)]
    px = torch.stack([clip_preprocess(im, agent.image_processor) for im in imgs])
    eos_row = agent.w["lm_head"][agent.eos_id].clone()
    for scale in (1.0, 1.5, 2.0, 3.0, 4.0, 6.0, 8.0):
        agent.w["lm_head"][agent.eos_id] = (eos_row.float() * scale).half()
        lengths = [len(agent.generate_ids(px[i], temperature=0, max_new_tokens=24)) for i in range(4)]
        if len(set(lengths)) > 1 and min(lengths) < 24:
            break
    return agent, imgs, px, folder, clip


def test_batched_logits_equal_per_image(small_llava):
    agent, _, px, _, _ = small_llava
    B, steps = 4, 12
    ids = agent.prompt_ids()
    x = agent.embed_prompt(ids, agent.vision_features(px[:B]))
    assert x.shape[0] == B
    for b in range(B):
        assert torch.equal(x[b], agent.embed_prompt(ids, agent.vision_features(px[b])))
    g = torch.Generator().manual_seed(3)
    forced = [torch.randint(3, 400, (steps,), generator=g).tolist() for _ in range(B)]
    ours = agent.forward_logits_batch(x, forced)
    assert len(ours) == steps + 1
    for b in range(B):
        one = agent.forward_logits(x[b], forced[b])
        for step in range(steps + 1):
            assert torch.equal(ours[step][b], one[step]), (b, step)


def test_batched_captions_equal_one_image_calls(small_llava):
    from upscale_a_video_b200 import llava
    agent, imgs, px, _, _ = small_llava
    # the rows of a batch end at different steps
    lengths = [len(t) for t in agent.generate_ids_batch(px[:8], temperature=0)]
    assert len(set(lengths)) > 1 and min(lengths) < 64, lengths
    calls = []
    real = agent.generate_ids_batch

    def counting(p, *a, **k):
        calls.append(p.shape[0])
        return real(p, *a, **k)

    agent.generate_ids_batch = counting
    try:
        gens = lambda: [torch.Generator().manual_seed(100 + i) for i in range(9)]
        caps = agent.gen_image_caption(imgs, generator=gens())
        assert calls == [8, 1]
        one = [agent.gen_image_caption([im], generator=g)[0] for im, g in zip(imgs, gens())]
        assert caps == one
        calls.clear()
        greedy = agent.gen_image_caption(imgs, temperature=0)
        assert calls == [8, 1]
        assert greedy == [agent.gen_image_caption([im], temperature=0)[0] for im in imgs]
        # sampled captions differ between images at all: the test compares something
        assert len(set(caps)) > 1
        calls.clear()
        agent.gen_image_caption(imgs[:3], generator=torch.Generator().manual_seed(1))  # one generator: one at a time
        assert calls == [1, 1, 1]
    finally:
        del agent.generate_ids_batch
    assert llava.CAPTION_BATCH == 8


# ---------------------------------------------------------------- the command
from test_cli_gpu import _bgr, model_dir  # noqa: E402,F401  (the synthetic Upscale-A-Video folder)


def test_cli_captions_a_group_of_clips(tmp_path, model_dir, small_llava, capsys, monkeypatch):
    import cv2
    from upscale_a_video_b200 import LLavaAgent, cli, video_io
    _, _, _, folder, clip = small_llava
    clips = tmp_path / "clips"
    clips.mkdir()
    names = ["a", "b", "c"]
    for k, name in enumerate(names):
        video_io.write_video(str(clips / f"{name}.mp4"), _bgr(3, 64, 64, 20 + k)[..., ::-1].copy(), 10)

    def pngs(out, name):
        d = out / "frame" / f"{name}_n120_g6_s2"
        return np.stack([cv2.imread(str(d / p)) for p in sorted(os.listdir(d))])

    calls = []
    real = LLavaAgent.gen_image_caption

    def counting(self, imgs, *a, **k):
        calls.append(len(imgs))
        return real(self, imgs, *a, **k)

    monkeypatch.setattr(LLavaAgent, "gen_image_caption", counting)
    capsys.readouterr()
    cli.main(["-i", str(clips), "-o", str(tmp_path / "all"), "--model_dir", str(model_dir), "-s", "2", "--save_image",
              "--llava_path", folder, "--llava_vision_path", clip])
    printed = capsys.readouterr().out
    assert calls == [3]
    monkeypatch.setattr(LLavaAgent, "gen_image_caption", real)
    agent = LLavaAgent(folder, vision_tower_path=clip)
    assert printed.count("Caption: ") == 3
    for name in names:
        path = str(clips / f"{name}.mp4")
        assert np.array_equal(video_io.read_first_frame(path), video_io.read_frames(path)[0][0])
        caption = cli.caption_frame(agent, video_io.read_first_frame(path))
        wrapped = textwrap.indent(textwrap.fill("Caption: " + caption, width=80), " " * 8)
        assert wrapped in printed, name
        cli.main(["-i", path, "-o", str(tmp_path / name), "--model_dir", str(model_dir), "-s", "2", "--save_image",
                  "--caption", caption])
        assert np.array_equal(pngs(tmp_path / "all", name), pngs(tmp_path / name, name)), name


# ---------------------------------------------------------------- the measurement tool runs in both modes
@pytest.mark.parametrize("extra", [[], ["--rows", "1,2"]], ids=["one-row", "rows"])
def test_bench_llava_runs(tmp_path, extra):
    import json
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = tmp_path / "r.json"
    r = subprocess.run([sys.executable, os.path.join(root, "tools", "bench_llava.py"), "--layers", "1", *extra,
                        "--json", str(out)], cwd=str(tmp_path), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    res = json.load(open(out))
    if extra:
        assert [row["rows"] for row in res["rows"]] == [1, 2]
        assert all(len(row["seconds_per_call"]) == 3 for row in res["rows"])
    else:
        assert res["ms_per_token"] > 0 and res["seconds_per_caption"] > 0 and len(res["gemv"]) == 5
