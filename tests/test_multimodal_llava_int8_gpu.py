"""The captioner with weight-only int8 decoder Linears on the GPU: quantization and dequantization bit-exact against
the CPU rule, the int8 GEMV against fp64 (no worse than the fp16 GEMV on the dequantized weight) and bitwise
independent of its batch, its argument checks, one 13B-shaped decoder layer, the reduced model against transformers'
LLaVA on the dequantized weights, batched captions, the load's memory, and the command with `--llava_int8`.

The name sorts after test_multimodal_llava_gpu.py for the reason given in test_multimodal_llava_batch_gpu.py: the
profiler-trace test of test_long_clip_gpu.py has been seen to miss its kernel when other GPU work runs before it."""
import numpy as np
import pytest
import torch

from llava_cases import text_config, vision_config, write_llava_folders
from llava_int8_cases import dequantize_ref, hand_rows, int8_decoder_bytes, quantize_rows_ref
from test_multimodal_llava_gpu import _layer_ref, _rel, _run_cli, cli_llava  # noqa: F401  (cli_llava: a fixture)
from test_cli_gpu import model_dir  # noqa: F401  (the synthetic Upscale-A-Video folder)

pytestmark = pytest.mark.gpu
SHAPES_13B = [(15360, 5120), (5120, 5120), (27648, 5120), (5120, 13824)]
SMALL = (77, 336)  # N not a multiple of 16, K not a multiple of 64


@pytest.fixture(autouse=True)
def _setup(uav_lib):
    """fp32 references without TF32; the process's setting is restored afterwards"""
    before = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = before


def _weights(N, K, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(N, K, generator=g) / K ** 0.5).half()


def _quantized(w):
    """Int8Rows of fp16 w (host) quantized on the device"""
    from upscale_a_video_b200 import ops
    from upscale_a_video_b200.llava import Int8Rows
    N, K = w.shape
    t = Int8Rows(torch.empty(N, K, dtype=torch.int8, device="cuda"), torch.empty(N, dtype=torch.float32, device="cuda"))
    ops.quantize_rows_int8(w.cuda(), t.q, t.absmax)
    return t


# ---------------------------------------------------------------- quantize / dequantize
@pytest.mark.parametrize("N,K", SHAPES_13B + [SMALL])
def test_quantize_and_dequantize_bit_exact(N, K):
    from upscale_a_video_b200 import ops
    w = _weights(N, K, N + K)
    q_ref, s_ref = quantize_rows_ref(w)
    # the source is a column slice of a wider buffer and the destination a row slice of a larger, sentinel-filled one
    src = torch.full((N, K + 24), float("nan"), dtype=torch.float16, device="cuda")
    src[:, 8:8 + K] = w.cuda()
    qb = torch.full((N + 6, K), 77, dtype=torch.int8, device="cuda")
    sb = torch.full((N + 6,), 1234.0, dtype=torch.float32, device="cuda")
    ops.quantize_rows_int8(src[:, 8:8 + K], qb[3:3 + N], sb[3:3 + N])
    assert torch.equal(qb[3:3 + N].cpu(), q_ref) and torch.equal(sb[3:3 + N].cpu(), s_ref)
    assert bool((qb[:3] == 77).all() and (qb[3 + N:] == 77).all() and (sb[:3] == 1234).all() and (sb[3 + N:] == 1234).all())
    out = ops.dequantize_rows_int8(qb[3:3 + N], sb[3:3 + N])
    assert torch.equal(out.cpu(), dequantize_ref(q_ref, s_ref))


def test_quantize_hand_made_rows():
    from upscale_a_video_b200 import ops
    w, expect = hand_rows()
    q = torch.empty(w.shape, dtype=torch.int8, device="cuda")
    s = torch.empty(w.shape[0], dtype=torch.float32, device="cuda")
    ops.quantize_rows_int8(w.cuda(), q, s)
    assert torch.equal(q.cpu(), expect)
    assert torch.equal(s.cpu(), quantize_rows_ref(w)[1])
    assert torch.equal(ops.dequantize_rows_int8(q, s).cpu(), dequantize_ref(expect, s.cpu()))


# ---------------------------------------------------------------- GEMV
@pytest.mark.parametrize("N,K", SHAPES_13B + [SMALL])
def test_gemv_rows_int8_accuracy_and_batch_invariance(N, K):
    from upscale_a_video_b200 import ops
    t = _quantized(_weights(N, K, 3 * N + K))
    w_exact = t.q.double() * (t.absmax.double() / 127)[:, None]       # decode's weight
    w_prefill = ops.dequantize_rows_int8(t.q, t.absmax)                # W'
    g = torch.Generator(device="cuda").manual_seed(N - K)
    x8 = torch.randn(8, K, generator=g, device="cuda").half()
    res8 = torch.randn(8, N, generator=g, device="cuda").half()
    pad = 64
    for rows in (1, 2, 3, 8):
        x, res = x8[:rows].contiguous(), res8[:rows].contiguous()
        for residual, dt in ((res, torch.float16), (None, torch.float16), (None, torch.float32)):
            buf = torch.full((rows * N + 2 * pad,), float("nan"), dtype=dt, device="cuda")
            out = buf[pad:pad + rows * N].view(rows, N)
            ops.gemv_rows_int8(t.q, t.absmax, x, residual=residual, out=out)
            assert bool(torch.isnan(buf[:pad]).all() and torch.isnan(buf[pad + rows * N:]).all()), "wrote outside out"
            first = out.clone()
            ops.gemv_rows_int8(t.q, t.absmax, x, residual=residual, out=out)
            assert torch.equal(first, out), "repeat launch differs"
            add = 0 if residual is None else residual.double()
            ref = ops.gemv_rows(w_prefill, x, residual=residual, out_dtype=dt)
            e_ours = _rel(out, x.double() @ w_exact.T + add)
            e_ref = _rel(ref, x.double() @ w_prefill.double().T + add)
            assert e_ours <= 1.5 * e_ref, (N, K, rows, residual is not None, dt, e_ours, e_ref)
            # a row's result does not depend on its batch
            for r in range(rows):
                one = ops.gemv_rows_int8(t.q, t.absmax, x[r:r + 1].contiguous(), out_dtype=dt,
                                         residual=None if residual is None else residual[r:r + 1].contiguous())
                assert torch.equal(out[r:r + 1], one), (N, K, rows, r, residual is not None, dt)


def test_gemv_rows_int8_rejects_bad_arguments():
    from upscale_a_video_b200 import _lib
    lib = _lib.load()
    q = torch.zeros(64, 14336 + 64, dtype=torch.int8, device="cuda")
    s = torch.ones(64, dtype=torch.float32, device="cuda")
    x = torch.zeros(9, 14336 + 64, dtype=torch.float16, device="cuda")
    out = torch.zeros(9, 64, dtype=torch.float16, device="cuda")
    good = (q.data_ptr(), s.data_ptr(), 64, 64, x.data_ptr(), 1, 0, out.data_ptr(), 0, 0)
    before = lib.uav_launch_count()
    cases = {"rows 0": dict(rows=0), "rows 9": dict(rows=9), "K % 16": dict(K=40),
             "rows * K over the limit": dict(K=14336, rows=8), "null absmax": dict(s=0),
             "misaligned q": dict(q=q.data_ptr() + 8), "misaligned x": dict(x=x.data_ptr() + 2),
             "fp32 out with a residual": dict(res=out.data_ptr(), dt=1)}
    for what, c in cases.items():
        args = list(good)
        for key, pos in (("q", 0), ("s", 1), ("K", 3), ("x", 4), ("rows", 5), ("res", 6), ("dt", 8)):
            if key in c:
                args[pos] = c[key]
        assert lib.uav_gemv_rows_int8(*args) != 0, what
    assert lib.uav_launch_count() == before, "a rejected call launched"
    assert lib.uav_gemv_rows_int8(*good) == 0
    torch.cuda.synchronize()


# ---------------------------------------------------------------- one 13B-shaped layer
def test_one_decoder_layer_13b_shape_int8():
    """prefill of 630 rows then one decode step through one 13B-shaped int8 layer, against fp32 torch on the
    dequantized weights W'; our error must be no worse than 1.5x that of the same torch layer in fp16"""
    from types import SimpleNamespace
    from upscale_a_video_b200 import ops
    from upscale_a_video_b200.llava import LLavaAgent, dequant_scratch
    H, heads, I, n = 5120, 40, 13824, 631
    g = torch.Generator(device="cuda").manual_seed(9)
    lin = lambda a, b, s=1.0: (torch.randn(a, b, generator=g, device="cuda") * (s / b ** 0.5)).half()
    w16 = {"qkv": torch.cat([lin(H, H, 2.0), lin(H, H, 2.0), lin(H, H)]), "o": lin(H, H), "gu": lin(2 * I, H),
           "down": lin(H, I)}
    q = {k: _quantized(v) for k, v in w16.items()}
    del w16
    w = {k: ops.dequantize_rows_int8(t.q, t.absmax) for k, t in q.items()}
    w["ln1"] = (1 + 0.1 * torch.randn(H, generator=g, device="cuda")).half()
    w["ln2"] = (1 + 0.1 * torch.randn(H, generator=g, device="cuda")).half()
    x = torch.randn(n, H, generator=g, device="cuda").half()
    agent = LLavaAgent.__new__(LLavaAgent)
    agent.config = SimpleNamespace(hidden_size=H, num_attention_heads=heads, rms_norm_eps=1e-5, rope_theta=10000.0)
    agent.device = torch.device("cuda")
    agent.w = {"qkv0": q["qkv"], "o0": q["o"], "gu0": q["gu"], "down0": q["down"], "ln1_0": w["ln1"], "ln2_0": w["ln2"]}
    agent._dq = dequant_scratch(agent.w, agent.device)
    rope = agent._rope_table(n)
    cache = torch.empty(2, n, H, dtype=torch.float16, device="cuda")
    with torch.no_grad():
        pre = agent._layer_prefill(0, x[:n - 1].clone(), cache[0], cache[1], rope)
        dec = agent._layer_decode(0, x[n - 1:].clone(), n - 1, cache[0], cache[1], rope)
        cfg = dict(hidden=H, heads=heads)
        r32 = _layer_ref(x, w, cfg, torch.float32)
        r16 = _layer_ref(x, w, cfg, torch.float16)
    for what, ours, a, b in (("prefill", pre, r32[:n - 1], r16[:n - 1]), ("decode", dec, r32[n - 1:], r16[n - 1:])):
        base = x[:n - 1] if what == "prefill" else x[n - 1:]
        e_ours, e_ref = _rel(ours.float() - base.float(), a - base.float()), _rel(b.float() - base.float(), a - base.float())
        print(f"13B int8 layer {what}: ours {e_ours:.3e}, torch fp16 {e_ref:.3e}")
        assert e_ours <= 1.5 * e_ref, (what, e_ours, e_ref)


# ---------------------------------------------------------------- the reduced model
@pytest.fixture(scope="module")
def reduced(tmp_path_factory):
    tc, vc = text_config(), vision_config()
    folder, clip, sd, vsd = write_llava_folders(str(tmp_path_factory.mktemp("llava_int8")), tc, vc)
    return tc, vc, folder, clip, sd, vsd


def _dequantized_state_dict(sd):
    """the released state dict with every Linear the int8 agent quantizes replaced by its W'"""
    out = dict(sd)
    for k, v in sd.items():
        if k.endswith("_proj.weight") or k in ("model.mm_projector.0.weight", "model.mm_projector.2.weight"):
            out[k] = dequantize_ref(*quantize_rows_ref(v))
    return out


def _px(agent, seed):
    from upscale_a_video_b200.llava import clip_preprocess, frame0_image
    frame = np.random.default_rng(seed).integers(0, 256, (90, 160, 3), dtype=np.uint8)
    return clip_preprocess(frame0_image(frame), agent.image_processor)


def test_whole_model_int8_against_transformers(reduced):
    from oracle.llava_oracle import build_llava, expand_image_ids
    from upscale_a_video_b200 import LLavaAgent
    tc, vc, folder, clip, sd, vsd = reduced
    agent = LLavaAgent(folder, vision_tower_path=clip, weights="int8")
    px = _px(agent, 4)
    ids = agent.prompt_ids()
    img_tok = tc["vocab_size"] - 1
    at = ids.index(-200)
    x = agent.embed_prompt(ids, agent.vision_features(px))
    n = x.shape[0]
    sdq = _dequantized_state_dict(sd)
    # transformers in fp32 and fp16 on W', and in fp32 on the original weights (printed, not asserted)
    models = {"fp32": (build_llava(tc, vc, sdq, vsd, img_tok, torch.float32).cuda(), torch.float32),
              "fp16": (build_llava(tc, vc, sdq, vsd, img_tok, torch.float16).cuda(), torch.float16),
              "original": (build_llava(tc, vc, sd, vsd, img_tok, torch.float32).cuda(), torch.float32)}
    input_ids = expand_image_ids(ids, img_tok, 576).cuda()
    feats, logit = {}, {}
    with torch.no_grad():
        m32 = models["fp32"][0]
        seq = input_ids
        for _ in range(17):  # teacher forcing: the fp32 oracle's own greedy continuation, fed to every model
            nxt = m32(input_ids=seq, pixel_values=px[None].cuda().float()).logits[0, -1].argmax()
            seq = torch.cat([seq, nxt.view(1, 1)], 1)
        forced = seq[0, n:].tolist()
        for name, (m, dt) in models.items():
            f = m.model.get_image_features(pixel_values=px[None].cuda().to(dt), vision_feature_layer=-2,
                                           vision_feature_select_strategy="default")
            f = getattr(f, "pooler_output", f)
            feats[name] = (torch.cat(list(f)) if isinstance(f, (list, tuple)) else f).reshape(-1, tc["hidden_size"])
            logit[name] = m(input_ids=seq[:, :-1], pixel_values=px[None].cuda().to(dt)).logits[0, n - 1:].float()
    ours_logits = torch.stack(agent.forward_logits(x, forced[:16]))
    ours_img = x[at:at + 576]
    for what, ours, pick in (("image features", ours_img, lambda d, k: d[k]),
                             ("prefill logits", ours_logits[0], lambda d, k: d[k][0]),
                             ("decode logits", ours_logits[1:], lambda d, k: d[k][1:17])):
        src = feats if what == "image features" else logit
        r32, r16, orig = pick(src, "fp32"), pick(src, "fp16"), pick(src, "original")
        e_ours, e_ref = _rel(ours, r32), _rel(r16, r32)
        print(f"int8 {what}: ours {e_ours:.3e}, transformers fp16 {e_ref:.3e} (against fp32 on W'); "
              f"against fp32 on the original fp16 weights {_rel(ours, orig):.3e}")
        assert e_ours <= 1.5 * e_ref, (what, e_ours, e_ref)


def test_batched_int8_captions_equal_one_image_captions(reduced):
    from upscale_a_video_b200 import LLavaAgent
    tc, vc, folder, clip, sd, vsd = reduced
    agent = LLavaAgent(folder, vision_tower_path=clip, weights="int8")
    px = torch.stack([_px(agent, 20 + i) for i in range(3)])
    greedy = agent.generate_ids_batch(px, temperature=0, max_new_tokens=24)
    assert greedy == [agent.generate_ids(px[i], temperature=0, max_new_tokens=24) for i in range(3)]
    gens = lambda: [torch.Generator().manual_seed(30 + i) for i in range(3)]
    sampled = agent.generate_ids_batch(px, generators=gens(), max_new_tokens=24)
    assert sampled == [agent.generate_ids(px[i], generator=g, max_new_tokens=24) for i, g in enumerate(gens())]


def test_int8_load_memory(reduced):
    from upscale_a_video_b200 import LLavaAgent
    from upscale_a_video_b200.llava import Int8Rows
    tc, vc, folder, clip, sd, vsd = reduced
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    agent = LLavaAgent(folder, vision_tower_path=clip, weights="int8")
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base

    def nbytes(t):
        return t.q.numel() + 4 * t.absmax.numel() if isinstance(t, Int8Rows) else t.numel() * t.element_size()
    w_bytes = sum(nbytes(t) for t in agent.w.values())
    assert w_bytes == int8_decoder_bytes(tc, vc["hidden_size"])
    assert all(isinstance(agent.w[k], Int8Rows) for k in ("qkv0", "o1", "gu0", "down1", "proj0_w", "proj2_w"))
    assert all(agent.w[k].dtype == torch.float16 for k in ("embed", "lm_head", "norm", "ln1_0"))
    tower_bytes = sum(t.numel() * t.element_size() for t in _tensors(agent.tower))
    largest = max(v.numel() for v in sd.values()) * 2
    print(f"int8 load: weights {w_bytes / 2**20:.1f} MiB, tower {tower_bytes / 2**20:.1f} MiB, "
          f"peak over baseline {peak / 2**20:.1f} MiB")
    assert peak <= w_bytes + tower_bytes + largest + 64 * 2**20, (peak, w_bytes, tower_bytes, largest)


def _tensors(obj):
    if isinstance(obj, torch.Tensor):
        yield obj
    elif isinstance(obj, (list, tuple)):
        for o in obj:
            yield from _tensors(o)
    elif hasattr(obj, "__dict__"):
        for o in vars(obj).values():
            yield from _tensors(o)


# ---------------------------------------------------------------- the command
def test_cli_llava_int8(tmp_path, model_dir, cli_llava, capsys):  # noqa: F811
    import textwrap
    from upscale_a_video_b200 import LLavaAgent, cli, video_io
    folder, clip = cli_llava
    flags = ["--llava_path", folder, "--llava_vision_path", clip, "--llava_int8"]
    printed, pngs = _run_cli(tmp_path, model_dir, "a", flags, capsys)
    # the caption the int8 captioner gives frame 0, printed as the reference prints it
    bgr, _, _ = video_io.read_frames(str(tmp_path / "clip"))
    caption = cli.caption_frame(LLavaAgent(folder, vision_tower_path=clip, weights="int8"), bgr[0])
    assert caption
    wrapped = textwrap.indent(textwrap.fill("Caption: " + caption, width=80), " " * 8)
    assert wrapped in printed and printed.count("Caption: ") == 1
    printed2, pngs2 = _run_cli(tmp_path, model_dir, "b", flags, capsys)
    assert wrapped in printed2 and printed2.count("Caption: ") == 1  # a second run prints the same caption
    assert np.array_equal(pngs, pngs2)
