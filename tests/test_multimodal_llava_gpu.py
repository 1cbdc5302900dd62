"""The LLaVA captioner on the GPU: its kernels at the 13B shapes against fp64 torch (operands read from NaN-filled
buffers, outputs written into slices of sentinel-filled buffers, every launch repeated and bitwise equal), the sampler,
the whole model at a reduced config against transformers' LlavaForConditionalGeneration, one decoder layer at the 13B
shape, and the command end to end on a synthetic folder.

The file sorts after test_long_clip_gpu.py on purpose.  That file's kernel-selection test reads a torch.profiler trace
in-process, after test_igemm_wide_gpu.py's traces.  When other GPU work runs between the two files, the trace has been
seen to miss the kernel it checks for.  The cuBLAS, transformers and captioner work here then runs after the last
in-process trace of the suite."""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

from attention_cases import GENERATORS, U32, Ref, assert_matches, make_inputs, softmax_ref
from llava_cases import text_config, vision_config, write_llava_folders

pytestmark = pytest.mark.gpu
SENTINEL = 1234.0
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(autouse=True)
def _setup(uav_lib):
    """fp32 references without TF32; the process's setting is restored afterwards"""
    before = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = before


def _nan_embed(x, pad=64):
    """x (contiguous) as a slice in the middle of a NaN-filled buffer"""
    buf = torch.full((x.numel() + 2 * pad,), float("nan"), dtype=x.dtype, device="cuda")
    view = buf[pad:pad + x.numel()].view(x.shape)
    view.copy_(x)
    return view


def _sentinel_out(n, dtype, pad=64):
    buf = torch.full((n + 2 * pad,), SENTINEL, dtype=dtype, device="cuda")
    return buf, buf[pad:pad + n]


def _check_sentinel(buf, n, pad=64):
    assert bool((buf[:pad] == SENTINEL).all() and (buf[pad + n:] == SENTINEL).all()), "wrote outside its output"


# ---------------------------------------------------------------- GEMV
@pytest.mark.parametrize("N,K", [(15360, 5120), (5120, 5120), (27648, 5120), (5120, 13824), (32000, 5120)])
def test_gemv(N, K):
    from upscale_a_video_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(N + K)
    w = (torch.randn(N, K, generator=g, device="cuda") / K ** 0.5).half()
    x = _nan_embed(torch.randn(K, generator=g, device="cuda").half())
    res = _nan_embed(torch.randn(N, generator=g, device="cuda").half())
    ref = w.double() @ x.double()
    bound = (w.double().abs() @ x.double().abs()) * 2 ** -20 * 4
    for residual, dt in ((None, torch.float16), (res, torch.float16), (None, torch.float32)):
        buf, out = _sentinel_out(N, dt)
        ops.gemv(w, x, residual=residual, out=out)
        _check_sentinel(buf, N)
        first = out.clone()
        ops.gemv(w, x, residual=residual, out=out)
        assert torch.equal(first, out), "repeat launch differs"
        want = ref + (0 if residual is None else residual.double())
        tol = bound + (want.abs() * 2 ** -11 if dt == torch.float16 else 0) + 1e-6
        err = (out.double() - want).abs()
        assert bool((err <= tol).all()), (N, K, residual is not None, dt, err.max().item())


# ---------------------------------------------------------------- RMSNorm, RoPE + KV append, SwiGLU
def test_rmsnorm_5120():
    from upscale_a_video_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(1)
    rows, C = 7, 5120
    xb = torch.full((rows, C + 64), float("nan"), dtype=torch.float16, device="cuda")
    xb[:, 32:32 + C] = (torch.randn(rows, C, generator=g, device="cuda") * 3).half()
    x = xb[:, 32:32 + C]
    wt = (1 + 0.1 * torch.randn(C, generator=g, device="cuda")).half()
    ob = torch.full((rows, C + 64), SENTINEL, dtype=torch.float16, device="cuda")
    out = ob[:, 16:16 + C]
    ops.rms_norm(x, wt, 1e-5, out=out)
    first = out.clone()
    ops.rms_norm(x, wt, 1e-5, out=out)
    assert torch.equal(first, out)
    assert bool((ob[:, :16] == SENTINEL).all() and (ob[:, 16 + C:] == SENTINEL).all())
    xd = x.double()
    normed = (xd * torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + 1e-5))
    # one fp16 rounding of the normalised value (either neighbour), then the fp16 product with the weight
    ref = wt.double() * normed
    tol = wt.double().abs() * normed.abs() * 2 ** -10 + ref.abs() * 2 ** -11 + 1e-7
    assert bool(((out.double() - ref).abs() <= tol).all())


def _rope_ref(x, pos, theta=10000.0):
    """rotate-half RoPE of (n, heads, 128) at positions pos, fp64"""
    inv = 1.0 / (theta ** (torch.arange(0, 128, 2, dtype=torch.float64, device=x.device) / 128))
    f = pos.double()[:, None] * inv[None]
    cos, sin = torch.cat([f.cos(), f.cos()], -1)[:, None], torch.cat([f.sin(), f.sin()], -1)[:, None]
    rot = torch.cat([-x[..., 64:], x[..., :64]], -1)
    return x * cos + rot * sin


@pytest.mark.parametrize("n,p0", [(1, 700), (630, 37)])
def test_rope_kv_append(n, p0):
    from upscale_a_video_b200 import ops
    from upscale_a_video_b200.llava import LLavaAgent
    heads, H = 40, 5120
    L = p0 + n + 5
    g = torch.Generator(device="cuda").manual_seed(n)
    qkv_b = torch.full((n, 3 * H + 64), float("nan"), dtype=torch.float16, device="cuda")
    qkv_b[:, :3 * H] = torch.randn(n, 3 * H, generator=g, device="cuda").half()
    qkv = qkv_b[:, :3 * H]
    src = qkv.clone()
    agent = LLavaAgent.__new__(LLavaAgent)
    agent.config, agent.device = type("C", (), {"rope_theta": 10000.0})(), torch.device("cuda")
    rope = agent._rope_table(L)
    cache = torch.full((2, L, H), SENTINEL, dtype=torch.float16, device="cuda")
    ops.rope_kv_append(qkv, heads, p0, rope, cache[0], cache[1])
    pos = torch.arange(p0, p0 + n, device="cuda")
    for got, want in ((qkv[:, :H], _rope_ref(src[:, :H].double().view(n, heads, 128), pos).view(n, H)),
                      (cache[0, p0:p0 + n], _rope_ref(src[:, H:2 * H].double().view(n, heads, 128), pos).view(n, H))):
        tol = want.abs() * 2 ** -11 + 1e-3 * src.double().abs().amax()
        assert bool(((got.double() - want).abs() <= tol).all())
    assert torch.equal(cache[1, p0:p0 + n], src[:, 2 * H:])
    assert bool((cache[:, :p0] == SENTINEL).all() and (cache[:, p0 + n:] == SENTINEL).all())
    assert bool(torch.isnan(qkv_b[:, 3 * H:]).all())


def test_swiglu():
    from upscale_a_video_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(2)
    for rows in (1, 630):
        gu = (torch.randn(rows, 2 * 13824, generator=g, device="cuda") * 2).half()
        out = ops.swiglu(gu)
        gd, ud = gu[:, :13824].double(), gu[:, 13824:].double()
        ref = gd * torch.sigmoid(gd) * ud
        assert bool(((out.double() - ref).abs() <= ref.abs() * 2 ** -10 + 1e-6).all())
        assert torch.equal(out, ops.swiglu(gu))


# ---------------------------------------------------------------- decode attention
@pytest.mark.parametrize("L", [1, 127, 128, 129, 700])
def test_attention_decode(L):
    from upscale_a_video_b200 import ops
    heads, H = 40, 5120
    g = torch.Generator(device="cuda").manual_seed(L)
    cache = torch.full((2, L + 64, H), float("nan"), dtype=torch.float16, device="cuda")
    cache[:, :L] = torch.randn(2, L, H, generator=g, device="cuda").half()
    q = torch.randn(H, generator=g, device="cuda").half()
    # a needle: head h's query picks key (h * 37) % L with a margin of ~30 nats in half the heads
    needle = torch.arange(heads, device="cuda") * 37 % L
    for h in range(0, heads, 2):
        cache[0, needle[h], h * 128:(h + 1) * 128] = (q[h * 128:(h + 1) * 128].float() * 0.6).half()
    buf, out = _sentinel_out(H, torch.float16)
    ops.attention_decode(q, cache[0], cache[1], L, heads, out=out)
    _check_sentinel(buf, H)
    first = out.clone()
    ops.attention_decode(q, cache[0], cache[1], L, heads, out=out)
    assert torch.equal(first, out)
    qd = q.double().view(heads, 1, 128)
    kd = cache[0, :L].double().view(L, heads, 128).transpose(0, 1)
    vd = cache[1, :L].double().view(L, heads, 128).transpose(0, 1)
    s = qd @ kd.transpose(-1, -2) * 128 ** -0.5
    ref = softmax_ref(s, vd, U32 * 128 * 128 ** -0.5 * qd.norm(dim=-1) * kd.norm(dim=-1).amax(-1, keepdim=True))
    ref = Ref(*(t.reshape(1, 1, H) for t in ref))
    assert_matches(out.view(1, 1, H), ref, L, f"decode L{L}")


# ---------------------------------------------------------------- causal prefill attention (wgmma, d = 128)
def _causal_ref(q, k, v, heads, d):
    B, n, C = q.shape
    mask = torch.ones(n, n, dtype=torch.bool, device="cuda").triu(1)
    qs = q.double().view(B, n, heads, d).transpose(1, 2)
    ks = k.double().view(B, n, heads, d).transpose(1, 2)
    vs = v.double().view(B, n, heads, d).transpose(1, 2)
    s = (qs @ ks.transpose(-1, -2) * d ** -0.5).masked_fill(mask, float("-inf"))
    ref = softmax_ref(s, vs, U32 * d * d ** -0.5 * qs.norm(dim=-1) * ks.norm(dim=-1).amax(-1, keepdim=True))
    return Ref(*(t.transpose(1, 2).reshape(B, n, C) for t in ref))


@pytest.mark.parametrize("n", [129, 630, 700])
def test_causal_prefill(n):
    from upscale_a_video_b200 import ops
    B, heads, d = 1, 8, 128
    C = heads * d
    for gen in GENERATORS:
        q, k, v = make_inputs(gen, B, heads, d, n, n, 1, device="cuda")
        W = 3 * C + 64
        buf = torch.full((n + 64, W), float("nan"), dtype=torch.float16, device="cuda")
        qs = buf[:n].view(1, n, W)[..., 8:8 + C]
        ks = buf[:n].view(1, n, W)[..., C + 16:2 * C + 16]
        vs = buf[:n].view(1, n, W)[..., 2 * C + 24:3 * C + 24]
        qs.copy_(q), ks.copy_(k), vs.copy_(v)
        ob = torch.full((n + 64, C + 64), SENTINEL, dtype=torch.float16, device="cuda")
        os_ = ob[:n].view(1, n, C + 64)[..., 8:8 + C]
        ops.attention_causal(qs, ks, vs, heads, out=os_)
        mask = torch.ones_like(ob, dtype=torch.bool)
        mask[:n].view(1, n, C + 64)[..., 8:8 + C] = False
        assert bool((ob[mask] == SENTINEL).all()), "wrote outside its output slice"
        first = os_.clone()
        ops.attention_causal(qs, ks, vs, heads, out=os_)
        assert torch.equal(first, os_)
        assert_matches(os_, _causal_ref(q, k, v, heads, d), n, f"causal {gen} n{n}")
    # needles at future keys: rows <= j0 must not change
    g = torch.Generator(device="cuda").manual_seed(n)
    qkv = torch.randn(B, n, 3 * C, generator=g, device="cuda").half()
    q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
    base = ops.attention_causal(q, k, v, heads)
    for j0 in (0, 127, 128, n // 2, n - 2):
        k2 = k.clone()
        k2[:, j0 + 1:] = q[:, j0 + 1:] * 2
        out = ops.attention_causal(q, k2, v, heads)
        assert torch.equal(out[:, :j0 + 1], base[:, :j0 + 1]), f"a future key changed row <= {j0}"
        assert_matches(out, _causal_ref(q, k2, v, heads, d), n, f"causal needle j0={j0} n{n}")


# ---------------------------------------------------------------- sampler
def _probs64(logits, temperature):
    return torch.softmax(logits.double() / temperature, -1)


def _host_pick(logits, temperature, top_p, u):
    """fp64 restatement: nucleus = tokens whose strictly more probable tokens have mass < top_p, inverse CDF in
    vocabulary order; also returns the distance of u * mass from the nearest CDF boundary"""
    p = _probs64(logits, temperature)
    order = torch.sort(p, descending=True).values
    above = torch.cumsum(order, 0) - order
    t = order[(above < top_p).nonzero().max()]
    keep = torch.where(p >= t, p, torch.zeros_like(p))
    cdf = torch.cumsum(keep, 0)
    target = u * cdf[-1]
    idx = int((cdf > target).nonzero()[0])
    return idx, (cdf - target).abs().min().item() / cdf[-1].item()


def test_sampler_argmax_ties():
    from upscale_a_video_b200 import ops
    for V, ties in ((32000, [5, 17, 31999]), (32000, [31998, 31999]), (100, [0, 1])):
        x = torch.randn(V, device="cuda")
        x[ties] = x.max() + 1
        assert int(ops.sample_top_p(x, 0.0, 0.7, 0.5)) == ties[0] == int(torch.argmax(x))
    x = torch.full((32000,), -float("inf"), device="cuda")
    x[123] = -1e30
    assert int(ops.sample_top_p(x, 0.0, 0.7, 0.0)) == 123


def test_sampler_matches_host_restatement():
    from upscale_a_video_b200 import ops
    g = torch.Generator().manual_seed(11)
    checked = 0
    for trial in range(30):
        x = torch.randn(32000, generator=g) * (1 + trial % 4)
        x[torch.randint(32000, (4,), generator=g)] += 4
        for temperature, top_p in ((0.2, 0.7), (1.0, 0.9), (0.7, 0.3)):
            for u in torch.rand(8, generator=g).tolist():
                want, dist = _host_pick(x, temperature, top_p, u)
                if dist < 1e-6:
                    continue
                got = int(ops.sample_top_p(x.cuda(), temperature, top_p, u))
                assert got == want, (trial, temperature, top_p, u)
                checked += 1
    assert checked > 500


def test_sampler_nucleus_equals_transformers():
    """for small nuclei, a fine grid of uniforms reaches every kept token: the tokens drawn are exactly the set that
    transformers' TopPLogitsWarper keeps"""
    from transformers.generation.logits_process import TemperatureLogitsWarper, TopPLogitsWarper
    from upscale_a_video_b200 import ops
    g = torch.Generator().manual_seed(12)
    for trial in range(12):
        x = torch.randn(32000, generator=g)
        hot = torch.randint(32000, (3 + trial % 5,), generator=g)
        x[hot] += torch.rand(len(hot), generator=g) * 2 + 8
        temperature, top_p = (0.2, 0.7) if trial % 2 else (1.0, 0.9)
        s = TopPLogitsWarper(top_p)(None, TemperatureLogitsWarper(temperature)(None, x[None]))[0]
        kept = set(torch.isfinite(s).nonzero().flatten().tolist())
        p = _probs64(x, temperature)
        if min(p[list(kept)]).item() < 2e-3 or len(kept) > 12:
            continue
        xc = x.cuda()
        drawn = {int(ops.sample_top_p(xc, temperature, top_p, (i + 0.5) / 2000)) for i in range(2000)}
        assert drawn == kept, (trial, sorted(drawn), sorted(kept))


# ---------------------------------------------------------------- the whole model against transformers
def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


@pytest.fixture(scope="module")
def reduced(tmp_path_factory):
    tc, vc = text_config(), vision_config()
    root = str(tmp_path_factory.mktemp("llava_reduced"))
    folder, clip, sd, vsd = write_llava_folders(root, tc, vc)
    return tc, vc, folder, clip, sd, vsd


def test_whole_model_against_transformers(reduced):
    from oracle.llava_oracle import build_llava, expand_image_ids
    from upscale_a_video_b200 import LLavaAgent
    from upscale_a_video_b200.llava import clip_preprocess, frame0_image
    tc, vc, folder, clip, sd, vsd = reduced
    agent = LLavaAgent(folder, vision_tower_path=clip)
    rng = np.random.default_rng(4)
    frame = rng.integers(0, 256, (90, 160, 3), dtype=np.uint8)
    px = clip_preprocess(frame0_image(frame), agent.image_processor)
    ids = agent.prompt_ids()
    img_tok = tc["vocab_size"] - 1
    at = ids.index(-200)

    ours_feat = agent.vision_features(px)
    x = agent.embed_prompt(ids, ours_feat)
    n = x.shape[0]
    oracle = {dt: build_llava(tc, vc, sd, vsd, img_tok, dt).cuda() for dt in (torch.float32, torch.float16)}
    input_ids = expand_image_ids(ids, img_tok, 576).cuda()
    with torch.no_grad():
        feats = {}
        for dt, m in oracle.items():
            f = m.model.get_image_features(pixel_values=px[None].cuda().to(dt), vision_feature_layer=-2,
                                           vision_feature_select_strategy="default")
            f = getattr(f, "pooler_output", f)
            feats[dt] = (torch.cat(list(f)) if isinstance(f, (list, tuple)) else f).reshape(-1, tc["hidden_size"])
        # teacher forcing: the fp32 oracle's own greedy continuation, fed to both models
        m32 = oracle[torch.float32]
        seq = input_ids
        for _ in range(17):
            nxt = m32(input_ids=seq, pixel_values=px[None].cuda().float()).logits[0, -1].argmax()
            seq = torch.cat([seq, nxt.view(1, 1)], 1)
        forced = seq[0, n:].tolist()
        logit = {dt: m(input_ids=seq[:, :-1], pixel_values=px[None].cuda().to(dt)).logits[0, n - 1:].float()
                 for dt, m in oracle.items()}
    ours_logits = torch.stack(agent.forward_logits(x, forced[:16]))
    ours_img = x[at:at + 576]
    for what, ours, r32, r16 in (("image features", ours_img, feats[torch.float32], feats[torch.float16]),
                                 ("prefill logits", ours_logits[0], logit[torch.float32][0], logit[torch.float16][0]),
                                 ("decode logits", ours_logits[1:], logit[torch.float32][1:17], logit[torch.float16][1:17])):
        e_ours, e_ref = _rel(ours, r32), _rel(r16, r32)
        print(f"{what}: ours {e_ours:.3e}, transformers fp16 {e_ref:.3e}")
        assert e_ours <= 1.5 * e_ref, (what, e_ours, e_ref)
    # greedy tokens: where the fp32 oracle's top-2 margin exceeds our deviation, the argmax agrees
    for step in range(17):
        r = logit[torch.float32][step]
        top2 = r.topk(2).values
        dev = (ours_logits[step] - r).abs().max().item()
        if (top2[0] - top2[1]).item() > 2 * dev:
            assert int(ours_logits[step].argmax()) == int(r.argmax()), step
    # a greedy caption run is reproducible and stops at EOS or 64 tokens
    a = agent.generate_ids(px, temperature=0)
    assert a == agent.generate_ids(px, temperature=0) and 1 <= len(a) <= 64
    gen = lambda: torch.Generator().manual_seed(10)
    assert agent.generate_ids(px, generator=gen()) == agent.generate_ids(px, generator=gen())


def _layer_ref(x, w, cfg, dtype):
    """one Llama decoder layer (prefill over all rows of x) in `dtype`, transformers' op order"""
    H, heads, eps = cfg["hidden"], cfg["heads"], 1e-5
    n = x.shape[0]

    def rms(t, wt):
        v = t.float().pow(2).mean(-1, keepdim=True)
        return wt.to(dtype) * (t.float() * torch.rsqrt(v + eps)).to(dtype)

    def rope(t):
        inv = 1.0 / (10000 ** (torch.arange(0, 128, 2, device=t.device).float() / 128))
        f = torch.arange(n, device=t.device).float()[:, None] * inv[None]
        cos = torch.cat([f.cos(), f.cos()], -1)[:, None].to(dtype)
        sin = torch.cat([f.sin(), f.sin()], -1)[:, None].to(dtype)
        t = t.view(n, heads, 128)
        return (t * cos + torch.cat([-t[..., 64:], t[..., :64]], -1) * sin)

    x = x.to(dtype)
    qkv = rms(x, w["ln1"]) @ w["qkv"].to(dtype).T
    q, k, v = rope(qkv[:, :H]), rope(qkv[:, H:2 * H]), qkv[:, 2 * H:].view(n, heads, 128)
    s = torch.einsum("qhd,khd->hqk", q.float(), k.float()) * 128 ** -0.5
    s = s.masked_fill(torch.ones(n, n, dtype=torch.bool, device=x.device).triu(1), float("-inf"))
    o = torch.einsum("hqk,khd->qhd", torch.softmax(s, -1).to(dtype).float(), v.float()).to(dtype).reshape(n, H)
    x = x + o @ w["o"].to(dtype).T
    gu = rms(x, w["ln2"]) @ w["gu"].to(dtype).T
    I = gu.shape[1] // 2
    a = torch.nn.functional.silu(gu[:, :I]) * gu[:, I:]
    return x + a @ w["down"].to(dtype).T


def test_one_decoder_layer_13b_shape():
    """prefill of 630 rows then one decode step through one 13B-shaped layer, against fp32 torch; our error must be no
    worse than 1.5x the error of the same torch layer in fp16"""
    from types import SimpleNamespace
    from upscale_a_video_b200.llava import LLavaAgent
    H, heads, I, n = 5120, 40, 13824, 631
    g = torch.Generator(device="cuda").manual_seed(9)
    lin = lambda a, b, s=1.0: (torch.randn(a, b, generator=g, device="cuda") * (s / b ** 0.5)).half()
    w = {"qkv": torch.cat([lin(H, H, 2.0), lin(H, H, 2.0), lin(H, H)]), "o": lin(H, H), "gu": lin(2 * I, H),
         "down": lin(H, I), "ln1": (1 + 0.1 * torch.randn(H, generator=g, device="cuda")).half(),
         "ln2": (1 + 0.1 * torch.randn(H, generator=g, device="cuda")).half()}
    x = torch.randn(n, H, generator=g, device="cuda").half()
    agent = LLavaAgent.__new__(LLavaAgent)
    agent.config = SimpleNamespace(hidden_size=H, num_attention_heads=heads, rms_norm_eps=1e-5, rope_theta=10000.0)
    agent.device = torch.device("cuda")
    agent.w = {"qkv0": w["qkv"], "o0": w["o"], "gu0": w["gu"], "down0": w["down"], "ln1_0": w["ln1"], "ln2_0": w["ln2"]}
    rope = agent._rope_table(n)
    cache = torch.empty(2, n, H, dtype=torch.float16, device="cuda")
    with torch.no_grad():
        pre = agent._layer_prefill(0, x[:n - 1].clone(), cache[0], cache[1], rope)
        dec = agent._layer_decode(0, x[n - 1:].clone(), n - 1, cache[0], cache[1], rope)
        cfg = dict(hidden=H, heads=heads)
        r32 = _layer_ref(x, w, cfg, torch.float32)
        r16 = _layer_ref(x, w, cfg, torch.float16)
    for what, ours, a, b in (("prefill", pre, r32[:n - 1], r16[:n - 1]), ("decode", dec, r32[n - 1:], r16[n - 1:])):
        # the residual stream carries x itself: compare the layer's update
        base = x[:n - 1] if what == "prefill" else x[n - 1:]
        e_ours, e_ref = _rel(ours.float() - base.float(), a - base.float()), _rel(b.float() - base.float(), a - base.float())
        print(f"13B layer {what}: ours {e_ours:.3e}, torch fp16 {e_ref:.3e}")
        assert e_ours <= 1.5 * e_ref, (what, e_ours, e_ref)


# ---------------------------------------------------------------- the command
from test_cli_gpu import _bgr, model_dir  # noqa: E402,F401  (the synthetic Upscale-A-Video folder)


@pytest.fixture(scope="module")
def cli_llava(tmp_path_factory):
    """a tiny LLaVA in the released format whose vocabulary is the golden sentencepiece tokenizer's, so that every
    generated id decodes"""
    tc = text_config(hidden=256, heads=2, layers=2, inter=512, vocab=400)
    vc = vision_config(hidden=128, heads=2, layers=2, inter=256)  # head_dim 64, as the attention kernels take
    folder, clip, _, _ = write_llava_folders(str(tmp_path_factory.mktemp("cli_llava")), tc, vc)
    return folder, clip


def _run_cli(tmp_path, model_dir, tag, extra, capsys):
    import cv2
    from upscale_a_video_b200 import cli, video_io
    clip = tmp_path / "clip"
    if not clip.exists():
        video_io.write_frames(str(clip), _bgr(3, 64, 64, 5))
    out = tmp_path / tag
    capsys.readouterr()
    cli.main(["-i", str(clip), "-o", str(out), "--model_dir", str(model_dir), "-s", "2", "--save_image", *extra])
    printed = capsys.readouterr().out
    d = out / "frame" / "clip_n120_g6_s2"
    pngs = np.stack([cv2.imread(str(d / p)) for p in sorted(os.listdir(d))])
    return printed, pngs


def test_cli_caption_end_to_end(tmp_path, model_dir, cli_llava, capsys):
    folder, clip = cli_llava
    flags = ["--llava_path", folder, "--llava_vision_path", clip]
    printed, pngs = _run_cli(tmp_path, model_dir, "a", flags, capsys)
    # the caption the command computes for frame 0, printed as the reference prints it
    from upscale_a_video_b200 import LLavaAgent, cli, video_io
    bgr, _, _ = video_io.read_frames(str(tmp_path / "clip"))
    caption = cli.caption_frame(LLavaAgent(folder, vision_tower_path=clip), bgr[0])
    assert caption
    wrapped = textwrap.indent(textwrap.fill("Caption: " + caption, width=80), " " * 8)
    assert wrapped in printed and printed.count("Caption: ") == 1
    printed2, pngs2 = _run_cli(tmp_path, model_dir, "b", flags, capsys)
    assert wrapped in printed2 and printed2.count("Caption: ") == 1  # a rerun prints the same caption
    assert np.array_equal(pngs, pngs2)
    # the prompt is caption + a_prompt: the PNGs equal those of a run given that caption
    _, pngs3 = _run_cli(tmp_path, model_dir, "c", ["--caption", caption], capsys)
    assert np.array_equal(pngs, pngs3)
    # --no_llava turns the captioner off
    printed4, pngs4 = _run_cli(tmp_path, model_dir, "d", flags + ["--no_llava"], capsys)
    assert "Caption:" not in printed4


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_cli_caption_torchrun(tmp_path, model_dir, cli_llava):
    """only rank 0 loads the captioner; both ranks use its caption (the PNGs equal the single-process run's)"""
    import cv2
    from upscale_a_video_b200 import cli, video_io
    folder, clip_dir = cli_llava
    clip = tmp_path / "clip"
    video_io.write_frames(str(clip), _bgr(3, 64, 64, 5))
    args = ["-i", str(clip), "--model_dir", str(model_dir), "-s", "2", "--save_image", "--llava_path", folder,
            "--llava_vision_path", clip_dir]
    cli.main(args + ["-o", str(tmp_path / "one")])
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nproc-per-node", "2", "--master-port", "29533",
                        "-m", "upscale_a_video_b200", *args, "-o", str(tmp_path / "two")],
                       cwd=ROOT, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.count("Loading LLaVA") == 1 and r.stdout.count("Caption: ") == 1
    d1, d2 = tmp_path / "one" / "frame" / "clip_n120_g6_s2", tmp_path / "two" / "frame" / "clip_n120_g6_s2"
    for p in sorted(os.listdir(d1)):
        assert np.array_equal(cv2.imread(str(d1 / p)), cv2.imread(str(d2 / p))), p
