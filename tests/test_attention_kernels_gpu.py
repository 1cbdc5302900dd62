"""Every attention kernel against an fp64 reference (tests/attention_cases.py) with inputs that expose dropped, stale and
unmasked key tiles: the dispatch boundaries of uav_attention with the kernel each case runs pinned by torch.profiler, the
pipeline's own shapes, what the kernels read and write around their operands, repeat launches, the temporal kernels
with a needle planted through the relative-position bias, and the causal kernel with needles at future keys."""
import json
import os
import subprocess
import sys

import pytest
import torch

from attention_cases import (GENERATORS, U16, U32, Ref, assert_matches, attention_ref, check_rows, make_inputs,
                             softmax_ref)

pytestmark = pytest.mark.gpu
SENTINEL = 1234.0  # exact in fp16
PAD = 64           # NaN columns beside each operand slice, and NaN rows after the last token


@pytest.fixture(autouse=True, scope="module")
def _release_memory(uav_lib):
    """build and load the library first; afterwards hand the pipeline-shape buffers (GBs) back to the driver, so that
    later tests' memory measurements start clean"""
    yield
    import gc
    gc.collect()
    torch.cuda.empty_cache()


def _in_subprocess(fn_name):
    """fn_name() of this module, run in a fresh interpreter.  The kernel traces are taken there: once the profiler has
    been used in a process, kernels whose modules load later in that process can be missing from its later traces,
    which would take the kernel-selection checks of the other test files with them."""
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.dirname(here), here, os.environ.get("PYTHONPATH", "")]))
    r = subprocess.run([sys.executable, "-c", f"import json, {__name__} as t; print(json.dumps(t.{fn_name}()))"],
                       cwd=os.path.dirname(here), env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def _kernels_run(calls, candidates):
    """{tag: the `candidates` kernel names that call() launched}, from one torch.profiler session.  Every call launches
    exactly one candidate kernel on the current stream, so the candidates of the trace in time order are the calls in
    order.  The kernels are loaded before the session: a launch that loads its module inside the window can be missing
    from the trace."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    for fn in calls.values():
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for fn in calls.values():
            fn()
        torch.cuda.synchronize()
    launched = sorted((e.time_range.start, e.name.replace(" ", "")) for e in prof.events()
                      if e.device_type == DeviceType.CUDA and any(c in e.name.replace(" ", "") for c in candidates))
    assert len(launched) == len(calls), (len(launched), len(calls), "the trace lost kernel records")
    return {tag: sorted(c for c in candidates if c in name) for tag, (_, name) in zip(calls, launched)}


def _embed(x, col0, width, fill):
    """x (b, n, C) as the column slice [col0, col0 + C) of one (b * n + PAD, width) buffer filled with `fill`: an
    access past the slice or past the last token reads (or writes) memory of this buffer"""
    b, n, C = x.shape
    buf = torch.full((b * n + PAD, width), fill, dtype=torch.float16, device="cuda")
    view = buf[:b * n].view(b, n, width)[..., col0:col0 + C]
    view.copy_(x)
    return buf, view


def run_attention(q, k, v, heads, kvd, scale=None):
    """ops.attention on q, k, v held as slices of NaN-filled buffers with token stride 3 C + PAD, into a slice of a
    sentinel-filled output buffer; checks the sentinel and that the output is finite, returns the output"""
    from upscale_a_video_b200 import ops
    B, nq, C = q.shape
    W = 3 * C + PAD
    nan = float("nan")
    _, qs = _embed(q, C + 8, W, nan)
    _, ks = _embed(k, 8, W, nan)
    _, vs = _embed(v, 2 * C + 16, W, nan)
    obuf = torch.full((B * nq + PAD, C + PAD), SENTINEL, dtype=torch.float16, device="cuda")
    os_ = obuf[:B * nq].view(B, nq, C + PAD)[..., 8:8 + C]
    ops.attention(qs, ks, vs, heads, kv_batch_div=kvd, scale=scale, out=os_)
    mask = torch.ones_like(obuf, dtype=torch.bool)
    mask[:B * nq].view(B, nq, C + PAD)[..., 8:8 + C] = False
    assert bool((obuf[mask] == SENTINEL).all()), "attention wrote outside its output slice"
    out = os_.clone()
    assert bool(torch.isfinite(out).all()), "non-finite output: a NaN outside the operands was read"
    return out


# ---------------------------------------------------------------- dispatch boundaries
# (B, heads, d, nq, nk, kv_batch_div, kernel).  uav_attention runs the cross kernel (80- or 128-key resident tile) for
# nk <= 128, nq >= 4 nk and d != 512, and the wgmma kernel for every other case (128 query rows per CTA; 128-key tiles
# for d = 64 and 128, 64-key tiles for d = 512).
CROSS64_5, CROSS64_8 = "cross_attn_kernel<64,5>", "cross_attn_kernel<64,8>"
CROSS128_5, CROSS128_8 = "cross_attn_kernel<128,5>", "cross_attn_kernel<128,8>"
TC64, TC128, TC512 = "fa_tc_kernel<64,64,128>", "fa_tc_kernel<128,128,128>", "fa_tc_kernel<512,256,64>"
DISPATCH = [
    (2, 8, 64, 4, 1, 1, CROSS64_5), (2, 8, 64, 3, 1, 1, TC64),
    (4, 8, 64, 64, 16, 2, CROSS64_5), (4, 8, 64, 63, 16, 2, TC64),
    (8, 8, 64, 308, 77, 8, CROSS64_5), (8, 8, 64, 307, 77, 8, TC64),
    (2, 8, 64, 320, 80, 1, CROSS64_5), (2, 8, 64, 324, 81, 1, CROSS64_8), (2, 8, 64, 323, 81, 1, TC64),
    (2, 8, 64, 508, 127, 2, CROSS64_8), (2, 8, 64, 512, 128, 1, CROSS64_8), (2, 8, 64, 511, 128, 1, TC64),
    (2, 8, 64, 516, 129, 1, TC64), (2, 4, 64, 129, 191, 1, TC64), (2, 4, 64, 127, 192, 1, TC64),
    (2, 4, 64, 193, 193, 1, TC64), (8, 2, 64, 65, 257, 8, TC64),
    (8, 8, 128, 308, 77, 8, CROSS128_5), (2, 8, 128, 324, 81, 1, CROSS128_8), (2, 8, 128, 512, 128, 2, CROSS128_8),
    (2, 8, 128, 511, 128, 2, TC128), (2, 8, 128, 516, 129, 1, TC128), (2, 8, 128, 307, 77, 1, TC128),
    (2, 4, 128, 256, 255, 1, TC128), (2, 4, 128, 129, 256, 1, TC128), (8, 2, 128, 127, 257, 8, TC128),
    (2, 1, 512, 4, 1, 1, TC512), (2, 1, 512, 64, 16, 2, TC512), (2, 1, 512, 129, 63, 1, TC512),
    (2, 1, 512, 256, 64, 1, TC512), (2, 1, 512, 127, 65, 1, TC512), (2, 1, 512, 385, 129, 2, TC512),
    (1, 1, 512, 300, 191, 1, TC512),
]
ATTENTION_KERNELS = {CROSS64_5, CROSS64_8, CROSS128_5, CROSS128_8, TC64, TC128, TC512}


def _id(c):
    return f"B{c[0]}h{c[1]}d{c[2]}nq{c[3]}nk{c[4]}kv{c[5]}"


def dispatch_kernels():
    """{case id: attention kernels it launched}"""
    from upscale_a_video_b200 import ops
    calls = {}
    for B, H, d, nq, nk, kvd, _ in DISPATCH:
        q, k, v = make_inputs("random", B, H, d, nq, nk, kvd, device="cuda")
        calls[_id((B, H, d, nq, nk, kvd))] = lambda q=q, k=k, v=v, H=H, kvd=kvd: ops.attention(q, k, v, H, kv_batch_div=kvd)
    return _kernels_run(calls, ATTENTION_KERNELS)


@pytest.fixture(scope="module")
def dispatched(uav_lib):
    return _in_subprocess("dispatch_kernels")


@pytest.mark.parametrize("case", DISPATCH, ids=lambda c: f"{_id(c)}-{c[6]}")  # the id names the kernel it pins
def test_dispatch_boundaries(case, dispatched):
    """each case runs the kernel of its row (and no other attention kernel), passes the criterion on every generator,
    keeps its operands' NaN surroundings out and its output sentinel intact, and repeats bit for bit"""
    B, H, d, nq, nk, kvd, kernel = case
    assert dispatched[_id(case)] == [kernel], (kernel, dispatched[_id(case)])
    for gen in GENERATORS:
        q, k, v = make_inputs(gen, B, H, d, nq, nk, kvd, seed=nq * 131 + nk, device="cuda")
        out = run_attention(q, k, v, H, kvd)
        assert torch.equal(out, run_attention(q, k, v, H, kvd)), f"{_id(case)} {gen}: repeat launch differs"
        assert_matches(out, attention_ref(q, k, v, H, kvd, d ** -0.5), nk, f"{_id(case)} {gen}")


def test_scale_other_than_default():
    """an explicit positive scale reaches every kernel path the same way as the default one"""
    for B, H, d, nq, nk, kvd in ((2, 8, 64, 308, 77, 1), (2, 8, 64, 300, 300, 1), (2, 8, 128, 300, 300, 1),
                                 (1, 1, 512, 200, 130, 1)):
        q, k, v = make_inputs("random", B, H, d, nq, nk, kvd, seed=3, device="cuda")
        assert_matches(run_attention(q, k, v, H, kvd, scale=0.31), attention_ref(q, k, v, H, kvd, 0.31), nk,
                       f"d{d} nk{nk} scale 0.31")


# ---------------------------------------------------------------- the pipeline's shapes
# (batch, heads, d, nq, nk, kv_batch_div) of every ops.attention call of one UNet forward (2 CFG halves x 8 frames) and
# of the first decode chunk (3 frames) of an 8-frame vae_3d decode, captured by recording the arguments of ops.attention
# during an ops.Profile of each at h720 (180x320 latents) and config 2 (320x576 latents).  The 384x384 tile of config 5
# follows the same pattern at 384x384 latents.
PIPELINE_SHAPES = [
    # UNet, h720: text cross-attention at h/2, h/4, h/8 and self-attention at h/8 (23x40 = 920 tokens)
    (16, 8, 64, 14400, 77, 8), (16, 8, 64, 3600, 77, 8), (16, 8, 128, 920, 77, 8), (16, 8, 128, 920, 920, 1),
    # UNet, config 2 (40x72 = 2880 tokens at h/8)
    (16, 8, 64, 46080, 77, 8), (16, 8, 64, 11520, 77, 8), (16, 8, 128, 2880, 77, 8), (16, 8, 128, 2880, 2880, 1),
    # UNet, config 5 tile (48x48 = 2304 tokens at h/8, no ragged key tile)
    (16, 8, 64, 36864, 77, 8), (16, 8, 64, 9216, 77, 8), (16, 8, 128, 2304, 77, 8), (16, 8, 128, 2304, 2304, 1),
    # VAE mid-block attention: one head, d = 512, every latent pixel of a frame
    (3, 1, 512, 57600, 57600, 1), (3, 1, 512, 184320, 184320, 1), (3, 1, 512, 147456, 147456, 1),
]


@pytest.mark.parametrize("shape", PIPELINE_SHAPES, ids=lambda s: "B{}h{}d{}nq{}nk{}kv{}".format(*s))
@pytest.mark.parametrize("gen", ["needle", "ramp_up", "random"])
def test_pipeline_shapes(shape, gen):
    """the kernel runs on every query row; the first and last query tile, the rows whose needle sits on a tile edge
    and 1024 random rows of every batch item are compared with the full-key fp64 reference"""
    from upscale_a_video_b200 import ops
    B, H, d, nq, nk, kvd = shape
    q, k, v = make_inputs(gen, B, H, d, nq, nk, kvd, seed=nq + nk, device="cuda")
    out = ops.attention(q, k, v, H, kv_batch_div=kvd)
    rows = check_rows(nq, nk).cuda()
    assert_matches(out[:, rows], attention_ref(q, k, v, H, kvd, d ** -0.5, rows=rows), nk,
                   f"B{B} h{H} d{d} nq{nq} nk{nk} {gen}")


# ---------------------------------------------------------------- temporal kernels
def _temporal_needle_inputs(B, Fr, HW, heads, d, seed):
    """q, k, v ~ N(0, 0.5^2) as slices of one qkv buffer; bias = N(0, 0.5^2) + 20 at bias[h, i, pi_h(i)] with pi_h a
    head-dependent, non-symmetric map of query frame i to a key frame, so the output of (h, i) is ~ v of frame pi_h(i)"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    C = heads * d
    qkv = (torch.randn(B, Fr, HW, 3 * C, generator=g, device="cuda") * 0.5).half()
    bias = torch.randn(heads, Fr, Fr, generator=g, device="cuda") * 0.5
    i = torch.arange(Fr, device="cuda")
    for h in range(heads):
        bias[h, i, (i * (2 * h + 1) + h + 1) % Fr] += 20.0
    freqs = 1.0 / (10000 ** (torch.arange(0, 32, 2).double() / 32))
    ang = torch.arange(Fr).double()[:, None] * freqs[None, :]
    rot = torch.stack([ang.cos(), ang.sin()], dim=-1).float().contiguous().cuda()
    return qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:], rot, bias.contiguous()


def _temporal_ref(q, k, v, heads, rot, bias) -> Ref:
    """fp64: rotary on the interleaved pairs of dims [0, 32) of q and k, scores q k^T / sqrt(d) + bias[h, i, j]"""
    B, Fr, HW, C = q.shape
    d = C // heads

    def seq(t):  # (B, F, HW, C) -> (B, HW, heads, F, d)
        return t.double().view(B, Fr, HW, heads, d).permute(0, 2, 3, 1, 4)

    def rope(t):
        c, s = rot.double()[..., 0], rot.double()[..., 1]  # (F, 16)
        x0, x1 = t[..., 0:32:2], t[..., 1:32:2]
        r = t.clone()
        r[..., 0:32:2], r[..., 1:32:2] = x0 * c - x1 * s, x1 * c + x0 * s
        return r

    qs, ks, vs = rope(seq(q)), rope(seq(k)), seq(v)
    sc = (qs @ ks.transpose(-1, -2)) * d ** -0.5 + bias.double()
    eps = U32 * d * d ** -0.5 * qs.norm(dim=-1) * ks.norm(dim=-1).amax(-1, keepdim=True)
    ref = softmax_ref(sc, vs, eps)
    return Ref(*(t.permute(0, 3, 1, 2, 4).reshape(B, Fr, HW, C) for t in ref))


TEMPORAL_CASES = [
    (2, 8, 40, 8, 64, "temporal_attn_mma_kernel"), (1, 5, 33, 8, 128, "temporal_attn_mma_kernel"),
    (2, 2, 17, 2, 64, "temporal_attn_mma_kernel"), (2, 8, 20, 3, 64, "temporal_attn_long_kernel"),
    (1, 9, 24, 8, 64, "temporal_attn_long_kernel"), (1, 17, 12, 8, 128, "temporal_attn_long_kernel"),
    (1, 40, 10, 2, 64, "temporal_attn_long_kernel"), (2, 1, 9, 8, 64, "temporal_attn_mma_kernel"),
    # the pipeline's calls, captured with the attention shapes above: (B, F, HW, heads, d) = (2, 8, h w / 4 | h w / 16 |
    # h w / 64, 8, 64 | 64 | 128) at h720 and config 2
    (2, 8, 14400, 8, 64, "temporal_attn_mma_kernel"), (2, 8, 3600, 8, 64, "temporal_attn_mma_kernel"),
    (2, 8, 920, 8, 128, "temporal_attn_mma_kernel"), (2, 8, 46080, 8, 64, "temporal_attn_mma_kernel"),
    (2, 8, 2880, 8, 128, "temporal_attn_mma_kernel")]


def temporal_kernels():
    """{case: temporal kernels it launched}"""
    from upscale_a_video_b200 import ops
    calls = {}
    for B, Fr, HW, heads, d, _ in TEMPORAL_CASES:
        q, k, v, rot, bias = _temporal_needle_inputs(B, Fr, HW, heads, d, seed=0)
        calls[f"temporal {B} {Fr} {HW} {heads} {d}"] = (
            lambda q=q, k=k, v=v, heads=heads, rot=rot, bias=bias: ops.temporal_attention(q, k, v, heads, rot, bias))
    return _kernels_run(calls, {"temporal_attn_mma_kernel", "temporal_attn_long_kernel"})


@pytest.fixture(scope="module")
def temporal_dispatched(uav_lib):
    return _in_subprocess("temporal_kernels")


@pytest.mark.parametrize("B,Fr,HW,heads,d,kernel", TEMPORAL_CASES)
def test_temporal_bias_needle(B, Fr, HW, heads, d, kernel, temporal_dispatched):
    """the needle planted through the relative-position bias pins its orientation (query frame, key frame) and head"""
    from upscale_a_video_b200 import ops
    ran = temporal_dispatched[f"temporal {B} {Fr} {HW} {heads} {d}"]
    assert ran == [kernel], (kernel, ran)
    q, k, v, rot, bias = _temporal_needle_inputs(B, Fr, HW, heads, d, seed=Fr * 7 + heads)
    out = ops.temporal_attention(q, k, v, heads, rot, bias)
    assert torch.equal(out, ops.temporal_attention(q, k, v, heads, rot, bias))
    # the pairs kernel rounds the rotated q and k to fp16 before the scores: 2 U16 |q_32| |k_32| / sqrt(d) more
    r32 = lambda t: t.float()[..., :32].reshape(-1, 32).norm(dim=-1).max().item()  # noqa: E731
    rotary_err = 2 * U16 * d ** -0.5 * r32(q) * r32(k)
    assert_matches(out, _temporal_ref(q, k, v, heads, rot, bias), Fr, f"temporal F{Fr} h{heads} d{d}",
                   score_err=rotary_err)


# ---------------------------------------------------------------- causal kernel (CLIP text encoder)
@pytest.mark.parametrize("n", [1, 2, 33, 77, 128])
def test_causal_future_needle(n):
    """key j > j0 is replaced by 2 q_j, a needle that query j picks (score ~16 nats): rows <= j0, for which those keys
    are in the future, must not change at all, and rows > j0 must follow their needle on the diagonal, both against the
    fp64 causal reference"""
    from upscale_a_video_b200 import ops
    B, heads, d = 2, 4, 64
    C = heads * d
    g = torch.Generator(device="cuda").manual_seed(n)
    qkv = torch.randn(B, n, 3 * C, generator=g, device="cuda").half()
    q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
    base = ops.attention_causal(q, k, v, heads)
    j0 = n // 2
    k2 = k.clone()
    k2[:, j0 + 1:] = q[:, j0 + 1:] * 2
    out = ops.attention_causal(q, k2, v, heads)
    assert torch.equal(out[:, :j0 + 1], base[:, :j0 + 1]), "a future key changed the output"
    mask = torch.ones(n, n, dtype=torch.bool, device="cuda").triu(1)
    for kk, got in ((k, base), (k2, out)):
        qs = q.double().view(B, n, heads, d).transpose(1, 2)
        ks = kk.double().view(B, n, heads, d).transpose(1, 2)
        vs = v.double().view(B, n, heads, d).transpose(1, 2)
        s = (qs @ ks.transpose(-1, -2) * d ** -0.5).masked_fill(mask, float("-inf"))
        ref = softmax_ref(s, vs, U32 * d * d ** -0.5 * qs.norm(dim=-1) * ks.norm(dim=-1).amax(-1, keepdim=True))
        ref = Ref(*(t.transpose(1, 2).reshape(B, n, C) for t in ref))
        assert_matches(got, ref, n, f"causal n{n}")
