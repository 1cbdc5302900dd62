"""GPU checks of the inputs beyond the pipeline's own shapes: temporal attention on more than 8 frames (the online-softmax
kernel), UNetVideoModel.forward on 12 and 40 frames against the reference's fixtures and on 64 frames against the oracle, and the area resize of the flows in
Propagation, bit-exact against torch on the same GPU."""
import json
import os
import zlib

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
PROP_MODES = (("nearest", "fuse", 0.001, 0.05), ("bilinear", "copy", 0.01, 0.5))


@pytest.fixture(autouse=True)
def _setup(uav_lib):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.manual_seed(0)


def _rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm()).item()


def _load(name):
    return torch.load(os.path.join(G, name), weights_only=False)


def _unet_long_case(name):
    """a case of unet_long.pt with its inputs redrawn: sample, low_res and the text embeddings are drawn in that order from a
    generator seeded with crc32(name) (oracle/make_golden_long.py); the stored sums catch a change of torch's generator"""
    c = dict(_load("unet_long.pt")[name])
    B, T, H, W = c["shape"]
    g = torch.Generator().manual_seed(zlib.crc32(name.encode()))
    c["sample"] = torch.randn(B, 4, T, H, W, generator=g)
    c["low_res"] = torch.randn(B, 3, T, H, W, generator=g)
    c["ctx"] = torch.randn(B, 77, 1024, generator=g) * 0.3
    for k, want in zip(("sample", "low_res", "ctx"), c["input_sums"]):
        assert abs(float(c[k].double().sum()) - want) < 1e-6 * (1 + abs(want)), f"{name}: redrawn {k} differs from the fixture's"
    return c


# ---------------------------------------------------------------- temporal attention, F > 8
def _temporal_inputs(B, Fr, HW, heads, d, q_gain=1.0):
    from oracle import uav_oracle as O
    C = heads * d
    qkv = torch.randn(B, Fr, HW, 3 * C, device="cuda").half()
    if q_gain != 1.0:
        qkv[..., :C] = (qkv[..., :C].float() * q_gain).half()
    q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
    freqs = 1.0 / (10000 ** (torch.arange(0, 32, 2).float() / 32))
    table = torch.randn(32, heads) * 0.5
    bias = O.rel_pos_bias({"b.relative_attention_bias.weight": table}, "b", Fr).contiguous().cuda()
    ang = torch.arange(Fr).float()[:, None] * freqs[None, :]
    rot = torch.stack([ang.cos(), ang.sin()], dim=-1).contiguous().cuda()
    return q, k, v, freqs, rot, bias


def _temporal_ref(q, k, v, heads, freqs, bias):
    """fp32 restatement of TemporalAttention._attention (attention.py:699-733), as in test_ops_gpu.test_temporal_attention"""
    from oracle import uav_oracle as O
    B, Fr, HW, C = q.shape
    d = C // heads

    def to_seq(t):  # (B,F,HW,C) -> ((B HW), heads, F, d)
        return t.float().permute(0, 2, 1, 3).reshape(B * HW, Fr, heads, d).permute(0, 2, 1, 3)

    qs, ks, vs = to_seq(q) * d ** -0.5, to_seq(k), to_seq(v)
    qs, ks = O.rotary(freqs.cuda(), qs), O.rotary(freqs.cuda(), ks)
    sc = torch.einsum("bhid,bhjd->bhij", qs, ks) + bias
    pr = (sc - sc.amax(-1, keepdim=True)).softmax(-1)
    return torch.einsum("bhij,bhjd->bhid", pr, vs).permute(0, 2, 1, 3).reshape(B, HW, Fr, C).permute(0, 2, 1, 3)


def _assert_close(got, ref, tol, what):
    err = (got.float() - ref.float()).abs()
    bad = (err > tol + tol * ref.float().abs()).sum().item()
    assert bad == 0, f"{what}: {bad}/{err.numel()} mismatches, max err {err.max().item():.4g}"


@pytest.mark.parametrize("B,Fr,HW,heads,d", [(2, 9, 96, 8, 64), (1, 12, 50, 8, 128), (2, 16, 33, 8, 64), (1, 17, 7, 8, 128),
                                             (2, 33, 19, 2, 128), (1, 40, 10, 3, 64), (1, 64, 2881, 8, 64)])
def test_temporal_attention_long(B, Fr, HW, heads, d):
    """q/k/v are strided slices of one qkv tensor; odd head counts and ragged last tiles included"""
    from upscale_a_video_b200 import ops
    q, k, v, freqs, rot, bias = _temporal_inputs(B, Fr, HW, heads, d)
    out = ops.temporal_attention(q, k, v, heads, rot, bias)
    _assert_close(out, _temporal_ref(q, k, v, heads, freqs, bias), 3e-3, f"temporal attention F={Fr}")


def test_temporal_attention_long_peaky_scores():
    """q x 6: the row maximum moves between key tiles, so O and the row sum are rescaled (online softmax)"""
    from upscale_a_video_b200 import ops
    B, Fr, HW, heads, d = 2, 40, 24, 8, 64
    q, k, v, freqs, rot, bias = _temporal_inputs(B, Fr, HW, heads, d, q_gain=6.0)
    out = ops.temporal_attention(q, k, v, heads, rot, bias)
    _assert_close(out, _temporal_ref(q, k, v, heads, freqs, bias), 3e-3, "temporal attention F=40 (peaky)")


def _kernels_run(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {e.key for e in prof.key_averages()}


def test_temporal_attention_kernel_selection():
    """F > 8 or an odd head count runs the online-softmax kernel; F <= 8 with an even head count keeps the mma kernel of
    the pipeline's windows"""
    from upscale_a_video_b200 import ops
    for Fr, heads, want, other in ((12, 8, "temporal_attn_long_kernel", "temporal_attn_mma_kernel"),
                                   (8, 8, "temporal_attn_mma_kernel", "temporal_attn_long_kernel"),
                                   (4, 3, "temporal_attn_long_kernel", "temporal_attn_mma_kernel")):
        q, k, v, _, rot, bias = _temporal_inputs(1, Fr, 40, heads, 64)
        names = _kernels_run(lambda: ops.temporal_attention(q, k, v, heads, rot, bias))
        assert any(want in n for n in names) and not any(other in n for n in names), (Fr, names)


# ---------------------------------------------------------------- UNet on long clips
@pytest.fixture(scope="module")
def unet(uav_lib):
    from oracle.weights import make_state_dict
    from upscale_a_video_b200.unet_video import UNetVideoModel
    meta = json.load(open(os.path.join(G, "meta.json")))
    cfg = json.load(open(os.path.join(os.path.dirname(__file__), "..", "upscale_a_video_b200", "configs",
                                      "unet_video_config.json")))
    sd = make_state_dict(json.load(open(os.path.join(G, "shapes_unet.json"))), meta["seed_unet"])
    m = UNetVideoModel.from_config(cfg)
    m.load_state_dict(sd, strict=True)
    return m.half().eval().cuda(), sd, cfg


@pytest.mark.parametrize("case", ["t12_16x24", "t40_8x8"])
def test_unet_long_clip_vs_golden(unet, case):
    """the acceptance band of test_unet_gpu.py: no worse than 1.5x the reference's own fp16 drift (or 5e-3)"""
    from oracle import uav_oracle as O
    m, sd, cfg = unet
    c = _unet_long_case(case)
    sample, low, ctx = c["sample"].cuda().half(), c["low_res"].cuda().half(), c["ctx"].cuda().half()
    out = m(sample, torch.tensor(c["timestep"]), low, encoder_hidden_states=ctx, class_labels=c["class_labels"].cuda()).sample
    assert out.shape == c["out"].shape and out.dtype == torch.float16
    torch.cuda.synchronize()
    err = _rel(out.cpu(), c["out"])
    sd16 = {k: v.cuda().half() for k, v in sd.items()}
    ref16 = O.unet_forward(sd16, cfg, sample, torch.tensor(c["timestep"]), low, ctx, c["class_labels"])
    err_ref = _rel(ref16.cpu(), c["out"])
    print(f"\n[unet {case}] rel L2 err vs fp32 golden: uav_b200 {err:.3e} | reference-fp16 (torch) {err_ref:.3e}")
    assert err <= max(1.5 * err_ref, 5e-3), (err, err_ref)
    out2 = m(sample, torch.tensor(c["timestep"]), low, encoder_hidden_states=ctx, class_labels=c["class_labels"].cuda()).sample
    assert torch.equal(out, out2)


def test_unet_long_clip_shared_cfg_prefix(unet):
    m, _, _ = unet
    c = _unet_long_case("t12_16x24")
    sample = c["sample"][:1].repeat(2, 1, 1, 1, 1).cuda().half()
    low = c["low_res"][:1].repeat(2, 1, 1, 1, 1).cuda().half()
    ctx = c["ctx"].cuda().half()
    a = m(sample, 601, low, encoder_hidden_states=ctx, class_labels=torch.tensor([120])).sample
    b = m(sample, 601, low, encoder_hidden_states=ctx, class_labels=torch.tensor([120]), cfg_shared_input=True).sample
    err = _rel(b, a)
    print(f"\n[unet t12 shared-prefix] rel L2 diff vs unshared {err:.3e}")
    assert err < 5e-3 and not torch.equal(a[0], a[1])


def test_unet_64_frames_small_spatial_vs_oracle(unet):
    """64 frames at 8x8: everything sized by b*t (GroupNorm statistics blocks, the concat slots, the shared CFG prefix, the
    fused tail) against the fp32 oracle run on the same GPU"""
    from oracle import uav_oracle as O
    m, sd, cfg = unet
    g = torch.Generator().manual_seed(64)
    sample, low = torch.randn(1, 4, 64, 8, 8, generator=g).repeat(2, 1, 1, 1, 1), torch.randn(1, 3, 64, 8, 8, generator=g)
    low = low.repeat(2, 1, 1, 1, 1)
    ctx = torch.randn(2, 77, 1024, generator=g) * 0.3
    sdc = {k: v.cuda() for k, v in sd.items()}
    ref = O.unet_forward(sdc, cfg, sample.cuda(), torch.tensor(400), low.cuda(), ctx.cuda(), torch.tensor([100])).cpu()
    s16, l16, c16 = sample.cuda().half(), low.cuda().half(), ctx.cuda().half()
    out = m(s16, 400, l16, encoder_hidden_states=c16, class_labels=torch.tensor([100])).sample
    shared = m(s16, 400, l16, encoder_hidden_states=c16, class_labels=torch.tensor([100]), cfg_shared_input=True).sample
    err, err_shared = _rel(out.cpu(), ref), _rel(shared.cpu(), ref)
    print(f"\n[unet t64_8x8] rel L2 err vs fp32 oracle {err:.3e}, shared prefix {err_shared:.3e}")
    assert out.shape == (2, 4, 64, 8, 8) and err < 5e-3 and err_shared < 5e-3


# ---------------------------------------------------------------- flow resize (bit exact vs torch on the GPU)
@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_flow_resize_area_matches_torch(dtype):
    from upscale_a_video_b200 import ops
    p = _load("propagation_resize.pt")
    t, h, w = p["x"].shape[2:]
    for name in ("up2x", "down2x", "ratio1_5", "t7"):
        for key in ("flows_forward", "flows_backward"):
            f = p[name][key].cuda().to(dtype)
            s = 1.0 * w / f.shape[-1]
            got = ops.flow_resize_area(f, (t - 1, h, w), s)
            ref = F.interpolate(f, (t - 1, h, w), mode="area") * s
            assert got.dtype == dtype and torch.equal(got, ref), (name, key, (got.float() - ref.float()).abs().max().item())
    # shapes beyond the fixtures: upsampling in every dimension, one output frame, several batch items
    g = torch.randn(3, 2, 5, 7, 11, device="cuda").to(dtype) * 4
    for size in ((9, 13, 29), (1, 2, 3), (5, 3, 4)):
        assert torch.equal(ops.flow_resize_area(g, size, 0.37), F.interpolate(g, size, mode="area") * 0.37), size


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("interp,mode,a1,a2", PROP_MODES)
def test_propagation_resized_flows_vs_torch_ops(dtype, interp, mode, a1, a2):
    """Propagation with flows at another size than the latents against the oracle's torch op sequence on the same GPU:
    bit-exact for fp16 and for nearest, the rule of test_ops_gpu.test_propagation_vs_torch_ops"""
    from oracle import uav_oracle as O
    from upscale_a_video_b200 import Propagation
    p = _load("propagation_resize.pt")
    x = p["x"].cuda().to(dtype)
    for name in ("up2x", "down2x", "ratio1_5", "t7"):
        ff, fb = p[name]["flows_forward"].cuda().to(dtype), p[name]["flows_backward"].cuda().to(dtype)
        ref = O.propagation(x, ff, fb, interp, mode, 0.5, a1, a2)
        got = Propagation(4, learnable=False)(x, ff, fb, interpolation=interp, mode=mode, fuse_scale=0.5, alpha1=a1,
                                              alpha2=a2)
        mism = (got != ref).float().mean().item()
        maxd = (got.float() - ref.float()).abs().max().item()
        if interp == "nearest" or dtype == torch.float16:
            assert mism == 0.0, f"{name} {dtype} {interp}: {mism * 100:.3f}% elements differ, max {maxd:.4g}"
        else:
            assert maxd <= 1e-6, f"{name} {dtype} {interp}: max abs diff {maxd:.4g}"
