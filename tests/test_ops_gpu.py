"""GPU parity of the non-GEMM kernels (norm / attention / data movement / sampler) through the C ABI.
Floating-point kernels are compared with a plain PyTorch fp32 reference of the same op (tolerances stated per
test); the sampler kernels are compared BIT-EXACTLY with the oracle's torch op sequence executed on the same GPU
(that is the arithmetic the reference performs, SURVEY.md Appendix B)."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _setup(uav_lib):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.manual_seed(0)


def _assert_close(got, ref, rtol, atol, what):
    got, ref = got.float(), ref.float()
    err = (got - ref).abs()
    bad = (err > atol + rtol * ref.abs()).sum().item()
    assert bad == 0, f"{what}: {bad}/{err.numel()} mismatches, max err {err.max().item():.4g}"


# ---------------------------------------------------------------- GroupNorm / LayerNorm
@pytest.mark.parametrize("B,T,H,W,C,G,silu", [(2, 3, 16, 24, 256, 32, True), (1, 8, 20, 28, 768, 32, True),
                                              (2, 1, 8, 8, 2048, 32, False), (1, 3, 32, 48, 128, 32, True),
                                              (2, 2, 9, 11, 512, 32, True), (1, 2, 16, 16, 1536, 32, True)])
def test_groupnorm_5d(B, T, H, W, C, G, silu):
    from upscale_a_video_b200 import ops
    x = (torch.randn(B, T, H, W, C, device="cuda") * 2 + 0.5).half()
    g = torch.randn(C, device="cuda") * 0.2 + 1
    b = torch.randn(C, device="cuda") * 0.1
    y = ops.group_norm(x, g, b, G, 1e-5, silu=silu, n_outer=B)
    ref = F.group_norm(x.float().permute(0, 4, 1, 2, 3), G, g, b, 1e-5)
    if silu:
        ref = F.silu(ref)
    _assert_close(y, ref.permute(0, 2, 3, 4, 1), 2e-3, 2e-3, "groupnorm5d")


def test_groupnorm_per_frame_and_small_c():
    from upscale_a_video_b200 import ops
    B, T, H, W, C = 2, 3, 12, 20, 512
    x = torch.randn(B, T, H, W, C, device="cuda").half()
    g = torch.randn(C, device="cuda") * 0.2 + 1
    b = torch.randn(C, device="cuda") * 0.1
    y = ops.group_norm(x, g, b, 32, 1e-6, silu=False, n_outer=B * T)
    ref = F.group_norm(x.float().reshape(B * T, H, W, C).permute(0, 3, 1, 2), 32, g, b, 1e-6).permute(0, 2, 3, 1)
    _assert_close(y.reshape(B * T, H, W, C), ref, 2e-3, 2e-3, "groupnorm per frame")
    # 3 channels stored with pixel stride 8 (condition_in of the video VAE: groups=3)
    buf = torch.zeros(1, 2, 16, 16, 8, device="cuda", dtype=torch.float16)
    buf[..., :3] = torch.randn(1, 2, 16, 16, 3, device="cuda").half()
    out = torch.zeros_like(buf)
    g3 = torch.tensor([1.0, 0.5, 2.0], device="cuda")
    b3 = torch.tensor([0.1, -0.2, 0.3], device="cuda")
    ops.group_norm(buf[..., :3], g3, b3, 3, 1e-6, silu=True, n_outer=1, out=out[..., :3])
    ref = F.silu(F.group_norm(buf[..., :3].float().permute(0, 4, 1, 2, 3), 3, g3, b3, 1e-6)).permute(0, 2, 3, 4, 1)
    _assert_close(out[..., :3], ref, 2e-3, 2e-3, "groupnorm C=3")
    assert out[..., 3:].abs().max().item() == 0


@pytest.mark.parametrize("rows,C", [(1000, 512), (777, 1024), (64, 2048), (5, 320)])
def test_layernorm(rows, C):
    from upscale_a_video_b200 import ops
    x = (torch.randn(rows, C, device="cuda") * 3 + 1).half()
    g = torch.randn(C, device="cuda") * 0.2 + 1
    b = torch.randn(C, device="cuda") * 0.1
    y = ops.layer_norm(x, g, b)
    _assert_close(y, F.layer_norm(x.float(), (C,), g, b, 1e-5), 2e-3, 2e-3, "layernorm")


# ---------------------------------------------------------------- attention
def _sdpa_ref(q, k, v, heads, kv_div=1):
    B, nq, C = q.shape
    d = C // heads
    k = k.repeat_interleave(kv_div, dim=0)
    v = v.repeat_interleave(kv_div, dim=0)
    dv = v.shape[-1] // heads
    qh = q.float().reshape(B, nq, heads, d).transpose(1, 2)
    kh = k.float().reshape(B, -1, heads, d).transpose(1, 2)
    vh = v.float().reshape(B, -1, heads, dv).transpose(1, 2)
    p = torch.softmax(qh @ kh.transpose(-1, -2) * d ** -0.5, dim=-1)
    return (p @ vh).transpose(1, 2).reshape(B, nq, heads * dv)


@pytest.mark.parametrize("B,heads,d,nq,nk,kv_div", [(4, 8, 128, 300, 300, 1), (6, 8, 64, 1000, 77, 3),
                                                    (2, 8, 128, 64, 77, 2), (3, 8, 64, 130, 130, 1),
                                                    (2, 1, 512, 400, 400, 1), (1, 1, 512, 2100, 2100, 1),
                                                    (2, 8, 128, 1500, 1500, 1), (3, 1, 512, 130, 70, 1),
                                                    (4, 8, 128, 2000, 77, 2), (2, 8, 64, 777, 100, 1), (8, 8, 64, 5000, 77, 4)])
def test_attention(B, heads, d, nq, nk, kv_div):
    from upscale_a_video_b200 import ops
    C = heads * d
    q = torch.randn(B, nq, C, device="cuda").half()
    k = torch.randn(B // kv_div, nk, C, device="cuda").half()
    v = torch.randn(B // kv_div, nk, C, device="cuda").half()
    out = ops.attention(q, k, v, heads, kv_batch_div=kv_div)
    _assert_close(out, _sdpa_ref(q, k, v, heads, kv_div), 2e-3, 2e-3, f"attention d={d}")
    # scores with a large dynamic range: exercises the online row-max rescaling of the attention kernel
    q2 = (q.float() * 6).half()
    out2 = ops.attention(q2, k, v, heads, kv_batch_div=kv_div)
    _assert_close(out2, _sdpa_ref(q2, k, v, heads, kv_div), 4e-3, 4e-3, f"attention d={d} (peaky)")


def test_attention_fused_qkv_slices():
    from upscale_a_video_b200 import ops
    B, n, heads, d = 2, 200, 8, 64
    C = heads * d
    qkv = torch.randn(B, n, 3 * C, device="cuda").half()
    q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
    out = ops.attention(q, k, v, heads)
    _assert_close(out, _sdpa_ref(q, k, v, heads), 2e-3, 2e-3, "attention qkv slices")


@pytest.mark.parametrize("B,Fr,HW,heads,d", [(2, 8, 96, 8, 64), (1, 3, 50, 8, 128), (2, 1, 33, 8, 64), (1, 5, 7, 8, 128),
                                             (1, 8, 2881, 8, 64), (2, 7, 19, 2, 128),
                                             (1, 4, 10, 3, 64)])  # odd head count: online-softmax kernel
def test_temporal_attention(B, Fr, HW, heads, d):
    """vs the oracle's TemporalAttention restatement (attention.py:699-733) in fp32"""
    from oracle import uav_oracle as O
    from upscale_a_video_b200 import ops
    C = heads * d
    qkv = torch.randn(B, Fr, HW, 3 * C, device="cuda").half()
    q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
    freqs = 1.0 / (10000 ** (torch.arange(0, 32, 2).float() / 32))
    table = torch.randn(32, heads) * 0.5
    bias = O.rel_pos_bias({"b.relative_attention_bias.weight": table}, "b", Fr).contiguous().cuda()
    ang = torch.arange(Fr).float()[:, None] * freqs[None, :]
    rot = torch.stack([ang.cos(), ang.sin()], dim=-1).contiguous().cuda()
    out = ops.temporal_attention(q, k, v, heads, rot, bias)

    def to_seq(t):  # (B,F,HW,C) -> ((B HW), heads, F, d)
        return t.float().cpu().permute(0, 2, 1, 3).reshape(B * HW, Fr, heads, d).permute(0, 2, 1, 3)

    qs, ks, vs = to_seq(q) * d ** -0.5, to_seq(k), to_seq(v)
    qs, ks = O.rotary(freqs, qs), O.rotary(freqs, ks)
    sc = torch.einsum("bhid,bhjd->bhij", qs, ks) + bias.cpu()
    pr = (sc - sc.amax(-1, keepdim=True)).softmax(-1)
    ref = torch.einsum("bhij,bhjd->bhid", pr, vs).permute(0, 2, 1, 3).reshape(B, HW, Fr, C).permute(0, 2, 1, 3)
    _assert_close(out.cpu(), ref, 3e-3, 3e-3, "temporal attention")


# ---------------------------------------------------------------- data movement
def test_layout_and_copies():
    from upscale_a_video_b200 import ops
    B, T, H, W = 2, 3, 10, 14
    sample = torch.randn(B, 4, T, H, W, device="cuda").half()
    low = torch.randn(B, 3, T, H, W, device="cuda")
    buf = torch.zeros(B, T, H, W, 8, device="cuda", dtype=torch.float16)
    ops.planar_to_channels_last(sample, buf, 0)
    ops.planar_to_channels_last(low, buf, 4, scale=0.5)
    ref = torch.cat([sample.float(), low * 0.5, torch.zeros(B, 1, T, H, W, device="cuda")], 1).permute(0, 2, 3, 4, 1)
    assert torch.equal(buf, ref.half())
    back = ops.channels_last_to_planar(buf, 4, torch.float32)
    assert torch.equal(back, sample.float())
    big = torch.randn(B, T, H, W, 4, device="cuda") * 2
    assert torch.equal(ops.channels_last_to_planar(big, 3, torch.float32, clamp=True),
                       big[..., :3].clamp(-1, 1).permute(0, 4, 1, 2, 3))
    a = torch.randn(B, T, H, W, 64, device="cuda").half()
    b = torch.randn(B, T, H, W, 128, device="cuda").half()
    assert torch.equal(ops.concat_channels(a, b), torch.cat([a, b], -1))
    up = ops.upsample_nearest(a)
    ref = F.interpolate(a.reshape(B * T, H, W, 64).permute(0, 3, 1, 2).float(), scale_factor=2, mode="nearest")
    assert torch.equal(up.reshape(B * T, 2 * H, 2 * W, 64), ref.permute(0, 2, 3, 1).half())
    up2 = ops.upsample_nearest(a, size=(13, 17))
    ref2 = F.interpolate(a.reshape(B * T, H, W, 64).permute(0, 3, 1, 2).float(), size=(13, 17), mode="nearest")
    assert torch.equal(up2.reshape(B * T, 13, 17, 64), ref2.permute(0, 2, 3, 1).half())
    x = torch.randn(5, 1024, device="cuda").half()
    _assert_close(ops.silu(x), F.silu(x.float()), 1e-3, 1e-3, "silu")
    t = torch.tensor([601.0, 34.0], device="cuda")
    from oracle import uav_oracle as O
    emb = ops.timestep_embedding(t, 256, True, 0.0)
    _assert_close(emb, O.timestep_embedding(t.cpu(), 256, True, 0).cuda(), 1e-3, 1e-3, "timestep embedding")


# ---------------------------------------------------------------- sampler (bit exact vs torch op sequence on the GPU)
@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_cfg_blend_addnoise(dtype):
    from upscale_a_video_b200 import ops
    p2 = torch.randn(2, 4, 5, 12, 16, device="cuda").to(dtype)
    u, t = p2.chunk(2)
    assert torch.equal(ops.cfg_combine(p2, 6.0), u + 6.0 * (t - u))
    dst = torch.randn(2, 4, 11, 6, 8, device="cuda").to(dtype)
    src = torch.randn(2, 4, 8, 6, 8, device="cuda").to(dtype)
    ref = dst.clone()
    for k in range(8):
        if k < 5:
            ref[:, :, 3 + k] = ref[:, :, 3 + k] * 0.5 + src[:, :, k] * 0.5
        else:
            ref[:, :, 3 + k] = src[:, :, k]
    ops.window_blend(dst, src, 3, 0b00011111)
    assert torch.equal(dst, ref)
    from upscale_a_video_b200 import _lib
    launches = _lib.launch_count()
    with pytest.raises(AssertionError):  # a non-contiguous src is rejected before the kernel would read it as dense
        ops.window_blend(dst, src.transpose(3, 4), 3, 0)
    assert _lib.launch_count() == launches and torch.equal(dst, ref)


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("cfg", ["eps_linear_clip", "v_scaled_offset", "sample_linear"])
def test_ddim_steps_bit_exact(dtype, cfg):
    import json, os
    from oracle import uav_oracle as O
    from upscale_a_video_b200.scheduling_ddim import DDIMScheduler
    meta = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "meta.json")))
    kw = meta["sched_cfgs"][cfg]
    ref, mine = O.DDIM(**kw), DDIMScheduler(**kw)
    x = torch.randn(1, 4, 3, 16, 16, device="cuda").to(dtype)
    mo = torch.randn(1, 4, 3, 16, 16, device="cuda").to(dtype)
    for steps in (30, 2):
        ref.set_timesteps(steps)
        mine.set_timesteps(steps, device="cuda")
        assert torch.equal(mine.timesteps.cpu(), ref.timesteps)
        for i in (0, steps // 2, steps - 1):
            t = ref.timesteps[i]
            x0 = mine.step_v0(mo, mine.timesteps[i], x).pred_original_sample
            assert torch.equal(x0, ref.step_v0(mo, t, x)), (cfg, dtype, steps, i)
            prev = mine.step_vt(x0, mo, mine.timesteps[i], x).prev_sample
            assert torch.equal(prev, ref.step_vt(x0, mo, t, x)), (cfg, dtype, steps, i)
    nz = mine.add_noise(x, mo, torch.tensor([120], device="cuda"))
    assert torch.equal(nz, ref.add_noise(x, mo, torch.tensor([120])))


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("interp,mode,a1,a2", [("nearest", "fuse", 0.001, 0.05), ("bilinear", "copy", 0.01, 0.5)])
def test_propagation_vs_torch_ops(dtype, interp, mode, a1, a2):
    """Propagation.forward(learnable=False) against the same torch op sequence on the same GPU."""
    import os
    from oracle import uav_oracle as O
    from upscale_a_video_b200.propagation_module import Propagation
    p = torch.load(os.path.join(os.path.dirname(__file__), "golden", "propagation.pt"), weights_only=False)["inputs"]
    x, ff, fb = (p[k].cuda().to(dtype) for k in ("x", "flows_forward", "flows_backward"))
    ref = O.propagation(x, ff, fb, interp, mode, 0.5, a1, a2)
    got = Propagation(4, learnable=False)(x, ff, fb, interpolation=interp, mode=mode, fuse_scale=0.5, alpha1=a1, alpha2=a2)
    mism = (got != ref).float().mean().item()
    maxd = (got.float() - ref.float()).abs().max().item()
    if interp == "nearest" or dtype == torch.float16:
        # the pipeline's mode (nearest + fuse, pipeline_upscale_a_video.py:655) and all fp16 modes: bit exact
        assert mism == 0.0, f"{dtype} {interp}: {mism * 100:.3f}% elements differ, max {maxd:.4g}"
    else:
        # fp32 bilinear (not used by the pipeline): ATen's grid_sampler contracts its fp32 weight/accumulate chain
        # differently from ours -> last-bit differences only
        assert maxd <= 1e-6, f"{dtype} {interp}: max abs diff {maxd:.4g}"
