"""GPU parity of the wgmma implicit-GEMM kernel (csrc/igemm.cu) through the C ABI against a
plain PyTorch fp32 reference of the same op (inputs rounded to fp16 first, fp32 math, TF32 off).
Tolerance: fp16 output rounding (rtol 1e-3) + fp32 accumulation-order noise (atol scaled by sqrt(K))."""
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


def _close(got, ref, K, what):
    got = got.float()
    ref = ref.float()
    err = (got - ref).abs()
    tol = 1e-3 * ref.abs() + 2e-3 * math.sqrt(K) * 0.02 + 1e-3
    bad = (err > tol).sum().item()
    assert bad == 0, f"{what}: {bad}/{err.numel()} mismatches, max err {err.max().item():.4g}, ref max {ref.abs().max().item():.4g}"


@pytest.mark.parametrize("M,K,N", [(128, 64, 16), (128, 64, 256), (1000, 512, 512), (300, 1024, 1024),
                                   (2, 256, 1024), (4096, 320, 128), (257, 72, 40), (130, 512, 4)])
def test_linear(M, K, N):
    from upscale_a_video_b200 import ops
    a = torch.randn(M, K, device="cuda").half()
    w = (torch.randn(N, K, device="cuda") * 0.05).half()
    b = torch.randn(N, device="cuda")
    out = ops.linear(a, w, b)
    ref = a.float() @ w.float().t() + b
    _close(out, ref, K, f"linear {M}x{K}x{N}")


def test_linear_epilogue_variants():
    from upscale_a_video_b200 import ops
    M, K, N = 777, 512, 512
    a = torch.randn(M, K, device="cuda").half()
    w = (torch.randn(N, K, device="cuda") * 0.05).half()
    b = torch.randn(N, device="cuda")
    res = torch.randn(M, N, device="cuda").half()
    rv = torch.randn(3, N, device="cuda").half()
    out = ops.linear(a, w, b, residual=res, rowvec=rv, rows_per_vec=259, act=ops.ACT_SILU)
    lin = a.float() @ w.float().t() + b + rv.float()[torch.arange(M, device="cuda") // 259]
    ref = F.silu(lin) + res.float()
    _close(out, ref, K, "linear+rowvec+silu+res")
    out32 = ops.linear(a, w, None, out_dtype=torch.float32)
    _close(out32, a.float() @ w.float().t(), K, "linear fp32 out")
    # write into a channel slice of a wider buffer
    buf = torch.zeros(M, N + 64, device="cuda", dtype=torch.float16)
    ops.linear(a, w, b, out=buf[:, 64:])
    _close(buf[:, 64:], a.float() @ w.float().t() + b, K, "linear slice out")
    assert buf[:, :64].abs().max().item() == 0


def test_geglu():
    from upscale_a_video_b200 import ops
    M, K, N = 515, 512, 4096
    a = torch.randn(M, K, device="cuda").half()
    w = (torch.randn(N, K, device="cuda") * 0.05).half()
    b = torch.randn(N, device="cuda") * 0.1
    out = ops.linear(a, w, b, act=ops.ACT_GEGLU)
    y = a.float() @ w.float().t() + b
    h, g = y.chunk(2, dim=-1)
    _close(out, h * F.gelu(g), K, "geglu")


def _conv_ref(x, w, b, stride=1, padding=1):
    # x (NB,H,W,C) channels-last; w (Cout,k,k,Cin)
    y = F.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), b, stride=stride, padding=padding)
    return y.permute(0, 2, 3, 1)


@pytest.mark.parametrize("NB,H,W,Cin,Cout,k", [
    (2, 16, 16, 64, 64, 3), (3, 40, 72, 128, 256, 3), (2, 33, 47, 64, 128, 3), (1, 64, 64, 8, 256, 3),
    (2, 24, 40, 256, 4, 3), (2, 20, 36, 768, 256, 3), (2, 20, 36, 192, 64, 1), (1, 8, 8, 512, 512, 3),
    (1, 128, 160, 64, 32, 3),
])
def test_conv2d(NB, H, W, Cin, Cout, k):
    from upscale_a_video_b200 import ops
    x = torch.randn(NB, H, W, Cin, device="cuda").half()
    w = (torch.randn(Cout, k, k, Cin, device="cuda") * 0.05).half()
    b = torch.randn(Cout, device="cuda")
    out = ops.conv2d(x, w, b)
    ref = _conv_ref(x, w, b, 1, k // 2)
    _close(out, ref, Cin * k * k, f"conv2d {NB}x{H}x{W} {Cin}->{Cout} k{k}")


@pytest.mark.parametrize("NB,H,W,Cin,Cout,pad_mode", [(2, 32, 48, 64, 64, 0), (3, 40, 72, 256, 256, 0),
                                                      (1, 18, 22, 128, 128, 0), (2, 32, 48, 128, 128, 1)])
def test_conv2d_stride2(NB, H, W, Cin, Cout, pad_mode):
    from upscale_a_video_b200 import ops
    x = torch.randn(NB, H, W, Cin, device="cuda").half()
    w = (torch.randn(Cout, 3, 3, Cin, device="cuda") * 0.05).half()
    b = torch.randn(Cout, device="cuda")
    out = ops.conv2d(x, w, b, stride=2, pad_mode=pad_mode)
    if pad_mode == 0:
        ref = _conv_ref(x, w, b, 2, 1)
    else:
        xp = F.pad(x.float().permute(0, 3, 1, 2), (0, 1, 0, 1))
        ref = F.conv2d(xp, w.float().permute(0, 3, 1, 2), b, stride=2).permute(0, 2, 3, 1)
    _close(out, ref, Cin * 9, f"conv2d s2 pad_mode{pad_mode}")


def test_conv2d_slice_in_and_residual_temb():
    from upscale_a_video_b200 import ops
    B, T, H, W, C0, C1, Cout = 2, 3, 20, 28, 64, 128, 128
    buf = torch.randn(B, T, H, W, C0 + C1, device="cuda").half()
    x = buf[..., C0:]
    w = (torch.randn(Cout, 3, 3, C1, device="cuda") * 0.05).half()
    b = torch.randn(Cout, device="cuda")
    temb = torch.randn(B, Cout, device="cuda").half()
    res = torch.randn(B, T, H, W, Cout, device="cuda").half()
    out = ops.conv2d(x, w, b, rowvec=temb, rows_per_vec=T * H * W, residual=res)
    ref = _conv_ref(x.reshape(B * T, H, W, C1), w, b).reshape(B, T, H, W, Cout)
    ref = ref + temb.float()[:, None, None, None, :] + res.float()
    _close(out, ref, C1 * 9, "conv2d slice+temb+res")


@pytest.mark.parametrize("B,T,H,W,Cin,Cout,k", [(2, 8, 12, 20, 64, 64, 3), (1, 5, 16, 24, 256, 256, 5),
                                                (2, 1, 9, 11, 128, 128, 3), (1, 3, 40, 40, 512, 512, 5)])
def test_conv_temporal(B, T, H, W, Cin, Cout, k):
    from upscale_a_video_b200 import ops
    x = torch.randn(B, T, H, W, Cin, device="cuda").half()
    w = (torch.randn(Cout, k, Cin, device="cuda") * 0.05).half()
    b = torch.randn(Cout, device="cuda")
    out = ops.conv_temporal(x, w, b)
    w5 = w.float().permute(0, 2, 1)[:, :, :, None, None]  # (Cout, Cin, k, 1, 1)
    ref = F.conv3d(x.float().permute(0, 4, 1, 2, 3), w5, b, padding=(k // 2, 0, 0)).permute(0, 2, 3, 4, 1)
    _close(out, ref, Cin * k, f"conv_temporal k{k}")


@pytest.mark.parametrize("B,T,H,W,Cin,Cout", [(1, 3, 16, 24, 64, 64), (2, 2, 20, 20, 128, 128)])
def test_conv3d(B, T, H, W, Cin, Cout):
    from upscale_a_video_b200 import ops
    x = torch.randn(B, T, H, W, Cin, device="cuda").half()
    w = (torch.randn(Cout, 3, 3, 3, Cin, device="cuda") * 0.05).half()
    b = torch.randn(Cout, device="cuda")
    out = ops.conv3d(x, w, b)
    ref = F.conv3d(x.float().permute(0, 4, 1, 2, 3), w.float().permute(0, 4, 1, 2, 3), b, padding=1)
    _close(out, ref.permute(0, 2, 3, 4, 1), Cin * 27, "conv3d")


# ---- large launches (>= 2 * num_SMs M-tiles: several tiles per persistent CTA); odd tile counts, ragged last tiles
@pytest.mark.parametrize("M,K,N,act", [(299 * 128 - 3, 512, 512, 0), (300 * 128, 320, 128, 0), (301 * 128 + 7, 512, 2048, 2),
                                       (298 * 128, 1024, 384, 1)])
def test_linear_cluster(M, K, N, act):
    from upscale_a_video_b200 import ops
    a = torch.randn(M, K, device="cuda").half()
    w = (torch.randn(N, K, device="cuda") * 0.05).half()
    b = torch.randn(N, device="cuda") * 0.1
    res = torch.randn(M, N // 2 if act == 2 else N, device="cuda").half() if act != 2 else None
    out = ops.linear(a, w, b, act=act, residual=res)
    y = a.float() @ w.float().t() + b
    if act == 2:
        h, g = y.chunk(2, dim=-1)
        ref = h * F.gelu(g)
    elif act == 1:
        ref = F.silu(y) + res.float()
    else:
        ref = y + res.float()
    _close(out, ref, K, f"cluster linear {M}x{K}x{N} act{act}")


@pytest.mark.parametrize("NB,H,W,Cin,Cout,k,stride", [(5, 96, 160, 128, 256, 3, 1), (3, 128, 208, 64, 128, 3, 1),
                                                      (7, 160, 144, 64, 256, 3, 2), (2, 168, 232, 256, 512, 1, 1)])
def test_conv2d_cluster(NB, H, W, Cin, Cout, k, stride):
    from upscale_a_video_b200 import ops
    x = torch.randn(NB, H, W, Cin, device="cuda").half()
    w = (torch.randn(Cout, k, k, Cin, device="cuda") * 0.05).half()
    b = torch.randn(Cout, device="cuda")
    out = ops.conv2d(x, w, b, stride=stride)
    ref = _conv_ref(x, w, b, stride, k // 2)
    _close(out, ref, Cin * k * k, f"cluster conv2d {NB}x{H}x{W} {Cin}->{Cout} k{k} s{stride}")


@pytest.mark.parametrize("NB,H,W,Cin,Cout", [(2, 12, 20, 64, 64), (3, 40, 72, 128, 256), (16, 20, 36, 512, 512), (1, 9, 7, 256, 128)])
def test_upsample2x_conv3x3(NB, H, W, Cin, Cout):
    """nearest x2 + 3x3 conv via four collapsed 2x2 phase filters == upsample then conv (weights summed in fp32 and
    rounded once, so the tolerance includes that extra fp16 weight rounding)"""
    from upscale_a_video_b200 import ops
    x = torch.randn(NB, H, W, Cin, device="cuda").half()
    w = (torch.randn(Cout, 3, 3, Cin, device="cuda") * 0.05).half()
    b = torch.randn(Cout, device="cuda")
    out = ops.upsample2x_conv3x3(x, ops.collapse_upsample_filter(w), b)
    up = F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2, mode="nearest")
    ref = F.conv2d(up, w.float().permute(0, 3, 1, 2), b, padding=1).permute(0, 2, 3, 1)
    assert out.shape == ref.shape
    _close(out, ref, Cin * 9, f"upsample2x+conv {NB}x{H}x{W} {Cin}->{Cout}")


# ------------------------------------------------------------------------------------------------------------------
# round 2: epilogue extensions — output scale, saturating fp16 stores, GroupNorm statistics emitted by the producer
# ------------------------------------------------------------------------------------------------------------------
from upscale_a_video_b200 import ops  # noqa: E402

DEV = "cuda"


def _rand(*shape, scale=1.0):
    return (torch.randn(*shape, device=DEV) * scale).half()


def _check(got, ref, atol=2e-3, rtol=2e-3):
    err = (got.float() - ref.float()).abs()
    bad = (err > atol + rtol * ref.float().abs()).sum().item()
    assert bad == 0, f"{bad}/{err.numel()} mismatches, max err {err.max().item():.4g}, ref max {ref.abs().max().item():.4g}"


def test_out_scale_and_saturation():
    a, w = _rand(300, 128, scale=1.0), _rand(256, 128, scale=0.1)
    res = _rand(300, 256, scale=100.0)
    bias = torch.randn(256, device=DEV)
    out = ops.linear(a, w, bias, residual=res, out_scale=2.0 ** -5)
    ref = (a.float() @ w.float().t() + bias) * 2.0 ** -5 + res.float()
    _check(out, ref)
    # conv with scale, no residual
    x, wc = _rand(2, 20, 24, 64), _rand(128, 3, 3, 64, scale=0.05)
    out = ops.conv2d(x, wc, None, out_scale=0.25)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), wc.float().permute(0, 3, 1, 2), padding=1).permute(0, 2, 3, 1) * 0.25
    _check(out, ref)
    # fp16 stores saturate instead of producing inf
    big = ops.linear(_rand(130, 64, scale=30.0), _rand(64, 64, scale=30.0), torch.full((64,), 1e5, device=DEV))
    assert torch.isfinite(big).all() and big.max().item() == 65504.0


def _gn_ref(x, gamma, beta, groups, eps, silu, n_outer):
    C = x.shape[-1]
    v = x.float().reshape(n_outer, -1, C).permute(0, 2, 1)
    y = F.group_norm(v, groups, gamma, beta, eps)
    if silu:
        y = F.silu(y)
    return y.permute(0, 2, 1).reshape(x.shape)


@pytest.mark.parametrize("case", ["conv3x3", "conv3x3_big", "conv_t", "linear", "conv1x1_res", "conv3d", "ragged"])
def test_groupnorm_statistics_from_the_producer_epilogue(case):
    """the producing GEMM emits {sum, sumsq} blocks of its OUTPUT (uav_epilogue_t.gn_partial); GroupNorm from those
    blocks == GroupNorm with its own statistics pass (same fp64 finalisation; the fused statistics see the fp32 values
    before the fp16 rounding, so the two differ by rounding noise only) == torch's group_norm"""
    torch.manual_seed(3)
    groups, eps = 32, 1e-5
    if case == "conv3x3":
        x, w = _rand(2, 4, 20, 28, 64), _rand(256, 3, 3, 64, scale=0.05)
        y = ops.conv2d(x, w, torch.randn(256, device=DEV), gn_stats=True)
        n_outer_list = [2, 8]
    elif case == "conv3x3_big":  # >= 2 M-tiles per SM: persistent loop, odd tile count
        x, w = _rand(1, 7, 80, 84, 64), _rand(128, 3, 3, 64, scale=0.05)   # 385 M-tiles (8 x 16 pixel boxes)
        y = ops.conv2d(x, w, None, residual=_rand(1, 7, 80, 84, 128), gn_stats=True)
        n_outer_list = [1, 7]
    elif case == "conv_t":
        x, w = _rand(2, 5, 12, 17, 128), _rand(256, 3, 128, scale=0.05)
        y = ops.conv_temporal(x, w, torch.randn(256, device=DEV), residual=_rand(2, 5, 12, 17, 256), gn_stats=True)
        n_outer_list = [2, 10]
    elif case == "linear":
        x, w = _rand(2, 4, 256, 128), _rand(512, 128, scale=0.1)
        y = ops.linear(x, w, torch.randn(512, device=DEV), residual=_rand(2, 4, 256, 512), gn_stats=True)
        n_outer_list = [2, 8]
    elif case == "conv1x1_res":
        x, w = _rand(2, 2, 16, 32, 256), _rand(256, 1, 1, 256, scale=0.1)
        y = ops.conv2d(x, w, torch.randn(256, device=DEV), residual=x, gn_stats=True)
        n_outer_list = [2, 4]
    elif case == "conv3d":
        x, w = _rand(1, 3, 10, 12, 64), _rand(128, 3, 3, 3, 64, scale=0.05)
        y = ops.conv3d(x, w, torch.randn(128, device=DEV), gn_stats=True, out_scale=0.125)
        n_outer_list = [1]
    else:  # rows per slab not a multiple of 128 for a Linear producer: the consumer must fall back to its own pass
        x, w = _rand(2, 3, 50, 128), _rand(256, 128, scale=0.1)
        y = ops.linear(x, w, None, gn_stats=True)
        assert y.uav_gn[0].slabs_for(2, 2) == 0
        n_outer_list = [2]
    st = y.uav_gn
    assert st and st[0].C == y.shape[-1]
    C = y.shape[-1]
    gamma, beta = torch.randn(C, device=DEV) * 0.2 + 1, torch.randn(C, device=DEV) * 0.1
    for n_outer in n_outer_list:
        fused = ops.group_norm(y, gamma, beta, groups, eps, silu=True, n_outer=n_outer, stats=st, batch=y.shape[0])
        plain = ops.group_norm(y, gamma, beta, groups, eps, silu=True, n_outer=n_outer)
        ref = _gn_ref(y, gamma, beta, groups, eps, True, n_outer)
        assert (fused.float() - plain.float()).abs().max().item() < 4e-3
        _check(fused, ref, atol=4e-3)


def test_groupnorm_statistics_of_a_concat_and_a_broadcast_skip():
    """torch.cat([x, skip]) -> GroupNorm (unet_blocks.py:573,645 + resnet.py:267): statistics come from BOTH producers;
    a skip computed once for the two classifier-free-guidance halves (batch 1) serves both slabs; 48 channels per group
    straddle the concat boundary (1024 + 512 channels)"""
    torch.manual_seed(4)
    B, T, H, W = 2, 2, 8, 16
    xa = ops.conv2d(_rand(B, T, H, W, 64), _rand(1024, 3, 3, 64, scale=0.05), None, gn_stats=True)
    xb1 = ops.conv2d(_rand(1, T, H, W, 64), _rand(512, 3, 3, 64, scale=0.05), None, gn_stats=True)
    cat = ops.concat_channels(xa, xb1)  # broadcasts the batch-1 skip
    assert len(cat.uav_gn) == 2
    C = 1536
    gamma, beta = torch.randn(C, device=DEV) * 0.2 + 1, torch.randn(C, device=DEV) * 0.1
    fused = ops.group_norm(cat, gamma, beta, 32, 1e-5, silu=True, n_outer=B, stats=cat.uav_gn, batch=B)
    ref = _gn_ref(cat, gamma, beta, 32, 1e-5, True, B)
    _check(fused, ref, atol=4e-3)
    rep = ops.repeat_batch(xb1, 2)
    fused = ops.group_norm(rep, gamma[:512].contiguous(), beta[:512].contiguous(), 32, 1e-5, silu=False, n_outer=2,
                           stats=rep.uav_gn, batch=2)
    _check(fused, _gn_ref(rep, gamma[:512], beta[:512], 32, 1e-5, False, 2), atol=4e-3)


@pytest.mark.parametrize("M,K,N", [(148 * 2 * 128 + 77, 512, 512), (40000, 128, 320), (5000, 256, 192)])
def test_residual_tile_through_tma(M, K, N):
    """the residual operand arrives as a TMA tile in shared memory (one tile ahead for single-tap GEMMs, in the staging
    tile for convolutions): residual = channel slice of a wider buffer, ragged last M-tile, N not a multiple of the tile"""
    a, w = _rand(M, K), _rand(N, K, scale=0.05)
    wide = _rand(M, N + 64)
    res = wide[:, 64:]
    out = ops.linear(a, w, None, residual=res, out_scale=0.5)
    _close(out, (a.float() @ w.float().t()) * 0.5 + res.float(), K, f"linear+res(slice) {M}x{K}x{N}")
    # convolution, residual in place of the staging tile, output written over a slice of a wider buffer
    x, wc = _rand(3, 40, 52, 64), _rand(192, 3, 3, 64, scale=0.05)
    r = _rand(3, 40, 52, 192)
    buf = torch.zeros(3, 40, 52, 256, device=DEV, dtype=torch.float16)
    ops.conv2d(x, wc, None, residual=r, out=buf[..., 64:])
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), wc.float().permute(0, 3, 1, 2), padding=1).permute(0, 2, 3, 1) + r.float()
    _close(buf[..., 64:], ref, 576, "conv+res -> slice")
    assert buf[..., :64].abs().max().item() == 0


def test_groupnorm_of_a_concat_that_is_never_built():
    """ops.group_norm_cat: GroupNorm(cat([x, skip])) -> dense tensor, the two inputs read in place (one apply launch per
    part), statistics from their producers; a batch-1 skip serves both batch items; groups straddle the boundary"""
    torch.manual_seed(5)
    B, T, H, W = 2, 3, 16, 24   # t*h*w = 9 x 128 rows per batch item: a Linear producer's blocks split per batch item
    for cx, cs, skip_b in ((1024, 512, 1), (512, 256, 2), (256, 256, 1)):
        x = ops.conv2d(_rand(B, T, H, W, 64), _rand(cx, 3, 3, 64, scale=0.05), None, gn_stats=True)
        skip = ops.linear(_rand(skip_b, T, H * W, 128), _rand(cs, 128, scale=0.1), torch.randn(cs, device=DEV), gn_stats=True)
        st = skip.uav_gn
        skip = skip.view(skip_b, T, H, W, cs)
        skip.uav_gn = st  # a reshaped view keeps its producer's statistics (layers._carry_gn)
        C = cx + cs
        gamma, beta = torch.randn(C, device=DEV) * 0.2 + 1, torch.randn(C, device=DEV) * 0.1
        got = ops.group_norm_cat([x, skip], gamma, beta, 32, 1e-5, silu=True, n_outer=B)
        assert got is not None and tuple(got.shape) == (B, T, H, W, C) and got.is_contiguous()
        cat = torch.cat([x, skip.expand(B, -1, -1, -1, -1)], dim=-1)
        _check(got, _gn_ref(cat, gamma, beta, 32, 1e-5, True, B), atol=4e-3)
    # a part without statistics -> None (the caller materialises the concat)
    assert ops.group_norm_cat([x, _rand(B, T, H, W, 256)], gamma, beta, 32, 1e-5, silu=True, n_outer=B) is None
