"""GPU parity of the 128x256 implicit-GEMM tiles (csrc/igemm.cu, BLOCK_N = 256) against fp32 PyTorch, with the kernel
instance that ran read from torch.profiler.

Convolutions and GEGLU take 256-column tiles when they cut the number of waves of persistent CTAs: each wide shape below
has at most one wave of 256-column tiles and two waves of 128-column tiles, so the wide instance must run.  A launch where
both widths fit in one wave, and a Linear without GEGLU, keep the 128-column tiles.  Tolerances are those of test_igemm_gpu.py."""
import math
import re

import pytest
import torch
import torch.nn.functional as F

from upscale_a_video_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(autouse=True)
def _setup(uav_lib):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.manual_seed(0)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _rand(*shape, scale=1.0):
    return (torch.randn(*shape, device=DEV) * scale).half()


def _close(got, ref, K, what):
    got = got.float()
    ref = ref.float()
    err = (got - ref).abs()
    tol = 1e-3 * ref.abs() + 2e-3 * math.sqrt(K) * 0.02 + 1e-3
    bad = (err > tol).sum().item()
    assert bad == 0, f"{what}: {bad}/{err.numel()} mismatches, max err {err.max().item():.4g}, ref max {ref.abs().max().item():.4g}"


def _check(got, ref, atol=2e-3, rtol=2e-3):
    err = (got.float() - ref.float()).abs()
    bad = (err > atol + rtol * ref.float().abs()).sum().item()
    assert bad == 0, f"{bad}/{err.numel()} mismatches, max err {err.max().item():.4g}, ref max {ref.abs().max().item():.4g}"


_INSTANCE = re.compile(r"igemm_kernel<(\d+), (true|false), (true|false), (true|false)>")


def _run(fn):
    """fn() under torch.profiler -> (its result, set of (BLOCK_N, GEGLU, TMA_EPI, AUX) instances that ran)"""
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    ran = set()
    for ev in prof.events():
        m = _INSTANCE.search(ev.name)
        if m:
            ran.add((int(m.group(1)), m.group(2) == "true", m.group(3) == "true", m.group(4) == "true"))
    assert ran, "no igemm_kernel launch in the trace"
    return out, ran


def _widths(ran):
    return {r[0] for r in ran}


def _m_tiles(n_wide_tiles):
    """M-tiles such that the launch is one wave of 256-column tiles and two waves of 128-column tiles"""
    m = _sms() // n_wide_tiles
    assert m * n_wide_tiles > _sms() // 2
    return m


# every 2-D shape below is W=64 x H=16 per image: pick_tile_2d covers it with 8 boxes of 64 x 2 pixels
PIX_W, PIX_H, TILES_PER_IMAGE = 64, 16, 8


def _images(n_wide_tiles):
    return _m_tiles(n_wide_tiles * TILES_PER_IMAGE)


def _temporal_ref(x, w, b, k):
    w5 = w.float().permute(0, 2, 1)[:, :, :, None, None]
    return F.conv3d(x.float().permute(0, 4, 1, 2, 3), w5, b, padding=(k // 2, 0, 0)).permute(0, 2, 3, 4, 1)


# temporal (3,1,1) conv over 1019-pixel frames: 8 M-tiles per frame, the last one ragged
HW_RAGGED = 1019


@pytest.mark.parametrize("N", [256, 512, 1024, 384, 264])
def test_conv_temporal_n_wide(N):
    K = 256
    T = _images((N + 255) // 256)
    x, w = _rand(1, T, 1, HW_RAGGED, K), _rand(N, 3, K, scale=0.05)
    b = torch.randn(N, device=DEV)
    out, ran = _run(lambda: ops.conv_temporal(x, w, b))
    assert _widths(ran) == {256}, ran
    _close(out, _temporal_ref(x, w, b, 3), 3 * K, f"conv_temporal {K}->{N}")


def test_geglu_wide():
    N, K = 4096, 512
    M = 128 * _m_tiles(N // 2 // 128) - 9
    a, w = _rand(M, K), _rand(N, K, scale=0.05)
    b = torch.randn(N, device=DEV) * 0.1
    out, ran = _run(lambda: ops.linear(a, w, b, act=ops.ACT_GEGLU))
    assert ran == {(256, True, True, False)}, ran
    h, g = (a.float() @ w.float().t() + b).chunk(2, dim=-1)
    _close(out, h * F.gelu(g), K, "geglu")


def test_single_tap_and_small_launches_keep_128_column_tiles():
    """a Linear keeps 128-column tiles at any size; so does a convolution that fits in one wave either way"""
    N, K = 512, 512
    M = 128 * _m_tiles(2)
    a, w = _rand(M, K), _rand(N, K, scale=0.05)
    out, ran = _run(lambda: ops.linear(a, w, None))
    assert _widths(ran) == {128}, ran
    _close(out, a.float() @ w.float().t(), K, "linear")
    T = _images(2) // 2
    x, wt = _rand(1, T, 1, HW_RAGGED, K), _rand(N, 3, K, scale=0.05)
    out, ran = _run(lambda: ops.conv_temporal(x, wt, None))
    assert _widths(ran) == {128}, ran
    _close(out, _temporal_ref(x, wt, None, 3), 3 * K, "conv_temporal, one wave")


def test_residual_through_tma_wide():
    """residual = channel slice of a wider buffer, loaded by TMA into the four output slabs; ragged last M-tile"""
    N, K = 512, 256
    T = _images(2)
    x, w = _rand(1, T, 1, HW_RAGGED, K), _rand(N, 3, K, scale=0.05)
    wide = _rand(1, T, 1, HW_RAGGED, N + 64)
    res = wide[..., 64:]
    out, ran = _run(lambda: ops.conv_temporal(x, w, None, residual=res, out_scale=0.5))
    assert ran == {(256, False, True, True)}, ran
    _close(out, _temporal_ref(x, w, None, 3) * 0.5 + res.float(), 3 * K, "conv_temporal+res(slice)")


def _conv_ref(x, w, b):
    return F.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), b, padding=1).permute(0, 2, 3, 1)


def test_rowvec_silu_wide():
    N, K, B = 512, 128, 2
    NB = _images(2)
    x, w = _rand(NB, PIX_H, PIX_W, K), _rand(N, 3, 3, K, scale=0.05)
    b = torch.randn(N, device=DEV)
    rv = _rand(B, N)
    rpv = NB // B * PIX_H * PIX_W
    out, ran = _run(lambda: ops.conv2d(x, w, b, rowvec=rv, rows_per_vec=rpv, act=ops.ACT_SILU))
    assert ran == {(256, False, True, True)}, ran
    ref = _conv_ref(x, w, b) + rv.float().repeat_interleave(NB // B, dim=0)[:, None, None, :]
    _close(out, F.silu(ref), 9 * K, "conv3x3+rowvec+silu")


def test_out_scale_and_saturation_wide():
    N, K = 512, 64
    NB = _images(2)
    x, w = _rand(NB, PIX_H, PIX_W, K), _rand(N, 3, 3, K, scale=0.1)
    res = _rand(NB, PIX_H, PIX_W, N, scale=100.0)
    bias = torch.randn(N, device=DEV)
    out, ran = _run(lambda: ops.conv2d(x, w, bias, residual=res, out_scale=2.0 ** -5))
    assert _widths(ran) == {256}, ran
    _check(out, _conv_ref(x, w, bias) * 2.0 ** -5 + res.float())
    big, ran = _run(lambda: ops.conv2d(_rand(NB, PIX_H, PIX_W, K, scale=30.0), _rand(N, 3, 3, K, scale=30.0),
                                       torch.full((N,), 1e5, device=DEV)))
    assert _widths(ran) == {256}, ran
    assert torch.isfinite(big).all() and big.max().item() == 65504.0


def test_fp32_output_direct_stores_wide():
    N, K = 512, 128
    NB = _images(2)
    x, w = _rand(NB, PIX_H, PIX_W, K), _rand(N, 3, 3, K, scale=0.05)
    out, ran = _run(lambda: ops.conv2d(x, w, None, out_dtype=torch.float32))
    assert ran == {(256, False, False, True)}, ran
    assert out.dtype == torch.float32
    _close(out, _conv_ref(x, w, None), 9 * K, "conv3x3 fp32 out")


def test_groupnorm_statistics_wide():
    """GroupNorm statistics blocks (16 rows x 8 columns) written by the 256-column epilogue"""
    torch.manual_seed(3)
    B = 2
    T = _images(2) // B
    C = 512
    x, w = _rand(B, T, PIX_H, PIX_W, 128), _rand(C, 3, 3, 128, scale=0.05)
    y, ran = _run(lambda: ops.conv2d(x, w, torch.randn(C, device=DEV), gn_stats=True))
    assert ran == {(256, False, True, True)}, ran
    st = y.uav_gn
    gamma, beta = torch.randn(C, device=DEV) * 0.2 + 1, torch.randn(C, device=DEV) * 0.1
    for n_outer in (B, B * T):
        fused = ops.group_norm(y, gamma, beta, 32, 1e-5, silu=True, n_outer=n_outer, stats=st, batch=B)
        plain = ops.group_norm(y, gamma, beta, 32, 1e-5, silu=True, n_outer=n_outer)
        v = y.float().reshape(n_outer, -1, C).permute(0, 2, 1)
        ref = F.silu(F.group_norm(v, 32, gamma, beta, 1e-5)).permute(0, 2, 1).reshape(y.shape)
        assert (fused.float() - plain.float()).abs().max().item() < 4e-3
        _check(fused, ref, atol=4e-3)


@pytest.mark.parametrize("Cin,Cout", [(256, 256), (128, 512)])
def test_conv3x3_wide(Cin, Cout):
    NB = _images(Cout // 256)
    x, w = _rand(NB, PIX_H, PIX_W, Cin), _rand(Cout, 3, 3, Cin, scale=0.05)
    b = torch.randn(Cout, device=DEV)
    out, ran = _run(lambda: ops.conv2d(x, w, b))
    assert _widths(ran) == {256}, ran
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), b, padding=1).permute(0, 2, 3, 1)
    _close(out, ref, Cin * 9, f"conv3x3 {Cin}->{Cout}")


@pytest.mark.parametrize("pad_mode", [0, 1])
def test_conv3x3_stride2_wide(pad_mode):
    Cin, Cout = 128, 512
    NB = _images(2)
    x, w = _rand(NB, 2 * PIX_H, 2 * PIX_W, Cin), _rand(Cout, 3, 3, Cin, scale=0.05)
    b = torch.randn(Cout, device=DEV)
    out, ran = _run(lambda: ops.conv2d(x, w, b, stride=2, pad_mode=pad_mode))
    assert _widths(ran) == {256}, ran
    xp = x.float().permute(0, 3, 1, 2)
    if pad_mode == 0:
        ref = F.conv2d(xp, w.float().permute(0, 3, 1, 2), b, stride=2, padding=1)
    else:
        ref = F.conv2d(F.pad(xp, (0, 1, 0, 1)), w.float().permute(0, 3, 1, 2), b, stride=2)
    _close(out, ref.permute(0, 2, 3, 1), Cin * 9, f"conv3x3 s2 pad_mode{pad_mode}")


def test_conv3d_wide():
    Cin, Cout = 64, 256
    B = 1
    T = _images(1)
    x, w = _rand(B, T, PIX_H, PIX_W, Cin), _rand(Cout, 3, 3, 3, Cin, scale=0.05)
    b = torch.randn(Cout, device=DEV)
    out, ran = _run(lambda: ops.conv3d(x, w, b))
    assert _widths(ran) == {256}, ran
    ref = F.conv3d(x.float().permute(0, 4, 1, 2, 3), w.float().permute(0, 4, 1, 2, 3), b, padding=1)
    _close(out, ref.permute(0, 2, 3, 4, 1), Cin * 27, "conv3d")


def test_conv2d_taps_wide():
    Cin, Cout, kh, kw = 128, 256, 1, 7
    NB = _images(1)
    x, w = _rand(NB, PIX_H, PIX_W, Cin), _rand(Cout, kh, kw, Cin, scale=0.05)
    b = torch.randn(Cout, device=DEV)
    out, ran = _run(lambda: ops.conv2d_taps(x, w, b, pad_top=0, pad_left=3))
    assert _widths(ran) == {256}, ran
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), b, padding=(0, 3)).permute(0, 2, 3, 1)
    _close(out, ref, Cin * kh * kw, "conv2d_taps 1x7")


def test_upsample2x_conv3x3_wide():
    """four phase launches, each writing a strided view of the 2x output through the TMA store"""
    Cin, Cout = 128, 512
    NB = _images(2)
    x, w = _rand(NB, PIX_H, PIX_W, Cin), _rand(Cout, 3, 3, Cin, scale=0.05)
    b = torch.randn(Cout, device=DEV)
    out, ran = _run(lambda: ops.upsample2x_conv3x3(x, ops.collapse_upsample_filter(w), b))
    assert ran == {(256, False, True, False)}, ran
    up = F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2, mode="nearest")
    ref = F.conv2d(up, w.float().permute(0, 3, 1, 2), b, padding=1).permute(0, 2, 3, 1)
    _close(out, ref, Cin * 9, "upsample2x+conv 128->512")

