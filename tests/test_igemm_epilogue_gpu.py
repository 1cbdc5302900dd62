"""GPU parity of the 128-column TMA-store epilogue of the implicit GEMM (csrc/igemm.cu, igemm_kernel<128, false, true,
AUX>: every Linear and 1x1 conv with N > 64) against fp32 PyTorch with the tolerance of test_igemm_gpu.py, and its
GroupNorm statistics block by block against torch's sums.

The shapes cover ragged M and N tiles, one k-block per tile (the producer runs several tiles ahead of an epilogue that
is slower than the main loop), a long K, and launches where every CTA runs at least three tiles so that the stage ring
and the residual barrier go through both phases more than once.  The same launch run twice must be bitwise equal."""
import math

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


def _rows(M, n_tiles_per_m):
    """M, or for M = "many": rows such that every persistent CTA runs at least three tiles, the last M-tile ragged"""
    if M != "many":
        return M
    return 128 * ((3 * _sms() + n_tiles_per_m - 1) // n_tiles_per_m + 1) - 5


@pytest.mark.parametrize("M,K,N", [
    (130, 512, 512),    # M tail: one full and one 2-row M-tile
    (1000, 512, 512),   # M tail
    (777, 256, 200),    # n_out tail: 128 + 72 columns
    (1000, 320, 328),   # n_out tail: 2 x 128 + 72 columns
    ("many", 8, 128),   # one k-block per tile: the epilogue is the slower side
    (1000, 4096, 256),  # 64 k-blocks per tile
    ("many", 512, 512),
])
def test_linear_bias(M, K, N):
    M = _rows(M, (N + 127) // 128)
    a, w = _rand(M, K), _rand(N, K, scale=0.05)
    b = torch.randn(N, device=DEV)
    out = ops.linear(a, w, b)
    _close(out, a.float() @ w.float().t() + b, K, f"linear {M}x{K}x{N}")


@pytest.mark.parametrize("M,K,N", [(1000, 512, 328), ("many", 512, 512), ("many", 8, 128)])
def test_linear_residual_out_scale(M, K, N):
    """residual (a channel slice of a wider buffer) loaded by TMA into the staging tile while the main loop runs"""
    M = _rows(M, (N + 127) // 128)
    a, w = _rand(M, K), _rand(N, K, scale=0.05)
    wide = _rand(M, N + 64)
    res = wide[:, 64:]
    out = ops.linear(a, w, None, residual=res, out_scale=0.5)
    _close(out, (a.float() @ w.float().t()) * 0.5 + res.float(), K, f"linear+res {M}x{K}x{N}")


def test_linear_rowvec_silu():
    K, N = 512, 256
    M = _rows("many", 2) // 3 * 3  # rows_per_vec divides M: every row has its row vector
    a, w = _rand(M, K), _rand(N, K, scale=0.05)
    b = torch.randn(N, device=DEV)
    rows_per_vec = M // 3
    rv = _rand(3, N)
    out = ops.linear(a, w, b, rowvec=rv, rows_per_vec=rows_per_vec, act=ops.ACT_SILU)
    idx = torch.arange(M, device=DEV) // rows_per_vec
    _close(out, F.silu(a.float() @ w.float().t() + b + rv.float()[idx]), K, "linear+rowvec+silu")


@pytest.mark.parametrize("M,N", [(1000, 328), ("many", 512)])
def test_gn_stats_blocks(M, N):
    """every {sum, sumsq} block of 16 rows x 8 columns against torch's sums over the same rows of the fp32 result"""
    K = 256
    M = _rows(M, (N + 127) // 128)
    a, w = _rand(M, K), _rand(N, K, scale=0.05)
    b = torch.randn(N, device=DEV)
    res = _rand(M, N)
    out = ops.linear(a, w, b, residual=res, gn_stats=True)
    ref = a.float() @ w.float().t() + b + res.float()
    _close(out, ref, K, "linear+res+gn_stats")
    st = out.uav_gn[0]
    blocks = st.blocks
    assert blocks == (M + 127) // 128 * 8
    pad = torch.zeros(blocks * 16, N, device=DEV)
    pad[:M] = ref
    v = pad.view(blocks, 16, N // 8, 8)
    want = torch.stack([v.sum(dim=(1, 3)), (v * v).sum(dim=(1, 3))], dim=-1).permute(1, 0, 2)
    scale = torch.stack([v.abs().sum(dim=(1, 3)), (v * v).sum(dim=(1, 3))], dim=-1).permute(1, 0, 2)
    err = (st.partial - want).abs()
    bad = (err > 2e-3 * scale + 1e-2).sum().item()
    assert bad == 0, f"{bad}/{err.numel()} statistics blocks off, max err {err.max().item():.4g}"


def test_conv3x3_narrow_tiles():
    """a 3x3 convolution of 128 output channels with a residual: 128-column tiles, nine taps per tile"""
    NB, H, W, Cin, Cout = 6, 40, 72, 128, 128
    x, w = _rand(NB, H, W, Cin), _rand(Cout, 3, 3, Cin, scale=0.05)
    b = torch.randn(Cout, device=DEV)
    r = _rand(NB, H, W, Cout)
    out = ops.conv2d(x, w, b, residual=r)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), b, padding=1).permute(0, 2, 3, 1)
    _close(out, ref + r.float(), Cin * 9, "conv3x3 128->128 + res")


def test_repeat_launch_is_bitwise_equal():
    """the same launch twice gives the same output and the same statistics, bit for bit"""
    M, K, N = _rows("many", 4), 512, 512
    a, w = _rand(M, K), _rand(N, K, scale=0.05)
    b = torch.randn(N, device=DEV)
    res = _rand(M, N)
    y0 = ops.linear(a, w, b, residual=res, gn_stats=True)
    y1 = ops.linear(a, w, b, residual=res, gn_stats=True)
    assert torch.equal(y0, y1)
    assert torch.equal(y0.uav_gn[0].partial, y1.uav_gn[0].partial)
    z0, z1 = ops.linear(a, w, b), ops.linear(a, w, b)
    assert torch.equal(z0, z1)
