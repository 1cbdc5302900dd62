"""GPU checks of the implicit GEMM's GroupNorm statistics, which the epilogue reduces over each warp's 16 rows with one
transposing warp reduction per pass (csrc/igemm.cu, warp_sum_transpose): every {sum, sumsq} block against torch's sums
at 64-, 128- and 256-column tiles, including ragged M and N, and the same launch run twice bitwise equal."""
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


def _rand(*shape, scale=1.0):
    return (torch.randn(*shape, device=DEV) * scale).half()


def _close(got, ref, K, what):
    err = (got.float() - ref).abs()
    tol = 1e-3 * ref.abs() + 2e-3 * math.sqrt(K) * 0.02 + 1e-3
    bad = (err > tol).sum().item()
    assert bad == 0, f"{what}: {bad}/{err.numel()} mismatches, max err {err.max().item():.4g}"


def _check_blocks(st, ref):
    """ref: (rows, n_out) fp32 in the launch's row order, 128-row M-tiles of 8 blocks of 16 rows"""
    M, N = ref.shape
    blocks = st.blocks
    assert blocks == (M + 127) // 128 * 8
    pad = torch.zeros(blocks * 16, N, device=DEV)
    pad[:M] = ref
    v = pad.view(blocks, 16, N // 8, 8)
    want = torch.stack([v.sum(dim=(1, 3)), (v * v).sum(dim=(1, 3))], dim=-1).permute(1, 0, 2)
    scale = torch.stack([v.abs().sum(dim=(1, 3)), (v * v).sum(dim=(1, 3))], dim=-1).permute(1, 0, 2)
    assert st.partial.shape == want.shape
    err = (st.partial - want).abs()
    bad = (err > 2e-3 * scale + 1e-2).sum().item()
    assert bad == 0, f"{bad}/{err.numel()} statistics blocks off, max err {err.max().item():.4g}"


@pytest.mark.parametrize("M,N,residual", [
    (1000, 64, False),  # 64-column tile: two lanes per statistics value
    (777, 64, True),
    (1000, 200, True),  # 128 + 72 columns
    (4000, 512, False),
])
def test_linear_stats_blocks(M, N, residual):
    K = 256
    a, w = _rand(M, K), _rand(N, K, scale=0.05)
    b = torch.randn(N, device=DEV)
    res = _rand(M, N) if residual else None
    out = ops.linear(a, w, b, residual=res, gn_stats=True)
    ref = a.float() @ w.float().t() + b + (res.float() if residual else 0.0)
    _close(out, ref, K, f"linear {M}x{K}x{N} gn_stats")
    _check_blocks(out.uav_gn[0], ref)


@pytest.mark.parametrize("Cout,residual", [
    (256, False),  # many waves: 256-column tiles, two epilogue passes per tile
    (256, True),
    (264, False),  # three 128-column tiles, the last one with 8 valid columns
])
def test_conv3x3_stats_blocks(Cout, residual):
    """W = 256 makes every M-tile one 128-pixel run of an image row, so the blocks follow the pixel order"""
    NB, H, W, Cin = 8, 40, 256, 64
    x, w = _rand(NB, H, W, Cin), _rand(Cout, 3, 3, Cin, scale=0.05)
    b = torch.randn(Cout, device=DEV)
    r = _rand(NB, H, W, Cout) if residual else None
    out = ops.conv2d(x, w, b, residual=r, gn_stats=True)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), b, padding=1).permute(0, 2, 3, 1)
    if residual:
        ref = ref + r.float()
    _close(out, ref, Cin * 9, f"conv3x3 {Cin}->{Cout} gn_stats")
    _check_blocks(out.uav_gn[0], ref.reshape(-1, Cout))


def test_stats_repeat_launch_is_bitwise_equal():
    """the same statistics-bearing launches twice give the same outputs and statistics, bit for bit"""
    a, w = _rand(5000, 512), _rand(512, 512, scale=0.05)
    res = _rand(5000, 512)
    x, wc = _rand(8, 40, 256, 64), _rand(256, 3, 3, 64, scale=0.05)
    for launch in (lambda: ops.linear(a, w, None, residual=res, out_scale=0.5, gn_stats=True),
                   lambda: ops.conv2d(x, wc, None, gn_stats=True)):
        y0, y1 = launch(), launch()
        assert torch.equal(y0, y1)
        assert torch.equal(y0.uav_gn[0].partial, y1.uav_gn[0].partial)
