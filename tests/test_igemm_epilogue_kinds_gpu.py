"""GPU checks of the implicit GEMM's specialised AUX epilogue bodies (csrc/igemm.cu, epilogue_kind): each feature set
that has a body of its own (row vector + statistics, residual + statistics, residual, statistics, out_scale, and the
residual with out_scale that shares the residual bodies) and the generic body that runs every other combination.

Each case runs at 64-, 128- or 256-column tiles (GEGLU only on the generic body), with ragged M or a ragged last N tile,
and most on launches where every persistent CTA runs at least three tiles.  One Linear has 7360 rows per row vector, so
some of its 128-row tiles straddle two row vectors.  Every case is checked against fp32 PyTorch with the tolerance of
test_igemm_epilogue_gpu.py, its statistics blocks against torch's sums, and bit for bit against itself run twice and
against the generic body: a bias that is not 8-byte aligned sends the same launch to the generic body, which must give
the same outputs and statistics.  One profiler trace pins the kernel instance each case runs on."""
import json
import math
import os
import re
import subprocess
import sys

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
    err = (got.float() - ref).abs()
    tol = 1e-3 * ref.abs() + 2e-3 * math.sqrt(K) * 0.02 + 1e-3
    bad = (err > tol).sum().item()
    assert bad == 0, f"{what}: {bad}/{err.numel()} mismatches, max err {err.max().item():.4g}"


def _check_blocks(st, ref, what):
    """ref: (rows, n_out) fp32 in the launch's row order, 128-row M-tiles of 8 blocks of 16 rows"""
    M, N = ref.shape
    blocks = st.blocks
    assert blocks == (M + 127) // 128 * 8
    pad = torch.zeros(blocks * 16, N, device=DEV)
    pad[:M] = ref
    v = pad.view(blocks, 16, N // 8, 8)
    want = torch.stack([v.sum(dim=(1, 3)), (v * v).sum(dim=(1, 3))], dim=-1).permute(1, 0, 2)
    scale = torch.stack([v.abs().sum(dim=(1, 3)), (v * v).sum(dim=(1, 3))], dim=-1).permute(1, 0, 2)
    err = (st.partial - want).abs()
    bad = (err > 2e-3 * scale + 1e-2).sum().item()
    assert bad == 0, f"{what}: {bad}/{err.numel()} statistics blocks off, max err {err.max().item():.4g}"


def _many(n_tiles_per_m):
    """rows such that every persistent CTA runs at least three tiles, the last M-tile ragged"""
    return 128 * ((3 * _sms() + n_tiles_per_m - 1) // n_tiles_per_m + 1) - 5


# name: (op, rows or "many" / conv (NB, H), K, N, features, BLOCK_N of the instance, GEGLU)
# Convolutions are 3x3 on W = 256 images, so every M-tile is one 128-pixel run of an image row and the statistics
# blocks follow the pixel order; NB x H = 330 gives 660 M-tiles, enough waves for 256-column tiles at N >= 256.
CASES = {
    # row vector + statistics
    "linear_rowvec_stats_straddle": ("linear", 6 * 7360, 256, 256, dict(rowvec=7360, stats=True), 128, False),
    "linear_rowvec_stats_n64": ("linear", "many", 128, 64, dict(rowvec="many", stats=True), 64, False),
    "conv_rowvec_stats_n256": ("conv", (6, 55), 64, 256, dict(rowvec=2, stats=True), 256, False),
    # residual + statistics (and with out_scale, the same body)
    "linear_res_stats_n200": ("linear", 1000, 256, 200, dict(res=True, stats=True), 128, False),
    "linear_res_stats_n64": ("linear", 777, 256, 64, dict(res=True, stats=True), 64, False),
    "conv_res_stats_n456": ("conv", (6, 55), 64, 456, dict(res=True, stats=True), 256, False),
    "conv_res_scale_stats_n456": ("conv", (6, 55), 64, 456, dict(res=True, scale=0.25, stats=True), 256, False),
    # residual (and with out_scale)
    "linear_res_many": ("linear", "many", 512, 512, dict(res=True), 128, False),
    "linear_res_scale_n200": ("linear", 1000, 320, 200, dict(res=True, scale=0.5), 128, False),
    "linear_res_n40": ("linear", "many", 64, 40, dict(res=True), 64, False),
    "conv_res_n456": ("conv", (6, 55), 64, 456, dict(res=True), 256, False),
    # statistics
    "linear_stats_nobias_n200": ("linear", "many", 256, 200, dict(stats=True, bias=False), 128, False),
    "linear_stats_n64": ("linear", 1000, 256, 64, dict(stats=True), 64, False),
    "conv_stats_n456": ("conv", (6, 55), 64, 456, dict(stats=True), 256, False),
    # out_scale
    "linear_scale_n200": ("linear", "many", 256, 200, dict(scale=0.125), 128, False),
    "linear_scale_n40": ("linear", 1000, 256, 40, dict(scale=0.125), 64, False),
    "conv_scale_n456": ("conv", (6, 55), 64, 456, dict(scale=0.125), 256, False),
    # generic body: an activation, a row vector without statistics, GEGLU
    "generic_linear_rowvec_silu_n200": ("linear", "many", 256, 200, dict(rowvec=7360, act=ops.ACT_SILU), 128, False),
    "generic_linear_rowvec_res_stats": ("linear", 1000, 256, 128, dict(rowvec=300, res=True, stats=True), 128, False),
    "generic_conv_rowvec_n456": ("conv", (6, 55), 64, 456, dict(rowvec=3), 256, False),
    "generic_geglu128_res": ("linear", 1000, 256, 128, dict(res=True, act=ops.ACT_GEGLU), 128, True),
    "generic_geglu256_res": ("linear", 660 * 128 - 5, 256, 512, dict(res=True, act=ops.ACT_GEGLU), 256, True),
}


def _inputs(case):
    op, M, K, N, f, _, _ = case
    act = f.get("act", ops.ACT_NONE)
    n_out = N // 2 if act == ops.ACT_GEGLU else N
    rnd = _rand
    if op == "linear":
        rows = _many((n_out + 127) // 128) if M == "many" else M
        x, w = rnd(rows, K), rnd(N, K, scale=0.05)
        lead = (rows,)
    else:
        NB, H = M
        rows = NB * H * 256
        x, w = rnd(NB, H, 256, K), rnd(N, 3, 3, K, scale=0.05)
        lead = (NB, H, 256)
    bias = torch.randn(N, device=DEV) if f.get("bias", True) else None
    rv = rpv = None
    if "rowvec" in f:
        rpv = f["rowvec"] if op == "linear" else f["rowvec"] * M[1] * 256  # conv: images per row vector
        if rpv == "many":
            rpv = rows // 3 + 1
        rv = rnd((rows + rpv - 1) // rpv, n_out)
    res = rnd(*lead, n_out) if f.get("res") else None
    return x, w, bias, rv, rpv, res, rows, n_out


def _launch(case, x, w, bias, rv, rpv, res):
    op, _, _, _, f, _, _ = case
    kw = dict(residual=res, rowvec=rv, rows_per_vec=rpv or 0, act=f.get("act", ops.ACT_NONE),
              out_scale=f.get("scale", 1.0), gn_stats=f.get("stats", False))
    if op == "linear":
        return ops.linear(x, w, bias, **kw)
    return ops.conv2d(x, w, bias, **kw)


def _misaligned(bias):
    """the same values at an address that is 4 but not 8 bytes aligned"""
    if bias is None:
        return None
    buf = torch.empty(bias.numel() + 1, device=DEV)
    b = buf[1:]
    b.copy_(bias)
    assert b.data_ptr() % 8 == 4
    return b


def _reference(case, x, w, bias, rv, rpv, res, rows, n_out):
    op, _, K, N, f, _, _ = case
    if op == "linear":
        y = x.float() @ w.float().t()
    else:
        y = F.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), padding=1).permute(0, 2, 3, 1)
    y = y.reshape(rows, N)
    if bias is not None:
        y = y + bias
    act = f.get("act", ops.ACT_NONE)
    if act == ops.ACT_GEGLU:
        y = y[:, :n_out] * F.gelu(y[:, n_out:])
    if rv is not None:
        y = y + rv.float()[torch.arange(rows, device=DEV) // rpv]
    if act == ops.ACT_SILU:
        y = F.silu(y)
    y = y * f.get("scale", 1.0)
    if res is not None:
        y = y + res.float().reshape(rows, n_out)
    return y, (K if op == "linear" else 9 * K)


@pytest.mark.parametrize("name", list(CASES))
def test_epilogue_kind(name):
    case = CASES[name]
    x, w, bias, rv, rpv, res, rows, n_out = _inputs(case)
    out = _launch(case, x, w, bias, rv, rpv, res)
    ref, k_eff = _reference(case, x, w, bias, rv, rpv, res, rows, n_out)
    _close(out.reshape(rows, n_out), ref, k_eff, name)
    stats = case[4].get("stats", False)
    if stats:
        _check_blocks(out.uav_gn[0], ref, name)
    again = _launch(case, x, w, bias, rv, rpv, res)
    assert torch.equal(out, again), f"{name}: a second launch differs"
    generic = _launch(case, x, w, _misaligned(bias), rv, rpv, res)
    assert torch.equal(out, generic), f"{name}: differs from the generic body"
    if stats:
        assert torch.equal(out.uav_gn[0].partial, again.uav_gn[0].partial), f"{name}: statistics of a second launch"
        assert torch.equal(out.uav_gn[0].partial, generic.uav_gn[0].partial), f"{name}: statistics of the generic body"


def _instances_trace():
    """(BLOCK_N, GEGLU, TMA_EPI, AUX) of the igemm_kernel launches of all cases, in launch order, from one
    torch.profiler session; the kernels are loaded before the session"""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    inputs = {name: _inputs(case) for name, case in CASES.items()}
    for name, case in CASES.items():
        _launch(case, *inputs[name][:6])
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for name, case in CASES.items():
            _launch(case, *inputs[name][:6])
        torch.cuda.synchronize()
    got = []
    for e in sorted((e for e in prof.events() if e.device_type == DeviceType.CUDA and "igemm_kernel" in e.name),
                    key=lambda e: e.time_range.start):
        m = re.search(r"igemm_kernel<(\d+), (true|false), (true|false), (true|false)>", e.name)
        assert m, e.name
        got.append([int(m.group(1)), m.group(2) == "true", m.group(3) == "true", m.group(4) == "true"])
    return got


def test_epilogue_kind_instances():
    """each case launches once, on the TMA-store AUX instance of its tile width.  The trace is taken in a fresh
    interpreter: once the profiler has been used in a process, kernels whose modules load later in that process can be
    missing from its later traces, which would take the kernel-selection checks of other test files with them."""
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.dirname(here), here, os.environ.get("PYTHONPATH", "")]))
    r = subprocess.run([sys.executable, "-c", f"import json, {__name__} as t; print(json.dumps(t._instances_trace()))"],
                       cwd=os.path.dirname(here), env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    got = [tuple(g) for g in json.loads(r.stdout.strip().splitlines()[-1])]
    want = [(case[5], case[6], True, True) for case in CASES.values()]
    assert got == want, [(name, g, w) for name, g, w in zip(CASES, got, want) if g != w] or (len(got), len(want))
