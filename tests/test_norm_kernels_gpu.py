"""Every normalisation kernel at the pipeline's own calls (tests/norm_cases.py PIPELINE_NORMS) against an fp64 reference,
with inputs whose statistics differ per group, slab, frame and token, so that a kernel using the wrong statistics, or
dropping part of them, moves outputs by O(1).  The producer-statistics path gets its data through a 1-tap temporal conv
with identity weights and `gn_stats=True`, whose fp16 output equals its input bit for bit.  Outputs start as NaN: every
element must be written and the padding beside a channel slice must keep its NaN.  A second launch must give the same
bits.  Where a clip's tensors would take more than the 8 GB the tests may use, it runs with fewer frames (printed)."""
import math

import pytest
import torch

import norm_cases as nc

pytestmark = pytest.mark.gpu
MEM_LIMIT = 8 * 2 ** 30   # peak extra device memory of one case
LIVE_BUDGET = 6 * 2 ** 30  # what the operands of one case may take (the fp64 reference chunks come on top)
NAN = float("nan")


@pytest.fixture(autouse=True, scope="module")
def _release_memory(uav_lib):
    yield
    import gc
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(autouse=True)
def _memory_bound():
    import gc
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    yield
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    assert peak < MEM_LIMIT, f"peak extra device memory {peak / 2 ** 30:.2f} GiB"


def _affine(C, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(C, device="cuda", generator=g) * 0.2 + 1, torch.randn(C, device="cuda", generator=g) * 0.1)


def _frames(call, bytes_per_frame):
    T = min(call.T, max(1, LIVE_BUDGET // bytes_per_frame))
    if T < call.T:
        print(f"\n[{call.name}] {T} of {call.T} frames (the whole clip exceeds the memory budget)")
    return T


def _identity_copy(x):
    """x (B, T, P, C) fp16 through a 1-tap temporal conv with identity weights, the statistics blocks requested: returns
    the conv's output, which carries them (`uav_gn`) and equals x bit for bit"""
    from upscale_a_video_b200 import ops
    B, T, P, C = x.shape
    w = torch.eye(C, dtype=torch.float16, device="cuda").view(C, 1, C).contiguous()
    y = ops.conv_temporal(x.view(B, T, P, 1, C), w, gn_stats=True)
    assert getattr(y, "uav_gn", None), "the producer did not emit statistics blocks"
    assert torch.equal(y.view(B, T, P, C), x)
    return y


def _report(call, gen, v, extra=""):
    print(f"\n[{call.name} {gen}] worst err/tol {v.worst:.3g}, {v.bad}/{v.n} out of bounds{extra}")
    assert v.bad == 0, f"{call.name} {gen}: {v.bad}/{v.n} elements out of bounds, worst err/tol {v.worst:.3g}"


GN_CASES = [(c, g) for c in nc.PIPELINE_NORMS if c.kind == "groupnorm" for g in nc.generators_for(c)]


@pytest.mark.parametrize("call,gen", GN_CASES, ids=[f"{c.name}-{g}" for c, g in GN_CASES])
def test_groupnorm(call, gen):
    from upscale_a_video_b200 import ops
    C, G, B = call.C, call.groups, call.B
    ld_in, ld_out = call.ld_in or C, call.ld_out or C
    T = _frames(call, 2 * B * call.HW * max(2 * ld_in, ld_in + ld_out))
    P = call.HW
    gamma, beta = _affine(C, 1)
    xbuf = torch.full((B, T, P, ld_in), NAN, dtype=torch.float16, device="cuda")
    x = nc.fill_groups(xbuf[..., :C], gen, G, seed=7, eps=call.eps)
    stats = None
    if call.source == "producer":
        y = _identity_copy(x)
        del x, xbuf
        x, stats = y.view(B, T, P, C), y.uav_gn
    n_outer = B * T if call.per_frame else B

    def launch():
        obuf = torch.full((B, T, P, ld_out), NAN, dtype=torch.float16, device="cuda")
        ops.group_norm(x, gamma, beta, G, call.eps, silu=call.silu, n_outer=n_outer, out=obuf[..., :C], stats=stats,
                       batch=B)
        return obuf

    out = launch()
    first = nc.fingerprint(out)
    if ld_out > C:
        assert out[..., C:].isnan().all(), "the kernel wrote beside its channel slice"
    xs = x.reshape(n_outer, -1, C) if ld_in == C else x.reshape(n_outer, -1, C).contiguous()
    v = nc.gn_verdict(out[..., :C].reshape(n_outer, -1, C), xs, nc.group_stats(xs, G), gamma, beta, call.eps, call.silu)
    del out
    assert nc.fingerprint(launch()) == first, "a second launch gave different bits"
    S = nc.split_count(n_outer, G, nc.producer_blocks_per_slab(call._replace(T=T))) if stats else 0
    _report(call, gen, v, f" (n_outer {n_outer}, {xs.shape[1]} px per slab" + (f", S = {S})" if S else ")"))


CAT_CASES = [(c, g) for c in nc.PIPELINE_NORMS if c.kind == "group_norm_cat" for g in nc.generators_for(c)]


@pytest.mark.parametrize("call,gen", CAT_CASES, ids=[f"{c.name}-{g}" for c, g in CAT_CASES])
def test_group_norm_cat(call, gen):
    from upscale_a_video_b200 import ops
    C, G, B, P = call.C, call.groups, call.B, call.HW
    T = _frames(call, 2 * 2 * B * P * C)
    gamma, beta = _affine(C, 2)
    parts, c0 = [], 0
    for i, cp in enumerate(call.parts):
        nb = 1 if (call.source == "concat_bcast" and i == len(call.parts) - 1) else B
        x0 = nc.fill_groups(torch.empty(nb, T, P, cp, dtype=torch.float16, device="cuda"), gen, G, seed=11 + i,
                            eps=call.eps, c0=c0, C_total=C)
        parts.append(_identity_copy(x0))
        del x0
        c0 += cp
    def launch():
        # the result is allocated inside group_norm_cat: hand it a block of NaN to be reused by the caching allocator
        tmp = torch.full((B, T, P, 1, C), NAN, dtype=torch.float16, device="cuda")
        ptr = tmp.data_ptr()
        del tmp
        out = ops.group_norm_cat(parts, gamma, beta, G, call.eps, silu=call.silu, n_outer=B)
        assert out is not None, "group_norm_cat refused parts that carry statistics"
        return out, out.data_ptr() == ptr

    first, ptr_reused = launch()
    fp_first = nc.fingerprint(first)
    # fp64 statistics of the virtual concatenation, from the parts (a batch-1 part serves every slab), in two passes
    st_parts = [p.view(p.shape[0], -1, p.shape[-1]) for p in parts]
    cpg, cnt = C // G, P * T * C // G
    s = torch.zeros(B, G, dtype=torch.float64, device="cuda")
    q = torch.zeros_like(s)
    for second in (False, True):
        c0 = 0
        for p in st_parts:
            cp = p.shape[-1]
            g_of = torch.arange(c0, c0 + cp, device="cuda") // cpg
            step = max(1, nc.CHUNK // (B * cp))
            for p0 in range(0, p.shape[1], step):
                xc = p[:, p0:p0 + step].double().expand(B, -1, -1)
                if second:
                    d = xc - mean[:, None, g_of]
                    q.index_add_(1, g_of, (d * d).sum(1))
                else:
                    s.index_add_(1, g_of, xc.sum(1))
            c0 += cp
        mean = s / cnt
    st = nc.Stats(mean, q / cnt)
    v = None
    out_v = first.view(B, -1, C)
    e_r, e_m = nc.stats_error(st.mean, st.var, call.eps)
    rstd = (st.var + call.eps).rsqrt()
    c0 = 0
    for p in st_parts:   # each part's channels against the statistics of the groups they belong to
        cp = p.shape[-1]
        sl = slice(c0, c0 + cp)
        g_of = torch.arange(c0, c0 + cp, device="cuda") // cpg
        step = max(1, nc.CHUNK // (B * cp))
        for p0 in range(0, p.shape[1], step):
            xh = (p[:, p0:p0 + step].double().expand(B, -1, -1) - st.mean[:, None, g_of]) * rstd[:, None, g_of]
            pre = xh * gamma[sl].double() + beta[sl].double()
            y = pre * torch.sigmoid(pre)
            tol = nc.tolerance(y, xh, gamma[sl].double(), e_r[:, None, g_of], e_m[:, None, g_of], rstd[:, None, g_of], True)
            v = nc.merge(v, nc.judge(out_v[:, p0:p0 + step, sl], y, tol))
        c0 += cp
    del first, out_v
    assert nc.fingerprint(launch()[0]) == fp_first, "a second launch gave different bits"
    _report(call, gen, v, f" ({'NaN-filled output' if ptr_reused else 'output block not reused: unwritten elements unchecked'})")


@pytest.mark.parametrize("gen", ["per_group", "offset16"])
def test_conv_out_fused_at_unet_output(gen):
    """GroupNorm + SiLU + conv_out in one kernel at the UNet output (2 x 8 x 320 x 576 x 256, statistics from the
    producer).  The conv has only its centre tap, so the output is a 256 -> 4 projection of the normalised tensor whose
    fp64 reference is cheap; every channel (and so every group) enters every output with weight +-1/16."""
    from upscale_a_video_b200 import ops
    call = next(c for c in nc.PIPELINE_NORMS if c.kind == "conv_out_fused")
    B, T, C, G, H, W, cout = call.B, call.T, call.C, call.groups, 320, 576, 4
    assert H * W == call.HW
    gamma, beta = _affine(C, 3)
    x0 = nc.fill_groups(torch.empty(B, T, H * W, C, dtype=torch.float16, device="cuda"), gen, G, seed=13)
    y = _identity_copy(x0)
    del x0
    x = y.view(B, T, H, W, C)
    x.uav_gn = stats = y.uav_gn
    gsign = torch.Generator(device="cuda").manual_seed(17)
    wc = (torch.randint(0, 2, (cout, C), generator=gsign, device="cuda").float() * 2 - 1) / 16
    w = torch.zeros(cout, 3, 3, C, dtype=torch.float16, device="cuda")
    w[:, 1, 1] = wc.half()
    bias = torch.linspace(-0.5, 0.5, cout, device="cuda")
    outs = []
    for _ in range(2):
        out = ops.conv_out_fused(x, gamma, beta, G, call.eps, w, bias, cout, torch.float32)
        outs.append(nc.fingerprint(out))
    assert outs[0] == outs[1], "a second launch gave different bits"
    xs = x.view(B, -1, C)
    st = nc.group_stats(xs, G)
    e_r, e_m = nc.stats_error(st.mean, st.var, call.eps)
    rstd = (st.var + call.eps).rsqrt()
    cpg = C // G
    per_c = lambda t: t.repeat_interleave(cpg, -1)[:, None, :]
    wd = wc.double()
    v = None
    step = max(1, nc.CHUNK // (B * C))
    o = out.permute(0, 2, 3, 4, 1).reshape(B, -1, cout)
    for p0 in range(0, xs.shape[1], step):
        y, xh, _ = nc.gn_apply_ref(xs[:, p0:p0 + step], st, gamma, beta, call.eps, True)
        tol_y = nc.tolerance(y, xh, gamma.double(), per_c(e_r), per_c(e_m), per_c(rstd), True)
        ref = y @ wd.t() + bias.double()
        tol = tol_y @ wd.abs().t() + nc.SAFETY * (C * nc.U32 * (y.abs() @ wd.abs().t()) + nc.U32 * ref.abs())
        v = nc.merge(v, nc.judge(o[:, p0:p0 + step], ref, tol))
    _report(call, gen, v, f" (statistics {'from the producer' if stats else 'by a read pass'})")


ROW_CASES = [(c, g) for c in nc.PIPELINE_NORMS if c.kind in ("layernorm", "rmsnorm") for g in nc.generators_for(c)]


@pytest.mark.parametrize("call,gen", ROW_CASES, ids=[f"{c.name}-{g}" for c, g in ROW_CASES])
def test_row_norm(call, gen):
    from upscale_a_video_b200 import ops
    C, rows = call.C, call.B * call.HW
    ld_out = call.ld_out or C
    x = nc.make_rows(gen, rows, C, seed=19, device="cuda", ld=call.ld_in or None)
    if call.kind == "layernorm":
        gamma, beta = _affine(C, 4)
    else:
        weight = (_affine(C, 4)[0]).half()
    outs = []
    for _ in range(2):
        obuf = torch.full((rows, ld_out), NAN, dtype=torch.float16, device="cuda")
        if call.kind == "layernorm":
            ops.layer_norm(x, gamma, beta, call.eps, out=obuf[:, :C])
        else:
            ops.rms_norm(x, weight, call.eps, out=obuf[:, :C])
        outs.append(nc.fingerprint(obuf))
        out = obuf
    assert outs[0] == outs[1], "a second launch gave different bits"
    if ld_out > C:
        assert out[:, C:].isnan().all(), "the kernel wrote beside its rows"
    v = None
    step = max(1, nc.CHUNK // C)
    for r0 in range(0, rows, step):
        xc = x[r0:r0 + step]
        if call.kind == "layernorm":
            ref, xh = nc.layer_norm_ref(xc, gamma, beta, call.eps)
            tol = nc.rows_tolerance(ref, xh, gamma, xc.double(), call.eps, C)
        else:
            ref, xr = nc.rms_norm_ref(xc, weight, call.eps)
            tol = nc.rms_tolerance(ref, xr, weight, C)
        v = nc.merge(v, nc.judge(out[r0:r0 + step, :C], ref, tol))
    _report(call, gen, v, f" ({rows} rows)")


IN_CASES = [(c, g) for c in nc.PIPELINE_NORMS if c.kind == "instnorm" for g in nc.generators_for(c)]


@pytest.mark.parametrize("call,gen", IN_CASES, ids=[f"{c.name}-{g}" for c, g in IN_CASES])
def test_instnorm(call, gen):
    from upscale_a_video_b200 import ops
    n, P, C = call.B, call.HW, call.C
    x = nc.fill_groups(torch.empty(n, 1, P, C, dtype=torch.float16, device="cuda"), gen, C, seed=23).view(n, P, 1, C)
    outs = []
    for _ in range(2):
        tmp = torch.full_like(x, NAN)
        ptr = tmp.data_ptr()
        del tmp
        y = ops.instnorm_relu(x, call.relu, call.eps)
        reused = y.data_ptr() == ptr
        outs.append(nc.fingerprint(y))
    assert outs[0] == outs[1], "a second launch gave different bits"
    xs = x.view(n, P, C)
    ones, zeros = torch.ones(C, device="cuda"), torch.zeros(C, device="cuda")
    v = nc.gn_verdict(y.view(n, P, C), xs, nc.group_stats(xs, C), ones, zeros, call.eps, "relu" if call.relu else False)
    _report(call, gen, v, " (NaN-filled output)" if reused else "")


@pytest.mark.parametrize("gen", nc.PLANE_GENERATORS)
def test_plane_stats(gen):
    from upscale_a_video_b200 import ops
    call = next(c for c in nc.PIPELINE_NORMS if c.kind == "plane_stats")
    x = nc.make_planes(gen, call.B, call.C, 1280, 2304, seed=29, device="cuda")
    m1, s1 = ops.plane_stats(x, call.eps)
    m2, s2 = ops.plane_stats(x, call.eps)
    assert torch.equal(m1, m2) and torch.equal(s1, s2), "a second launch gave different bits"
    m, s, var = nc.plane_stats_ref(x, call.eps)
    n = x[0, 0].numel()
    U64 = 2.0 ** -53
    e_sum = 64 * math.sqrt(n) * U64
    ma = x.double().abs().flatten(2).mean(-1)
    tol_m = nc.SAFETY * (nc.U32 * m.abs() + e_sum * ma)
    e_var = e_sum * (m * m + var) * 4
    tol_s = nc.SAFETY * (2 * nc.U32 * s + e_var / (2 * s))
    vm = nc.judge(m1.view_as(m), m, tol_m)
    vs = nc.judge(s1.view_as(s), s, tol_s)
    _report(call, gen, nc.merge(vm, vs), f" (mean {vm.worst:.3g}, std {vs.worst:.3g})")
