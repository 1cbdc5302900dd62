"""CPU checks of tests/norm_cases.py: its fp64 references equal torch's, its pass criterion rejects the faults the GPU
tests are built to catch (on a CPU emulator of the kernels' blocking: per-block partials with a ragged grid-stride
tail, the GEMM epilogue's 16-row x 8-channel statistics blocks reduced in S splits, the per-source apply at a channel
offset, a batch-1 skip serving every batch item, U tokens per warp), and `PIPELINE_NORMS` covers every normalisation
call the pipeline's modules make."""
import collections
import json
import math
import os

import pytest
import torch
import torch.nn.functional as F

import emu_ops
import norm_cases as nc

G_DIR = os.path.join(os.path.dirname(__file__), "golden")
CFG = os.path.join(os.path.dirname(__file__), "..", "upscale_a_video_b200", "configs")


# ---------------------------------------------------------------------------------------------------------------------
# 1. the references
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gen", nc.GN_GENERATORS)
def test_group_norm_reference_matches_torch(gen):
    N, T, P, C, G = 2, 3, 50, 96, 32
    x = nc.fill_groups(torch.empty(N, T, P, C, dtype=torch.float16), gen, G, seed=1, eps=nc.EPS_SCALED)
    g, b = torch.randn(C, dtype=torch.float64), torch.randn(C, dtype=torch.float64)
    eps = nc.EPS_SCALED if gen == "scaled" else 1e-5
    for per_frame in (False, True):
        xs = x.reshape(N * T if per_frame else N, -1, C)
        ref = nc.gn_reference(xs, G, g, b, eps, True)
        tr = F.silu(F.group_norm(xs.double().transpose(1, 2), G, g, b, eps)).transpose(1, 2)
        assert torch.allclose(ref, tr, rtol=1e-10, atol=1e-10)
        # chunked statistics equal the one-piece ones
        st = nc.group_stats(xs, G)
        assert torch.allclose(st.var, xs.double().reshape(xs.shape[0], -1, G, C // G).transpose(1, 2)
                              .reshape(xs.shape[0], G, -1).var(-1, unbiased=False), rtol=1e-10, atol=1e-30)


def test_scaled_generator_has_constant_and_near_constant_groups():
    x = nc.fill_groups(torch.empty(1, 3, 400, 64, dtype=torch.float16), "scaled", 32, seed=2, eps=nc.EPS_SCALED)
    st = nc.group_stats(x.reshape(1, -1, 64), 32)
    assert (st.var[0, 6::8] == 0).all()                                      # exactly constant: eps alone
    assert ((st.var[0, 3::8] > 0.2 * nc.EPS_SCALED) & (st.var[0, 3::8] < 5 * nc.EPS_SCALED)).all()  # eps governs
    from upscale_a_video_b200 import autoencoder_kl_cond_video as A
    assert A.VAE_STREAM_SCALE == nc.VAE_STREAM_SCALE


def test_row_and_instance_and_plane_references_match_torch():
    x = nc.make_rows("rows", 37, 64, seed=3)
    g, b = torch.randn(64, dtype=torch.float64), torch.randn(64, dtype=torch.float64)
    assert torch.allclose(nc.layer_norm_ref(x, g, b, 1e-5)[0], F.layer_norm(x.double(), (64,), g, b, 1e-5), atol=1e-10)
    w = torch.randn(64, dtype=torch.float64)
    assert torch.allclose(nc.rms_norm_ref(x, w, 1e-5)[0], F.rms_norm(x.double(), (64,), w, 1e-5), atol=1e-10)
    xi = nc.fill_groups(torch.empty(3, 1, 70, 32, dtype=torch.float16), "per_group", 32, seed=4).reshape(3, 7, 10, 32)
    y = nc.instance_norm_ref(xi, 1e-5, False)[0]
    tr = F.instance_norm(xi.double().permute(0, 3, 1, 2), eps=1e-5).permute(0, 2, 3, 1)
    assert torch.allclose(y, tr, atol=1e-10)
    for gen in nc.PLANE_GENERATORS:
        p = nc.make_planes(gen, 2, 3, 9, 11, seed=5)
        m, s, _ = nc.plane_stats_ref(p, 1e-5)
        v = p.double().flatten(2)
        assert torch.allclose(m, v.mean(-1), atol=1e-14) and torch.allclose(s, (v.var(-1) + 1e-5).sqrt(), rtol=1e-12)


def test_criterion_is_never_looser_than_the_old_band():
    y = torch.linspace(-8, 8, 101, dtype=torch.float64)
    tol = nc.tolerance(y, y, torch.ones(1, dtype=torch.float64), 1.0, 1.0, 1.0, True)
    assert (tol <= nc.LEGACY_ATOL + nc.LEGACY_RTOL * y.abs()).all()


# ---------------------------------------------------------------------------------------------------------------------
# 2. a CPU emulator of the kernels' blocking, and the faults the criterion must reject
# ---------------------------------------------------------------------------------------------------------------------
def _own_sums(xs, G, nb, drop_tail):
    """norm.cu gn_stats_kernel: block b of nb adds pixels b, b + nb, ... 4 strides at a time, then the ragged tail;
    returns fp64 (slabs, G, 2) sums of the per-block partials in block order"""
    S_, P, C = xs.shape
    cpg = C // G
    out = torch.zeros(S_, G, 2, dtype=torch.float64)
    for b in range(nb):
        p = b
        idx = []
        while p + 3 * nb < P:
            idx += [p, p + nb, p + 2 * nb, p + 3 * nb]
            p += 4 * nb
        if not drop_tail:
            idx += list(range(p, P, nb))
        v = xs[:, idx].reshape(S_, len(idx), G, cpg)
        out[..., 0] += v.sum((1, 3))
        out[..., 1] += (v * v).sum((1, 3))
    return out


def _producer_sums(part, oct0, G, cpg, S, fault):
    """the statistics blocks of one concat part (slabs, P, Cp): 16 rows x 8 channels each, reduced per group in S splits
    of the slab's blocks (norm.cu gn_reduce_partials_kernel) -> (slabs, G, S, 2)"""
    n_sl, P, Cp = part.shape
    bps = -(-P // 16)
    sums = torch.zeros(n_sl, G, S, 2, dtype=torch.float64)
    for o in range(Cp // 8):
        g = (oct0 + o) * 8 // cpg
        blk = part[:, :, o * 8:(o + 1) * 8]
        for sp in range(S):
            if fault == "split_drop" and sp == S - 1 and S > 1:
                continue
            for k in range(bps * sp // S, bps * (sp + 1) // S):
                v = blk[:, 16 * k:16 * (k + 1)]
                reps = 2 if fault == "block_twice" and k == 0 and o == 0 else 1
                sums[:, g, sp, 0] += reps * v.sum((1, 2))
                sums[:, g, sp, 1] += reps * (v * v).sum((1, 2))
    return sums


def emulate_groupnorm(parts, G, eps, gamma, beta, silu, *, per_frame, source, fault=None, nb=7, S=3):
    """GroupNorm(+SiLU) of torch.cat(parts, -1) as the kernels block it, in fp64.  parts: (Nk, T, P, Ck) with Nk = N or 1
    (a batch-1 part serves every batch item: concat sources only).  Returns (N, T, P, C) with NaN where nothing was
    written."""
    N = max(p.shape[0] for p in parts)
    _, T, P, _ = parts[0].shape
    C = sum(p.shape[-1] for p in parts)
    cpg = C // G
    if fault == "eps_unscaled":
        eps = eps / nc.VAE_STREAM_SCALE ** 2
    stat_frame = per_frame != (fault in ("clip_for_frame", "frame_for_clip"))  # the slabs statistics are taken over

    def slabs(p, frame):
        return p.reshape(p.shape[0] * p.shape[1], P, -1) if frame else p.reshape(p.shape[0], p.shape[1] * P, -1)

    if source == "own":
        full = torch.cat([p.expand(N, *p.shape[1:]) for p in parts], -1)
        if fault == "frame_for_clip":
            full = full[:, :1]  # per-frame statistics: those of the clip's first frame
        sums = _own_sums(slabs(full, stat_frame), G, nb, fault == "tail")[:, :, None]
        cnt = (P if stat_frame else T * P) * cpg
        bsl = [1] * len(parts)
    else:
        sums, oct0 = 0, 0
        bsl = [1 if p.shape[0] == N else 0 for p in parts]   # slab_mul: 0 = every n reads the same blocks
        if fault == "bcast_wrong_slab":
            bsl = [0] * len(parts)
        for p, mul in zip(parts, bsl):
            s = _producer_sums(slabs(p, stat_frame), oct0, G, cpg, S, fault)
            n_sl = N * T if stat_frame else N
            sums = sums + (s if mul and s.shape[0] == n_sl else s[:1].expand(n_sl, *s.shape[1:]))
            oct0 += p.shape[-1] // 8
        cnt = (P if stat_frame else T * P) * cpg
    s, q = sums[..., 0].sum(-1), sums[..., 1].sum(-1)       # (slabs, G): the S splits in order
    mean = s / cnt
    rstd = ((q / cnt - mean * mean).clamp_min(0) + eps).rsqrt()
    n_sl = mean.shape[0]
    if per_frame and not stat_frame:          # clip_for_frame: frame slab (n, t) reads clip n
        mean, rstd = mean.repeat_interleave(T, 0), rstd.repeat_interleave(T, 0)
    n_out = N * T if per_frame else N
    if fault == "slab_prev":
        perm = [(n - 1) % n_out for n in range(n_out)]
        mean, rstd = mean[perm], rstd[perm]
    if fault == "slab0":
        mean, rstd = mean[:1].expand(n_out, -1), rstd[:1].expand(n_out, -1)
    y = torch.full((n_out, (P if per_frame else T * P), C), math.nan, dtype=torch.float64)
    chan = 0
    for i, p in enumerate(parts):
        Cp = p.shape[-1]
        off = chan + (8 if fault == "concat_plus8" and i == 1 else -8 if fault == "concat_minus8" and i == 1 else 0)
        cs = torch.arange(off, off + Cp)
        keep = (cs >= 0) & (cs < C)
        cs = cs[keep]
        grp = cs // cpg
        if fault == "neighbour":
            grp = (grp + 1) % G
        xv = slabs(p.expand(N, *p.shape[1:]), per_frame)[..., keep]
        pre = (xv - mean[:, None, grp]) * rstd[:, None, grp] * gamma[cs] + beta[cs]
        y[..., cs] = pre * torch.sigmoid(pre) if silu else pre
        chan += Cp
    return y.reshape(N, T, P, C)


def _gn_case(gen, per_frame, source, *, parts=(64,), G=8, eps=1e-5, bcast=False, N=3, T=3, P=40, seed=0):
    eps = nc.EPS_SCALED if gen == "scaled" else eps
    C = sum(parts)
    full = nc.fill_groups(torch.empty(N, T, P, C, dtype=torch.float16), gen, G, seed, eps).double()
    xs, c0 = [], 0
    for i, cp in enumerate(parts):
        x = full[..., c0:c0 + cp]
        xs.append(x[:1] if bcast and i == 1 else x)
        c0 += cp
    g = torch.randn(C, dtype=torch.float64, generator=torch.Generator().manual_seed(seed)) * 0.2 + 1
    b = torch.randn(C, dtype=torch.float64, generator=torch.Generator().manual_seed(seed + 1)) * 0.1
    ref_x = torch.cat([x.expand(N, *x.shape[1:]) for x in xs], -1)
    return xs, ref_x, g, b, eps


def _gn_judge(y, ref_x, G, g, b, eps, per_frame, silu=True):
    N, T, P, C = ref_x.shape
    xs = ref_x.reshape(N * T if per_frame else N, -1, C)
    return nc.gn_verdict(y.reshape(xs.shape), xs, nc.group_stats(xs, G), g, b, eps, silu)


# the call each fault needs (source, per_frame, parts, broadcast skip) and the generator it shows up under
GN_FAULTS = {
    "neighbour": ("per_group", "own", False, (64,), False),
    "slab_prev": ("per_group", "producer", False, (64,), False),
    "slab0": ("per_group", "own", True, (64,), False),
    "clip_for_frame": ("per_frame", "producer", True, (64,), False),
    "frame_for_clip": ("per_frame", "own", False, (64,), False),
    "tail": ("per_frame", "own", False, (64,), False),
    "split_drop": ("offset16", "producer", False, (64,), False),
    "block_twice": ("offset16", "producer", False, (64,), False),
    "concat_plus8": ("per_group", "concat", False, (40, 32), False),
    "concat_minus8": ("per_group", "concat", False, (40, 32), False),
    "bcast_wrong_slab": ("per_group", "concat", False, (40, 32), True),
    "eps_unscaled": ("scaled", "own", False, (64,), False),
}


@pytest.mark.parametrize("source,per_frame,parts,bcast", [("own", False, (64,), False), ("own", True, (64,), False),
                                                          ("producer", False, (64,), False), ("producer", True, (64,), False),
                                                          ("concat", False, (40, 32), False),
                                                          ("concat", False, (40, 32), True)])
@pytest.mark.parametrize("gen", nc.GN_GENERATORS)
def test_emulator_without_faults_passes(gen, source, per_frame, parts, bcast):
    G = 3 if parts != (64,) else 8   # 72 channels in 3 groups of 24: groups straddle octets and the concat boundary
    xs, ref_x, g, b, eps = _gn_case(gen, per_frame, source, parts=parts, G=G, bcast=bcast)
    y = emulate_groupnorm(xs, G, eps, g, b, True, per_frame=per_frame, source="own" if source == "own" else "producer")
    v = _gn_judge(y, ref_x, G, g, b, eps, per_frame)
    assert v.bad == 0, v


@pytest.mark.parametrize("fault", sorted(GN_FAULTS))
def test_emulated_fault_is_rejected(fault):
    gen, source, per_frame, parts, bcast = GN_FAULTS[fault]
    G = 3 if parts != (64,) else 8
    xs, ref_x, g, b, eps = _gn_case(gen, per_frame, source, parts=parts, G=G, bcast=bcast)
    src = "own" if source == "own" else "producer"
    clean = _gn_judge(emulate_groupnorm(xs, G, eps, g, b, True, per_frame=per_frame, source=src), ref_x, G, g, b, eps,
                      per_frame)
    v = _gn_judge(emulate_groupnorm(xs, G, eps, g, b, True, per_frame=per_frame, source=src, fault=fault), ref_x, G, g, b,
                  eps, per_frame)
    print(f"\n[fault {fault} on {gen}] {v.bad}/{v.n} out of bounds, worst err/tol {v.worst:.3g} (no fault: {clean.worst:.3g})")
    assert clean.bad == 0 and v.bad > 0 and v.worst >= 10


def emulate_layernorm(x, gamma, beta, eps, nwarps=4, U=2, fault=None):
    """layernorm_kernel: warp w handles tokens row0 + u * nwarps, u < U, of each step; fault token_prev: token u uses the
    statistics of the token before it in flight"""
    xd = x.double()
    m = xd.mean(-1)
    v = ((xd - m[:, None]) ** 2).mean(-1)
    idx = torch.arange(x.shape[0])
    if fault == "token_prev":
        u = (idx // nwarps) % U
        idx = torch.where(u > 0, idx - nwarps, idx)
    return (xd - m[idx, None]) * (v[idx, None] + eps).rsqrt() * gamma + beta


@pytest.mark.parametrize("fault", [None, "token_prev"])
def test_emulated_token_fault(fault):
    x = nc.make_rows("rows", 64, 64, seed=6)
    g = torch.randn(64, dtype=torch.float64) * 0.2 + 1
    b = torch.randn(64, dtype=torch.float64) * 0.1
    ref, xh = nc.layer_norm_ref(x, g, b, 1e-5)
    v = nc.judge(emulate_layernorm(x, g, b, 1e-5, fault=fault), ref, nc.rows_tolerance(ref, xh, g, x.double(), 1e-5, 64))
    print(f"\n[layernorm fault {fault}] {v.bad}/{v.n} out of bounds, worst err/tol {v.worst:.3g}")
    assert (v.bad == 0) if fault is None else (v.bad > 0 and v.worst >= 10)


# ---------------------------------------------------------------------------------------------------------------------
# 3. PIPELINE_NORMS covers the calls the modules make
# ---------------------------------------------------------------------------------------------------------------------
def _signature(c: nc.NormCall):
    return (c.kind, c.C, c.groups, float(c.eps), c.per_frame, c.source)


def test_pipeline_norms_table_is_consistent():
    names = [c.name for c in nc.PIPELINE_NORMS]
    assert len(names) == len(set(names))
    for c in nc.PIPELINE_NORMS:
        if c.groups:
            assert c.C % c.groups == 0 and sum(c.parts or (c.C,)) == c.C
            assert (c.source in ("concat", "concat_bcast")) == bool(c.parts)
            if c.source != "own":
                assert c.cpg % 8 == 0
        assert nc.generators_for(c)
    kinds = {c.kind for c in nc.PIPELINE_NORMS}
    assert kinds == {"groupnorm", "group_norm_cat", "conv_out_fused", "layernorm", "rmsnorm", "instnorm", "plane_stats"}
    assert {c.cpg for c in nc.PIPELINE_NORMS if c.kind == "group_norm_cat"} >= {24, 48, 64}
    assert max(c.pixels for c in nc.PIPELINE_NORMS if c.groups) == 3 * 1280 * 2304


class _Recorder:
    """emu_ops with the normalisation wrappers recording the signature of every call"""

    def __init__(self):
        self.calls = collections.Counter()
        for n in dir(emu_ops):
            if not n.startswith("_"):
                setattr(self, n, getattr(emu_ops, n))
        self.group_norm, self.group_norm_cat = self._gn, self._gn_cat
        self.layer_norm, self.conv_out_fused = self._ln, self._cof

    def _gn(self, x, gamma, beta, groups, eps, *, silu, n_outer, out=None, stats=None, batch=None):
        src = "producer" if stats and (x.shape[-1] // groups) % 8 == 0 else "own"  # as ops._gn_sources decides
        self.calls[("groupnorm", x.shape[-1], groups, float(eps), n_outer != x.shape[0], src)] += 1
        return emu_ops.group_norm(x, gamma, beta, groups, eps, silu=silu, n_outer=n_outer, out=out)

    def _gn_cat(self, parts, gamma, beta, groups, eps, *, silu, n_outer):
        src = "concat" if all(p.shape[0] == parts[0].shape[0] for p in parts) else "concat_bcast"
        self.calls[("group_norm_cat", sum(p.shape[-1] for p in parts), groups, float(eps), False, src)] += 1
        return emu_ops.group_norm_cat(parts, gamma, beta, groups, eps, silu=silu, n_outer=n_outer)

    def _ln(self, x, gamma, beta, eps=1e-5, out=None):
        self.calls[("layernorm", x.shape[-1], 0, float(eps), False, "own")] += 1
        return emu_ops.layer_norm(x, gamma, beta, eps, out)

    def _cof(self, x, gamma, beta, groups, eps, *a, **k):
        src = "producer" if getattr(x, "uav_gn", None) else "own"
        self.calls[("conv_out_fused", x.shape[-1], groups, float(eps), False, src)] += 1
        return emu_ops.conv_out_fused(x, gamma, beta, groups, eps, *a, **k)


def test_pipeline_norms_covers_the_modules_calls(monkeypatch):
    """the UNet (batch-2 and shared-guidance-prefix calls) and both VAE decoders, run on small inputs with emulated
    kernels: every distinct (kind, C, groups, eps, per-frame, statistics source) they ask for is in PIPELINE_NORMS"""
    from oracle.weights import make_state_dict
    from upscale_a_video_b200 import (AutoencoderKLVideo, _lib, autoencoder_kl_cond_video, layers, pipeline_upscale_a_video,
                                      unet_video)
    from upscale_a_video_b200.unet_video import UNetVideoModel
    rec = _Recorder()
    for mod in (layers, unet_video, autoencoder_kl_cond_video, pipeline_upscale_a_video):
        monkeypatch.setattr(mod, "ops", rec)
    monkeypatch.setattr(_lib, "require_cuda", lambda t, who: None)
    meta = json.load(open(os.path.join(G_DIR, "meta.json")))
    v = torch.load(os.path.join(G_DIR, "vae.pt"), weights_only=False)
    for kind, key in (("vae_3d", "vae3d_decode"), ("vae_video", "vaevideo_decode")):
        m = AutoencoderKLVideo.from_config(json.load(open(os.path.join(CFG, f"{kind}_config.json"))))
        m.load_state_dict(make_state_dict(json.load(open(os.path.join(G_DIR, f"shapes_{kind}.json"))), meta["seed_vae"]))
        c = v[key]
        m.eval().decode(c["z"], c["img"], c["w_lr"])
    m = UNetVideoModel.from_config(json.load(open(os.path.join(CFG, "unet_video_config.json"))))
    m.load_state_dict(make_state_dict(json.load(open(os.path.join(G_DIR, "shapes_unet.json"))), meta["seed_unet"]))
    m = m.half().eval()
    c = torch.load(os.path.join(G_DIR, "unet.pt"), weights_only=False)["t3_16x24"]
    ctx = c["ctx"].half()
    m(c["sample"].half(), torch.tensor(c["timestep"]), c["low_res"].half(), encoder_hidden_states=ctx,
      class_labels=c["class_labels"])
    s, lo = c["sample"][:1].repeat(2, 1, 1, 1, 1).half(), c["low_res"][:1].repeat(2, 1, 1, 1, 1).half()
    m(s, 601, lo, encoder_hidden_states=ctx, class_labels=torch.tensor([120]), cfg_shared_input=True)
    table = {_signature(c) for c in nc.PIPELINE_NORMS}
    seen = set(rec.calls)
    print(f"\n{len(seen)} distinct normalisation calls recorded, {len(table)} in PIPELINE_NORMS")
    missing = sorted(s for s in seen if s not in table)
    assert not missing, f"calls the modules make that PIPELINE_NORMS lacks: {missing}"
    # and every GroupNorm / LayerNorm signature in the table is one the modules make (RAFT, LLaVA, CLIP text and the
    # colour fix are not part of these runs)
    extra = sorted(s for s in table if s[0] in ("groupnorm", "group_norm_cat", "conv_out_fused") and s not in seen)
    assert not extra, f"PIPELINE_NORMS entries no module call matches: {extra}"
