"""Inputs, fp64 references and the pass criterion shared by the normalisation kernel tests (importable without a GPU).

With i.i.d. inputs every group, slab and frame has the same statistics up to sampling noise, so a kernel that reads a
neighbour's statistics, a stale slab, per-clip statistics where per-frame ones are asked for, or that drops part of
its partial sums moves its outputs by that noise only.  The generators here give every (slab, group), every frame and
every token its own mean and scale, so each of those faults moves outputs by O(1) (`per_group`, `per_frame`,
`rows`); `offset16` / `offset64` put a common DC offset under the data, which is what the raw-moment statistics
(E[x^2] - E[x]^2 from fp32 partials) are sensitive to; `scaled` is the VAE decoder's residual stream (x 2^-7, eps
x 2^-14) with near-constant and exactly constant groups, where eps governs; `flat` is a fade to black for the colour
fix's plane statistics.

`PIPELINE_NORMS` lists the distinct normalisation calls of one config-2 run (8 frames 320x576 -> 1280x2304, 30 DDIM
steps, classifier-free guidance, the 3-D VAE decoding 3 frames at a time, RAFT flows on the input frames, the LLaVA
captioner) at their real sizes, plus the video VAE's two calls the 3-D VAE does not make (config 4's 180x320 input).
"""
from __future__ import annotations

import math
from typing import NamedTuple, Optional, Tuple

import torch

U16 = 2.0 ** -11          # unit roundoff of fp16 (round to nearest)
U32 = 2.0 ** -24          # unit roundoff of fp32
FP16_TINY = 2.0 ** -24    # spacing of fp16 subnormals: the absolute floor of an fp16 rounding
GAMMA_STATS = 4 * U32     # relative error of the kernels' summed {x, x^2} (fp32 per thread / per block, fp64 across)
LEGACY_RTOL = LEGACY_ATOL = 2e-3   # the band the normalisation tests used before: the criterion is never looser
SAFETY = 2.0
CHUNK = 1 << 22           # elements per generated / reference chunk (keeps full-size references at a few hundred MB)
VAE_STREAM_SCALE = 2.0 ** -7       # autoencoder_kl_cond_video.VAE_STREAM_SCALE (pinned in test_norm_cases_host)
EPS_SCALED = 1e-6 * VAE_STREAM_SCALE ** 2
NUM_SMS = 132             # H100 SXM: the split count of the producer-statistics path depends on it

GN_GENERATORS = ("iid", "per_group", "per_frame", "offset16", "offset64", "scaled")
ROW_GENERATORS = ("iid", "rows", "offset16")
PLANE_GENERATORS = ("iid", "per_group", "flat")


# ---------------------------------------------------------------------------------------------------------------------
# generators
# ---------------------------------------------------------------------------------------------------------------------
def group_moments(gen: str, N: int, T: int, G: int, eps: float = 1e-6, device="cpu"):
    """(mu, sd) of every (slab n, frame t, group g), each (N, T, G) fp32: x = mu + sd * z with z ~ N(0, 1).

    per_group: k = (2g + 3n) mod 5 - 2, mu = 4k, sd = 2^((g + n) mod 3 - 1): neighbouring groups and slabs differ by
    >= 8 >= 4 std in mean and x2 or x4 in scale.  per_frame: the same with t added to both indices (frames differ by 4
    in mean).  scaled: per_group x 2^-7, and groups g = 3 mod 8 near-constant (sd = sqrt(eps), mean 2 sd), g = 6 mod 8
    exactly constant (sd = 0) at a mean that sums exactly in fp32."""
    n = torch.arange(N, device=device).view(N, 1, 1)
    t = torch.arange(T, device=device).view(1, T, 1)
    g = torch.arange(G, device=device).view(1, 1, G)
    shape = (N, T, G)
    if gen == "iid":
        return torch.full(shape, 0.5, device=device), torch.full(shape, 2.0, device=device)
    if gen in ("offset16", "offset64"):
        return torch.full(shape, float(gen[6:]), device=device), torch.ones(shape, device=device)
    tt = t if gen == "per_frame" else 0 * t
    k = (2 * g + 3 * n + tt) % 5 - 2
    mu = (4.0 * k).float().expand(shape)
    sd = torch.pow(2.0, ((g + n + tt) % 3 - 1).float()).expand(shape)
    if gen in ("per_group", "per_frame"):
        return mu.contiguous(), sd.contiguous()
    assert gen == "scaled", gen
    s = VAE_STREAM_SCALE
    mu, sd = (mu * s).clone(), (sd * s).clone()
    near = (g % 8 == 3).expand(shape)
    const = (g % 8 == 6).expand(shape)
    sd[near] = math.sqrt(eps)
    mu[near] = 2 * math.sqrt(eps)
    sd[const] = 0.0
    mu[const] = (k.expand(shape)[const] + 3).float() * 2.0 ** -5 * s
    return mu, sd


def fill_groups(x: torch.Tensor, gen: str, G: int, seed: int, eps: float = 1e-6, c0: int = 0, C_total: int = 0):
    """fills x (N, T, P, C) fp16 in place (any device, any strides of the pixel dim) from `group_moments`, chunk by
    chunk over pixels with a generator on x's device: deterministic for a given seed, shape and device.  x may be
    channels [c0, c0 + C) of a C_total-channel tensor (one part of a concatenation): its groups are that tensor's."""
    N, T, P, C = x.shape
    mu, sd = group_moments(gen, N, T, G, eps, x.device)
    cpg = (C_total or C) // G
    mu_c = mu.repeat_interleave(cpg, -1)[:, :, None, c0:c0 + C]   # (N, T, 1, C)
    sd_c = sd.repeat_interleave(cpg, -1)[:, :, None, c0:c0 + C]
    rng = torch.Generator(device=x.device).manual_seed(seed)
    step = max(1, CHUNK // max(1, N * T * C))
    for p0 in range(0, P, step):
        p1 = min(P, p0 + step)
        z = torch.randn(N, T, p1 - p0, C, generator=rng, device=x.device)
        x[:, :, p0:p1] = (mu_c + sd_c * z).half()
    return x


def make_rows(gen: str, rows: int, C: int, seed: int, device="cpu", ld: Optional[int] = None):
    """(rows, C) fp16 tokens (a column slice of a (rows, ld) buffer when ld > C).  rows: token r has mean
    4((3r) mod 5 - 2) and scale 2^(r mod 3 - 1), so neighbouring tokens, and the U tokens one warp keeps in flight,
    differ by >= 8 in mean and x2 in scale"""
    ld = C if ld is None else ld
    buf = torch.full((rows, ld), float("nan"), dtype=torch.float16, device=device)
    x = buf[:, :C]
    r = torch.arange(rows, device=device, dtype=torch.float32)[:, None]
    if gen == "iid":
        mu, sd = torch.full_like(r, 1.0), torch.full_like(r, 3.0)
    elif gen in ("offset16", "offset64"):
        mu, sd = torch.full_like(r, float(gen[6:])), torch.ones_like(r)
    else:
        assert gen == "rows", gen
        mu, sd = 4.0 * ((3 * r) % 5 - 2), torch.pow(2.0, r % 3 - 1)
    rng = torch.Generator(device=device).manual_seed(seed)
    step = max(1, CHUNK // C)
    for r0 in range(0, rows, step):
        r1 = min(rows, r0 + step)
        x[r0:r1] = (mu[r0:r1] + sd[r0:r1] * torch.randn(r1 - r0, C, generator=rng, device=device)).half()
    return x


def make_planes(gen: str, t: int, c: int, h: int, w: int, seed: int, device="cpu"):
    """(t, c, h, w) fp32 frames.  per_group: plane (t, c) has mean 0.25((2c + 3t) mod 5 - 2), scale 2^-((c + t) mod 3 + 2);
    flat: a fade to black, -1 plus 1e-4 noise"""
    rng = torch.Generator(device=device).manual_seed(seed)
    x = torch.randn(t, c, h, w, generator=rng, device=device)
    if gen == "iid":
        return x * 0.5
    if gen == "flat":
        return x * 1e-4 - 1.0
    assert gen == "per_group", gen
    tt = torch.arange(t, device=device).view(t, 1, 1, 1)
    cc = torch.arange(c, device=device).view(1, c, 1, 1)
    return 0.25 * ((2 * cc + 3 * tt) % 5 - 2) + x * torch.pow(2.0, -((cc + tt) % 3 + 2).float())


# ---------------------------------------------------------------------------------------------------------------------
# fp64 references
# ---------------------------------------------------------------------------------------------------------------------
class Stats(NamedTuple):
    """fp64 (mean, var) of every statistics slab, (N, K) each (K = groups, or channels for InstanceNorm)"""
    mean: torch.Tensor
    var: torch.Tensor


def group_stats(x: torch.Tensor, G: int) -> Stats:
    """per-(slab, group) mean and biased variance of x (N, P, C) (any strides), in fp64 chunks over pixels: two passes
    (mean first, then the centred second moment), so the reference itself has no cancellation"""
    N, P, C = x.shape
    cpg = C // G
    step = max(1, CHUNK // max(1, N * C))
    s = torch.zeros(N, G, dtype=torch.float64, device=x.device)
    for p0 in range(0, P, step):
        s += x[:, p0:p0 + step].double().reshape(N, -1, G, cpg).sum((1, 3))
    mean = s / (P * cpg)
    q = torch.zeros_like(s)
    for p0 in range(0, P, step):
        d = x[:, p0:p0 + step].double().reshape(N, -1, G, cpg) - mean[:, None, :, None]
        q += (d * d).sum((1, 3))
    return Stats(mean, q / (P * cpg))


def gn_apply_ref(x: torch.Tensor, st: Stats, gamma, beta, eps: float, silu: bool):
    """fp64 (y, xhat, pre) of GroupNorm(+SiLU) of x (N, p, C) given the slab statistics: y the output, xhat the
    normalised value, pre the affine value before SiLU"""
    N, p, C = x.shape
    G = st.mean.shape[1]
    cpg = C // G
    rstd = (st.var + eps).rsqrt()
    xh = (x.double().view(N, p, G, cpg) - st.mean[:, None, :, None]) * rstd[:, None, :, None]
    xh = xh.reshape(N, p, C)
    pre = xh * gamma.double() + beta.double()
    y = pre.clamp_min(0) if silu == "relu" else pre * torch.sigmoid(pre) if silu else pre
    return y, xh, pre


def gn_reference(x, G, gamma, beta, eps, silu):
    """GroupNorm(+SiLU) of x (N, P, C) in fp64 (small inputs: one piece)"""
    return gn_apply_ref(x, group_stats(x, G), gamma, beta, eps, silu)[0]


def layer_norm_ref(x, gamma, beta, eps):
    """(y, xhat) of LayerNorm over the last dim, fp64"""
    xd = x.double()
    m = xd.mean(-1, keepdim=True)
    v = ((xd - m) ** 2).mean(-1, keepdim=True)
    xh = (xd - m) / (v + eps).sqrt()
    return xh * gamma.double() + beta.double(), xh


def rms_norm_ref(x, weight, eps):
    """(y, x * rstd) of LlamaRMSNorm, fp64"""
    xd = x.double()
    xr = xd * (xd.pow(2).mean(-1, keepdim=True) + eps).rsqrt()
    return xr * weight.double(), xr


def instance_norm_ref(x, eps, relu):
    """(y, xhat, Stats) of InstanceNorm2d (no affine, biased variance) (+ ReLU) of x (n, h, w, C) channels-last, fp64"""
    n, C = x.shape[0], x.shape[-1]
    st = group_stats(x.reshape(n, -1, C), C)
    xh = (x.double().reshape(n, -1, C) - st.mean[:, None]) * (st.var + eps).rsqrt()[:, None]
    y = xh.clamp_min(0) if relu else xh
    return y.reshape(x.shape), xh.reshape(x.shape), st


def plane_stats_ref(x, eps):
    """calc_mean_std: (mean, sqrt(unbiased var + eps)) per (t, c) plane of x (t, c, h, w), fp64, each (t, c)"""
    v = x.double().flatten(2)
    m = v.mean(-1)
    var = ((v - m[..., None]) ** 2).sum(-1) / (v.shape[-1] - 1)
    return m, (var + eps).sqrt(), var


# ---------------------------------------------------------------------------------------------------------------------
# pass criterion
# ---------------------------------------------------------------------------------------------------------------------
def stats_error(mean, var, eps, gamma_s=GAMMA_STATS):
    """(relative error of rstd, absolute error of the mean) the raw-moment statistics may carry: E[x^2] and E[x] from
    sums with relative error gamma_s, so var is off by gamma_s (mean^2 + var) + the fp32 rounding of the mean"""
    m2 = mean * mean
    e_var = gamma_s * (m2 + var) + 2 * U32 * m2
    return 0.5 * e_var / (var + eps) + 2 * U32, gamma_s * mean.abs() + U32 * mean.abs()


def tolerance(y, xh, scale, e_rstd, e_mean, rstd, silu: bool, extra=0.0):
    """per-element bound on |kernel - ref| for a normalisation y = act(xhat * scale + shift), times SAFETY:

    * the fp16 output rounding: U16 |y| + 2^-24;
    * the statistics: |scale| (|xhat| e_rstd + rstd e_mean) (SiLU's slope is below 1.1);
    * the fp32 affine x * sc + sh: 4 U32 |scale| (|xhat| + rstd |mean|) is inside the statistics term's 2 U32 terms;
    * `extra`: a rounding the kernel does on top (the fp16 product of RMSNorm).

    The result is capped at the band the tests used before (2e-3 + 2e-3 |ref|): the criterion is never looser."""
    slope = 1.1 if silu else 1.0
    b = U16 * y.abs() + FP16_TINY + slope * scale.abs() * (xh.abs() * e_rstd + rstd * e_mean) + extra
    return torch.minimum(SAFETY * b, LEGACY_ATOL + LEGACY_RTOL * y.abs())


class Verdict(NamedTuple):
    bad: int          # elements out of bounds (NaN counts as out of bounds)
    worst: float      # max |err| / tol
    n: int


def judge(got: torch.Tensor, ref: torch.Tensor, tol: torch.Tensor) -> Verdict:
    err = (got.double() - ref).abs()
    ratio = torch.nan_to_num(err / tol, nan=math.inf)
    return Verdict(int((~(err <= tol)).sum()), float(ratio.max()) if ratio.numel() else 0.0, err.numel())


def fingerprint(t: torch.Tensor) -> float:
    """a position-weighted sum of the bit patterns of a dense tensor, in chunks: equal for bit-identical tensors (the
    determinism check of outputs too large to keep twice)"""
    flat = t.reshape(-1).view(torch.int16 if t.element_size() == 2 else torch.int32)
    s = 0.0
    for i0 in range(0, flat.numel(), CHUNK):
        c = flat[i0:i0 + CHUNK].double()
        w = torch.arange(i0, i0 + c.numel(), device=c.device, dtype=torch.float64) % 65521 + 1
        s += float((c * w).sum())
    return s


def merge(a: Optional[Verdict], b: Verdict) -> Verdict:
    return b if a is None else Verdict(a.bad + b.bad, max(a.worst, b.worst), a.n + b.n)


def gn_verdict(got, x, st: Stats, gamma, beta, eps, silu, pixel_chunks=True) -> Verdict:
    """judge a GroupNorm(+SiLU) output got (N, P, C) of x (N, P, C) against the fp64 reference, in pixel chunks
    (silu: True, False or "relu", for InstanceNorm + ReLU with G = C)"""
    N, P, C = x.shape
    G = st.mean.shape[1]
    cpg = C // G
    e_r, e_m = stats_error(st.mean, st.var, eps)
    rstd = (st.var + eps).rsqrt()
    per_c = lambda t: t.repeat_interleave(cpg, -1)[:, None, :]  # (N, 1, C)
    scale = gamma.double()[None, None, :]
    step = max(1, CHUNK // max(1, N * C)) if pixel_chunks else P
    v = None
    for p0 in range(0, P, step):
        xs = x[:, p0:p0 + step]
        y, xh, _ = gn_apply_ref(xs, st, gamma, beta, eps, silu)
        tol = tolerance(y, xh, scale, per_c(e_r), per_c(e_m), per_c(rstd), silu is True)
        v = merge(v, judge(got[:, p0:p0 + step], y, tol))
    return v


def rows_tolerance(y, xh, gamma, xd, eps, C):
    """LayerNorm bound: the mean and the centred second moment are fp32 warp sums (C / 256 + 32 rounding steps deep),
    rstd is rsqrtf (2 ulp)"""
    m = xd.mean(-1, keepdim=True)
    v = ((xd - m) ** 2).mean(-1, keepdim=True)
    depth = (C / 256 + 32) * U32
    e_m = depth * xd.abs().mean(-1, keepdim=True)
    e_r = 0.5 * depth + 2 * U32 + (2 * m.abs() * e_m) / (v + eps)
    return tolerance(y, xh, gamma.double(), e_r, e_m, (v + eps).rsqrt(), False)


def rms_tolerance(y, xr, weight, C):
    """RMSNorm bound: sum of squares in fp32 (C / 2048 + 16 steps deep per thread and tree), rsqrtf, x * r rounded to
    fp16 before the fp16 product with the weight (LlamaRMSNorm's `weight * x.to(fp16)`)"""
    w = weight.double().abs()
    e_r = (C / 2048 + 16) * U32 + 2 * U32
    inner = U16 * xr.abs() * w + FP16_TINY * w
    return tolerance(y, xr, weight.double(), e_r, 0.0, 0.0, False, extra=inner)


# ---------------------------------------------------------------------------------------------------------------------
# the pipeline's normalisation calls
# ---------------------------------------------------------------------------------------------------------------------
class NormCall(NamedTuple):
    name: str
    kind: str              # groupnorm | group_norm_cat | conv_out_fused | layernorm | rmsnorm | instnorm | plane_stats
    C: int                 # channels (features for layernorm / rmsnorm, planes' channels for plane_stats)
    groups: int            # GroupNorm groups (0 elsewhere)
    eps: float
    per_frame: bool        # statistics per frame (n_outer = B * T) instead of per clip (n_outer = B)
    B: int                 # batch items (images for instnorm, rows' batch for layernorm / rmsnorm)
    T: int                 # frames per batch item
    HW: int                # pixels per frame (rows per batch item for layernorm / rmsnorm)
    source: str            # own (read pass) | producer (the GEMM epilogue's 16 x 8 blocks) | concat | concat_bcast
    parts: Tuple[int, ...] = ()   # channels of each concat part
    silu: bool = True
    ld_in: int = 0         # pixel / row stride of the input when wider than C (0: dense)
    ld_out: int = 0        # pixel / row stride of the output when wider than C (0: dense)
    relu: bool = False

    @property
    def cpg(self) -> int:
        return self.C // self.groups

    @property
    def n_outer(self) -> int:
        return self.B * self.T if self.per_frame else self.B

    @property
    def pixels(self) -> int:
        """pixels per statistics slab"""
        return self.HW if self.per_frame else self.T * self.HW


def split_count(n_outer: int, groups: int, blocks_per_slab: int, num_sms: int = NUM_SMS) -> int:
    """S, the number of fp64 partials per (slab, group) of the producer-statistics path (norm.cu gn_reduce_plan)"""
    S = -(-4 * num_sms // (groups * n_outer))
    return max(1, min(S, blocks_per_slab // 256, 32))


def producer_blocks_per_slab(call: NormCall) -> int:
    """statistics blocks per slab when the producer is a 1-tap temporal conv over (B, T, H*W): 16-row blocks per frame"""
    per_frame = -(-call.HW // 128) * 8
    return per_frame if call.per_frame else call.T * per_frame


# config 2: UNet on (B = 2, T = 8) windows at the 320x576 latent; levels 0..3 at 320x576, 160x288, 80x144, 40x72
_L = {0: 320 * 576, 1: 160 * 288, 2: 80 * 144, 3: 40 * 72}
# 3-D VAE decoder on (1, 3) chunks: the latent size, x2 and x4
_V = {1: 320 * 576, 2: 640 * 1152, 4: 1280 * 2304}


def _unet(name, C, eps, lvl, source, *, per_frame=False, silu=True, parts=()):
    return NormCall(f"unet_{name}", "groupnorm" if not parts else "group_norm_cat", C, 32, eps, per_frame, 2, 8, _L[lvl],
                    source, parts, silu and not per_frame)


def _vae(name, C, eps, up, source, *, per_frame=False, silu=True):
    return NormCall(f"vae_{name}", "groupnorm", C, 32, eps, per_frame, 1, 3, _V[up], source, (), silu and not per_frame)


PIPELINE_NORMS = (
    # UNet ResNet blocks: norm1 of conv_in's output and of the upsampled tensors by a read pass, the rest from the
    # producing conv's statistics blocks; eps 1e-5 (norm_eps) or 1e-6 (the blocks' resnet_eps)
    _unet("conv_in_norm1", 256, 1e-5, 0, "own"),
    _unet("l0_256", 256, 1e-5, 0, "producer"),
    _unet("l0_256_e6", 256, 1e-6, 0, "producer"),
    _unet("l0_512_up", 512, 1e-5, 0, "own"),
    _unet("l0_512_up_e6", 512, 1e-6, 0, "own"),
    _unet("l0_512_e6", 512, 1e-6, 0, "producer"),
    _unet("l1_256_e6", 256, 1e-6, 1, "producer"),
    _unet("l1_256", 256, 1e-5, 1, "producer"),
    _unet("l1_512", 512, 1e-5, 1, "producer"),
    _unet("l1_512_e6", 512, 1e-6, 1, "producer"),
    _unet("l1_512_up_e6", 512, 1e-6, 1, "own"),
    _unet("l2_512", 512, 1e-5, 2, "producer"),
    _unet("l2_512_e6", 512, 1e-6, 2, "producer"),
    _unet("l2_1024_up_e6", 1024, 1e-6, 2, "own"),
    _unet("l2_1024_e6", 1024, 1e-6, 2, "producer"),
    _unet("l3_512", 512, 1e-5, 3, "producer"),
    _unet("l3_512_e6", 512, 1e-6, 3, "producer"),
    _unet("l3_1024", 1024, 1e-5, 3, "producer"),
    _unet("l3_1024_e6", 1024, 1e-6, 3, "producer"),
    # Transformer3DModel.norm: per frame (n_outer = B T), no SiLU
    _unet("l1_attn_512", 512, 1e-6, 1, "producer", per_frame=True),
    _unet("l2_attn_512", 512, 1e-6, 2, "producer", per_frame=True),
    _unet("l3_attn_1024", 1024, 1e-6, 3, "producer", per_frame=True),
    # up-block norm1 over torch.cat([x, skip]) without the concat: 768 / 1536 / 2048 channels (cpg 24, 48, 64), and the
    # skip computed once for both guidance halves (batch 1, broadcast)
    _unet("l3_cat_2048", 2048, 1e-5, 3, "concat", parts=(1024, 1024)),
    _unet("l3_cat_1536", 1536, 1e-5, 3, "concat", parts=(1024, 512)),
    _unet("l2_cat_1536", 1536, 1e-5, 2, "concat", parts=(1024, 512)),
    _unet("l2_cat_1024", 1024, 1e-5, 2, "concat", parts=(512, 512)),
    _unet("l1_cat_1024", 1024, 1e-5, 1, "concat", parts=(512, 512)),
    _unet("l1_cat_768", 768, 1e-5, 1, "concat", parts=(512, 256)),
    _unet("l0_cat_768", 768, 1e-5, 0, "concat", parts=(512, 256)),
    _unet("l0_cat_512", 512, 1e-5, 0, "concat", parts=(256, 256)),
    _unet("l1_cat_768_bcast", 768, 1e-5, 1, "concat_bcast", parts=(512, 256)),
    _unet("l0_cat_768_bcast", 768, 1e-5, 0, "concat_bcast", parts=(512, 256)),
    _unet("l0_cat_512_bcast", 512, 1e-5, 0, "concat_bcast", parts=(256, 256)),
    # conv_norm_out + SiLU + conv_out in one kernel (uav_groupnorm_affine -> uav_conv_out_fused)
    NormCall("unet_conv_norm_out", "conv_out_fused", 256, 32, 1e-5, False, 2, 8, _L[0], "producer"),
    # 3-D VAE decoder: the scaled residual stream's norms (eps 1e-6 x 2^-14), the branch-internal norm2 (eps 1e-6), the
    # mid block's AttentionBlock per frame, and conv_norm_out at 1280x2304
    _vae("mid_norm1", 512, EPS_SCALED, 1, "own"),
    _vae("l1_512_s", 512, EPS_SCALED, 1, "producer"),
    _vae("l1_512", 512, 1e-6, 1, "producer"),
    _vae("mid_attn", 512, EPS_SCALED, 1, "producer", per_frame=True),
    _vae("up1_norm1", 512, EPS_SCALED, 2, "own"),
    _vae("l2_256_s", 256, EPS_SCALED, 2, "producer"),
    _vae("l2_256", 256, 1e-6, 2, "producer"),
    _vae("up2_norm1", 256, EPS_SCALED, 4, "own"),
    # (4 channels per group: the producer's 8-channel blocks cannot serve, so these read x once more)
    _vae("l4_128_s", 128, EPS_SCALED, 4, "own"),
    _vae("l4_128", 128, 1e-6, 4, "own"),
    # video VAE (config 4, 180x320 input): the 3-channel condition frames in an 8-channel buffer (generic kernels) and
    # the 640-channel concat of the condition features
    NormCall("vaevideo_cond_c3", "groupnorm", 3, 3, 1e-6, False, 1, 3, 180 * 320, "own", (), True, 8, 8),
    NormCall("vaevideo_cond_640", "groupnorm", 640, 32, 1e-6, False, 1, 3, 180 * 320, "own"),
    # LayerNorm of the UNet transformers (B T H W tokens), CLIP text (77 tokens), the LLaVA vision tower (8 x 577)
    NormCall("unet_ln_l1", "layernorm", 512, 0, 1e-5, False, 16, 1, _L[1], "own"),
    NormCall("unet_ln_l2", "layernorm", 512, 0, 1e-5, False, 16, 1, _L[2], "own"),
    NormCall("unet_ln_l3", "layernorm", 1024, 0, 1e-5, False, 16, 1, _L[3], "own"),
    NormCall("clip_text_ln", "layernorm", 1024, 0, 1e-5, False, 2, 1, 77, "own"),
    NormCall("llava_vision_ln", "layernorm", 1024, 0, 1e-5, False, 8, 1, 577, "own"),
    # LlamaRMSNorm of the LLaVA-1.5 decoder (hidden 4096): prefill of 8 prompts, and decode rows in a wider buffer
    NormCall("llava_rms_prefill", "rmsnorm", 4096, 0, 1e-5, False, 8, 1, 640, "own"),
    NormCall("llava_rms_decode", "rmsnorm", 4096, 0, 1e-5, False, 8, 1, 1, "own", (), False, 4096 * 3, 4096 * 2),
    # RAFT feature encoder (instance norm, both directions of 7 frame pairs = 28 images at 320x576 / 2, / 4, / 8)
    NormCall("raft_in_64", "instnorm", 64, 0, 1e-5, False, 28, 1, 160 * 288, "own", relu=True),
    NormCall("raft_in_96", "instnorm", 96, 0, 1e-5, False, 28, 1, 80 * 144, "own", relu=True),
    NormCall("raft_in_128", "instnorm", 128, 0, 1e-5, False, 28, 1, 40 * 72, "own", relu=False),
    # colour fix (AdaIN): per-plane statistics of 3 decoded frames x 3 channels at 1280x2304
    NormCall("colorfix_planes", "plane_stats", 3, 0, 1e-5, False, 3, 1, 1280 * 2304, "own"),
)


def generators_for(call: NormCall) -> Tuple[str, ...]:
    """the generators a call is tested with: the ones its faults show up under"""
    if call.kind in ("layernorm", "rmsnorm"):
        return ("rows", "offset16") if call.kind == "layernorm" else ("rows",)
    if call.kind == "plane_stats":
        return PLANE_GENERATORS
    if call.kind == "instnorm":
        return ("per_group", "offset64")
    if call.eps == EPS_SCALED:
        return ("per_group", "scaled")
    g = ["per_group"]
    if call.per_frame:
        g.append("per_frame")
    if call.source == "own":
        g.append("offset64")
    elif call.source == "producer" and not call.per_frame:
        g.append("offset16")
    if call.C == 3:
        g = ["iid", "per_frame"]
    return tuple(g)
