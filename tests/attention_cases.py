"""Inputs, fp64 reference and pass criterion shared by the attention kernel tests (importable without a GPU).

Random q/k make the softmax nearly uniform at long sequences, so a dropped, stale or unmasked key tile moves each output
by far less than any sensible tolerance.  The generators here are built so that such a fault moves outputs by O(1)
(`needle`), changes the running maximum in every tile (`ramp_up`) or only in the first (`ramp_down`), or changes the
number of keys averaged over (`flat`); `random` and `peaky` keep the plain inputs.
"""
from __future__ import annotations

import math
from typing import NamedTuple, Optional

import torch

GENERATORS = ("random", "peaky", "needle", "ramp_up", "ramp_down", "flat")
U16 = 2.0 ** -11      # unit roundoff of fp16 (round to nearest)
U32 = 2.0 ** -24      # unit roundoff of fp32
NEEDLE_LOGIT = 48.0   # scaled score of the planted key, in nats
RAMP_LOGITS = 8.0     # scaled score range of the ramps, in nats


def needle_keys(nq: int, nk: int, seed: int) -> torch.Tensor:
    """pi(i), the planted key of query row i.  Rows [0, S) take the S special keys in order: every key when nk <= 256,
    else the first and last key of every 64- and 128-key tile (the last one is the last valid key of the ragged tile)
    and key nk - 1; the other rows take random keys."""
    if nk <= 256:
        special = list(range(nk))
    else:
        s = {nk - 1}
        for bn in (64, 128):
            for t0 in range(0, nk, bn):
                s.update((t0, min(t0 + bn - 1, nk - 1)))
        special = sorted(s)
    g = torch.Generator().manual_seed(seed + 17)
    pi = torch.randint(0, nk, (nq,), generator=g)
    n = min(nq, len(special))
    pi[:n] = torch.tensor(special[:n])
    return pi


def num_special(nk: int) -> int:
    return nk if nk <= 256 else len({nk - 1} | {t for bn in (64, 128) for t0 in range(0, nk, bn)
                                                 for t in (t0, min(t0 + bn - 1, nk - 1))})


def make_inputs(gen: str, B: int, heads: int, d: int, nq: int, nk: int, kv_batch_div: int = 1, seed: int = 0,
                device="cpu", scale: Optional[float] = None):
    """fp16 q (B, nq, heads*d), k and v (B / kv_batch_div, nk, heads*d), deterministic from `seed` on a given device"""
    assert gen in GENERATORS, gen
    scale = d ** -0.5 if scale is None else scale
    C, Bk = heads * d, B // kv_batch_div
    g = torch.Generator(device=device).manual_seed(seed)

    def randn(*shape):
        return torch.randn(*shape, generator=g, device=device)

    if gen in ("random", "peaky"):
        q, k, v = randn(B, nq, C), randn(Bk, nk, C), randn(Bk, nk, C)
        if gen == "peaky":
            q = q * 6
        return q.half(), k.half(), v.half()
    if gen == "needle":
        # unit keys: the planted key scores NEEDLE_LOGIT, every other key NEEDLE_LOGIT * cos, cos ~ N(0, 1/d), so the
        # others carry at most nk exp(NEEDLE_LOGIT^2 / 2d - NEEDLE_LOGIT) < 1e-7 of the mass and out[i] ~ v[pi(i)]
        k = randn(Bk, nk, heads, d)
        k = (k / k.norm(dim=-1, keepdim=True)).half()
        kf = k.float()
        pi = needle_keys(nq, nk, seed).to(device)
        kp = kf[:, pi]                                              # (Bk, nq, heads, d)
        q = kp * (NEEDLE_LOGIT / scale) / (kp * kp).sum(-1, keepdim=True)
        q = q.repeat_interleave(kv_batch_div, dim=0).reshape(B, nq, C)
        return q.half(), k.reshape(Bk, nk, C), randn(Bk, nk, C).half()
    if gen in ("ramp_up", "ramp_down"):
        # score(i, j) ~ RAMP_LOGITS * t_j + small noise, t rising (falling) linearly over the keys
        u = torch.full((d,), d ** -0.5, device=device)
        t = torch.linspace(0.0, 1.0, nk, device=device)
        if gen == "ramp_down":
            t = 1.0 - t
        k = t[None, :, None, None] * u + 0.05 * randn(Bk, nk, heads, d)
        q = (RAMP_LOGITS / scale) * u + 0.3 * randn(B, nq, heads, d)
        return q.reshape(B, nq, C).half(), k.reshape(Bk, nk, C).half(), randn(Bk, nk, C).half()
    # flat: q = 0, every score is 0 and out = the exact mean of v over exactly nk keys
    q = torch.zeros(B, nq, C, device=device)
    v = (1.0 + 0.5 * torch.arange(nk, device=device, dtype=torch.float32) / nk)[None, :, None].expand(Bk, nk, C)
    return q.half(), randn(Bk, nk, C).half(), v.contiguous().half()


class Ref(NamedTuple):
    """fp64 attention of the selected rows, (B, R, C) each: `out`; `mag` = sum_j p_ij |v_jc| (p normalised);
    `sub` = sum_j |v_jc| / l_i with l_i = sum_j exp(s_ij - max_j s_ij) (the fp16-subnormal term of P); `eps` = a bound
    on the fp32 rounding of the scaled score of row i (in nats), broadcast over the head's columns."""
    out: torch.Tensor
    mag: torch.Tensor
    sub: torch.Tensor
    eps: torch.Tensor


def softmax_ref(s: torch.Tensor, v: torch.Tensor, eps: torch.Tensor) -> Ref:
    """Ref of softmax(s) v for fp64 scaled scores s (..., n, nk), -inf where masked, v (..., nk, d) and the per-row
    score error eps (..., n); the fields keep the (..., n, d) layout"""
    m = s.amax(-1, keepdim=True)
    e = torch.exp(s - m)
    l = e.sum(-1, keepdim=True)
    p = e / l
    va = v.abs()
    return Ref(p @ v, p @ va, va.sum(-2, keepdim=True) / l, eps[..., None].expand(p.shape[:-1] + (v.shape[-1],)))


def attention_ref(q, k, v, heads: int, kv_batch_div: int, scale: float, rows=None) -> Ref:
    """softmax(q k^T scale) v in fp64 on q's device, for query rows `rows` (all by default) against EVERY key, evaluated
    in blocks of query rows so that the score block stays under 2^26 elements"""
    B, nq, C = q.shape
    Bk, nk, _ = k.shape
    d = C // heads
    dev = q.device
    rows = torch.arange(nq, device=dev) if rows is None else torch.as_tensor(rows, device=dev)
    R = rows.numel()
    res = [torch.empty(B, R, C, dtype=torch.float64, device=dev) for _ in range(4)]
    blk = max(1, (1 << 26) // (heads * nk))
    for bk in range(Bk):
        kb = k[bk].double().view(nk, heads, d).permute(1, 0, 2)   # (heads, nk, d)
        vb = v[bk].double().view(nk, heads, d).permute(1, 0, 2)
        kmax = kb.norm(dim=-1).amax(-1)                             # (heads,)
        for b in range(bk * kv_batch_div, (bk + 1) * kv_batch_div):
            for r0 in range(0, R, blk):
                rr = rows[r0:r0 + blk]
                qb = q[b, rr].double().view(-1, heads, d).permute(1, 0, 2)  # (heads, n, d)
                outs = softmax_ref((qb @ kb.transpose(1, 2)) * scale, vb,
                                   U32 * d * scale * qb.norm(dim=-1) * kmax[:, None])
                for dst, x in zip(res, outs):
                    dst[b, r0:r0 + rr.numel()] = x.permute(1, 0, 2).reshape(-1, C)
    return Ref(*res)


def tolerance(ref: Ref, nk: int, score_err: float = 0.0, safety: float = 2.0) -> torch.Tensor:
    """Per-element bound on |kernel - ref| from the roundings the kernels do, times `safety`:

    * P is rounded to fp16 before P V while the row sum l uses the unrounded fp32 P: relative error U16 per p_ij, plus
      an absolute 2^-25 where p_ij (max 1) falls in the fp16 subnormal range -> U16 * mag + 2^-25 * sub;
    * the scaled score is fp32 (fp16 products, fp32 accumulation over d, times scale * log2 e, ex2.approx): each p_ij is
      off by a factor exp(+-eps_i), which moves the normalised output by at most (exp(eps_i) - 1) (mag + |out|);
      `score_err` adds an input rounding the kernel does on top (the fp16 rotary of the temporal kernels);
    * O and l accumulate in fp32 over at most nk / 64 tiles of up to 128 terms, with a rescale per tile:
      gamma = (nk / 64 + 128) * U32 relative to mag + |out|;
    * the output is rounded to fp16: U16 * |out| + 2^-25."""
    gamma = (nk / 64 + 128) * U32
    es = torch.expm1(ref.eps + score_err + 2.0 ** -20)
    a = ref.out.abs()
    bound = U16 * ref.mag + 2.0 ** -25 * ref.sub + (es + gamma) * (ref.mag + a) + U16 * a + 2.0 ** -25
    return safety * bound


def compare(got: torch.Tensor, ref: Ref, nk: int, score_err: float = 0.0):
    """(number of elements out of bounds, rel L2 error); `got` holds the same rows as `ref`"""
    g = got.double()
    err = (g - ref.out).abs()
    tol = tolerance(ref, nk, score_err)
    bad = int((~(err <= tol)).sum())
    rel = float((g - ref.out).norm() / ref.out.norm().clamp_min(1e-300))
    return bad, rel


def assert_matches(got, ref: Ref, nk: int, what: str, score_err: float = 0.0):
    bad, rel = compare(got, ref, nk, score_err)
    print(f"[{what}] rel L2 {rel:.3e}, {bad} elements out of bounds")
    if bad:
        err = (got.double() - ref.out).abs()
        ratio = err / tolerance(ref, nk, score_err)
        i = int(torch.nan_to_num(ratio, nan=math.inf).flatten().argmax())
        raise AssertionError(f"{what}: {bad}/{err.numel()} elements out of bounds, rel L2 {rel:.3e}, worst "
                             f"|err| {err.flatten()[i].item():.4g} = {ratio.flatten()[i].item():.3g} x bound "
                             f"(ref {ref.out.flatten()[i].item():.4g}, got {got.flatten()[i].item():.4g})")


def check_rows(nq: int, nk: int, n_random: int = 1024, seed: int = 0, tile: int = 128) -> torch.Tensor:
    """query rows a long case compares: the first and the last query tile, the rows whose needle is a special key and
    `n_random` random rows"""
    g = torch.Generator().manual_seed(seed + 99)
    parts = [torch.arange(min(nq, max(tile, num_special(nk)))), torch.arange(max(0, nq - tile), nq),
             torch.randint(0, nq, (n_random,), generator=g)]
    return torch.unique(torch.cat(parts))
