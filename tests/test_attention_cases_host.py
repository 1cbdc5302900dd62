"""CPU checks of the attention test inputs and pass criterion (tests/attention_cases.py): a CPU emulator of the tiled
online-softmax kernels (fp32 scores and accumulators, P and the output rounded to fp16) passes the criterion on every
generator, and each tile-level fault injected into it is rejected by at least one generator in the shape class it
targets, so the GPU tests of tests/test_attention_kernels_gpu.py would reject the same fault in a kernel.  Also: a
non-positive or non-finite softmax scale is rejected before anything launches."""
import math

import pytest
import torch

from attention_cases import GENERATORS, attention_ref, compare, make_inputs

def emulate(q, k, v, heads, kv_batch_div, scale, BM, BN, fault=None):
    """out (B, ceil(nq / BM) * BM, C) as the kernels compute it: query tiles of BM rows, kv tiles of BN keys with a
    zero-filled ragged tail, the running row maximum of the scaled scores, P rounded to fp16 for P V while l sums the
    fp32 P, O and l rescaled when the maximum moves, fp16 output.  Rows >= nq hold the NaN that was there before unless
    a fault writes them."""
    B, nq, C = q.shape
    Bk, nk, _ = k.shape
    d = C // heads
    nt = -(-nk // BN)
    kf = torch.zeros(Bk, nt * BN, heads, d)
    vf = torch.zeros(Bk, nt * BN, heads, d)
    kf[:, :nk] = k.float().view(Bk, nk, heads, d)
    vf[:, :nk] = v.float().view(Bk, nk, heads, d)
    if fault == "v_halves_swapped":
        vf = torch.cat([vf[..., d // 2:], vf[..., :d // 2]], -1)
    bidx = torch.arange(B) % Bk if fault == "kv_batch" else torch.arange(B) // kv_batch_div
    kf, vf = kf[bidx].transpose(1, 2), vf[bidx].transpose(1, 2)          # (B, heads, keys, d)
    nqp = -(-nq // BM) * BM
    qf = torch.zeros(B, heads, nqp, d)
    qf[:, :, :nq] = q.float().view(B, nq, heads, d).transpose(1, 2)
    m = torch.full((B, heads, nqp, 1), -math.inf)
    l = torch.zeros(B, heads, nqp, 1)
    o = torch.zeros(B, heads, nqp, d)
    for j in range(nt - 1 if fault == "drop_last" else nt):
        jk = j - 1 if fault == "stale_k" and j > 0 else j
        jv = j - 1 if fault == "stale_v" and j > 0 else j
        s = qf @ kf[:, :, jk * BN:(jk + 1) * BN].transpose(-1, -2) * scale
        valid = nk - j * BN
        if fault == "mask_minus1":
            valid -= 1
        elif fault == "mask_plus1":
            valid += 1
        if valid < BN and fault != "unmasked":
            s[..., valid:] = -math.inf
        mn = torch.maximum(m, s.amax(-1, keepdim=True))
        alpha = torch.exp(m - mn)
        p = torch.exp(s - mn)
        l = (l if fault == "no_rescale_l" else l * alpha) + p.sum(-1, keepdim=True)
        o = (o if fault == "no_rescale_o" else o * alpha) + p.half().float() @ vf[:, :, jv * BN:(jv + 1) * BN]
        m = mn
    out = (o / l).half().transpose(1, 2).reshape(B, nqp, C)
    if fault != "q_tail_written":
        out[:, nq:] = math.nan
    return out


def rejects(out, ref, nq, nk):
    """True when the criterion rejects `out`: an element out of bounds, or a row >= nq written"""
    if not torch.isnan(out[:, nq:].float()).all():
        return True
    return compare(out[:, :nq], ref, nk)[0] > 0


# shape classes at reduced size: (B, heads, d, nq, nk, kv_batch_div, BM, BN).  The cross kernel takes 64 query rows at a
# time and holds every key in one tile of 80 (nk <= 80) or 128; the wgmma kernel takes 128 query rows per CTA and
# streams tiles of 128 keys for d = 64 and 128, and of 64 keys for d = 512 with the output split into two 256-column
# halves.
CLASSES = {
    "cross d64 nk77": (4, 2, 64, 308, 77, 2, 64, 80),
    "cross d128 nk100": (2, 2, 128, 400, 100, 1, 64, 128),
    "wgmma d64 nk140": (2, 2, 64, 130, 140, 1, 128, 128),
    "wgmma d128 nk300": (4, 2, 128, 129, 300, 2, 128, 128),
    "wgmma d512 nk140": (1, 1, 512, 100, 140, 1, 128, 64),
}
FAULTS = {
    "unmasked": list(CLASSES),
    "mask_minus1": list(CLASSES),
    "mask_plus1": list(CLASSES),
    "drop_last": ["wgmma d64 nk140", "wgmma d128 nk300", "wgmma d512 nk140"],
    "stale_k": ["wgmma d64 nk140", "wgmma d128 nk300", "wgmma d512 nk140"],
    "stale_v": ["wgmma d64 nk140", "wgmma d128 nk300", "wgmma d512 nk140"],
    "no_rescale_l": ["wgmma d64 nk140", "wgmma d128 nk300", "wgmma d512 nk140"],
    "no_rescale_o": ["wgmma d64 nk140", "wgmma d128 nk300", "wgmma d512 nk140"],
    "kv_batch": ["cross d64 nk77", "wgmma d128 nk300"],
    "v_halves_swapped": ["wgmma d512 nk140"],
    "q_tail_written": list(CLASSES),
}


@pytest.fixture(scope="module")
def cases():
    """inputs and fp64 reference of every (class, generator)"""
    out = {}
    for name, (B, H, d, nq, nk, kvd, BM, BN) in CLASSES.items():
        for gen in GENERATORS:
            q, k, v = make_inputs(gen, B, H, d, nq, nk, kvd, seed=7)
            out[name, gen] = (q, k, v, attention_ref(q, k, v, H, kvd, d ** -0.5))
    return out


def test_emulator_passes_every_generator(cases):
    for (name, gen), (q, k, v, ref) in cases.items():
        B, H, d, nq, nk, kvd, BM, BN = CLASSES[name]
        out = emulate(q, k, v, H, kvd, d ** -0.5, BM, BN)
        bad, rel = compare(out[:, :nq], ref, nk)
        assert bad == 0 and not rejects(out, ref, nq, nk), (name, gen, bad, rel)


def test_needle_output_is_the_planted_value(cases):
    """the needle carries the mass: out[i] ~ v[pi(i)], so a fault that loses the planted key moves out[i] by O(1)"""
    from attention_cases import needle_keys
    for name, (B, H, d, nq, nk, kvd, BM, BN) in CLASSES.items():
        q, k, v, ref = cases[name, "needle"]
        pi = needle_keys(nq, nk, 7)
        want = v.double()[torch.arange(B) // kvd][:, pi]
        assert (ref.out - want).abs().max() < 1e-6, name


@pytest.mark.parametrize("fault", list(FAULTS))
def test_fault_is_rejected(cases, fault):
    for name in FAULTS[fault]:
        B, H, d, nq, nk, kvd, BM, BN = CLASSES[name]
        caught = []
        for gen in GENERATORS:
            q, k, v, ref = cases[name, gen]
            if rejects(emulate(q, k, v, H, kvd, d ** -0.5, BM, BN, fault), ref, nq, nk):
                caught.append(gen)
        print(f"{fault:18s} {name:18s} rejected by {', '.join(caught) or 'NOTHING'}")
        assert caught, f"fault {fault} on {name} passes every generator"


def test_attention_rejects_bad_scale_before_launch(uav_lib):
    """the cross and wgmma kernels scale the row maximum of the raw scores, which is the maximum of the scaled scores only
    for scale > 0: zero, negative, infinite and NaN scales are rejected with a message and launch nothing, on every
    kernel path (cross, wgmma d = 64, 128 and 512).  The pointers are never dereferenced."""
    A = 1 << 20
    launches = uav_lib.uav_launch_count()
    for heads, d, nq, nk in ((8, 64, 4096, 77), (8, 64, 300, 300), (8, 128, 920, 920), (1, 512, 1024, 1024)):
        C = heads * d
        for scale in (0.0, -0.125, -0.0, math.inf, -math.inf, math.nan):
            st = uav_lib.uav_attention(A, A, A, A, 1, heads, d, nq, nk, C, C, C, C, 1, scale, None)
            msg = uav_lib.uav_last_error_string()
            assert st == 1 and b"uav_attention: scale must be finite and > 0" in msg, (d, nk, scale, st, msg)
    assert uav_lib.uav_launch_count() == launches
