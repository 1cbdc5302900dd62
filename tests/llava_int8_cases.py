"""The captioner's weight-only int8 rule restated on the CPU (bitsandbytes' row-wise int8 quantization), hand-made
rows with their expected int8 values, and the byte count of a decoder held in int8."""
from fractions import Fraction

import torch

HALF_MAX = 65504.0
SUB = 2.0 ** -24  # the smallest fp16 subnormal


def quantize_rows_ref(w: torch.Tensor):
    """(q int8, absmax fp32) of fp16 w (N, K): absmax = max |w| per row in fp32, q = round_half_even((w * 127) /
    absmax) in fp32, q = 0 on a row with absmax 0"""
    wf = w.float()
    s = wf.abs().amax(1)
    q = torch.round(wf * 127 / s[:, None])
    q = torch.where(s[:, None] == 0, torch.zeros_like(q), q)
    return q.to(torch.int8), s


def dequantize_ref(q: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """W' = fp16((q * absmax) / 127), the prefill's weight"""
    return ((q.float() * s[:, None]) / 127).half()


def _exact_q(row):
    """round_half_even(w * 127 / max |w|) of each fp16 value of `row`, in exact rational arithmetic"""
    s = max(abs(Fraction(v)) for v in row)
    return [0 if s == 0 else round(Fraction(v) * 127 / s) for v in row]  # Fraction rounds half to even


def hand_rows(K: int = 32):
    """(fp16 rows (6, K), expected q (6, K) int8): exact .5 ties, a zero row, one outlier, an absmax taken from a
    negative value, +-65504, and subnormals.  Unlisted columns are 0."""
    rows = [
        [127.0, 0.5, 1.5, 2.5, -0.5, -1.5, -2.5, 126.5, 3.5, -125.5],    # absmax 127: q = w, ties to even
        [0.0],                                                           # absmax 0: q = 0
        [100.0, 0.3, -0.3, 0.4, 0.39, -0.4, 0.01, -99.0],                # one outlier
        [-3.0, 1.0, 2.0, -1.5, 0.75, 2.99],                              # absmax from -3; -1.5 -> -63.5 -> -64
        [HALF_MAX, -HALF_MAX, HALF_MAX / 2, 1.0, -16376.0, 0.0],         # 32752 -> 63.5 -> 64
        [5 * SUB, -3 * SUB, SUB, 2 * SUB, 4 * SUB, -5 * SUB, 1023 * SUB],  # subnormals, absmax 1023 * 2^-24
    ]
    w = torch.zeros(len(rows), K, dtype=torch.float16)
    for i, r in enumerate(rows):
        w[i, :len(r)] = torch.tensor(r, dtype=torch.float32).half()
    expect = torch.tensor([_exact_q(r) for r in w.float().tolist()], dtype=torch.int8)
    return w, expect


def int8_decoder_bytes(tc: dict, mm_hidden: int) -> int:
    """device bytes of the decoder and projector weights with int8 Linears (N K + 4 N each), fp16 embed_tokens,
    lm_head and RMSNorm weights, and fp32 projector biases"""
    H, I, V, L = tc["hidden_size"], tc["intermediate_size"], tc["vocab_size"], tc["num_hidden_layers"]
    lin = lambda n, k: n * k + 4 * n
    per_layer = lin(3 * H, H) + lin(H, H) + lin(2 * I, H) + lin(H, I) + 2 * 2 * H
    return L * per_layer + 2 * (2 * V * H) + 2 * H + lin(H, mm_hidden) + lin(H, H) + 2 * 4 * H
