"""VAE-sized single-head d=512 attention and UNet d=128 self-attention: CUDA-event timing of uav_attention"""
import os, sys, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from upscale_a_video_b200 import ops, build
build.build()
def timeit(fn, iters=3, warmup=1):
    for _ in range(warmup): fn()
    torch.cuda.synchronize()
    s = torch.cuda.Event(enable_timing=True); e = torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters): fn()
    e.record(); torch.cuda.synchronize()
    return s.elapsed_time(e) / iters
# the d = 64 self-attention rows are no pipeline shape (the UNet's d = 64 attention is text cross-attention): they time
# the d = 64 instance of the wgmma kernel that d = 128 runs on
for name, B, heads, d, n, iters in [("vae d512 N=46080", 1, 1, 512, 46080, 3),
                                    ("vae d512 N=184320", 1, 1, 512, 184320, 3),
                                    ("unet self d128 N=2880 x16 frames", 16, 8, 128, 2880, 3),
                                    ("self d64 N=920 x16", 16, 8, 64, 920, 200),
                                    ("self d64 N=2880 x16", 16, 8, 64, 2880, 50),
                                    ("self d64 N=14400 x16", 16, 8, 64, 14400, 10)]:
    C = heads * d
    qkv = torch.randn(B, n, 3 * C, device="cuda").half()
    out = torch.empty(B, n, C, device="cuda", dtype=torch.float16)
    ms = timeit(lambda: ops.attention(qkv[..., :C], qkv[..., C:2*C], qkv[..., 2*C:], heads, out=out), iters=iters)
    print(json.dumps({"name": name, "ms": ms, "tflops_alg": 4.0 * B * n * n * C / ms / 1e9}))

# temporal attention at the top UNet level (B=2, T=8, 160x288, 8 heads x 64): 8 B/element stream
import math
B, Fr, HW, heads, d = 2, 8, 160 * 288, 8, 64
C = heads * d
qkv = torch.randn(B, Fr, HW, 3 * C, device="cuda").half()
q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
freqs = 1.0 / (10000 ** (torch.arange(0, 32, 2).float() / 32))
ang = torch.arange(Fr).float()[:, None] * freqs[None, :]
rot = torch.stack([ang.cos(), ang.sin()], dim=-1).contiguous().cuda()
bias = (torch.randn(heads, Fr, Fr) * 0.3).cuda()
out = torch.empty(B, Fr, HW, C, device="cuda", dtype=torch.float16)
ms = timeit(lambda: ops.temporal_attention(q, k, v, heads, rot, bias, out=out), iters=10, warmup=3)
print(json.dumps({"name": "temporal attn 2x8x46080 h8 d64",
                  "ms": ms, "GBps": 4 * B * Fr * HW * C * 2 / ms / 1e6}))

# clips longer than 8 frames (online-softmax kernel) at the largest temporal-attention site of the h720 UNet:
# B=2, 90x160 pixels, 8 heads x 64
for Fr in (16, 32):
    B, HW, heads, d = 2, 90 * 160, 8, 64
    C = heads * d
    qkv = torch.randn(B, Fr, HW, 3 * C, device="cuda").half()
    q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
    ang = torch.arange(Fr).float()[:, None] * freqs[None, :]
    rot = torch.stack([ang.cos(), ang.sin()], dim=-1).contiguous().cuda()
    bias = (torch.randn(heads, Fr, Fr) * 0.3).cuda()
    out = torch.empty(B, Fr, HW, C, device="cuda", dtype=torch.float16)
    ms = timeit(lambda: ops.temporal_attention(q, k, v, heads, rot, bias, out=out), iters=10, warmup=3)
    print(json.dumps({"name": f"temporal attn 2x{Fr}x{HW} h8 d64",
                      "ms": ms, "GBps": 4 * B * Fr * HW * C * 2 / ms / 1e6}))

# text cross-attention at the top UNet level: 16 frames x 46080 queries, 77 keys, 8 heads x 64 (4 B/element stream of q, o)
B, heads, d, nq, nk = 16, 8, 64, 46080, 77
C = heads * d
q = torch.randn(B, nq, C, device="cuda").half()
kv = torch.randn(2, nk, 2 * C, device="cuda").half()
out = torch.empty(B, nq, C, device="cuda", dtype=torch.float16)
ms = timeit(lambda: ops.attention(q, kv[..., :C], kv[..., C:], heads, kv_batch_div=8, out=out), iters=10, warmup=3)
print(json.dumps({"name": "cross attn b16 h8 d64 nq46080 nk77", "ms": ms, "GBps": 2 * B * nq * C * 2 / ms / 1e6}))
