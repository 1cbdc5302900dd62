"""Micro-benchmark of the implicit-GEMM kernel on UNet shapes (SURVEY.md Appendix A and the h720 clip of bench.py).
CUDA-event timing; "block_n" is the tile width of the igemm_kernel instance that ran (from torch.profiler)."""
import json
import re
import sys
import os

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from upscale_a_video_b200 import build, ops

build.build()
torch.manual_seed(0)
dev = "cuda"


def timeit(fn, iters=10, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    s = torch.cuda.Event(enable_timing=True)
    e = torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def block_n(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sorted({int(m.group(1)) for ev in prof.events() for m in [re.search(r"igemm_kernel<(\d+),", ev.name)] if m})


cases = []
# (name, NB, H, W, Cin, Cout, k); NB = 16 is the two guidance halves of an 8-frame clip
for name, NB, H, W, Cin, Cout, k in [
    ("h720 conv3x3 256->256 @180x320", 16, 180, 320, 256, 256, 3),
    ("h720 conv3x3 768->256 @180x320", 16, 180, 320, 768, 256, 3),
    ("h720 conv3x3 512->512 @90x160", 16, 90, 160, 512, 512, 3),
    ("h720 conv3x3 512->512 @45x80", 16, 45, 80, 512, 512, 3),
    ("h720 conv3x3 1024->1024 @23x40", 16, 23, 40, 1024, 1024, 3),
    ("conv3x3 512->512 @160x288", 16, 160, 288, 512, 512, 3),
    ("conv3x3 256->256 @320x576", 16, 320, 576, 256, 256, 3),
    ("conv3x3 1024->1024 @40x72", 16, 40, 72, 1024, 1024, 3),
    ("conv3x3 512->512 @320x576", 8, 320, 576, 512, 512, 3),
    ("conv1x1 512->512 @160x288", 16, 160, 288, 512, 512, 1),
]:
    x = torch.randn(NB, H, W, Cin, device=dev).half()
    w = (torch.randn(Cout, k, k, Cin, device=dev) * 0.02).half()
    b = torch.zeros(Cout, device=dev)
    out = torch.empty(NB, H, W, Cout, device=dev, dtype=torch.float16)
    ms = timeit(lambda: ops.conv2d(x, w, b, out=out))
    fl = 2.0 * NB * H * W * Cin * Cout * k * k
    cases.append({"name": name, "ms": ms, "tflops": fl / ms / 1e9, "block_n": block_n(lambda: ops.conv2d(x, w, b, out=out))})
    del x, w, out

for name, M, K, N, act in [("h720 linear 512->512 M=230400", 230400, 512, 512, 0),
                           ("h720 geglu 512->4096 M=230400", 230400, 512, 4096, 2),
                           ("h720 linear 2048->512 M=230400", 230400, 2048, 512, 0),
                           ("linear 512->512 M=737280", 737280, 512, 512, 0),
                           ("geglu 512->4096 M=184320", 184320, 512, 4096, 2),
                           ("linear 2048->512 M=184320", 184320, 2048, 512, 0)]:
    a = torch.randn(M, K, device=dev).half()
    w = (torch.randn(N, K, device=dev) * 0.02).half()
    b = torch.zeros(N, device=dev)
    ms = timeit(lambda: ops.linear(a, w, b, act=act))
    cases.append({"name": name, "ms": ms, "tflops": 2.0 * M * K * N / ms / 1e9, "block_n": block_n(lambda: ops.linear(a, w, b, act=act))})
    del a, w

x = torch.randn(2, 8, 160, 288, 512, device=dev).half()
w = (torch.randn(512, 3, 512, device=dev) * 0.02).half()
b = torch.zeros(512, device=dev)
ms = timeit(lambda: ops.conv_temporal(x, w, b))
cases.append({"name": "conv_t3 512 @160x288", "ms": ms, "tflops": 2.0 * x.numel() * 512 * 3 / ms / 1e9,
              "block_n": block_n(lambda: ops.conv_temporal(x, w, b))})
for c in cases:
    print(json.dumps(c))
