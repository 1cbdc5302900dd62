"""GroupNorm(+SiLU) apply pass alone, CUDA events, buffers rotated so that no launch finds its input in L2."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from upscale_a_video_b200 import ops

dev = torch.device("cuda")
SHAPES = [(16, 160, 288, 512), (16, 320, 576, 256), (16, 320, 576, 512), (16, 80, 144, 512), (16, 40, 72, 1024)]
for shp in SHAPES:
    n, h, w, c = shp
    nbuf = max(2, int(1.5e9 // (n * h * w * c * 2)) + 1)
    xs = [torch.randn(shp, device=dev).half() for _ in range(nbuf)]
    out = torch.empty(shp, device=dev, dtype=torch.float16)
    g, b = torch.rand(c, device=dev) + 0.5, torch.randn(c, device=dev) * 0.1
    for silu in (True, False):
        for x in xs[:2]:
            ops.group_norm(x, g, b, 32, 1e-5, silu=silu, n_outer=n, out=out)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        iters = 4 * nbuf
        e0.record()
        for i in range(iters):
            ops.group_norm(xs[i % nbuf], g, b, 32, 1e-5, silu=silu, n_outer=n, out=out)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / iters
        gb = 3 * n * h * w * c * 2 / 1e9   # statistics read + apply read + write
        print(f"gn {n}x{h}x{w} C{c} silu={int(silu)}: {ms * 1000:8.1f} us  {gb / ms * 1000:7.0f} GB/s (3 passes)")
    del xs, out
    torch.cuda.empty_cache()
