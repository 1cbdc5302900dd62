"""Linear K=512 -> N=512 at M = 737 280 (the most frequent launch of a UNet forward: 39 of 319) alone, with and without
the residual operand / statistics / out_scale / row vector epilogue, the single-tap GEMMs of the default h720 clip (16 x 90x160,
45x80 and 23x40 tokens per level, the VAE's 16 x 180x320 pixels), and the two few-wave h720 3x3 convolutions plus one
many-wave one that WIDE_TILE_COST in igemm.cu is calibrated on, each also with GroupNorm statistics and with a residual,
and the conv1 / conv2 epilogues of a ResNet block at 16 x 180x320 x 256 and 16 x 90x160 x 512.
Inputs rotated past L2.  Prints ms, TFLOP/s and the HBM rate of the algorithmic bytes, with the card and its power
limit."""
import os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from upscale_a_video_b200 import ops

dev = torch.device("cuda")
print({k: v for k, v in os.environ.items() if k.startswith("UAV_")})
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip()
print(f"device: {torch.cuda.get_device_name()} | {smi}")


def timed(one, iters):
    for i in range(3):
        one(i)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        one(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def run(M, K, N, residual, gn_stats, act=0, nbuf=3, iters=12, out_scale=1.0, rowvec=False):
    a = [torch.randn(16, M // 16, K, device=dev).half() for _ in range(nbuf)]
    w = (torch.randn(N, K, device=dev) * 0.02).half()
    b = torch.zeros(N, device=dev)
    n_out = N // 2 if act == 2 else N
    outs = [torch.empty(16, M // 16, n_out, device=dev, dtype=torch.float16) for _ in range(nbuf)]
    res = [torch.randn(16, M // 16, n_out, device=dev).half() for _ in range(nbuf)] if residual else None
    rv = torch.randn(16, n_out, device=dev).half() if rowvec else None  # one row vector per image, as conv1's temb

    def one(i):
        ops.linear(a[i % nbuf], w, b, out=outs[i % nbuf], residual=res[i % nbuf] if residual else None, act=act,
                   gn_stats=gn_stats, out_scale=out_scale, rowvec=rv, rows_per_vec=M // 16)
    ms = timed(one, iters)
    gb = 2.0 * (M * K + M * n_out * (2 if residual else 1) + N * K) / 1e9
    print(f"linear M{M} K{K} N{N} act{act} residual={int(residual)} gn_stats={int(gn_stats)}"
          f"{' rowvec=1' if rowvec else ''}"
          f"{f' out_scale={out_scale}' if out_scale != 1.0 else ''}: {ms * 1000:7.1f} us  "
          f"{2.0 * M * K * N / ms / 1e9:6.0f} TF/s  {gb / ms * 1000:6.0f} GB/s")


def conv3x3(NB, H, W, Cin, Cout, slices=1, nbuf=3, iters=12, residual=False, gn_stats=False, rowvec=False):
    """3x3 conv; slices > 1 runs it as that many launches of Cout / slices channels each (128 -> 128-column tiles)"""
    x = [torch.randn(NB, H, W, Cin, device=dev).half() for _ in range(nbuf)]
    w = (torch.randn(Cout, 3, 3, Cin, device=dev) * 0.02).half()
    b = torch.zeros(Cout, device=dev)
    outs = [torch.empty(NB, H, W, Cout, device=dev, dtype=torch.float16) for _ in range(nbuf)]
    res = [torch.randn(NB, H, W, Cout, device=dev).half() for _ in range(nbuf)] if residual else None
    rv = torch.randn(NB, Cout, device=dev).half() if rowvec else None  # one row vector per image, as conv1's temb
    step = Cout // slices
    ws = [w[s * step:(s + 1) * step].contiguous() for s in range(slices)]
    bs = [b[s * step:(s + 1) * step].contiguous() for s in range(slices)]

    def one(i):
        for s in range(slices):
            ops.conv2d(x[i % nbuf], ws[s], bs[s], out=outs[i % nbuf][..., s * step:(s + 1) * step],
                       residual=res[i % nbuf][..., s * step:(s + 1) * step] if residual else None, gn_stats=gn_stats,
                       rowvec=rv[:, s * step:(s + 1) * step] if rowvec else None, rows_per_vec=H * W)
    ms = timed(one, iters)
    print(f"conv3x3 {NB}x{H}x{W} {Cin}->{Cout} in {slices} launch(es) residual={int(residual)} gn_stats={int(gn_stats)}"
          f"{' rowvec=1' if rowvec else ''}: "
          f"{ms * 1000:7.1f} us  "
          f"{2.0 * NB * H * W * Cin * Cout * 9 / ms / 1e9:6.0f} TF/s")


for residual, gn in ((False, False), (True, False), (True, True), (False, True)):
    run(737280, 512, 512, residual, gn)
run(737280, 512, 512, False, False, out_scale=0.5)  # AUX code without the residual's wait
run(737280, 512, 512, False, True, rowvec=True)
run(737280, 512, 1536, False, False)
run(737280, 2048, 512, True, False)
run(737280, 512, 4096, False, False, act=2)
run(184320, 512, 512, True, False, nbuf=8, iters=32)
run(46080, 1024, 1024, True, False, nbuf=16, iters=64)
# h720: 16 x 90x160 tokens at level 1, 45x80 at level 2, 23x40 at level 3, the VAE at 16 x 180x320
run(230400, 512, 512, False, False, nbuf=4, iters=24)
run(230400, 512, 512, True, True, nbuf=4, iters=24)
run(230400, 512, 1536, False, False, nbuf=4, iters=24)
run(230400, 2048, 512, True, False, nbuf=4, iters=24)
run(57600, 512, 512, True, False, nbuf=16, iters=64)
run(14720, 1024, 1024, True, False, nbuf=16, iters=64)
run(921600, 256, 256, True, False, nbuf=3, iters=12)
for residual, gn in ((False, False), (False, True), (True, True)):
    conv3x3(16, 45, 80, 512, 512, iters=32, residual=residual, gn_stats=gn)
    conv3x3(16, 23, 40, 1024, 1024, iters=32, residual=residual, gn_stats=gn)
    conv3x3(16, 90, 160, 512, 512, residual=residual, gn_stats=gn)
conv3x3(16, 90, 160, 512, 512, slices=4)
# the epilogues of conv1 (row vector + statistics) and conv2 (residual + statistics) of the h720 ResNet blocks at the
# VAE's 180x320 x 256 channels and the UNet's 90x160 x 512
for residual, rowvec in ((False, False), (False, True), (True, False)):
    conv3x3(16, 180, 320, 256, 256, residual=residual, gn_stats=residual or rowvec, rowvec=rowvec)
    conv3x3(16, 90, 160, 512, 512, residual=residual, gn_stats=residual or rowvec, rowvec=rowvec)
