"""Implicit-GEMM time of one h720 UNet forward (B=2 = the two CFG halves, T=8, 180x320, as the pipeline calls it),
bucketed by the kind of fused epilogue (bias only, or which of residual / statistics / row vector / activation /
out_scale it carries) and by single-tap (Linear, 1x1 and (1,1,1) convs) against multi-tap launches.  Per-launch CUDA
events from `ops.Profile`; prints the card and its power limit."""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from upscale_a_video_b200 import UNetVideoModel, ops
from upscale_a_video_b200.synthetic import seeded_state_dict

smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip()
print(f"device: {torch.cuda.get_device_name()} | {smi}")


def single_tap(fn, args):
    if fn == "uav_linear":
        return True
    if fn == "uav_conv2d":
        return args[8] == 1 and args[9] == 1  # ksize, stride
    if fn == "uav_conv_temporal":
        return args[8] == 1
    return False


def epilogue_kind(e):
    parts = [name for name, on in (("residual", bool(e.residual)), ("stats", bool(e.gn_partial)),
                                   ("rowvec", bool(e.rowvec)),
                                   ("act", e.act not in (ops.ACT_NONE, ops.ACT_GEGLU)),
                                   ("out_scale", e.out_scale not in (0.0, 1.0))) if on]
    return "+".join(parts) if parts else ("geglu" if e.act == ops.ACT_GEGLU else "bias")


_igemm = ops._igemm


def tagged_igemm(fn, args, out, e, st, flops, nbytes, tag=""):
    kind = f"{'single' if single_tap(fn, args) else 'multi'}-tap {epilogue_kind(e)}"
    return _igemm(fn, args, out, e, st, flops, nbytes, f"{kind}|{tag}")


ops._igemm = tagged_igemm

dev = torch.device("cuda")
cfg = json.load(open(os.path.join(os.path.dirname(__file__), "..", "upscale_a_video_b200", "configs",
                                  "unet_video_config.json")))
unet = UNetVideoModel.from_config(cfg)
unet.load_state_dict(seeded_state_dict(unet, 1234))
unet = unet.half().eval().to(dev)
H, W = 180, 320
lat = torch.randn(1, 4, 8, H, W, device=dev, dtype=torch.float16).repeat(2, 1, 1, 1, 1)
low = torch.randn(1, 3, 8, H, W, device=dev, dtype=torch.float16).repeat(2, 1, 1, 1, 1)
ctx = (torch.randn(2, 77, 1024, device=dev) * 0.3).half()
kw = dict(encoder_hidden_states=ctx, class_labels=torch.tensor([120]), cfg_shared_input=True)

for _ in range(2):
    unet(lat, 500, low, **kw)
with ops.Profile() as prof:
    unet(lat, 500, low, **kw)
buckets = {}
total = 0.0
for (kind, tag), d in prof.by_tag().items():
    if kind != "igemm":
        continue
    b = buckets.setdefault(tag.split("|")[0], dict(ms=0.0, launches=0, flops=0.0))
    b["ms"] += d["ms"]
    b["launches"] += d["launches"]
    b["flops"] += d["flops"]
    total += d["ms"]
print(f"igemm total {total:.1f} ms per forward")
for k, b in sorted(buckets.items(), key=lambda kv: -kv[1]["ms"]):
    print(f"{b['ms']:8.2f} ms {100 * b['ms'] / total:5.1f}%  x{b['launches']:3d}  {b['flops'] / b['ms'] / 1e9:6.0f} TF/s  {k}")
