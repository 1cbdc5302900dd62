"""per-shape timing of one UNet forward (B=2 = the two CFG halves of one clip, T=8) as the pipeline calls it
(cfg_shared_input=True): --config c2 (320x576, the default) or h720 (180x320, the clip bench.py times by default)"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from upscale_a_video_b200 import UNetVideoModel, ops
from upscale_a_video_b200.synthetic import seeded_state_dict

SIZES = {"c2": (320, 576), "h720": (180, 320)}
ap = argparse.ArgumentParser()
ap.add_argument("--config", default="c2", choices=sorted(SIZES))
H, W = SIZES[ap.parse_args().config]

dev = torch.device("cuda")
cfg = json.load(open(os.path.join(os.path.dirname(__file__), "..", "upscale_a_video_b200", "configs", "unet_video_config.json")))
unet = UNetVideoModel.from_config(cfg)
unet.load_state_dict(seeded_state_dict(unet, 1234))
unet = unet.half().eval().to(dev)
lat = torch.randn(1, 4, 8, H, W, device=dev, dtype=torch.float16).repeat(2, 1, 1, 1, 1)
low = torch.randn(1, 3, 8, H, W, device=dev, dtype=torch.float16).repeat(2, 1, 1, 1, 1)
ctx = (torch.randn(2, 77, 1024, device=dev) * 0.3).half()
kw = dict(encoder_hidden_states=ctx, class_labels=torch.tensor([120]), cfg_shared_input=True)


def run(tag, detail=False):
    for _ in range(2):
        unet(lat, 500, low, **kw)
    with ops.Profile() as prof:
        unet(lat, 500, low, **kw)
    bt = prof.by_tag()
    tot = sum(d["ms"] for d in bt.values())
    kinds = {}
    for (kind, _), d in bt.items():
        kinds[kind] = kinds.get(kind, 0.0) + d["ms"]
    print(f"[{tag}] total {tot:.1f} ms  " + "  ".join(f"{k} {v:.1f}" for k, v in sorted(kinds.items(), key=lambda kv: -kv[1])))
    if detail:
        for (kind, t), d in sorted(bt.items(), key=lambda kv: -kv[1]["ms"])[:60]:
            tf = d["flops"] / d["ms"] / 1e9 if d["flops"] else 0
            gb = d["bytes"] / d["ms"] / 1e6
            print(f"{d['ms']:8.2f} ms {100 * d['ms'] / tot:5.1f}%  x{d['launches']:3d}  {tf:7.0f} TF/s {gb:7.0f} GB/s  {kind:10s} {t}")
    return tot


run("default", detail=True)
