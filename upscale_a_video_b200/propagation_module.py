"""Propagation — drop-in for /root/reference/models_video/propagation_module.py:152-281 (`learnable=False`,
the only branch alive at inference: inference_upscale_a_video.py:126).

Bidirectional recurrent flow-guided warp of the x0 latents with a forward/backward-consistency mask.  The
reference issues ~10 tiny ATen kernels per frame (meshgrid, 2x grid_sample, square/sum/compare, blends); here
each frame update is one fused kernel (`uav_propagate_step`, csrc/sampler.cu) that replays the reference's fp16
rounding sequence (SURVEY.md fact 8: coordinates are fp16, nearest sampling).  The recurrence over frames is
inherently sequential (each warp reads arbitrary pixels of the previous result), so there are 2*(T-1) launches."""
from __future__ import annotations

import torch
from torch import nn

from . import ops
from . import _lib


class Propagation(nn.Module):
    def __init__(self, in_channels, mid_channels=256, max_residue_magnitude=10, num_blocks=2, learnable=True):
        super().__init__()
        self.learnable = learnable
        self.module = ["backward_prop", "forward_prop"]
        if learnable:
            raise NotImplementedError(
                "Propagation(learnable=True) (DeformableAlignment / ConvResidualBlocks) is dead code at inference "
                "(inference_upscale_a_video.py:126 builds learnable=False) and is out of scope of the uav_b200 path")

    @torch.no_grad()
    def forward(self, x, flows_forward, flows_backward, interpolation="bilinear", mode="fuse", fuse_scale=0.5,
                alpha1=0.01, alpha2=0.5):
        """x: (b, c, t, h, w); flows: (b, 2, t_f, h_f, w_f) on x's device.  Returns (b, c, t, h, w).
        Flows of another shape than (t-1, h, w) are area-resized to it and scaled by w / w_f, in their own dtype, as the
        reference does (propagation_module.py:206-209); at (t-1, h, w) that resize is the identity and is skipped."""
        _lib.require_cuda(x, "Propagation")
        b, c, t, h, w = x.shape
        if interpolation not in ("nearest", "bilinear") or mode not in ("fuse", "copy"):
            raise ValueError(f"unsupported interpolation/mode {interpolation}/{mode}")
        s = 1.0 * w / flows_forward.shape[-1]  # both flows take the forward flow's width ratio, as in the reference
        if tuple(flows_forward.shape[2:]) != (t - 1, h, w) or s != 1.0:
            flows_forward = ops.flow_resize_area(flows_forward, (t - 1, h, w), s)
        if tuple(flows_backward.shape[2:]) != (t - 1, h, w) or s != 1.0:
            flows_backward = ops.flow_resize_area(flows_backward, (t - 1, h, w), s)
        x = x.contiguous()
        ff = flows_forward.to(x.dtype).contiguous()
        fb = flows_backward.to(x.dtype).contiguous()
        cur = x
        for name in self.module:
            out = torch.empty_like(x)
            if "backward" in name:
                frame_idx = list(range(t))[::-1]
                flow_idx = frame_idx
                f_prop, f_check = ff, fb
            else:
                frame_idx = list(range(t))
                flow_idx = list(range(-1, t - 1))
                f_prop, f_check = fb, ff
            for bi in range(b):
                prev = None
                for i, idx in enumerate(frame_idx):
                    if i == 0:
                        out[bi, :, idx].copy_(cur[bi, :, idx])
                    else:
                        ops.propagate_step(out[bi, :, prev], cur[bi, :, idx], f_prop[bi, :, flow_idx[i]],
                                           f_check[bi, :, flow_idx[i]], out[bi, :, idx],
                                           nearest=(interpolation == "nearest"), fuse=(mode == "fuse"),
                                           fuse_scale=float(fuse_scale), alpha1=float(alpha1), alpha2=float(alpha2),
                                           half_grid_sample=False)
                    prev = idx
            cur = out
        return cur


class EmptyPropagation(nn.Module):
    def forward(self, feats_in, flows_forward, flows_backward):
        return feats_in
