"""Parameter containers with the reference's module / state-dict names + the channels-last CUDA forward of
every block on the sampling path.

The classes mirror /root/reference/models_video/{resnet,attention,temporal_module,unet_blocks}.py by NAME and by
parameter layout (so `load_state_dict(strict=True)` of a reference checkpoint works), but they hold parameters
only: the arithmetic is in `csrc/` behind the C ABI and is driven by the `forward` methods below on fp16
channels-last tensors (b, t, h, w, c).  `torch.nn.{Conv2d,Conv3d,Linear,GroupNorm,LayerNorm,Embedding}` are used
purely as parameter holders (their own forward is never called).

Kernel-ready weights (K-major fp16 conv filters, fused q/k/v matrices, fp32 affine vectors) are packed lazily by
`Packed` and cached until the parameters change (`_apply` / `load_state_dict`).
"""
from __future__ import annotations

from typing import Dict, Optional

import torch
from torch import nn

from . import ops


# ------------------------------------------------------------------------------------------------
# packed weights
# ------------------------------------------------------------------------------------------------
def _pad8(n: int) -> int:
    return (n + 7) // 8 * 8


class Packed:
    """kernel-ready views of a module tree's parameters, keyed by parameter name"""

    def __init__(self, root: nn.Module):
        self.root = root
        self.cache: Dict[str, torch.Tensor] = {}

    def clear(self):
        self.cache.clear()

    def conv(self, m: nn.Module, bias_scale: float = 1.0):
        """-> (weight [Cout][taps...][Cin_pad8] fp16, bias fp32 | None); `bias_scale`: the bias of a conv that maps a
        residual stream kept at `bias_scale` x the reference's values onto itself (linear in x: only the bias rescales)"""
        if bias_scale != 1.0:
            key = (id(m), "bias_scale", bias_scale)
            if key not in self.cache:
                w, b = self.conv(m)
                self.cache[key] = (w, None if b is None else (b * bias_scale).contiguous())
            return self.cache[key]
        key = id(m)
        if key not in self.cache:
            w = m.weight.detach()
            cin = w.shape[1]
            if w.dim() == 4:
                wp = w.permute(0, 2, 3, 1)
            elif w.shape[3] == 1 and w.shape[4] == 1:
                wp = w[:, :, :, 0, 0].permute(0, 2, 1)
            else:
                wp = w.permute(0, 2, 3, 4, 1)
            if cin % 8:
                wp = torch.nn.functional.pad(wp, (0, _pad8(cin) - cin))
            self.cache[key] = (wp.to(torch.float16).contiguous(),
                               None if m.bias is None else m.bias.detach().float().contiguous())
        return self.cache[key]

    def linear(self, m: nn.Module):
        key = id(m)
        if key not in self.cache:
            self.cache[key] = (m.weight.detach().to(torch.float16).contiguous(),
                               None if m.bias is None else m.bias.detach().float().contiguous())
        return self.cache[key]

    def fused_linear(self, key: str, mods):
        """row-concatenated weights of several Linear layers sharing one input (q|k|v, k|v, all temb projections)"""
        if key not in self.cache:
            w = torch.cat([m.weight.detach().to(torch.float16) for m in mods], dim=0).contiguous()
            if all(m.bias is None for m in mods):
                b = None
            else:
                b = torch.cat([(m.bias.detach().float() if m.bias is not None else
                                torch.zeros(m.weight.shape[0], device=w.device)) for m in mods]).contiguous()
            self.cache[key] = (w, b)
        return self.cache[key]

    def affine(self, m: nn.Module):
        key = id(m)
        if key not in self.cache:
            self.cache[key] = (m.weight.detach().float().contiguous(), m.bias.detach().float().contiguous())
        return self.cache[key]

    def tensor(self, key: str, fn):
        if key not in self.cache:
            self.cache[key] = fn()
        return self.cache[key]


class PackedModule(nn.Module):
    """root module mixin: owns the Packed cache and invalidates it when parameters move / change"""

    def _packed(self) -> Packed:
        pk = self.__dict__.get("_pk")
        if pk is None:
            pk = Packed(self)
            self.__dict__["_pk"] = pk
        return pk

    def _apply(self, fn, *args, **kwargs):
        r = super()._apply(fn, *args, **kwargs)
        if self.__dict__.get("_pk") is not None:
            self.__dict__["_pk"].clear()
        return r

    def load_state_dict(self, *args, **kwargs):
        r = super().load_state_dict(*args, **kwargs)
        if self.__dict__.get("_pk") is not None:
            self.__dict__["_pk"].clear()
        return r


# ------------------------------------------------------------------------------------------------
# forward context
# ------------------------------------------------------------------------------------------------
class Ctx:
    """per-forward state: packed weights, the batched time-embedding projections, cached prompt K/V"""

    def __init__(self, pk: Packed):
        self.pk = pk
        self.temb_all: Optional[torch.Tensor] = None    # (B, sum Cout) fp16
        self.temb_slices: Dict[int, tuple] = {}          # id(resnet) -> (col0, col1)
        self.ctx_kv: Optional[torch.Tensor] = None       # (B*77, sum 2C) fp16
        self.ctx_slices: Dict[int, tuple] = {}           # id(attn) -> (col0, C)
        self.ctx_len = 0
        self.rot: Optional[torch.Tensor] = None
        self.rel_bias: Dict[int, torch.Tensor] = {}

    def temb(self, resnet):
        if self.temb_all is None or id(resnet) not in self.temb_slices:
            return None
        c0, c1 = self.temb_slices[id(resnet)]
        return self.temb_all[:, c0:c1]


# ------------------------------------------------------------------------------------------------
# resnet.py
# ------------------------------------------------------------------------------------------------
class InflatedConv3d(nn.Conv2d):
    """resnet.py:94-101 — parameter holder; executed by `ops.conv2d` on (b, t, h, w, c)"""

    def run(self, c: Ctx, x, bias_scale: float = 1.0, **epi):
        w, b = c.pk.conv(self, bias_scale)
        stride = self.stride[0]
        if stride == 2:
            pad_mode = 0 if self.padding[0] == 1 else 1
            H, W = x.shape[-3], x.shape[-2]
            if H % 2 or W % 2:  # zero row/col == the conv's own zero padding (exact)
                xp = torch.zeros(*x.shape[:-3], H + H % 2, W + W % 2, x.shape[-1], dtype=x.dtype, device=x.device)
                xp[..., :H, :W, :].copy_(x)  # strided plumbing copy (only for odd sizes, e.g. 45 -> 23 at 180x320)
                x = xp
            y = self._launch(x, w, b, dict(stride=2, pad_mode=pad_mode), epi)
            if pad_mode == 1 and (H % 2 or W % 2):
                # F.pad (0,1,0,1) + unpadded stride-2 conv (resnet.py:188-192) yields floor((H - 2) / 2) + 1 rows: for an odd
                # H the even-padded launch computed one extra row / column from padding only — drop it
                ho, wo = (H - 2) // 2 + 1, (W - 2) // 2 + 1
                if (ho, wo) != tuple(y.shape[-3:-1]):
                    y = y[..., :ho, :wo, :].contiguous()
            return y
        return self._launch(x, w, b, {}, epi)

    @staticmethod
    def _launch(x, w, b, kw, epi):
        cout = w.shape[0]
        if cout % 8 and epi.get("out") is None and epi.get("out_dtype", torch.float16) == torch.float16:
            # keep the channels-last invariant "pixel stride % 8 == 0": zero-padded buffer, conv writes [:cout];
            # downstream filters are zero-padded on Cin, so the pad channels contribute exactly 0
            H, W = x.shape[-3], x.shape[-2]
            if kw.get("stride", 1) == 2:
                H, W = H // 2, W // 2
            buf = torch.zeros(*x.shape[:-3], H, W, _pad8(cout), dtype=torch.float16, device=x.device)
            ops.conv2d(x, w, b, out=buf[..., :cout], **kw, **epi)
            return buf
        return ops.conv2d(x, w, b, **kw, **epi)


def _gn(c: Ctx, norm: nn.GroupNorm, x, silu: bool, n_outer: int, stream_scale: float = 1.0):
    """`stream_scale`: x holds stream_scale x the reference's values; GroupNorm(s x) with eps s^2 == GroupNorm(x) with eps"""
    g, b = c.pk.affine(norm)
    C = norm.num_channels
    eps = norm.eps * stream_scale * stream_scale
    if x.shape[-1] != C:  # logical C channels inside a zero-padded buffer (e.g. the 3-channel LR frames)
        out = torch.zeros_like(x)
        ops.group_norm(x[..., :C], g, b, norm.num_groups, eps, silu=silu, n_outer=n_outer, out=out[..., :C])
        return out
    return ops.group_norm(x, g, b, norm.num_groups, eps, silu=silu, n_outer=n_outer, stats=getattr(x, "uav_gn", None),
                          batch=x.shape[0])


def _split_1x1(conv, cx: int):
    """1x1 conv weight (Cout, Cx + Cs, 1, 1) -> ([Cout][Cx], [Cout][Cs]) fp16 K-major blocks + fp32 bias"""
    w = conv.weight.detach()[:, :, 0, 0]
    return (w[:, :cx].to(torch.float16).contiguous(), w[:, cx:].to(torch.float16).contiguous(),
            None if conv.bias is None else conv.bias.detach().float().contiguous())


def _carry_gn(dst, src):
    """a reshaped view of a produced tensor keeps the producer's GroupNorm statistics and its concat-buffer membership"""
    for name in ("uav_gn", "uav_cat"):
        st = getattr(src, name, None)
        if st is not None:
            setattr(dst, name, st)
    return dst


# skip-connection concat without the copy of the main branch (unet_blocks.py:573,645 `torch.cat([hidden_states,
# res_hidden_states], dim=1)`): the concat buffer is allocated BEFORE the layer that produces hidden_states runs, the skip
# is copied into its tail (a skip computed once for both classifier-free-guidance halves is broadcast there) and the
# producer's epilogue stores straight into the head slice (`out=`).
# ... and where both halves carry the GroupNorm statistics of their producers, the concat is never built at all
# (ResnetBlock3D.forward_cat): norm1 normalises the two tensors straight into ONE dense tensor (ops.group_norm_cat) and the
# 1x1 conv_shortcut over the concat is split into its two column blocks.
def new_cat_slot(skip, cx: int, batch: int, producer_has_stats: bool = False):
    """-> the head slice (batch, t, h, w, cx) of a fresh concat buffer whose tail already holds `skip`; the producer of
    the main branch writes into it and `cat_with_skip` later returns the whole buffer.  None (plain allocation by the
    producer) when the concat will not be materialised at all."""
    if producer_has_stats and getattr(skip, "uav_gn", None):
        return None
    cs = skip.shape[-1]
    buf = torch.empty(batch, *skip.shape[1:-1], cx + cs, dtype=skip.dtype, device=skip.device)
    if skip.shape[0] == 1 and batch > 1:
        for i in range(batch):
            ops.copy_channels(skip, buf[i:i + 1, ..., cx:])
    else:
        ops.copy_channels(skip, buf[..., cx:])
    slot = buf[..., :cx]
    slot.uav_cat = (buf, skip)
    return slot


def cat_with_skip(x, skip):
    cat = getattr(x, "uav_cat", None)
    if cat is not None and cat[1] is skip:
        buf = cat[0]
        ga, gb = getattr(x, "uav_gn", None), getattr(skip, "uav_gn", None)
        if ga and gb:
            buf.uav_gn = list(ga) + list(gb)
        return buf
    return ops.concat_channels(x, skip)


class ResnetBlock3D(nn.Module):
    """resnet.py:200-294"""

    def __init__(self, *, in_channels, out_channels=None, temb_channels=512, groups=32, groups_out=None, eps=1e-6,
                 output_scale_factor=1.0, **_):
        super().__init__()
        out_channels = in_channels if out_channels is None else out_channels
        groups_out = groups if groups_out is None else groups_out
        self.in_channels, self.out_channels = in_channels, out_channels
        assert output_scale_factor == 1.0, "output_scale_factor != 1 is not used by any shipped config"
        self.norm1 = nn.GroupNorm(groups, in_channels, eps=eps, affine=True)
        self.conv1 = InflatedConv3d(in_channels, out_channels, kernel_size=3, stride=1, padding=1)
        self.time_emb_proj = nn.Linear(temb_channels, out_channels) if temb_channels is not None else None
        self.norm2 = nn.GroupNorm(groups_out, out_channels, eps=eps, affine=True)
        self.conv2 = InflatedConv3d(out_channels, out_channels, kernel_size=3, stride=1, padding=1)
        self.conv_shortcut = (InflatedConv3d(in_channels, out_channels, kernel_size=1, stride=1, padding=0)
                              if in_channels != out_channels else None)

    def _convs(self, c, h, which, **epi):
        return getattr(self, which).run(c, h, **epi)

    def forward_cat(self, c: Ctx, x, skip, out=None):
        """forward(torch.cat([x, skip], channel)) (unet_blocks.py:573,645) without building the concatenation when both
        tensors carry their producers' GroupNorm statistics; otherwise through the (in-place) concat buffer"""
        h = None
        if (self.conv_shortcut is not None and isinstance(self.conv_shortcut, InflatedConv3d)
                and getattr(x, "uav_cat", None) is None):
            g, b = c.pk.affine(self.norm1)
            h = ops.group_norm_cat([x, skip], g, b, self.norm1.num_groups, self.norm1.eps, silu=True, n_outer=x.shape[0])
        if h is None:
            return self.forward(c, cat_with_skip(x, skip), out=out)
        B = x.shape[0]
        thw = x.shape[1] * x.shape[2] * x.shape[3]
        temb = c.temb(self) if self.time_emb_proj is not None else None
        h = self._convs(c, h, "conv1", rowvec=temb, rows_per_vec=thw, gn_stats=True)
        h = _gn(c, self.norm2, h, True, B)
        # conv_shortcut(cat) = Wx x + Ws skip + b: the skip half first (once, if the skip is shared by the batch items)
        cx = x.shape[-1]
        wx, ws, bias = c.pk.tensor(f"shortcut_split{id(self.conv_shortcut)}_{cx}", lambda: _split_1x1(self.conv_shortcut, cx))
        s1 = ops.linear(skip, ws, None)
        if skip.shape[0] == B:
            xs = ops.linear(x, wx, bias, residual=s1)
        else:
            xs = torch.empty(*x.shape[:-1], wx.shape[0], dtype=torch.float16, device=x.device)
            for n in range(B):
                ops.linear(x[n:n + 1], wx, bias, residual=s1, out=xs[n:n + 1])
        return self._convs(c, h, "conv2", residual=xs, gn_stats=True, out=out)

    def forward(self, c: Ctx, x, stream_scale: float = 1.0, out=None):
        """`stream_scale` (VAE decoder): x and the result are stream_scale x the reference's residual stream;
        `out`: destination view (e.g. the head slice of the next concat buffer)"""
        B = x.shape[0]
        thw = x.shape[1] * x.shape[2] * x.shape[3]
        h = _gn(c, self.norm1, x, True, B, stream_scale)
        temb = c.temb(self) if self.time_emb_proj is not None else None
        h = self._convs(c, h, "conv1", rowvec=temb, rows_per_vec=thw, gn_stats=True)
        h = _gn(c, self.norm2, h, True, B)
        xs = x if self.conv_shortcut is None else self._convs(c, x, "conv_shortcut", bias_scale=stream_scale)
        return self._convs(c, h, "conv2", residual=xs, out_scale=stream_scale, gn_stats=True, out=out)


class TemporalConv(nn.Conv3d):
    """nn.Conv3d (k,1,1) / (1,1,1) / (3,3,3) parameter holder (resnet.py:332,348,361,461)"""

    def run(self, c: Ctx, x, bias_scale: float = 1.0, **epi):
        w, b = c.pk.conv(self, bias_scale)
        if w.dim() == 3:
            return ops.conv_temporal(x, w, b, **epi)
        epi.pop("rowvec", None)
        epi.pop("rows_per_vec", None)
        return ops.conv3d(x, w, b, **epi)


class ResnetBlock3DCNN(ResnetBlock3D):
    """resnet.py:297-393 — temporal (k,1,1) convolutions"""

    def __init__(self, *, in_channels, out_channels=None, kernel=(3, 1, 1), temb_channels=512, groups=32, eps=1e-6, **_):
        nn.Module.__init__(self)
        out_channels = in_channels if out_channels is None else out_channels
        self.in_channels, self.out_channels = in_channels, out_channels
        self.norm1 = nn.GroupNorm(groups, in_channels, eps=eps, affine=True)
        pad = tuple((k - 1) // 2 for k in kernel)
        self.conv1 = TemporalConv(in_channels, out_channels, kernel_size=kernel, stride=(1, 1, 1), padding=pad)
        self.time_emb_proj = nn.Linear(temb_channels, out_channels) if temb_channels is not None else None
        self.norm2 = nn.GroupNorm(groups, out_channels, eps=eps, affine=True)
        self.conv2 = TemporalConv(out_channels, out_channels, kernel_size=(3, 1, 1), stride=(1, 1, 1), padding=(1, 0, 0))
        self.conv_shortcut = (TemporalConv(in_channels, out_channels, kernel_size=(1, 1, 1))
                              if in_channels != out_channels else None)


class ResnetBlock3D_plus(ResnetBlock3D):
    """resnet.py:396-500 — ResnetBlock3D + GN -> SiLU -> zero-init Conv3d 3x3x3 residual (video VAE)"""

    def __init__(self, *, in_channels, out_channels=None, temb_channels=512, groups=32, groups_out=None, eps=1e-6, **kw):
        super().__init__(in_channels=in_channels, out_channels=out_channels, temb_channels=temb_channels, groups=groups,
                         groups_out=groups_out, eps=eps)
        go = groups if groups_out is None else groups_out
        self.norm_3d = nn.GroupNorm(go, self.out_channels, eps=eps, affine=True)
        self.conv_3d = TemporalConv(self.out_channels, self.out_channels, kernel_size=(3, 3, 3), stride=(1, 1, 1),
                                    padding=(1, 1, 1))
        nn.init.zeros_(self.conv_3d.weight)
        nn.init.zeros_(self.conv_3d.bias)

    def forward(self, c: Ctx, x, stream_scale: float = 1.0):
        out = super().forward(c, x, stream_scale)
        h = _gn(c, self.norm_3d, out, True, x.shape[0], stream_scale)
        return self.conv_3d.run(c, h, residual=out, out_scale=stream_scale, gn_stats=True)


class Upsample3D(nn.Module):
    """resnet.py:104-158"""

    def __init__(self, channels, use_conv=False, out_channels=None, **_):
        super().__init__()
        self.channels = channels
        self.out_channels = out_channels or channels
        self.conv = InflatedConv3d(channels, self.out_channels, 3, padding=1) if use_conv else None

    def forward(self, c: Ctx, x, output_size=None, stream_scale: float = 1.0, out=None):
        assert x.shape[-1] == self.channels
        exact2x = output_size is None or tuple(output_size[-2:]) == (2 * x.shape[-3], 2 * x.shape[-2])
        if (self.conv is not None and exact2x and self.out_channels >= 64
                and self.out_channels % 8 == 0 and self.channels % 8 == 0):
            # nearest x2 + 3x3 conv as four 2x2 phase convs on the source (4/9 of the MACs, no 4x intermediate)
            w4 = c.pk.tensor(f"up4_{id(self.conv)}",
                             lambda: ops.collapse_upsample_filter(self.conv.weight.detach().permute(0, 2, 3, 1)))
            _, b = c.pk.conv(self.conv, stream_scale)
            return ops.upsample2x_conv3x3(x, w4, b, out=out)
        x = ops.upsample_nearest(x, None if output_size is None else tuple(output_size[-2:]))
        if self.conv is None:
            assert out is None
            return x
        return self.conv.run(c, x, bias_scale=stream_scale, gn_stats=True, out=out)


class Downsample3D(nn.Module):
    """resnet.py:161-197 (use_conv=True; name='op')"""

    def __init__(self, channels, use_conv=True, out_channels=None, padding=1, name="conv"):
        super().__init__()
        assert use_conv
        self.channels, self.out_channels, self.padding = channels, out_channels or channels, padding
        self.conv = InflatedConv3d(channels, self.out_channels, 3, stride=2, padding=padding)

    def forward(self, c: Ctx, x):
        assert x.shape[-1] == self.channels
        return self.conv.run(c, x, gn_stats=True)


# ------------------------------------------------------------------------------------------------
# attention.py
# ------------------------------------------------------------------------------------------------
class CrossAttention(nn.Module):
    """attention.py:44-238 parameter holder"""

    def __init__(self, query_dim, cross_attention_dim=None, heads=8, dim_head=64, bias=False):
        super().__init__()
        inner = dim_head * heads
        self.is_cross = cross_attention_dim is not None
        kv_dim = cross_attention_dim if cross_attention_dim is not None else query_dim
        self.heads, self.dim_head, self.scale = heads, dim_head, dim_head ** -0.5
        self._use_memory_efficient_attention_xformers = False
        self.to_q = nn.Linear(query_dim, inner, bias=bias)
        self.to_k = nn.Linear(kv_dim, inner, bias=bias)
        self.to_v = nn.Linear(kv_dim, inner, bias=bias)
        self.to_out = nn.ModuleList([nn.Linear(inner, query_dim), nn.Dropout(0.0)])

    def forward(self, c: Ctx, norm, hs, frames: int):
        """hs: residual stream (B, T, HW, C); returns to_out(attn(LayerNorm(hs))) + hs."""
        B, T, HW, C = hs.shape
        if self.is_cross:
            q = _ln_linear(c, norm, [self.to_q], f"lnq{id(self)}", hs).view(B * T, HW, C)
            c0, cc = c.ctx_slices[id(self)]
            kv = c.ctx_kv.view(B, c.ctx_len, -1)
            k, v = kv[:, :, c0:c0 + cc], kv[:, :, c0 + cc:c0 + 2 * cc]
            o = ops.attention(q, k, v, self.heads, kv_batch_div=T)
        else:
            qkv = _ln_linear(c, norm, [self.to_q, self.to_k, self.to_v], f"lnqkv{id(self)}", hs).view(B * T, HW, 3 * C)
            o = ops.attention(qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:], self.heads)
        wo, bo = c.pk.linear(self.to_out[0])
        return ops.linear(o.view(B, T, HW, C), wo, bo, residual=hs)


def _ln_linear(c: Ctx, norm: nn.LayerNorm, mods, key: str, hs, **kw):
    """Linear(s) `mods` applied to LayerNorm(hs): LayerNorm kernel + one GEMM on the row-concatenated weights"""
    g, bt = c.pk.affine(norm)
    n = ops.layer_norm(hs, g, bt, norm.eps)
    w, b = c.pk.fused_linear(key, mods) if len(mods) > 1 else c.pk.linear(mods[0])
    return ops.linear(n, w, b, **kw)


class RotaryEmbedding(nn.Module):
    """rotary-embedding-torch 0.2.3 parameter holder (unet_video.py:203): `freqs` = theta^(-2j/dim)"""

    def __init__(self, dim, theta=10000):
        super().__init__()
        self.freqs = nn.Parameter(1.0 / (theta ** (torch.arange(0, dim, 2)[: dim // 2].float() / dim)), requires_grad=False)

    def table(self, n: int) -> torch.Tensor:
        """(n, dim/2, 2) fp32: cos/sin of position * freq"""
        f = self.freqs.detach().float()
        ang = torch.arange(n, device=f.device, dtype=torch.float32)[:, None] * f[None, :]
        return torch.stack([ang.cos(), ang.sin()], dim=-1).contiguous()


class RelativePositionBias(nn.Module):
    """attention.py:735-773"""

    def __init__(self, heads=8, num_buckets=32, max_distance=128):
        super().__init__()
        self.num_buckets, self.max_distance = num_buckets, max_distance
        self.relative_attention_bias = nn.Embedding(num_buckets, heads)

    def table(self, n: int) -> torch.Tensor:
        """(heads, n, n) fp32 — host-side index math (attention.py:747-773), one tiny gather on device"""
        import math
        q = torch.arange(n)
        rel = q[None, :] - q[:, None]
        nb = self.num_buckets // 2
        neg = -rel
        ret = (neg < 0).long() * nb
        a = neg.abs()
        max_exact = nb // 2
        large = max_exact + (torch.log(a.float().clamp(min=1) / max_exact) / math.log(self.max_distance / max_exact)
                             * (nb - max_exact)).long()
        large = torch.min(large, torch.full_like(large, nb - 1))
        bucket = ret + torch.where(a < max_exact, a, large)
        w = self.relative_attention_bias.weight.detach().float()
        return w[bucket.to(w.device)].permute(2, 0, 1).contiguous()


class TemporalAttention(CrossAttention):
    """attention.py:626-733"""

    def __init__(self, query_dim, heads=8, dim_head=64, bias=False, rotary_emb=None):
        super().__init__(query_dim, None, heads, dim_head, bias)
        self.time_rel_pos_bias = RelativePositionBias(heads=heads, max_distance=32)
        self.rotary_emb = rotary_emb  # shared module: the reference state dict carries `...rotary_emb.freqs` per site

    def forward(self, c: Ctx, norm, hs, frames: int):
        B, T, HW, C = hs.shape
        qkv = _ln_linear(c, norm, [self.to_q, self.to_k, self.to_v], f"lnqkv{id(self)}", hs)
        bias = c.pk.tensor(f"relbias{id(self)}_{T}", lambda: self.time_rel_pos_bias.table(T))
        o = ops.temporal_attention(qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:], self.heads, c.rot, bias)
        wo, bo = c.pk.linear(self.to_out[0])
        return ops.linear(o, wo, bo, residual=hs)


class GEGLU(nn.Module):
    def __init__(self, dim_in, dim_out):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out * 2)


class FeedForward(nn.Module):
    """diffusers FeedForward(activation_fn='geglu') parameter holder (attention.py:18,493)"""

    def __init__(self, dim, mult=4):
        super().__init__()
        self.net = nn.ModuleList([GEGLU(dim, dim * mult), nn.Dropout(0.0), nn.Linear(dim * mult, dim)])

    def forward(self, c: Ctx, norm, hs):
        g = _ln_linear(c, norm, [self.net[0].proj], f"lnff{id(self)}", hs, act=ops.ACT_GEGLU)
        w2, b2 = c.pk.linear(self.net[2])
        return ops.linear(g, w2, b2, residual=hs)


class BasicTransformerBlock(nn.Module):
    """attention.py:414-564"""

    def __init__(self, dim, num_attention_heads, attention_head_dim, cross_attention_dim=None, attention_bias=False,
                 only_cross_attention=False, rotary_emb=None):
        super().__init__()
        self.only_cross_attention = only_cross_attention
        self.attn1 = CrossAttention(dim, cross_attention_dim if only_cross_attention else None, num_attention_heads,
                                    attention_head_dim, attention_bias)
        self.norm1 = nn.LayerNorm(dim)
        if cross_attention_dim is not None:
            self.attn2 = CrossAttention(dim, cross_attention_dim, num_attention_heads, attention_head_dim, attention_bias)
            self.norm2 = nn.LayerNorm(dim)
        else:
            self.attn2, self.norm2 = None, None
        self.attn_temporal = TemporalAttention(dim, num_attention_heads, attention_head_dim, attention_bias, rotary_emb)
        nn.init.zeros_(self.attn_temporal.to_out[0].weight.data)
        self.norm_temporal = nn.LayerNorm(dim)
        self.ff = FeedForward(dim)
        self.norm3 = nn.LayerNorm(dim)

    def _ln(self, c, m, x):
        g, b = c.pk.affine(m)
        return ops.layer_norm(x, g, b, m.eps)

    def forward(self, c: Ctx, hs):
        T = hs.shape[1]
        hs = self.attn1(c, self.norm1, hs, T)
        if self.attn2 is not None:
            hs = self.attn2(c, self.norm2, hs, T)
        hs = self.attn_temporal(c, self.norm_temporal, hs, T)
        return self.ff(c, self.norm3, hs)


class Transformer3DModel(nn.Module):
    """attention.py:292-411 (use_linear_projection=True)"""

    def __init__(self, num_attention_heads=16, attention_head_dim=88, in_channels=None, num_layers=1,
                 norm_num_groups=32, cross_attention_dim=None, use_linear_projection=False, only_cross_attention=False,
                 rotary_emb=None, **_):
        super().__init__()
        assert use_linear_projection, "only use_linear_projection=True (shipped config) is implemented"
        inner = num_attention_heads * attention_head_dim
        self.in_channels = in_channels
        self.resblock_temporal = ResnetBlock3DCNN(in_channels=in_channels, kernel=(3, 1, 1), temb_channels=None)
        self.norm = nn.GroupNorm(norm_num_groups, in_channels, eps=1e-6, affine=True)
        self.proj_in = nn.Linear(in_channels, inner)
        self.transformer_blocks = nn.ModuleList([
            BasicTransformerBlock(inner, num_attention_heads, attention_head_dim, cross_attention_dim=cross_attention_dim,
                                  only_cross_attention=only_cross_attention, rotary_emb=rotary_emb)
            for _ in range(num_layers)])
        self.proj_out = nn.Linear(in_channels, inner)

    def forward(self, c: Ctx, x, out=None):
        B, T, H, W, C = x.shape
        x = self.resblock_temporal(c, x)
        hs = _gn(c, self.norm, x, False, B * T)
        w, b = c.pk.linear(self.proj_in)
        hs = ops.linear(hs.view(B, T, H * W, C), w, b)
        for blk in self.transformer_blocks:
            hs = blk(c, hs)
        w, b = c.pk.linear(self.proj_out)
        dst = None if out is None else out.view(B, T, H * W, C)
        y = ops.linear(hs, w, b, residual=x.view(B, T, H * W, C), gn_stats=True, out=dst)
        if out is not None:
            return _carry_gn(out, y)
        return _carry_gn(y.view(B, T, H, W, C), y)


# ------------------------------------------------------------------------------------------------
# temporal_module.py
# ------------------------------------------------------------------------------------------------
class TemporalModule3D(nn.Module):
    """temporal_module.py:98-194 with attention_block_types=("","") (shipped config): no attention inside"""

    def __init__(self, in_channels=None, out_channels=None, temb_channels=512, attention_block_types=("", ""), **_):
        super().__init__()
        if tuple(attention_block_types) != ("", ""):
            raise NotImplementedError("TemporalTransformer3DModel is dead under the shipped config and out of scope")
        self.resblocks_3d_temporal = ResnetBlock3DCNN(in_channels=in_channels, out_channels=in_channels, kernel=(5, 1, 1),
                                                      temb_channels=temb_channels)
        self.resblocks_3d_spatial = ResnetBlock3D(in_channels=in_channels, out_channels=in_channels,
                                                  temb_channels=temb_channels, groups=32, groups_out=32)
        self.shift_conv = InflatedConv3d(in_channels, in_channels, kernel_size=1, stride=1, padding=0)
        nn.init.zeros_(self.shift_conv.weight)
        nn.init.zeros_(self.shift_conv.bias)

    def forward(self, c: Ctx, x, out=None):
        h = self.resblocks_3d_temporal(c, x)
        h = self.resblocks_3d_spatial(c, h)
        return self.shift_conv.run(c, h, residual=x, gn_stats=True, out=out)


class EmptyTemporalModule3D(nn.Module):
    def forward(self, c: Ctx, x, out=None):
        assert out is None
        return x


# ------------------------------------------------------------------------------------------------
# unet_blocks.py (UNet side)
# ------------------------------------------------------------------------------------------------
def _t3d(heads, channels, cross_dim, groups, only_cross, rotary):
    return Transformer3DModel(heads, channels // heads, in_channels=channels, num_layers=1, cross_attention_dim=cross_dim,
                              norm_num_groups=groups, use_linear_projection=True, only_cross_attention=only_cross,
                              rotary_emb=rotary)


class DownBlock3D(nn.Module):
    """unet_blocks.py:415-487"""
    has_cross_attention = False

    def __init__(self, in_channels, out_channels, temb_channels, num_layers=1, resnet_eps=1e-6, resnet_groups=32,
                 add_downsample=True, downsample_padding=1, **_):
        super().__init__()
        self.resnets = nn.ModuleList([
            ResnetBlock3D(in_channels=in_channels if i == 0 else out_channels, out_channels=out_channels,
                          temb_channels=temb_channels, eps=resnet_eps, groups=resnet_groups) for i in range(num_layers)])
        self.attentions = None
        self.downsamplers = (nn.ModuleList([Downsample3D(out_channels, True, out_channels, downsample_padding, "op")])
                             if add_downsample else None)

    def forward(self, c: Ctx, x, expand_batch_to: int = 0):
        """`expand_batch_to`: the input is the text-independent prefix computed for ONE classifier-free-guidance half;
        it is broadcast to the full batch right before the first text-dependent op (the first Transformer3DModel)."""
        outs = []
        for i, r in enumerate(self.resnets):
            x = r(c, x)
            if self.attentions is not None:
                if expand_batch_to and x.shape[0] != expand_batch_to:
                    x = ops.repeat_batch(x, expand_batch_to)
                x = self.attentions[i](c, x)
            outs.append(x)
        if self.downsamplers is not None:
            x = self.downsamplers[0](c, x)
            outs.append(x)
        return x, outs


class CrossAttnDownBlock3D(DownBlock3D):
    """unet_blocks.py:270-412"""
    has_cross_attention = True

    def __init__(self, in_channels, out_channels, temb_channels, num_layers=1, resnet_eps=1e-6, resnet_groups=32,
                 attn_num_head_channels=1, cross_attention_dim=1280, add_downsample=True, downsample_padding=1,
                 only_cross_attention=False, rotary_emb=None, **_):
        super().__init__(in_channels, out_channels, temb_channels, num_layers, resnet_eps, resnet_groups, add_downsample,
                         downsample_padding)
        self.attentions = nn.ModuleList([_t3d(attn_num_head_channels, out_channels, cross_attention_dim, resnet_groups,
                                              only_cross_attention, rotary_emb) for _ in range(num_layers)])


class UNetMidBlock3DCrossAttn(nn.Module):
    """unet_blocks.py:180-267"""
    has_cross_attention = True

    def __init__(self, in_channels, temb_channels, resnet_eps=1e-6, resnet_groups=32, attn_num_head_channels=1,
                 cross_attention_dim=1280, rotary_emb=None, **_):
        super().__init__()
        mk = lambda: ResnetBlock3D(in_channels=in_channels, out_channels=in_channels, temb_channels=temb_channels,  # noqa
                                   eps=resnet_eps, groups=resnet_groups)
        self.attentions = nn.ModuleList([_t3d(attn_num_head_channels, in_channels, cross_attention_dim, resnet_groups,
                                              False, rotary_emb)])
        self.resnets = nn.ModuleList([mk(), mk()])

    def forward(self, c: Ctx, x, out=None):
        x = self.resnets[0](c, x)
        x = self.attentions[0](c, x)
        return self.resnets[1](c, x, out=out)


class UpBlock3D(nn.Module):
    """unet_blocks.py:588-660"""
    has_cross_attention = False

    def __init__(self, in_channels, prev_output_channel, out_channels, temb_channels, num_layers=1, resnet_eps=1e-6,
                 resnet_groups=32, add_upsample=True, **_):
        super().__init__()
        res = []
        for i in range(num_layers):
            skip = in_channels if i == num_layers - 1 else out_channels
            rin = prev_output_channel if i == 0 else out_channels
            res.append(ResnetBlock3D(in_channels=rin + skip, out_channels=out_channels, temb_channels=temb_channels,
                                     eps=resnet_eps, groups=resnet_groups))
        self.resnets = nn.ModuleList(res)
        self.attentions = None
        self.upsamplers = nn.ModuleList([Upsample3D(out_channels, True, out_channels)]) if add_upsample else None

    def forward(self, c: Ctx, x, skips, upsample_size=None, out=None):
        """`out`: destination of the block's result (the head slice of the NEXT concat buffer, see new_cat_slot)"""
        n = len(self.resnets)
        B = x.shape[0]
        for i, r in enumerate(self.resnets):
            last = i == n - 1
            # the main branch of the next concat is produced by this stage's last layer: let it store there directly
            # (unless that concat will not be materialised at all: both halves carry GroupNorm statistics)
            nxt = (out if self.upsamplers is None else None) if last else \
                new_cat_slot(skips[-2 - i], r.out_channels, B, True)
            if self.attentions is not None:
                x = r.forward_cat(c, x, skips[-1 - i])
                x = self.attentions[i](c, x, out=nxt)
            else:
                x = r.forward_cat(c, x, skips[-1 - i], out=nxt)
        if self.upsamplers is not None:
            x = self.upsamplers[0](c, x, upsample_size, out=out)
        return x


class CrossAttnUpBlock3D(UpBlock3D):
    """unet_blocks.py:490-585"""
    has_cross_attention = True

    def __init__(self, in_channels, out_channels, prev_output_channel, temb_channels, num_layers=1, resnet_eps=1e-6,
                 resnet_groups=32, attn_num_head_channels=1, cross_attention_dim=1280, add_upsample=True,
                 only_cross_attention=False, rotary_emb=None, **_):
        super().__init__(in_channels, prev_output_channel, out_channels, temb_channels, num_layers, resnet_eps,
                         resnet_groups, add_upsample)
        self.attentions = nn.ModuleList([_t3d(attn_num_head_channels, out_channels, cross_attention_dim, resnet_groups,
                                              only_cross_attention, rotary_emb) for _ in range(num_layers)])


# ------------------------------------------------------------------------------------------------
# VAE side of unet_blocks.py / vae_video.py
# ------------------------------------------------------------------------------------------------
class AttentionBlock(nn.Module):
    """diffusers AttentionBlock (unet_blocks.py:16,703-713; in-tree copy diffusers_attention.py:249-381):
    per-frame single-head attention over all h*w positions, d = channels."""

    def __init__(self, channels, num_head_channels=None, norm_num_groups=32, rescale_output_factor=1.0, eps=1e-5):
        super().__init__()
        self.channels = channels
        self.num_heads = channels // num_head_channels if num_head_channels is not None else 1
        assert rescale_output_factor == 1.0
        self.group_norm = nn.GroupNorm(num_channels=channels, num_groups=norm_num_groups, eps=eps, affine=True)
        self.query = nn.Linear(channels, channels)
        self.key = nn.Linear(channels, channels)
        self.value = nn.Linear(channels, channels)
        self.proj_attn = nn.Linear(channels, channels, bias=True)
        self._use_memory_efficient_attention_xformers = False  # read by the pipeline (pipeline...:673)

    def forward(self, c: Ctx, x, stream_scale: float = 1.0):
        B, T, H, W, C = x.shape
        n = _gn(c, self.group_norm, x, False, B * T, stream_scale)
        w, b = c.pk.fused_linear(f"qkv{id(self)}", [self.query, self.key, self.value])
        qkv = ops.linear(n.view(B * T, H * W, C), w, b)
        o = ops.attention(qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:], self.num_heads,
                          scale=(C // self.num_heads) ** -0.5)
        wo, bo = c.pk.linear(self.proj_attn)
        out = ops.linear(o.view(B, T, H * W, C), wo, bo, residual=x.view(B, T, H * W, C), out_scale=stream_scale,
                         gn_stats=True)
        return _carry_gn(out.view(B, T, H, W, C), out)


def _vae_resnet(plus: bool, cin, cout, eps, groups):
    cls = ResnetBlock3D_plus if plus else ResnetBlock3D
    return cls(in_channels=cin, out_channels=cout, temb_channels=None, eps=eps, groups=groups)


class UNetMidBlock3D(nn.Module):
    """unet_blocks.py:663-745 (and the `_plus` variant :848-915)"""
    PLUS = False

    def __init__(self, in_channels, resnet_eps=1e-6, resnet_groups=32, attn_num_head_channels=None, **_):
        super().__init__()
        self.resnets = nn.ModuleList([_vae_resnet(self.PLUS, in_channels, in_channels, resnet_eps, resnet_groups)
                                      for _ in range(2)])
        self.attentions = nn.ModuleList([AttentionBlock(in_channels, num_head_channels=attn_num_head_channels,
                                                        eps=resnet_eps, norm_num_groups=resnet_groups)])

    def forward(self, c: Ctx, x, stream_scale: float = 1.0):
        x = self.resnets[0](c, x, stream_scale)
        x = self.attentions[0](c, x, stream_scale)
        return self.resnets[1](c, x, stream_scale)


class UNetMidBlock3D_plus(UNetMidBlock3D):
    PLUS = True


class DownEncoderBlock3D(nn.Module):
    """unet_blocks.py:748-805"""

    def __init__(self, in_channels, out_channels, num_layers=1, resnet_eps=1e-6, resnet_groups=32, add_downsample=True,
                 downsample_padding=1, **_):
        super().__init__()
        self.resnets = nn.ModuleList([_vae_resnet(False, in_channels if i == 0 else out_channels, out_channels,
                                                  resnet_eps, resnet_groups) for i in range(num_layers)])
        self.downsamplers = (nn.ModuleList([Downsample3D(out_channels, True, out_channels, downsample_padding, "op")])
                             if add_downsample else None)

    def forward(self, c: Ctx, x):
        for r in self.resnets:
            x = r(c, x)
        if self.downsamplers is not None:
            x = self.downsamplers[0](c, x)
        return x


class UpDecoderBlock3D(nn.Module):
    """unet_blocks.py:808-845 (and `_plus` :918-993)"""
    PLUS = False

    def __init__(self, in_channels, out_channels, num_layers=1, resnet_eps=1e-6, resnet_groups=32, add_upsample=True, **_):
        super().__init__()
        self.resnets = nn.ModuleList([_vae_resnet(self.PLUS, in_channels if i == 0 else out_channels, out_channels,
                                                  resnet_eps, resnet_groups) for i in range(num_layers)])
        self.upsamplers = nn.ModuleList([Upsample3D(out_channels, True, out_channels)]) if add_upsample else None

    def forward(self, c: Ctx, x, stream_scale: float = 1.0):
        for r in self.resnets:
            x = r(c, x, stream_scale)
        if self.upsamplers is not None:
            x = self.upsamplers[0](c, x, None, stream_scale)
        return x


class UpDecoderBlock3D_plus(UpDecoderBlock3D):
    PLUS = True


class Fuse_sft_block(nn.Module):
    """resnet.py:63-79"""

    def __init__(self, enc_ch, dec_ch):
        super().__init__()
        self.shared = nn.Sequential(ResnetBlock3D(in_channels=enc_ch + dec_ch, out_channels=dec_ch, temb_channels=None),
                                    ResnetBlock3D(in_channels=dec_ch, out_channels=dec_ch, temb_channels=None))
        self.scale = InflatedConv3d(dec_ch, dec_ch, 3, 1, 1)
        self.shift = InflatedConv3d(dec_ch, dec_ch, 3, 1, 1)

    def forward(self, c: Ctx, enc_feat, dec_feat, w=1, out_scale: float = 1.0):
        e = ops.concat_channels(enc_feat, dec_feat)
        e = self.shared[0](c, e)
        e = self.shared[1](c, e)
        return ops.sft_fuse(dec_feat, self.scale.run(c, e), self.shift.run(c, e), float(w), out_scale)
