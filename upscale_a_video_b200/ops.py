"""Thin torch-tensor wrappers over the C ABI (include/uav_b200.h).

All activations are channels-last fp16 CUDA tensors: a reference "b c t h w" tensor is held as
(b, t, h, w, c).  A tensor may be a channel slice `buf[..., c0:c1]` of a wider buffer (its pixel
stride `ld` is then the buffer's channel count).  PyTorch is used for memory and streams only.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _lib
from ._lib import Epilogue

ACT_NONE, ACT_SILU, ACT_GEGLU = 0, 1, 2
F16, F32 = 0, 1


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


class Profile:
    """Opt-in per-launch timing (CUDA events on the launching stream) + algorithmic work counters, used by bench.py
    for the roofline numbers.  Disabled (zero overhead) unless entered as a context manager."""
    active: "Optional[Profile]" = None

    def __init__(self):
        self.records = []  # (kind, flops, bytes, start_event, end_event)

    def __enter__(self):
        Profile.active = self
        return self

    def __exit__(self, *a):
        Profile.active = None

    def by_tag(self):
        """per (kind, tag) totals: launches, flops, ms — for finding the expensive shapes"""
        torch.cuda.synchronize()
        out = {}
        for kind, fl, by, s, e, tag in self.records:
            d = out.setdefault((kind, tag), dict(launches=0, flops=0.0, bytes=0.0, ms=0.0))
            d["launches"] += 1
            d["flops"] += fl
            d["bytes"] += by
            d["ms"] += s.elapsed_time(e)
        return out

    def summary(self):
        torch.cuda.synchronize()
        out = {}
        for kind, fl, by, s, e, _tag in self.records:
            d = out.setdefault(kind, dict(launches=0, flops=0.0, bytes=0.0, ms=0.0))
            d["launches"] += 1
            d["flops"] += fl
            d["bytes"] += by
            d["ms"] += s.elapsed_time(e)
        return out


class _timed:
    __slots__ = ("kind", "flops", "bytes", "s", "tag")

    def __init__(self, kind, flops=0.0, nbytes=0.0, tag=""):
        self.kind, self.flops, self.bytes, self.tag = kind, flops, nbytes, tag

    def __enter__(self):
        if Profile.active is not None:
            self.s = torch.cuda.Event(enable_timing=True)
            self.s.record()

    def __exit__(self, *a):
        p = Profile.active
        if p is not None:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            p.records.append((self.kind, self.flops, self.bytes, self.s, e, self.tag))


def _pixel_ld(x: torch.Tensor) -> int:
    """element distance between consecutive pixels; validates the channels-last layout"""
    assert x.is_cuda, "uav_b200 ops need CUDA tensors (no CPU fallback)"
    # kernels launch on the CURRENT device's stream: a tensor living elsewhere would be dereferenced on the wrong GPU
    assert x.device.index == torch.cuda.current_device(), \
        f"tensor on cuda:{x.device.index} but the current device is cuda:{torch.cuda.current_device()} (torch.cuda.set_device first)"
    assert x.stride(-1) == 1 or x.shape[-1] == 1, "channel dim must be contiguous"
    if x.dim() == 1:
        return x.shape[0]
    # the pixel stride is the stride of the innermost pixel dim of extent > 1 (a size-1 dim reports an arbitrary stride:
    # e.g. the (b, t, h*w = 1, c) view of a channel slice of a wider buffer)
    ld = None
    exp = None
    for d in range(x.dim() - 2, -1, -1):
        if x.shape[d] != 1:
            if ld is None:
                ld = x.stride(d)
                exp = ld
            assert x.stride(d) == exp, f"tensor is not a dense channels-last view: {x.shape} {x.stride()}"
        if exp is not None:
            exp *= x.shape[d]
    return x.shape[-1] if ld is None else ld


class GnStats:
    """GroupNorm statistics blocks of ONE tensor, written by the epilogue of the implicit-GEMM launch that produced it
    (uav_epilogue_t.gn_partial): fp32 [C / 8][blocks][2].  `images` x `rows_per_image` is the row geometry of that launch
    (M-tiles never straddle images), `batch` the number of batch items the tensor spans.  Attached to the produced tensor
    as `tensor.uav_gn = [GnStats]`; a channel concatenation carries the list of its parts."""
    __slots__ = ("partial", "blocks", "C", "images", "rows_per_image", "batch")

    def __init__(self, partial, blocks, C, images, rows_per_image, batch):
        self.partial, self.blocks, self.C = partial, blocks, C
        self.images, self.rows_per_image, self.batch = images, rows_per_image, batch

    def slabs_for(self, n_outer: int, batch: int) -> int:
        """number of slabs this source splits into for a consumer normalising `n_outer` slabs over `batch` batch items;
        0 = unusable (the consumer then runs its own statistics pass)"""
        per_item = n_outer // batch
        if self.batch == batch:
            want = n_outer
        elif self.batch == 1 and per_item == 1:
            return 1  # computed once for both classifier-free-guidance halves: every n reads the same blocks
        else:
            return 0
        if self.images % want == 0:
            return want
        rows = self.images * self.rows_per_image
        if self.images == 1 and rows % want == 0 and (rows // want) % 128 == 0:
            return want
        return 0


def _gn_request(out: torch.Tensor, n_out: int, w: int, h: int, images: int, batch: int, e: Epilogue):
    """arm the epilogue to emit the statistics blocks of `out`; returns the GnStats to attach after the launch"""
    if out.dtype != torch.float16 or n_out < 64 or n_out % 8:
        return None
    blocks = int(_lib.load().uav_gn_partial_blocks(w, h, images))
    partial = torch.empty(n_out // 8, blocks, 2, dtype=torch.float32, device=out.device)
    e.gn_partial = partial.data_ptr()
    e.gn_blocks = blocks
    return GnStats(partial, blocks, n_out, images, w * h, batch)


def _epi(out: torch.Tensor, bias=None, rowvec=None, rows_per_vec=0, residual=None, act=ACT_NONE, out_scale=1.0) -> Epilogue:
    e = Epilogue()
    e.out_scale = out_scale
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.is_contiguous()
        e.bias = bias.data_ptr()
    if rowvec is not None:
        assert rowvec.dtype == torch.float16 and rowvec.stride(-1) == 1
        e.rowvec = rowvec.data_ptr()
        e.rows_per_vec = rows_per_vec
        e.ld_rowvec = rowvec.stride(0) if rowvec.dim() > 1 else rowvec.shape[0]
    if residual is not None:
        assert residual.dtype == torch.float16
        e.residual = residual.data_ptr()
        e.ld_res = _pixel_ld(residual)
    e.act = act
    e.out_dtype = F16 if out.dtype == torch.float16 else F32
    assert out.dtype in (torch.float16, torch.float32)
    e.ld_out = _pixel_ld(out)
    return e


def _igemm(fn: str, args, out: torch.Tensor, e: Epilogue, st: Optional[GnStats], flops, nbytes, tag=""):
    """launch the implicit-GEMM entry point `fn`(*args, out, e, stream), timed as "igemm"; `st` (the statistics requested
    from `e`, or None) is attached to `out`"""
    lib = _lib.load()
    with _timed("igemm", flops, nbytes, tag):
        _lib.check(getattr(lib, fn)(*args, out.data_ptr(), C.byref(e), _stream()), fn)
    if st is not None:
        out.uav_gn = [st]
    return out


def linear(a: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, *, out=None,
           residual=None, rowvec=None, rows_per_vec=0, act=ACT_NONE, out_dtype=torch.float16, out_scale=1.0,
           gn_stats=False):
    """out[..., N] = epilogue(a[..., K] @ w[N, K]^T); a fp16 (rows may be a channel-slice view)."""
    assert a.dtype == torch.float16 and w.dtype == torch.float16 and w.is_contiguous()
    K = a.shape[-1]
    N = w.shape[0]
    assert w.shape[1] == K
    M = a.numel() // K
    n_out = N // 2 if act == ACT_GEGLU else N
    if out is None:
        out = torch.empty(*a.shape[:-1], n_out, dtype=out_dtype, device=a.device)
    assert out.shape[-1] == n_out and out.numel() // n_out == M
    e = _epi(out, bias, rowvec, rows_per_vec, residual, act, out_scale)
    st = _gn_request(out, n_out, M, 1, 1, a.shape[0] if a.dim() > 2 else 1, e) if gn_stats and act != ACT_GEGLU else None
    return _igemm("uav_linear", (a.data_ptr(), M, K, _pixel_ld(a) if a.dim() > 1 else K, w.data_ptr(), N), out, e, st,
                  2.0 * M * N * K, 2.0 * (M * K + N * K + M * n_out), f"linear M{M} K{K} N{N} act{act}")


def conv2d(x: torch.Tensor, w: torch.Tensor, bias=None, *, stride=1, pad_mode=0, out=None, residual=None,
           rowvec=None, rows_per_vec=0, act=ACT_NONE, out_dtype=torch.float16, out_scale=1.0, gn_stats=False):
    """x: (..., H, W, Cin) channels-last fp16 (leading dims = images); w: (Cout, k, k, Cin) fp16."""
    assert x.dtype == torch.float16 and w.dtype == torch.float16 and w.is_contiguous()
    *lead, H, W, Cin = x.shape
    Cout, k, k2, Cin_w = w.shape
    assert k == k2 and Cin_w == Cin
    NB = 1
    for d in lead:
        NB *= d
    Ho, Wo = (H, W) if stride == 1 else (H // 2, W // 2)
    if out is None:
        out = torch.empty(*lead, Ho, Wo, Cout, dtype=out_dtype, device=x.device)
    assert tuple(out.shape) == (*lead, Ho, Wo, Cout), (out.shape, (*lead, Ho, Wo, Cout))
    e = _epi(out, bias, rowvec, rows_per_vec, residual, act, out_scale)
    st = None
    if gn_stats:
        st = (_gn_request(out, Cout, NB * Ho * Wo, 1, 1, lead[0] if lead else 1, e) if (k == 1 and stride == 1) else
              _gn_request(out, Cout, Wo, Ho, NB, lead[0] if lead else 1, e))
    return _igemm("uav_conv2d", (x.data_ptr(), NB, H, W, Cin, _pixel_ld(x), w.data_ptr(), Cout, k, stride, pad_mode), out,
                  e, st, 2.0 * NB * Ho * Wo * Cout * Cin * k * k,
                  2.0 * (NB * H * W * Cin + w.numel()) + out.element_size() * NB * Ho * Wo * Cout,
                  f"conv{k}x{k}s{stride} {NB}x{H}x{W} {Cin}->{Cout}")


def upsample2x_conv3x3(x: torch.Tensor, w4: torch.Tensor, bias=None, out=None):
    """nearest x2 upsample + 3x3 conv without the upsampled intermediate.  x: (..., H, W, Cin); w4: (4, Cout, 2, 2, Cin)
    phase filters from `collapse_upsample_filter`."""
    assert x.dtype == torch.float16 and w4.dtype == torch.float16 and w4.is_contiguous()
    *lead, H, W, Cin = x.shape
    Cout = w4.shape[1]
    assert tuple(w4.shape) == (4, Cout, 2, 2, Cin)
    NB = 1
    for d in lead:
        NB *= d
    if out is None:
        out = torch.empty(*lead, 2 * H, 2 * W, Cout, dtype=torch.float16, device=x.device)
    assert tuple(out.shape) == (*lead, 2 * H, 2 * W, Cout) and out.dtype == torch.float16
    e = _epi(out, bias)
    return _igemm("uav_upsample2x_conv3x3", (x.data_ptr(), NB, H, W, Cin, _pixel_ld(x), w4.data_ptr(), Cout), out, e,
                  None, 2.0 * NB * 4 * H * W * Cout * Cin * 4,
                  2.0 * (NB * H * W * Cin + w4.numel() + out.numel()), f"up2x+conv {NB}x{H}x{W} {Cin}->{Cout}")


def collapse_upsample_filter(w: torch.Tensor) -> torch.Tensor:
    """(Cout, 3, 3, Cin) conv filter applied after a nearest x2 upsample -> (4, Cout, 2, 2, Cin) phase filters
    (summed in fp32, rounded to fp16 once).  Phase p = a*2+b produces output pixel (2y+a, 2x+b); its taps read source
    rows {y-1, y} (a=0) or {y, y+1} (a=1), columns likewise."""
    w = w.float()
    rows = [torch.stack([w[:, 0], w[:, 1] + w[:, 2]], dim=1), torch.stack([w[:, 0] + w[:, 1], w[:, 2]], dim=1)]  # (Cout,2,3,Cin)
    out = []
    for a in range(2):
        r = rows[a]
        cols = [torch.stack([r[:, :, 0], r[:, :, 1] + r[:, :, 2]], dim=2), torch.stack([r[:, :, 0] + r[:, :, 1], r[:, :, 2]], dim=2)]
        for b in range(2):
            out.append(cols[b])
    return torch.stack(out, dim=0).to(torch.float16).contiguous()


def conv_temporal(x: torch.Tensor, w: torch.Tensor, bias=None, *, out=None, residual=None, rowvec=None,
                  rows_per_vec=0, act=ACT_NONE, out_dtype=torch.float16, out_scale=1.0, gn_stats=False):
    """x: (B, T, H, W, Cin); w: (Cout, k, Cin) — nn.Conv3d (k,1,1), zero padding (k-1)/2 in t."""
    assert x.dtype == torch.float16 and w.dtype == torch.float16 and w.is_contiguous()
    B, T, H, W, Cin = x.shape
    Cout, k, Cin_w = w.shape
    assert Cin_w == Cin
    if out is None:
        out = torch.empty(B, T, H, W, Cout, dtype=out_dtype, device=x.device)
    e = _epi(out, bias, rowvec, rows_per_vec, residual, act, out_scale)
    st = _gn_request(out, Cout, H * W, 1, B * T, B, e) if gn_stats else None
    return _igemm("uav_conv_temporal", (x.data_ptr(), B, T, H * W, Cin, _pixel_ld(x), w.data_ptr(), Cout, k), out, e, st,
                  2.0 * B * T * H * W * Cout * Cin * k, 2.0 * (x.numel() + w.numel() + B * T * H * W * Cout),
                  f"conv_t{k} {B}x{T}x{H}x{W} {Cin}->{Cout}")


def conv3d(x: torch.Tensor, w: torch.Tensor, bias=None, *, out=None, residual=None, act=ACT_NONE,
           out_dtype=torch.float16, out_scale=1.0, gn_stats=False):
    """x: (B, T, H, W, Cin); w: (Cout, 3, 3, 3, Cin) — nn.Conv3d 3x3x3, padding 1."""
    assert x.dtype == torch.float16 and w.dtype == torch.float16 and w.is_contiguous()
    B, T, H, W, Cin = x.shape
    Cout = w.shape[0]
    assert tuple(w.shape) == (Cout, 3, 3, 3, Cin)
    if out is None:
        out = torch.empty(B, T, H, W, Cout, dtype=out_dtype, device=x.device)
    e = _epi(out, bias, None, 0, residual, act, out_scale)
    st = _gn_request(out, Cout, W, H, B * T, B, e) if gn_stats else None
    return _igemm("uav_conv3d", (x.data_ptr(), B, T, H, W, Cin, _pixel_ld(x), w.data_ptr(), Cout), out, e, st,
                  2.0 * B * T * H * W * Cout * Cin * 27, 2.0 * (x.numel() + w.numel() + B * T * H * W * Cout))


# ------------------------------------------------------------------------------------------------
# normalisation
# ------------------------------------------------------------------------------------------------
_gn_ws = {}


def _gn_workspace(device, n_outer: int, groups: int):
    """the GroupNorm scratch of the current stream, grown to uav_groupnorm_workspace_bytes(n_outer, groups)"""
    nbytes = _lib.load().uav_groupnorm_workspace_bytes(n_outer, groups)
    key = (device, torch.cuda.current_stream().cuda_stream)
    ws = _gn_ws.get(key)
    if ws is None or ws.numel() < nbytes:
        ws = torch.empty(max(nbytes, 1 << 16), dtype=torch.uint8, device=device)
        _gn_ws[key] = ws
    return ws


def _gn_sources(stats, C: int, groups: int, n_outer: int, batch: int, parts=None):
    """ctypes uav_gn_source_t table of a C-channel GroupNorm over the channel concatenation whose parts' producers emitted
    `stats` (one GnStats per part), or None when they cannot serve.  `parts`: the parts themselves, for a concatenation
    that is never built (a batch-1 part serves every batch item)."""
    if not (stats and (C // groups) % 8 == 0 and len(stats) <= 4 and sum(s.C for s in stats) == C):
        return None
    slabs = [s.slabs_for(n_outer, batch) for s in stats]
    if not all(slabs):
        return None
    srcs = (_lib.GnSource * len(stats))()
    for i, (s, sl) in enumerate(zip(stats, slabs)):
        srcs[i].partial, srcs[i].blocks, srcs[i].C, srcs[i].slabs = s.partial.data_ptr(), s.blocks, s.C, sl
        if parts is not None:
            p = parts[i]
            ld = _pixel_ld(p)
            srcs[i].x, srcs[i].ld = p.data_ptr(), ld
            srcs[i].slab_stride = p.numel() // p.shape[-1] // p.shape[0] * ld if p.shape[0] > 1 else 0
    return srcs


def group_norm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, groups: int, eps: float, *, silu: bool,
               n_outer: int, out: Optional[torch.Tensor] = None, stats=None, batch: Optional[int] = None):
    """x: channels-last (..., C) fp16; statistics per (outer index, group) where the leading `n_outer` slabs of
    x.numel()/C/n_outer pixels each are normalised independently (5-D GN: n_outer=b; per-frame GN: n_outer=b*t).
    `stats`: list of GnStats of the tensors x is the channel concatenation of (emitted by their producers' epilogues):
    the statistics read pass is then skipped."""
    assert x.dtype == torch.float16 and gamma.dtype == torch.float32 and beta.dtype == torch.float32
    C = x.shape[-1]
    total_pix = x.numel() // C
    assert total_pix % n_outer == 0
    pixels = total_pix // n_outer
    if out is None:
        out = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    lib = _lib.load()
    ws = _gn_workspace(x.device, n_outer, groups)
    srcs = _gn_sources(stats, C, groups, n_outer, x.shape[0] if batch is None else batch)
    if srcs is not None:
        with _timed("groupnorm", 0.0, 2.0 * 2 * total_pix * C, f"gn(fused stats) {total_pix}px C{C}"):  # read + write
            _lib.check(lib.uav_groupnorm_silu_from_partials(x.data_ptr(), n_outer, pixels, C, _pixel_ld(x), groups,
                                                            gamma.data_ptr(), beta.data_ptr(), eps, 1 if silu else 0,
                                                            out.data_ptr(), _pixel_ld(out), srcs, len(stats), ws.data_ptr(),
                                                            ws.numel(), _stream()), "uav_groupnorm_silu_from_partials")
        return out
    with _timed("groupnorm", 0.0, 2.0 * 3 * total_pix * C, f"gn {total_pix}px C{C}"):  # read (stats) + read + write
        _lib.check(lib.uav_groupnorm_silu(x.data_ptr(), n_outer, pixels, C, _pixel_ld(x), groups, gamma.data_ptr(),
                                          beta.data_ptr(), eps, 1 if silu else 0, out.data_ptr(), _pixel_ld(out),
                                          ws.data_ptr(), ws.numel(), _stream()), "uav_groupnorm_silu")
    return out


def group_norm_cat(parts, gamma: torch.Tensor, beta: torch.Tensor, groups: int, eps: float, *, silu: bool, n_outer: int):
    """GroupNorm(+SiLU) of torch.cat(parts, channel) WITHOUT building the concatenation (unet_blocks.py:573,645 followed by
    resnet.py:267): every part carries the statistics blocks its producer emitted; one reduction over all of them, then one
    apply launch per part writing its channel range of the dense result.  A part with batch 1 (computed once for both
    classifier-free-guidance halves) serves every batch item.  Returns None when a part cannot serve (no statistics,
    misaligned slabs): the caller then materialises the concat."""
    B = max(p.shape[0] for p in parts)
    C = sum(p.shape[-1] for p in parts)
    lead = tuple(parts[0].shape[1:-1])
    stats = []
    for p in parts:
        st = getattr(p, "uav_gn", None)
        if (not st or len(st) != 1 or st[0].C != p.shape[-1] or p.dtype != torch.float16 or p.shape[0] not in (1, B)
                or tuple(p.shape[1:-1]) != lead):
            return None
        stats.append(st[0])
    srcs = _gn_sources(stats, C, groups, n_outer, B, parts) if n_outer == B else None
    if srcs is None:
        return None
    out = torch.empty(B, *lead, C, dtype=torch.float16, device=parts[0].device)
    pixels = out.numel() // C // n_outer
    lib = _lib.load()
    ws = _gn_workspace(out.device, n_outer, groups)
    with _timed("groupnorm", 0.0, 2.0 * 2 * out.numel(), f"gn(virtual concat) {out.numel() // C}px C{C}"):
        _lib.check(lib.uav_groupnorm_silu_from_partials(None, n_outer, pixels, C, C, groups, gamma.data_ptr(), beta.data_ptr(),
                                                        eps, 1 if silu else 0, out.data_ptr(), C, srcs, len(parts),
                                                        ws.data_ptr(), ws.numel(), _stream()),
                   "uav_groupnorm_silu_from_partials")
    return out


def conv_out_fused(x: torch.Tensor, gamma, beta, groups: int, eps: float, w: torch.Tensor, bias, cout: int, out_dtype,
                   cfg_step: Optional[dict] = None):
    """conv_out(SiLU(GroupNorm(x))) -> planar (B, cout, T, H, W): x (B, T, H, W, 256) fp16 raw, w (cout, 3, 3, 256) fp16
    (unet_video.py:567-569).  GroupNorm statistics from x's producer when it emitted them, else by a read pass.
    `cfg_step` (B == 2, fp16): dict(guidance_scale, pred_type, sqrt_alpha, sqrt_beta, clip, clip_range, sample) — the
    classifier-free-guidance combine and DDIMScheduler.step_v0 run in the kernel's epilogue; returns (noise_pred, x0), both
    (1, cout, T, H, W) fp16, bit-identical to cfg_combine + ddim_step_v0 on the unfused output."""
    B, T, H, W, Cc = x.shape
    assert x.dtype == torch.float16 and w.dtype == torch.float16 and w.is_contiguous() and tuple(w.shape[1:]) == (3, 3, Cc)
    lib = _lib.load()
    ws = _gn_workspace(x.device, B, groups)
    affine = torch.empty(B, Cc, 2, dtype=torch.float32, device=x.device)
    stats = getattr(x, "uav_gn", None)
    srcs = _gn_sources(stats, Cc, groups, B, B)
    with _timed("groupnorm", 0.0, 2.0 * x.numel() if srcs is None else 0.0, f"gn affine {x.numel() // Cc}px C{Cc}"):
        _lib.check(lib.uav_groupnorm_affine(x.data_ptr(), B, T * H * W, Cc, _pixel_ld(x), groups, gamma.data_ptr(),
                                            beta.data_ptr(), eps, srcs, 0 if srcs is None else len(stats),
                                            affine.data_ptr(), ws.data_ptr(), ws.numel(), _stream()), "uav_groupnorm_affine")
    bias_p = None if bias is None else bias.data_ptr()
    if cfg_step is not None:
        sample = cfg_step["sample"]
        assert B == 2 and sample.dtype == torch.float16 and sample.is_contiguous() and tuple(sample.shape) == (1, cout, T, H, W)
        noise_pred, x0 = torch.empty_like(sample), torch.empty_like(sample)
        st = _lib.CfgStep(float(cfg_step["guidance_scale"]), int(cfg_step["pred_type"]), float(cfg_step["sqrt_alpha"]),
                          float(cfg_step["sqrt_beta"]), 1 if cfg_step["clip"] else 0, float(cfg_step["clip_range"]),
                          sample.data_ptr(), noise_pred.data_ptr(), x0.data_ptr())
        with _timed("conv_io", 2.0 * B * T * H * W * cout * Cc * 9, 2.0 * x.numel() + 6.0 * sample.numel(),
                    f"conv_out+cfg+step_v0 {B * T}x{H}x{W} {Cc}->{cout}"):
            _lib.check(lib.uav_conv_out_cfg_step(x.data_ptr(), T, H, W, Cc, _pixel_ld(x), affine.data_ptr(), w.data_ptr(),
                                                 bias_p, cout, C.byref(st), _stream()), "uav_conv_out_cfg_step")
        return noise_pred, x0
    out = torch.empty(B, cout, T, H, W, dtype=out_dtype, device=x.device)
    with _timed("conv_io", 2.0 * B * T * H * W * cout * Cc * 9, 2.0 * x.numel() + out.numel() * out.element_size(),
                f"conv_out_fused {B * T}x{H}x{W} {Cc}->{cout}"):
        _lib.check(lib.uav_conv_out_fused(x.data_ptr(), B, T, H, W, Cc, _pixel_ld(x), affine.data_ptr(), w.data_ptr(),
                                          bias_p, cout, out.data_ptr(), F16 if out_dtype == torch.float16 else F32,
                                          _stream()), "uav_conv_out_fused")
    return out


def layer_norm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float = 1e-5, out=None):
    assert x.dtype == torch.float16 and gamma.dtype == torch.float32
    C = x.shape[-1]
    rows = x.numel() // C
    if out is None:
        out = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    lib = _lib.load()
    with _timed("layernorm", 0.0, 2.0 * 2 * rows * C):
        _lib.check(lib.uav_layernorm(x.data_ptr(), rows, C, _pixel_ld(x), gamma.data_ptr(), beta.data_ptr(), eps,
                                     out.data_ptr(), _pixel_ld(out), _stream()), "uav_layernorm")
    return out


# ------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------
def attention(q, k, v, heads: int, *, kv_batch_div: int = 1, scale: Optional[float] = None, out=None):
    """q: (batch, nq, heads*d) fp16 (may be a column slice of a fused qkv buffer); k, v: (batch/kv_batch_div, nk, heads*d).
    `scale` (default d ** -0.5) multiplies the scores before the softmax; it must be finite and > 0, anything else is
    rejected before a launch."""
    batch, nq, C = q.shape
    d = C // heads
    nk = k.shape[1]
    assert k.shape[0] * kv_batch_div == batch and v.shape[:2] == k.shape[:2]
    if out is None:
        out = torch.empty(batch, nq, C, dtype=torch.float16, device=q.device)
    if scale is None:
        scale = d ** -0.5
    for t in (q, k, v, out):
        assert t.dtype == torch.float16 and t.stride(-1) == 1 and t.stride(0) == t.shape[1] * t.stride(1)
    lib = _lib.load()
    with _timed("attention", 4.0 * batch * nq * nk * C, 2.0 * (2 * batch * nq * C + 2 * k.shape[0] * nk * C),
                f"attn b{batch} h{heads} d{d} nq{nq} nk{nk}"):
        _lib.check(lib.uav_attention(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), batch, heads, d, nq, nk,
                                     q.stride(1), k.stride(1), v.stride(1), out.stride(1), kv_batch_div, scale,
                                     _stream()), "uav_attention")
    return out


def temporal_attention(q, k, v, heads: int, rot: torch.Tensor, bias: torch.Tensor, *, out=None):
    """q, k, v: (B, F, HW, heads*d) fp16 (column slices allowed); rot: (F,16,2) fp32 cos/sin; bias: (heads,F,F) fp32."""
    B, F, HW, C = q.shape
    d = C // heads
    if out is None:
        out = torch.empty(B, F, HW, C, dtype=torch.float16, device=q.device)
    assert rot.dtype == torch.float32 and rot.is_contiguous() and tuple(rot.shape) == (F, 16, 2)
    assert bias.dtype == torch.float32 and bias.is_contiguous() and tuple(bias.shape) == (heads, F, F)
    lib = _lib.load()
    with _timed("temporal_attention", 4.0 * B * HW * F * F * C, 2.0 * 4 * B * F * HW * C):
        _lib.check(lib.uav_temporal_attention(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), B, F, HW, heads, d,
                                              _pixel_ld(q), _pixel_ld(k), _pixel_ld(v), _pixel_ld(out), d ** -0.5,
                                              rot.data_ptr(), bias.data_ptr(), _stream()), "uav_temporal_attention")
    return out


# ------------------------------------------------------------------------------------------------
# data movement
# ------------------------------------------------------------------------------------------------
def copy_channels(src: torch.Tensor, dst: torch.Tensor):
    """dst[..., :C] = src (both channels-last views with the same pixel count)"""
    C = src.shape[-1]
    assert dst.shape[-1] == C and src.numel() == dst.numel()
    lib = _lib.load()
    with _timed("copy", 0.0, 4.0 * src.numel()):
        _lib.check(lib.uav_copy_channels(src.data_ptr(), _pixel_ld(src), dst.data_ptr(), _pixel_ld(dst), C,
                                         src.numel() // C, _stream()), "uav_copy_channels")
    return dst


def concat_channels(a: torch.Tensor, b: torch.Tensor):
    """torch.cat([a, b], dim=channel) for channels-last tensors.  `b` may have batch 1 while `a` has batch > 1 (a skip
    connection computed once for both classifier-free-guidance halves): it is then broadcast over the batch."""
    out = torch.empty(*a.shape[:-1], a.shape[-1] + b.shape[-1], dtype=a.dtype, device=a.device)
    copy_channels(a, out[..., : a.shape[-1]])
    if b.shape[0] == 1 and a.shape[0] > 1:
        for i in range(a.shape[0]):
            copy_channels(b, out[i:i + 1, ..., a.shape[-1]:])
    else:
        copy_channels(b, out[..., a.shape[-1]:])
    ga, gb = getattr(a, "uav_gn", None), getattr(b, "uav_gn", None)
    if ga and gb:
        out.uav_gn = list(ga) + list(gb)
    return out


def repeat_batch(x: torch.Tensor, n: int):
    """x (1, ...) -> (n, ...) by copy (channels-last)"""
    assert x.shape[0] == 1
    out = torch.empty(n, *x.shape[1:], dtype=x.dtype, device=x.device)
    for i in range(n):
        copy_channels(x, out[i:i + 1])
    if getattr(x, "uav_gn", None):
        out.uav_gn = x.uav_gn  # batch-1 statistics serve every batch item (GnStats.slabs_for)
    return out


def upsample_nearest(x: torch.Tensor, size=None):
    """x: (..., H, W, C); nearest x2 in H, W (or to explicit (Ho, Wo))"""
    *lead, H, W, C = x.shape
    Ho, Wo = (2 * H, 2 * W) if size is None else size
    NB = 1
    for d in lead:
        NB *= d
    out = torch.empty(*lead, Ho, Wo, C, dtype=x.dtype, device=x.device)
    lib = _lib.load()
    with _timed("copy", 0.0, 2.0 * (x.numel() + out.numel())):
        _lib.check(lib.uav_upsample_nearest(x.data_ptr(), _pixel_ld(x), NB, H, W, C, out.data_ptr(), _pixel_ld(out), Ho,
                                            Wo, _stream()), "uav_upsample_nearest")
    return out


def planar_to_channels_last(src: torch.Tensor, dst: torch.Tensor, c_off: int = 0, scale: float = 1.0):
    """src: (B, C, T, H, W) fp16/fp32 contiguous -> dst[(B,T,H,W), c_off:c_off+C] (fp16 channels-last)"""
    assert src.is_contiguous() and dst.dtype == torch.float16
    B, Cc = src.shape[:2]
    thw = src.numel() // (B * Cc)
    lib = _lib.load()
    _lib.check(lib.uav_planar_to_channels_last(src.data_ptr(), F16 if src.dtype == torch.float16 else F32, B, Cc, thw,
                                               dst.data_ptr(), _pixel_ld(dst), c_off, scale, _stream()),
               "uav_planar_to_channels_last")
    return dst


def channels_last_to_planar(src: torch.Tensor, C: int, out_dtype, clamp: bool = False):
    """src: (B, T, H, W, ld) channels-last (fp16/fp32) -> (B, C, T, H, W) of out_dtype"""
    B, T, H, W, _ = src.shape
    out = torch.empty(B, C, T, H, W, dtype=out_dtype, device=src.device)
    lib = _lib.load()
    _lib.check(lib.uav_channels_last_to_planar(src.data_ptr(), F16 if src.dtype == torch.float16 else F32,
                                               _pixel_ld(src), B, C, T * H * W, out.data_ptr(),
                                               F16 if out_dtype == torch.float16 else F32, 1 if clamp else 0,
                                               _stream()), "uav_channels_last_to_planar")
    return out


def silu(x: torch.Tensor):
    assert x.dtype == torch.float16 and x.is_contiguous()
    out = torch.empty_like(x)
    lib = _lib.load()
    _lib.check(lib.uav_silu(x.data_ptr(), out.data_ptr(), x.numel(), _stream()), "uav_silu")
    return out


def sft_fuse(dec: torch.Tensor, scale: torch.Tensor, shift: torch.Tensor, w: float, out_scale: float = 1.0):
    """(dec + w * (dec * scale + shift)) * out_scale (Fuse_sft_block, resnet.py:77-78); dense fp16 tensors of equal shape"""
    for t in (dec, scale, shift):
        assert t.dtype == torch.float16 and t.is_contiguous() and t.shape == dec.shape
    out = torch.empty_like(dec)
    lib = _lib.load()
    _lib.check(lib.uav_sft_fuse(dec.data_ptr(), scale.data_ptr(), shift.data_ptr(), float(w), float(out_scale), out.data_ptr(), dec.numel(),
                                _stream()), "uav_sft_fuse")
    return out


def timestep_embedding(t: torch.Tensor, dim: int, flip_sin_to_cos: bool, freq_shift: float):
    assert t.dtype == torch.float32 and t.is_contiguous()
    out = torch.empty(t.shape[0], dim, dtype=torch.float16, device=t.device)
    lib = _lib.load()
    _lib.check(lib.uav_timestep_embedding(t.data_ptr(), t.shape[0], dim, 1 if flip_sin_to_cos else 0, freq_shift,
                                          out.data_ptr(), _stream()), "uav_timestep_embedding")
    return out


# ------------------------------------------------------------------------------------------------
# sampler (operate on the reference's b c t h w latents)
# ------------------------------------------------------------------------------------------------
def _dt(x):
    assert x.dtype in (torch.float16, torch.float32) and x.is_contiguous() and x.is_cuda
    return F16 if x.dtype == torch.float16 else F32


def cfg_combine(pred2: torch.Tensor, guidance_scale: float):
    assert pred2.shape[0] % 2 == 0
    out = torch.empty(pred2.shape[0] // 2, *pred2.shape[1:], dtype=pred2.dtype, device=pred2.device)
    lib = _lib.load()
    _lib.check(lib.uav_cfg_combine(pred2.data_ptr(), out.data_ptr(), out.numel(), guidance_scale, _dt(pred2), _stream()),
               "uav_cfg_combine")
    return out


def window_blend(dst: torch.Tensor, src: torch.Tensor, t0: int, covered_mask: int):
    """dst: (B, C, T, H, W); src: (B, C, Tw, H, W)"""
    B, Cc, T, H, W = dst.shape
    Tw = src.shape[2]
    assert src.dtype == dst.dtype
    _dt(src)
    lib = _lib.load()
    _lib.check(lib.uav_window_blend(dst.data_ptr(), T, src.data_ptr(), Tw, t0, covered_mask, B * Cc, H * W, _dt(dst),
                                    _stream()), "uav_window_blend")
    return dst


def ddim_step_v0(model_output, sample, pred_type: int, sqrt_alpha: float, sqrt_beta: float, clip: bool, clip_range: float):
    out = torch.empty_like(sample)
    lib = _lib.load()
    assert model_output.dtype == sample.dtype
    _dt(model_output)
    _lib.check(lib.uav_ddim_step_v0(model_output.data_ptr(), sample.data_ptr(), out.data_ptr(), sample.numel(), pred_type,
                                    sqrt_alpha, sqrt_beta, 1 if clip else 0, clip_range, _dt(sample), _stream()),
               "uav_ddim_step_v0")
    return out


def ddim_step_vt(x0, model_output, sample, pred_type: int, sqrt_alpha, sqrt_beta, sqrt_alpha_prev, dir_coef, clip: bool,
                 clip_range: float, std_dev: float = 0.0, noise=None):
    out = torch.empty_like(sample)
    lib = _lib.load()
    for t in (x0, model_output):
        assert t.dtype == sample.dtype
        _dt(t)
    _lib.check(lib.uav_ddim_step_vt(x0.data_ptr(), model_output.data_ptr(), sample.data_ptr(), out.data_ptr(),
                                    sample.numel(), pred_type, sqrt_alpha, sqrt_beta, sqrt_alpha_prev, dir_coef,
                                    1 if clip else 0, clip_range, std_dev,
                                    noise.data_ptr() if noise is not None else None, _dt(sample), _stream()),
               "uav_ddim_step_vt")
    return out


def add_noise(x, noise, sqrt_alpha: float, sqrt_one_minus_alpha: float):
    out = torch.empty_like(x)
    assert noise.dtype == x.dtype
    _dt(noise)
    lib = _lib.load()
    _lib.check(lib.uav_add_noise(x.data_ptr(), noise.data_ptr(), out.data_ptr(), x.numel(), sqrt_alpha,
                                 sqrt_one_minus_alpha, _dt(x), _stream()), "uav_add_noise")
    return out


def propagate_step(feat_prop, feat_cur, flow_prop, flow_check, out, *, nearest: bool, fuse: bool, fuse_scale: float,
                   alpha1: float, alpha2: float, half_grid_sample: bool):
    """all tensors are (C|2, H, W) views with contiguous planes (stride(-1)==1, stride(-2)==W).
    `half_grid_sample`: how the grid sample rounds half inputs.  Only False is implemented: the opmath form of torch's
    CUDA grid_sampler (fp32 coordinates and weights, one final rounding); True raises."""
    if half_grid_sample:
        raise _lib.UavError("propagate_step: only the opmath grid sample (half_grid_sample=False) is implemented")
    Cc, H, W = feat_prop.shape
    for t in (feat_prop, feat_cur, flow_prop, flow_check, out):
        assert t.stride(-1) == 1 and t.stride(-2) == W and t.dtype == feat_prop.dtype and t.is_cuda
    dt = F16 if feat_prop.dtype == torch.float16 else F32
    lib = _lib.load()
    _lib.check(lib.uav_propagate_step(feat_prop.data_ptr(), feat_cur.data_ptr(), flow_prop.data_ptr(),
                                      flow_check.data_ptr(), out.data_ptr(), Cc, H, W, feat_prop.stride(0),
                                      feat_cur.stride(0), out.stride(0), flow_prop.stride(0), flow_check.stride(0),
                                      1 if nearest else 0, 1 if fuse else 0, fuse_scale, alpha1, alpha2,
                                      dt, _stream()), "uav_propagate_step")
    return out


def flow_resize_area(flows: torch.Tensor, size, scale: float):
    """F.interpolate(flows, size, mode='area') * scale, bit-identical to torch on the GPU.  flows: (b, c, t, h, w) fp16/fp32;
    size: (t_out, h_out, w_out)."""
    b, c, t, h, w = flows.shape
    to, ho, wo = (int(s) for s in size)
    x = flows.contiguous()
    out = torch.empty(b, c, to, ho, wo, dtype=x.dtype, device=x.device)
    lib = _lib.load()
    _lib.check(lib.uav_flow_resize_area(x.data_ptr(), out.data_ptr(), b * c, t, h, w, to, ho, wo, float(scale), _dt(x),
                                        _stream()), "uav_flow_resize_area")
    return out


# ---------------------------------------------------------------------------------------
# after the decode: colour fix + output packing (csrc/postprocess.cu) — planar fp32 "t c h w" frames
# ---------------------------------------------------------------------------------------
def _f32_planes(x: torch.Tensor) -> torch.Tensor:
    assert x.is_cuda and x.dim() == 4, "expected a CUDA (t, c, h, w) tensor"
    return x.float().contiguous()


def bicubic_upsample(x: torch.Tensor, scale: int = 4) -> torch.Tensor:
    """F.interpolate(x, scale_factor=scale, mode='bicubic') for a (t, c, h, w) fp32 tensor"""
    x = _f32_planes(x)
    t, c, h, w = x.shape
    out = torch.empty(t, c, h * scale, w * scale, dtype=torch.float32, device=x.device)
    lib = _lib.load()
    _lib.check(lib.uav_bicubic_upsample(x.data_ptr(), t * c, h, w, scale, out.data_ptr(), _stream()), "uav_bicubic_upsample")
    return out


def plane_stats(x: torch.Tensor, eps: float = 1e-5):
    """calc_mean_std: (mean, sqrt(unbiased var + eps)) per (t, c) plane, each shaped (t, c, 1, 1)"""
    x = _f32_planes(x)
    t, c, h, w = x.shape
    lib = _lib.load()
    ws = torch.empty(lib.uav_plane_stats_workspace_bytes(t * c), dtype=torch.uint8, device=x.device)
    mean = torch.empty(t, c, 1, 1, dtype=torch.float32, device=x.device)
    std = torch.empty_like(mean)
    _lib.check(lib.uav_plane_stats(x.data_ptr(), t * c, h * w, eps, ws.data_ptr(), mean.data_ptr(), std.data_ptr(),
                                   _stream()), "uav_plane_stats")
    return mean, std


def adain_apply(content: torch.Tensor, c_mean, c_std, s_mean, s_std) -> torch.Tensor:
    content = _f32_planes(content)
    t, c, h, w = content.shape
    out = torch.empty_like(content)
    lib = _lib.load()
    _lib.check(lib.uav_adain_apply(content.data_ptr(), t * c, h * w, c_mean.data_ptr(), c_std.data_ptr(),
                                   s_mean.data_ptr(), s_std.data_ptr(), out.data_ptr(), _stream()), "uav_adain_apply")
    return out


def wavelet_level(image: torch.Tensor, radius: int, *, low: Optional[torch.Tensor] = None,
                  high: Optional[torch.Tensor] = None, high_first: bool = False, add: Optional[torch.Tensor] = None):
    """one a-trous level: low <- blur(image) (+ add), high (+)= image - blur(image)"""
    t, c, h, w = image.shape
    for x in (image, low, high, add):
        assert x is None or (x.is_cuda and x.dtype == torch.float32 and x.is_contiguous() and x.shape == image.shape)
    lib = _lib.load()
    _lib.check(lib.uav_wavelet_level(image.data_ptr(), t * c, h, w, radius, low.data_ptr() if low is not None else None,
                                     high.data_ptr() if high is not None else None, 1 if high_first else 0,
                                     add.data_ptr() if add is not None else None, _stream()), "uav_wavelet_level")


def pack_video_uint8(frames: torch.Tensor) -> torch.Tensor:
    """(t, c, h, w) in [-1, 1] -> (t, h, w, c) uint8, as the reference packs frames for imageio"""
    frames = _f32_planes(frames)
    t, c, h, w = frames.shape
    out = torch.empty(t, h, w, c, dtype=torch.uint8, device=frames.device)
    lib = _lib.load()
    _lib.check(lib.uav_pack_video_uint8(frames.data_ptr(), t, c, h, w, out.data_ptr(), _stream()), "uav_pack_video_uint8")
    return out


def pack_frames_png(frames: torch.Tensor) -> torch.Tensor:
    """(t, c, h, w) -> (t, h, w, c) uint8 with the rounding of save_image(normalize=True, value_range=(-1, 1))"""
    frames = _f32_planes(frames)
    t, c, h, w = frames.shape
    out = torch.empty(t, h, w, c, dtype=torch.uint8, device=frames.device)
    lib = _lib.load()
    _lib.check(lib.uav_pack_frames_png(frames.data_ptr(), t, c, h, w, out.data_ptr(), _stream()), "uav_pack_frames_png")
    return out


def unpack_video_uint8(frames: torch.Tensor, size=None, channels_last: bool = False) -> torch.Tensor:
    """(t, h, w, 3) uint8 BGR frames on the GPU -> (1, 3, t, h_out, w_out) fp32 RGB in [-1, 1]; `size` = (h_out, w_out)
    area-downsamples in the same pass (None: no resize), rounded as torch's area resize rounds NCHW frames, or
    channels-last frames when `channels_last`"""
    assert frames.is_cuda and frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[-1] == 3, \
        "expected CUDA (t, h, w, 3) uint8 frames"
    frames = frames.contiguous()
    t, h, w, _ = frames.shape
    ho, wo = (h, w) if size is None else (int(s) for s in size)
    out = torch.empty(1, 3, t, ho, wo, dtype=torch.float32, device=frames.device)
    lib = _lib.load()
    _lib.check(lib.uav_unpack_video_uint8(frames.data_ptr(), t, h, w, ho, wo, 1 if channels_last else 0, out.data_ptr(),
                                          _stream()),
               "uav_unpack_video_uint8")
    return out


# ---------------------------------------------------------------------------------------
# RAFT optical flow (csrc/raft.cu + uav_conv2d_taps): channels-last fp16 activations, fp32 correlation / coordinates
# ---------------------------------------------------------------------------------------
ACT_RELU, ACT_SIGMOID, ACT_TANH = 3, 4, 5


def conv2d_taps(x: torch.Tensor, w: torch.Tensor, bias=None, *, pad_top: int, pad_left: int, out=None, residual=None,
                act=ACT_NONE, out_dtype=torch.float16):
    """stride-1 same-size conv with a (kh, kw) window and asymmetric padding; x (N, H, W, Cin) fp16 (channel-slice views
    allowed), w (Cout, kh, kw, Cin) fp16"""
    assert x.dtype == torch.float16 and w.dtype == torch.float16 and w.is_contiguous() and x.dim() == 4
    NB, H, W, Cin = x.shape
    Cout, kh, kw, Cin_w = w.shape
    assert Cin_w == Cin, (Cin_w, Cin)
    if out is None:
        out = torch.empty(NB, H, W, Cout, dtype=out_dtype, device=x.device)
    assert tuple(out.shape) == (NB, H, W, Cout)
    e = _epi(out, bias, None, 0, residual, act)
    return _igemm("uav_conv2d_taps", (x.data_ptr(), NB, H, W, Cin, _pixel_ld(x), w.data_ptr(), Cout, kh, kw, pad_top,
                                      pad_left), out, e, None, 2.0 * NB * H * W * Cout * Cin * kh * kw,
                  2.0 * (NB * H * W * Cin + w.numel()) + out.element_size() * NB * H * W * Cout,
                  f"conv{kh}x{kw}taps {NB}x{H}x{W} {Cin}->{Cout}")


def instnorm_relu(x: torch.Tensor, relu: bool = True, eps: float = 1e-5) -> torch.Tensor:
    """(N, H, W, C) fp16 contiguous -> InstanceNorm2d (no affine) (+ ReLU)"""
    assert x.is_cuda and x.dtype == torch.float16 and x.is_contiguous() and x.dim() == 4
    n, h, w, c = x.shape
    lib = _lib.load()
    ws = torch.empty(lib.uav_instnorm_workspace_bytes(n, c), dtype=torch.uint8, device=x.device)
    y = torch.empty_like(x)
    _lib.check(lib.uav_instnorm_relu(x.data_ptr(), n, h * w, c, eps, 1 if relu else 0, y.data_ptr(), ws.data_ptr(), _stream()),
               "uav_instnorm_relu")
    return y


def add_relu(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    assert a.shape == b.shape and a.dtype == b.dtype == torch.float16 and a.is_contiguous() and b.is_contiguous()
    y = torch.empty_like(a)
    lib = _lib.load()
    _lib.check(lib.uav_add_relu(a.data_ptr(), b.data_ptr(), y.data_ptr(), a.numel(), _stream()), "uav_add_relu")
    return y


def raft_split_tanh_relu(cnet: torch.Tensor, net: torch.Tensor, inp_a: torch.Tensor, inp_b: Optional[torch.Tensor]):
    """cnet (rows, 2C) fp16 contiguous; net / inp_* are (rows, C) channel-slice views"""
    rows, c2 = cnet.shape
    lib = _lib.load()
    _lib.check(lib.uav_raft_split_tanh_relu(cnet.data_ptr(), rows, c2 // 2, net.data_ptr(), net.stride(0), inp_a.data_ptr(),
                                            inp_a.stride(0), inp_b.data_ptr() if inp_b is not None else None,
                                            inp_b.stride(0) if inp_b is not None else 0, _stream()), "uav_raft_split_tanh_relu")


def avgpool2x2_f32(x: torch.Tensor) -> torch.Tensor:
    """(planes, h, w) fp32 -> (planes, h // 2, w // 2)"""
    assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous() and x.dim() == 3
    planes, h, w = x.shape
    out = torch.empty(planes, h // 2, w // 2, dtype=torch.float32, device=x.device)
    lib = _lib.load()
    _lib.check(lib.uav_avgpool2x2_f32(x.data_ptr(), planes, h, w, out.data_ptr(), _stream()), "uav_avgpool2x2_f32")
    return out


def raft_corr_lookup(levels, coords: torch.Tensor, out: torch.Tensor):
    """levels: 4 fp32 tensors (pixels, h_i, w_i); coords (pixels, 2) fp32; out (pixels, >= 324) fp16 contiguous"""
    assert len(levels) == 4 and coords.dtype == torch.float32 and coords.is_contiguous() and out.dtype == torch.float16
    pixels = coords.shape[0]
    ptrs = (C.c_void_p * 4)(*[lv.data_ptr() for lv in levels])
    hs = (C.c_int32 * 4)(*[lv.shape[1] for lv in levels])
    ws = (C.c_int32 * 4)(*[lv.shape[2] for lv in levels])
    for lv in levels:
        assert lv.dtype == torch.float32 and lv.is_contiguous() and lv.shape[0] == pixels
    lib = _lib.load()
    _lib.check(lib.uav_raft_corr_lookup(ptrs, hs, ws, coords.data_ptr(), pixels, out.data_ptr(), out.stride(0), _stream()),
               "uav_raft_corr_lookup")
    return out


def raft_gru_rh(zr: torch.Tensor, h: torch.Tensor, out: torch.Tensor):
    rows, c = h.shape
    lib = _lib.load()
    _lib.check(lib.uav_raft_gru_rh(zr.data_ptr(), zr.stride(0), h.data_ptr(), h.stride(0), out.data_ptr(), out.stride(0), rows, c,
                                   _stream()), "uav_raft_gru_rh")


def raft_gru_update(zr: torch.Tensor, q: torch.Tensor, h: torch.Tensor):
    rows, c = h.shape
    lib = _lib.load()
    _lib.check(lib.uav_raft_gru_update(zr.data_ptr(), zr.stride(0), q.data_ptr(), q.stride(0), h.data_ptr(), h.stride(0), rows, c,
                                       _stream()), "uav_raft_gru_update")


def raft_flow_update(coords1: torch.Tensor, delta: Optional[torch.Tensor], h8: int, w8: int, flow16=None, dst_a=None, dst_b=None):
    """coords1 (rows, 2) fp32 in place (+= delta (rows, >= 2) fp32); fp16 flow into channels [0, 2) of the given views"""
    rows = coords1.shape[0]
    lib = _lib.load()

    def pl(t):
        return (t.data_ptr(), t.stride(0)) if t is not None else (None, 0)

    _lib.check(lib.uav_raft_flow_update(coords1.data_ptr(), delta.data_ptr() if delta is not None else None,
                                        delta.stride(0) if delta is not None else 0, rows, h8, w8, *pl(flow16), *pl(dst_a),
                                        *pl(dst_b), _stream()), "uav_raft_flow_update")


def raft_convex_upsample(coords1: torch.Tensor, mask: torch.Tensor, nimg: int, h8: int, w8: int) -> torch.Tensor:
    out = torch.empty(nimg, 2, 8 * h8, 8 * w8, dtype=torch.float32, device=coords1.device)
    lib = _lib.load()
    _lib.check(lib.uav_raft_convex_upsample(coords1.data_ptr(), mask.data_ptr(), mask.stride(0), nimg, h8, w8, out.data_ptr(),
                                            _stream()), "uav_raft_convex_upsample")
    return out


# ---------------------------------------------------------------------------------------
# CLIP text encoder: causal attention over the 77-token prompt, GELU epilogues
# ---------------------------------------------------------------------------------------
ACT_GELU, ACT_QUICK_GELU = 6, 7


def attention_causal(q, k, v, heads: int, *, scale: Optional[float] = None, out=None):
    """q, k, v: (batch, n, heads*d) fp16 (column slices of a fused qkv buffer allowed), n <= 128"""
    batch, n, Cc = q.shape
    d = Cc // heads
    if out is None:
        out = torch.empty(batch, n, Cc, dtype=torch.float16, device=q.device)
    if scale is None:
        scale = d ** -0.5
    for t in (q, k, v, out):
        assert t.is_cuda and t.dtype == torch.float16 and t.stride(-1) == 1 and t.stride(0) == t.shape[1] * t.stride(1)
    lib = _lib.load()
    _lib.check(lib.uav_attention_causal(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), batch, heads, d, n,
                                        q.stride(1), k.stride(1), v.stride(1), out.stride(1), scale, _stream()),
               "uav_attention_causal")
    return out


# ---------------------------------------------------------------------------------------
# LLaVA-1.5 captioner (llava.py): the Llama decoder's kernels and the sampler
# ---------------------------------------------------------------------------------------
def _rows(x: torch.Tensor):
    """(rows, row stride) of a 2-D fp16 tensor whose last dim is dense"""
    assert x.is_cuda and x.dtype == torch.float16 and x.dim() == 2 and x.stride(-1) == 1
    return x.shape[0], x.stride(0)


def rms_norm(x: torch.Tensor, weight: torch.Tensor, eps: float, out=None):
    """transformers LlamaRMSNorm of the rows of x (rows, C) fp16 (a row slice or column slice allowed); weight fp16 (C,)"""
    rows, ldx = _rows(x)
    assert weight.dtype == torch.float16 and weight.is_contiguous() and weight.numel() == x.shape[1]
    if out is None:
        out = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    _, ldo = _rows(out)
    with _timed("rmsnorm", 0.0, 2.0 * 2 * x.numel()):
        _lib.check(_lib.load().uav_rmsnorm(x.data_ptr(), rows, x.shape[1], ldx, weight.data_ptr(), eps, out.data_ptr(),
                                           ldo, _stream()), "uav_rmsnorm")
    return out


def rope_kv_append(qkv: torch.Tensor, heads: int, p0: int, cos_sin: torch.Tensor, k_cache: torch.Tensor,
                   v_cache: torch.Tensor):
    """rotate q (in place) and k of the fused q|k|v rows qkv (n, >= 3 heads 128) at positions [p0, p0 + n); rotated k
    and v go to rows [p0, p0 + n) of k_cache / v_cache (L_max, heads 128).  cos_sin: fp32 (positions, 64, 2)"""
    n, ld = _rows(qkv)
    rows, ld_kv = _rows(k_cache)
    assert v_cache.shape == k_cache.shape and v_cache.stride() == k_cache.stride()
    assert cos_sin.dtype == torch.float32 and cos_sin.is_contiguous() and cos_sin.shape[1:] == (64, 2)
    _lib.check(_lib.load().uav_rope_kv_append(qkv.data_ptr(), ld, n, heads, 128, p0, cos_sin.data_ptr(), cos_sin.shape[0],
                                              k_cache.data_ptr(), v_cache.data_ptr(), ld_kv, rows, _stream()),
               "uav_rope_kv_append")


def swiglu(gate_up: torch.Tensor, out=None):
    """silu(gate) * up of the fused (rows, 2 I) gate|up GEMM output -> (rows, I) fp16"""
    rows, ld = _rows(gate_up)
    inter = gate_up.shape[1] // 2
    if out is None:
        out = torch.empty(rows, inter, dtype=torch.float16, device=gate_up.device)
    _, ldo = _rows(out)
    _lib.check(_lib.load().uav_swiglu(gate_up.data_ptr(), ld, rows, inter, out.data_ptr(), ldo, _stream()), "uav_swiglu")
    return out


def gemv(w: torch.Tensor, x: torch.Tensor, *, residual=None, out=None, out_dtype=torch.float16):
    """out (N,) = w (N, K) @ x (K,) (+ residual (N,)), the one-row weight stream of a decode step; fp16 or fp32 out"""
    assert w.is_cuda and w.dtype == torch.float16 and w.is_contiguous() and w.dim() == 2
    N, K = w.shape
    assert x.dtype == torch.float16 and x.numel() == K and x.is_contiguous()
    if out is None:
        out = torch.empty(N, dtype=out_dtype, device=w.device)
    assert out.numel() == N and out.is_contiguous() and out.dtype in (torch.float16, torch.float32)
    if residual is not None:
        assert residual.dtype == torch.float16 and residual.numel() == N and residual.is_contiguous()
    with _timed("gemv", 2.0 * N * K, 2.0 * (N * K + K + N), f"gemv N{N} K{K}"):
        _lib.check(_lib.load().uav_gemv(w.data_ptr(), N, K, x.data_ptr(), 0 if residual is None else residual.data_ptr(),
                                        out.data_ptr(), F16 if out.dtype == torch.float16 else F32, _stream()),
                   "uav_gemv")
    return out


def attention_decode(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, L: int, heads: int, *,
                     scale: Optional[float] = None, out=None):
    """one query row q (heads 128,) fp16 against rows [0, L) of the KV cache (L_max, heads 128) -> (heads 128,) fp16"""
    _, ld_kv = _rows(k_cache)
    assert v_cache.stride() == k_cache.stride() and q.dtype == torch.float16 and q.is_contiguous()
    if out is None:
        out = torch.empty(heads * 128, dtype=torch.float16, device=q.device)
    lib = _lib.load()
    ws_bytes = int(lib.uav_attention_decode_workspace_bytes(heads, L))
    ws = torch.empty(ws_bytes // 4, dtype=torch.float32, device=q.device)
    _lib.check(lib.uav_attention_decode(q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(), ld_kv, L, heads, 128,
                                        128 ** -0.5 if scale is None else scale, out.data_ptr(), ws.data_ptr(), ws_bytes,
                                        _stream()), "uav_attention_decode")
    return out


def sample_top_p(logits: torch.Tensor, temperature: float, top_p: float, u: float, out=None) -> torch.Tensor:
    """next token id (a device int64 scalar) from fp32 logits (V,): temperature, top-p nucleus, inverse CDF at u in
    [0, 1); temperature 0 = argmax (first index on ties)"""
    assert logits.is_cuda and logits.dtype == torch.float32 and logits.is_contiguous()
    if out is None:
        out = torch.empty((), dtype=torch.int64, device=logits.device)
    _lib.check(_lib.load().uav_sample_top_p(logits.data_ptr(), logits.numel(), temperature, top_p, u, out.data_ptr(),
                                            _stream()), "uav_sample_top_p")
    return out


# batched decode: B sequences per step (llava.py captions up to 8 images per weight pass); each row's result is
# bit-identical to the one-row op on that row
def gemv_rows(w: torch.Tensor, x: torch.Tensor, *, residual=None, out=None, out_dtype=torch.float16):
    """out (rows, N) = x (rows, K) @ w (N, K)^T (+ residual (rows, N)), 1 <= rows <= 8, w streamed once for all rows"""
    assert w.is_cuda and w.dtype == torch.float16 and w.is_contiguous() and w.dim() == 2
    N, K = w.shape
    assert x.dtype == torch.float16 and x.dim() == 2 and x.shape[1] == K and x.is_contiguous()
    rows = x.shape[0]
    assert 1 <= rows <= 8, rows
    if out is None:
        out = torch.empty(rows, N, dtype=out_dtype, device=w.device)
    assert out.shape == (rows, N) and out.is_contiguous() and out.dtype in (torch.float16, torch.float32)
    if residual is not None:
        assert residual.dtype == torch.float16 and residual.shape == (rows, N) and residual.is_contiguous()
    with _timed("gemv", 2.0 * rows * N * K, 2.0 * (N * K + rows * (K + N)), f"gemv_rows{rows} N{N} K{K}"):
        _lib.check(_lib.load().uav_gemv_rows(w.data_ptr(), N, K, x.data_ptr(), rows,
                                             0 if residual is None else residual.data_ptr(), out.data_ptr(),
                                             F16 if out.dtype == torch.float16 else F32, _stream()),
                   "uav_gemv_rows")
    return out


def _batched_cache(k_cache: torch.Tensor, v_cache: torch.Tensor):
    """(batch, rows, batch stride, row stride) of per-sequence KV caches (B, L_max, heads 128) fp16"""
    assert k_cache.is_cuda and k_cache.dtype == torch.float16 and k_cache.dim() == 3 and k_cache.stride(-1) == 1
    assert v_cache.shape == k_cache.shape and v_cache.stride() == k_cache.stride() and v_cache.dtype == torch.float16
    return k_cache.shape[0], k_cache.shape[1], k_cache.stride(0), k_cache.stride(1)


def rope_kv_append_batched(qkv: torch.Tensor, heads: int, p0: int, cos_sin: torch.Tensor, k_cache: torch.Tensor,
                           v_cache: torch.Tensor):
    """rope_kv_append on B sequences: qkv (B, n, >= 3 heads 128) fused q|k|v rows at positions [p0, p0 + n) of every
    sequence (q rotated in place); k_cache / v_cache (B, L_max, heads 128)"""
    assert qkv.is_cuda and qkv.dtype == torch.float16 and qkv.dim() == 3 and qkv.stride(-1) == 1
    B, n, _ = qkv.shape
    Bc, rows, kv_bs, ld_kv = _batched_cache(k_cache, v_cache)
    assert Bc == B, (Bc, B)
    assert cos_sin.dtype == torch.float32 and cos_sin.is_contiguous() and cos_sin.shape[1:] == (64, 2)
    _lib.check(_lib.load().uav_rope_kv_append_batched(qkv.data_ptr(), qkv.stride(1), qkv.stride(0), B, n, heads, 128,
                                                      p0, cos_sin.data_ptr(), cos_sin.shape[0], k_cache.data_ptr(),
                                                      v_cache.data_ptr(), ld_kv, kv_bs, rows, _stream()),
               "uav_rope_kv_append_batched")


def attention_decode_batched(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, L: int, heads: int, *,
                             scale: Optional[float] = None, out=None):
    """attention_decode on B sequences: q (B, heads 128) fp16 (a column slice of the fused q|k|v rows allowed)
    against rows [0, L) of each sequence's cache (B, L_max, heads 128) -> (B, heads 128) fp16"""
    B, _, kv_bs, ld_kv = _batched_cache(k_cache, v_cache)
    assert q.is_cuda and q.dtype == torch.float16 and q.shape == (B, heads * 128) and q.stride(-1) == 1
    if out is None:
        out = torch.empty(B, heads * 128, dtype=torch.float16, device=q.device)
    assert out.dtype == torch.float16 and out.shape == (B, heads * 128) and out.stride(-1) == 1
    lib = _lib.load()
    ws_bytes = int(lib.uav_attention_decode_batched_workspace_bytes(B, heads, L))
    ws = torch.empty(ws_bytes // 4, dtype=torch.float32, device=q.device)
    _lib.check(lib.uav_attention_decode_batched(q.data_ptr(), q.stride(0), k_cache.data_ptr(), v_cache.data_ptr(),
                                                ld_kv, kv_bs, B, L, heads, 128, 128 ** -0.5 if scale is None else scale,
                                                out.data_ptr(), out.stride(0), ws.data_ptr(), ws_bytes, _stream()),
               "uav_attention_decode_batched")
    return out


def sample_top_p_batched(logits: torch.Tensor, temperature: float, top_p: float, u, out=None) -> torch.Tensor:
    """sample_top_p on each row of fp32 logits (B, V), B <= 8, row b at uniform u[b] -> (B,) device int64 tokens"""
    assert logits.is_cuda and logits.dtype == torch.float32 and logits.dim() == 2 and logits.stride(-1) == 1
    B, V = logits.shape
    assert 1 <= B <= 8 and len(u) == B, (B, len(u))
    if out is None:
        out = torch.empty(B, dtype=torch.int64, device=logits.device)
    assert out.dtype == torch.int64 and out.shape == (B,) and out.is_contiguous()
    us = (C.c_float * B)(*u)
    _lib.check(_lib.load().uav_sample_top_p_batched(logits.data_ptr(), logits.stride(0), B, V, temperature, top_p, us,
                                                    out.data_ptr(), _stream()), "uav_sample_top_p_batched")
    return out


# weight-only int8 decoder Linears (include/uav_b200_int8.h): q int8 (N, K) with an fp32 per-row absmax (N,)
def quantize_rows_int8(w: torch.Tensor, q: torch.Tensor, absmax: torch.Tensor):
    """q[n] = round_half_even((w[n] * 127) / absmax[n]), absmax[n] = max |w[n]| (bitsandbytes' row-wise rule) of fp16
    w (N, K) (a row slice of a wider matrix allowed), into int8 q (N, K) and fp32 absmax (N,), which may be row slices
    of a larger destination"""
    assert w.is_cuda and w.dtype == torch.float16 and w.dim() == 2 and w.stride(1) == 1
    N, K = w.shape
    assert q.dtype == torch.int8 and q.shape == (N, K) and q.is_contiguous()
    assert absmax.dtype == torch.float32 and absmax.shape == (N,) and absmax.is_contiguous()
    with _timed("quantize_int8", 0.0, 2.0 * N * K + N * K + 4.0 * N, f"quantize_int8 N{N} K{K}"):
        _lib.check(_lib.load().uav_quantize_rows_int8(w.data_ptr(), N, K, w.stride(0), q.data_ptr(), absmax.data_ptr(),
                                                      _stream()), "uav_quantize_rows_int8")


def dequantize_rows_int8(q: torch.Tensor, absmax: torch.Tensor, out=None) -> torch.Tensor:
    """fp16((q * absmax[n]) / 127) of int8 q (N, K) -> fp16 (N, K), the prefill's weight"""
    assert q.is_cuda and q.dtype == torch.int8 and q.dim() == 2 and q.is_contiguous()
    N, K = q.shape
    assert absmax.dtype == torch.float32 and absmax.shape == (N,) and absmax.is_contiguous()
    if out is None:
        out = torch.empty(N, K, dtype=torch.float16, device=q.device)
    assert out.dtype == torch.float16 and out.shape == (N, K) and out.is_contiguous()
    with _timed("dequantize_int8", 0.0, N * K + 4.0 * N + 2.0 * N * K, f"dequantize_int8 N{N} K{K}"):
        _lib.check(_lib.load().uav_dequantize_rows_int8(q.data_ptr(), absmax.data_ptr(), N, K, out.data_ptr(),
                                                        _stream()), "uav_dequantize_rows_int8")
    return out


def gemv_rows_int8(q: torch.Tensor, absmax: torch.Tensor, x: torch.Tensor, *, residual=None, out=None,
                   out_dtype=torch.float16):
    """out (rows, N) = (x (rows, K) @ q (N, K)^T) * absmax / 127 (+ residual (rows, N)), 1 <= rows <= 8, the int8
    weight stream of a decode step; each row's result does not depend on the other rows"""
    assert q.is_cuda and q.dtype == torch.int8 and q.dim() == 2 and q.is_contiguous()
    N, K = q.shape
    assert absmax.dtype == torch.float32 and absmax.shape == (N,) and absmax.is_contiguous()
    assert x.dtype == torch.float16 and x.dim() == 2 and x.shape[1] == K and x.is_contiguous()
    rows = x.shape[0]
    assert 1 <= rows <= 8, rows
    if out is None:
        out = torch.empty(rows, N, dtype=out_dtype, device=q.device)
    assert out.shape == (rows, N) and out.is_contiguous() and out.dtype in (torch.float16, torch.float32)
    if residual is not None:
        assert residual.dtype == torch.float16 and residual.shape == (rows, N) and residual.is_contiguous()
    with _timed("gemv", 2.0 * rows * N * K, N * K + 4.0 * N + 2.0 * rows * (K + N), f"gemv_rows_int8 {rows} N{N} K{K}"):
        _lib.check(_lib.load().uav_gemv_rows_int8(q.data_ptr(), absmax.data_ptr(), N, K, x.data_ptr(), rows,
                                                  0 if residual is None else residual.data_ptr(), out.data_ptr(),
                                                  F16 if out.dtype == torch.float16 else F32, _stream()),
                   "uav_gemv_rows_int8")
    return out
