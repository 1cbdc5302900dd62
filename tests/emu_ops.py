"""emu_ops.py — plain-torch stand-ins for the kernel wrappers of `upscale_a_video_b200/ops.py` (TEST INFRASTRUCTURE).

Each function re-states the CONTRACT of one wrapper (argument meaning, channels-last layouts, channel-slice views,
`out=` placement, fused-epilogue order, fp32 math with ONE rounding to the fp16 output) so that the host logic of the
package — weight packing, buffer plumbing, batching, caching, the module graph — can be exercised on a CPU-only box
against the reference fixtures (`tests/test_host_emulated.py`).  The kernels themselves are validated on the GPU
(`-m gpu`); the product never imports this file and keeps refusing CPU tensors (`_lib.require_cuda`), which the emulated
tests stub explicitly."""
import math

import torch
import torch.nn.functional as F

ACT_NONE, ACT_SILU, ACT_GEGLU = 0, 1, 2


def _epilogue(acc, bias, rowvec, rows_per_vec, residual, act, out, out_dtype, out_scale=1.0):
    """acc: (..., N) fp32 pre-bias accumulators flattened over rows in the output's row order"""
    n = acc.shape[-1]
    v = acc.reshape(-1, n)
    if bias is not None:
        v = v + bias.float()
    if rowvec is not None:
        idx = torch.arange(v.shape[0]) // max(int(rows_per_vec), 1)
        v = v + rowvec.float().reshape(-1, rowvec.shape[-1])[idx][:, :n]
    if act == ACT_SILU:
        v = F.silu(v)
    elif act == ACT_GEGLU:
        half = n // 2
        v = v[:, :half] * F.gelu(v[:, half:])
    if out_scale != 1.0:
        v = v * out_scale
    if residual is not None:
        v = v + residual.float().reshape(-1, residual.shape[-1])[:, :v.shape[-1]]
    return v


class EmuStats:
    """stand-in for ops.GnStats: marks a tensor whose producer "emitted" GroupNorm statistics, so that the host logic
    around them (virtual concat, slot allocation) runs on the CPU; the emulated GroupNorm recomputes its statistics"""

    def __init__(self, C, batch):
        self.C, self.batch = C, batch

    def slabs_for(self, n_outer, batch):
        return n_outer if self.batch == batch else (1 if self.batch == 1 and n_outer == batch else 0)


def _finish(v, lead_shape, out, out_dtype, gn_stats=False):
    v = v.reshape(*lead_shape, v.shape[-1])
    if out is None:
        out = v.to(out_dtype)
    else:
        out.copy_(v)
    if gn_stats and out.dtype == torch.float16 and out.shape[-1] >= 64 and out.shape[-1] % 8 == 0:
        out.uav_gn = [EmuStats(out.shape[-1], out.shape[0] if out.dim() > 2 else 1)]
    return out


def group_norm_cat(parts, gamma, beta, groups, eps, *, silu, n_outer):
    B = max(p.shape[0] for p in parts)
    C = sum(p.shape[-1] for p in parts)
    if (C // groups) % 8 or n_outer != B:
        return None
    for p in parts:
        st = getattr(p, "uav_gn", None)
        if not st or len(st) != 1 or not st[0].slabs_for(n_outer, B):
            return None
    cat = torch.cat([p.expand(B, *p.shape[1:]) for p in parts], dim=-1)
    return group_norm(cat, gamma, beta, groups, eps, silu=silu, n_outer=n_outer)


def linear(a, w, bias=None, *, out=None, residual=None, rowvec=None, rows_per_vec=0, act=ACT_NONE, out_dtype=torch.float16,
           out_scale=1.0, gn_stats=False):
    acc = a.float().reshape(-1, a.shape[-1]) @ w.float().t()
    v = _epilogue(acc, bias, rowvec, rows_per_vec, residual, act, out, out_dtype, out_scale)
    return _finish(v, a.shape[:-1], out, out_dtype, gn_stats and act != ACT_GEGLU)


def _conv_nhwc(x4, w, stride, pads):
    """x4 (N, H, W, C) fp32, w (Cout, kh, kw, Cin); pads = (left, right, top, bottom)"""
    xp = F.pad(x4.permute(0, 3, 1, 2), pads)
    return F.conv2d(xp, w.float().permute(0, 3, 1, 2), stride=stride).permute(0, 2, 3, 1)


def conv2d(x, w, bias=None, *, stride=1, pad_mode=0, out=None, residual=None, rowvec=None, rows_per_vec=0, act=ACT_NONE,
           out_dtype=torch.float16, out_scale=1.0, gn_stats=False):
    *lead, H, W, Cin = x.shape
    k = w.shape[1]
    x4 = x.float().reshape(-1, H, W, Cin)
    if stride == 1:
        p = k // 2
        y = _conv_nhwc(x4, w, 1, (p, p, p, p))
    elif pad_mode == 0:
        y = _conv_nhwc(x4, w, 2, (1, 1, 1, 1))
    else:  # F.pad (0, 1, 0, 1) then no padding
        y = _conv_nhwc(x4, w, 2, (0, 1, 0, 1))
    v = _epilogue(y, bias, rowvec, rows_per_vec, residual, act, out, out_dtype, out_scale)
    return _finish(v, (*lead, y.shape[1], y.shape[2]), out, out_dtype, gn_stats)


def collapse_upsample_filter(w):
    from upscale_a_video_b200 import ops as real_ops  # pure torch math, no kernel involved
    return real_ops.collapse_upsample_filter(w)


def upsample2x_conv3x3(x, w4, bias=None, out=None):
    """phase p = a*2+b -> output pixel (2y+a, 2x+b); taps read rows {y-1, y} (a=0) or {y, y+1} (a=1), columns likewise"""
    *lead, H, W, Cin = x.shape
    Cout = w4.shape[1]
    x4 = x.float().reshape(-1, H, W, Cin)
    out_, out = out, torch.zeros(x4.shape[0], 2 * H, 2 * W, Cout)
    for a in range(2):
        for b in range(2):
            pads = (1 - b, b, 1 - a, a)  # left, right, top, bottom
            y = _conv_nhwc(x4, w4[a * 2 + b], 1, pads)
            out[:, a::2, b::2] = y
    acc = out
    if bias is not None:
        acc = acc + bias.float()
    res = acc.reshape(*lead, 2 * H, 2 * W, Cout).half()
    if out_ is not None:
        out_.copy_(res)
        return out_
    return res


def conv_temporal(x, w, bias=None, *, out=None, residual=None, rowvec=None, rows_per_vec=0, act=ACT_NONE, out_dtype=torch.float16,
                  out_scale=1.0, gn_stats=False):
    B, T, H, W, Cin = x.shape
    Cout, k, _ = w.shape
    xp = F.pad(x.float().permute(0, 4, 1, 2, 3), (0, 0, 0, 0, k // 2, k // 2))
    y = F.conv3d(xp, w.float().permute(0, 2, 1)[:, :, :, None, None]).permute(0, 2, 3, 4, 1)
    v = _epilogue(y, bias, rowvec, rows_per_vec, residual, act, out, out_dtype, out_scale)
    return _finish(v, (B, T, H, W), out, out_dtype, gn_stats)


def conv3d(x, w, bias=None, *, out=None, residual=None, act=ACT_NONE, out_dtype=torch.float16, out_scale=1.0, gn_stats=False):
    B, T, H, W, Cin = x.shape
    y = F.conv3d(x.float().permute(0, 4, 1, 2, 3), w.float().permute(0, 4, 1, 2, 3), padding=1).permute(0, 2, 3, 4, 1)
    v = _epilogue(y, bias, None, 0, residual, act, out, out_dtype, out_scale)
    return _finish(v, (B, T, H, W), out, out_dtype, gn_stats)


def group_norm(x, gamma, beta, groups, eps, *, silu, n_outer, out=None, stats=None, batch=None):
    C = x.shape[-1]
    v = x.float().reshape(n_outer, -1, C).permute(0, 2, 1)  # (n, C, pixels)
    y = F.group_norm(v, groups, gamma.float(), beta.float(), eps)
    if silu:
        y = F.silu(y)
    y = y.permute(0, 2, 1).reshape(x.shape)
    if out is None:
        return y.half()
    out.copy_(y)
    return out


def layer_norm(x, gamma, beta, eps=1e-5, out=None):
    y = F.layer_norm(x.float(), (x.shape[-1],), gamma.float(), beta.float(), eps)
    if out is None:
        return y.half()
    out.copy_(y)
    return out


def attention(q, k, v, heads, *, kv_batch_div=1, scale=None, out=None):
    batch, nq, C = q.shape
    d = C // heads
    scale = d ** -0.5 if scale is None else scale
    kk = k.float().repeat_interleave(kv_batch_div, dim=0).reshape(batch, -1, heads, d).permute(0, 2, 1, 3)
    vv = v.float().repeat_interleave(kv_batch_div, dim=0).reshape(batch, -1, heads, d).permute(0, 2, 1, 3)
    qq = q.float().reshape(batch, nq, heads, d).permute(0, 2, 1, 3)
    p = torch.softmax(qq @ kk.transpose(-1, -2) * scale, dim=-1)
    o = (p @ vv).permute(0, 2, 1, 3).reshape(batch, nq, C)
    if out is None:
        return o.half()
    out.copy_(o)
    return out


def temporal_attention(q, k, v, heads, rot, bias, *, out=None):
    """q, k, v (B, F, HW, heads*d); rot (F, 16, 2) cos / sin of frame * freq_pair; bias (heads, F, F); rotary on the first 32
    dims of every head, interleaved pairs (x0, x1) -> (x0 c - x1 s, x1 c + x0 s)"""
    B, Fr, HW, C = q.shape
    d = C // heads

    def seq(t):  # -> (B*HW, heads, F, d)
        return t.float().permute(0, 2, 1, 3).reshape(B * HW, Fr, heads, d).permute(0, 2, 1, 3)

    def rotary(t):
        cos, sin = rot[:, :, 0].float(), rot[:, :, 1].float()  # (F, 16)
        r = t[..., :32].reshape(*t.shape[:-1], 16, 2)
        x0, x1 = r[..., 0], r[..., 1]
        rr = torch.stack([x0 * cos - x1 * sin, x1 * cos + x0 * sin], dim=-1).reshape(*t.shape[:-1], 32)
        return torch.cat([rr, t[..., 32:]], dim=-1)

    qs, ks, vs = rotary(seq(q) * d ** -0.5), rotary(seq(k)).half().float(), seq(v)
    p = torch.softmax(qs @ ks.transpose(-1, -2) + bias.float(), dim=-1)
    o = (p @ vs).permute(0, 2, 1, 3).reshape(B, HW, Fr, C).permute(0, 2, 1, 3)
    if out is None:
        return o.half()
    out.copy_(o)
    return out


def copy_channels(src, dst):
    dst.copy_(src)
    return dst


def concat_channels(a, b):
    if b.shape[0] == 1 and a.shape[0] > 1:
        b = b.expand(a.shape[0], *b.shape[1:])
    return torch.cat([a, b], dim=-1)


def repeat_batch(x, n):
    return _carry(_repeat_batch(x, n), x)


def _carry(dst, src):
    if getattr(src, "uav_gn", None):
        dst.uav_gn = src.uav_gn
    return dst


def _repeat_batch(x, n):
    return x.repeat(n, *([1] * (x.dim() - 1)))


def upsample_nearest(x, size=None):
    *lead, H, W, C = x.shape
    x4 = x.reshape(-1, H, W, C).permute(0, 3, 1, 2).float()
    y = F.interpolate(x4, scale_factor=2, mode="nearest") if size is None else F.interpolate(x4, size=tuple(size), mode="nearest")
    return y.permute(0, 2, 3, 1).reshape(*lead, y.shape[-2], y.shape[-1], C).to(x.dtype)


def planar_to_channels_last(src, dst, c_off=0, scale=1.0):
    dst[..., c_off:c_off + src.shape[1]] = (src.float() * scale).permute(0, 2, 3, 4, 1)
    return dst


def channels_last_to_planar(src, C, out_dtype, clamp=False):
    y = src[..., :C].float().permute(0, 4, 1, 2, 3)
    if clamp:
        y = y.clamp(-1, 1)
    return y.to(out_dtype).contiguous()


def silu(x):
    return F.silu(x.float()).half()


def sft_fuse(dec, scale, shift, w, out_scale=1.0):
    d = dec.float()
    return ((d + w * (d * scale.float() + shift.float())) * out_scale).half()


def timestep_embedding(t, dim, flip_sin_to_cos, freq_shift):
    """diffusers.models.embeddings.get_timestep_embedding (max_period 10000, scale 1)"""
    half = dim // 2
    exponent = -math.log(10000) * torch.arange(half, dtype=torch.float32) / (half - freq_shift)
    emb = t.float()[:, None] * torch.exp(exponent)[None, :]
    emb = torch.cat([torch.sin(emb), torch.cos(emb)], dim=-1)
    if flip_sin_to_cos:
        emb = torch.cat([emb[:, half:], emb[:, :half]], dim=-1)
    return emb.half()


# ---------------------------------------------------------------------------------------
# sampler ops on the reference's "b c t h w" latents: torch op sequences (one rounding per op in the tensor dtype, which
# is what the kernels replay)
# ---------------------------------------------------------------------------------------
def cfg_combine(pred2, guidance_scale):
    u, t = pred2.chunk(2)
    return u + guidance_scale * (t - u)


def window_blend(dst, src, t0, covered_mask):
    for k in range(src.shape[2]):
        if (covered_mask >> k) & 1:
            dst[:, :, t0 + k] = dst[:, :, t0 + k] * 0.5 + src[:, :, k] * 0.5
        else:
            dst[:, :, t0 + k] = src[:, :, k]
    return dst


def ddim_step_v0(model_output, sample, pred_type, sqrt_alpha, sqrt_beta, clip, clip_range):
    if pred_type == 0:
        r = (sample - sqrt_beta * model_output) * (1.0 / sqrt_alpha)
    elif pred_type == 1:
        r = model_output.clone()
    else:
        r = sqrt_alpha * sample - sqrt_beta * model_output
    return r.clamp(-clip_range, clip_range) if clip else r


def ddim_step_vt(x0, model_output, sample, pred_type, sqrt_alpha, sqrt_beta, sqrt_alpha_prev, dir_coef, clip, clip_range,
                 std_dev=0.0, noise=None):
    if pred_type == 0:
        eps = model_output
    elif pred_type == 1:
        eps = (sample - sqrt_alpha * x0) * (1.0 / sqrt_beta)
    else:
        eps = sqrt_alpha * model_output + sqrt_beta * sample
    if clip:
        x0 = x0.clamp(-clip_range, clip_range)
    r = sqrt_alpha_prev * x0 + dir_coef * eps
    if noise is not None:
        r = r + std_dev * noise
    return r


def add_noise(x, noise, sqrt_alpha, sqrt_one_minus_alpha):
    return sqrt_alpha * x + sqrt_one_minus_alpha * noise


def propagate_step(feat_prop, feat_cur, flow_prop, flow_check, out, *, nearest, fuse, fuse_scale, alpha1, alpha2,
                   half_grid_sample):
    """one recurrence step of Propagation.forward (propagation_module.py:234-254) on (C|2, H, W) planes of one frame"""
    from oracle import uav_oracle as O
    fp, fc = flow_prop[None].float(), flow_check[None].float()
    mask = O.fb_consistency(fp, fc, alpha1, alpha2)
    warped = O.flow_warp(feat_prop[None].float(), fp.permute(0, 2, 3, 1), "nearest" if nearest else "bilinear")
    cur = feat_cur[None].float()
    if fuse:
        warped = warped * fuse_scale + cur * (1 - fuse_scale)
    out.copy_((mask * warped + (1 - mask) * cur)[0])
    return out


# ---------------------------------------------------------------------------------------
# post-decode colour fix + packing (csrc/postprocess.cu): planar fp32 "t c h w" frames
# ---------------------------------------------------------------------------------------
def bicubic_upsample(x, scale=4):
    return F.interpolate(x.float(), scale_factor=scale, mode="bicubic")


def plane_stats(x, eps=1e-5):
    x = x.float()
    t, c = x.shape[:2]
    v = x.reshape(t, c, -1)
    return v.mean(-1).reshape(t, c, 1, 1), (v.var(-1) + eps).sqrt().reshape(t, c, 1, 1)


def adain_apply(content, c_mean, c_std, s_mean, s_std):
    return (content.float() - c_mean) / c_std * s_std + s_mean


def wavelet_level(image, radius, *, low=None, high=None, high_first=False, add=None):
    from oracle import color_oracle as co
    blur = co.wavelet_blur(image, radius)
    if high is not None:
        d = image - blur
        high.copy_(d if high_first else high + d)
    if low is not None:
        low.copy_(blur if add is None else add + blur)


def pack_video_uint8(frames):
    v = (frames.float() / 2 + 0.5).clamp(0, 1) * 255
    return v.permute(0, 2, 3, 1).contiguous().to(torch.int32).to(torch.uint8)


def conv_out_fused(x, gamma, beta, groups, eps, w, bias, cout, out_dtype, cfg_step=None):
    """stand-in of ops.conv_out_fused: GroupNorm + SiLU (fp32, no rounding of the normalised tensor: the kernel applies it on
    the way into shared memory, rounded to fp16 there), 3x3 conv, planar output; optional guidance + step_v0 epilogue"""
    B, T, H, W, C = x.shape
    y = group_norm(x, gamma, beta, groups, eps, silu=True, n_outer=B)
    o = conv2d(y, w, bias, out_dtype=torch.float32)[..., :cout]
    out = o.permute(0, 4, 1, 2, 3).contiguous()
    if cfg_step is None:
        return out.to(out_dtype)
    npred = cfg_combine(out.half(), cfg_step["guidance_scale"])
    x0 = ddim_step_v0(npred, cfg_step["sample"], cfg_step["pred_type"], cfg_step["sqrt_alpha"], cfg_step["sqrt_beta"],
                      cfg_step["clip"], cfg_step["clip_range"])
    return npred, x0
