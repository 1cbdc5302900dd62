// postprocess.cu — the step right after the decode (SURVEY.md §8f rank 4): bicubic x4 of the low-resolution
// frames, AdaIN / wavelet colour fix against them, and the uint8 THWC packing of the result for the mp4 and the PNG
// frames (inference_upscale_a_video.py:323-357, models_video/color_correction.py:45-118); and the frame ingest before
// sampling (uint8 frames -> normalised, area-resized fp32 clip, inference_upscale_a_video.py:180-188).
//
// All tensors are the reference's own planar fp32 "t c h w" frames.  Every kernel is a single streaming pass
// (HBM-bound: the 4x frames are the largest tensors of the whole job, 283 MB per 8-frame 1280x2304 clip):
//   * plane statistics are deterministic (per-block fp64 partials, fixed-order finalize, no atomics);
//   * the arithmetic replays the reference's op order with one rounding per torch op (`__fmul_rn` & co. keep nvcc
//     from contracting into FMAs), so AdaIN / packing are bit-identical given bit-identical statistics, and the
//     wavelet levels accumulate `high += image - low` level by level exactly as color_correction.py:95-103 does
//     (not the telescoped image_0 - low_5, which rounds differently).
#include "uav_common.cuh"

namespace uav {

// ---------------------------------------------------------------------------------------
// bicubic upsampling, align_corners=False, A=-0.75, border-clamped taps
// (F.interpolate(vframes, scale_factor=4, mode='bicubic'), inference_upscale_a_video.py:327)
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ float cubic1(float x, float A) { return ((A + 2.f) * x - (A + 3.f)) * x * x + 1.f; }
__device__ __forceinline__ float cubic2(float x, float A) { return ((A * x - 5.f * A) * x + 8.f * A) * x - 4.f * A; }
__device__ __forceinline__ void cubic_coeffs(float t, float (&c)[4]) {
  const float A = -0.75f;
  c[0] = cubic2(t + 1.f, A);
  c[1] = cubic1(t, A);
  const float u = 1.f - t;
  c[2] = cubic1(u, A);
  c[3] = cubic2(u + 1.f, A);
}

__global__ void bicubic_kernel(const float* __restrict__ in, int64_t planes, int h, int w, int oh, int ow,
                               float scale_h, float scale_w, float* __restrict__ out) {
  const int64_t total = planes * oh * ow;
  UAV_GRID_STRIDE(i, total) {
    const int ox = static_cast<int>(i % ow);
    const int oy = static_cast<int>((i / ow) % oh);
    const int64_t pl = i / (static_cast<int64_t>(ow) * oh);
    const float rx = scale_w * (ox + 0.5f) - 0.5f, ry = scale_h * (oy + 0.5f) - 0.5f;
    const float fx = floorf(rx), fy = floorf(ry);
    const int ix = static_cast<int>(fx), iy = static_cast<int>(fy);
    float cx[4], cy[4];
    cubic_coeffs(rx - fx, cx);
    cubic_coeffs(ry - fy, cy);
    const float* src = in + pl * h * w;
    float rows[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int yy = min(max(iy - 1 + k, 0), h - 1);
      const float* r = src + static_cast<int64_t>(yy) * w;
      const float x0 = __ldg(r + min(max(ix - 1, 0), w - 1)), x1 = __ldg(r + min(max(ix, 0), w - 1)),
                  x2 = __ldg(r + min(max(ix + 1, 0), w - 1)), x3 = __ldg(r + min(max(ix + 2, 0), w - 1));
      rows[k] = x0 * cx[0] + x1 * cx[1] + x2 * cx[2] + x3 * cx[3];
    }
    out[i] = rows[0] * cy[0] + rows[1] * cy[1] + rows[2] * cy[2] + rows[3] * cy[3];
  }
}

// ---------------------------------------------------------------------------------------
// per-plane mean / sqrt(unbiased var + eps)   (calc_mean_std, color_correction.py:45-58)
// ---------------------------------------------------------------------------------------
constexpr int PS_THREADS = 256;
constexpr int PS_BLOCKS_PER_PLANE = 64;

__global__ void plane_stats_partial_kernel(const float* __restrict__ x, int64_t hw, double2* __restrict__ partial) {
  const int64_t pl = blockIdx.y;
  const float* src = x + pl * hw;
  double s = 0.0, ss = 0.0;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * PS_THREADS + threadIdx.x; i < hw;
       i += static_cast<int64_t>(PS_BLOCKS_PER_PLANE) * PS_THREADS) {
    const double v = static_cast<double>(__ldg(src + i));
    s += v;
    ss += v * v;
  }
  __shared__ double sh_s[PS_THREADS], sh_ss[PS_THREADS];
  sh_s[threadIdx.x] = s;
  sh_ss[threadIdx.x] = ss;
  __syncthreads();
  for (int off = PS_THREADS / 2; off > 0; off >>= 1) {  // fixed tree: deterministic
    if (threadIdx.x < off) {
      sh_s[threadIdx.x] += sh_s[threadIdx.x + off];
      sh_ss[threadIdx.x] += sh_ss[threadIdx.x + off];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) partial[pl * PS_BLOCKS_PER_PLANE + blockIdx.x] = make_double2(sh_s[0], sh_ss[0]);
}

__global__ void plane_stats_finalize_kernel(const double2* __restrict__ partial, int64_t planes, int64_t hw, float eps,
                                            float* __restrict__ mean, float* __restrict__ stdv) {
  const int64_t pl = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (pl >= planes) return;
  double s = 0.0, ss = 0.0;
  for (int b = 0; b < PS_BLOCKS_PER_PLANE; ++b) {
    const double2 v = partial[pl * PS_BLOCKS_PER_PLANE + b];
    s += v.x;
    ss += v.y;
  }
  const double n = static_cast<double>(hw);
  const double m = s / n;
  double var = (ss - s * m) / (n - 1.0);  // unbiased, as Tensor.var() defaults to
  if (var < 0.0) var = 0.0;
  // feat_var = var + eps (fp32 tensor op), feat_std = sqrt(feat_var)
  const float var_f = __fadd_rn(static_cast<float>(var), eps);
  mean[pl] = static_cast<float>(m);
  stdv[pl] = __fsqrt_rn(var_f);
}

// normalized = (content - c_mean) / c_std ; out = normalized * s_std + s_mean   (color_correction.py:69-73)
__global__ void adain_apply_kernel(const float* __restrict__ content, int64_t planes, int64_t hw,
                                   const float* __restrict__ c_mean, const float* __restrict__ c_std,
                                   const float* __restrict__ s_mean, const float* __restrict__ s_std,
                                   float* __restrict__ out) {
  const int64_t total = planes * hw;
  UAV_GRID_STRIDE(i, total) {
    const int64_t pl = i / hw;
    const float n = __fdiv_rn(__fsub_rn(content[i], c_mean[pl]), c_std[pl]);
    out[i] = __fadd_rn(__fmul_rn(n, s_std[pl]), s_mean[pl]);
  }
}

// ---------------------------------------------------------------------------------------
// one level of the a-trous wavelet decomposition (color_correction.py:75-103):
//   low = depthwise 3x3 [1 2 1; 2 4 2; 1 2 1]/16, dilation = radius, replicate padding
//   high (+)= image - low                (content chain)
//   out  = low + add                     (last level of the style chain: content_high + style_low)
// ---------------------------------------------------------------------------------------
__global__ void wavelet_level_kernel(const float* __restrict__ img, int64_t planes, int H, int W, int radius,
                                     float* __restrict__ low, float* __restrict__ high, int high_first,
                                     const float* __restrict__ add) {
  const int64_t hw = static_cast<int64_t>(H) * W;
  const int64_t total = planes * hw;
  UAV_GRID_STRIDE(i, total) {
    const int x = static_cast<int>(i % W);
    const int y = static_cast<int>((i / W) % H);
    const float* src = img + (i / hw) * hw;
    const int xm = max(x - radius, 0), xp = min(x + radius, W - 1);
    const int ym = max(y - radius, 0), yp = min(y + radius, H - 1);
    const float* r0 = src + static_cast<int64_t>(ym) * W;
    const float* r1 = src + static_cast<int64_t>(y) * W;
    const float* r2 = src + static_cast<int64_t>(yp) * W;
    const float c = __ldg(r1 + x);
    // row-major accumulation from zero; the weights are powers of two, so every product is exact
    float acc = 0.0625f * __ldg(r0 + xm);
    acc = __fadd_rn(acc, 0.125f * __ldg(r0 + x));
    acc = __fadd_rn(acc, 0.0625f * __ldg(r0 + xp));
    acc = __fadd_rn(acc, 0.125f * __ldg(r1 + xm));
    acc = __fadd_rn(acc, 0.25f * c);
    acc = __fadd_rn(acc, 0.125f * __ldg(r1 + xp));
    acc = __fadd_rn(acc, 0.0625f * __ldg(r2 + xm));
    acc = __fadd_rn(acc, 0.125f * __ldg(r2 + x));
    acc = __fadd_rn(acc, 0.0625f * __ldg(r2 + xp));
    if (high != nullptr) {
      const float d = __fsub_rn(c, acc);
      high[i] = high_first ? d : __fadd_rn(high[i], d);
    }
    if (add != nullptr) acc = __fadd_rn(add[i], acc);
    if (low != nullptr) low[i] = acc;
  }
}

// ---------------------------------------------------------------------------------------
// "t c h w" fp32 -> "t h w c" uint8 by truncation, with one of two roundings:
//   video (inference…:354-356):  (x / 2 + 0.5).clamp(0, 1) * 255, then numpy astype
//   PNG   (torchvision save_image(normalize=True, value_range=(-1, 1)), inference…:350):
//         clamp(-1, 1), (x - (-1)) / 2, * 255, + 0.5, clamp(0, 255), then Tensor.to(uint8)
// ---------------------------------------------------------------------------------------
template <bool PNG>
__global__ void pack_uint8_kernel(const float* __restrict__ x, int64_t T, int C, int64_t hw, uint8_t* __restrict__ out) {
  const int64_t total = T * hw;
  UAV_GRID_STRIDE(i, total) {
    const int64_t t = i / hw, px = i % hw;
    const float* src = x + t * C * hw + px;
    uint8_t* dst = out + i * C;
    for (int c = 0; c < C; ++c) {
      float v;
      if (PNG) {
        v = fminf(fmaxf(src[c * hw], -1.f), 1.f);
        v = __fmul_rn(__fadd_rn(v, 1.f), 0.5f);  // the halving is exact, as is the reference's division by 2
        v = __fadd_rn(__fmul_rn(v, 255.f), 0.5f);
        v = fminf(fmaxf(v, 0.f), 255.f);
      } else {
        v = __fadd_rn(__fmul_rn(src[c * hw], 0.5f), 0.5f);  // x / 2 is exact either way
        v = fminf(fmaxf(v, 0.f), 1.f);
        v = __fmul_rn(v, 255.f);
      }
      dst[c] = static_cast<uint8_t>(static_cast<int>(v));  // NaN -> 0 (numpy gives an unspecified value)
    }
  }
}

// ---------------------------------------------------------------------------------------
// frame ingest (inference…:180-188): uint8 "t h w c" BGR frames (OpenCV's decode order) -> planar fp32 RGB "c t h w".
//   * normalisation (v / 255. - 0.5) * 2 with the three roundings of the reference's CPU ops (an IEEE division, not
//     the reciprocal multiply torch uses for a scalar divisor on the GPU);
//   * area resize to (h_out, w_out) in the same pass, as ATen's adaptive_avg_pool2d CUDA kernels: fp32 sum over the
//     window in (row, column) order from 0, then, for NCHW frames, two divisions sum / kh / kw, and for channels-last
//     frames (NHWC) one multiply by the fp32 reciprocal 1 / (kh * kw).  The two differ once kh * kw is not a power of
//     two, i.e. for overlapping windows (and both differ from the single divide of the 3-D kernel behind
//     uav_flow_resize_area).  A 1 x 1 window (no resize) returns the normalised value unchanged.
// One thread per output pixel reads the 3 bytes of each input pixel of its window.
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ float normalize_u8(uint8_t u) {
  return __fmul_rn(__fsub_rn(__fdiv_rn(static_cast<float>(u), 255.f), 0.5f), 2.f);
}

template <bool NHWC>
__global__ void unpack_uint8_kernel(const uint8_t* __restrict__ in, int64_t T, int64_t H, int64_t W, int64_t h_out,
                                    int64_t w_out, float* __restrict__ out) {
  const int64_t hw_out = h_out * w_out;
  const int64_t total = T * hw_out;
  UAV_GRID_STRIDE(i, total) {
    const int64_t ox = i % w_out, oy = (i / w_out) % h_out, t = i / hw_out;
    const int64_t y0 = area_start(oy, h_out, H), y1 = area_end(oy, h_out, H);
    const int64_t x0 = area_start(ox, w_out, W), x1 = area_end(ox, w_out, W);
    float sum[3] = {0.f, 0.f, 0.f};
    for (int64_t y = y0; y < y1; ++y) {
      const uint8_t* row = in + (t * H + y) * W * 3;
      for (int64_t x = x0; x < x1; ++x) {
#pragma unroll
        for (int c = 0; c < 3; ++c) sum[c] = __fadd_rn(sum[c], normalize_u8(__ldg(row + x * 3 + c)));
      }
    }
    const float kh = static_cast<float>(y1 - y0), kw = static_cast<float>(x1 - x0);
    const float factor = __fdiv_rn(1.f, static_cast<float>((y1 - y0) * (x1 - x0)));
#pragma unroll
    for (int c = 0; c < 3; ++c)  // BGR -> RGB
      out[(2 - c) * total + i] = NHWC ? __fmul_rn(sum[c], factor) : __fdiv_rn(__fdiv_rn(sum[c], kh), kw);
  }
}

}  // namespace uav

using namespace uav;

extern "C" {

uav_status_t uav_bicubic_upsample(const float* in, int64_t planes, int64_t h, int64_t w, int scale, float* out,
                                  uav_stream_t stream) {
  UAV_REQUIRE(in && out && planes > 0 && h > 0 && w > 0 && scale >= 1 && scale <= 8, "uav_bicubic_upsample: bad argument");
  UAV_REQUIRE(h * scale < (1 << 30) && w * scale < (1 << 30), "uav_bicubic_upsample: frame too large");
  const int oh = static_cast<int>(h * scale), ow = static_cast<int>(w * scale);
  const int64_t total = planes * oh * ow;
  const float s = 1.0f / static_cast<float>(scale);  // scale_factor given -> ATen uses 1 / scale_factor
  bicubic_kernel<<<stream_grid(total, 256, 8), 256, 0, (cudaStream_t)stream>>>(in, planes, (int)h, (int)w, oh, ow, s, s, out);
  UAV_LAUNCHED();
  return UAV_OK;
}

size_t uav_plane_stats_workspace_bytes(int64_t planes) {
  return planes > 0 ? static_cast<size_t>(planes) * PS_BLOCKS_PER_PLANE * sizeof(double2) : 0;
}

uav_status_t uav_plane_stats(const float* x, int64_t planes, int64_t hw, float eps, void* workspace, float* mean,
                             float* stdv, uav_stream_t stream) {
  UAV_REQUIRE(x && workspace && mean && stdv && planes > 0 && hw > 1, "uav_plane_stats: bad argument");
  UAV_REQUIRE(planes <= 65535, "uav_plane_stats: more than 65535 planes");
  UAV_REQUIRE_ALIGNED16("uav_plane_stats", workspace);
  double2* partial = reinterpret_cast<double2*>(workspace);
  plane_stats_partial_kernel<<<dim3(PS_BLOCKS_PER_PLANE, (unsigned)planes), PS_THREADS, 0, (cudaStream_t)stream>>>(
      x, hw, partial);
  UAV_LAUNCHED();
  plane_stats_finalize_kernel<<<(unsigned)((planes + 63) / 64), 64, 0, (cudaStream_t)stream>>>(partial, planes, hw, eps,
                                                                                               mean, stdv);
  UAV_LAUNCHED();
  return UAV_OK;
}

uav_status_t uav_adain_apply(const float* content, int64_t planes, int64_t hw, const float* c_mean, const float* c_std,
                             const float* s_mean, const float* s_std, float* out, uav_stream_t stream) {
  UAV_REQUIRE(content && c_mean && c_std && s_mean && s_std && out && planes > 0 && hw > 0, "uav_adain_apply: bad argument");
  adain_apply_kernel<<<stream_grid(planes * hw, 256, 8), 256, 0, (cudaStream_t)stream>>>(content, planes, hw, c_mean, c_std,
                                                                                          s_mean, s_std, out);
  UAV_LAUNCHED();
  return UAV_OK;
}

uav_status_t uav_wavelet_level(const float* image, int64_t planes, int64_t H, int64_t W, int radius, float* low,
                               float* high, int high_first, const float* add, uav_stream_t stream) {
  UAV_REQUIRE(image && planes > 0 && H > 0 && W > 0 && radius >= 1, "uav_wavelet_level: bad argument");
  UAV_REQUIRE(H < (1 << 30) && W < (1 << 30), "uav_wavelet_level: frame too large");
  UAV_REQUIRE(low != nullptr || high != nullptr, "uav_wavelet_level: nothing to write");
  UAV_REQUIRE(low != image && high != image, "uav_wavelet_level: outputs must not alias the input (neighbour reads)");
  wavelet_level_kernel<<<stream_grid(planes * H * W, 256, 8), 256, 0, (cudaStream_t)stream>>>(image, planes, (int)H, (int)W,
                                                                                              radius, low, high, high_first, add);
  UAV_LAUNCHED();
  return UAV_OK;
}

uav_status_t uav_pack_video_uint8(const float* frames, int64_t T, int64_t C, int64_t H, int64_t W, uint8_t* out,
                                  uav_stream_t stream) {
  UAV_REQUIRE(frames && out && T > 0 && C > 0 && C <= 4 && H > 0 && W > 0, "uav_pack_video_uint8: bad argument");
  pack_uint8_kernel<false><<<stream_grid(T * H * W, 256, 8), 256, 0, (cudaStream_t)stream>>>(frames, T, (int)C, H * W, out);
  UAV_LAUNCHED();
  return UAV_OK;
}

uav_status_t uav_pack_frames_png(const float* frames, int64_t T, int64_t C, int64_t H, int64_t W, uint8_t* out,
                                 uav_stream_t stream) {
  UAV_REQUIRE(frames && out && T > 0 && C > 0 && C <= 4 && H > 0 && W > 0, "uav_pack_frames_png: bad argument");
  pack_uint8_kernel<true><<<stream_grid(T * H * W, 256, 8), 256, 0, (cudaStream_t)stream>>>(frames, T, (int)C, H * W, out);
  UAV_LAUNCHED();
  return UAV_OK;
}

uav_status_t uav_unpack_video_uint8(const uint8_t* frames, int64_t T, int64_t H, int64_t W, int64_t h_out, int64_t w_out,
                                    int nhwc, float* out, uav_stream_t stream) {
  UAV_REQUIRE(frames && out && T > 0 && H > 0 && W > 0, "uav_unpack_video_uint8: bad argument");
  UAV_REQUIRE(h_out > 0 && h_out <= H && w_out > 0 && w_out <= W,
              "uav_unpack_video_uint8: output %lldx%lld must be between 1x1 and the input's %lldx%lld (downsampling only)",
              (long long)h_out, (long long)w_out, (long long)H, (long long)W);
  // torch reduces to a 1 x 1 output with a mean, whose summation order this kernel does not reproduce
  UAV_REQUIRE(h_out > 1 || w_out > 1 || (H == 1 && W == 1), "uav_unpack_video_uint8: a 1x1 output is not supported");
  UAV_REQUIRE(H < (1 << 30) && W < (1 << 30), "uav_unpack_video_uint8: frame too large");
  const unsigned grid = stream_grid(T * h_out * w_out, 256, 8);
  if (nhwc)
    unpack_uint8_kernel<true><<<grid, 256, 0, (cudaStream_t)stream>>>(frames, T, H, W, h_out, w_out, out);
  else
    unpack_uint8_kernel<false><<<grid, 256, 0, (cudaStream_t)stream>>>(frames, T, H, W, h_out, w_out, out);
  UAV_LAUNCHED();
  return UAV_OK;
}

}  // extern "C"
