// elementwise.cu — HBM-bound data-movement kernels around the implicit-GEMM core:
// channel-slice copies (skip-connection concat, unet_blocks.py:573,645), nearest upsampling
// (Upsample3D, resnet.py:143-146), the API-edge layout converters between the reference's
// "b c t h w" tensors and the channels-last working layout, SiLU on the time embedding, and the
// timestep sinusoid (diffusers Timesteps, unet_video.py:173,472).
#include "uav_common.cuh"

namespace uav {

// dst[p][0:C] = src[p][0:C]  (C % 8 == 0, 16-byte aligned)
__global__ void __launch_bounds__(256)
    copy_channels_kernel(const __half* __restrict__ src, int64_t ld_src, __half* __restrict__ dst,
                         int64_t ld_dst, int octs, int64_t pixels) {
  const int64_t total = pixels * octs;
  UAV_GRID_STRIDE(i, total) {
    const int64_t p = i / octs;
    const int o = static_cast<int>(i - p * octs);
    stg16(dst + p * ld_dst + o * 8, ldg16(src + p * ld_src + o * 8));
  }
}

// nearest-neighbour resize of NB images (channels-last): src index = floor(dst * in / out),
// which for out = 2*in is dst >> 1 (F.interpolate(mode="nearest"))
__global__ void __launch_bounds__(256)
    upsample_nearest_kernel(const __half* __restrict__ src, int64_t ld_src, int Hi, int Wi,
                            __half* __restrict__ dst, int64_t ld_dst, int Ho, int Wo, int octs,
                            int64_t NB) {
  const int64_t total = NB * Ho * Wo * octs;
  const float sy = static_cast<float>(Hi) / Ho, sx = static_cast<float>(Wi) / Wo;
  UAV_GRID_STRIDE(i, total) {
    const int o = static_cast<int>(i % octs);
    int64_t r = i / octs;
    const int x = static_cast<int>(r % Wo);
    r /= Wo;
    const int y = static_cast<int>(r % Ho);
    const int64_t n = r / Ho;
    int ys = (Ho == 2 * Hi) ? (y >> 1) : min(static_cast<int>(floorf(y * sy)), Hi - 1);
    int xs = (Wo == 2 * Wi) ? (x >> 1) : min(static_cast<int>(floorf(x * sx)), Wi - 1);
    stg16(dst + ((n * Ho + y) * Wo + x) * ld_dst + o * 8,
          ldg16(src + ((n * Hi + ys) * Wi + xs) * ld_src + o * 8));
  }
}

// (B, C, T*H*W) planar [fp16|fp32] -> channels-last fp16 [B][THW][ld_dst] at channel offset c_off
template <typename T>
__global__ void __launch_bounds__(256)
    planar_to_cl_kernel(const T* __restrict__ src, int C, int64_t thw, int64_t B,
                        __half* __restrict__ dst, int64_t ld_dst, int c_off, float scale) {
  const int64_t total = B * thw;
  UAV_GRID_STRIDE(i, total) {
    const int64_t b = i / thw, p = i - b * thw;
    for (int c = 0; c < C; ++c)
      dst[i * ld_dst + c_off + c] =
          __float2half_rn(static_cast<float>(src[(b * C + c) * thw + p]) * scale);
  }
}

// channels-last [fp16|fp32] [B][THW][ld_src] (first C channels) -> planar (B, C, THW) [fp16|fp32]
template <typename TI, typename TO>
__global__ void __launch_bounds__(256)
    cl_to_planar_kernel(const TI* __restrict__ src, int64_t ld_src, int C, int64_t thw, int64_t B,
                        TO* __restrict__ dst, int clamp) {
  const int64_t total = B * thw;
  UAV_GRID_STRIDE(i, total) {
    const int64_t b = i / thw, p = i - b * thw;
    for (int c = 0; c < C; ++c) {
      float v = static_cast<float>(src[i * ld_src + c]);
      if (clamp) v = fminf(fmaxf(v, -1.f), 1.f);
      dst[(b * C + c) * thw + p] = static_cast<TO>(v);
    }
  }
}

__global__ void __launch_bounds__(256)
    silu_kernel(const __half* __restrict__ x, __half* __restrict__ y, int64_t n) {
  UAV_GRID_STRIDE(i, n)
    y[i] = __float2half_rn(silu_f(__half2float(x[i])));
}

// out[b][0:half] = cos(t_b * f_i), out[b][half:2*half] = sin(t_b * f_i), f_i = exp(-ln(1e4) i /
// (half - shift)) — diffusers get_timestep_embedding with flip_sin_to_cos=True (fp32 math).
__global__ void timestep_embedding_kernel(const float* __restrict__ t, int B, int dim,
                                          int flip_sin_to_cos, float freq_shift,
                                          __half* __restrict__ out) {
  const int half = dim / 2;
  UAV_GRID_STRIDE(i, B * half) {
    const int b = static_cast<int>(i / half), j = static_cast<int>(i % half);
    const float f = expf(-logf(10000.f) * j / (half - freq_shift));
    const float a = t[b] * f;
    const float s = sinf(a), c = cosf(a);
    out[b * dim + j] = __float2half_rn(flip_sin_to_cos ? c : s);
    out[b * dim + half + j] = __float2half_rn(flip_sin_to_cos ? s : c);
  }
}


// Fuse_sft_block tail (resnet.py:77-78): out = dec + w * (dec * scale + shift), 8 halfs per thread
__global__ void __launch_bounds__(256)
    sft_fuse_kernel(const __half* __restrict__ dec, const __half* __restrict__ scale,
                    const __half* __restrict__ shift, float w, float out_scale, __half* __restrict__ out, int64_t n8) {
  UAV_GRID_STRIDE(i, n8) {
    const uint4 d = ldg16(dec + i * 8), sc = ldg16(scale + i * 8), sh = ldg16(shift + i * 8);
    const __half2* dh = reinterpret_cast<const __half2*>(&d);
    const __half2* ch = reinterpret_cast<const __half2*>(&sc);
    const __half2* hh = reinterpret_cast<const __half2*>(&sh);
    uint4 o;
    uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 a = __half22float2(dh[j]), b = __half22float2(ch[j]), c = __half22float2(hh[j]);
      ow[j] = pack_half2_sat((a.x + w * (a.x * b.x + c.x)) * out_scale, (a.y + w * (a.y * b.y + c.y)) * out_scale);
    }
    stg16(out + i * 8, o);
  }
}

}  // namespace uav

using namespace uav;

extern "C" {

uav_status_t uav_copy_channels(const void* src, int64_t ld_src, void* dst, int64_t ld_dst,
                               int64_t C, int64_t pixels, uav_stream_t stream) {
  UAV_REQUIRE(src && dst && C > 0 && C % 8 == 0 && ld_src % 8 == 0 && ld_dst % 8 == 0 &&
                  ld_src >= C && ld_dst >= C,
              "uav_copy_channels: bad shape / alignment (C=%lld)", (long long)C);
  UAV_REQUIRE(pixels >= 0, "uav_copy_channels: pixels must be >= 0");
  UAV_REQUIRE_ALIGNED16("uav_copy_channels", src);
  UAV_REQUIRE_ALIGNED16("uav_copy_channels", dst);
  if (pixels == 0) return UAV_OK;
  copy_channels_kernel<<<stream_grid(pixels * (C / 8), 256 * 4, 16), 256, 0, (cudaStream_t)stream>>>(
      (const __half*)src, ld_src, (__half*)dst, ld_dst, (int)(C / 8), pixels);
  UAV_LAUNCHED();
  return UAV_OK;
}

uav_status_t uav_upsample_nearest(const void* src, int64_t ld_src, int64_t NB, int64_t Hi,
                                  int64_t Wi, int64_t C, void* dst, int64_t ld_dst, int64_t Ho,
                                  int64_t Wo, uav_stream_t stream) {
  UAV_REQUIRE(src && dst && C > 0 && C % 8 == 0 && ld_src % 8 == 0 && ld_dst % 8 == 0,
              "uav_upsample_nearest: bad shape / alignment");
  UAV_REQUIRE(ld_src >= C && ld_dst >= C, "uav_upsample_nearest: ld_src and ld_dst must be >= C");
  UAV_REQUIRE(NB > 0 && Hi > 0 && Wi > 0 && Ho > 0 && Wo > 0, "uav_upsample_nearest: bad shape");
  UAV_REQUIRE(Hi < (1 << 30) && Wi < (1 << 30) && Ho < (1 << 30) && Wo < (1 << 30),
              "uav_upsample_nearest: Hi, Wi, Ho and Wo must be < 2^30");
  UAV_REQUIRE_ALIGNED16("uav_upsample_nearest", src);
  UAV_REQUIRE_ALIGNED16("uav_upsample_nearest", dst);
  upsample_nearest_kernel<<<stream_grid(NB * Ho * Wo * (C / 8), 256 * 4, 16), 256, 0, (cudaStream_t)stream>>>(
      (const __half*)src, ld_src, (int)Hi, (int)Wi, (__half*)dst, ld_dst, (int)Ho, (int)Wo,
      (int)(C / 8), NB);
  UAV_LAUNCHED();
  return UAV_OK;
}

uav_status_t uav_planar_to_channels_last(const void* src, int src_dtype, int64_t B, int64_t C,
                                         int64_t thw, void* dst, int64_t ld_dst, int64_t c_off,
                                         float scale, uav_stream_t stream) {
  UAV_REQUIRE(src && dst && B > 0 && C > 0 && thw > 0 && c_off >= 0 && c_off + C <= ld_dst,
              "uav_planar_to_channels_last: bad shape");
  UAV_REQUIRE(src_dtype == UAV_F16 || src_dtype == UAV_F32, "uav_planar_to_channels_last: unsupported src_dtype %d",
              src_dtype);
  const unsigned g = stream_grid(B * thw, 256, 16);
  if (src_dtype == UAV_F16)
    planar_to_cl_kernel<__half><<<g, 256, 0, (cudaStream_t)stream>>>(
        (const __half*)src, (int)C, thw, B, (__half*)dst, ld_dst, (int)c_off, scale);
  else
    planar_to_cl_kernel<float><<<g, 256, 0, (cudaStream_t)stream>>>(
        (const float*)src, (int)C, thw, B, (__half*)dst, ld_dst, (int)c_off, scale);
  UAV_LAUNCHED();
  return UAV_OK;
}

uav_status_t uav_channels_last_to_planar(const void* src, int src_dtype, int64_t ld_src, int64_t B,
                                         int64_t C, int64_t thw, void* dst, int dst_dtype,
                                         int clamp, uav_stream_t stream) {
  UAV_REQUIRE(src && dst && B > 0 && C > 0 && thw > 0 && ld_src >= C,
              "uav_channels_last_to_planar: bad shape");
  const unsigned g = stream_grid(B * thw, 256, 16);
  cudaStream_t s = (cudaStream_t)stream;
  if (src_dtype == UAV_F16 && dst_dtype == UAV_F16)
    cl_to_planar_kernel<__half, __half><<<g, 256, 0, s>>>((const __half*)src, ld_src, (int)C, thw,
                                                          B, (__half*)dst, clamp);
  else if (src_dtype == UAV_F16 && dst_dtype == UAV_F32)
    cl_to_planar_kernel<__half, float><<<g, 256, 0, s>>>((const __half*)src, ld_src, (int)C, thw, B,
                                                         (float*)dst, clamp);
  else if (src_dtype == UAV_F32 && dst_dtype == UAV_F32)
    cl_to_planar_kernel<float, float><<<g, 256, 0, s>>>((const float*)src, ld_src, (int)C, thw, B,
                                                        (float*)dst, clamp);
  else {
    set_last_error("uav_channels_last_to_planar: unsupported dtype pair");
    return UAV_ERR_UNSUPPORTED;
  }
  UAV_LAUNCHED();
  return UAV_OK;
}

uav_status_t uav_silu(const void* x, void* y, int64_t n, uav_stream_t stream) {
  UAV_REQUIRE(x && y && n >= 0, "uav_silu: bad argument");
  if (n == 0) return UAV_OK;
  silu_kernel<<<stream_grid(n, 256, 16), 256, 0, (cudaStream_t)stream>>>((const __half*)x, (__half*)y, n);
  UAV_LAUNCHED();
  return UAV_OK;
}

uav_status_t uav_timestep_embedding(const float* t, int64_t B, int64_t dim, int flip_sin_to_cos,
                                    float freq_shift, void* out, uav_stream_t stream) {
  UAV_REQUIRE(t && out && B > 0 && dim > 0 && dim % 2 == 0, "uav_timestep_embedding: bad shape");
  timestep_embedding_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(t, (int)B, (int)dim,
                                                                flip_sin_to_cos, freq_shift,
                                                                (__half*)out);
  UAV_LAUNCHED();
  return UAV_OK;
}

uav_status_t uav_sft_fuse(const void* dec, const void* scale, const void* shift, float w, float out_scale, void* out,
                          int64_t n, uav_stream_t stream) {
  UAV_REQUIRE(dec && scale && shift && out && n >= 0 && n % 8 == 0, "uav_sft_fuse: bad argument");
  UAV_REQUIRE_ALIGNED16("uav_sft_fuse", dec);
  UAV_REQUIRE_ALIGNED16("uav_sft_fuse", scale);
  UAV_REQUIRE_ALIGNED16("uav_sft_fuse", shift);
  UAV_REQUIRE_ALIGNED16("uav_sft_fuse", out);
  if (n == 0) return UAV_OK;
  sft_fuse_kernel<<<stream_grid(n / 8, 256 * 4, 16), 256, 0, (cudaStream_t)stream>>>(
      (const __half*)dec, (const __half*)scale, (const __half*)shift, w, out_scale == 0.f ? 1.f : out_scale, (__half*)out, n / 8);
  UAV_LAUNCHED();
  return UAV_OK;
}

}  // extern "C"
