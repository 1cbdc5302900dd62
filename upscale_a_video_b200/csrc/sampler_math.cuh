// sampler_math.cuh — torch's per-op rounding of the sampler's elementwise math, and the two steps that both the sampler
// kernels (sampler.cu) and the fused conv_out epilogue (conv_io.cu) evaluate, so that the fused step is bit-identical
// to the separate kernels by construction.
//
// In fp16 the reference rounds after EVERY torch op (0-dim fp32 scalars x fp16 CUDA tensors -> fp16; SURVEY.md
// Appendix B): Num<true> is fp32 math + one round-to-half (`rh`) per op, Num<false> plain fp32.
#pragma once
#include "uav_common.cuh"

namespace uav {

template <bool HALF>
struct Num;
template <>
struct Num<true> {
  using T = __half;
  static __device__ __forceinline__ float ld(const __half* p, int64_t i) { return __half2float(p[i]); }
  static __device__ __forceinline__ void st(__half* p, int64_t i, float v) { p[i] = __float2half_rn(v); }
  static __device__ __forceinline__ float rh(float v) { return __half2float(__float2half_rn(v)); }
  static __device__ __forceinline__ float mul(float a, float b) { return rh(__fmul_rn(a, b)); }
  static __device__ __forceinline__ float add(float a, float b) { return rh(__fadd_rn(a, b)); }
  static __device__ __forceinline__ float sub(float a, float b) { return rh(__fsub_rn(a, b)); }
};
template <>
struct Num<false> {
  using T = float;
  static __device__ __forceinline__ float ld(const float* p, int64_t i) { return p[i]; }
  static __device__ __forceinline__ void st(float* p, int64_t i, float v) { p[i] = v; }
  static __device__ __forceinline__ float rh(float v) { return v; }
  // one torch op == one rounding: intrinsics keep nvcc from contracting a*b+c into an FMA
  static __device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
  static __device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
  static __device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
};

// noise_pred = uncond + g * (text - uncond)   (pipeline_upscale_a_video.py:644-645)
template <bool HALF>
__device__ __forceinline__ float cfg_combine(float uncond, float text, float g) {
  using N = Num<HALF>;
  return N::add(uncond, N::mul(g, N::sub(text, uncond)));
}

// x0 of DDIMScheduler.step_v0 (scheduling_ddim.py:383-433) from the model output m and the sample s.
// pred_type: 0 epsilon, 1 sample, 2 v
template <bool HALF>
__device__ __forceinline__ float ddim_x0(float m, float s, int pred_type, float sa, float sb, float inv_sa, int clip,
                                         float clip_range) {
  using N = Num<HALF>;
  float r;
  if (pred_type == 0) {
    // (sample - beta^0.5 * eps) / alpha^0.5 ; CUDA divides by a CPU scalar as mul-by-reciprocal
    r = N::mul(N::sub(s, N::mul(sb, m)), inv_sa);
  } else if (pred_type == 1) {
    r = m;
  } else {
    r = N::sub(N::mul(sa, s), N::mul(sb, m));
  }
  if (clip) r = fminf(fmaxf(r, -clip_range), clip_range);
  return r;
}

}  // namespace uav
