// sampler.cu — the per-step elementwise part of VideoUpscalePipeline.__call__
// (SURVEY.md §8a rows a15, a16, a17): classifier-free-guidance combine, window blend, the
// split DDIM step (step_v0 / step_vt), add_noise and flow-guided latent propagation with its
// area resize of the flows.
//
// These run on the reference's own "b c t h w" latents (4 channels).  In fp16 the reference
// rounds after EVERY torch op (0-dim fp32 scalars x fp16 CUDA tensors -> fp16; SURVEY.md
// Appendix B), so each kernel replays that exact op sequence with a round-to-half after each
// step (`rh`), in one launch instead of 3-10: results are bit-identical to the op-by-op
// torch sequence while reading/writing each tensor once.
#include "uav_common.cuh"

#include <atomic>

namespace uav {
extern std::atomic<uint64_t> g_launches;

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

#define UAV_GRID_STRIDE(i, n)                                                         \
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < (n); \
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)

// noise_pred = uncond + g * (text - uncond)   (pipeline_upscale_a_video.py:644-645)
template <bool HALF>
__global__ void cfg_kernel(const void* pred2_, void* out_, int64_t n, float g) {
  using N = Num<HALF>;
  const typename N::T* pred2 = reinterpret_cast<const typename N::T*>(pred2_);
  typename N::T* out = reinterpret_cast<typename N::T*>(out_);
  UAV_GRID_STRIDE(i, n) {
    const float u = N::ld(pred2, i), t = N::ld(pred2, n + i);
    const float d = N::sub(t, u);
    const float m = N::mul(g, d);
    N::st(out, i, N::add(u, m));
  }
}

// window blend (pipeline_upscale_a_video.py:630-634): per frame k of the window,
// dst[:, :, t0+k] = covered ? dst*0.5 + src*0.5 : src ; tensors are (outer=b*c, T, hw)
template <bool HALF>
__global__ void window_blend_kernel(void* dst_, int64_t T, const void* src_, int64_t Tw, int t0,
                                    uint32_t covered_mask, int64_t outer, int64_t hw) {
  using N = Num<HALF>;
  typename N::T* dst = reinterpret_cast<typename N::T*>(dst_);
  const typename N::T* src = reinterpret_cast<const typename N::T*>(src_);
  const int64_t n = outer * Tw * hw;
  UAV_GRID_STRIDE(i, n) {
    const int64_t p = i % hw;
    const int64_t k = (i / hw) % Tw;
    const int64_t o = i / (hw * Tw);
    const int64_t di = (o * T + t0 + k) * hw + p;
    const float s = N::ld(src, i);
    if ((covered_mask >> k) & 1u) {
      const float a = N::mul(N::ld(dst, di), 0.5f), b = N::mul(s, 0.5f);
      N::st(dst, di, N::add(a, b));
    } else {
      N::st(dst, di, s);
    }
  }
}

// DDIMScheduler.step_v0 (scheduling_ddim.py:383-433).  pred_type: 0 epsilon, 1 sample, 2 v
template <bool HALF>
__global__ void ddim_v0_kernel(const void* mo_, const void* x_, void* x0_, int64_t n, int pred_type,
                               float sa, float sb, float inv_sa, int clip, float clip_range) {
  using N = Num<HALF>;
  const typename N::T* mo = reinterpret_cast<const typename N::T*>(mo_);
  const typename N::T* x = reinterpret_cast<const typename N::T*>(x_);
  typename N::T* x0 = reinterpret_cast<typename N::T*>(x0_);
  UAV_GRID_STRIDE(i, n) {
    const float m = N::ld(mo, i), s = N::ld(x, i);
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
    N::st(x0, i, r);
  }
}

// DDIMScheduler.step_vt (scheduling_ddim.py:436-520)
template <bool HALF>
__global__ void ddim_vt_kernel(const void* x0_, const void* mo_, const void* x_, void* prev_,
                               int64_t n, int pred_type, float sa, float sb, float inv_sb,
                               float sa_prev, float c_dir, int clip, float clip_range, float std,
                               const void* noise_) {
  using N = Num<HALF>;
  const typename N::T* x0p = reinterpret_cast<const typename N::T*>(x0_);
  const typename N::T* mo = reinterpret_cast<const typename N::T*>(mo_);
  const typename N::T* x = reinterpret_cast<const typename N::T*>(x_);
  const typename N::T* noise = reinterpret_cast<const typename N::T*>(noise_);
  typename N::T* prev = reinterpret_cast<typename N::T*>(prev_);
  UAV_GRID_STRIDE(i, n) {
    float x0 = N::ld(x0p, i);
    const float m = N::ld(mo, i), s = N::ld(x, i);
    float eps;
    if (pred_type == 0) eps = m;
    else if (pred_type == 1) eps = N::mul(N::sub(s, N::mul(sa, x0)), inv_sb);
    else eps = N::add(N::mul(sa, m), N::mul(sb, s));
    if (clip) x0 = fminf(fmaxf(x0, -clip_range), clip_range);
    const float dir = N::mul(c_dir, eps);
    float r = N::add(N::mul(sa_prev, x0), dir);
    if (noise != nullptr) r = N::add(r, N::mul(std, N::ld(noise, i)));
    N::st(prev, i, r);
  }
}

// add_noise (scheduling_ddim.py:524-545): a, s are already rounded to the sample dtype
template <bool HALF>
__global__ void add_noise_kernel(const void* x_, const void* nz_, void* out_, int64_t n, float a,
                                 float s) {
  using N = Num<HALF>;
  const typename N::T* x = reinterpret_cast<const typename N::T*>(x_);
  const typename N::T* nz = reinterpret_cast<const typename N::T*>(nz_);
  typename N::T* out = reinterpret_cast<typename N::T*>(out_);
  UAV_GRID_STRIDE(i, n) {
    N::st(out, i, N::add(N::mul(a, N::ld(x, i)), N::mul(s, N::ld(nz, i))));
  }
}

// ---------------------------------------------------------------------------------------
// one recurrence step of Propagation.forward, learnable=False (propagation_module.py:234-254):
//   mask = fbConsistencyCheck(flow_prop, flow_check, alpha1, alpha2)      (bilinear warp)
//   warped = flow_warp(feat_prop, flow_prop, interpolation)
//   fuse:  warped = warped * fuse_scale + cur * (1 - fuse_scale)
//   out = mask * warped + (1 - mask) * cur
// feat_* are (C, H, W) planes of one frame (frame stride given), flows are (2, H, W).
// Grid sampling follows torch's CUDA grid_sampler for half inputs in opmath: fp32 coordinates
// and weights, one final rounding.
// ---------------------------------------------------------------------------------------
template <bool HALF>
struct GridSample {
  using N = Num<HALF>;
  // source index from a normalised coordinate, align_corners=True
  static __device__ __forceinline__ float unnorm(float coord, int size) {
    return __fmul_rn(__fadd_rn(coord, 1.f) * 0.5f, static_cast<float>(size - 1));
  }
  static __device__ __forceinline__ float bilinear(const typename N::T* plane, int H, int W,
                                                   float ix, float iy) {
    const int ix_nw = static_cast<int>(floorf(ix)), iy_nw = static_cast<int>(floorf(iy));
    const int ix_ne = ix_nw + 1, iy_ne = iy_nw, ix_sw = ix_nw, iy_sw = iy_nw + 1;
    const int ix_se = ix_nw + 1, iy_se = iy_nw + 1;
    const float nw = __fmul_rn(ix_se - ix, iy_se - iy);
    const float ne = __fmul_rn(ix - ix_sw, iy_sw - iy);
    const float sw = __fmul_rn(ix_ne - ix, iy - iy_ne);
    const float se = __fmul_rn(ix - ix_nw, iy - iy_nw);
    float acc = 0.f;
    auto in = [&](int y, int x) { return y >= 0 && y < H && x >= 0 && x < W; };
    // `out_acc += inp * w` in ATen's grid_sampler kernel: an FMA per corner
    auto accum = [&](float v, float w) { acc = __fmaf_rn(v, w, acc); };
    if (in(iy_nw, ix_nw)) accum(N::ld(plane, (int64_t)iy_nw * W + ix_nw), nw);
    if (in(iy_ne, ix_ne)) accum(N::ld(plane, (int64_t)iy_ne * W + ix_ne), ne);
    if (in(iy_sw, ix_sw)) accum(N::ld(plane, (int64_t)iy_sw * W + ix_sw), sw);
    if (in(iy_se, ix_se)) accum(N::ld(plane, (int64_t)iy_se * W + ix_se), se);
    return N::rh(acc);
  }
  static __device__ __forceinline__ float nearest(const typename N::T* plane, int H, int W,
                                                  float ix, float iy) {
    const int xn = static_cast<int>(nearbyintf(ix)), yn = static_cast<int>(nearbyintf(iy));
    if (yn >= 0 && yn < H && xn >= 0 && xn < W) return N::ld(plane, (int64_t)yn * W + xn);
    return 0.f;
  }
};

template <bool HALF>
__global__ void propagate_step_kernel(const void* feat_prop_, const void* feat_cur_,
                                      const void* flow_prop_, const void* flow_check_, void* out_,
                                      int C, int H, int W, int64_t cs_prop, int64_t cs_cur,
                                      int64_t cs_out, int64_t cs_fp, int64_t cs_fc, int nearest,
                                      int fuse, float fuse_scale, float alpha1, float alpha2,
                                      float inv_wm1, float inv_hm1) {
  using N = Num<HALF>;
  using T = typename N::T;
  using GS = GridSample<HALF>;
  const T* feat_prop = reinterpret_cast<const T*>(feat_prop_);
  const T* feat_cur = reinterpret_cast<const T*>(feat_cur_);
  const T* flow_prop = reinterpret_cast<const T*>(flow_prop_);
  const T* flow_check = reinterpret_cast<const T*>(flow_check_);
  T* out = reinterpret_cast<T*>(out_);
  const int64_t hw = static_cast<int64_t>(H) * W;
  UAV_GRID_STRIDE(i, hw) {
    const int y = static_cast<int>(i / W), x = static_cast<int>(i % W);
    const float fpx = N::ld(flow_prop, i), fpy = N::ld(flow_prop, cs_fp + i);
    // flow_warp(): vgrid = grid + flow ; 2.0 * v / max(size-1, 1) - 1.0  (each op rounds)
    const float gx = N::add(static_cast<float>(x), fpx), gy = N::add(static_cast<float>(y), fpy);
    const float vx = N::sub(N::mul(N::mul(2.0f, gx), inv_wm1), 1.0f);
    const float vy = N::sub(N::mul(N::mul(2.0f, gy), inv_hm1), 1.0f);
    const float ix = GS::unnorm(vx, W), iy = GS::unnorm(vy, H);
    // fbConsistencyCheck
    const float bwx = GS::bilinear(flow_check, H, W, ix, iy);
    const float bwy = GS::bilinear(flow_check + cs_fc, H, W, ix, iy);
    const float dx = N::add(fpx, bwx), dy = N::add(fpy, bwy);
    const float lsq_f = N::add(N::mul(fpx, fpx), N::mul(fpy, fpy));
    const float lsq_b = N::add(N::mul(bwx, bwx), N::mul(bwy, bwy));
    const float mag = N::add(lsq_f, lsq_b);
    const float thr = N::add(N::mul(alpha1, mag), alpha2);
    const float lsq_d = N::add(N::mul(dx, dx), N::mul(dy, dy));
    const float mask = (lsq_d < thr) ? 1.f : 0.f;
    for (int c = 0; c < C; ++c) {
      const T* plane = feat_prop + c * cs_prop;
      float w = nearest ? GS::nearest(plane, H, W, ix, iy) : GS::bilinear(plane, H, W, ix, iy);
      const float cur = N::ld(feat_cur, c * cs_cur + i);
      if (fuse) w = N::add(N::mul(w, fuse_scale), N::mul(cur, 1.f - fuse_scale));
      const float r = N::add(N::mul(mask, w), N::mul(N::sub(1.f, mask), cur));
      N::st(out, c * cs_out + i, r);
    }
  }
}

// ---------------------------------------------------------------------------------------
// flow resize of Propagation.forward (propagation_module.py:206-209):
//   F.interpolate(flows, (t_out, h_out, w_out), mode='area') * scale
// = adaptive_avg_pool3d: output (ot, oh, ow) averages the input window [floor(i*in/out),
// ceil((i+1)*in/out)) in each dimension.  As torch's CUDA kernel: fp32 sum in (t, h, w) order,
// one divide by the window size, rounded to the storage dtype; then `* scale` in fp32 opmath and
// rounded again.  in/out are (planes, t, h, w) contiguous.  Window bounds: area_start / area_end (uav_common.cuh).
// ---------------------------------------------------------------------------------------
template <bool HALF>
__global__ void flow_resize_area_kernel(const void* in_, void* out_, int64_t planes, int64_t t_in,
                                        int64_t h_in, int64_t w_in, int64_t t_out, int64_t h_out,
                                        int64_t w_out, float scale) {
  using N = Num<HALF>;
  const typename N::T* in = reinterpret_cast<const typename N::T*>(in_);
  typename N::T* out = reinterpret_cast<typename N::T*>(out_);
  const int64_t n = planes * t_out * h_out * w_out;
  UAV_GRID_STRIDE(i, n) {
    const int64_t ow = i % w_out, oh = (i / w_out) % h_out, ot = (i / (w_out * h_out)) % t_out;
    const int64_t pl = i / (w_out * h_out * t_out);
    const int64_t t0 = area_start(ot, t_out, t_in), t1 = area_end(ot, t_out, t_in);
    const int64_t y0 = area_start(oh, h_out, h_in), y1 = area_end(oh, h_out, h_in);
    const int64_t x0 = area_start(ow, w_out, w_in), x1 = area_end(ow, w_out, w_in);
    float sum = 0.f;
    for (int64_t t = t0; t < t1; ++t) {
      const int64_t base = (pl * t_in + t) * h_in;
      for (int64_t y = y0; y < y1; ++y)
        for (int64_t x = x0; x < x1; ++x) sum = __fadd_rn(sum, N::ld(in, (base + y) * w_in + x));
    }
    const float avg = N::rh(__fdiv_rn(sum, static_cast<float>((t1 - t0) * (y1 - y0) * (x1 - x0))));
    N::st(out, i, N::mul(avg, scale));
  }
}

static inline unsigned sgrid(int64_t n) {
  int64_t g = (n + 255) / 256;
  const int64_t cap = static_cast<int64_t>(num_sms()) * 16;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return static_cast<unsigned>(g);
}

}  // namespace uav

using namespace uav;

#define UAV_DISPATCH_DTYPE(dtype, KERNEL, grid, stream, ...)                                   \
  do {                                                                                         \
    if ((dtype) == UAV_F16) KERNEL<true><<<grid, 256, 0, (cudaStream_t)stream>>>(__VA_ARGS__); \
    else if ((dtype) == UAV_F32) KERNEL<false><<<grid, 256, 0, (cudaStream_t)stream>>>(__VA_ARGS__); \
    else {                                                                                     \
      set_last_error("unsupported dtype %d", (int)(dtype));                                    \
      return UAV_ERR_INVALID;                                                                  \
    }                                                                                          \
    UAV_CHECK_CUDA(cudaGetLastError());                                                        \
    g_launches.fetch_add(1, std::memory_order_relaxed);                                        \
  } while (0)

extern "C" {

uav_status_t uav_cfg_combine(const void* pred2, void* out, int64_t n, float guidance_scale,
                             int dtype, uav_stream_t stream) {
  UAV_REQUIRE(pred2 && out && n >= 0, "uav_cfg_combine: bad argument");
  if (n == 0) return UAV_OK;
  UAV_DISPATCH_DTYPE(dtype, cfg_kernel, sgrid(n), stream, pred2, out, n, guidance_scale);
  return UAV_OK;
}

uav_status_t uav_window_blend(void* dst, int64_t T, const void* src, int64_t Tw, int64_t t0,
                              uint32_t covered_mask, int64_t outer, int64_t hw, int dtype,
                              uav_stream_t stream) {
  UAV_REQUIRE(dst && src && T > 0 && Tw > 0 && Tw <= 32 && t0 >= 0 && t0 + Tw <= T && outer > 0 &&
                  hw > 0,
              "uav_window_blend: bad shape");
  UAV_DISPATCH_DTYPE(dtype, window_blend_kernel, sgrid(outer * Tw * hw), stream, dst, T, src, Tw,
                     (int)t0, covered_mask, outer, hw);
  return UAV_OK;
}

uav_status_t uav_ddim_step_v0(const void* model_output, const void* sample, void* x0, int64_t n,
                              int pred_type, float sqrt_alpha, float sqrt_beta, int clip,
                              float clip_range, int dtype, uav_stream_t stream) {
  UAV_REQUIRE(model_output && sample && x0 && n >= 0 && pred_type >= 0 && pred_type <= 2,
              "uav_ddim_step_v0: bad argument");
  if (n == 0) return UAV_OK;
  UAV_DISPATCH_DTYPE(dtype, ddim_v0_kernel, sgrid(n), stream, model_output, sample, x0, n,
                     pred_type, sqrt_alpha, sqrt_beta, 1.0f / sqrt_alpha, clip, clip_range);
  return UAV_OK;
}

uav_status_t uav_ddim_step_vt(const void* x0, const void* model_output, const void* sample,
                              void* prev, int64_t n, int pred_type, float sqrt_alpha,
                              float sqrt_beta, float sqrt_alpha_prev, float dir_coef, int clip,
                              float clip_range, float std_dev, const void* noise, int dtype,
                              uav_stream_t stream) {
  UAV_REQUIRE(x0 && model_output && sample && prev && n >= 0 && pred_type >= 0 && pred_type <= 2,
              "uav_ddim_step_vt: bad argument");
  if (n == 0) return UAV_OK;
  UAV_DISPATCH_DTYPE(dtype, ddim_vt_kernel, sgrid(n), stream, x0, model_output, sample, prev, n,
                     pred_type, sqrt_alpha, sqrt_beta, 1.0f / sqrt_beta, sqrt_alpha_prev, dir_coef,
                     clip, clip_range, std_dev, noise);
  return UAV_OK;
}

uav_status_t uav_add_noise(const void* x, const void* noise, void* out, int64_t n,
                           float sqrt_alpha, float sqrt_one_minus_alpha, int dtype,
                           uav_stream_t stream) {
  UAV_REQUIRE(x && noise && out && n >= 0, "uav_add_noise: bad argument");
  if (n == 0) return UAV_OK;
  UAV_DISPATCH_DTYPE(dtype, add_noise_kernel, sgrid(n), stream, x, noise, out, n, sqrt_alpha,
                     sqrt_one_minus_alpha);
  return UAV_OK;
}

uav_status_t uav_propagate_step(const void* feat_prop, const void* feat_cur, const void* flow_prop,
                                const void* flow_check, void* out, int64_t C, int64_t H, int64_t W,
                                int64_t cs_prop, int64_t cs_cur, int64_t cs_out, int64_t cs_flow_prop,
                                int64_t cs_flow_check, int nearest, int fuse, float fuse_scale,
                                float alpha1, float alpha2, int dtype, uav_stream_t stream) {
  UAV_REQUIRE(feat_prop && feat_cur && flow_prop && flow_check && out && C > 0 && H > 0 && W > 0,
              "uav_propagate_step: bad argument");
  const float inv_wm1 = 1.0f / static_cast<float>(W > 1 ? W - 1 : 1);
  const float inv_hm1 = 1.0f / static_cast<float>(H > 1 ? H - 1 : 1);
  UAV_DISPATCH_DTYPE(dtype, propagate_step_kernel, sgrid(H * W), stream, feat_prop, feat_cur,
                     flow_prop, flow_check, out, (int)C, (int)H, (int)W, cs_prop, cs_cur, cs_out,
                     cs_flow_prop, cs_flow_check, nearest, fuse, fuse_scale, alpha1, alpha2, inv_wm1,
                     inv_hm1);
  return UAV_OK;
}

uav_status_t uav_flow_resize_area(const void* in, void* out, int64_t planes, int64_t t_in, int64_t h_in,
                                  int64_t w_in, int64_t t_out, int64_t h_out, int64_t w_out, float scale,
                                  int dtype, uav_stream_t stream) {
  UAV_REQUIRE(in && out, "uav_flow_resize_area: null pointer");
  UAV_REQUIRE(planes > 0 && t_in > 0 && h_in > 0 && w_in > 0 && t_out > 0 && h_out > 0 && w_out > 0,
              "uav_flow_resize_area: bad shape");
  UAV_DISPATCH_DTYPE(dtype, flow_resize_area_kernel, sgrid(planes * t_out * h_out * w_out), stream, in,
                     out, planes, t_in, h_in, w_in, t_out, h_out, w_out, scale);
  return UAV_OK;
}

}  // extern "C"
