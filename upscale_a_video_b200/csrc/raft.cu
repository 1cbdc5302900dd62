// raft.cu — the non-GEMM kernels of the RAFT bidirectional optical flow that produces `flows_bi`
// (SURVEY.md §8f rank 1; reference: models_video/RAFT/{raft,corr,update,extractor}.py).  All convolutions and the
// all-pairs correlation run on the implicit-GEMM kernel (igemm.cu: uav_conv2d_taps / uav_linear); this file holds
//   * InstanceNorm(+ReLU) of the feature encoder (extractor.py:27-31,129-130), deterministic like the GroupNorm kernels;
//   * relu(a + b) of the residual blocks (extractor.py:57);
//   * the 2x2 average-pooling pyramid of the correlation volume and the fused 4-level (2r+1)^2 bilinear lookup
//     (corr.py:24-50) — the role of upstream's `alt_cuda_corr`, whose source the reference does not ship;
//   * the SepConvGRU gate arithmetic (update.py:47-60), the tanh / relu split of the context features (raft.py:117-120),
//     the coordinate update and the convex 8x upsampling (raft.py:73-84,122-139).
// Activations are channels-last fp16 [pixel][C]; coordinates, the correlation volume and the flows are fp32.
#include "uav_common.cuh"

namespace uav {

// ---------------------------------------------------------------------------------------
// InstanceNorm2d (no affine, biased variance, eps) + optional ReLU on [n][hw][C] fp16, C % 8 == 0, C <= 2048
// ---------------------------------------------------------------------------------------
constexpr int IN_THREADS = 256;
constexpr int IN_BLOCKS = 64;  // statistics blocks per sample

__global__ void __launch_bounds__(IN_THREADS)
    instnorm_stats_kernel(const __half* __restrict__ x, int64_t hw, int C, float2* __restrict__ partial) {
  extern __shared__ float in_smem[];  // [pixel lanes][C][2]
  const int n = blockIdx.y;
  const int octs = C >> 3;
  const int lanes = IN_THREADS / octs;
  const int my_lane = threadIdx.x / octs, oct = threadIdx.x % octs;
  const __half* xn = x + static_cast<int64_t>(n) * hw * C;
  float s[8], q[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) s[j] = q[j] = 0.f;
  if (my_lane < lanes) {
    for (int64_t p = static_cast<int64_t>(blockIdx.x) * lanes + my_lane; p < hw; p += static_cast<int64_t>(IN_BLOCKS) * lanes) {
      const uint4 v = ldg16(xn + p * C + oct * 8);
      const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __half22float2(h[j]);
        s[2 * j] += f.x;
        q[2 * j] += f.x * f.x;
        s[2 * j + 1] += f.y;
        q[2 * j + 1] += f.y * f.y;
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      in_smem[(my_lane * C + oct * 8 + j) * 2] = s[j];
      in_smem[(my_lane * C + oct * 8 + j) * 2 + 1] = q[j];
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += IN_THREADS) {
    float ts = 0.f, tq = 0.f;
    for (int l = 0; l < lanes; ++l) {  // fixed order: deterministic
      ts += in_smem[(l * C + c) * 2];
      tq += in_smem[(l * C + c) * 2 + 1];
    }
    partial[(static_cast<int64_t>(n) * IN_BLOCKS + blockIdx.x) * C + c] = make_float2(ts, tq);
  }
}

__global__ void instnorm_finalize_kernel(const float2* __restrict__ partial, int64_t total, int C, int64_t hw, float eps,
                                         float2* __restrict__ stats) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;  // (n, c)
  if (i >= total) return;
  const int64_t n = i / C;
  const int c = static_cast<int>(i % C);
  double s = 0.0, q = 0.0;
  for (int b = 0; b < IN_BLOCKS; ++b) {
    const float2 v = partial[(n * IN_BLOCKS + b) * C + c];
    s += v.x;
    q += v.y;
  }
  const double mean = s / static_cast<double>(hw);
  double var = q / static_cast<double>(hw) - mean * mean;  // biased, as F.instance_norm
  if (var < 0.0) var = 0.0;
  stats[i] = make_float2(static_cast<float>(mean), static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps))));
}

__global__ void instnorm_apply_kernel(const __half* __restrict__ x, int64_t hw, int C, const float2* __restrict__ stats,
                                      int relu, __half* __restrict__ y, int64_t total_octs) {
  const int octs = C >> 3;
  UAV_GRID_STRIDE(i, total_octs) {
    const int oct = static_cast<int>(i % octs);
    const int64_t pix = i / octs;
    const int64_t n = pix / hw;
    const uint4 v = ldg16(x + pix * C + oct * 8);
    const __half2* h = reinterpret_cast<const __half2*>(&v);
    uint4 o;
    uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __half22float2(h[j]);
      const float2 s0 = stats[n * C + oct * 8 + 2 * j], s1 = stats[n * C + oct * 8 + 2 * j + 1];
      float a = (f.x - s0.x) * s0.y, b = (f.y - s1.x) * s1.y;
      if (relu) {
        a = fmaxf(a, 0.f);
        b = fmaxf(b, 0.f);
      }
      __half2 r = __floats2half2_rn(a, b);
      ow[j] = *reinterpret_cast<uint32_t*>(&r);
    }
    stg16(y + pix * C + oct * 8, o);
  }
}

// y = relu(a + b), n8 groups of 8 halfs
__global__ void add_relu_kernel(const __half* __restrict__ a, const __half* __restrict__ b, __half* __restrict__ y, int64_t n8) {
  UAV_GRID_STRIDE(i, n8) {
    const uint4 va = ldg16(a + i * 8), vb = ldg16(b + i * 8);
    const __half2* ha = reinterpret_cast<const __half2*>(&va);
    const __half2* hb = reinterpret_cast<const __half2*>(&vb);
    uint4 o;
    uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 fa = __half22float2(ha[j]), fb = __half22float2(hb[j]);
      // the reference adds in fp32 (fp32 network); one rounding here
      __half2 r = __floats2half2_rn(fmaxf(fa.x + fb.x, 0.f), fmaxf(fa.y + fb.y, 0.f));
      ow[j] = *reinterpret_cast<uint32_t*>(&r);
    }
    stg16(y + i * 8, o);
  }
}

// net = tanh(cnet[:, :C]), inp = relu(cnet[:, C:2C])   (raft.py:117-120); writes inp to two destinations
__global__ void split_tanh_relu_kernel(const __half* __restrict__ cnet, int64_t rows, int C, __half* __restrict__ net,
                                       int64_t ld_net, __half* __restrict__ inp_a, int64_t ld_a, __half* __restrict__ inp_b,
                                       int64_t ld_b) {
  const int64_t total = rows * C;
  UAV_GRID_STRIDE(i, total) {
    const int64_t r = i / C;
    const int c = static_cast<int>(i % C);
    const float a = __half2float(cnet[r * 2 * C + c]), b = __half2float(cnet[r * 2 * C + C + c]);
    net[r * ld_net + c] = __float2half_rn(1.0f - 2.0f * rcp_ftz(1.0f + ex2_ftz(2.8853900817779268f * a)));
    const __half rb = __float2half_rn(fmaxf(b, 0.f));
    inp_a[r * ld_a + c] = rb;
    if (inp_b != nullptr) inp_b[r * ld_b + c] = rb;
  }
}

// ---------------------------------------------------------------------------------------
// correlation pyramid: F.avg_pool2d(corr, 2, stride=2) on [planes][h][w] fp32 (floor output size)
// ---------------------------------------------------------------------------------------
__global__ void avgpool2_kernel(const float* __restrict__ in, int64_t planes, int h, int w, float* __restrict__ out) {
  const int oh = h / 2, ow = w / 2;
  const int64_t total = planes * oh * ow;
  UAV_GRID_STRIDE(i, total) {
    const int x = static_cast<int>(i % ow), y = static_cast<int>((i / ow) % oh);
    const int64_t pl = i / (static_cast<int64_t>(ow) * oh);
    const float* src = in + (pl * h + 2 * y) * w + 2 * x;
    out[i] = (src[0] + src[1] + src[w] + src[w + 1]) * 0.25f;
  }
}

// ---------------------------------------------------------------------------------------
// fused 4-level lookup (corr.py:30-50): for query pixel p with current target coordinate (cx, cy), level i and window
// index (a, b): sample level i of ITS correlation plane at (cx / 2^i + d[a], cy / 2^i + d[b]), d = -r..r — the first
// window index offsets x and the second y (upstream quirk, see oracle/raft_oracle.py) — bilinear, zero outside,
// align_corners=True (pixel coordinates).  One warp per query pixel; out: fp16 [pixel][ld_out], channel = i*81 + a*9 + b.
// ---------------------------------------------------------------------------------------
struct LookupParams {
  const float* level[4];
  int h[4], w[4];
  const float* coords;  // [pixels][2]
  __half* out;
  int64_t ld_out;
  int64_t pixels;
  int pad_from, pad_to;  // channels [pad_from, pad_to) are written as zero
};

__global__ void __launch_bounds__(256)
    corr_lookup_kernel(const LookupParams p) {
  const int lane = threadIdx.x & 31;
  const int64_t pix = static_cast<int64_t>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (pix >= p.pixels) return;
  const float cx = p.coords[pix * 2], cy = p.coords[pix * 2 + 1];
  __half* o = p.out + pix * p.ld_out;
#pragma unroll
  for (int lvl = 0; lvl < 4; ++lvl) {
    const int h = p.h[lvl], w = p.w[lvl];
    const float* plane = p.level[lvl] + pix * h * w;
    const float sc = 1.0f / static_cast<float>(1 << lvl);
    const float bx = cx * sc, by = cy * sc;
    for (int k = lane; k < 81; k += 32) {
      const int a = k / 9, b = k % 9;
      const float x = bx + static_cast<float>(a - 4), y = by + static_cast<float>(b - 4);
      const float fx = floorf(x), fy = floorf(y);
      const int x0 = static_cast<int>(fx), y0 = static_cast<int>(fy);
      const float tx = x - fx, ty = y - fy;
      float v00 = 0.f, v01 = 0.f, v10 = 0.f, v11 = 0.f;
      const bool xin0 = x0 >= 0 && x0 < w, xin1 = x0 + 1 >= 0 && x0 + 1 < w;
      const bool yin0 = y0 >= 0 && y0 < h, yin1 = y0 + 1 >= 0 && y0 + 1 < h;
      if (yin0 && xin0) v00 = __ldg(plane + y0 * w + x0);
      if (yin0 && xin1) v01 = __ldg(plane + y0 * w + x0 + 1);
      if (yin1 && xin0) v10 = __ldg(plane + (y0 + 1) * w + x0);
      if (yin1 && xin1) v11 = __ldg(plane + (y0 + 1) * w + x0 + 1);
      const float v = (v00 * (1.f - tx) + v01 * tx) * (1.f - ty) + (v10 * (1.f - tx) + v11 * tx) * ty;
      o[lvl * 81 + k] = __float2half_rn(v);
    }
  }
  for (int c = p.pad_from + lane; c < p.pad_to; c += 32) o[c] = __float2half_rn(0.f);
}

// ---------------------------------------------------------------------------------------
// SepConvGRU gates (update.py:47-60).  zr: [rows][2C] = sigmoid(convz | convr)
// ---------------------------------------------------------------------------------------
__global__ void gru_rh_kernel(const __half* __restrict__ zr, int64_t ld_zr, const __half* __restrict__ h, int64_t ld_h,
                              __half* __restrict__ out, int64_t ld_out, int64_t rows, int C) {
  const int64_t total = rows * C;
  UAV_GRID_STRIDE(i, total) {
    const int64_t r = i / C;
    const int c = static_cast<int>(i % C);
    out[r * ld_out + c] = __float2half_rn(__half2float(zr[r * ld_zr + C + c]) * __half2float(h[r * ld_h + c]));
  }
}
__global__ void gru_update_kernel(const __half* __restrict__ zr, int64_t ld_zr, const __half* __restrict__ q, int64_t ld_q,
                                  __half* __restrict__ h, int64_t ld_h, int64_t rows, int C) {
  const int64_t total = rows * C;
  UAV_GRID_STRIDE(i, total) {
    const int64_t r = i / C;
    const int c = static_cast<int>(i % C);
    const float z = __half2float(zr[r * ld_zr + c]);
    const float hv = __half2float(h[r * ld_h + c]);
    h[r * ld_h + c] = __float2half_rn((1.f - z) * hv + z * __half2float(q[r * ld_q + c]));
  }
}

// coords1 += delta (fp32); flow = coords1 - coords0 with coords0 = (x, y) of the 1/8-resolution grid; the fp16 flow is
// written as channels [0, 2) of `flow16` ([rows][ld16], remaining channels untouched) and optionally scattered into two
// more buffers (the motion-feature tail of the GRU input)
__global__ void flow_update_kernel(float* __restrict__ coords1, const float* __restrict__ delta, int64_t ld_delta, int64_t rows,
                                   int w8, int h8, __half* __restrict__ flow16, int64_t ld16, __half* __restrict__ dst_a,
                                   int64_t ld_a, __half* __restrict__ dst_b, int64_t ld_b) {
  UAV_GRID_STRIDE(r, rows) {
    float cx = coords1[r * 2], cy = coords1[r * 2 + 1];
    if (delta != nullptr) {
      cx += delta[r * ld_delta];
      cy += delta[r * ld_delta + 1];
      coords1[r * 2] = cx;
      coords1[r * 2 + 1] = cy;
    }
    const int x = static_cast<int>(r % w8), y = static_cast<int>((r / w8) % h8);
    const __half fx = __float2half_rn(cx - static_cast<float>(x)), fy = __float2half_rn(cy - static_cast<float>(y));
    if (flow16 != nullptr) {
      flow16[r * ld16] = fx;
      flow16[r * ld16 + 1] = fy;
    }
    if (dst_a != nullptr) {
      dst_a[r * ld_a] = fx;
      dst_a[r * ld_a + 1] = fy;
    }
    if (dst_b != nullptr) {
      dst_b[r * ld_b] = fx;
      dst_b[r * ld_b + 1] = fy;
    }
  }
}

// convex 8x upsampling (raft.py:73-84): out[n][c][8i+a][8j+b] = sum_k softmax_k(mask[n,i,j][k*64+a*8+b]) * 8 * flow[n, i+ky-1, j+kx-1][c]
// with k = ky*3+kx and zero flow outside the grid; flow = coords1 - coords0.
__global__ void convex_upsample_kernel(const float* __restrict__ coords1, const __half* __restrict__ mask, int64_t ld_mask,
                                       int64_t nimg, int h8, int w8, float* __restrict__ out) {
  const int H = 8 * h8, W = 8 * w8;
  const int64_t total = nimg * H * W;
  UAV_GRID_STRIDE(i, total) {
    const int X = static_cast<int>(i % W), Y = static_cast<int>((i / W) % H);
    const int64_t n = i / (static_cast<int64_t>(W) * H);
    const int ci = Y >> 3, a = Y & 7, cj = X >> 3, b = X & 7;
    const __half* m = mask + ((n * h8 + ci) * w8 + cj) * ld_mask + a * 8 + b;
    float mv[9], mx = -INFINITY;
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      mv[k] = __half2float(m[k * 64]);
      mx = fmaxf(mx, mv[k]);
    }
    float den = 0.f;
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      mv[k] = __expf(mv[k] - mx);
      den += mv[k];
    }
    const float inv = 1.f / den;
    float ox = 0.f, oy = 0.f;
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      const int yy = ci + k / 3 - 1, xx = cj + k % 3 - 1;
      if (yy >= 0 && yy < h8 && xx >= 0 && xx < w8) {
        const int64_t r = (n * h8 + yy) * w8 + xx;
        const float fx = 8.f * (coords1[r * 2] - static_cast<float>(xx)), fy = 8.f * (coords1[r * 2 + 1] - static_cast<float>(yy));
        ox += mv[k] * inv * fx;
        oy += mv[k] * inv * fy;
      }
    }
    out[((n * 2 + 0) * H + Y) * W + X] = ox;
    out[((n * 2 + 1) * H + Y) * W + X] = oy;
  }
}

}  // namespace uav

using namespace uav;

extern "C" {

size_t uav_instnorm_workspace_bytes(int64_t n, int64_t C) {
  if (n <= 0 || C <= 0) return 0;
  return static_cast<size_t>(n) * C * (IN_BLOCKS + 1) * sizeof(float2);
}

uav_status_t uav_instnorm_relu(const void* x, int64_t n, int64_t hw, int64_t C, float eps, int relu, void* y, void* workspace,
                               uav_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  UAV_REQUIRE(x && y && workspace && n > 0 && hw > 0, "uav_instnorm_relu: bad argument");
  UAV_REQUIRE(C >= 8 && C % 8 == 0 && C <= 2048, "uav_instnorm_relu: C must be a multiple of 8 in [8, 2048]");
  UAV_REQUIRE(n <= 65535, "uav_instnorm_relu: n must be at most 65535");
  UAV_REQUIRE_ALIGNED16("uav_instnorm_relu", x);
  UAV_REQUIRE_ALIGNED16("uav_instnorm_relu", y);
  UAV_REQUIRE_ALIGNED16("uav_instnorm_relu", workspace);
  float2* partial = reinterpret_cast<float2*>(workspace);
  float2* stats = partial + n * IN_BLOCKS * C;
  // lanes * C * 8 bytes = floor(256 / octs) * octs * 64 <= 16 KB: no opt-in needed
  const size_t smem = static_cast<size_t>(IN_THREADS / (C / 8)) * C * 2 * sizeof(float);
  instnorm_stats_kernel<<<dim3(IN_BLOCKS, (unsigned)n), IN_THREADS, smem, stream>>>(reinterpret_cast<const __half*>(x), hw,
                                                                                   (int)C, partial);
  UAV_LAUNCHED();
  instnorm_finalize_kernel<<<(unsigned)((n * C + 127) / 128), 128, 0, stream>>>(partial, n * C, (int)C, hw, eps, stats);
  UAV_LAUNCHED();
  const int64_t total_octs = n * hw * (C / 8);
  instnorm_apply_kernel<<<stream_grid(total_octs, 256, 8), 256, 0, stream>>>(reinterpret_cast<const __half*>(x), hw, (int)C,
                                                                            stats, relu, reinterpret_cast<__half*>(y),
                                                                            total_octs);
  UAV_LAUNCHED();
  return UAV_OK;
}

uav_status_t uav_add_relu(const void* a, const void* b, void* y, int64_t n, uav_stream_t stream) {
  UAV_REQUIRE(a && b && y && n > 0 && n % 8 == 0, "uav_add_relu: n must be a positive multiple of 8");
  UAV_REQUIRE_ALIGNED16("uav_add_relu", a);
  UAV_REQUIRE_ALIGNED16("uav_add_relu", b);
  UAV_REQUIRE_ALIGNED16("uav_add_relu", y);
  add_relu_kernel<<<stream_grid(n / 8, 256, 8), 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const __half*>(a), reinterpret_cast<const __half*>(b), reinterpret_cast<__half*>(y), n / 8);
  UAV_LAUNCHED();
  return UAV_OK;
}

uav_status_t uav_raft_split_tanh_relu(const void* cnet, int64_t rows, int64_t C, void* net, int64_t ld_net, void* inp_a,
                                      int64_t ld_a, void* inp_b, int64_t ld_b, uav_stream_t stream) {
  UAV_REQUIRE(cnet && net && inp_a && rows > 0 && C > 0 && C <= INT32_MAX, "uav_raft_split_tanh_relu: bad argument");
  UAV_REQUIRE(ld_net >= C && ld_a >= C && (inp_b == nullptr || ld_b >= C),
              "uav_raft_split_tanh_relu: ld_net, ld_a and ld_b must be >= C");
  split_tanh_relu_kernel<<<stream_grid(rows * C, 256, 8), 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const __half*>(cnet), rows, (int)C, reinterpret_cast<__half*>(net), ld_net,
      reinterpret_cast<__half*>(inp_a), ld_a, reinterpret_cast<__half*>(inp_b), ld_b);
  UAV_LAUNCHED();
  return UAV_OK;
}

uav_status_t uav_avgpool2x2_f32(const float* in, int64_t planes, int64_t h, int64_t w, float* out, uav_stream_t stream) {
  UAV_REQUIRE(in && out && planes > 0 && h >= 2 && w >= 2 && h < (1 << 20) && w < (1 << 20), "uav_avgpool2x2_f32: bad argument");
  const int64_t total = planes * (h / 2) * (w / 2);
  avgpool2_kernel<<<stream_grid(total, 256, 8), 256, 0, (cudaStream_t)stream>>>(in, planes, (int)h, (int)w, out);
  UAV_LAUNCHED();
  return UAV_OK;
}

uav_status_t uav_raft_corr_lookup(const float* const* levels, const int32_t* hs, const int32_t* ws, const float* coords,
                                  int64_t pixels, void* out, int64_t ld_out, uav_stream_t stream) {
  UAV_REQUIRE(levels && hs && ws && coords && out && pixels > 0 && ld_out >= 324, "uav_raft_corr_lookup: bad argument");
  UAV_REQUIRE(ld_out <= INT32_MAX, "uav_raft_corr_lookup: ld_out must be < 2^31");
  LookupParams p;
  for (int i = 0; i < 4; ++i) {
    UAV_REQUIRE(levels[i] != nullptr && hs[i] >= 1 && ws[i] >= 1, "uav_raft_corr_lookup: bad pyramid level %d", i);
    p.level[i] = levels[i];
    p.h[i] = hs[i];
    p.w[i] = ws[i];
  }
  p.coords = coords;
  p.out = reinterpret_cast<__half*>(out);
  p.ld_out = ld_out;
  p.pixels = pixels;
  p.pad_from = 324;
  p.pad_to = (int)ld_out;
  corr_lookup_kernel<<<(unsigned)((pixels + 7) / 8), 256, 0, (cudaStream_t)stream>>>(p);
  UAV_LAUNCHED();
  return UAV_OK;
}

uav_status_t uav_raft_gru_rh(const void* zr, int64_t ld_zr, const void* h, int64_t ld_h, void* out, int64_t ld_out, int64_t rows,
                             int64_t C, uav_stream_t stream) {
  UAV_REQUIRE(zr && h && out && rows > 0 && C > 0 && C <= INT32_MAX, "uav_raft_gru_rh: bad argument");
  UAV_REQUIRE(ld_zr >= 2 * C, "uav_raft_gru_rh: ld_zr must be >= 2C (the r half is read)");
  UAV_REQUIRE(ld_h >= C && ld_out >= C, "uav_raft_gru_rh: ld_h and ld_out must be >= C");
  gru_rh_kernel<<<stream_grid(rows * C, 256, 8), 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const __half*>(zr), ld_zr,
                                                                                 reinterpret_cast<const __half*>(h), ld_h,
                                                                                 reinterpret_cast<__half*>(out), ld_out, rows,
                                                                                 (int)C);
  UAV_LAUNCHED();
  return UAV_OK;
}

uav_status_t uav_raft_gru_update(const void* zr, int64_t ld_zr, const void* q, int64_t ld_q, void* h, int64_t ld_h, int64_t rows,
                                 int64_t C, uav_stream_t stream) {
  UAV_REQUIRE(zr && q && h && rows > 0 && C > 0 && C <= INT32_MAX, "uav_raft_gru_update: bad argument");
  UAV_REQUIRE(ld_zr >= C && ld_q >= C && ld_h >= C, "uav_raft_gru_update: ld_zr, ld_q and ld_h must be >= C");
  gru_update_kernel<<<stream_grid(rows * C, 256, 8), 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const __half*>(zr),
                                                                                     ld_zr, reinterpret_cast<const __half*>(q),
                                                                                     ld_q, reinterpret_cast<__half*>(h), ld_h,
                                                                                     rows, (int)C);
  UAV_LAUNCHED();
  return UAV_OK;
}

uav_status_t uav_raft_flow_update(float* coords1, const float* delta, int64_t ld_delta, int64_t rows, int64_t h8, int64_t w8,
                                  void* flow16, int64_t ld16, void* dst_a, int64_t ld_a, void* dst_b, int64_t ld_b,
                                  uav_stream_t stream) {
  UAV_REQUIRE(coords1 && rows > 0 && h8 > 0 && w8 > 0 && rows % (h8 * w8) == 0, "uav_raft_flow_update: bad argument");
  UAV_REQUIRE(h8 <= INT32_MAX && w8 <= INT32_MAX, "uav_raft_flow_update: h8 and w8 must be < 2^31");
  UAV_REQUIRE((delta == nullptr || ld_delta >= 2) && (flow16 == nullptr || ld16 >= 2) && (dst_a == nullptr || ld_a >= 2) &&
                  (dst_b == nullptr || ld_b >= 2),
              "uav_raft_flow_update: ld_delta, ld16, ld_a and ld_b must be >= 2");
  flow_update_kernel<<<stream_grid(rows, 256, 8), 256, 0, (cudaStream_t)stream>>>(coords1, delta, ld_delta, rows, (int)w8,
                                                                                  (int)h8, reinterpret_cast<__half*>(flow16),
                                                                                  ld16, reinterpret_cast<__half*>(dst_a), ld_a,
                                                                                  reinterpret_cast<__half*>(dst_b), ld_b);
  UAV_LAUNCHED();
  return UAV_OK;
}

uav_status_t uav_raft_convex_upsample(const float* coords1, const void* mask, int64_t ld_mask, int64_t nimg, int64_t h8,
                                      int64_t w8, float* out, uav_stream_t stream) {
  UAV_REQUIRE(coords1 && mask && out && nimg > 0 && h8 > 0 && w8 > 0 && ld_mask >= 576, "uav_raft_convex_upsample: bad argument");
  UAV_REQUIRE(h8 < (1 << 28) && w8 < (1 << 28), "uav_raft_convex_upsample: h8 and w8 must be < 2^28 (8 h8 and 8 w8 are int)");
  convex_upsample_kernel<<<stream_grid(nimg * 64 * h8 * w8, 256, 8), 256, 0, (cudaStream_t)stream>>>(
      coords1, reinterpret_cast<const __half*>(mask), ld_mask, nimg, (int)h8, (int)w8, out);
  UAV_LAUNCHED();
  return UAV_OK;
}

}  // extern "C"
