// norm.cu — GroupNorm(+SiLU) over channels-last video tensors and LayerNorm over tokens.
// HBM-bound kernels (SURVEY.md §8a rows a6, a8): 128-bit coalesced loads, fp32 statistics
// (fp64 for the cross-block accumulation), fused affine + SiLU on the way out.
//
// GroupNorm semantics follow nn.GroupNorm applied to the reference's 5-D "b c t h w" tensors
// (resnet.py:231,267,278): one (mean, var) per (batch item, group) over (C/G)*T*H*W elements —
// statistics span all frames of the chunk.  The per-frame 4-D case (attention.py:374,
// AttentionBlock) is the same kernel with n_outer = b*t and pixels = h*w.
#include "uav_common.cuh"

#include <limits.h>
#include <string.h>

namespace uav {

constexpr int GN_THREADS = 256;

// ---------------------------------------------------------------------------------------
// stats, deterministic (no atomics): every block writes its {sum, sumsq} per group to
// partial[n][block][g]; gn_finalize_kernel reduces the blocks in a fixed order in fp64.
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(GN_THREADS)
    gn_stats_kernel(const __half* __restrict__ x, int64_t pixels, int C, int64_t ld, int G,
                    float2* __restrict__ partial) {
  // [pixel lane][unit] partial sums; pixel lanes * units == 2 * GN_THREADS
  __shared__ float s_sum[2 * GN_THREADS];
  __shared__ float s_sq[2 * GN_THREADS];
  const int n = blockIdx.y;
  const int octs = C >> 3;   // 8-channel vectors per pixel (<= 256)
  const int units = C >> 2;  // 4-channel units
  const __half* xn = x + static_cast<int64_t>(n) * pixels * ld;
  const int pix_per_iter = GN_THREADS / octs;
  const int my_pix = threadIdx.x / octs;
  const int oct = threadIdx.x % octs;
  float a0 = 0.f, q0 = 0.f, a1 = 0.f, q1 = 0.f;
  if (my_pix < pix_per_iter) {
    // 4 independent 16-byte loads in flight per thread (memory-level parallelism), fixed order
    const int64_t stride = static_cast<int64_t>(gridDim.x) * pix_per_iter;
    auto acc = [&](const uint4& v) {
      const __half2* h = reinterpret_cast<const __half2*>(&v);
      const float2 f0 = __half22float2(h[0]), f1 = __half22float2(h[1]);
      const float2 f2 = __half22float2(h[2]), f3 = __half22float2(h[3]);
      a0 += f0.x + f0.y + f1.x + f1.y;
      q0 += f0.x * f0.x + f0.y * f0.y + f1.x * f1.x + f1.y * f1.y;
      a1 += f2.x + f2.y + f3.x + f3.y;
      q1 += f2.x * f2.x + f2.y * f2.y + f3.x * f3.x + f3.y * f3.y;
    };
    int64_t p = static_cast<int64_t>(blockIdx.x) * pix_per_iter + my_pix;
    for (; p + 3 * stride < pixels; p += 4 * stride) {
      const uint4 v0 = ldg16(xn + p * ld + oct * 8);
      const uint4 v1 = ldg16(xn + (p + stride) * ld + oct * 8);
      const uint4 v2 = ldg16(xn + (p + 2 * stride) * ld + oct * 8);
      const uint4 v3 = ldg16(xn + (p + 3 * stride) * ld + oct * 8);
      acc(v0);
      acc(v1);
      acc(v2);
      acc(v3);
    }
    for (; p < pixels; p += stride) acc(ldg16(xn + p * ld + oct * 8));
    s_sum[my_pix * units + oct * 2] = a0;
    s_sq[my_pix * units + oct * 2] = q0;
    s_sum[my_pix * units + oct * 2 + 1] = a1;
    s_sq[my_pix * units + oct * 2 + 1] = q1;
  }
  __syncthreads();
  const int units_per_group = units / G;  // (C/G)/4
  for (int g = threadIdx.x; g < G; g += GN_THREADS) {
    float s = 0.f, q = 0.f;
    for (int pl = 0; pl < pix_per_iter; ++pl)
      for (int u = 0; u < units_per_group; ++u) {
        s += s_sum[pl * units + g * units_per_group + u];
        q += s_sq[pl * units + g * units_per_group + u];
      }
    partial[(static_cast<int64_t>(n) * gridDim.x + blockIdx.x) * G + g] = make_float2(s, q);
  }
}

// generic scalar statistics (any C, any G): used for tiny channel counts (C = 3)
__global__ void __launch_bounds__(GN_THREADS)
    gn_stats_generic_kernel(const __half* __restrict__ x, int64_t pixels, int C, int64_t ld, int G,
                            float2* __restrict__ partial) {
  __shared__ float s_s[GN_THREADS / 32], s_q[GN_THREADS / 32];
  const int n = blockIdx.y;
  const int cpg = C / G;
  const __half* xn = x + static_cast<int64_t>(n) * pixels * ld;
  for (int g = 0; g < G; ++g) {
    float s = 0.f, q = 0.f;
    for (int64_t p = static_cast<int64_t>(blockIdx.x) * GN_THREADS + threadIdx.x; p < pixels;
         p += static_cast<int64_t>(gridDim.x) * GN_THREADS) {
      for (int c = 0; c < cpg; ++c) {
        const float v = __half2float(xn[p * ld + g * cpg + c]);
        s += v;
        q += v * v;
      }
    }
    for (int o = 16; o > 0; o >>= 1) {
      s += __shfl_xor_sync(0xffffffff, s, o);
      q += __shfl_xor_sync(0xffffffff, q, o);
    }
    if ((threadIdx.x & 31) == 0) {
      s_s[threadIdx.x >> 5] = s;
      s_q[threadIdx.x >> 5] = q;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      float ts = 0.f, tq = 0.f;
      for (int w = 0; w < GN_THREADS / 32; ++w) {
        ts += s_s[w];
        tq += s_q[w];
      }
      partial[(static_cast<int64_t>(n) * gridDim.x + blockIdx.x) * G + g] = make_float2(ts, tq);
    }
    __syncthreads();
  }
}

// sums[n][g] = fp64 reduction of the per-block partials in a fixed order
__global__ void __launch_bounds__(256)
    gn_finalize_kernel(const float2* __restrict__ partial, int nblocks, int G,
                       double* __restrict__ sums) {
  // one CTA per (sample, group): thread t adds blocks t, t+256, ... in fp64, then a fixed shared-memory tree
  // (deterministic for a given launch geometry).  The first version used one warp per group in ONE CTA per sample:
  // 64 dependent strided loads per lane = 15 us per GroupNorm, as long as the statistics pass of the small layers.
  __shared__ double sh_s[256], sh_q[256];
  const int n = blockIdx.y, g = blockIdx.x;
  double s = 0.0, q = 0.0;
  for (int b = threadIdx.x; b < nblocks; b += 256) {
    const float2 v = partial[(static_cast<int64_t>(n) * nblocks + b) * G + g];
    s += v.x;
    q += v.y;
  }
  sh_s[threadIdx.x] = s;
  sh_q[threadIdx.x] = q;
  __syncthreads();
  for (int off = 128; off > 0; off >>= 1) {
    if (threadIdx.x < off) {
      sh_s[threadIdx.x] += sh_s[threadIdx.x + off];
      sh_q[threadIdx.x] += sh_q[threadIdx.x + off];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    sums[(static_cast<int64_t>(n) * G + g) * 2] = sh_s[0];
    sums[(static_cast<int64_t>(n) * G + g) * 2 + 1] = sh_q[0];
  }
}

// ---------------------------------------------------------------------------------------
// apply: y = (x - mean) * rstd * gamma + beta, optional SiLU; fp16 out
// ---------------------------------------------------------------------------------------
// {scale, shift} = {gamma[c] * rstd, beta[c] - mean * gamma[c] * rstd} of channel c in group g of slab n, from the
// fp64 {sum, sumsq} of (n, g) given as `nsplit` partials (added in a fixed order) over cnt elements.  gamma / beta are
// read after the fp64 math on purpose: passed as values, their loads are hoisted and the kernels' code changes.
__device__ __forceinline__ float2 gn_scale_shift(const double* __restrict__ sums, int nsplit, int n, int G, int g,
                                                 double cnt, const float* __restrict__ gamma,
                                                 const float* __restrict__ beta, int c, float eps) {
  double s = 0.0, q = 0.0;
  for (int k = 0; k < nsplit; ++k) {
    s += sums[((static_cast<int64_t>(n) * G + g) * nsplit + k) * 2];
    q += sums[((static_cast<int64_t>(n) * G + g) * nsplit + k) * 2 + 1];
  }
  const double mean = s / cnt;
  double var = q / cnt - mean * mean;
  if (var < 0.0) var = 0.0;
  const float rstd = static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps)));
  const float sc = gamma[c] * rstd;
  return make_float2(sc, beta[c] - static_cast<float>(mean) * sc);
}

// scalar apply for C % 8 != 0 (the C = 3 GroupNorm of the video VAE's condition input); statistics with nsplit = 1
__global__ void __launch_bounds__(GN_THREADS)
    gn_apply_kernel(const __half* __restrict__ x, int64_t pixels, int C, int64_t ld_in, int G,
                    const double* __restrict__ sums, const float* __restrict__ gamma,
                    const float* __restrict__ beta, float eps, int silu, __half* __restrict__ y,
                    int64_t ld_out) {
  extern __shared__ float2 s_aff[];  // [C] {scale, shift}
  const int n = blockIdx.y;
  const int cpg = C / G;
  const double cnt = static_cast<double>(pixels) * cpg;
  for (int c = threadIdx.x; c < C; c += GN_THREADS)
    s_aff[c] = gn_scale_shift(sums, 1, n, G, c / cpg, cnt, gamma, beta, c, eps);
  __syncthreads();
  const __half* xn = x + static_cast<int64_t>(n) * pixels * ld_in;
  __half* yn = y + static_cast<int64_t>(n) * pixels * ld_out;
  const int64_t total = pixels * C;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * GN_THREADS + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * GN_THREADS) {
    const int64_t p = i / C;
    const int c = static_cast<int>(i - p * C);
    float a = __half2float(xn[p * ld_in + c]) * s_aff[c].x + s_aff[c].y;
    if (silu) a = silu_f(a);
    yn[p * ld_out + c] = __float2half_rn(a);
  }
}

// vector path of the apply pass: thread = (pixel lane, 8-channel octet) like the stats kernel, so the 8 scale
// and 8 shift values of its channels live in registers for the whole pixel loop — no shared-memory
// lookups per element (a shared-memory table read per element saturates the LSU pipe at ~3 TB/s).
__global__ void __launch_bounds__(GN_THREADS)
    gn_apply_vec_kernel(const __half* __restrict__ x, int64_t pixels, int C, int64_t ld_in, int G,
                        const double* __restrict__ sums, int nsplit, const float* __restrict__ gamma,
                        const float* __restrict__ beta, float eps, int silu, __half* __restrict__ y,
                        int64_t ld_out, int c_total, int chan_off, int64_t x_slab_stride) {
  // C channels of THIS launch = channels [chan_off, chan_off + C) of a c_total-channel GroupNorm whose input is the
  // channel concatenation of several tensors (x_slab_stride: elements between the statistics slabs of this source, 0 when
  // the same rows serve every n); the plain case is c_total == C, chan_off == 0, x_slab_stride == pixels * ld_in
  const int n = blockIdx.y;
  const int octs = C >> 3;
  const int cpg = c_total / G;
  const int pix_per_iter = GN_THREADS / octs;
  const int my_pix = threadIdx.x / octs;
  const int oct = threadIdx.x % octs;
  if (my_pix >= pix_per_iter) return;
  const double cnt = static_cast<double>(pixels) * cpg;
  float sc[8], sh[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = chan_off + oct * 8 + j;
    const float2 a = gn_scale_shift(sums, nsplit, n, G, c / cpg, cnt, gamma, beta, c, eps);
    sc[j] = a.x;
    sh[j] = a.y;
  }
  const __half* xn = x + static_cast<int64_t>(n) * x_slab_stride + oct * 8;
  __half* yn = y + static_cast<int64_t>(n) * pixels * ld_out + chan_off + oct * 8;
  auto one = [&](int64_t p, const uint4& v) {
    const __half2* h = reinterpret_cast<const __half2*>(&v);
    uint4 o;
    uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __half22float2(h[j]);
      float a = f.x * sc[2 * j] + sh[2 * j];
      float b = f.y * sc[2 * j + 1] + sh[2 * j + 1];
      if (silu) silu2_f(a, b);  // two values per reciprocal (uav_common.cuh)
      ow[j] = pack_half2_sat(a, b);
    }
    stg16(yn + p * ld_out, o);
  };
  const int64_t stride = static_cast<int64_t>(gridDim.x) * pix_per_iter;
  int64_t p = static_cast<int64_t>(blockIdx.x) * pix_per_iter + my_pix;
  for (; p + 3 * stride < pixels; p += 4 * stride) {  // 4 loads in flight per thread
    const uint4 v0 = ldg16(xn + p * ld_in), v1 = ldg16(xn + (p + stride) * ld_in);
    const uint4 v2 = ldg16(xn + (p + 2 * stride) * ld_in), v3 = ldg16(xn + (p + 3 * stride) * ld_in);
    one(p, v0);
    one(p + stride, v1);
    one(p + 2 * stride, v2);
    one(p + 3 * stride, v3);
  }
  for (; p < pixels; p += stride) one(p, ldg16(xn + p * ld_in));
}

// ---------------------------------------------------------------------------------------
// statistics from the producers' epilogues (igemm.cu: uav_epilogue_t.gn_partial): x is the channel concatenation of up
// to 4 sources, each with fp32 {sum, sumsq} blocks [C_src / 8][blocks] over 8 channels x 16 rows.  One CTA per
// (group, n, split) adds its share of the blocks in fp64 in a fixed order -> sums[n][g][split].
// ---------------------------------------------------------------------------------------
struct GnSrc {
  const float2* p;
  int64_t blocks;     // blocks per octet row
  int64_t bps;        // blocks per statistics slab
  int64_t slab_mul;   // 1: slab n starts at n * bps; 0: every n reads the same blocks
  int oct0, octs;     // octet range of this source inside x
};
struct GnReduceParams {
  GnSrc src[4];
  int nsrc, oct_per_group, G;
};

__global__ void __launch_bounds__(256)
    gn_reduce_partials_kernel(const GnReduceParams prm, double* __restrict__ sums) {
  __shared__ double sh_s[256], sh_q[256];
  const int g = blockIdx.x, n = blockIdx.y, sp = blockIdx.z, S = gridDim.z;
  double s = 0.0, q = 0.0;
  for (int o = g * prm.oct_per_group; o < (g + 1) * prm.oct_per_group; ++o) {
    int k = 0;
    while (k + 1 < prm.nsrc && o >= prm.src[k].oct0 + prm.src[k].octs) ++k;
    const GnSrc& sr = prm.src[k];
    const float2* base = sr.p + static_cast<int64_t>(o - sr.oct0) * sr.blocks + static_cast<int64_t>(n) * sr.slab_mul * sr.bps;
    const int64_t b0 = sr.bps * sp / S, b1 = sr.bps * (sp + 1) / S;
    int64_t b = b0 + threadIdx.x;
    for (; b + 768 < b1; b += 1024) {  // 4 loads in flight
      const float2 v0 = base[b], v1 = base[b + 256], v2 = base[b + 512], v3 = base[b + 768];
      s += (static_cast<double>(v0.x) + v1.x) + (static_cast<double>(v2.x) + v3.x);
      q += (static_cast<double>(v0.y) + v1.y) + (static_cast<double>(v2.y) + v3.y);
    }
    for (; b < b1; b += 256) {
      const float2 v = base[b];
      s += v.x;
      q += v.y;
    }
  }
  sh_s[threadIdx.x] = s;
  sh_q[threadIdx.x] = q;
  __syncthreads();
  for (int off = 128; off > 0; off >>= 1) {
    if (threadIdx.x < off) {
      sh_s[threadIdx.x] += sh_s[threadIdx.x + off];
      sh_q[threadIdx.x] += sh_q[threadIdx.x + off];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const int64_t i = (static_cast<int64_t>(n) * prm.G + g) * S + sp;
    sums[i * 2] = sh_s[0];
    sums[i * 2 + 1] = sh_q[0];
  }
}

// affine[n][c] = {gamma[c] * rstd, beta[c] - mean * gamma[c] * rstd}: the per-(slab, channel) scale / shift of a GroupNorm,
// for consumers that apply it themselves (uav_conv_out_fused)
__global__ void gn_affine_kernel(const double* __restrict__ sums, int nsplit, int G, int C, double cnt,
                                 const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                 float2* __restrict__ affine) {
  const int n = blockIdx.y;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  affine[static_cast<int64_t>(n) * C + c] = gn_scale_shift(sums, nsplit, n, G, c / (C / G), cnt, gamma, beta, c, eps);
}

// ---------------------------------------------------------------------------------------
// LayerNorm over the last dim (C % 8 == 0, C <= 2048): one warp per token
// ---------------------------------------------------------------------------------------
template <int MAX_OCT, int U>
__global__ void __launch_bounds__(256)
    layernorm_kernel(const __half* __restrict__ x, int64_t rows, int C, int64_t ld_in,
                     const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                     __half* __restrict__ y, int64_t ld_out) {
  // warp per token, grid-stride over tokens: gamma / beta live in registers for the whole kernel (the first version
  // re-read them per token: 8 of its 12 load/store instructions per token, LSU-bound at 4.1 TB/s), U tokens in flight
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = static_cast<int64_t>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  const int64_t nwarps = static_cast<int64_t>(gridDim.x) * 8;
  const int octs = C >> 3;
  const float inv_c = 1.0f / C;
  float gg[MAX_OCT][8], bb[MAX_OCT][8];
#pragma unroll
  for (int i = 0; i < MAX_OCT; ++i) {
    const int oct = lane + i * 32;
    if (oct < octs) {
      const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + oct * 8));
      const float4 g1 = __ldg(reinterpret_cast<const float4*>(gamma + oct * 8 + 4));
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + oct * 8));
      const float4 b1 = __ldg(reinterpret_cast<const float4*>(beta + oct * 8 + 4));
      gg[i][0] = g0.x; gg[i][1] = g0.y; gg[i][2] = g0.z; gg[i][3] = g0.w;
      gg[i][4] = g1.x; gg[i][5] = g1.y; gg[i][6] = g1.z; gg[i][7] = g1.w;
      bb[i][0] = b0.x; bb[i][1] = b0.y; bb[i][2] = b0.z; bb[i][3] = b0.w;
      bb[i][4] = b1.x; bb[i][5] = b1.y; bb[i][6] = b1.z; bb[i][7] = b1.w;
    }
  }
  for (int64_t row0 = warp0; row0 < rows; row0 += U * nwarps) {
    int64_t rws[U];
#pragma unroll
    for (int u = 0; u < U; ++u) rws[u] = row0 + u * nwarps;
    uint4 v[U][MAX_OCT];
#pragma unroll
    for (int u = 0; u < U; ++u) {
#pragma unroll
      for (int i = 0; i < MAX_OCT; ++i) {
        const int oct = lane + i * 32;
        v[u][i] = (oct < octs && rws[u] < rows) ? ldg16(x + rws[u] * ld_in + oct * 8) : make_uint4(0, 0, 0, 0);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (rws[u] >= rows) continue;  // warp-uniform
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < MAX_OCT; ++i) {
        const __half2* h = reinterpret_cast<const __half2*>(&v[u][i]);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = __half22float2(h[j]);
          s += f.x + f.y;
        }
      }
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffff, s, o);
      const float mean = s * inv_c;
      float q = 0.f;
#pragma unroll
      for (int i = 0; i < MAX_OCT; ++i) {
        const int oct = lane + i * 32;
        if (oct < octs) {
          const __half2* h = reinterpret_cast<const __half2*>(&v[u][i]);
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float2 f = __half22float2(h[j]);
            q += (f.x - mean) * (f.x - mean) + (f.y - mean) * (f.y - mean);
          }
        }
      }
      for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffff, q, o);
      const float rstd = rsqrtf(q * inv_c + eps);
#pragma unroll
      for (int i = 0; i < MAX_OCT; ++i) {
        const int oct = lane + i * 32;
        if (oct < octs) {
          const __half2* h = reinterpret_cast<const __half2*>(&v[u][i]);
          uint4 o;
          uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float2 f = __half22float2(h[j]);
            __half2 r = __floats2half2_rn((f.x - mean) * rstd * gg[i][2 * j] + bb[i][2 * j],
                                          (f.y - mean) * rstd * gg[i][2 * j + 1] + bb[i][2 * j + 1]);
            ow[j] = *reinterpret_cast<uint32_t*>(&r);
          }
          stg16(y + rws[u] * ld_out + oct * 8, o);
        }
      }
    }
  }
}

}  // namespace uav

using namespace uav;

extern "C" {

static constexpr int GN_MAX_BLOCKS_PER_N = 2048;  // upper bound of gridDim.x of the stats kernels
static constexpr int GN_MAX_SPLIT = 32;            // partial sums per (n, group) of the from-partials path

size_t uav_groupnorm_workspace_bytes(int64_t n_outer, int groups) {
  // fp64 {sum, sumsq} per (n, group)  +  fp32 {sum, sumsq} per (n, block, group)
  return static_cast<size_t>(n_outer) * groups * (2 * sizeof(double) + GN_MAX_BLOCKS_PER_N * sizeof(float2));
}

// gridDim.x of a grid-stride pass over `items` per slab: about `per_sm` CTAs per SM over all n_outer slabs, at most one
// per `per_block` items, at least one
static int64_t gn_blocks(int per_sm, int64_t n_outer, int64_t items, int64_t per_block) {
  const int64_t want = ((int64_t)num_sms() * per_sm + n_outer - 1) / n_outer;
  const int64_t most = (items + per_block - 1) / per_block;
  const int64_t b = want < most ? want : most;
  return b < 1 ? 1 : b;
}

// statistics stage, read pass over x: per-block partials (the vector kernel when x allows 16-byte loads of whole 4-channel
// units of a group, else the generic one), then their fp64 reduction -> sums[n][g][S = 1][2] at the head of `workspace`
static uav_status_t gn_stats_pass(const void* x, int64_t n_outer, int64_t pixels, int64_t C, int64_t ld_in, int groups,
                                  void* workspace, cudaStream_t stream) {
  double* sums = reinterpret_cast<double*>(workspace);
  float2* partial = reinterpret_cast<float2*>(sums + n_outer * groups * 2);
  const __half* xh = reinterpret_cast<const __half*>(x);
  const bool vec = (C % 8 == 0) && ((C / groups) % 4 == 0) && (ld_in % 8 == 0) && aligned16(x);
  // vector kernel: >= ~16 pixels per thread to amortise the block reduction
  int64_t gx = vec ? gn_blocks(8, n_outer, pixels, GN_THREADS / (C / 8) * 16) : gn_blocks(4, n_outer, pixels, GN_THREADS);
  if (gx > GN_MAX_BLOCKS_PER_N) gx = GN_MAX_BLOCKS_PER_N;
  const dim3 grid((unsigned)gx, (unsigned)n_outer);
  if (vec)
    gn_stats_kernel<<<grid, GN_THREADS, 0, stream>>>(xh, pixels, (int)C, ld_in, groups, partial);
  else
    gn_stats_generic_kernel<<<grid, GN_THREADS, 0, stream>>>(xh, pixels, (int)C, ld_in, groups, partial);
  UAV_LAUNCHED();
  gn_finalize_kernel<<<dim3((unsigned)groups, (unsigned)n_outer), 256, 0, stream>>>(partial, (int)gx, groups, sums);
  UAV_LAUNCHED();
  return UAV_OK;
}

// statistics stage from the producers' blocks, checks: the sources of a C-channel GroupNorm -> `prm` and the split count
// *S.  Launches nothing, so that a caller can finish its own checks before gn_reduce_sources.
static uav_status_t gn_reduce_plan(int64_t n_outer, int64_t C, int groups, const uav_gn_source_t* sources, int n_sources,
                                   size_t workspace_bytes, GnReduceParams* prm, int* S_out) {
  const int cpg = (int)(C / groups);
  UAV_REQUIRE(cpg % 8 == 0, "groupnorm from partials: channels per group (%d) must be a multiple of 8", cpg);
  UAV_REQUIRE(n_sources >= 1 && n_sources <= 4, "groupnorm from partials: 1..4 sources");
  UAV_REQUIRE(workspace_bytes >= uav_groupnorm_workspace_bytes(n_outer, groups), "groupnorm from partials: workspace too small");
  memset(prm, 0, sizeof(*prm));
  int oct = 0;
  int64_t min_bps = INT64_MAX;
  for (int i = 0; i < n_sources; ++i) {
    const uav_gn_source_t& sc = sources[i];
    UAV_REQUIRE(sc.partial && sc.C > 0 && sc.C % 8 == 0 && sc.blocks > 0 && (sc.slabs == n_outer || sc.slabs == 1) &&
                    sc.blocks % sc.slabs == 0,
                "groupnorm from partials: bad source %d (C=%lld blocks=%lld slabs=%lld)", i, (long long)sc.C,
                (long long)sc.blocks, (long long)sc.slabs);
    prm->src[i].p = reinterpret_cast<const float2*>(sc.partial);
    prm->src[i].blocks = sc.blocks;
    prm->src[i].bps = sc.blocks / sc.slabs;
    prm->src[i].slab_mul = sc.slabs == n_outer ? 1 : 0;
    prm->src[i].oct0 = oct;
    prm->src[i].octs = (int)(sc.C / 8);
    oct += (int)(sc.C / 8);
    if (prm->src[i].bps < min_bps) min_bps = prm->src[i].bps;
  }
  UAV_REQUIRE(oct * 8 == C, "groupnorm from partials: sources cover %d channels, x has %lld", oct * 8, (long long)C);
  prm->nsrc = n_sources;
  prm->oct_per_group = cpg / 8;
  prm->G = groups;
  // enough CTAs to pull the blocks at HBM speed, at least ~256 blocks per split; GN_MAX_SPLIT doubles fit the workspace
  int64_t S = (4 * (int64_t)num_sms() + groups * n_outer - 1) / (groups * n_outer);
  if (S > min_bps / 256) S = min_bps / 256;
  if (S > GN_MAX_SPLIT) S = GN_MAX_SPLIT;
  if (S < 1) S = 1;
  *S_out = (int)S;
  return UAV_OK;
}

// statistics stage from the producers' blocks, launch: fp64 reduction -> sums[n][g][S][2] at the head of `workspace`
static uav_status_t gn_reduce_sources(const GnReduceParams& prm, int64_t n_outer, int S, void* workspace,
                                      cudaStream_t stream) {
  gn_reduce_partials_kernel<<<dim3((unsigned)prm.G, (unsigned)n_outer, (unsigned)S), 256, 0, stream>>>(
      prm, reinterpret_cast<double*>(workspace));
  UAV_LAUNCHED();
  return UAV_OK;
}

// apply stage, vector path: channels [chan, chan + Cs) of a C-channel GroupNorm from sums[n][g][S][2] at the head of
// `workspace`.  x: 16-byte aligned fp16 rows of ld_in elements (Cs, ld_in, ld_out % 8 == 0), slab n at n * x_slab_stride.
static uav_status_t gn_apply(const void* x, int64_t n_outer, int64_t pixels, int64_t Cs, int64_t ld_in,
                             int64_t x_slab_stride, int groups, const void* workspace, int S, const float* gamma,
                             const float* beta, float eps, int silu, void* y, int64_t ld_out, int64_t C, int chan,
                             cudaStream_t stream) {
  const int64_t gx = gn_blocks(16, n_outer, pixels, GN_THREADS / (Cs / 8) * 4);
  gn_apply_vec_kernel<<<dim3((unsigned)gx, (unsigned)n_outer), GN_THREADS, 0, stream>>>(
      reinterpret_cast<const __half*>(x), pixels, (int)Cs, ld_in, groups, reinterpret_cast<const double*>(workspace), S,
      gamma, beta, eps, silu, reinterpret_cast<__half*>(y), ld_out, (int)C, chan, x_slab_stride);
  UAV_LAUNCHED();
  return UAV_OK;
}

uav_status_t uav_groupnorm_silu(const void* x, int64_t n_outer, int64_t pixels, int64_t C,
                                int64_t ld_in, int groups, const float* gamma, const float* beta,
                                float eps, int silu, void* y, int64_t ld_out, void* workspace,
                                size_t workspace_bytes, uav_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  UAV_REQUIRE(x && y && gamma && beta && workspace, "uav_groupnorm_silu: null pointer");
  UAV_REQUIRE(n_outer > 0 && pixels > 0 && C > 0 && groups > 0 && C % groups == 0 && ld_in >= C &&
                  ld_out >= C,
              "uav_groupnorm_silu: bad shape (C=%lld groups=%d)", (long long)C, groups);
  UAV_REQUIRE(C <= 2048, "uav_groupnorm_silu: C > 2048 unsupported");
  UAV_REQUIRE(n_outer <= 65535, "uav_groupnorm_silu: n_outer too large");
  UAV_REQUIRE(workspace_bytes >= uav_groupnorm_workspace_bytes(n_outer, groups),
              "uav_groupnorm_silu: workspace too small");
  UAV_REQUIRE(C % 8 != 0 || (ld_in % 8 == 0 && ld_out % 8 == 0 && aligned16(x) && aligned16(y)),
              "uav_groupnorm_silu: C %% 8 == 0 tensors must be 16-byte aligned with ld %% 8 == 0");
  uav_status_t st = gn_stats_pass(x, n_outer, pixels, C, ld_in, groups, workspace, stream);
  if (st != UAV_OK) return st;
  if (C % 8 == 0)
    return gn_apply(x, n_outer, pixels, C, ld_in, pixels * ld_in, groups, workspace, 1, gamma, beta, eps, silu, y, ld_out,
                    C, 0, stream);
  gn_apply_kernel<<<dim3((unsigned)gn_blocks(16, n_outer, pixels * C, GN_THREADS * 4), (unsigned)n_outer), GN_THREADS,
                    2 * C * sizeof(float), stream>>>(reinterpret_cast<const __half*>(x), pixels, (int)C, ld_in, groups,
                                                     reinterpret_cast<const double*>(workspace), gamma, beta, eps, silu,
                                                     reinterpret_cast<__half*>(y), ld_out);
  UAV_LAUNCHED();
  return UAV_OK;
}

uav_status_t uav_groupnorm_affine(const void* x, int64_t n_outer, int64_t pixels, int64_t C, int64_t ld_in, int groups,
                                  const float* gamma, const float* beta, float eps, const uav_gn_source_t* sources,
                                  int n_sources, float* affine, void* workspace, size_t workspace_bytes,
                                  uav_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  UAV_REQUIRE(gamma && beta && affine && workspace, "uav_groupnorm_affine: null pointer");
  UAV_REQUIRE(n_outer > 0 && n_outer <= 65535 && pixels > 0 && C > 0 && C <= 2048 && groups > 0 && C % groups == 0,
              "uav_groupnorm_affine: bad shape (C=%lld groups=%d)", (long long)C, groups);
  int S = 1;
  uav_status_t st;
  if (n_sources > 0) {
    UAV_REQUIRE(sources != nullptr, "uav_groupnorm_affine: null sources");
    GnReduceParams prm;
    st = gn_reduce_plan(n_outer, C, groups, sources, n_sources, workspace_bytes, &prm, &S);
    if (st == UAV_OK) st = gn_reduce_sources(prm, n_outer, S, workspace, stream);
  } else {
    UAV_REQUIRE(x != nullptr && ld_in >= C && C % 8 == 0 && (C / groups) % 4 == 0 && ld_in % 8 == 0 && aligned16(x),
                "uav_groupnorm_affine: without sources x must be an aligned fp16 tensor with C %% 8 == 0");
    UAV_REQUIRE(workspace_bytes >= uav_groupnorm_workspace_bytes(n_outer, groups), "uav_groupnorm_affine: workspace too small");
    st = gn_stats_pass(x, n_outer, pixels, C, ld_in, groups, workspace, stream);
  }
  if (st != UAV_OK) return st;
  gn_affine_kernel<<<dim3((unsigned)((C + 255) / 256), (unsigned)n_outer), 256, 0, stream>>>(
      reinterpret_cast<const double*>(workspace), S, groups, (int)C, static_cast<double>(pixels) * (C / groups), gamma,
      beta, eps, reinterpret_cast<float2*>(affine));
  UAV_LAUNCHED();
  return UAV_OK;
}

uav_status_t uav_groupnorm_silu_from_partials(const void* x, int64_t n_outer, int64_t pixels, int64_t C,
                                              int64_t ld_in, int groups, const float* gamma, const float* beta,
                                              float eps, int silu, void* y, int64_t ld_out,
                                              const uav_gn_source_t* sources, int n_sources, void* workspace,
                                              size_t workspace_bytes, uav_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  UAV_REQUIRE(y && gamma && beta && workspace && sources, "uav_groupnorm_silu_from_partials: null pointer");
  UAV_REQUIRE(x != nullptr || sources[0].x != nullptr, "uav_groupnorm_silu_from_partials: no input tensor");
  UAV_REQUIRE(n_outer > 0 && n_outer <= 65535 && pixels > 0 && C > 0 && C <= 2048 && groups > 0 && C % groups == 0 &&
                  ld_out >= C,
              "uav_groupnorm_silu_from_partials: bad shape (C=%lld groups=%d)", (long long)C, groups);
  UAV_REQUIRE(C % 8 == 0 && (x == nullptr || (ld_in % 8 == 0 && ld_in >= C)) && ld_out % 8 == 0 && aligned16(x) &&
                  aligned16(y),
              "uav_groupnorm_silu_from_partials: tensors must be 16-byte aligned with ld %% 8 == 0");
  GnReduceParams prm;
  int S = 1;
  uav_status_t st = gn_reduce_plan(n_outer, C, groups, sources, n_sources, workspace_bytes, &prm, &S);
  if (st != UAV_OK) return st;
  // apply: one launch over x, or — when the sources carry their own tensors (a concat that was never materialised) — one
  // launch per source, each writing its channel range of the dense output
  const bool per_source = sources[0].x != nullptr;
  for (int i = 0; per_source && i < n_sources; ++i) {
    const uav_gn_source_t& sc = sources[i];
    UAV_REQUIRE(sc.x != nullptr && sc.ld >= sc.C && sc.ld % 8 == 0 && aligned16(sc.x) && sc.C <= 2048,
                "uav_groupnorm_silu_from_partials: bad tensor of source %d", i);
  }
  st = gn_reduce_sources(prm, n_outer, S, workspace, stream);
  if (st != UAV_OK) return st;
  if (!per_source)
    return gn_apply(x, n_outer, pixels, C, ld_in, pixels * ld_in, groups, workspace, S, gamma, beta, eps, silu, y, ld_out,
                    C, 0, stream);
  int chan = 0;
  for (int i = 0; i < n_sources; ++i) {
    const uav_gn_source_t& sc = sources[i];
    st = gn_apply(sc.x, n_outer, pixels, sc.C, sc.ld, sc.slab_stride, groups, workspace, S, gamma, beta, eps, silu, y,
                  ld_out, C, chan, stream);
    if (st != UAV_OK) return st;
    chan += (int)sc.C;
  }
  return UAV_OK;
}

uav_status_t uav_layernorm(const void* x, int64_t rows, int64_t C, int64_t ld_in,
                           const float* gamma, const float* beta, float eps, void* y,
                           int64_t ld_out, uav_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  UAV_REQUIRE(x && y && gamma && beta, "uav_layernorm: null pointer");
  UAV_REQUIRE(rows >= 0 && C > 0 && C % 8 == 0 && C <= 2048 && ld_in >= C && ld_out >= C &&
                  ld_in % 8 == 0 && ld_out % 8 == 0,
              "uav_layernorm: bad shape (C=%lld)", (long long)C);
  UAV_REQUIRE_ALIGNED16("uav_layernorm", x);
  UAV_REQUIRE_ALIGNED16("uav_layernorm", y);
  UAV_REQUIRE_ALIGNED16("uav_layernorm", gamma);
  UAV_REQUIRE_ALIGNED16("uav_layernorm", beta);
  if (rows == 0) return UAV_OK;
  // grid-stride over tokens: 8 warps per block, at most 8 blocks per SM
  const unsigned grid = stream_grid(rows, 8, 8);
  const int octs = (int)(C / 8);
  if (octs <= 64)
    layernorm_kernel<2, 2><<<grid, 256, 0, stream>>>(reinterpret_cast<const __half*>(x), rows, (int)C,
                                                  ld_in, gamma, beta, eps,
                                                  reinterpret_cast<__half*>(y), ld_out);
  else if (octs <= 128)
    layernorm_kernel<4, 1><<<grid, 256, 0, stream>>>(reinterpret_cast<const __half*>(x), rows, (int)C,
                                                  ld_in, gamma, beta, eps,
                                                  reinterpret_cast<__half*>(y), ld_out);
  else
    layernorm_kernel<8, 1><<<grid, 256, 0, stream>>>(reinterpret_cast<const __half*>(x), rows, (int)C,
                                                  ld_in, gamma, beta, eps,
                                                  reinterpret_cast<__half*>(y), ld_out);
  UAV_LAUNCHED();
  return UAV_OK;
}

}  // extern "C"
