// llava.cu — the kernels of the LLaVA-1.5 captioner (llava.py) that the shared GEMM / attention kernels do not cover:
// the Llama decoder's RMSNorm, rotary embedding with the KV-cache append, SwiGLU, the one-row weight stream of every
// decoded token (GEMV), attention of one query row against the KV cache, and the top-p sampler.
//
// A decoded token reads every decoder weight once (about 25.7 GB at 13B) and does 2 FLOP per weight, so the decode
// step is bound by HBM bandwidth; the GEMV is built to keep enough bytes in flight on every SM.  Every reduction here
// runs in a fixed order: repeated launches are bitwise equal.
#include "uav_common.cuh"

namespace uav {

// ---------------------------------------------------------------------------------------
// RMSNorm (transformers LlamaRMSNorm): fp32 mean of squares, x * rsqrt(var + eps) rounded to fp16, then weight * that
// in fp16.  One CTA of 256 threads per row.
// ---------------------------------------------------------------------------------------
constexpr int RMS_THREADS = 256;

__device__ __forceinline__ float block_sum_256(float v, float* red) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < RMS_THREADS / 32; ++w) t += red[w];  // same order in every thread
  return t;
}

__global__ void __launch_bounds__(RMS_THREADS)
    rmsnorm_kernel(const __half* __restrict__ x, int64_t ldx, const __half* __restrict__ w, int C, float eps,
                   __half* __restrict__ out, int64_t ldo) {
  __shared__ float red[RMS_THREADS / 32];
  const __half* xr = x + blockIdx.x * ldx;
  __half* orow = out + blockIdx.x * ldo;
  float ss = 0.f;
  for (int c = threadIdx.x * 8; c < C; c += RMS_THREADS * 8) {
    const uint4 u = ldg16(xr + c);
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 f = __half22float2(h[e]);
      ss = fmaf(f.x, f.x, ss);
      ss = fmaf(f.y, f.y, ss);
    }
  }
  const float r = rsqrtf(block_sum_256(ss, red) / C + eps);
  for (int c = threadIdx.x * 8; c < C; c += RMS_THREADS * 8) {
    const uint4 u = ldg16(xr + c), g = ldg16(w + c);
    const __half2* h = reinterpret_cast<const __half2*>(&u);
    const __half2* gw = reinterpret_cast<const __half2*>(&g);
    uint4 o;
    __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 f = __half22float2(h[e]);
      oh[e] = __hmul2(gw[e], __floats2half2_rn(f.x * r, f.y * r));
    }
    stg16(orow + c, o);
  }
}

// ---------------------------------------------------------------------------------------
// Rotary embedding in rotate-half form on the q and k columns of n fused q|k|v rows at positions [p0, p0 + n), head_dim
// 128: q is rotated in place, rotated k and v are written to rows [p0, p0 + n) of the layer's KV cache.  cos_sin is
// fp32 [positions][64][2] (cos, sin of position * inv_freq[i]).  One thread per (row, head, i < 64) pair (i, i + 64).
// ---------------------------------------------------------------------------------------
__global__ void rope_kv_append_kernel(__half* __restrict__ qkv, int64_t ld_qkv, int n, int heads, int p0,
                                      const float2* __restrict__ cos_sin, __half* __restrict__ kc,
                                      __half* __restrict__ vc, int64_t ld_kv) {
  const int64_t items = static_cast<int64_t>(n) * heads * 64;
  const int C = heads * 128;
  UAV_GRID_STRIDE(t, items) {
    const int i = static_cast<int>(t & 63);
    const int64_t rh = t >> 6;
    const int h = static_cast<int>(rh % heads), r = static_cast<int>(rh / heads);
    const float2 cs = cos_sin[static_cast<int64_t>(p0 + r) * 64 + i];
    __half* row = qkv + r * ld_qkv + h * 128 + i;
    const int64_t krow = static_cast<int64_t>(p0 + r) * ld_kv + h * 128 + i;
    // x1 = x[i], x2 = x[i + 64]:  out[i] = x1 cos - x2 sin,  out[i + 64] = x2 cos + x1 sin
    const float q1 = __half2float(row[0]), q2 = __half2float(row[64]);
    row[0] = __float2half_rn(q1 * cs.x - q2 * cs.y);
    row[64] = __float2half_rn(q2 * cs.x + q1 * cs.y);
    const float k1 = __half2float(row[C]), k2 = __half2float(row[C + 64]);
    kc[krow] = __float2half_rn(k1 * cs.x - k2 * cs.y);
    kc[krow + 64] = __float2half_rn(k2 * cs.x + k1 * cs.y);
    vc[krow] = row[2 * C];
    vc[krow + 64] = row[2 * C + 64];
  }
}

// ---------------------------------------------------------------------------------------
// SwiGLU (transformers LlamaMLP): out[r][c] = silu(gu[r][c]) * gu[r][I + c], from the fused gate|up output
// ---------------------------------------------------------------------------------------
__global__ void swiglu_kernel(const __half* __restrict__ gu, int64_t ld_gu, int64_t rows, int I, __half* __restrict__ out,
                              int64_t ldo) {
  const int64_t per_row = I / 8;
  UAV_GRID_STRIDE(t, rows * per_row) {
    const int64_t r = t / per_row;
    const int c = static_cast<int>(t % per_row) * 8;
    const uint4 g = ldg16(gu + r * ld_gu + c), u = ldg16(gu + r * ld_gu + I + c);
    const __half2* gh = reinterpret_cast<const __half2*>(&g);
    const __half2* uh = reinterpret_cast<const __half2*>(&u);
    uint4 o;
    uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 gf = __half22float2(gh[e]), uf = __half22float2(uh[e]);
      ow[e] = pack_half2_rn(gf.x / (1.f + expf(-gf.x)) * uf.x, gf.y / (1.f + expf(-gf.y)) * uf.y);
    }
    stg16(out + r * ldo + c, o);
  }
}

// ---------------------------------------------------------------------------------------
// GEMV: y[N] = W[N][K] . x[K] for one row, fp32 accumulation.  x is staged in shared memory.  A CTA of 8 warps takes
// 8 / S rows at a time; the S warps of a row split K (split-K), each lane streams 16-byte chunks of the row with
// non-coherent, L1-bypassing loads, GEMV_UNROLL chunks in flight per lane.  The S x 32 partial sums of a row are
// combined in a fixed order (a butterfly in each warp, then the S warps in order), so results are deterministic.
// Epilogue: fp16 out (optionally + fp16 residual, one rounding) or fp32 out.
// ---------------------------------------------------------------------------------------
constexpr int GEMV_THREADS = 256;
constexpr int GEMV_UNROLL = 4;
constexpr int GEMV_MAX_K = 16384;

__device__ __forceinline__ uint4 ldg16_stream(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::256B.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

__device__ __forceinline__ float dot8(const uint4& w, const uint4& x, float acc) {
  const __half2* wh = reinterpret_cast<const __half2*>(&w);
  const __half2* xh = reinterpret_cast<const __half2*>(&x);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 a = __half22float2(wh[e]), b = __half22float2(xh[e]);
    acc = fmaf(a.x, b.x, acc);
    acc = fmaf(a.y, b.y, acc);
  }
  return acc;
}

__global__ void __launch_bounds__(GEMV_THREADS)
    gemv_kernel(const __half* __restrict__ w, const __half* __restrict__ x, int N, int K, int S,
                const __half* __restrict__ residual, void* __restrict__ out, int out_f32) {
  extern __shared__ __align__(16) uint8_t gemv_smem[];
  __half* sx = reinterpret_cast<__half*>(gemv_smem);
  float* red = reinterpret_cast<float*>(gemv_smem + static_cast<size_t>(K) * 2);  // [8 warps]
  const int chunks = K / 8;
  for (int c = threadIdx.x; c < chunks; c += GEMV_THREADS)
    reinterpret_cast<uint4*>(sx)[c] = ldg16(x + 8 * c);
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rows_per_cta = (GEMV_THREADS / 32) / S;
  const int part = warp % S;
  // the S warps of a row take interleaved 16-byte chunks: chunk c = (i * S + part) * 32 + lane
  const int stride = S * 32;
  for (int row0 = blockIdx.x * rows_per_cta; row0 < N; row0 += gridDim.x * rows_per_cta) {
    const int row = row0 + warp / S;
    float acc = 0.f;
    if (row < N) {
      const __half* wr = w + static_cast<int64_t>(row) * K;
      int c = part * 32 + lane;
      for (; c + (GEMV_UNROLL - 1) * stride < chunks; c += GEMV_UNROLL * stride) {
        uint4 wv[GEMV_UNROLL];
#pragma unroll
        for (int u = 0; u < GEMV_UNROLL; ++u) wv[u] = ldg16_stream(wr + 8 * (c + u * stride));
#pragma unroll
        for (int u = 0; u < GEMV_UNROLL; ++u)
          acc = dot8(wv[u], reinterpret_cast<const uint4*>(sx)[c + u * stride], acc);
      }
      for (; c < chunks; c += stride) acc = dot8(ldg16_stream(wr + 8 * c), reinterpret_cast<const uint4*>(sx)[c], acc);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    if (lane == 0) red[warp] = acc;
    __syncthreads();
    if (threadIdx.x < rows_per_cta && row0 + (int)threadIdx.x < N) {
      const int r = row0 + threadIdx.x;
      float y = 0.f;
      for (int s = 0; s < S; ++s) y += red[threadIdx.x * S + s];
      if (out_f32) {
        reinterpret_cast<float*>(out)[r] = y;
      } else {
        if (residual) y += __half2float(residual[r]);
        reinterpret_cast<__half*>(out)[r] = __float2half_rn(y);
      }
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------
// Decode attention (flash-decoding): one query row per head against L cached keys, head_dim 128.  Stage 1: CTA (head,
// chunk of DEC_CHUNK keys), 4 warps, each warp a quarter of the chunk with an online softmax (lane = 4 of the 128 dims),
// the 4 warps merged in order -> (m, l, o[128]) of the chunk.  Stage 2: one CTA per head merges the chunks in order.
// ---------------------------------------------------------------------------------------
constexpr int DEC_CHUNK = 64;
constexpr int DEC_PART = 2 + 128;  // m, l, o[128] (fp32) per (head, chunk)

__global__ void __launch_bounds__(128)
    attn_decode_chunk_kernel(const __half* __restrict__ q, const __half* __restrict__ kc, const __half* __restrict__ vc,
                             int64_t ld_kv, int L, float scale_log2, float* __restrict__ part) {
  __shared__ float sm[4][DEC_PART];
  const int h = blockIdx.y, chunk = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint2 qu = *reinterpret_cast<const uint2*>(q + h * 128 + 4 * lane);
  const __half2* qh = reinterpret_cast<const __half2*>(&qu);
  const float2 q01 = __half22float2(qh[0]), q23 = __half22float2(qh[1]);
  float m = -INFINITY, l = 0.f, o[4] = {0.f, 0.f, 0.f, 0.f};
  const int k0 = chunk * DEC_CHUNK + warp * (DEC_CHUNK / 4);
  const int k1 = min(k0 + DEC_CHUNK / 4, L);
  for (int j = k0; j < k1; ++j) {
    const int64_t off = static_cast<int64_t>(j) * ld_kv + h * 128 + 4 * lane;
    const uint2 ku = *reinterpret_cast<const uint2*>(kc + off);
    const uint2 vu = *reinterpret_cast<const uint2*>(vc + off);
    const __half2* kh = reinterpret_cast<const __half2*>(&ku);
    const float2 k01 = __half22float2(kh[0]), k23 = __half22float2(kh[1]);
    float s = q01.x * k01.x;
    s = fmaf(q01.y, k01.y, s);
    s = fmaf(q23.x, k23.x, s);
    s = fmaf(q23.y, k23.y, s);
#pragma unroll
    for (int off2 = 16; off2 > 0; off2 >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off2);
    s *= scale_log2;
    const float m_new = fmaxf(m, s);
    const float alpha = exp2f(m - m_new), p = exp2f(s - m_new);
    m = m_new;
    l = l * alpha + p;
    const __half2* vh = reinterpret_cast<const __half2*>(&vu);
    const float2 v01 = __half22float2(vh[0]), v23 = __half22float2(vh[1]);
    o[0] = fmaf(p, v01.x, o[0] * alpha);
    o[1] = fmaf(p, v01.y, o[1] * alpha);
    o[2] = fmaf(p, v23.x, o[2] * alpha);
    o[3] = fmaf(p, v23.y, o[3] * alpha);
  }
  if (lane == 0) {
    sm[warp][0] = m;
    sm[warp][1] = l;
  }
#pragma unroll
  for (int e = 0; e < 4; ++e) sm[warp][2 + 4 * lane + e] = o[e];
  __syncthreads();
  // merge the 4 warps in order; thread t owns output column t (warps that saw no key have m = -inf, l = 0)
  float M = -INFINITY;
#pragma unroll
  for (int w2 = 0; w2 < 4; ++w2) M = fmaxf(M, sm[w2][0]);
  float Ls = 0.f, Os = 0.f;
#pragma unroll
  for (int w2 = 0; w2 < 4; ++w2) {
    const float a = sm[w2][0] == -INFINITY ? 0.f : exp2f(sm[w2][0] - M);
    Ls = fmaf(sm[w2][1], a, Ls);
    Os = fmaf(sm[w2][2 + threadIdx.x], a, Os);
  }
  float* pp = part + (static_cast<int64_t>(h) * gridDim.x + chunk) * DEC_PART;
  if (threadIdx.x == 0) {
    pp[0] = M;
    pp[1] = Ls;
  }
  pp[2 + threadIdx.x] = Os;
}

__global__ void __launch_bounds__(128)
    attn_decode_merge_kernel(const float* __restrict__ part, int chunks, __half* __restrict__ out) {
  const int h = blockIdx.x;
  const float* ph = part + static_cast<int64_t>(h) * chunks * DEC_PART;
  float M = -INFINITY;
  for (int c = 0; c < chunks; ++c) M = fmaxf(M, ph[c * DEC_PART]);
  float Ls = 0.f, Os = 0.f;
  for (int c = 0; c < chunks; ++c) {
    const float a = exp2f(ph[c * DEC_PART] - M);  // every chunk holds at least one key: m is finite
    Ls = fmaf(ph[c * DEC_PART + 1], a, Ls);
    Os = fmaf(ph[c * DEC_PART + 2 + threadIdx.x], a, Os);
  }
  out[h * 128 + threadIdx.x] = __float2half_rn(Os / Ls);
}

// ---------------------------------------------------------------------------------------
// Top-p sampling (transformers TemperatureLogitsWarper + TopPLogitsWarper + multinomial), one CTA of 1024 threads.
// p = softmax(logits / T) in fp32, held in shared memory.  TopPLogitsWarper drops the ascending-sorted prefix whose
// cumulative mass is <= 1 - top_p and keeps at least one token; for distinct probabilities that keeps exactly the
// tokens whose strictly more probable tokens have mass < top_p.  That mass is monotone in p, so the smallest kept
// probability t is found by bisecting its fp32 bit pattern (31 block reductions, no sort); the nucleus is {p >= t}.
// The token is the inverse CDF of the nucleus in vocabulary order at u * (nucleus mass), u in [0, 1) supplied by the
// caller.  temperature == 0 returns the argmax (first index on ties).
// ---------------------------------------------------------------------------------------
constexpr int SMP_THREADS = 1024;
constexpr int SMP_MAX_V = 49152;

template <class T, class Op>
__device__ __forceinline__ T block_reduce_1024(T v, T* red, Op op) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, off));
  __syncthreads();  // red may still be read by the previous reduction
  if (lane == 0) red[warp] = v;
  __syncthreads();
  T t = red[0];
#pragma unroll
  for (int w = 1; w < 32; ++w) t = op(t, red[w]);
  return t;
}

__global__ void __launch_bounds__(SMP_THREADS)
    sample_top_p_kernel(const float* __restrict__ logits, int V, float temperature, float top_p, float u,
                        int64_t* __restrict__ token) {
  extern __shared__ __align__(16) float sp[];  // [V] probabilities
  __shared__ float redf[32];
  __shared__ unsigned long long redu[32];
  __shared__ float scan[SMP_THREADS];
  const int tid = threadIdx.x;
  const auto fmax_op = [](float a, float b) { return fmaxf(a, b); };
  const auto fadd_op = [](float a, float b) { return a + b; };
  if (temperature == 0.f) {
    // argmax, first index on ties: minimise (order-flipped value bits, index) packed in 64 bits; NaN never wins
    unsigned long long best = ~0ull;
    for (int i = tid; i < V; i += SMP_THREADS) {
      const float v = logits[i];
      if (v != v) continue;
      const uint32_t b = __float_as_uint(v);
      const uint32_t key = (b & 0x80000000u) ? b : ~b & 0x7fffffffu;  // larger value -> smaller key
      const unsigned long long k = (static_cast<unsigned long long>(key) << 32) | static_cast<uint32_t>(i);
      best = k < best ? k : best;
    }
    best = block_reduce_1024(best, redu, [](unsigned long long a, unsigned long long b) { return a < b ? a : b; });
    if (tid == 0) *token = best == ~0ull ? 0 : static_cast<int64_t>(best & 0xffffffffu);
    return;
  }
  float mx = -INFINITY;
  for (int i = tid; i < V; i += SMP_THREADS) mx = fmaxf(mx, logits[i] / temperature);
  mx = block_reduce_1024(mx, redf, fmax_op);
  float sum = 0.f;
  for (int i = tid; i < V; i += SMP_THREADS) {
    const float e = expf(logits[i] / temperature - mx);
    sp[i] = e;
    sum += e;
  }
  const float inv_sum = 1.f / block_reduce_1024(sum, redf, fadd_op);
  for (int i = tid; i < V; i += SMP_THREADS) sp[i] *= inv_sum;
  __syncthreads();
  // smallest t (as fp32 bits) with mass(p > t) < top_p; t = max p satisfies it (mass 0)
  float pm = 0.f;
  for (int i = tid; i < V; i += SMP_THREADS) pm = fmaxf(pm, sp[i]);
  uint32_t lo = 0, hi = __float_as_uint(block_reduce_1024(pm, redf, fmax_op));
  while (lo < hi) {
    const uint32_t mid = lo + (hi - lo) / 2;
    const float t = __uint_as_float(mid);
    float above = 0.f;
    for (int i = tid; i < V; i += SMP_THREADS) above += sp[i] > t ? sp[i] : 0.f;
    if (block_reduce_1024(above, redf, fadd_op) < top_p) hi = mid;
    else lo = mid + 1;
  }
  const float t = __uint_as_float(lo);
  // inverse CDF over the nucleus in vocabulary order: thread `tid` owns the contiguous range [tid * per, +per)
  const int per = (V + SMP_THREADS - 1) / SMP_THREADS;
  const int b0 = min(tid * per, V), b1 = min(b0 + per, V);
  float own = 0.f;
  for (int i = b0; i < b1; ++i) own += sp[i] >= t ? sp[i] : 0.f;
  scan[tid] = own;
  __syncthreads();
  if (tid == 0) {  // exclusive prefix sums in order, then the target
    float run = 0.f;
    for (int w = 0; w < SMP_THREADS; ++w) {
      const float v = scan[w];
      scan[w] = run;
      run += v;
    }
    redf[0] = u * run;
    redu[0] = ~0ull;
  }
  __syncthreads();
  const float target = redf[0];
  float run = scan[tid];
  int pick = -1, last = -1;
  for (int i = b0; i < b1; ++i) {
    if (sp[i] < t) continue;
    last = i;
    run += sp[i];
    if (run > target) {
      pick = i;
      break;
    }
  }
  // the first thread (in vocabulary order) whose range crosses the target wins; rounding can leave the target
  // uncrossed, and then the last nucleus token is taken
  unsigned long long key = pick >= 0 ? static_cast<unsigned long long>(pick) : ~0ull;
  key = block_reduce_1024(key, redu, [](unsigned long long a, unsigned long long b) { return a < b ? a : b; });
  unsigned long long lastk = last >= 0 ? static_cast<unsigned long long>(last) : 0ull;
  lastk = block_reduce_1024(lastk, redu, [](unsigned long long a, unsigned long long b) { return a > b ? a : b; });
  if (tid == 0) *token = static_cast<int64_t>(key != ~0ull ? key : lastk);
}

}  // namespace uav

using namespace uav;

extern "C" {

uav_status_t uav_rmsnorm(const void* x, int64_t rows, int64_t C, int64_t ldx, const void* weight, float eps, void* out,
                         int64_t ldo, uav_stream_t stream) {
  UAV_REQUIRE(x && weight && out, "uav_rmsnorm: null pointer");
  UAV_REQUIRE(rows > 0 && rows <= INT32_MAX && C > 0 && C <= INT32_MAX && C % 8 == 0 && ldx % 8 == 0 && ldo % 8 == 0,
              "uav_rmsnorm: rows > 0, C % 8 == 0 and strides % 8 == 0 (got rows=%lld C=%lld)", (long long)rows,
              (long long)C);
  UAV_REQUIRE(eps >= 0.f, "uav_rmsnorm: eps must be >= 0");
  UAV_REQUIRE_ALIGNED16("uav_rmsnorm", x);
  UAV_REQUIRE_ALIGNED16("uav_rmsnorm", weight);
  UAV_REQUIRE_ALIGNED16("uav_rmsnorm", out);
  rmsnorm_kernel<<<(unsigned)rows, RMS_THREADS, 0, (cudaStream_t)stream>>>(
      (const __half*)x, ldx, (const __half*)weight, (int)C, eps, (__half*)out, ldo);
  UAV_LAUNCHED();
  return UAV_OK;
}

uav_status_t uav_rope_kv_append(void* qkv, int64_t ld_qkv, int64_t n, int heads, int head_dim, int64_t p0,
                                const float* cos_sin, int64_t positions, void* k_cache, void* v_cache, int64_t ld_kv,
                                int64_t cache_rows, uav_stream_t stream) {
  UAV_REQUIRE(qkv && cos_sin && k_cache && v_cache, "uav_rope_kv_append: null pointer");
  if (head_dim != 128) {
    set_last_error("uav_rope_kv_append: head_dim %d unsupported (128)", head_dim);
    return UAV_ERR_UNSUPPORTED;
  }
  UAV_REQUIRE(n > 0 && heads > 0 && p0 >= 0 && ld_qkv >= 3 * heads * 128 && ld_kv >= heads * 128,
              "uav_rope_kv_append: bad shape");
  UAV_REQUIRE(p0 + n <= positions && p0 + n <= cache_rows,
              "uav_rope_kv_append: positions [%lld, %lld) exceed the rotary table (%lld) or the cache (%lld)",
              (long long)p0, (long long)(p0 + n), (long long)positions, (long long)cache_rows);
  const int64_t items = n * heads * 64;
  rope_kv_append_kernel<<<stream_grid(items, 256, 8), 256, 0, (cudaStream_t)stream>>>(
      (__half*)qkv, ld_qkv, (int)n, heads, (int)p0, (const float2*)cos_sin, (__half*)k_cache, (__half*)v_cache, ld_kv);
  UAV_LAUNCHED();
  return UAV_OK;
}

uav_status_t uav_swiglu(const void* gate_up, int64_t ld_gu, int64_t rows, int64_t inter, void* out, int64_t ldo,
                        uav_stream_t stream) {
  UAV_REQUIRE(gate_up && out, "uav_swiglu: null pointer");
  UAV_REQUIRE(rows > 0 && inter > 0 && inter % 8 == 0 && inter <= INT32_MAX && ld_gu >= 2 * inter && ld_gu % 8 == 0 &&
                  ldo >= inter && ldo % 8 == 0,
              "uav_swiglu: bad shape (rows=%lld inter=%lld)", (long long)rows, (long long)inter);
  UAV_REQUIRE_ALIGNED16("uav_swiglu", gate_up);
  UAV_REQUIRE_ALIGNED16("uav_swiglu", out);
  swiglu_kernel<<<stream_grid(rows * (inter / 8), 256, 8), 256, 0, (cudaStream_t)stream>>>(
      (const __half*)gate_up, ld_gu, rows, (int)inter, (__half*)out, ldo);
  UAV_LAUNCHED();
  return UAV_OK;
}

uav_status_t uav_gemv(const void* w, int64_t N, int64_t K, const void* x, const void* residual, void* out, int out_dtype,
                      uav_stream_t stream) {
  UAV_REQUIRE(w && x && out, "uav_gemv: null pointer");
  UAV_REQUIRE(N > 0 && N <= INT32_MAX && K > 0 && K % 8 == 0 && K <= GEMV_MAX_K,
              "uav_gemv: N > 0 and K %% 8 == 0, K <= %d (got N=%lld K=%lld)", GEMV_MAX_K, (long long)N, (long long)K);
  UAV_REQUIRE(out_dtype == UAV_F16 || (out_dtype == UAV_F32 && !residual),
              "uav_gemv: out is fp16 (with an optional residual) or fp32");
  UAV_REQUIRE_ALIGNED16("uav_gemv", w);
  UAV_REQUIRE_ALIGNED16("uav_gemv", x);
  // warps per row: split K until the rows give every SM at least 48 warps (HBM needs many loads in flight per SM)
  const int64_t want_warps = static_cast<int64_t>(num_sms()) * 48;
  int S = 1;
  while (S < 8 && N * S < want_warps) S *= 2;
  const int rows_per_cta = (GEMV_THREADS / 32) / S;
  const int smem = (int)K * 2 + (GEMV_THREADS / 32) * 4;
  const int64_t ctas = (N + rows_per_cta - 1) / rows_per_cta;
  // resident CTAs: 64 KB of shared memory per SM is left to L1; spread the rows evenly over one wave
  int per_sm = 8;
  while (per_sm > 1 && per_sm * smem > 160 * 1024) --per_sm;
  const int64_t cap = static_cast<int64_t>(num_sms()) * per_sm;
  const int64_t waves = (ctas + cap - 1) / cap;
  const unsigned grid = (unsigned)((ctas + waves - 1) / waves);
  const uav_status_t st = opt_in_smem<gemv_kernel>(GEMV_MAX_K * 2 + (GEMV_THREADS / 32) * 4);
  if (st != UAV_OK) return st;
  gemv_kernel<<<grid, GEMV_THREADS, smem, (cudaStream_t)stream>>>((const __half*)w, (const __half*)x, (int)N, (int)K, S,
                                                                  (const __half*)residual, out,
                                                                  out_dtype == UAV_F32 ? 1 : 0);
  UAV_LAUNCHED();
  return UAV_OK;
}

size_t uav_attention_decode_workspace_bytes(int heads, int64_t L) {
  return static_cast<size_t>(heads) * ((L + DEC_CHUNK - 1) / DEC_CHUNK) * DEC_PART * sizeof(float);
}

uav_status_t uav_attention_decode(const void* q, const void* k_cache, const void* v_cache, int64_t ld_kv, int64_t L,
                                  int heads, int head_dim, float scale, void* out, void* workspace, size_t ws_bytes,
                                  uav_stream_t stream) {
  UAV_REQUIRE(q && k_cache && v_cache && out && workspace, "uav_attention_decode: null pointer");
  if (head_dim != 128) {
    set_last_error("uav_attention_decode: head_dim %d unsupported (128)", head_dim);
    return UAV_ERR_UNSUPPORTED;
  }
  UAV_REQUIRE(L > 0 && L <= INT32_MAX && heads > 0 && heads <= 65535 && ld_kv >= heads * 128 && ld_kv % 4 == 0,
              "uav_attention_decode: bad shape (L=%lld heads=%d)", (long long)L, heads);
  UAV_REQUIRE(scale > 0.f && scale < INFINITY, "uav_attention_decode: scale must be finite and > 0");
  UAV_REQUIRE(ws_bytes >= uav_attention_decode_workspace_bytes(heads, L), "uav_attention_decode: workspace too small");
  UAV_REQUIRE((reinterpret_cast<uintptr_t>(q) & 7) == 0 && (reinterpret_cast<uintptr_t>(k_cache) & 7) == 0 &&
                  (reinterpret_cast<uintptr_t>(v_cache) & 7) == 0,
              "uav_attention_decode: q and the caches must be 8-byte aligned");
  const int chunks = (int)((L + DEC_CHUNK - 1) / DEC_CHUNK);
  attn_decode_chunk_kernel<<<dim3((unsigned)chunks, (unsigned)heads), 128, 0, (cudaStream_t)stream>>>(
      (const __half*)q, (const __half*)k_cache, (const __half*)v_cache, ld_kv, (int)L, scale * 1.4426950408889634f,
      (float*)workspace);
  UAV_LAUNCHED();
  attn_decode_merge_kernel<<<(unsigned)heads, 128, 0, (cudaStream_t)stream>>>((const float*)workspace, chunks,
                                                                               (__half*)out);
  UAV_LAUNCHED();
  return UAV_OK;
}

uav_status_t uav_sample_top_p(const float* logits, int64_t V, float temperature, float top_p, float u, int64_t* token,
                              uav_stream_t stream) {
  UAV_REQUIRE(logits && token, "uav_sample_top_p: null pointer");
  UAV_REQUIRE(V > 0 && V <= SMP_MAX_V, "uav_sample_top_p: vocabulary of 1..%d tokens (got %lld)", SMP_MAX_V,
              (long long)V);
  UAV_REQUIRE(temperature >= 0.f && temperature < INFINITY, "uav_sample_top_p: temperature must be finite and >= 0");
  UAV_REQUIRE(top_p > 0.f && top_p <= 1.f, "uav_sample_top_p: top_p must be in (0, 1]");
  UAV_REQUIRE(u >= 0.f && u < 1.f, "uav_sample_top_p: u must be in [0, 1)");
  return launch_opted_in<sample_top_p_kernel>(dim3(1), SMP_THREADS, (int)(SMP_MAX_V * sizeof(float)),
                                              (cudaStream_t)stream, logits, (int)V, temperature, top_p, u, token);
}

}  // extern "C"
