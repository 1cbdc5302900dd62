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
// `batch` sequences at once: sequence b's rows start at qkv + b * qkv_bs and its cache at kc / vc + b * kv_bs.
// ---------------------------------------------------------------------------------------
__global__ void rope_kv_append_kernel(__half* __restrict__ qkv, int64_t ld_qkv, int64_t qkv_bs, int batch, int n,
                                      int heads, int p0, const float2* __restrict__ cos_sin, __half* __restrict__ kc,
                                      __half* __restrict__ vc, int64_t ld_kv, int64_t kv_bs) {
  const int64_t items = static_cast<int64_t>(batch) * n * heads * 64;
  const int C = heads * 128;
  UAV_GRID_STRIDE(t, items) {
    const int i = static_cast<int>(t & 63);
    const int64_t rh = t >> 6;
    const int64_t br = rh / heads;
    const int h = static_cast<int>(rh % heads), r = static_cast<int>(br % n), b = static_cast<int>(br / n);
    const float2 cs = cos_sin[static_cast<int64_t>(p0 + r) * 64 + i];
    __half* row = qkv + b * qkv_bs + r * ld_qkv + h * 128 + i;
    const int64_t krow = b * kv_bs + static_cast<int64_t>(p0 + r) * ld_kv + h * 128 + i;
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
// GEMV: y[r][N] = W[N][K] . x[r][K] for ROWS input rows, fp32 accumulation, W streamed once for all rows.  x is
// staged in shared memory.  A CTA of THREADS / 32 warps takes (THREADS / 32) / S weight rows at a time; the S warps of
// a weight row split K (split-K), each lane streams 16-byte chunks of the row with non-coherent, L1-bypassing loads,
// GEMV_UNROLL chunks in flight per lane, and applies each chunk to every input row.  The S x 32 partial sums of an
// output are combined in a fixed order (a butterfly in each warp, then the S warps in order), so results are
// deterministic, and each input row gets the same operations in the same order whatever ROWS and THREADS are: a row's
// result does not depend on the other rows of its batch.  Epilogue: fp16 out (optionally + fp16 residual, one
// rounding) or fp32 out.
// ---------------------------------------------------------------------------------------
constexpr int GEMV_THREADS = 256;        // one input row (uav_gemv)
constexpr int GEMV_ROWS_THREADS = 1024;  // 2..8 input rows: x fills up to 216 KB, so one CTA may be all an SM holds
constexpr int GEMV_UNROLL = 4;
constexpr int GEMV_MAX_K = 16384;
constexpr int GEMV_MAX_ROWS = 8;
constexpr int GEMV_ROWS_MAX_X = 8 * 13824;  // rows * K of x held in shared memory (216 KB: 8 rows of Llama-13B's down)

__device__ __forceinline__ uint4 ldg16_stream(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::256B.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

// acc[r] += w . x[r] over one 16-byte chunk (8 halves) for each input row r, in element order
template <int ROWS>
__device__ __forceinline__ void dot8_rows(const uint4& w, const uint4* __restrict__ sx, int chunks, float (&acc)[ROWS]) {
  const __half2* wh = reinterpret_cast<const __half2*>(&w);
  float2 a[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) a[e] = __half22float2(wh[e]);
#pragma unroll
  for (int r = 0; r < ROWS; ++r) {
    const uint4 x = sx[r * chunks];
    const __half2* xh = reinterpret_cast<const __half2*>(&x);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 b = __half22float2(xh[e]);
      acc[r] = fmaf(a[e].x, b.x, acc[r]);
      acc[r] = fmaf(a[e].y, b.y, acc[r]);
    }
  }
}

// x, residual: fp16 [ROWS][K] / [ROWS][N] dense; out [ROWS][N] dense
template <int ROWS, int THREADS>
__global__ void __launch_bounds__(THREADS, THREADS == GEMV_THREADS ? 0 : 1)
    gemv_kernel(const __half* __restrict__ w, const __half* __restrict__ x, int N, int K, int S,
                const __half* __restrict__ residual, void* __restrict__ out, int out_f32) {
  constexpr int WARPS = THREADS / 32;
  extern __shared__ __align__(16) uint8_t gemv_smem[];
  const uint4* sx = reinterpret_cast<const uint4*>(gemv_smem);                                // [ROWS][K / 8]
  float* red = reinterpret_cast<float*>(gemv_smem + static_cast<size_t>(ROWS) * K * 2);  // [ROWS][WARPS]
  const int chunks = K / 8;
  for (int c = threadIdx.x; c < ROWS * chunks; c += THREADS)
    reinterpret_cast<uint4*>(gemv_smem)[c] = ldg16(x + 8 * c);
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rows_per_cta = WARPS / S;
  const int part = warp % S;
  // the S warps of a row take interleaved 16-byte chunks: chunk c = (i * S + part) * 32 + lane
  const int stride = S * 32;
  for (int row0 = blockIdx.x * rows_per_cta; row0 < N; row0 += gridDim.x * rows_per_cta) {
    const int row = row0 + warp / S;
    float acc[ROWS];
#pragma unroll
    for (int r = 0; r < ROWS; ++r) acc[r] = 0.f;
    if (row < N) {
      const __half* wr = w + static_cast<int64_t>(row) * K;
      int c = part * 32 + lane;
      for (; c + (GEMV_UNROLL - 1) * stride < chunks; c += GEMV_UNROLL * stride) {
        uint4 wv[GEMV_UNROLL];
#pragma unroll
        for (int u = 0; u < GEMV_UNROLL; ++u) wv[u] = ldg16_stream(wr + 8 * (c + u * stride));
#pragma unroll
        for (int u = 0; u < GEMV_UNROLL; ++u) dot8_rows<ROWS>(wv[u], sx + c + u * stride, chunks, acc);
      }
      for (; c < chunks; c += stride) dot8_rows<ROWS>(ldg16_stream(wr + 8 * c), sx + c, chunks, acc);
    }
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) acc[r] += __shfl_xor_sync(0xffffffffu, acc[r], off);
      if (lane == 0) red[r * WARPS + warp] = acc[r];
    }
    __syncthreads();
    // thread t writes output (input row t / rows_per_cta, weight row row0 + t % rows_per_cta)
    const int slot = ROWS == 1 ? threadIdx.x : threadIdx.x % rows_per_cta;
    const int xr = ROWS == 1 ? 0 : threadIdx.x / rows_per_cta;
    if (slot < rows_per_cta && xr < ROWS && row0 + slot < N) {
      const int64_t o = static_cast<int64_t>(xr) * N + row0 + slot;
      float y = 0.f;
      for (int s = 0; s < S; ++s) y += red[xr * WARPS + slot * S + s];
      if (out_f32) {
        reinterpret_cast<float*>(out)[o] = y;
      } else {
        if (residual) y += __half2float(residual[o]);
        reinterpret_cast<__half*>(out)[o] = __float2half_rn(y);
      }
    }
    __syncthreads();
  }
}

template <int ROWS, int THREADS>
uav_status_t launch_gemv(const void* w, int64_t N, int64_t K, const void* x, const void* residual, void* out,
                         int out_dtype, cudaStream_t stream) {
  // warps per row: split K until the rows give every SM at least 48 warps (HBM needs many loads in flight per SM).
  // S depends on N only, so every row count runs the same split and combine.
  const int64_t want_warps = static_cast<int64_t>(num_sms()) * 48;
  int S = 1;
  while (S < 8 && N * S < want_warps) S *= 2;
  constexpr int WARPS = THREADS / 32;
  const int rows_per_cta = WARPS / S;
  const int smem = ROWS * (int)K * 2 + ROWS * WARPS * 4;
  const int64_t ctas = (N + rows_per_cta - 1) / rows_per_cta;
  // resident CTAs: 64 KB of shared memory per SM is left to L1; spread the rows evenly over one wave.  A CTA of
  // GEMV_ROWS_THREADS uses up to 64 registers per thread: one fits an SM.
  int per_sm = THREADS == GEMV_THREADS ? 8 : 1;
  while (per_sm > 1 && per_sm * smem > 160 * 1024) --per_sm;
  const int64_t cap = static_cast<int64_t>(num_sms()) * per_sm;
  const int64_t waves = (ctas + cap - 1) / cap;
  const unsigned grid = (unsigned)((ctas + waves - 1) / waves);
  constexpr int max_x = ROWS == 1 ? GEMV_MAX_K : GEMV_ROWS_MAX_X;
  const uav_status_t st = opt_in_smem<gemv_kernel<ROWS, THREADS>>(max_x * 2 + ROWS * WARPS * 4);
  if (st != UAV_OK) return st;
  gemv_kernel<ROWS, THREADS><<<grid, THREADS, smem, stream>>>((const __half*)w, (const __half*)x, (int)N, (int)K, S,
                                                              (const __half*)residual, out, out_dtype == UAV_F32 ? 1 : 0);
  UAV_LAUNCHED();
  return UAV_OK;
}

// ---------------------------------------------------------------------------------------
// Decode attention (flash-decoding): one query row per head against L cached keys, head_dim 128.  Stage 1: CTA (head,
// chunk of DEC_CHUNK keys), 4 warps, each warp a quarter of the chunk with an online softmax (lane = 4 of the 128 dims),
// the 4 warps merged in order -> (m, l, o[128]) of the chunk.  Stage 2: one CTA per head merges the chunks in order.
// Sequences of a batch (grid z of stage 1, grid y of stage 2) run the same CTAs on their own query row, cache and
// workspace slice: a sequence's result does not depend on the others.
// ---------------------------------------------------------------------------------------
constexpr int DEC_CHUNK = 64;
constexpr int DEC_PART = 2 + 128;  // m, l, o[128] (fp32) per (head, chunk)

// (128, 1): with the batch offsets, ptxas's default target of 40 registers spills; it takes 48, with no spills
__global__ void __launch_bounds__(128, 1)
    attn_decode_chunk_kernel(const __half* __restrict__ q, int64_t ldq, const __half* __restrict__ kc,
                             const __half* __restrict__ vc, int64_t ld_kv, int64_t kv_bs, int L, float scale_log2,
                             float* __restrict__ part) {
  __shared__ float sm[4][DEC_PART];
  const int h = blockIdx.y, chunk = blockIdx.x;
  q += blockIdx.z * ldq;
  const int64_t kv0 = blockIdx.z * kv_bs;  // this sequence's cache rows
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint2 qu = *reinterpret_cast<const uint2*>(q + h * 128 + 4 * lane);
  const __half2* qh = reinterpret_cast<const __half2*>(&qu);
  const float2 q01 = __half22float2(qh[0]), q23 = __half22float2(qh[1]);
  float m = -INFINITY, l = 0.f, o[4] = {0.f, 0.f, 0.f, 0.f};
  const int k0 = chunk * DEC_CHUNK + warp * (DEC_CHUNK / 4);
  const int k1 = min(k0 + DEC_CHUNK / 4, L);
  for (int j = k0; j < k1; ++j) {
    const int64_t off = kv0 + static_cast<int64_t>(j) * ld_kv + h * 128 + 4 * lane;
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
  float* pp = part + ((static_cast<int64_t>(blockIdx.z) * gridDim.y + h) * gridDim.x + chunk) * DEC_PART;
  if (threadIdx.x == 0) {
    pp[0] = M;
    pp[1] = Ls;
  }
  pp[2 + threadIdx.x] = Os;
}

__global__ void __launch_bounds__(128)
    attn_decode_merge_kernel(const float* __restrict__ part, int chunks, __half* __restrict__ out, int64_t ldo) {
  const int h = blockIdx.x;
  part += static_cast<int64_t>(blockIdx.y) * gridDim.x * chunks * DEC_PART;
  out += blockIdx.y * ldo;
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

uav_status_t launch_attention_decode(const void* q, int64_t ldq, const void* k_cache,
                                     const void* v_cache, int64_t ld_kv, int64_t kv_bs, int64_t batch, int64_t L,
                                     int heads, float scale, void* out, int64_t ldo, void* workspace,
                                     cudaStream_t stream) {
  const int chunks = (int)((L + DEC_CHUNK - 1) / DEC_CHUNK);
  attn_decode_chunk_kernel<<<dim3((unsigned)chunks, (unsigned)heads, (unsigned)batch), 128, 0, stream>>>(
      (const __half*)q, ldq, (const __half*)k_cache, (const __half*)v_cache, ld_kv, kv_bs, (int)L,
      scale * 1.4426950408889634f, (float*)workspace);
  UAV_LAUNCHED();
  attn_decode_merge_kernel<<<dim3((unsigned)heads, (unsigned)batch), 128, 0, stream>>>((const float*)workspace, chunks,
                                                                                      (__half*)out, ldo);
  UAV_LAUNCHED();
  return UAV_OK;
}

// ---------------------------------------------------------------------------------------
// Top-p sampling (transformers TemperatureLogitsWarper + TopPLogitsWarper + multinomial), one CTA of 1024 threads.
// p = softmax(logits / T) in fp32, held in shared memory.  TopPLogitsWarper drops the ascending-sorted prefix whose
// cumulative mass is <= 1 - top_p and keeps at least one token; for distinct probabilities that keeps exactly the
// tokens whose strictly more probable tokens have mass < top_p.  That mass is monotone in p, so the smallest kept
// probability t is found by bisecting its fp32 bit pattern (31 block reductions, no sort); the nucleus is {p >= t}.
// The token is the inverse CDF of the nucleus in vocabulary order at u * (nucleus mass), u in [0, 1) supplied by the
// caller.  temperature == 0 returns the argmax (first index on ties).  Batched: CTA b samples logits row b with
// uniform u.u[b] into token[b], with the one-row arithmetic.
// ---------------------------------------------------------------------------------------
constexpr int SMP_THREADS = 1024;
constexpr int SMP_MAX_V = 49152;
constexpr int SMP_MAX_ROWS = 8;

struct SampleUniforms {  // passed by value: no host-to-device copy per step
  float u[SMP_MAX_ROWS];
};

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
    sample_top_p_kernel(const float* __restrict__ logits, int64_t ld_logits, int V, float temperature, float top_p,
                        SampleUniforms us, int64_t* __restrict__ token) {
  extern __shared__ __align__(16) float sp[];  // [V] probabilities
  __shared__ float redf[32];
  __shared__ unsigned long long redu[32];
  __shared__ float scan[SMP_THREADS];
  const int tid = threadIdx.x;
  logits += blockIdx.x * ld_logits;
  token += blockIdx.x;
  const float u = us.u[blockIdx.x];
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
      (__half*)qkv, ld_qkv, 0, 1, (int)n, heads, (int)p0, (const float2*)cos_sin, (__half*)k_cache, (__half*)v_cache,
      ld_kv, 0);
  UAV_LAUNCHED();
  return UAV_OK;
}

uav_status_t uav_rope_kv_append_batched(void* qkv, int64_t ld_qkv, int64_t qkv_batch_stride, int64_t batch, int64_t n,
                                        int heads, int head_dim, int64_t p0, const float* cos_sin, int64_t positions,
                                        void* k_cache, void* v_cache, int64_t ld_kv, int64_t kv_batch_stride,
                                        int64_t cache_rows, uav_stream_t stream) {
  UAV_REQUIRE(qkv && cos_sin && k_cache && v_cache, "uav_rope_kv_append_batched: null pointer");
  if (head_dim != 128) {
    set_last_error("uav_rope_kv_append_batched: head_dim %d unsupported (128)", head_dim);
    return UAV_ERR_UNSUPPORTED;
  }
  UAV_REQUIRE(batch > 0 && batch <= 65535 && n > 0 && n <= INT32_MAX && heads > 0 && p0 >= 0 &&
                  ld_qkv >= 3 * heads * 128 && ld_kv >= heads * 128,
              "uav_rope_kv_append_batched: bad shape (batch=%lld n=%lld heads=%d)", (long long)batch, (long long)n,
              heads);
  UAV_REQUIRE(p0 + n <= positions && p0 + n <= cache_rows && p0 + n <= INT32_MAX,
              "uav_rope_kv_append_batched: positions [%lld, %lld) exceed the rotary table (%lld) or the cache (%lld)",
              (long long)p0, (long long)(p0 + n), (long long)positions, (long long)cache_rows);
  // sequences must not overlap: each one's rows and cache lie between its batch stride and the next one's
  UAV_REQUIRE(batch == 1 || (qkv_batch_stride >= n * ld_qkv && kv_batch_stride >= cache_rows * ld_kv),
              "uav_rope_kv_append_batched: batch strides (%lld, %lld) overlap the rows (%lld x %lld, %lld x %lld)",
              (long long)qkv_batch_stride, (long long)kv_batch_stride, (long long)n, (long long)ld_qkv,
              (long long)cache_rows, (long long)ld_kv);
  const int64_t items = batch * n * heads * 64;
  rope_kv_append_kernel<<<stream_grid(items, 256, 8), 256, 0, (cudaStream_t)stream>>>(
      (__half*)qkv, ld_qkv, qkv_batch_stride, (int)batch, (int)n, heads, (int)p0, (const float2*)cos_sin,
      (__half*)k_cache, (__half*)v_cache, ld_kv, kv_batch_stride);
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
  return launch_gemv<1, GEMV_THREADS>(w, N, K, x, residual, out, out_dtype, (cudaStream_t)stream);
}

uav_status_t uav_gemv_rows(const void* w, int64_t N, int64_t K, const void* x, int64_t rows, const void* residual,
                           void* out, int out_dtype, uav_stream_t stream) {
  UAV_REQUIRE(w && x && out, "uav_gemv_rows: null pointer");
  UAV_REQUIRE(rows >= 1 && rows <= GEMV_MAX_ROWS, "uav_gemv_rows: rows must be in 1..%d (got %lld)", GEMV_MAX_ROWS,
              (long long)rows);
  UAV_REQUIRE(N > 0 && N <= INT32_MAX / GEMV_MAX_ROWS && K > 0 && K % 8 == 0 && K <= GEMV_MAX_K &&
                  (rows == 1 || rows * K <= GEMV_ROWS_MAX_X),
              "uav_gemv_rows: N > 0, K %% 8 == 0, K <= %d and rows * K <= %d (got N=%lld K=%lld rows=%lld)", GEMV_MAX_K,
              GEMV_ROWS_MAX_X, (long long)N, (long long)K, (long long)rows);
  UAV_REQUIRE(out_dtype == UAV_F16 || (out_dtype == UAV_F32 && !residual),
              "uav_gemv_rows: out is fp16 (with an optional residual) or fp32");
  UAV_REQUIRE_ALIGNED16("uav_gemv_rows", w);
  UAV_REQUIRE_ALIGNED16("uav_gemv_rows", x);
  const cudaStream_t s = (cudaStream_t)stream;
  switch (rows) {
    case 1: return launch_gemv<1, GEMV_THREADS>(w, N, K, x, residual, out, out_dtype, s);
    case 2: return launch_gemv<2, GEMV_ROWS_THREADS>(w, N, K, x, residual, out, out_dtype, s);
    case 3: return launch_gemv<3, GEMV_ROWS_THREADS>(w, N, K, x, residual, out, out_dtype, s);
    case 4: return launch_gemv<4, GEMV_ROWS_THREADS>(w, N, K, x, residual, out, out_dtype, s);
    case 5: return launch_gemv<5, GEMV_ROWS_THREADS>(w, N, K, x, residual, out, out_dtype, s);
    case 6: return launch_gemv<6, GEMV_ROWS_THREADS>(w, N, K, x, residual, out, out_dtype, s);
    case 7: return launch_gemv<7, GEMV_ROWS_THREADS>(w, N, K, x, residual, out, out_dtype, s);
    default: return launch_gemv<8, GEMV_ROWS_THREADS>(w, N, K, x, residual, out, out_dtype, s);
  }
}

size_t uav_attention_decode_workspace_bytes(int heads, int64_t L) {
  return static_cast<size_t>(heads) * ((L + DEC_CHUNK - 1) / DEC_CHUNK) * DEC_PART * sizeof(float);
}

size_t uav_attention_decode_batched_workspace_bytes(int64_t batch, int heads, int64_t L) {
  return static_cast<size_t>(batch) * uav_attention_decode_workspace_bytes(heads, L);
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
  return launch_attention_decode(q, 0, k_cache, v_cache, ld_kv, 0, 1, L, heads, scale, out, 0,
                                 workspace, (cudaStream_t)stream);
}

uav_status_t uav_attention_decode_batched(const void* q, int64_t ldq, const void* k_cache, const void* v_cache,
                                          int64_t ld_kv, int64_t kv_batch_stride, int64_t batch, int64_t L, int heads,
                                          int head_dim, float scale, void* out, int64_t ldo, void* workspace,
                                          size_t ws_bytes, uav_stream_t stream) {
  UAV_REQUIRE(q && k_cache && v_cache && out && workspace, "uav_attention_decode_batched: null pointer");
  if (head_dim != 128) {
    set_last_error("uav_attention_decode_batched: head_dim %d unsupported (128)", head_dim);
    return UAV_ERR_UNSUPPORTED;
  }
  UAV_REQUIRE(batch > 0 && batch <= 65535 && L > 0 && L <= INT32_MAX && heads > 0 && heads <= 65535 &&
                  ld_kv >= heads * 128 && ld_kv % 4 == 0,
              "uav_attention_decode_batched: bad shape (batch=%lld L=%lld heads=%d)", (long long)batch, (long long)L,
              heads);
  UAV_REQUIRE(batch == 1 || (ldq >= heads * 128 && ldq % 4 == 0 && ldo >= heads * 128 &&
                             kv_batch_stride >= L * ld_kv && kv_batch_stride % 4 == 0),
              "uav_attention_decode_batched: strides ldq=%lld ldo=%lld (>= heads * 128, ldq %% 4 == 0) and "
              "kv_batch_stride=%lld (>= L * ld_kv, %% 4 == 0)",
              (long long)ldq, (long long)ldo, (long long)kv_batch_stride);
  UAV_REQUIRE(scale > 0.f && scale < INFINITY, "uav_attention_decode_batched: scale must be finite and > 0");
  UAV_REQUIRE(ws_bytes >= uav_attention_decode_batched_workspace_bytes(batch, heads, L),
              "uav_attention_decode_batched: workspace too small");
  UAV_REQUIRE((reinterpret_cast<uintptr_t>(q) & 7) == 0 && (reinterpret_cast<uintptr_t>(k_cache) & 7) == 0 &&
                  (reinterpret_cast<uintptr_t>(v_cache) & 7) == 0,
              "uav_attention_decode_batched: q and the caches must be 8-byte aligned");
  return launch_attention_decode(q, ldq, k_cache, v_cache, ld_kv, kv_batch_stride,
                                 batch, L, heads, scale, out, ldo, workspace, (cudaStream_t)stream);
}

uav_status_t uav_sample_top_p(const float* logits, int64_t V, float temperature, float top_p, float u, int64_t* token,
                              uav_stream_t stream) {
  UAV_REQUIRE(logits && token, "uav_sample_top_p: null pointer");
  UAV_REQUIRE(V > 0 && V <= SMP_MAX_V, "uav_sample_top_p: vocabulary of 1..%d tokens (got %lld)", SMP_MAX_V,
              (long long)V);
  UAV_REQUIRE(temperature >= 0.f && temperature < INFINITY, "uav_sample_top_p: temperature must be finite and >= 0");
  UAV_REQUIRE(top_p > 0.f && top_p <= 1.f, "uav_sample_top_p: top_p must be in (0, 1]");
  UAV_REQUIRE(u >= 0.f && u < 1.f, "uav_sample_top_p: u must be in [0, 1)");
  SampleUniforms us{};
  us.u[0] = u;
  return launch_opted_in<sample_top_p_kernel>(dim3(1), SMP_THREADS, (int)(SMP_MAX_V * sizeof(float)),
                                              (cudaStream_t)stream, logits, (int64_t)0, (int)V, temperature, top_p, us,
                                              token);
}

uav_status_t uav_sample_top_p_batched(const float* logits, int64_t ld_logits, int64_t rows, int64_t V,
                                      float temperature, float top_p, const float* u, int64_t* tokens,
                                      uav_stream_t stream) {
  UAV_REQUIRE(logits && u && tokens, "uav_sample_top_p_batched: null pointer");
  UAV_REQUIRE(rows >= 1 && rows <= SMP_MAX_ROWS, "uav_sample_top_p_batched: rows must be in 1..%d (got %lld)",
              SMP_MAX_ROWS, (long long)rows);
  UAV_REQUIRE(V > 0 && V <= SMP_MAX_V && (rows == 1 || ld_logits >= V),
              "uav_sample_top_p_batched: vocabulary of 1..%d tokens, ld_logits >= V (got V=%lld ld=%lld)", SMP_MAX_V,
              (long long)V, (long long)ld_logits);
  UAV_REQUIRE(temperature >= 0.f && temperature < INFINITY,
              "uav_sample_top_p_batched: temperature must be finite and >= 0");
  UAV_REQUIRE(top_p > 0.f && top_p <= 1.f, "uav_sample_top_p_batched: top_p must be in (0, 1]");
  SampleUniforms us{};
  for (int64_t r = 0; r < rows; ++r) {
    UAV_REQUIRE(u[r] >= 0.f && u[r] < 1.f, "uav_sample_top_p_batched: u[%lld] must be in [0, 1)", (long long)r);
    us.u[r] = u[r];
  }
  return launch_opted_in<sample_top_p_kernel>(dim3((unsigned)rows), SMP_THREADS, (int)(SMP_MAX_V * sizeof(float)),
                                              (cudaStream_t)stream, logits, ld_logits, (int)V, temperature, top_p, us,
                                              tokens);
}

}  // extern "C"
