// llava_int8.cu — weight-only int8 (W8A16) decoder Linears of the LLaVA captioner (llava.py, weights="int8"): the
// row-wise quantization applied while the checkpoint is read, the dequantization that feeds the prefill GEMMs, and the
// int8 weight stream of every decoded token.
//
// An int8 decode step reads half the bytes of an fp16 one.  The fp16 GEMV (llava.cu) does one FFMA per weight and
// input row; at 8 rows it is issue-bound, and a 16-byte int8 chunk holds twice the weights of an fp16 one.  So the
// int8 GEMV converts its weights to fp16 in registers (exact: |q| <= 127) and hands them to mma.sync as the A operand,
// with the <= 8 input rows as the MMA's 8 columns: 16 weights x 8 rows per MMA.
#include "uav_common.cuh"
#include "../../include/uav_b200_int8.h"

namespace uav {

constexpr int Q8_MAX_K = 16384;
constexpr int Q8_MAX_ROWS = 8;
constexpr int Q8_MAX_X = 8 * 13824;  // rows * K of x in shared memory, as uav_gemv_rows
constexpr int Q8_THREADS = 256;
constexpr int Q8_WARPS = Q8_THREADS / 32;
constexpr int Q8_UNROLL = 4;   // 64-column blocks per warp per step: 2 x Q8_UNROLL 16-byte loads in flight per lane
constexpr int Q8_XPAD = 8;     // halves of padding per x row in shared memory: B-fragment loads are conflict-free
constexpr int Q8_RED = Q8_WARPS * 16 * 8;  // fp32 partial sums [warp][16 weight rows][8 input rows]

// ---------------------------------------------------------------------------------------
// quantize: one warp per row, 8 halves per lane per step; the max is exact in any order
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
    quantize_rows_int8_kernel(const __half* __restrict__ w, int N, int K, int64_t ldw, int8_t* __restrict__ q,
                              float* __restrict__ absmax) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = static_cast<int64_t>(gridDim.x) * (blockDim.x >> 5);
  for (int64_t n = static_cast<int64_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5); n < N; n += warps) {
    const __half* wr = w + n * ldw;
    float m = 0.f;
    for (int c = lane * 8; c < K; c += 256) {
      const uint4 u = ldg16(wr + c);
      const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = __half22float2(h[e]);
        m = fmaxf(m, fmaxf(fabsf(f.x), fabsf(f.y)));
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
    if (lane == 0) absmax[n] = m;
    int8_t* qr = q + n * K;
    for (int c = lane * 8; c < K; c += 256) {
      const uint4 u = ldg16(wr + c);
      const __half2* h = reinterpret_cast<const __half2*>(&u);
      uint32_t packed[2] = {0u, 0u};
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float2 f = __half22float2(h[e / 2]);
        const float v = (e & 1) ? f.y : f.x;
        // (v * 127) is exact in fp32; the quotient is IEEE-rounded, then rounded half to even
        const int qi = m == 0.f ? 0 : __float2int_rn(__fdiv_rn(v * 127.f, m));
        packed[e / 4] |= static_cast<uint32_t>(qi & 0xff) << (8 * (e & 3));
      }
      *reinterpret_cast<uint2*>(qr + c) = make_uint2(packed[0], packed[1]);
    }
  }
}

// ---------------------------------------------------------------------------------------
// dequantize: 16 weights per thread, two 16-byte stores
// ---------------------------------------------------------------------------------------
__global__ void dequantize_rows_int8_kernel(const int8_t* __restrict__ q, const float* __restrict__ absmax, int64_t N,
                                            int K, __half* __restrict__ out) {
  const int per_row = K / 16;
  UAV_GRID_STRIDE(t, N * per_row) {
    const int64_t n = t / per_row;
    const uint4 u = ldg16(q + 16 * t);
    const int8_t* b = reinterpret_cast<const int8_t*>(&u);
    const float s = absmax[n];
    uint4 o[2];
    uint32_t* ow = reinterpret_cast<uint32_t*>(o);
#pragma unroll
    for (int e = 0; e < 8; ++e)
      ow[e] = pack_half2_rn(__fdiv_rn(static_cast<float>(b[2 * e]) * s, 127.f),
                            __fdiv_rn(static_cast<float>(b[2 * e + 1]) * s, 127.f));
    stg16(out + 16 * t, o[0]);
    stg16(out + 16 * t + 8, o[1]);
  }
}

// ---------------------------------------------------------------------------------------
// GEMV on int8 weights with mma.sync.m16n8k16 (fp16 in, fp32 accumulate).
//
// A warp owns a tile of 16 weight rows; lane (g = lane / 4, t = lane % 4) loads the 16 bytes at columns
// [64 b + 16 t, +16) of rows g and g + 8 for each 64-column block b it takes.  Those 16 columns feed 4 MMAs: in MMA j
// the lane's A k-slots (2t, 2t+1, 2t+8, 2t+9) hold columns 64 b + 16 t + 4 j + (0, 1, 2, 3), and the B fragment of
// column g (input row g) takes x[g] at the same four columns, so each MMA sums 16 distinct columns of the block.
// Input rows >= rows are zero columns.  An output element's sum depends only on its own weight row and input row
// (MMA columns are independent), and the k-order is fixed by N and K: a row's result is the same in every batch.
//
// int8 -> fp16 without a convert per element: q ^ 0x80 = q + 128 is a byte u; the fp16 with bits 0x64uu is 1024 + u,
// exactly, so one PRMT builds a half2 of (1024 + u0, 1024 + u1) and one HSUB2 of 1152 gives (q0, q1).
//
// The S warps of a tile split its blocks: warp part p takes blocks [U (p + i S), U (p + i S) + U) for i = 0, 1, ...
// (256 contiguous bytes per row per step); the S partial sums are combined in order p = 0 .. S - 1 in shared memory.
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ void q8_to_half2x2(uint32_t word, uint32_t& lo, uint32_t& hi) {
  const uint32_t u = word ^ 0x80808080u;
  const uint32_t magic = 0x64646464u, bias = 0x64806480u;  // bias: half2 (1152, 1152)
  uint32_t a, b;
  asm("prmt.b32 %0, %1, %2, 0x5140;" : "=r"(a) : "r"(u), "r"(magic));  // (1024 + u0, 1024 + u1)
  asm("prmt.b32 %0, %1, %2, 0x7362;" : "=r"(b) : "r"(u), "r"(magic));  // (1024 + u2, 1024 + u3)
  asm("sub.f16x2 %0, %1, %2;" : "=r"(lo) : "r"(a), "r"(bias));
  asm("sub.f16x2 %0, %1, %2;" : "=r"(hi) : "r"(b), "r"(bias));
}

// acc += the 16 x 8 product of one 64-column block: w0 / w1 = the lane's 16 bytes of rows g / g + 8, xb = its 16
// halves of x[g] at the same columns (zero for g >= rows).  The block's 4 MMAs accumulate from zero and the block
// sum is added with an IEEE fp32 add: the tensor core's own accumulation only ever spans 64 products.
__device__ __forceinline__ void q8_block_mma(float (&acc)[4], const uint4& w0, const uint4& w1, const uint4 (&xb)[2]) {
  const uint32_t* r0 = reinterpret_cast<const uint32_t*>(&w0);
  const uint32_t* r1 = reinterpret_cast<const uint32_t*>(&w1);
  const uint32_t* xw = reinterpret_cast<const uint32_t*>(xb);
  float blk[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    uint32_t a[4];
    q8_to_half2x2(r0[j], a[0], a[2]);  // row g:     k-slots (2t, 2t+1) and (2t+8, 2t+9)
    q8_to_half2x2(r1[j], a[1], a[3]);  // row g + 8: the same k-slots
    mma16816(blk, a, xw[2 * j], xw[2 * j + 1]);
  }
#pragma unroll
  for (int e = 0; e < 4; ++e) acc[e] += blk[e];
}

__global__ void __launch_bounds__(Q8_THREADS, 2)
    gemv_rows_int8_kernel(const int8_t* __restrict__ q, const float* __restrict__ absmax, int N, int K,
                          const __half* __restrict__ x, int rows, int S, const __half* __restrict__ residual,
                          void* __restrict__ out, int out_f32) {
  extern __shared__ __align__(16) uint8_t q8_smem[];
  const int ldx = K + Q8_XPAD;
  __half* sx = reinterpret_cast<__half*>(q8_smem);                                        // [rows][ldx]
  float* red = reinterpret_cast<float*>(q8_smem + static_cast<size_t>(rows) * ldx * 2);  // [Q8_WARPS][16][8]
  const int xchunks = K / 8;
  for (int c = threadIdx.x; c < rows * xchunks; c += Q8_THREADS) {
    const int r = c / xchunks, k8 = c % xchunks;
    stg16(sx + r * ldx + 8 * k8, ldg16(x + static_cast<int64_t>(r) * K + 8 * k8));
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int tiles_per_cta = Q8_WARPS / S;
  const int part = warp % S;
  const int blocks = (K + 63) / 64, kchunks = K / 16;
  const __half* xg = sx + (g < rows ? g : 0) * ldx + 16 * t;
  const uint4 zero_w = make_uint4(0x80808080u, 0x80808080u, 0x80808080u, 0x80808080u);  // q = 0
  const int tiles = (N + 15) / 16;
  for (int tile0 = blockIdx.x * tiles_per_cta; tile0 < tiles; tile0 += gridDim.x * tiles_per_cta) {
    const int row0 = (tile0 + warp / S) * 16;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    if (row0 < N) {
      const int8_t* w0 = q + static_cast<int64_t>(min(row0 + g, N - 1)) * K + 16 * t;
      const int8_t* w1 = q + static_cast<int64_t>(min(row0 + g + 8, N - 1)) * K + 16 * t;
      const bool ok0 = row0 + g < N, ok1 = row0 + g + 8 < N;
      for (int b0 = part * Q8_UNROLL; b0 < blocks; b0 += S * Q8_UNROLL) {
        uint4 wa[Q8_UNROLL], wb[Q8_UNROLL];
#pragma unroll
        for (int u = 0; u < Q8_UNROLL; ++u) {
          const int c = (b0 + u) * 4 + t;  // this lane's 16-column chunk
          const bool in = c < kchunks;
          wa[u] = in && ok0 ? ldg16_stream(w0 + 64 * (b0 + u)) : zero_w;
          wb[u] = in && ok1 ? ldg16_stream(w1 + 64 * (b0 + u)) : zero_w;
        }
#pragma unroll
        for (int u = 0; u < Q8_UNROLL; ++u) {
          if (b0 + u >= blocks) break;  // warp-uniform
          const int c = (b0 + u) * 4 + t;
          uint4 xb[2] = {make_uint4(0u, 0u, 0u, 0u), make_uint4(0u, 0u, 0u, 0u)};
          if (g < rows && c < kchunks) {
            xb[0] = *reinterpret_cast<const uint4*>(xg + 64 * (b0 + u));
            xb[1] = *reinterpret_cast<const uint4*>(xg + 64 * (b0 + u) + 8);
          }
          q8_block_mma(acc, wa[u], wb[u], xb);
        }
      }
    }
    // acc: (weight row g, input rows 2t, 2t+1) and (weight row g + 8, the same input rows)
    float* rw = red + warp * 128;
    rw[g * 8 + 2 * t] = acc[0];
    rw[g * 8 + 2 * t + 1] = acc[1];
    rw[(g + 8) * 8 + 2 * t] = acc[2];
    rw[(g + 8) * 8 + 2 * t + 1] = acc[3];
    __syncthreads();
    // output i of the CTA: input row i / (16 tiles_per_cta), weight row tile0 * 16 + i % (16 tiles_per_cta)
    const int per_xr = 16 * tiles_per_cta;
    for (int i = threadIdx.x; i < rows * per_xr; i += Q8_THREADS) {
      const int xr = i / per_xr, slot = i % per_xr;
      const int n = tile0 * 16 + slot;
      if (n >= N) continue;
      const int tl = slot / 16, m = slot % 16;
      float y = 0.f;
      for (int s = 0; s < S; ++s) y += red[(tl * S + s) * 128 + m * 8 + xr];
      y *= __fdiv_rn(absmax[n], 127.f);
      const int64_t o = static_cast<int64_t>(xr) * N + n;
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

}  // namespace uav

using namespace uav;

extern "C" {

uav_status_t uav_quantize_rows_int8(const void* w, int64_t N, int64_t K, int64_t ldw, void* q, float* absmax,
                                    uav_stream_t stream) {
  UAV_REQUIRE(w && q && absmax, "uav_quantize_rows_int8: null pointer");
  UAV_REQUIRE(N > 0 && N <= INT32_MAX && K > 0 && K % 16 == 0 && K <= INT32_MAX && ldw >= K && ldw % 8 == 0,
              "uav_quantize_rows_int8: N > 0, K %% 16 == 0, ldw >= K and ldw %% 8 == 0 (got N=%lld K=%lld ldw=%lld)",
              (long long)N, (long long)K, (long long)ldw);
  UAV_REQUIRE_ALIGNED16("uav_quantize_rows_int8", w);
  UAV_REQUIRE_ALIGNED16("uav_quantize_rows_int8", q);
  UAV_REQUIRE((reinterpret_cast<uintptr_t>(absmax) & 3) == 0, "uav_quantize_rows_int8: absmax must be 4-byte aligned");
  quantize_rows_int8_kernel<<<stream_grid(N, 8, 8), 256, 0, (cudaStream_t)stream>>>(
      (const __half*)w, (int)N, (int)K, ldw, (int8_t*)q, absmax);
  UAV_LAUNCHED();
  return UAV_OK;
}

uav_status_t uav_dequantize_rows_int8(const void* q, const float* absmax, int64_t N, int64_t K, void* out,
                                      uav_stream_t stream) {
  UAV_REQUIRE(q && absmax && out, "uav_dequantize_rows_int8: null pointer");
  UAV_REQUIRE(N > 0 && K > 0 && K % 16 == 0 && K <= INT32_MAX,
              "uav_dequantize_rows_int8: N > 0 and K %% 16 == 0 (got N=%lld K=%lld)", (long long)N, (long long)K);
  UAV_REQUIRE_ALIGNED16("uav_dequantize_rows_int8", q);
  UAV_REQUIRE_ALIGNED16("uav_dequantize_rows_int8", out);
  UAV_REQUIRE((reinterpret_cast<uintptr_t>(absmax) & 3) == 0, "uav_dequantize_rows_int8: absmax must be 4-byte aligned");
  dequantize_rows_int8_kernel<<<stream_grid(N * (K / 16), 256, 8), 256, 0, (cudaStream_t)stream>>>(
      (const int8_t*)q, absmax, N, (int)K, (__half*)out);
  UAV_LAUNCHED();
  return UAV_OK;
}

uav_status_t uav_gemv_rows_int8(const void* q, const float* absmax, int64_t N, int64_t K, const void* x, int64_t rows,
                                const void* residual, void* out, int out_dtype, uav_stream_t stream) {
  UAV_REQUIRE(q && absmax && x && out, "uav_gemv_rows_int8: null pointer");
  UAV_REQUIRE(rows >= 1 && rows <= Q8_MAX_ROWS, "uav_gemv_rows_int8: rows must be in 1..%d (got %lld)", Q8_MAX_ROWS,
              (long long)rows);
  UAV_REQUIRE(N > 0 && N <= INT32_MAX / Q8_MAX_ROWS && K > 0 && K % 16 == 0 && K <= Q8_MAX_K && rows * K <= Q8_MAX_X,
              "uav_gemv_rows_int8: N > 0, K %% 16 == 0, K <= %d and rows * K <= %d (got N=%lld K=%lld rows=%lld)",
              Q8_MAX_K, Q8_MAX_X, (long long)N, (long long)K, (long long)rows);
  UAV_REQUIRE(out_dtype == UAV_F16 || (out_dtype == UAV_F32 && !residual),
              "uav_gemv_rows_int8: out is fp16 (with an optional residual) or fp32");
  UAV_REQUIRE_ALIGNED16("uav_gemv_rows_int8", q);
  UAV_REQUIRE_ALIGNED16("uav_gemv_rows_int8", x);
  UAV_REQUIRE((reinterpret_cast<uintptr_t>(absmax) & 3) == 0, "uav_gemv_rows_int8: absmax must be 4-byte aligned");
  UAV_REQUIRE((reinterpret_cast<uintptr_t>(out) & (out_dtype == UAV_F32 ? 3 : 1)) == 0 &&
                  (reinterpret_cast<uintptr_t>(residual) & 1) == 0,
              "uav_gemv_rows_int8: out and residual must be aligned to their element size");
  // warps per 16-row tile: split K until the tiles give every SM 16 warps (two CTAs, each lane with 8 16-byte loads in
  // flight).  S depends on N only, so every row count runs the same split and combine.
  const int64_t tiles = (N + 15) / 16;
  const int64_t want_warps = static_cast<int64_t>(num_sms()) * 2 * Q8_WARPS;
  int S = 1;
  while (S < Q8_WARPS && tiles * S < want_warps) S *= 2;
  const int tiles_per_cta = Q8_WARPS / S;
  const int smem = (int)(rows * (K + Q8_XPAD) * 2) + Q8_RED * 4;
  const int64_t ctas = (tiles + tiles_per_cta - 1) / tiles_per_cta;
  int per_sm = 2;  // __launch_bounds__(Q8_THREADS, 2) (90 registers, no spills); 64 KB of shared memory per SM is left to L1
  while (per_sm > 1 && per_sm * smem > 160 * 1024) --per_sm;
  const int64_t cap = static_cast<int64_t>(num_sms()) * per_sm;
  const int64_t waves = (ctas + cap - 1) / cap;
  const unsigned grid = (unsigned)((ctas + waves - 1) / waves);
  constexpr int max_smem = (Q8_MAX_X + Q8_MAX_ROWS * Q8_XPAD) * 2 + Q8_RED * 4;
  const uav_status_t st = opt_in_smem<gemv_rows_int8_kernel>(max_smem);
  if (st != UAV_OK) return st;
  gemv_rows_int8_kernel<<<grid, Q8_THREADS, smem, (cudaStream_t)stream>>>(
      (const int8_t*)q, absmax, (int)N, (int)K, (const __half*)x, (int)rows, S, (const __half*)residual, out,
      out_dtype == UAV_F32 ? 1 : 0);
  UAV_LAUNCHED();
  return UAV_OK;
}

}  // extern "C"
