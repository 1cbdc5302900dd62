// clip_text.cu — the one kernel the CLIP text encoder needs besides the shared GEMM / LayerNorm kernels
// (SURVEY.md §8f rank 3; reference: `self.text_encoder(...)` in pipeline_upscale_a_video.py:239-245, a transformers
// CLIPTextModel): causal self-attention over the 77-token prompt.
#include "uav_common.cuh"

// ---------------------------------------------------------------------------------------
// CLIP text encoder (SURVEY.md §8f rank 3): causal self-attention over a short sequence (77 tokens).  Longer sequences
// with head_dim 128 (the LLaVA decoder's prefill) run on the causal wgmma kernel of attention_tc.cu.  One CTA per (batch, head): K and V of the head in shared memory, one warp per query row,
// lane j scores key j (j <= i), fp32 softmax, then lanes own output columns.  n <= 128, d <= 128, d % 2 == 0.
// (transformers CLIPAttention with the causal mask of CLIPTextTransformer; run once per prompt: clarity over speed.)
// ---------------------------------------------------------------------------------------
namespace uav {
constexpr int CA_MAX_N = 128;

// dynamic shared memory of a launch over n tokens of head_dim d
constexpr size_t ca_smem_bytes(int64_t n, int64_t d) {
  return n * (d + 2) * 2 + n * d * 2 + 4 * CA_MAX_N * sizeof(float) + 4 * d * sizeof(float);
}

__global__ void __launch_bounds__(128)
    causal_attn_kernel(const __half* __restrict__ q, const __half* __restrict__ k, const __half* __restrict__ v,
                       __half* __restrict__ o, int n, int d, int64_t ldq, int64_t ldk, int64_t ldv, int64_t ldo, float scale) {
  extern __shared__ __align__(16) uint8_t ca_smem[];
  const int dp = d + 2;  // padded row (halfs): lanes reading different rows hit different banks
  __half* sk = reinterpret_cast<__half*>(ca_smem);           // [n][dp]
  __half* sv = sk + static_cast<size_t>(n) * dp;             // [n][d]
  float* sp = reinterpret_cast<float*>(sv + static_cast<size_t>(n) * d);  // [4 warps][CA_MAX_N] probabilities
  float* sq = sp + 4 * CA_MAX_N;                             // [4 warps][d] query row
  const int h = blockIdx.x, b = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const __half* qb = q + static_cast<int64_t>(b) * n * ldq + h * d;
  const __half* kb = k + static_cast<int64_t>(b) * n * ldk + h * d;
  const __half* vb = v + static_cast<int64_t>(b) * n * ldv + h * d;
  __half* ob = o + static_cast<int64_t>(b) * n * ldo + h * d;
  for (int i = threadIdx.x; i < n * d; i += blockDim.x) {
    const int r = i / d, c = i % d;
    sk[r * dp + c] = kb[r * ldk + c];
    sv[r * d + c] = vb[r * ldv + c];
  }
  __syncthreads();
  float* myp = sp + warp * CA_MAX_N;
  float* myq = sq + warp * d;
  for (int i = warp; i < n; i += 4) {
    for (int c = lane; c < d; c += 32) myq[c] = __half2float(qb[i * ldq + c]) * scale;
    __syncwarp();
    float sc[CA_MAX_N / 32];
    float mx = -INFINITY;
#pragma unroll
    for (int t = 0; t < CA_MAX_N / 32; ++t) {
      const int j = lane + 32 * t;
      float acc = -INFINITY;
      if (j <= i) {
        acc = 0.f;
        for (int c = 0; c < d; ++c) acc += myq[c] * __half2float(sk[j * dp + c]);
      }
      sc[t] = acc;
      mx = fmaxf(mx, acc);
    }
    for (int off = 16; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
    float den = 0.f;
#pragma unroll
    for (int t = 0; t < CA_MAX_N / 32; ++t) {
      const int j = lane + 32 * t;
      const float e = (j <= i) ? __expf(sc[t] - mx) : 0.f;
      den += e;
      if (j < CA_MAX_N) myp[j] = e;
    }
    for (int off = 16; off > 0; off >>= 1) den += __shfl_xor_sync(0xffffffffu, den, off);
    __syncwarp();
    const float inv = 1.f / den;
    for (int c = lane; c < d; c += 32) {
      float acc = 0.f;
      for (int j = 0; j <= i; ++j) acc += myp[j] * __half2float(sv[j * d + c]);
      ob[i * ldo + c] = __float2half_rn(acc * inv);
    }
    __syncwarp();
  }
}
uav_status_t attention_tc(const void* q, const void* k, const void* v, void* out, int64_t batch,
                          int heads, int head_dim, int64_t nq, int64_t nk, int64_t ldq, int64_t ldk,
                          int64_t ldv, int64_t ldo, int64_t kv_batch_div, float scale,
                          cudaStream_t stream, bool causal);  // attention_tc.cu (wgmma)
}  // namespace uav

extern "C" {

uav_status_t uav_attention_causal(const void* q, const void* k, const void* v, void* out, int64_t batch, int heads, int head_dim,
                                  int64_t n, int64_t ldq, int64_t ldk, int64_t ldv, int64_t ldo, float scale,
                                  uav_stream_t stream) {
  UAV_REQUIRE(q && k && v && out && batch > 0 && heads > 0, "uav_attention_causal: bad argument");
  if (head_dim == 128 && n > uav::CA_MAX_N) {
    UAV_REQUIRE(n <= INT32_MAX && batch * heads <= 65535, "uav_attention_causal: n or batch*heads too large");
    UAV_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0,
                "uav_attention_causal: token strides must be multiples of 8");
    UAV_REQUIRE(scale > 0.f && scale < INFINITY, "uav_attention_causal: scale must be finite and > 0 (got %g)",
                (double)scale);
    UAV_REQUIRE_ALIGNED16("uav_attention_causal", q);
    UAV_REQUIRE_ALIGNED16("uav_attention_causal", k);
    UAV_REQUIRE_ALIGNED16("uav_attention_causal", v);
    UAV_REQUIRE_ALIGNED16("uav_attention_causal", out);
    return uav::attention_tc(q, k, v, out, batch, heads, head_dim, n, n, ldq, ldk, ldv, ldo, 1, scale,
                             (cudaStream_t)stream, true);
  }
  UAV_REQUIRE(n >= 1 && n <= uav::CA_MAX_N && head_dim >= 2 && head_dim <= 128 && head_dim % 2 == 0,
              "uav_attention_causal: sequence <= %d tokens (any length for head_dim 128) and even head_dim <= 128 "
              "(got n=%lld d=%d)", uav::CA_MAX_N,
              (long long)n, head_dim);
  UAV_REQUIRE(batch <= 65535, "uav_attention_causal: batch too large");
  const uav_status_t st = uav::opt_in_smem<uav::causal_attn_kernel>((int)uav::ca_smem_bytes(uav::CA_MAX_N, 128));
  if (st != UAV_OK) return st;
  const size_t smem = uav::ca_smem_bytes(n, head_dim);
  uav::causal_attn_kernel<<<dim3((unsigned)heads, (unsigned)batch), 128, smem, (cudaStream_t)stream>>>(
      reinterpret_cast<const __half*>(q), reinterpret_cast<const __half*>(k), reinterpret_cast<const __half*>(v),
      reinterpret_cast<__half*>(out), (int)n, head_dim, ldq, ldk, ldv, ldo, scale);
  UAV_LAUNCHED();
  return UAV_OK;
}

}  // extern "C"
