// attention_tc.cu — wgmma FlashAttention forward for the two dense attention cores of
// the sampling path (SURVEY.md §8a rows a9, a19):
//   * VAE mid-block AttentionBlock: 1 head, d = 512, N = h*w tokens per frame (184 320 at
//     320x576 -> 70 TFLOP per frame, 71 % of VAE-decode FLOPs): fa_tc_kernel<512, 256, 64>;
//   * UNet spatial self-attention: 8 heads, d = 128, N = 2880: fa_tc_kernel<128, 128, 128>.
// d = 64 (no pipeline shape: the UNet's d = 64 attention is text cross-attention, attention.cu) runs on
// fa_tc_kernel<64, 64, 128>.  Causal self-attention with d = 128 over more than 128 tokens (the LLaVA decoder's prefill,
// llava.py) runs on fa_tc_causal_kernel<128, 128, 128>: the same body, which skips the key tiles past the diagonal and
// masks the keys after each query row in the diagonal tile.
//
// One CTA = 128 query rows x DVT output columns; warpgroup 0 is the TMA producer (one thread), warpgroups 1 and 2 each
// own 64 query rows.  Per kv tile of BN rows a consumer warpgroup computes S = Q K^T with wgmma from shared memory
// (m64 x BN, fp32 in registers), runs the online softmax on its registers (a row is spread over the 4 lanes of a quad),
// and feeds P as fp16 register fragments straight into O += P V (wgmma with A from registers, V as an MN-major shared
// memory operand): P never touches shared memory.  For d = 512 the output accumulator of 64 x 512 fp32 does not fit the
// register file, so two CTAs each own a 256-wide half of O (QK^T is recomputed: 1.5x the minimal MMA work; K tiles are
// shared through L2).  The two consumer warpgroups run independently (no ping-pong ordering between them), so the warp
// schedulers may overlap one's softmax with the other's MMAs, but nothing enforces it.
//
// Shared memory: Q (128 x DQK fp16, up to 128 KB) + a ring of [BN kv][64 d] slots.  A kv tile streams DQK/64 K slots
// (K-major B operand of QK^T) followed by DVT/64 V slots ([BN kv][64 dv], exactly as TMA writes them = MN-major B
// operand of P V).
#include "uav_common.cuh"

#include <string.h>

namespace uav {

constexpr int TC_BM = 128;      // query rows per CTA (two warpgroups of 64)
constexpr int TC_THREADS = 384;

struct alignas(64) FaTcParams {
  CUtensorMap map_q, map_k, map_v;
  __half* out;
  int64_t ldo, bso;   // output token stride / batch stride (elements)
  int nq, nk, heads, kv_batch_div;
  float scale_log2;
};

template <int DQK, int DVT, int BN>
struct FaTcCfg {
  static constexpr int QSLABS = DQK / 64;
  static constexpr int VBLKS = DVT / 64;
  static constexpr int Q_SLAB_BYTES = TC_BM * 128;
  static constexpr int Q_BYTES = QSLABS * Q_SLAB_BYTES;
  static constexpr int SLOT_BYTES = BN * 128;
  static constexpr int STAGES_RAW = (SMEM_OPT_IN_LIMIT - 1024 - 1024 - Q_BYTES) / SLOT_BYTES;
  static constexpr int STAGES = STAGES_RAW > 16 ? 16 : STAGES_RAW;
  static_assert(STAGES >= 2, "ring does not fit");
  static constexpr int SMEM_BYTES = Q_BYTES + STAGES * SLOT_BYTES + 1024 + 1024;
};

template <int DQK, int DVT, int BN, bool CAUSAL>
__device__ __forceinline__ void fa_tc_body(const FaTcParams& p) {
  using Cfg = FaTcCfg<DQK, DVT, BN>;
  constexpr int STAGES = Cfg::STAGES;
  constexpr int QSLABS = Cfg::QSLABS;
  constexpr int VBLKS = Cfg::VBLKS;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sq = smem_align1024(smem_raw);
  uint8_t* slots = sq + Cfg::Q_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(slots + STAGES * Cfg::SLOT_BYTES);
  const RingBarriers<STAGES> ring(bars);
  uint64_t* q_bar = bars + 2 * STAGES;

  const int warp_idx = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * TC_BM;
  const int dv_off = blockIdx.y * DVT;          // which slice of the value / output columns
  const int bh = blockIdx.z;
  const int b = bh / p.heads, h = bh % p.heads;
  const int bkv = b / p.kv_batch_div;
  int ntiles = (p.nk + BN - 1) / BN;
  if constexpr (CAUSAL) ntiles = min(ntiles, (q0 + TC_BM + BN - 1) / BN);  // no key of a later tile is <= a row of this CTA

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.map_q);
    tma_prefetch_desc(&p.map_k);
    tma_prefetch_desc(&p.map_v);
    ring.init(8);  // the 8 consumer warps
    mbar_init(q_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp_idx < 4) {
    // =============================== TMA producer ===============================
    setmaxnreg_dec<PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      mbar_expect_tx(q_bar, Cfg::Q_BYTES);
      for (int c = 0; c < QSLABS; ++c)
        tma_load_3d(&p.map_q, q_bar, sq + c * Cfg::Q_SLAB_BYTES, h * DQK + c * 64, q0, b);
      RingPos<STAGES> pos;
      auto load_slot = [&](const CUtensorMap* map, int col, int row) {
        uint64_t* full = ring.acquire(pos, Cfg::SLOT_BYTES);
        tma_load_3d(map, full, slots + pos.stage * Cfg::SLOT_BYTES, col, row, bkv);
        pos.advance();
      };
      // same order as the consumers: K_j slots, then V_j slots
      for (int j = 0; j < ntiles; ++j) {
        for (int c = 0; c < QSLABS; ++c) load_slot(&p.map_k, h * DQK + c * 64, j * BN);
        for (int c = 0; c < VBLKS; ++c) load_slot(&p.map_v, h * (DVT * (int)gridDim.y) + dv_off + c * 64, j * BN);
      }
    }
    return;
  }

  // =============================== consumers: QK^T, softmax, PV, epilogue ===============================
  setmaxnreg_inc<CONSUMER_REGS>();
  const int wg = (threadIdx.x >> 7) - 1;  // query rows [64 wg, +64) of the CTA
  const int lq = lane >> 2, lr = lane & 3;
  float o[VBLKS][32];
#pragma unroll
  for (int c = 0; c < VBLKS; ++c)
#pragma unroll
    for (int i = 0; i < 32; ++i) o[c][i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};  // rows lq and lq + 8 of this warp's 16
  RingPos<STAGES> pos;
  mbar_wait(q_bar, 0);

  for (int j = 0; j < ntiles; ++j) {
    // ---- S = Q K_j^T ----
    float s[BN / 2];
    const int k_first = pos.stage;
#pragma unroll 1
    for (int c = 0; c < QSLABS; ++c) {
      ring.wait_full(pos);
      const uint64_t adesc = gmma_desc_sw128(smem_u32(sq + c * Cfg::Q_SLAB_BYTES) + wg * (64 * 128));
      const uint64_t bdesc = gmma_desc_sw128(smem_u32(slots + pos.stage * Cfg::SLOT_BYTES));
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_ss(s, adesc + 2 * k, bdesc + 2 * k, (c | k) != 0);
      wgmma_commit();
      pos.advance();
    }
    wgmma_wait<0>();
    wgmma_fence_operands(s);
    if (lane == 0)
      for (int c = 0; c < QSLABS; ++c) mbar_arrive(&ring.empty[(k_first + c) % STAGES]);

    // ---- online softmax on the registers: s[i] is row lq + 8 ((i / 2) % 2), column 8 (i / 4) + 2 lr + i % 2 ----
    const int valid = p.nk - j * BN;  // columns >= valid are padding
    if (valid < BN) {
#pragma unroll
      for (int i = 0; i < BN / 2; ++i)
        if (8 * (i / 4) + 2 * lr + (i % 2) >= valid) s[i] = -INFINITY;
    }
    if constexpr (CAUSAL) {
      // key j * BN + col is masked for query row q0 + row0 + 8 ((i / 2) % 2) when it lies after the row; key 0 is in the
      // first tile, so every row keeps a finite maximum
      const int row0 = q0 + 64 * wg + 16 * (warp_idx & 3) + lq - j * BN;
      if (j * BN + BN - 1 > q0 + 64 * wg) {
#pragma unroll
        for (int i = 0; i < BN / 2; ++i)
          if (8 * (i / 4) + 2 * lr + (i % 2) > row0 + 8 * ((i / 2) & 1)) s[i] = -INFINITY;
      }
    }
    float alpha[2], neg_m[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float mx = -INFINITY;
#pragma unroll
      for (int i = 0; i < BN / 2; ++i)
        if (((i / 2) & 1) == r) mx = fmaxf(mx, s[i]);
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[r], mx * p.scale_log2);  // scale > 0; every tile has a valid column
      alpha[r] = ex2_ftz(m_run[r] - m_new);                      // 0 on the first tile (m_run = -inf)
      m_run[r] = m_new;
      neg_m[r] = -m_new;
      l_run[r] *= alpha[r];
    }
#pragma unroll
    for (int c = 0; c < VBLKS; ++c)
#pragma unroll
      for (int i = 0; i < 32; ++i) o[c][i] *= alpha[(i / 2) & 1];
    // P = exp2(S * scale - m) as fp16 A fragments of m64 x k16 (the accumulator layout, pairs packed)
    uint32_t pa[BN / 16][4];
#pragma unroll
    for (int kk = 0; kk < BN / 16; ++kk)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int r = e & 1;
        const float p0 = ex2_ftz(fmaf(s[8 * kk + 2 * e], p.scale_log2, neg_m[r]));
        const float p1 = ex2_ftz(fmaf(s[8 * kk + 2 * e + 1], p.scale_log2, neg_m[r]));
        l_run[r] += p0 + p1;
        pa[kk][e] = pack_half2_rn(p0, p1);
      }

    // ---- O += P V_j ----
    const int v_first = pos.stage;
#pragma unroll
    for (int c = 0; c < VBLKS; ++c) {
      ring.wait_full(pos);
      const uint64_t bdesc = gmma_desc_sw128(smem_u32(slots + pos.stage * Cfg::SLOT_BYTES));
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < BN / 16; ++kk)  // 16 kv rows per step: B + 16 rows * 128 B
        wgmma_rs_tb(o[c], pa[kk], bdesc + 128 * kk, 1u);
      wgmma_commit();
      pos.advance();
    }
    wgmma_wait<0>();
#pragma unroll
    for (int c = 0; c < VBLKS; ++c) wgmma_fence_operands(o[c]);
    if (lane == 0)
      for (int c = 0; c < VBLKS; ++c) mbar_arrive(&ring.empty[(v_first + c) % STAGES]);
  }

  // ---- epilogue: O / l -> global ----
  const int wrow = q0 + 64 * wg + 16 * (warp_idx & 3) + lq;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    float l = l_run[r];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = l > 0.f ? 1.f / l : 0.f;
    const int row = wrow + 8 * r;
    if (row >= p.nq) continue;
    __half* orow = p.out + static_cast<int64_t>(b) * p.bso + static_cast<int64_t>(row) * p.ldo +
                   static_cast<int64_t>(h) * (DVT * gridDim.y) + dv_off;
#pragma unroll
    for (int c = 0; c < VBLKS; ++c)
#pragma unroll
      for (int jb = 0; jb < 8; ++jb)
        *reinterpret_cast<uint32_t*>(orow + c * 64 + jb * 8 + 2 * lr) =
            pack_half2_rn(o[c][4 * jb + 2 * r] * inv, o[c][4 * jb + 2 * r + 1] * inv);
  }
}

template <int DQK, int DVT, int BN>
__global__ void __launch_bounds__(TC_THREADS, 1)
    fa_tc_kernel(const __grid_constant__ FaTcParams p) {
  fa_tc_body<DQK, DVT, BN, false>(p);
}

template <int DQK, int DVT, int BN>
__global__ void __launch_bounds__(TC_THREADS, 1)
    fa_tc_causal_kernel(const __grid_constant__ FaTcParams p) {
  fa_tc_body<DQK, DVT, BN, true>(p);
}


template <int DQK, int DVT, int BN, bool CAUSAL = false>
static uav_status_t launch_fa_tc(FaTcParams& p, int64_t batch, int dv_splits, cudaStream_t stream) {
  const dim3 grid((p.nq + TC_BM - 1) / TC_BM, dv_splits, (unsigned)(batch * p.heads));
  if constexpr (CAUSAL)
    return launch_opted_in<fa_tc_causal_kernel<DQK, DVT, BN>>(grid, TC_THREADS, FaTcCfg<DQK, DVT, BN>::SMEM_BYTES,
                                                              stream, p);
  else
    return launch_opted_in<fa_tc_kernel<DQK, DVT, BN>>(grid, TC_THREADS, FaTcCfg<DQK, DVT, BN>::SMEM_BYTES, stream, p);
}


// entry used by uav_attention (attention.cu), which has validated the arguments, for head_dim 64, 128 and 512 (one
// head), and by uav_attention_causal (clip_text.cu) for head_dim 128 with causal = true and nq = nk
uav_status_t attention_tc(const void* q, const void* k, const void* v, void* out, int64_t batch,
                          int heads, int head_dim, int64_t nq, int64_t nk, int64_t ldq, int64_t ldk,
                          int64_t ldv, int64_t ldo, int64_t kv_batch_div, float scale,
                          cudaStream_t stream, bool causal) {
  FaTcParams p;
  memset(&p, 0, sizeof(p));
  const int64_t C = (int64_t)heads * head_dim;
  // kv tile rows: 64 for d = 512 (the 64 x 256 fp32 O slice takes 128 registers per thread), else 128
  const uint32_t bn = head_dim == 512 ? 64 : 128;
  // (batch, rows, C) at token stride ld, loaded in boxes of 64 columns x box_rows tokens of one batch item
  auto map_3d = [C](CUtensorMap* map, const void* base, int64_t rows, int64_t nbatch, int64_t ld, uint32_t box_rows,
                    const char* what) {
    const cuuint64_t dims[3] = {(cuuint64_t)C, (cuuint64_t)rows, (cuuint64_t)nbatch};
    const cuuint64_t strides[2] = {(cuuint64_t)ld * 2, (cuuint64_t)(rows * ld) * 2};
    const cuuint32_t box[3] = {64, box_rows, 1};
    return encode_tensor_map(map, base, 3, dims, strides, box, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, what);
  };
  uav_status_t st;
  if ((st = map_3d(&p.map_q, q, nq, batch, ldq, TC_BM, "attention_tc(Q)")) != UAV_OK) return st;
  if ((st = map_3d(&p.map_k, k, nk, batch / kv_batch_div, ldk, bn, "attention_tc(K)")) != UAV_OK) return st;
  if ((st = map_3d(&p.map_v, v, nk, batch / kv_batch_div, ldv, bn, "attention_tc(V)")) != UAV_OK) return st;
  p.out = reinterpret_cast<__half*>(out);
  p.ldo = ldo;
  p.bso = nq * ldo;
  p.nq = (int)nq;
  p.nk = (int)nk;
  p.heads = heads;
  p.kv_batch_div = (int)kv_batch_div;
  p.scale_log2 = scale * 1.4426950408889634f;
  if (causal) return launch_fa_tc<128, 128, 128, true>(p, batch, 1, stream);
  if (head_dim == 512) return launch_fa_tc<512, 256, 64>(p, batch, 2, stream);
  if (head_dim == 64) return launch_fa_tc<64, 64, 128>(p, batch, 1, stream);
  return launch_fa_tc<128, 128, 128>(p, batch, 1, stream);
}

}  // namespace uav
