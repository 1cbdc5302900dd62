// attention.cu — attention cores of the sampling path (SURVEY.md §8a rows a9, a10, a11, a19).
//
//  * uav_attention: softmax(Q K^T * scale) V without materialising the score matrix
//    (the reference materialises it: attention.py:209-238, 2.1 GB per call at 320x576).
//    Short key sequences (the text cross-attention: Nk = 77, d = 64/128, K/V shared by all
//    frames of a batch item) run on a resident-KV mma.sync kernel.  Every other case (UNet
//    spatial self-attention, d = 128, N = h*w; VAE mid-block attention, d = 512, 1 head; and
//    d = 64 off the pipeline's shapes) runs on the wgmma kernel of attention_tc.cu.
//  * uav_temporal_attention: the seq = T per-pixel attention with rotary embedding on the
//    first 32 dims and the T5-style relative-position bias (attention.py:699-733).  T <= 8 (the
//    pipeline's windows) with an even head count runs on an mma.sync kernel for a pair of heads;
//    every other case runs on an mma.sync kernel for one head with an online softmax over
//    16-frame key tiles.  Both read q/k/v in the (b, f, hw, c) layout, so the reference's two
//    "(b f) d c <-> (b d) f c" rearrange copies (attention.py:555,560) do not exist.
//
// All three kernels are built from the warp-tile helpers below: S = Q K^T, the P fragment, O += P V and the output
// staging are written once.
#include "uav_common.cuh"

namespace uav {

// ---------------------------------------------------------------------------------------
// warp tiles: a warp owns 16 query rows.  Lane l holds rows l / 4 and l / 4 + 8 of every 16 x 8 accumulator block,
// columns 2 (l % 4) + {0, 1} (mma16816).  Q, K and V are tile_ptr<D> tiles of D halfs per row.
// ---------------------------------------------------------------------------------------
// s[n] += Q K^T for keys [8 n, 8 n + 8): the 16 Q rows of sQ from which the lane loads row arow (row0 + (lane & 7) +
// 8 ((lane >> 3) & 1)), key rows [0, 16 NB16) of sK, over the k-steps of 16 dims [KK_BEGIN, D / 16)
template <int D, int NB16, int KK_BEGIN = 0>
__device__ __forceinline__ void warp_qk(float (&s)[NB16 * 2][4], __half* sQ, int arow, __half* sK, int lane) {
  const int brow = (lane & 7) + (lane >> 4) * 8, bchk = (lane >> 3) & 1;
#pragma unroll
  for (int kk = KK_BEGIN; kk < D / 16; ++kk) {
    uint32_t a[4];
    ldmatrix_x4(a, tile_ptr<D>(sQ, arow, kk * 2 + (lane >> 4)));
#pragma unroll
    for (int nb = 0; nb < NB16; ++nb) {
      uint32_t bfr[4];
      ldmatrix_x4(bfr, tile_ptr<D>(sK, nb * 16 + brow, kk * 2 + bchk));
      mma16816(s[nb * 2], a, bfr[0], bfr[1]);
      mma16816(s[nb * 2 + 1], a, bfr[2], bfr[3]);
    }
  }
}

// P of the accumulator block of keys [8 j, 8 j + 8) of a k16 step (p0, p1: row lane / 4; p2, p3: row lane / 4 + 8) ->
// its half of the step's A fragment
__device__ __forceinline__ void pack_p(uint32_t (&a)[4], int j, float p0, float p1, float p2, float p3) {
  a[2 * j] = pack_half2_rn(p0, p1);
  a[2 * j + 1] = pack_half2_rn(p2, p3);
}

// o[n] += P V for output columns [8 n, 8 n + 8): a is P of the 16 keys at rows [krow, krow + 16) of sV
template <int D>
__device__ __forceinline__ void warp_pv(float (&o)[D / 8][4], const uint32_t (&a)[4], __half* sV, int krow, int lane) {
  const int vrow = krow + (lane & 7) + ((lane >> 3) & 1) * 8;
#pragma unroll
  for (int nb = 0; nb < D / 16; ++nb) {
    uint32_t bfr[4];
    ldmatrix_x4_trans(bfr, tile_ptr<D>(sV, vrow, nb * 2 + (lane >> 4)));
    mma16816(o[nb * 2], a, bfr[0], bfr[1]);
    mma16816(o[nb * 2 + 1], a, bfr[2], bfr[3]);
  }
}

// max / sum over the 4 lanes of a quad, which together hold one accumulator row.  The temporal kernels reduce their
// two rows with the shuffles interleaved instead.
__device__ __forceinline__ float quad_max(float x) {
  x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 1));
  return fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 2));
}
__device__ __forceinline__ float quad_sum(float x) {
  x += __shfl_xor_sync(0xffffffffu, x, 1);
  return x + __shfl_xor_sync(0xffffffffu, x, 2);
}

// fp16 of the lane's accumulator rows times i0 (tile row r0) and i1 (tile row r0 + 8), t4 = lane % 4
template <int D>
__device__ __forceinline__ void stage_rows(__half* tile, int r0, const float (&o)[D / 8][4], float i0, float i1,
                                           int t4) {
#pragma unroll
  for (int n = 0; n < D / 8; ++n) {
    const __half2 v0 = __floats2half2_rn(o[n][0] * i0, o[n][1] * i0);
    const __half2 v1 = __floats2half2_rn(o[n][2] * i1, o[n][3] * i1);
    *reinterpret_cast<__half2*>(tile_ptr<D>(tile, r0, n) + t4 * 2) = v0;
    *reinterpret_cast<__half2*>(tile_ptr<D>(tile, r0 + 8, n) + t4 * 2) = v1;
  }
}

constexpr int FA_BM = 64;   // query rows per CTA (4 warps x 16)
constexpr int FA_THREADS = 128;

struct FaParams {
  const __half* q;
  const __half* k;
  const __half* v;
  __half* o;
  int64_t ldq, ldk, ldv, ldo;        // token stride (elements)
  int64_t bsq, bsk, bsv, bso;        // batch stride (elements)
  int nq, nk, heads, kv_batch_div;
  float scale_log2;                  // softmax scale * log2(e)
};

// ---------------------------------------------------------------------------------------
// text cross-attention (nk <= 128, typically 77): K and V of one (batch, head) stay resident in
// shared memory, the CTA streams query tiles past them (double-buffered cp.async), the whole
// score row fits in registers (single-pass softmax), and each warp stages its 16 output rows in
// the Q buffer it has just consumed.  A kernel that streams KV tiles past one query tile per CTA
// spends most of its time in the per-CTA prologue / epilogue when there are only one or two KV
// tiles (an mma.sync one with 64-key tiles measured 1.0 TB/s at h/2).
// ---------------------------------------------------------------------------------------
template <int D, int NB16>
__global__ void __launch_bounds__(FA_THREADS)
    cross_attn_kernel(const FaParams p) {
  constexpr int NKP = NB16 * 16;
  extern __shared__ __align__(16) uint8_t fa_smem[];
  __half* sk = reinterpret_cast<__half*>(fa_smem);   // [NKP][D]
  __half* sv = sk + NKP * D;                          // [NKP][D]
  __half* sq = sv + NKP * D;                          // [2][64][D]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  // the head is the FASTEST block index: the CTAs that read the 2*D-byte head slices of the same token rows run side
  // by side, so each 1 KB token row is fetched from DRAM within one burst instead of once per head pass
  const int b = blockIdx.y, h = blockIdx.x % p.heads;
  const int tile_stride = gridDim.x / p.heads;
  const __half* qg = p.q + b * p.bsq + static_cast<int64_t>(h) * D;
  const __half* kg = p.k + (b / p.kv_batch_div) * p.bsk + static_cast<int64_t>(h) * D;
  const __half* vg = p.v + (b / p.kv_batch_div) * p.bsv + static_cast<int64_t>(h) * D;
  __half* og = p.o + b * p.bso + static_cast<int64_t>(h) * D;
  constexpr int QC = D / 8;
  const int ntiles = (p.nq + FA_BM - 1) / FA_BM;

  for (int i = tid; i < NKP * QC; i += FA_THREADS) {
    const int r = i / QC, c = i % QC;
    const bool ok = r < p.nk;
    cp_async16(tile_ptr<D>(sk, r, c), kg + static_cast<int64_t>(ok ? r : 0) * p.ldk + c * 8, ok);
    cp_async16(tile_ptr<D>(sv, r, c), vg + static_cast<int64_t>(ok ? r : 0) * p.ldv + c * 8, ok);
  }
  auto load_q = [&](int tile, int buf) {
    const int q0 = tile * FA_BM;
    __half* sqb = sq + buf * FA_BM * D;
    for (int i = tid; i < FA_BM * QC; i += FA_THREADS) {
      const int r = i / QC, c = i % QC;
      const bool ok = q0 + r < p.nq;
      cp_async16(tile_ptr<D>(sqb, r, c), qg + static_cast<int64_t>(ok ? q0 + r : 0) * p.ldq + c * 8, ok);
    }
  };
  int tile = blockIdx.x / p.heads;
  if (tile < ntiles) load_q(tile, 0);
  cp_async_commit();

  const int g = lane >> 2, t4 = lane & 3;
  const int arow = warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
  int it = 0;
  for (; tile < ntiles; tile += tile_stride, ++it) {
    const int buf = it & 1;
    const int next = tile + tile_stride;
    if (next < ntiles) load_q(next, buf ^ 1);
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    __half* sqb = sq + buf * FA_BM * D;

    // S = Q K^T  (16 x NKP per warp)
    float s[NB16 * 2][4];
#pragma unroll
    for (int i = 0; i < NB16 * 2; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
    warp_qk<D, NB16>(s, sqb, arow, sk, lane);
    // row maxima of the raw scores (scale > 0); only 8-column blocks past nk hold padded keys
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int nb = 0; nb < NB16 * 2; ++nb) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        if ((nb + 1) * 8 > p.nk) {  // block-uniform test, false for all but the tail blocks
          const int col = nb * 8 + t4 * 2 + (e & 1);
          if (col >= p.nk) s[nb][e] = -INFINITY;
        }
        mx[e >> 1] = fmaxf(mx[e >> 1], s[nb][e]);
      }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) mx[r] = quad_max(mx[r]) * p.scale_log2;
    float rs[2] = {0.f, 0.f};
    uint32_t pf[NB16][4];  // P as the A fragments of the k16 steps
#pragma unroll
    for (int nb = 0; nb < NB16 * 2; ++nb) {
      // exp2(s * scale - max): one FFMA + one MUFU per score
      const float p0 = ex2_ftz(fmaf(s[nb][0], p.scale_log2, -mx[0])), p1 = ex2_ftz(fmaf(s[nb][1], p.scale_log2, -mx[0]));
      const float p2 = ex2_ftz(fmaf(s[nb][2], p.scale_log2, -mx[1])), p3 = ex2_ftz(fmaf(s[nb][3], p.scale_log2, -mx[1]));
      rs[0] += p0 + p1;
      rs[1] += p2 + p3;
      pack_p(pf[nb >> 1], nb & 1, p0, p1, p2, p3);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) rs[r] = 1.f / quad_sum(rs[r]);
    // O = P V
    float o_acc[D / 8][4];
#pragma unroll
    for (int i = 0; i < D / 8; ++i) o_acc[i][0] = o_acc[i][1] = o_acc[i][2] = o_acc[i][3] = 0.f;
#pragma unroll
    for (int kk = 0; kk < NB16; ++kk) warp_pv<D>(o_acc, pf[kk], sv, kk * 16, lane);
    // stage this warp's 16 rows in its own (already consumed) rows of the Q buffer, then 16-byte stores
    __syncwarp();
    stage_rows<D>(sqb, warp * 16 + g, o_acc, rs[0], rs[1], t4);
    __syncwarp();
    const int q0 = tile * FA_BM;
    for (int i = lane; i < 16 * QC; i += 32) {
      const int r = warp * 16 + i / QC, c = i % QC;
      if (q0 + r < p.nq)
        stg16(og + static_cast<int64_t>(q0 + r) * p.ldo + c * 8,
              *reinterpret_cast<const uint4*>(tile_ptr<D>(sqb, r, c)));
    }
    __syncthreads();  // buffer `buf` is refilled by the prefetch issued in the next iteration
  }
  cp_async_wait<0>();
}

// ---------------------------------------------------------------------------------------
// temporal attention: one warp per (batch, pixel) and one head (temporal_attn_long_kernel) or a pair of heads
// (temporal_attn_mma_kernel)
// ---------------------------------------------------------------------------------------
struct TaParams {
  const __half* q;
  const __half* k;
  const __half* v;
  __half* o;
  int64_t ldq, ldk, ldv, ldo;  // token stride (elements); tokens ordered (b, f, hw)
  int B, F, heads;
  int64_t HW;
  float scale;
  const float* rot;   // [F][16][2] cos, sin of frame * freq_pair
  const float* bias;  // [heads][F][F]
};

// ---------------------------------------------------------------------------------------
// temporal attention for F <= 8 and an even head count, on mma.sync: one warp per PAIR of heads of one (batch, pixel).
// The two items' 8 frames are stacked into one 16-row tile, so that
//   S  = [Q_a; Q_b] K_a^T , [Q_a; Q_b] K_b^T   (two m16n8k16 n-blocks per k-step; the cross terms are discarded)
//   O  = diag(P_a, P_b) [V_a; V_b]              (ONE k-step: the block-diagonal P is exactly the A fragment
//                                                {P_a, 0, 0, P_b} built from the S accumulators in registers)
// ~125 instructions per (pixel, head) instead of ~700 for a warp-shuffle formulation with one lane per (frame, quarter
// of the head dim): the kernel becomes a pure 8 B/element stream.  Rotary (first 32 dims, interleaved pairs) is applied
// to the 16-byte chunks on their way into shared memory; scale and the relative-position bias are applied to the fp32
// scores.
// ---------------------------------------------------------------------------------------
template <int D>
__global__ void __launch_bounds__(128)
    temporal_attn_mma_kernel(const TaParams p) {
  constexpr int CH = D / 8;             // 16-byte chunks per row
  constexpr int LD_ITERS = 16 * CH / 32;  // chunks per lane and tensor
  __shared__ __align__(16) __half smem[4][3][16 * D];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int hp = p.heads >> 1;
  const int64_t pw = static_cast<int64_t>(blockIdx.x) * 4 + warp;
  const int64_t total = static_cast<int64_t>(p.B) * p.HW * hp;
  if (pw >= total) return;  // whole warp
  const int h0 = static_cast<int>(pw % hp) * 2;
  const int64_t pix = (pw / hp) % p.HW;
  const int64_t b = pw / (static_cast<int64_t>(hp) * p.HW);
  __half* sQ = smem[warp][0];
  __half* sK = smem[warp][1];
  __half* sV = smem[warp][2];

  // ---- global -> (rotary) -> swizzled smem tiles: row = item * 8 + frame.  All loads are issued before the first
  // use so that 3 * LD_ITERS 16-byte requests per lane are in flight ----
  uint4 v[3][LD_ITERS];
#pragma unroll
  for (int tsr = 0; tsr < 3; ++tsr) {
    const __half* src = tsr == 0 ? p.q : (tsr == 1 ? p.k : p.v);
    const int64_t ld = tsr == 0 ? p.ldq : (tsr == 1 ? p.ldk : p.ldv);
#pragma unroll
    for (int i = 0; i < LD_ITERS; ++i) {
      const int id = lane + 32 * i;
      const int row = id / CH, chunk = id % CH;
      const int item = row >> 3, frame = row & 7;
      v[tsr][i] = make_uint4(0, 0, 0, 0);
      if (frame < p.F) {
        const int64_t tok = (b * p.F + frame) * p.HW + pix;
        v[tsr][i] = ldg16(src + tok * ld + (h0 + item) * D + chunk * 8);
      }
    }
  }
#pragma unroll
  for (int tsr = 0; tsr < 3; ++tsr) {
    __half* dst = smem[warp][tsr];
#pragma unroll
    for (int i = 0; i < LD_ITERS; ++i) {
      const int id = lane + 32 * i;
      const int row = id / CH, chunk = id % CH;
      const int frame = row & 7;
      if (tsr < 2 && chunk < 4 && frame < p.F) {
        // rotary pairs 4*chunk .. 4*chunk+3 of this frame: (x0, x1) -> (x0 c - x1 s, x1 c + x0 s)
        const float4 r0 = __ldg(reinterpret_cast<const float4*>(p.rot + (frame * 16 + chunk * 4) * 2));
        const float4 r1 = __ldg(reinterpret_cast<const float4*>(p.rot + (frame * 16 + chunk * 4) * 2 + 4));
        const float cs[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
        __half2* h = reinterpret_cast<__half2*>(&v[tsr][i]);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = __half22float2(h[j]);
          const float c = cs[2 * j], sn = cs[2 * j + 1];
          h[j] = __floats2half2_rn(f.x * c - f.y * sn, f.y * c + f.x * sn);
        }
      }
      *reinterpret_cast<uint4*>(tile_ptr<D>(dst, row, chunk)) = v[tsr][i];
    }
  }
  __syncwarp();

  const int g = lane >> 2, t4 = lane & 3;
  // ---- S = Q K^T: the two n-blocks are the keys of item a (s[0]) and of item b (s[1]) ----
  float s[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
  warp_qk<D, 1>(s, sQ, (lane & 7) + ((lane >> 3) & 1) * 8, sK, lane);
  // ---- softmax over the <= 8 keys of each item: row g of item a lives in s[0][0..1], row g of item b in s[1][2..3] ----
  uint32_t pa, pb;
  {
    const int j0 = 2 * t4, j1 = j0 + 1;
    const bool row_ok = g < p.F;
    float xa0 = -INFINITY, xa1 = -INFINITY, xb0 = -INFINITY, xb1 = -INFINITY;
    if (row_ok && j0 < p.F) {
      xa0 = s[0][0] * p.scale + __ldg(p.bias + (h0 * p.F + g) * p.F + j0);
      xb0 = s[1][2] * p.scale + __ldg(p.bias + ((h0 + 1) * p.F + g) * p.F + j0);
    }
    if (row_ok && j1 < p.F) {
      xa1 = s[0][1] * p.scale + __ldg(p.bias + (h0 * p.F + g) * p.F + j1);
      xb1 = s[1][3] * p.scale + __ldg(p.bias + ((h0 + 1) * p.F + g) * p.F + j1);
    }
    float ma = fmaxf(xa0, xa1), mb = fmaxf(xb0, xb1);
    ma = fmaxf(ma, __shfl_xor_sync(0xffffffffu, ma, 1));
    mb = fmaxf(mb, __shfl_xor_sync(0xffffffffu, mb, 1));
    ma = fmaxf(ma, __shfl_xor_sync(0xffffffffu, ma, 2));
    mb = fmaxf(mb, __shfl_xor_sync(0xffffffffu, mb, 2));
    if (!row_ok) ma = mb = 0.f;  // padded query rows: all keys masked, keep the arithmetic finite
    const float ea0 = __expf(xa0 - ma), ea1 = __expf(xa1 - ma), eb0 = __expf(xb0 - mb), eb1 = __expf(xb1 - mb);
    float da = ea0 + ea1, db = eb0 + eb1;
    da += __shfl_xor_sync(0xffffffffu, da, 1);
    db += __shfl_xor_sync(0xffffffffu, db, 1);
    da += __shfl_xor_sync(0xffffffffu, da, 2);
    db += __shfl_xor_sync(0xffffffffu, db, 2);
    const float ia = da > 0.f ? 1.f / da : 0.f, ib = db > 0.f ? 1.f / db : 0.f;
    pa = pack_half2_rn(ea0 * ia, ea1 * ia);
    pb = pack_half2_rn(eb0 * ib, eb1 * ib);
  }
  // ---- O = diag(P_a, P_b) [V_a; V_b] ----
  float o[D / 8][4];
#pragma unroll
  for (int i = 0; i < D / 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  const uint32_t a[4] = {pa, 0u, 0u, pb};
  warp_pv<D>(o, a, sV, 0, lane);
  // ---- O (P is normalised) -> smem (Q tile) -> 16-byte stores ----
  __syncwarp();
#pragma unroll
  for (int n = 0; n < D / 8; ++n) {
    *reinterpret_cast<__half2*>(tile_ptr<D>(sQ, g, n) + 2 * t4) = __floats2half2_rn(o[n][0], o[n][1]);
    *reinterpret_cast<__half2*>(tile_ptr<D>(sQ, g + 8, n) + 2 * t4) = __floats2half2_rn(o[n][2], o[n][3]);
  }
  __syncwarp();
#pragma unroll
  for (int i = 0; i < LD_ITERS; ++i) {
    const int id = lane + 32 * i;
    const int row = id / CH, chunk = id % CH;
    const int item = row >> 3, frame = row & 7;
    if (frame < p.F) {
      const int64_t tok = (b * p.F + frame) * p.HW + pix;
      stg16(p.o + tok * p.ldo + (h0 + item) * D + chunk * 8, *reinterpret_cast<const uint4*>(tile_ptr<D>(sQ, row, chunk)));
    }
  }
}

// ---------------------------------------------------------------------------------------
// temporal attention for any F and head count (all but the even-head F <= 8 windows of the pipeline): one warp per
// (batch, pixel, head).  Queries are taken in 16-frame tiles; keys and values stream through per-warp
// shared memory in 16-frame tiles and the softmax is online (running fp32 row max and sum, O
// rescaled), so F has no upper bound.  Rotary is applied in fp32 while the mma fragments of dims
// [0, 32) are built, as hi + lo fp16 pairs.  Padded key columns are masked to -inf; padded query
// rows compute on zeros and are never stored.
// ---------------------------------------------------------------------------------------
template <int D>
__global__ void __launch_bounds__(128)
    temporal_attn_long_kernel(const TaParams p) {
  constexpr int CH = D / 8;               // 16-byte chunks per row
  constexpr int LD_ITERS = 16 * CH / 32;  // chunks per lane and tile
  __shared__ __align__(16) __half smem[4][3][16 * D];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t wid = static_cast<int64_t>(blockIdx.x) * 4 + warp;
  const int64_t total = static_cast<int64_t>(p.B) * p.HW * p.heads;
  if (wid >= total) return;  // whole warp
  const int h = static_cast<int>(wid % p.heads);
  const int64_t pix = (wid / p.heads) % p.HW;
  const int64_t b = wid / (static_cast<int64_t>(p.heads) * p.HW);
  const int64_t F = p.F;
  __half* sQ = smem[warp][0];
  __half* sK = smem[warp][1];
  __half* sV = smem[warp][2];
  const float* bias_h = p.bias + static_cast<int64_t>(h) * F * F;

  // 16 frames from f0 of one tensor -> swizzled smem tile with cp.async (zero fill past F).  A lane always holds
  // chunk lane % CH of rows lane / CH + i * (32 / CH).
  const int chunk = lane % CH;
  auto load_tile = [&](__half* dst, const __half* src, int64_t ld, int64_t f0) {
#pragma unroll 1
    for (int i = 0; i < LD_ITERS; ++i) {
      const int row = lane / CH + i * (32 / CH);
      const int64_t frame = f0 + row;
      const bool ok = frame < F;
      cp_async16(tile_ptr<D>(dst, row, chunk), src + ((b * F + (ok ? frame : 0)) * p.HW + pix) * ld + h * D + chunk * 8,
                 ok);
    }
  };
  // rotary on dims [0, 32), computed in fp32 straight into mma fragments and split into hi + lo fp16 parts, so that the
  // scores see the rotated operands to ~2^-22 instead of one fp16 rounding: pair (x0, x1) of frame f at dims
  // [dim, dim + 1] -> (x0 c - x1 s, x1 c + x0 s) with (c, s) = rot[f][dim / 2]
  auto rope_pair = [&](const __half* tile, int row, int dim, int64_t frame, uint32_t& hi, uint32_t& lo) {
    const float2 x = __half22float2(*reinterpret_cast<const __half2*>(tile_ptr<D>(const_cast<__half*>(tile), row, dim >> 3) +
                                                                       (dim & 7)));
    const float2 cs = __ldg(reinterpret_cast<const float2*>(p.rot) + (frame < F ? frame : F - 1) * 16 + (dim >> 1));
    const float r0 = x.x * cs.x - x.y * cs.y, r1 = x.y * cs.x + x.x * cs.y;
    const __half2 h = __floats2half2_rn(r0, r1);
    const float2 hf = __half22float2(h);
    const __half2 l = __floats2half2_rn(r0 - hf.x, r1 - hf.y);
    hi = *reinterpret_cast<const uint32_t*>(&h);
    lo = *reinterpret_cast<const uint32_t*>(&l);
  };

  const int g = lane >> 2, t4 = lane & 3;
  const int arow = (lane & 7) + ((lane >> 3) & 1) * 8;
#pragma unroll 1
  for (int64_t q0 = 0; q0 < F; q0 += 16) {
    __syncwarp();  // the previous tile's output rows have left sQ
    load_tile(sQ, p.q, p.ldq, q0);
    cp_async_commit();
    cp_async_wait<0>();
    __syncwarp();
    const int64_t r0 = q0 + g, r1 = q0 + g + 8;  // the two query rows of this lane
    // A fragments of the rotated dims [0, 32): a[j] = rows g + 8 (j & 1), dims kk*16 + 2 t4 + 8 (j >> 1)
    uint32_t qh[2][4], ql[2][4];
#pragma unroll
    for (int kk = 0; kk < 2; ++kk)
#pragma unroll
      for (int j = 0; j < 4; ++j)
        rope_pair(sQ, g + (j & 1) * 8, kk * 16 + 2 * t4 + (j >> 1) * 8, j & 1 ? r1 : r0, qh[kk][j], ql[kk][j]);
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
    float o[D / 8][4];
#pragma unroll
    for (int i = 0; i < D / 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;

#pragma unroll 1
    for (int64_t k0 = 0; k0 < F; k0 += 16) {
      __syncwarp();  // every lane is done with the previous K/V tile
      load_tile(sK, p.k, p.ldk, k0);
      load_tile(sV, p.v, p.ldv, k0);
      cp_async_commit();
      cp_async_wait<0>();
      __syncwarp();
      // ---- S = Q K^T: s[nb] holds keys k0 + nb*8 + 2*t4 + {0, 1} of rows g ([0..1]) and g + 8 ([2..3]) ----
      float s[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
      // rotated dims [0, 32): Qh Kh + Qh Kl + Ql Kh; B fragment of n-block nb = key nb*8 + g, dims kk*16 + 2 t4 + {0, 8}
#pragma unroll
      for (int kk = 0; kk < 2; ++kk) {
#pragma unroll
        for (int nb = 0; nb < 2; ++nb) {
          uint32_t kh[2], kl[2];
#pragma unroll
          for (int j = 0; j < 2; ++j)
            rope_pair(sK, nb * 8 + g, kk * 16 + 2 * t4 + j * 8, k0 + nb * 8 + g, kh[j], kl[j]);
          mma16816(s[nb], qh[kk], kh[0], kh[1]);
          mma16816(s[nb], qh[kk], kl[0], kl[1]);
          mma16816(s[nb], ql[kk], kh[0], kh[1]);
        }
      }
      warp_qk<D, 1, 2>(s, sQ, arow, sK, lane);  // dims [32, D)
      float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
      for (int nb = 0; nb < 2; ++nb) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int64_t col = k0 + nb * 8 + 2 * t4 + j;
          float x0 = -INFINITY, x1 = -INFINITY;
          if (col < F) {
            x0 = s[nb][j] * p.scale + (r0 < F ? __ldg(bias_h + r0 * F + col) : 0.f);
            x1 = s[nb][2 + j] * p.scale + (r1 < F ? __ldg(bias_h + r1 * F + col) : 0.f);
          }
          s[nb][j] = x0;
          s[nb][2 + j] = x1;
          mx0 = fmaxf(mx0, x0);
          mx1 = fmaxf(mx1, x1);
        }
      }
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
      // key column k0 is always valid, so the new maxima are finite; exp(-inf) = 0 covers the first tile
      const float n0 = fmaxf(m0, mx0), n1 = fmaxf(m1, mx1);
      const float c0 = __expf(m0 - n0), c1 = __expf(m1 - n1);
      m0 = n0;
      m1 = n1;
      float ps0 = 0.f, ps1 = 0.f;
#pragma unroll
      for (int nb = 0; nb < 2; ++nb) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          s[nb][j] = __expf(s[nb][j] - n0);
          s[nb][2 + j] = __expf(s[nb][2 + j] - n1);
          ps0 += s[nb][j];
          ps1 += s[nb][2 + j];
        }
      }
      l0 = l0 * c0 + ps0;  // per-lane partial sums: the quad is reduced once at the end
      l1 = l1 * c1 + ps1;
#pragma unroll
      for (int i = 0; i < D / 8; ++i) {
        o[i][0] *= c0;
        o[i][1] *= c0;
        o[i][2] *= c1;
        o[i][3] *= c1;
      }
      // ---- O += P V: the S accumulators are the A fragment of the k = 16 keys step ----
      uint32_t a[4];
      pack_p(a, 0, s[0][0], s[0][1], s[0][2], s[0][3]);
      pack_p(a, 1, s[1][0], s[1][1], s[1][2], s[1][3]);
      warp_pv<D>(o, a, sV, 0, lane);
    }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
    l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float i0 = 1.f / l0, i1 = 1.f / l1;
    // ---- O -> smem (Q tile) -> 16-byte stores of the rows < F ----
    __syncwarp();
    stage_rows<D>(sQ, g, o, i0, i1, t4);
    __syncwarp();
#pragma unroll
    for (int i = 0; i < LD_ITERS; ++i) {
      const int row = lane / CH + i * (32 / CH);
      const int64_t frame = q0 + row;
      if (frame < F) {
        stg16(p.o + ((b * F + frame) * p.HW + pix) * p.ldo + h * D + chunk * 8,
              *reinterpret_cast<const uint4*>(tile_ptr<D>(sQ, row, chunk)));
      }
    }
  }
}

uav_status_t attention_tc(const void* q, const void* k, const void* v, void* out, int64_t batch,
                          int heads, int head_dim, int64_t nq, int64_t nk, int64_t ldq, int64_t ldk,
                          int64_t ldv, int64_t ldo, int64_t kv_batch_div, float scale,
                          cudaStream_t stream, bool causal = false);  // attention_tc.cu (wgmma)

template <int D, int NB16>
static uav_status_t launch_cross(const FaParams& p, int batch, cudaStream_t stream) {
  const int ntiles = (p.nq + FA_BM - 1) / FA_BM;
  // enough CTAs to fill the GPU ~4x over, each streaming several query tiles past its resident K/V
  int gx = (num_sms() * 8 + batch * p.heads - 1) / (batch * p.heads);
  if (gx > ntiles) gx = ntiles;
  if (gx < 1) gx = 1;
  return launch_opted_in<cross_attn_kernel<D, NB16>>(dim3(gx * p.heads, batch), FA_THREADS,
                                                     (2 * NB16 * 16 * D + 2 * FA_BM * D) * 2, stream, p);
}

// blocks of 4 warps, one warp per (batch, pixel) and pair of heads (pairs) or head
template <int D>
static void launch_temporal(const TaParams& p, bool pairs, unsigned blocks, cudaStream_t stream) {
  if (pairs) temporal_attn_mma_kernel<D><<<blocks, 128, 0, stream>>>(p);
  else temporal_attn_long_kernel<D><<<blocks, 128, 0, stream>>>(p);
}

}  // namespace uav

using namespace uav;

extern "C" {

uav_status_t uav_attention(const void* q, const void* k, const void* v, void* out, int64_t batch,
                           int heads, int head_dim, int64_t nq, int64_t nk, int64_t ldq,
                           int64_t ldk, int64_t ldv, int64_t ldo, int64_t kv_batch_div,
                           float scale, uav_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  UAV_REQUIRE(q && k && v && out, "uav_attention: null pointer");
  UAV_REQUIRE(batch > 0 && heads > 0 && nq > 0 && nk > 0 && kv_batch_div > 0,
              "uav_attention: bad shape");
  UAV_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0,
              "uav_attention: token strides must be multiples of 8");
  UAV_REQUIRE(batch * heads <= 65535, "uav_attention: batch*heads too large");
  UAV_REQUIRE(batch % kv_batch_div == 0, "uav_attention: batch must be a multiple of kv_batch_div");
  if (head_dim != 64 && head_dim != 128 && head_dim != 512) {
    set_last_error("uav_attention: head_dim %d unsupported (64, 128, 512)", head_dim);
    return UAV_ERR_UNSUPPORTED;
  }
  UAV_REQUIRE(head_dim != 512 || heads == 1, "uav_attention: head_dim 512 supports a single head");
  UAV_REQUIRE(nq <= INT32_MAX && nk <= INT32_MAX, "uav_attention: nq or nk too large");
  // the cross and wgmma kernels take the row maximum of the raw scores and scale it afterwards, which is the maximum of
  // the scaled scores only for scale > 0 (scale = 0 would also turn the masked columns into -inf * 0 = NaN)
  UAV_REQUIRE(scale > 0.f && scale < INFINITY, "uav_attention: scale must be finite and > 0 (got %g)", (double)scale);
  UAV_REQUIRE_ALIGNED16("uav_attention", q);
  UAV_REQUIRE_ALIGNED16("uav_attention", k);
  UAV_REQUIRE_ALIGNED16("uav_attention", v);
  UAV_REQUIRE_ALIGNED16("uav_attention", out);

  // short key/value sequences (the 77 prompt tokens) run on the resident-KV streaming kernel; everything else (UNet
  // self-attention at h/8, d = 128; VAE AttentionBlock, d = 512; d = 64 off the pipeline's shapes) on the wgmma kernel
  const bool cross = nk <= 128 && nq >= 4 * nk && head_dim != 512;
  if (!cross)
    return attention_tc(q, k, v, out, batch, heads, head_dim, nq, nk, ldq, ldk, ldv, ldo, kv_batch_div, scale,
                        stream);
  FaParams p;
  p.q = (const __half*)q; p.k = (const __half*)k; p.v = (const __half*)v; p.o = (__half*)out;
  p.ldq = ldq; p.ldk = ldk; p.ldv = ldv; p.ldo = ldo;
  p.bsq = nq * ldq; p.bsk = nk * ldk; p.bsv = nk * ldv; p.bso = nq * ldo;
  p.nq = (int)nq; p.nk = (int)nk; p.heads = heads; p.kv_batch_div = (int)kv_batch_div;
  p.scale_log2 = scale * 1.4426950408889634f;
  if (head_dim == 64) return nk <= 80 ? launch_cross<64, 5>(p, (int)batch, stream) : launch_cross<64, 8>(p, (int)batch, stream);
  return nk <= 80 ? launch_cross<128, 5>(p, (int)batch, stream) : launch_cross<128, 8>(p, (int)batch, stream);
}

uav_status_t uav_temporal_attention(const void* q, const void* k, const void* v, void* out,
                                    int64_t B, int64_t F, int64_t HW, int heads, int head_dim,
                                    int64_t ldq, int64_t ldk, int64_t ldv, int64_t ldo,
                                    float scale, const float* rot_cos_sin, const float* rel_bias,
                                    uav_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  UAV_REQUIRE(q && k && v && out && rot_cos_sin && rel_bias,
              "uav_temporal_attention: null pointer");
  UAV_REQUIRE(B > 0 && F >= 1 && HW > 0 && heads > 0, "uav_temporal_attention: bad shape");
  UAV_REQUIRE(B <= INT32_MAX && F <= INT32_MAX, "uav_temporal_attention: B or F too large");
  UAV_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0,
              "uav_temporal_attention: token strides must be multiples of 8");
  if (head_dim != 64 && head_dim != 128) {
    set_last_error("uav_temporal_attention: head_dim %d unsupported (64, 128)", head_dim);
    return UAV_ERR_UNSUPPORTED;
  }
  UAV_REQUIRE_ALIGNED16("uav_temporal_attention", q);
  UAV_REQUIRE_ALIGNED16("uav_temporal_attention", k);
  UAV_REQUIRE_ALIGNED16("uav_temporal_attention", v);
  UAV_REQUIRE_ALIGNED16("uav_temporal_attention", out);
  UAV_REQUIRE_ALIGNED16("uav_temporal_attention", rot_cos_sin);
  // the pipeline's windows (F <= 8, even head count): one warp per pair of heads; everything else: one warp per head
  const bool pairs = F <= 8 && heads % 2 == 0;
  const int64_t blocks = (B * HW * (pairs ? heads / 2 : heads) + 3) / 4;  // 4 warps per CTA
  UAV_REQUIRE(blocks <= INT32_MAX, "uav_temporal_attention: too many (pixel, head) items");
  TaParams p;
  p.q = (const __half*)q; p.k = (const __half*)k; p.v = (const __half*)v; p.o = (__half*)out;
  p.ldq = ldq; p.ldk = ldk; p.ldv = ldv; p.ldo = ldo;
  p.B = (int)B; p.F = (int)F; p.heads = heads; p.HW = HW;
  p.scale = scale; p.rot = rot_cos_sin; p.bias = rel_bias;
  if (head_dim == 64) launch_temporal<64>(p, pairs, (unsigned)blocks, stream);
  else launch_temporal<128>(p, pairs, (unsigned)blocks, stream);
  UAV_LAUNCHED();
  return UAV_OK;
}

}  // extern "C"
