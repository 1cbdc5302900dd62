// igemm.cu — the wgmma implicit-GEMM kernel behind every convolution and Linear on the
// Upscale-A-Video sampling path (SURVEY.md §8a rows a3, a4, a5, a8, a12, a13, a18, a20).
//
//   out[pixel][n] = epilogue( sum_{tap, c} A[pixel + off(tap)][c] * W[n][tap][c] )
//
// Design (sm_90a, not a cuDNN translation):
//  * activations stay channels-last, so an M-tile of 128 output pixels is a rectangular box
//    of the input tensor and ONE TMA box load per filter tap (shifted coordinates, hardware
//    zero fill outside the image = the convolution's zero padding) lands directly in the
//    128B-swizzled K-major layout wgmma consumes — no im2col buffer, no layout copies
//    (the reference pays two permute copies per conv: resnet.py:97-99).
//  * persistent CTAs (one per SM), warp-specialised: one TMA producer thread, two consumer warpgroups that each issue
//    wgmma m64 x BLOCK_N x 16 on their 64 rows of the stage and run the fused epilogue from the register accumulators
//    (bias/temb/act/residual/statistics -> swizzled smem staging -> TMA store); an mbarrier ring of {A 128x64,
//    B BLOCK_Nx64} fp16 stages fills the rest of the 227 KB of shared memory.
//  * tiles are 128 x BLOCK_N with BLOCK_N up to 256: the producer warpgroup gives up registers (setmaxnreg.dec 40) so
//    that each consumer thread can hold the 128 fp32 accumulators of an m64n256 tile (setmaxnreg.inc 232).  A 256-wide
//    tile fetches every A box once per 256 output channels instead of once per 128.
//  * stride-2 convs read a 5-D "phase" view (2C, W/2, 2, H/2, NB) of the same buffer, the
//    temporal (k,1,1) conv a (C, HW, T, B) view, Conv3d a (C, W, H, T, B) view, Linear a
//    (K, M) view: all the same kernel, only the tensor map and the tap table differ.
#include <stdarg.h>
#include <stdlib.h>
#include <stdio.h>
#include <string.h>

#include <atomic>
#include <initializer_list>
#include <iterator>
#include <mutex>

#include "uav_common.cuh"

namespace uav {

// ---------------------------------------------------------------------------------------
// host-side globals shared by all translation units
// ---------------------------------------------------------------------------------------
static thread_local char g_err[1024] = "";
void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
std::atomic<uint64_t> g_launches{0};

int current_device() {
  int dev = 0;
  cudaGetDevice(&dev);
  return dev;
}

int num_sms() {
  static int n[64] = {0};  // per device (a process may drive several GPUs)
  const int dev = current_device() & 63;
  if (n[dev] == 0) {
    int v = 0;
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    n[dev] = v > 0 ? v : 132;
  }
  return n[dev];
}

// TMA descriptor encode through the driver entry point (no link-time libcuda dependency)
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled get_encode_tiled() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) ==
            cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  });
  return fn;
}

uav_status_t encode_tensor_map(CUtensorMap* map, const void* base, int rank, const cuuint64_t* dims,
                               const cuuint64_t* strides, const cuuint32_t* box, CUtensorMapL2promotion l2,
                               const char* what) {
  PFN_encodeTiled encode = get_encode_tiled();
  UAV_REQUIRE(encode != nullptr, "%s: cuTensorMapEncodeTiled entry point unavailable", what);
  const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  const CUresult r = encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, rank, const_cast<void*>(base), dims, strides, box,
                            estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, l2,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  UAV_REQUIRE(r == CUDA_SUCCESS, "%s: cuTensorMapEncodeTiled failed with %d", what, (int)r);
  return UAV_OK;
}

// ---------------------------------------------------------------------------------------
// kernel
// ---------------------------------------------------------------------------------------
constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;  // fp16 elements: one 128-byte swizzle row
constexpr int MAX_TAPS = 49;  // up to 7 x 7 (RAFT motion encoder)
constexpr int NUM_THREADS = 384;      // warpgroup 0: TMA producer (one thread); warpgroups 1-2: wgmma + epilogue
constexpr int NUM_EPI_THREADS = 256;
constexpr int A_STAGE_BYTES = BLOCK_M * BLOCK_K * 2;
constexpr int SLAB_BYTES = BLOCK_M * 128;  // 128 rows x 64 fp16 output columns, 128B-swizzled

struct alignas(64) IgemmParams {
  CUtensorMap map_a;
  CUtensorMap map_b;
  CUtensorMap map_out;           // only valid when tma_store != 0
  CUtensorMap map_res;           // residual operand as a TMA tensor (same box geometry as map_out); valid when res_tma != 0
  int32_t tap_off[MAX_TAPS][5];  // coordinate offset of each tap (dim0 = channel offset)
  int32_t num_taps;
  int32_t kblocks_per_tap;
  int32_t k_per_tap;
  uint32_t box[5];       // box[0] = 64, box[1..4] = M-tile extents (product 128)
  uint32_t tiles[5];     // tiles along dims 1..4
  uint32_t out_dims[5];  // output extents along dims 1..4
  uint32_t n_tiles, num_tiles;
  int32_t N;      // rows of B
  int32_t n_out;  // output columns (N, or N/2 with GEGLU)
  int32_t tma_store;
  // residual operand of the TMA-store epilogue, loaded by TMA into the output staging tile itself at the start of the
  // tile (the load hides behind the main loop and costs no extra shared memory)
  int32_t res_tma;
  const float* bias;
  const __half* rowvec;
  int64_t rows_per_vec, ld_rowvec;
  const __half* residual;
  int64_t ld_res;
  int32_t act, out_dtype;
  int64_t ld_out;
  void* out;
  float out_scale;     // applied before the residual add (1 = off)
  float* gn_partial;   // [n_out / 8][gn_blocks][2] GroupNorm statistics of the output, or nullptr
  int64_t gn_blocks;
  int32_t epi_kind;    // EPI_* feature set of a specialised AUX epilogue body, or EPI_GENERIC
};

// Feature sets of the AUX epilogue of the TMA-store instance that have a body of their own, compiled with only their
// features (no activation, no GEGLU).  A residual is added as fmaf(x, out_scale, r) whatever out_scale is, so EPI_SCALE
// only marks out_scale without a residual.  Every other combination runs the generic body (EPI_GENERIC).
constexpr int EPI_ROWVEC = 1, EPI_RES = 2, EPI_STATS = 4, EPI_SCALE = 8, EPI_GENERIC = -1;
template <int F>
struct EpiKindTag {
  static constexpr int value = F;
};

template <int BLOCK_N, bool GEGLU>
struct IgemmCfg {
  static constexpr int OUT_TILE_N = GEGLU ? BLOCK_N / 2 : BLOCK_N;
  static constexpr int B_STAGE_BYTES = BLOCK_N * BLOCK_K * 2;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static constexpr int STAGING_BYTES = (OUT_TILE_N >= 64) ? (OUT_TILE_N / 64) * SLAB_BYTES : 0;
  static constexpr int AUX_BYTES = 1024;  // mbarriers
  // everything left of the 227 KB after the output staging tile is the {A, B} stage ring
  static constexpr int STAGES_RAW = (SMEM_OPT_IN_LIMIT - 1024 - STAGING_BYTES - AUX_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_RAW > 8 ? 8 : STAGES_RAW;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + STAGING_BYTES + AUX_BYTES + 1024 /*align*/;
  static constexpr int ACC = BLOCK_N / 2;  // fp32 accumulator registers per thread: m64 x BLOCK_N per warpgroup
  static_assert(SMEM_BYTES <= SMEM_OPT_IN_LIMIT, "stage ring + output staging exceed the shared memory of a block");
};

// The tile of work item w: its N-tile, its M-tile and the origin of the M-tile's box along view dims 1..4
struct IgemmTile {
  uint32_t n_tile, m_tile;
  uint32_t t1, t2, t3, t4;
};
__device__ __forceinline__ IgemmTile igemm_tile(const IgemmParams& p, uint32_t w) {
  IgemmTile t;
  t.n_tile = w % p.n_tiles;
  t.m_tile = w / p.n_tiles;
  uint32_t idx = t.m_tile;
  t.t1 = (idx % p.tiles[1]) * p.box[1];
  idx /= p.tiles[1];
  t.t2 = (idx % p.tiles[2]) * p.box[2];
  idx /= p.tiles[2];
  t.t3 = (idx % p.tiles[3]) * p.box[3];
  idx /= p.tiles[3];
  t.t4 = idx * p.box[4];
  return t;
}

// pointwise activations of the fused epilogue (GEGLU is handled separately: it pairs two accumulator columns)
__device__ __forceinline__ float apply_act(float x, int act) {
  switch (act) {
    case UAV_ACT_SILU: return silu_f(x);
    case UAV_ACT_RELU: return fmaxf(x, 0.f);
    case UAV_ACT_SIGMOID: return rcp_ftz(1.0f + ex2_ftz(-1.4426950408889634f * x));
    case UAV_ACT_TANH: return 1.0f - 2.0f * rcp_ftz(1.0f + ex2_ftz(2.8853900817779268f * x));
    case UAV_ACT_GELU: return gelu_erf_f(x);
    case UAV_ACT_QUICK_GELU: return x * rcp_ftz(1.0f + ex2_ftz(-2.4554669595930156f * x));  // x * sigmoid(1.702 x)
    default: return x;
  }
}
// the activation of an epilogue body compiled for ACT: UAV_ACT_NONE (also GEGLU, which apply_act leaves alone), one
// activation, or ACT_RUNTIME for the run-time `act`
constexpr int ACT_RUNTIME = -1;
template <int ACT>
struct ActTag {
  static constexpr int value = ACT;
};
template <int ACT>
__device__ __forceinline__ float epi_act(float x, int act) {
  if constexpr (ACT == UAV_ACT_NONE) return x;
  else if constexpr (ACT == ACT_RUNTIME) return act != UAV_ACT_NONE ? apply_act(x, act) : x;
  else return apply_act(x, ACT);
}
// Sums each of the NV values of a lane over the 32 lanes of the warp (NV a power of two <= 32) and returns sum number
// lane >> (5 - log2 NV).  Recursive halving: at the step of offset o a lane keeps the half of its values that bit o of
// its lane index picks and adds its partner's partial of that half, so the warp shuffles NV - 1 times (plus once per
// step left over when NV < 32) instead of 5 NV times.  Each partial adds the same two lanes' partials as the butterfly
// v += shfl_xor(v, o), o = 16 .. 1, so every sum is bitwise the butterfly's.
template <int NV, int O = 16>
__device__ __forceinline__ float warp_sum_transpose(float (&v)[NV], int lane) {
  static_assert(NV >= 1 && NV <= 32 && (NV & (NV - 1)) == 0, "NV must be a power of two <= 32");
  constexpr int HALF = NV * O / 32;  // values a lane still holds after this step
  if constexpr (HALF >= 1) {
    const bool upper = (lane & O) != 0;
#pragma unroll
    for (int i = 0; i < HALF; ++i) {
      const float send = upper ? v[i] : v[i + HALF];
      const float keep = upper ? v[i + HALF] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, O);
    }
  } else {
    v[0] += __shfl_xor_sync(0xffffffffu, v[0], O);
  }
  if constexpr (O > 1) return warp_sum_transpose<NV, O / 2>(v, lane);
  else return v[0];
}

// TMA_EPI: smem-staged TMA-store epilogue (aligned fp16 output, >= 64-column tiles) vs direct per-element stores.
// AUX: the epilogue has a row vector / residual / activation / statistics on top of the bias (compiled out otherwise:
// the hot bias-only GEMMs get a small loop body).
//
// Persistent CTAs (one per SM) walk the tiles; thread 0 streams {A 128x64, B BLOCK_Nx64} stages through an mbarrier
// ring, warpgroup g of the two consumer warpgroups multiplies rows [64 g, 64 g + 64) of every stage into its register
// accumulator (wgmma m64 x BLOCK_N x 16) and runs the epilogue of those rows.  The producer runs ahead into the next tile
// while the epilogue of the current one executes.
template <int BLOCK_N, bool GEGLU, bool TMA_EPI, bool AUX>
__global__ void __launch_bounds__(NUM_THREADS, 1)
    igemm_kernel(const __grid_constant__ IgemmParams p) {
  using Cfg = IgemmCfg<BLOCK_N, GEGLU>;
  static_assert(!TMA_EPI || Cfg::OUT_TILE_N >= 64, "TMA-store epilogue needs >= 64-column output tiles");
  constexpr int OUT_TILE_N = Cfg::OUT_TILE_N;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align1024(smem_raw);
  uint8_t* staging = smem + STAGES * Cfg::STAGE_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(staging + Cfg::STAGING_BYTES);
  const RingBarriers<STAGES> ring(bars);  // one arrival per consumer warp on `empty`
  uint64_t* res_bar = bars + 2 * STAGES;  // residual tile landed in the staging tile

  const int warp_idx = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.map_a);
    tma_prefetch_desc(&p.map_b);
    if (TMA_EPI) tma_prefetch_desc(&p.map_out);
    if (TMA_EPI && p.res_tma) tma_prefetch_desc(&p.map_res);
    ring.init(NUM_EPI_THREADS / 32);
    mbar_init(res_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  const int num_kb = p.num_taps * p.kblocks_per_tap;

  if (warp_idx < 4) {
    // =============================== TMA producer ===============================
    setmaxnreg_dec<PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      RingPos<STAGES> pos;
      for (uint32_t w = blockIdx.x; w < p.num_tiles; w += gridDim.x) {
        const IgemmTile t = igemm_tile(p, w);
        for (int tap = 0; tap < p.num_taps; ++tap) {
          const int o0 = p.tap_off[tap][0], o1 = p.tap_off[tap][1], o2 = p.tap_off[tap][2],
                    o3 = p.tap_off[tap][3], o4 = p.tap_off[tap][4];
          for (int kc = 0; kc < p.kblocks_per_tap; ++kc) {
            // out-of-bounds parts of a box (image border = zero padding, K tail, N tail) are zero-filled and counted
            uint64_t* full = ring.acquire(pos, Cfg::STAGE_BYTES);
            uint8_t* sa = smem + pos.stage * Cfg::STAGE_BYTES;
            uint8_t* sb = sa + A_STAGE_BYTES;
            tma_load_5d(&p.map_a, full, sa, kc * BLOCK_K + o0, (int)t.t1 + o1, (int)t.t2 + o2, (int)t.t3 + o3,
                        (int)t.t4 + o4);
            const int kcoord = tap * p.k_per_tap + kc * BLOCK_K;
            if (GEGLU) {  // value rows, then the matching gate rows
              tma_load_2d(&p.map_b, full, sb, kcoord, t.n_tile * (BLOCK_N / 2));
              tma_load_2d(&p.map_b, full, sb + Cfg::B_STAGE_BYTES / 2, kcoord, p.N / 2 + t.n_tile * (BLOCK_N / 2));
            } else {
              tma_load_2d(&p.map_b, full, sb, kcoord, t.n_tile * BLOCK_N);
            }
            pos.advance();
          }
        }
      }
    }
    return;
  }

  // =============================== wgmma consumers + epilogue ===============================
  setmaxnreg_inc<CONSUMER_REGS>();
  const int et = threadIdx.x - 128;  // 0..255
  const int wg = et >> 7;            // rows [64 wg, +64) of the tile
  const int cw = et >> 5;            // rows [16 cw, +16): the accumulator rows of this warp
  const int lq = lane >> 2, lr = lane & 3;
  uint32_t lrow[2], l1[2], l2[2], l3[2], l4[2];  // tile rows of this thread and their box coordinates
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    uint32_t r = 16 * cw + lq + 8 * h;
    lrow[h] = r;
    l1[h] = r % p.box[1];
    r /= p.box[1];
    l2[h] = r % p.box[2];
    r /= p.box[2];
    l3[h] = r % p.box[3];
    r /= p.box[3];
    l4[h] = r;
  }
  RingPos<STAGES> pos;
  uint32_t res_phase = 0;
  float acc[Cfg::ACC];
#pragma unroll
  for (int i = 0; i < Cfg::ACC; ++i) acc[i] = 0.f;

  for (uint32_t w = blockIdx.x; w < p.num_tiles; w += gridDim.x) {
    const IgemmTile tile = igemm_tile(p, w);
    const int n_base = tile.n_tile * OUT_TILE_N;

    if constexpr (TMA_EPI) {
      if (et == 0) {
        // the store of the previous tile must have read the staging tile before it is refilled
        tma_store_wait_read<0>();
        if (AUX && p.res_tma) {
          uint32_t bytes = 0;
#pragma unroll
          for (int sl = 0; sl < OUT_TILE_N / 64; ++sl)
            if (n_base + sl * 64 < p.n_out) bytes += SLAB_BYTES;
          mbar_expect_tx(res_bar, bytes);
#pragma unroll
          for (int sl = 0; sl < OUT_TILE_N / 64; ++sl)
            if (n_base + sl * 64 < p.n_out)
              tma_load_5d(&p.map_res, res_bar, staging + sl * SLAB_BYTES, n_base + sl * 64, (int)tile.t1,
                          (int)tile.t2, (int)tile.t3, (int)tile.t4);
        }
      }
    }

    // ---- main loop: one stage = 4 k16 steps; the stage of step kb - 1 is released once step kb is in flight ----
    int prev = 0;
    for (int kb = 0; kb < num_kb; ++kb) {
      ring.wait_full(pos);
      const uint32_t sa = smem_u32(smem + pos.stage * Cfg::STAGE_BYTES) + wg * (64 * 128);
      const uint32_t sb = smem_u32(smem + pos.stage * Cfg::STAGE_BYTES + A_STAGE_BYTES);
      const uint64_t adesc = gmma_desc_sw128(sa), bdesc = gmma_desc_sw128(sb);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BLOCK_K / 16; ++k) wgmma_ss(acc, adesc + 2 * k, bdesc + 2 * k, (kb | k) != 0);
      wgmma_commit();
      if (kb > 0) {
        wgmma_wait<1>();
        if (lane == 0) mbar_arrive(&ring.empty[prev]);
      }
      prev = pos.stage;
      pos.advance();
    }
    wgmma_wait<0>();
    wgmma_fence_operands(acc);
    if (lane == 0) mbar_arrive(&ring.empty[prev]);

    // ---- epilogue ----
    bool row_ok[2];
    int64_t out_row[2];
    const __half* rv[2];
    const __half* res[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint32_t o1 = tile.t1 + l1[h], o2 = tile.t2 + l2[h], o3 = tile.t3 + l3[h], o4 = tile.t4 + l4[h];
      row_ok[h] = o1 < p.out_dims[1] && o2 < p.out_dims[2] && o3 < p.out_dims[3] && o4 < p.out_dims[4];
      out_row[h] = ((static_cast<int64_t>(o4) * p.out_dims[3] + o3) * p.out_dims[2] + o2) * p.out_dims[1] + o1;
      rv[h] = (AUX && p.rowvec != nullptr && row_ok[h]) ? p.rowvec + (out_row[h] / p.rows_per_vec) * p.ld_rowvec
                                                         : nullptr;
      res[h] = (AUX && !TMA_EPI && p.residual != nullptr && row_ok[h]) ? p.residual + out_row[h] * p.ld_res : nullptr;
    }
    if constexpr (TMA_EPI) {
      bar_sync<1, NUM_EPI_THREADS>();  // thread 0 saw the previous store release the staging tile
      if constexpr (AUX) {
        if (p.res_tma) {
          mbar_wait(res_bar, res_phase);
          res_phase ^= 1;
        }
      }
    }
    // The epilogue runs in passes of at most 128 columns over acc[0, EPI_ACC), shifting the next columns down after
    // each pass: an unrolled 256-column AUX epilogue would be twice the code and no longer fit the instruction cache.
    constexpr int EPI_N = GEGLU ? OUT_TILE_N : (OUT_TILE_N < 128 ? OUT_TILE_N : 128);
    constexpr int EPI_ACC = EPI_N / 2;
    // GroupNorm statistics of one pass: stats[2 jb], stats[2 jb + 1] = {sum, sum of squares} of column group jb over the
    // thread's rows; the warp's 16 rows x 8 columns per group are one block
    auto store_stats = [&](auto& stats, int pass) {
      // lane l ends up with the warp's sum of stats[l >> SHIFT]
      constexpr int SHIFT = EPI_N == 128 ? 0 : 1;
      static_assert(!TMA_EPI || EPI_N / 4 == (32 >> SHIFT), "one statistics value per 2^SHIFT lanes");
      const float s = warp_sum_transpose(stats, lane);
      const int value = lane >> SHIFT;
      const int oct = ((n_base + pass * EPI_N) >> 3) + (value >> 1);
      const int64_t blk = static_cast<int64_t>(tile.m_tile) * 8 + cw;
      if ((lane & ((1 << SHIFT) - 1)) == 0 && blk < p.gn_blocks && oct * 8 < p.n_out)
        p.gn_partial[(static_cast<int64_t>(oct) * p.gn_blocks + blk) * 2 + (value & 1)] = s;
    };
    auto epilogue = [&](auto act_tag) {
      [[maybe_unused]] constexpr int ACT = decltype(act_tag)::value;
#pragma unroll 1
      for (int pass = 0; pass < OUT_TILE_N / EPI_N; ++pass) {
        // GroupNorm statistics of 8-column group jb over the thread's rows: sum at [2 jb], sum of squares at [2 jb + 1]
        [[maybe_unused]] float stats[EPI_N / 4];
#pragma unroll
        for (int jb = 0; jb < EPI_N / 8; ++jb) {
          const int col = pass * EPI_N + jb * 8 + 2 * lr;  // column inside the output tile (this thread: col, col + 1)
          const int n = n_base + col;
          const bool ok0 = n < p.n_out, ok1 = n + 1 < p.n_out;
          float b0 = 0.f, b1 = 0.f, g0 = 0.f, g1 = 0.f;
          if (p.bias != nullptr) {
            if (ok0) b0 = __ldg(p.bias + n);
            if (ok1) b1 = __ldg(p.bias + n + 1);
            if (GEGLU) {
              if (ok0) g0 = __ldg(p.bias + p.N / 2 + n);
              if (ok1) g1 = __ldg(p.bias + p.N / 2 + n + 1);
            }
          }
          float gs = 0.f, gq = 0.f;  // GroupNorm statistics of this 8-column group over the thread's rows
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const float a0 = acc[4 * jb + 2 * h], a1 = acc[4 * jb + 2 * h + 1];
            float x0, x1;
            if constexpr (GEGLU) {
              constexpr int GJ = OUT_TILE_N / 8;  // gate columns start at accumulator column OUT_TILE_N
              const float q0 = acc[4 * (jb + GJ) + 2 * h], q1 = acc[4 * (jb + GJ) + 2 * h + 1];
              x0 = (a0 + b0) * gelu_erf_f(q0 + g0);
              x1 = (a1 + b1) * gelu_erf_f(q1 + g1);
            } else {
              x0 = a0 + b0;
              x1 = a1 + b1;
            }
            // staging address of (row, col): 16-byte chunk (col & 63) / 8 of the row, CU_TENSOR_MAP_SWIZZLE_128B
            const uint32_t row = lrow[h];
            uint8_t* sp = staging + (col >> 6) * SLAB_BYTES + row * 128 + ((((col & 63) >> 3) ^ (row & 7)) << 4) + (col & 7) * 2;
            if constexpr (AUX) {
              if (rv[h] != nullptr) {
                if (ok0) x0 += __half2float(rv[h][n]);
                if (ok1) x1 += __half2float(rv[h][n + 1]);
              }
              x0 = epi_act<ACT>(x0, p.act);
              x1 = epi_act<ACT>(x1, p.act);
              if (TMA_EPI && p.res_tma) {  // residual of this row from the staging tile (same swizzle as the store)
                const float2 r = __half22float2(*reinterpret_cast<const __half2*>(sp));
                x0 = fmaf(x0, p.out_scale, r.x);
                x1 = fmaf(x1, p.out_scale, r.y);
              } else if (res[h] != nullptr) {
                x0 = fmaf(x0, p.out_scale, ok0 ? __half2float(res[h][n]) : 0.f);
                x1 = fmaf(x1, p.out_scale, ok1 ? __half2float(res[h][n + 1]) : 0.f);
              } else if (p.out_scale != 1.0f) {
                x0 *= p.out_scale;
                x1 *= p.out_scale;
              }
              if (row_ok[h] && ok0) {
                gs += x0 + x1;
                gq = fmaf(x0, x0, fmaf(x1, x1, gq));
              }
            }
            if constexpr (TMA_EPI) {
              *reinterpret_cast<uint32_t*>(sp) = pack_half2_sat(x0, x1);
            } else if (row_ok[h]) {
              if (p.out_dtype == UAV_F16) {
                __half* op = reinterpret_cast<__half*>(p.out) + out_row[h] * p.ld_out + n;
                if (ok0) op[0] = __float2half_rn(fminf(fmaxf(x0, -65504.f), 65504.f));
                if (ok1) op[1] = __float2half_rn(fminf(fmaxf(x1, -65504.f), 65504.f));
              } else {
                float* op = reinterpret_cast<float*>(p.out) + out_row[h] * p.ld_out + n;
                if (ok0) op[0] = x0;
                if (ok1) op[1] = x1;
              }
            }
          }
          if constexpr (AUX && TMA_EPI) {
            stats[2 * jb] = gs;
            stats[2 * jb + 1] = gq;
          }
        }
        if constexpr (AUX && TMA_EPI) {
          if (p.gn_partial != nullptr) store_stats(stats, pass);  // warp-uniform
        }
        if (pass + 1 < OUT_TILE_N / EPI_N) {
#pragma unroll
          for (int i = 0; i + EPI_ACC < Cfg::ACC; ++i) acc[i] = acc[i + EPI_ACC];
        }
      }
    };
    // The AUX body of one feature set (EPI_*) of the TMA-store epilogue without activation.  It makes each of the generic
    // body's run-time decisions once per tile or once per 8-column group instead of once per element pair, and keeps its
    // fp32 operations and their order: (acc + bias) + rowvec, fmaf(x, out_scale, residual) or x * out_scale, statistics,
    // saturating fp16, so outputs and statistics are bitwise the generic body's.
    auto epilogue_kind = [&](auto kind_tag) {
      constexpr int F = decltype(kind_tag)::value;
      constexpr bool ROWVEC = (F & EPI_ROWVEC) != 0, RES = (F & EPI_RES) != 0, STATS = (F & EPI_STATS) != 0,
                     SCALE = (F & EPI_SCALE) != 0;
      const bool has_bias = p.bias != nullptr;  // float2 loads: the host checked 8-byte alignment
      // row vectors of the thread's two rows; a row outside the output takes the other row's (its value is never
      // stored or counted), and when both rows share one, it is loaded once per column group
      [[maybe_unused]] const __half* rvp[2];
      [[maybe_unused]] bool rv_shared = true;
      if constexpr (ROWVEC) {
        rvp[0] = rv[0] != nullptr ? rv[0] : (rv[1] != nullptr ? rv[1] : p.rowvec);
        rvp[1] = rv[1] != nullptr ? rv[1] : rvp[0];
        rv_shared = rvp[0] == rvp[1];
      }
#pragma unroll 1
      for (int pass = 0; pass < OUT_TILE_N / EPI_N; ++pass) {
        [[maybe_unused]] float stats[EPI_N / 4];
#pragma unroll
        for (int jb = 0; jb < EPI_N / 8; ++jb) {
          const int col = pass * EPI_N + jb * 8 + 2 * lr;
          const int n = n_base + col;
          float gs = 0.f, gq = 0.f;
          // n_out % 8 == 0 on the TMA-store path: a group of 8 columns is wholly inside or wholly outside the output
          if (n_base + pass * EPI_N + jb * 8 < p.n_out) {
            float2 b = make_float2(0.f, 0.f);
            if (has_bias) b = __ldg(reinterpret_cast<const float2*>(p.bias + n));
            [[maybe_unused]] float2 rvf[2];
            if constexpr (ROWVEC) {
              rvf[0] = __half22float2(__ldg(reinterpret_cast<const __half2*>(rvp[0] + n)));
              rvf[1] = rv_shared ? rvf[0] : __half22float2(__ldg(reinterpret_cast<const __half2*>(rvp[1] + n)));
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              float x0 = acc[4 * jb + 2 * h] + b.x, x1 = acc[4 * jb + 2 * h + 1] + b.y;
              const uint32_t row = lrow[h];
              uint8_t* sp = staging + (col >> 6) * SLAB_BYTES + row * 128 + ((((col & 63) >> 3) ^ (row & 7)) << 4) + (col & 7) * 2;
              if constexpr (ROWVEC) {
                x0 += rvf[h].x;
                x1 += rvf[h].y;
              }
              if constexpr (RES) {
                const float2 r = __half22float2(*reinterpret_cast<const __half2*>(sp));
                x0 = fmaf(x0, p.out_scale, r.x);
                x1 = fmaf(x1, p.out_scale, r.y);
              } else if constexpr (SCALE) {
                x0 *= p.out_scale;
                x1 *= p.out_scale;
              }
              if constexpr (STATS) {
                if (row_ok[h]) {
                  gs += x0 + x1;
                  gq = fmaf(x0, x0, fmaf(x1, x1, gq));
                }
              }
              *reinterpret_cast<uint32_t*>(sp) = pack_half2_sat(x0, x1);
            }
          }
          if constexpr (STATS) {
            stats[2 * jb] = gs;
            stats[2 * jb + 1] = gq;
          }
        }
        if constexpr (STATS) store_stats(stats, pass);
        if (pass + 1 < OUT_TILE_N / EPI_N) {
#pragma unroll
          for (int i = 0; i + EPI_ACC < Cfg::ACC; ++i) acc[i] = acc[i + EPI_ACC];
        }
      }
    };
    // The activation is the same for the whole launch, so it is picked here, once per tile, and each epilogue body is
    // compiled for one activation: the run-time switch inlined at every element pair made the AUX epilogue several
    // times as long as the one without activation, and launches without one or with SiLU pay for none of it.  The
    // feature sets the UNet and the VAE launch have bodies of their own, picked the same way.
    auto epilogue_generic = [&] {
      if (p.act == UAV_ACT_SILU) epilogue(ActTag<UAV_ACT_SILU>{});
      else if (p.act == UAV_ACT_NONE || p.act == UAV_ACT_GEGLU) epilogue(ActTag<UAV_ACT_NONE>{});
      else epilogue(ActTag<ACT_RUNTIME>{});
    };
    if constexpr (AUX && TMA_EPI && !GEGLU) {
      switch (p.epi_kind) {
        case EPI_ROWVEC | EPI_STATS: epilogue_kind(EpiKindTag<EPI_ROWVEC | EPI_STATS>{}); break;
        case EPI_RES | EPI_STATS: epilogue_kind(EpiKindTag<EPI_RES | EPI_STATS>{}); break;
        case EPI_RES: epilogue_kind(EpiKindTag<EPI_RES>{}); break;
        case EPI_STATS: epilogue_kind(EpiKindTag<EPI_STATS>{}); break;
        case EPI_SCALE: epilogue_kind(EpiKindTag<EPI_SCALE>{}); break;
        default: epilogue_generic();
      }
    } else if constexpr (AUX) {
      epilogue_generic();
    } else {
      epilogue(ActTag<UAV_ACT_NONE>{});
    }
    if constexpr (TMA_EPI) {
      // publish the staged tile to the async proxy and store it with TMA (clips OOB rows)
      fence_proxy_async();
      bar_sync<1, NUM_EPI_THREADS>();
      if (et == 0) {
#pragma unroll
        for (int sl = 0; sl < OUT_TILE_N / 64; ++sl)
          if (n_base + sl * 64 < p.n_out)
            tma_store_5d(&p.map_out, staging + sl * SLAB_BYTES, n_base + sl * 64, (int)tile.t1, (int)tile.t2,
                         (int)tile.t3, (int)tile.t4);
        tma_store_commit();
      }
    }
  }
  if (TMA_EPI && et == 0) tma_store_wait_read<0>();
}

// ---------------------------------------------------------------------------------------
// host: descriptor + launch
// ---------------------------------------------------------------------------------------
// Input view and tap table of one launch.  The view has the channels in dim 0 and the pixels in dims 1..4, which the
// M-tile box (extents multiplying to 128) tiles; the output pixels have the extents out_dims[1..4].
struct IgemmDesc {
  const void* a = nullptr;
  uint64_t a_dims[5] = {};     // dim0 = channels
  uint64_t a_strides[5] = {};  // elements; a_strides[0] == 1
  uint32_t box[5] = {};        // box[0] = 64
  uint32_t tiles[5] = {};
  uint32_t out_dims[5] = {};
  int num_taps = 0;
  int32_t tap_off[MAX_TAPS][5] = {};
  int k_per_tap = 0;
  // optional strided output view (elements) for dims 1..4; 0 = dense (derived from ld_out / out_dims).
  // Only the TMA-store epilogue understands it (used by the fused nearest-x2 upsample + 3x3 conv).
  uint64_t out_strides[5] = {};
};

// persistent launch: one CTA per SM, or per tile when there are fewer tiles
template <int BLOCK_N, bool GEGLU>
static uav_status_t launch_instance(IgemmParams& p, cudaStream_t stream) {
  using Cfg = IgemmCfg<BLOCK_N, GEGLU>;
  constexpr int smem = Cfg::SMEM_BYTES;
  const uint32_t sms = (uint32_t)num_sms();
  const dim3 grid(p.num_tiles < sms ? p.num_tiles : sms);
  const bool aux = p.rowvec != nullptr || p.residual != nullptr || (p.act != UAV_ACT_NONE && p.act != UAV_ACT_GEGLU) ||
                   p.out_scale != 1.0f || p.gn_partial != nullptr;
  p.epi_kind = EPI_GENERIC;
  if (p.tma_store && !GEGLU && p.act == UAV_ACT_NONE && (reinterpret_cast<uintptr_t>(p.bias) & 7) == 0) {
    const int kind = (p.rowvec != nullptr ? EPI_ROWVEC : 0) | (p.res_tma ? EPI_RES : 0) |
                     (p.gn_partial != nullptr ? EPI_STATS : 0) |
                     (p.residual == nullptr && p.out_scale != 1.0f ? EPI_SCALE : 0);
    for (int k : {EPI_ROWVEC | EPI_STATS, EPI_RES | EPI_STATS, EPI_RES, EPI_STATS, EPI_SCALE})
      if (kind == k) p.epi_kind = kind;
  }
  if constexpr (Cfg::OUT_TILE_N >= 64) {
    if (p.tma_store) {
      return aux ? launch_opted_in<igemm_kernel<BLOCK_N, GEGLU, true, true>>(grid, NUM_THREADS, smem, stream, p)
                 : launch_opted_in<igemm_kernel<BLOCK_N, GEGLU, true, false>>(grid, NUM_THREADS, smem, stream, p);
    }
  }
  return launch_opted_in<igemm_kernel<BLOCK_N, GEGLU, false, true>>(grid, NUM_THREADS, smem, stream, p);
}

// Time of one 256-column tile over one 128-column tile of the same GEMM (GEGLU: 128 over 64 output columns), from
// tools/bench_igemm.py on an H100 80GB HBM3 at 700 W.  On launches of many waves (twice the ratio of the kernel times at
// the two widths) 3x3 convs give 1.46 to 1.62, the (3,1,1) temporal conv 1.55 and GEGLU 512->4096 1.69 and 1.90.  Launches
// of few waves gain less: the h720 convs 512->512 on 16 x 45x80 (8 wide against 15 narrow waves) and 1024->1024 on
// 16 x 23x40 (5 against 9) took 0.47 and 0.56 ms with 256-column tiles against 0.41 and 0.49 ms with 128-column tiles.
// 1.9 keeps both of those at 128 columns and still takes the wide tiles for the GEGLU and the many-wave convolutions.
constexpr double WIDE_TILE_COST = 1.9;

// A persistent launch takes ceil(tiles / SMs) waves; the wide tiles win when their fewer waves, each WIDE_TILE_COST times
// as long, finish before the narrow ones.  out_wide = output columns of a wide tile.
static bool wide_tile_pays(uint64_t m_tiles, int64_t n_out, int64_t out_wide) {
  const uint64_t sms = (uint64_t)num_sms();
  const uint64_t waves_wide = (m_tiles * ((n_out + out_wide - 1) / out_wide) + sms - 1) / sms;
  const uint64_t waves_narrow = (m_tiles * ((2 * n_out + out_wide - 1) / out_wide) + sms - 1) / sms;
  return (double)waves_wide * WIDE_TILE_COST < (double)waves_narrow;
}

// out[pixel][n] = epilogue(sum over the taps of d of A[pixel + tap][c] * w[n][tap][c]) for the N rows of w
static uav_status_t launch_igemm(const IgemmDesc& d, const void* w, int64_t N, void* out, const uav_epilogue_t* e,
                                 cudaStream_t stream) {
  UAV_REQUIRE(e != nullptr, "igemm: epilogue descriptor is NULL");
  UAV_REQUIRE(d.a && w && out, "igemm: null pointer");
  UAV_REQUIRE(d.k_per_tap > 0 && d.k_per_tap % 8 == 0,
              "igemm: input channels (%d) must be a positive multiple of 8", d.k_per_tap);
  UAV_REQUIRE(aligned16(d.a) && aligned16(w), "igemm: operands must be 16-byte aligned");
  const bool geglu = e->act == UAV_ACT_GEGLU;
  UAV_REQUIRE(!geglu || (N % 128 == 0), "igemm: GEGLU needs N %% 128 == 0 (N=%lld)",
              (long long)N);

  IgemmParams p;
  memset(&p, 0, sizeof(p));
  uint64_t m_tiles = 1;
  for (int i = 1; i < 5; ++i) m_tiles *= d.tiles[i];
  // 256-column tiles (128 output columns with GEGLU) for convolutions and GEGLU with N >= 256, unless they lose to wave
  // quantisation; 128-column tiles for the rest of N > 64.  Single-tap GEMMs without GEGLU (Linear, 1x1 conv) keep
  // 128-column tiles: their short main loop does not hide the twice as long epilogue of a 256-column tile (measured: no
  // gain at K = 2048, 10% slower at K = 512).  GEGLU-256 needs N % 256 == 0 so that the value box never reads gate rows.
  const int64_t n_out = geglu ? N / 2 : N;
  int block_n;
  if (geglu) block_n = (N % 256 == 0 && wide_tile_pays(m_tiles, n_out, 128)) ? 256 : 128;
  else if (N >= 256 && d.num_taps > 1 && wide_tile_pays(m_tiles, n_out, 256)) block_n = 256;
  else if (N > 64) block_n = 128;
  else if (N > 32) block_n = 64;
  else if (N > 16) block_n = 32;
  else block_n = 16;

  // A map.  L2 promotion 256B: a 128-byte k-block fetch also brings the neighbouring 128 bytes of the row into L2, i.e.
  // the next k-block of the same rows
  for (int i = 0; i < 5; ++i)
    UAV_REQUIRE(d.a_dims[i] >= 1 && d.box[i] >= 1 && d.box[i] <= 256, "igemm: bad A dim/box %d", i);
  cuuint64_t a_strides[4];
  for (int i = 1; i < 5; ++i) {
    a_strides[i - 1] = d.a_strides[i] * 2;
    UAV_REQUIRE(a_strides[i - 1] % 16 == 0, "igemm: A stride %d not 16-byte aligned", i);
  }
  uav_status_t st;
  if ((st = encode_tensor_map(&p.map_a, d.a, 5, d.a_dims, a_strides, d.box, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                              "igemm(A)")) != UAV_OK)
    return st;
  // B map: [N][K_total] K-major
  const int64_t k_total = (int64_t)d.num_taps * d.k_per_tap;
  const cuuint64_t b_dims[2] = {(cuuint64_t)k_total, (cuuint64_t)N}, b_stride = (cuuint64_t)k_total * 2;
  const cuuint32_t b_box[2] = {64, (cuuint32_t)(geglu ? block_n / 2 : block_n)};
  if ((st = encode_tensor_map(&p.map_b, w, 2, b_dims, &b_stride, b_box, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                              "igemm(B)")) != UAV_OK)
    return st;
  UAV_REQUIRE(d.num_taps >= 1 && d.num_taps <= MAX_TAPS, "igemm: bad tap count %d", d.num_taps);
  memcpy(p.tap_off, d.tap_off, sizeof(int32_t) * 5 * d.num_taps);
  p.num_taps = d.num_taps;
  p.k_per_tap = d.k_per_tap;
  p.kblocks_per_tap = (d.k_per_tap + BLOCK_K - 1) / BLOCK_K;
  uint32_t box_prod = 1;
  for (int i = 0; i < 5; ++i) {
    p.box[i] = d.box[i];
    p.tiles[i] = d.tiles[i];
    p.out_dims[i] = d.out_dims[i];
    if (i >= 1) box_prod *= d.box[i];
  }
  UAV_REQUIRE(box_prod == BLOCK_M && d.box[0] == 64, "igemm: M-tile box must cover 128 rows");
  p.N = (int32_t)N;
  p.n_out = (int32_t)n_out;
  const int out_tile_n = geglu ? block_n / 2 : block_n;
  p.n_tiles = (uint32_t)((p.n_out + out_tile_n - 1) / out_tile_n);
  UAV_REQUIRE(m_tiles * p.n_tiles < (1ull << 31), "igemm: too many tiles");
  p.num_tiles = (uint32_t)(m_tiles * p.n_tiles);
  const bool can_tma = out_tile_n >= 64 && e->out_dtype == UAV_F16 && p.n_out % 8 == 0 && e->ld_out % 8 == 0 &&
                       aligned16(out) &&
                       (e->residual == nullptr || (e->ld_res % 8 == 0 && aligned16(e->residual))) &&
                       (e->rowvec == nullptr || (e->ld_rowvec % 8 == 0 && aligned16(e->rowvec)));
  p.res_tma = (can_tma && e->residual != nullptr) ? 1 : 0;
  p.bias = e->bias;
  p.rowvec = reinterpret_cast<const __half*>(e->rowvec);
  p.rows_per_vec = e->rows_per_vec > 0 ? e->rows_per_vec : 1;
  p.ld_rowvec = e->ld_rowvec;
  p.residual = reinterpret_cast<const __half*>(e->residual);
  p.ld_res = e->ld_res;
  p.act = e->act;
  p.out_dtype = e->out_dtype;
  p.ld_out = e->ld_out;
  p.out = out;
  p.out_scale = e->out_scale == 0.0f ? 1.0f : e->out_scale;
  p.gn_partial = reinterpret_cast<float*>(e->gn_partial);
  p.gn_blocks = e->gn_blocks;
  UAV_REQUIRE(!(geglu && p.out_scale != 1.0f), "igemm: out_scale is not supported with GEGLU");
  UAV_REQUIRE(p.ld_out >= p.n_out, "igemm: ld_out (%lld) < output columns (%d)",
              (long long)p.ld_out, p.n_out);
  UAV_REQUIRE(e->out_dtype == UAV_F16 || e->out_dtype == UAV_F32, "igemm: bad out_dtype");
  UAV_REQUIRE(e->act >= UAV_ACT_NONE && e->act <= UAV_ACT_QUICK_GELU, "igemm: bad activation");
  if (p.num_tiles == 0) return UAV_OK;

  // TMA-store epilogue (smem-staged, fully coalesced, clips partial tiles) whenever the output
  // is an aligned fp16 tensor with at least 64-column tiles; otherwise per-row direct stores.
  p.tma_store = can_tma ? 1 : 0;
  if (p.gn_partial != nullptr) {
    UAV_REQUIRE(can_tma && !geglu && d.out_strides[1] == 0,
                "igemm: GroupNorm statistics need the dense fp16 TMA-store epilogue (n_out >= 33, 16-byte aligned) without GEGLU");
    UAV_REQUIRE(p.gn_blocks == (int64_t)m_tiles * 8, "igemm: gn_blocks is %lld, this launch produces %lld blocks",
                (long long)p.gn_blocks, (long long)m_tiles * 8);
  }
  UAV_REQUIRE(d.out_strides[1] == 0 || (can_tma && p.residual == nullptr && p.rowvec == nullptr),
              "igemm: a strided output view needs the TMA-store epilogue without residual / row vector");
  if (can_tma) {
    // output and residual: n_out columns over the output pixels, stored in boxes of 64 columns x the M-tile box
    cuuint64_t o_dims[5] = {(cuuint64_t)p.n_out}, o_strides[4], r_strides[4];
    uint64_t o_el = (uint64_t)p.ld_out, r_el = (uint64_t)p.ld_res;
    for (int i = 1; i < 5; ++i) {
      o_dims[i] = d.out_dims[i];
      o_strides[i - 1] = (d.out_strides[i] ? d.out_strides[i] : o_el) * 2;
      r_strides[i - 1] = r_el * 2;
      o_el *= d.out_dims[i];
      r_el *= d.out_dims[i];
    }
    if ((st = encode_tensor_map(&p.map_out, out, 5, o_dims, o_strides, d.box, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                                "igemm(out)")) != UAV_OK)
      return st;
    if (p.res_tma && (st = encode_tensor_map(&p.map_res, p.residual, 5, o_dims, r_strides, d.box,
                                             CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "igemm(residual)")) != UAV_OK)
      return st;
  }

  if (geglu) return block_n == 256 ? launch_instance<256, true>(p, stream) : launch_instance<128, true>(p, stream);
  switch (block_n) {
    case 256: return launch_instance<256, false>(p, stream);
    case 128: return launch_instance<128, false>(p, stream);
    case 64: return launch_instance<64, false>(p, stream);
    case 32: return launch_instance<32, false>(p, stream);
    default: return launch_instance<16, false>(p, stream);
  }
}

// The (tw, th) rectangle with tw * th == 128 that wastes the fewest rows of a W x H image: the M-tile box of every launch
// over images, and the tiling uav_gn_partial_blocks counts statistics blocks over.
struct TileRect {
  uint32_t w, h;
};
static TileRect pick_tile_2d(int64_t W, int64_t H) {
  TileRect best_rect{};
  int64_t best = -1;
  for (uint32_t w = 128; w >= 1; w >>= 1) {
    const uint32_t h = 128 / w;
    const int64_t cover = ((W + w - 1) / w) * w * ((H + h - 1) / h) * h;
    if (best < 0 || cover < best) {
      best = cover;
      best_rect = {w, h};
    }
  }
  return best_rect;
}

// Dense channels-last input view: `channels` channels at pixel stride `ld`, under the outer extents ext (innermost
// first), tiled by the M-tile box.  The output pixels have the same extents.
static void dense_view(IgemmDesc& d, const void* x, int64_t ld, int64_t channels, const int64_t (&ext)[4],
                       const uint32_t (&box)[4]) {
  d.a = x;
  d.k_per_tap = (int)channels;
  d.a_dims[0] = (uint64_t)channels;
  d.a_strides[0] = 1;
  d.box[0] = 64;
  d.tiles[0] = 1;
  d.out_dims[0] = 1;
  uint64_t stride = (uint64_t)ld;
  for (int i = 1; i < 5; ++i) {
    d.a_dims[i] = (uint64_t)ext[i - 1];
    d.a_strides[i] = stride;
    d.box[i] = box[i - 1];
    d.tiles[i] = (uint32_t)((ext[i - 1] + box[i - 1] - 1) / box[i - 1]);
    d.out_dims[i] = (uint32_t)ext[i - 1];
    stride *= (uint64_t)ext[i - 1];
  }
}

// One axis of a tap grid: `extent` taps along view dim `dim`, at offsets start, start + 1, ...
struct TapAxis {
  int dim, extent, start;
};
// Appends every tap of the grid in the order the weights are packed: the first axis outermost, the last one fastest.
static void add_tap_grid(IgemmDesc& d, std::initializer_list<TapAxis> axes) {
  int count = 1;
  for (const TapAxis& ax : axes) count *= ax.extent;
  for (int t = 0; t < count; ++t) {
    int32_t* o = d.tap_off[d.num_taps++];
    int rest = t;
    for (auto ax = std::rbegin(axes); ax != std::rend(axes); ++ax) {
      o[ax->dim] = ax->start + rest % ax->extent;
      rest /= ax->extent;
    }
  }
}

// stride-1 convolution that keeps the image size: a kh x kw window padded by pad_top rows and pad_left columns, weights
// (Cout, kh, kw, Cin)
static uav_status_t conv2d_same(const void* x, int64_t NB, int64_t H, int64_t W, int64_t Cin, int64_t ld_in,
                                const void* w, int64_t Cout, int kh, int kw, int pad_top, int pad_left, void* out,
                                const uav_epilogue_t* epi, cudaStream_t stream) {
  const TileRect t = pick_tile_2d(W, H);
  IgemmDesc d;
  dense_view(d, x, ld_in, Cin, {W, H, NB, 1}, {t.w, t.h, 1, 1});
  add_tap_grid(d, {{2, kh, -pad_top}, {1, kw, -pad_left}});
  return launch_igemm(d, w, Cout, out, epi, stream);
}

}  // namespace uav

using namespace uav;

extern "C" {

int64_t uav_gn_partial_blocks(int64_t w, int64_t h, int64_t images) {
  if (w <= 0 || h <= 0 || images <= 0) return 0;
  // One block per 16 rows of a 128-row M-tile (the accumulator rows of one consumer warp).  This must agree block for
  // block with the launch whose epilogue writes the statistics, so the M-tiles come from pick_tile_2d as in the launches;
  // for h == 1 it gives (128, 1), the box of uav_linear and uav_conv_temporal.
  const TileRect t = pick_tile_2d(w, h);
  return ((w + t.w - 1) / t.w) * ((h + t.h - 1) / t.h) * images * 8;
}

const char* uav_version(void) { return "uav_b200 0.3 (sm_90a)"; }
const char* uav_last_error_string(void) { return g_err; }
uint64_t uav_launch_count(void) { return g_launches.load(); }

uav_status_t uav_linear(const void* a, int64_t M, int64_t K, int64_t lda, const void* w,
                        int64_t N, void* out, const uav_epilogue_t* epi, uav_stream_t stream) {
  UAV_REQUIRE(M >= 0 && K > 0 && N > 0 && lda >= K, "uav_linear: bad shape");
  if (M == 0) return UAV_OK;
  IgemmDesc d;
  dense_view(d, a, lda, K, {M, 1, 1, 1}, {128, 1, 1, 1});
  d.num_taps = 1;  // at offset 0
  return launch_igemm(d, w, N, out, epi, (cudaStream_t)stream);
}

uav_status_t uav_conv2d(const void* x, int64_t NB, int64_t H, int64_t W, int64_t Cin,
                        int64_t ld_in, const void* w, int64_t Cout, int ksize, int stride,
                        int pad_mode, void* out, const uav_epilogue_t* epi,
                        uav_stream_t stream) {
  UAV_REQUIRE(NB > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0 && ld_in >= Cin,
              "uav_conv2d: bad shape");
  UAV_REQUIRE(ksize == 1 || ksize == 3, "uav_conv2d: ksize must be 1 or 3");
  UAV_REQUIRE(stride == 1 || stride == 2, "uav_conv2d: stride must be 1 or 2");
  UAV_REQUIRE(pad_mode == 0 || (pad_mode == 1 && stride == 2 && ksize == 3),
              "uav_conv2d: pad_mode 1 needs a stride-2 3x3 conv");
  // a 1x1 stride-1 convolution is a plain GEMM over the NB*H*W pixels (always-full 128-row tiles)
  if (ksize == 1 && stride == 1) return uav_linear(x, NB * H * W, Cin, ld_in, w, Cout, out, epi, stream);
  const int pad = ksize / 2;
  if (stride == 1)
    return conv2d_same(x, NB, H, W, Cin, ld_in, w, Cout, ksize, ksize, pad, pad, out, epi, (cudaStream_t)stream);
  UAV_REQUIRE(H % 2 == 0 && W % 2 == 0, "uav_conv2d: stride 2 needs even H, W (got %lldx%lld)",
              (long long)H, (long long)W);
  UAV_REQUIRE(ld_in == Cin, "uav_conv2d: stride 2 needs a dense input (ld_in == Cin)");
  const int64_t Wo = W / 2, Ho = H / 2;
  const TileRect t = pick_tile_2d(Wo, Ho);
  IgemmDesc d;
  d.a = x;
  d.k_per_tap = (int)Cin;
  // phase view: (2C [px*C + c], W/2, 2 [py], H/2, NB)
  const uint64_t dims[5] = {(uint64_t)(2 * Cin), (uint64_t)Wo, 2, (uint64_t)Ho, (uint64_t)NB};
  const uint64_t strides[5] = {1, (uint64_t)(2 * Cin), (uint64_t)(W * Cin),
                               (uint64_t)(2 * W * Cin), (uint64_t)(H * W * Cin)};
  const uint32_t box[5] = {64, t.w, 1, t.h, 1};
  const uint32_t tiles[5] = {1, (uint32_t)((Wo + t.w - 1) / t.w), 1,
                             (uint32_t)((Ho + t.h - 1) / t.h), (uint32_t)NB};
  const uint32_t odims[5] = {1, (uint32_t)Wo, 1, (uint32_t)Ho, (uint32_t)NB};
  for (int i = 0; i < 5; ++i) {
    d.a_dims[i] = dims[i];
    d.a_strides[i] = strides[i];
    d.box[i] = box[i];
    d.tiles[i] = tiles[i];
    d.out_dims[i] = odims[i];
  }
  d.num_taps = 9;
  for (int ky = 0; ky < 3; ++ky)
    for (int kx = 0; kx < 3; ++kx) {
      // input coordinate = 2*o + k - pad  (pad = 1 for pad_mode 0, 0 for pad_mode 1)
      const int iy = ky - (pad_mode == 0 ? 1 : 0);  // in {-1,0,1} or {0,1,2}
      const int ix = kx - (pad_mode == 0 ? 1 : 0);
      const int py = ((iy % 2) + 2) % 2, px = ((ix % 2) + 2) % 2;
      const int oy = (iy - py) / 2, ox = (ix - px) / 2;  // exact
      int32_t* o = d.tap_off[ky * 3 + kx];
      o[0] = px * (int)Cin;
      o[1] = ox;
      o[2] = py;
      o[3] = oy;
    }
  return launch_igemm(d, w, Cout, out, epi, (cudaStream_t)stream);
}

uav_status_t uav_conv2d_taps(const void* x, int64_t NB, int64_t H, int64_t W, int64_t Cin, int64_t ld_in,
                             const void* w, int64_t Cout, int kh, int kw, int pad_top, int pad_left, void* out,
                             const uav_epilogue_t* epi, uav_stream_t stream) {
  UAV_REQUIRE(NB > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0 && ld_in >= Cin, "uav_conv2d_taps: bad shape");
  UAV_REQUIRE(kh >= 1 && kw >= 1 && kh * kw <= MAX_TAPS, "uav_conv2d_taps: at most %d taps (got %d x %d)", MAX_TAPS, kh,
              kw);
  UAV_REQUIRE(pad_top >= 0 && pad_top < kh && pad_left >= 0 && pad_left < kw, "uav_conv2d_taps: bad padding");
  return conv2d_same(x, NB, H, W, Cin, ld_in, w, Cout, kh, kw, pad_top, pad_left, out, epi, (cudaStream_t)stream);
}

uav_status_t uav_conv_temporal(const void* x, int64_t B, int64_t T, int64_t HW, int64_t Cin,
                               int64_t ld_in, const void* w, int64_t Cout, int k, void* out,
                               const uav_epilogue_t* epi, uav_stream_t stream) {
  UAV_REQUIRE(B > 0 && T > 0 && HW > 0 && Cin > 0 && Cout > 0 && ld_in >= Cin,
              "uav_conv_temporal: bad shape");
  UAV_REQUIRE(k == 1 || k == 3 || k == 5, "uav_conv_temporal: k must be 1, 3 or 5");
  IgemmDesc d;
  dense_view(d, x, ld_in, Cin, {HW, T, B, 1}, {128, 1, 1, 1});
  add_tap_grid(d, {{2, k, -k / 2}});
  return launch_igemm(d, w, Cout, out, epi, (cudaStream_t)stream);
}

uav_status_t uav_conv3d(const void* x, int64_t B, int64_t T, int64_t H, int64_t W, int64_t Cin,
                        int64_t ld_in, const void* w, int64_t Cout, void* out,
                        const uav_epilogue_t* epi, uav_stream_t stream) {
  UAV_REQUIRE(B > 0 && T > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0 && ld_in >= Cin,
              "uav_conv3d: bad shape");
  const TileRect t = pick_tile_2d(W, H);
  IgemmDesc d;
  dense_view(d, x, ld_in, Cin, {W, H, T, B}, {t.w, t.h, 1, 1});
  add_tap_grid(d, {{3, 3, -1}, {2, 3, -1}, {1, 3, -1}});
  return launch_igemm(d, w, Cout, out, epi, (cudaStream_t)stream);
}

uav_status_t uav_upsample2x_conv3x3(const void* x, int64_t NB, int64_t H, int64_t W, int64_t Cin,
                                    int64_t ld_in, const void* w4, int64_t Cout, void* out,
                                    const uav_epilogue_t* epi, uav_stream_t stream) {
  UAV_REQUIRE(NB > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0 && ld_in >= Cin && epi != nullptr,
              "uav_upsample2x_conv3x3: bad shape");
  UAV_REQUIRE(epi->residual == nullptr && epi->rowvec == nullptr && epi->out_dtype == UAV_F16 && Cout >= 33,
              "uav_upsample2x_conv3x3: bias-only fp16 epilogue with Cout > 32 required");
  const int64_t ld_out = epi->ld_out;
  const TileRect t = pick_tile_2d(W, H);
  for (int a = 0; a < 2; ++a)
    for (int b = 0; b < 2; ++b) {
      IgemmDesc d;
      dense_view(d, x, ld_in, Cin, {W, H, NB, 1}, {t.w, t.h, 1, 1});
      // source taps of the collapsed 2x2 filter: phase 0 reads {-1, 0}, phase 1 reads {0, +1}
      add_tap_grid(d, {{2, 2, a - 1}, {1, 2, b - 1}});
      // output phase (a, b): pixel (2y + a, 2x + b) of the [NB][2H][2W][ld_out] tensor
      d.out_strides[1] = 2 * (uint64_t)ld_out;
      d.out_strides[2] = 2 * 2 * (uint64_t)W * ld_out;
      d.out_strides[3] = 4 * (uint64_t)H * W * ld_out;
      d.out_strides[4] = 4 * (uint64_t)H * W * ld_out * NB;
      const __half* w_phase = reinterpret_cast<const __half*>(w4) + static_cast<int64_t>(a * 2 + b) * Cout * 4 * Cin;
      __half* out_phase = reinterpret_cast<__half*>(out) + (static_cast<int64_t>(a) * 2 * W + b) * ld_out;
      const uav_status_t st = launch_igemm(d, w_phase, Cout, out_phase, epi, (cudaStream_t)stream);
      if (st != UAV_OK) return st;
    }
  return UAV_OK;
}

}  // extern "C"
