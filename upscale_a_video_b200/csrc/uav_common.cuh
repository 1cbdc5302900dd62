// uav_common.cuh — sm_90a PTX wrappers shared by the uav kernels.
// mbarrier / TMA (cp.async.bulk.tensor) / wgmma (warpgroup MMA with shared-memory descriptors) helpers.
// No torch, no CUTLASS: plain CUDA + inline PTX. Bit layouts of the wgmma shared-memory matrix
// descriptors follow the PTX ISA "Matrix Descriptor Format" table of the asynchronous warpgroup MMA.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda.h>
#include <stdint.h>

#include <atomic>
#include <utility>

#include "../../include/uav_b200.h"

namespace uav {

// ---------------------------------------------------------------------------------------
// error plumbing (host)
// ---------------------------------------------------------------------------------------
void set_last_error(const char* fmt, ...);
#define UAV_CHECK_CUDA(expr)                                                             \
  do {                                                                                   \
    cudaError_t _e = (expr);                                                             \
    if (_e != cudaSuccess) {                                                             \
      uav::set_last_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr,                  \
                          cudaGetErrorString(_e));                                       \
      return UAV_ERR_CUDA;                                                               \
    }                                                                                    \
  } while (0)
#define UAV_REQUIRE(cond, ...)                                                           \
  do {                                                                                   \
    if (!(cond)) {                                                                       \
      uav::set_last_error(__VA_ARGS__);                                                  \
      return UAV_ERR_INVALID;                                                            \
    }                                                                                    \
  } while (0)

int num_sms();         // of the current device
int current_device();

// ---------------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier ----
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "LAB_WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1, %2;\n\t"
      "@P1 bra DONE;\n\t"
      "bra LAB_WAIT;\n\t"
      "DONE:\n\t"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity), "r"(0x989680u)
      : "memory");
}

// ---- TMA ----
__device__ __forceinline__ void tma_prefetch_desc(const void* desc) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(desc)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(const void* desc, uint64_t* bar, void* smem, int c0,
                                            int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(desc)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(const void* desc, uint64_t* bar, void* smem, int c0,
                                            int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(desc)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(const void* desc, uint64_t* bar, void* smem, int c0,
                                            int c1, int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6, %7}], [%2];" ::"r"(smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(desc)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
      "r"(c3), "r"(c4)
      : "memory");
}
// shared -> global store of a box, in the bulk group that the next tma_store_commit() closes
__device__ __forceinline__ void tma_store_5d(const void* desc, const void* smem, int c0, int c1, int c2, int c3,
                                             int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.global.shared::cta.bulk_group"
      " [%0, {%2, %3, %4, %5, %6}], [%1];" ::"l"(reinterpret_cast<uint64_t>(desc)),
      "r"(smem_u32(smem)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// waits until at most N committed store groups still have to read their shared memory
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}

// ---- warp-specialised TMA -> wgmma pipelines ----
constexpr int SMEM_OPT_IN_LIMIT = 232448;  // opt-in shared memory per block on sm_90 (227 KB)
// Register split of a 384-thread block with one producer and two consumer warpgroups: 128 x 40 + 256 x 232 fit the
// 64 K register file.
constexpr int PRODUCER_REGS = 40;
constexpr int CONSUMER_REGS = 232;
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N) : "memory");
}

// dynamic shared memory rounded up to 1024 bytes (the SWIZZLE_128B atom) in the shared address space
__device__ __forceinline__ uint8_t* smem_align1024(uint8_t* smem_raw) {
  const uint32_t raw_addr = smem_u32(smem_raw);
  return smem_raw + (((raw_addr + 1023u) & ~1023u) - raw_addr);
}

// named barrier ID over the first THREADS threads that reach it
template <int ID, int THREADS>
__device__ __forceinline__ void bar_sync() {
  asm volatile("bar.sync %0, %1;" ::"n"(ID), "n"(THREADS) : "memory");
}

// Position in a ring of STAGES slots.  The phase flips at every wrap: a slot's barrier completes once per pass.
template <int STAGES>
struct RingPos {
  uint32_t phase = 0;
  int stage = 0;
  __device__ __forceinline__ void advance() {
    if (++stage == STAGES) {
      stage = 0;
      phase ^= 1;
    }
  }
};

// The mbarriers of a ring of STAGES shared-memory slots, filled by TMA and drained by consumer warps: the 2 * STAGES
// barriers at `bars`.  Each consumer warp releases a slot with one mbar_arrive(&empty[stage]) from its lane 0 once its
// MMAs have read it.
template <int STAGES>
struct RingBarriers {
  uint64_t* full;   // [STAGES]: the slot's TMA bytes have landed
  uint64_t* empty;  // [STAGES]: every consumer warp has released the slot
  __device__ __forceinline__ explicit RingBarriers(uint64_t* bars) : full(bars), empty(bars + STAGES) {}
  // one thread, before fence_barrier_init()
  __device__ __forceinline__ void init(uint32_t consumer_warps) const {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], consumer_warps);
    }
  }
  // producer: waits for the consumers to release the slot at `pos`, then arms its full barrier for `bytes` of TMA loads
  // and returns it
  __device__ __forceinline__ uint64_t* acquire(const RingPos<STAGES>& pos, uint32_t bytes) const {
    mbar_wait(&empty[pos.stage], pos.phase ^ 1);
    mbar_expect_tx(&full[pos.stage], bytes);
    return &full[pos.stage];
  }
  // consumer: waits for the slot at `pos` to be filled
  __device__ __forceinline__ void wait_full(const RingPos<STAGES>& pos) const {
    mbar_wait(&full[pos.stage], pos.phase);
  }
};

// ---- wgmma (sm_90a warpgroup MMA) ----
// All four warps of a warpgroup execute these.  The accumulator fragment of m64nNk16 (fp32) in thread t of the
// warpgroup: d[i] holds row 16 * (t / 32) + (t % 32) / 4 + 8 * ((i / 2) % 2), column 8 * (i / 4) + 2 * (t % 4) + i % 2.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void wgmma_fence_operands(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Shared-memory matrix descriptor of a tile stored as rows of 128 bytes with the 128B swizzle (what a TMA box with a
// 128-byte inner extent and CU_TENSOR_MAP_SWIZZLE_128B writes): 8-row atoms of 1024 bytes (SBO = 1024).  K-major
// operands: LBO unused.  MN-major operands (rows = K, 64 MN elements per row): LBO would be the stride between 64-wide MN
// blocks, unused for N <= 64.  Advancing 16 fp16 along K inside a K-major row is +32 bytes (+2 in the address field).
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);  // [0,14) start address >> 4
  d |= static_cast<uint64_t>(1) << 16;                      // [16,30) LBO >> 4
  d |= static_cast<uint64_t>(1024 >> 4) << 32;              // [32,46) SBO >> 4
  d |= static_cast<uint64_t>(1) << 62;                      // [62,64) layout: SWIZZLE_128B
  return d;
}

// D (+)= A[smem] * B[smem]^T, A 64 x 16 and B N x 16 both K-major (scale_d == 0: D = A B^T)

__device__ __forceinline__ void wgmma_ss(float (&d)[8], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\n"
      "setp.ne.b32 p, %10, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_ss(float (&d)[16], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\n"
      "setp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_ss(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\n"
      "setp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_ss(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\n"
      "setp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_ss(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\n"
      "setp.ne.b32 p, %130, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, 0, 0;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
// D (+)= A[registers] * B[smem], A 64 x 16 fp16 (the layout of an m64 accumulator fragment converted to fp16
// pairs), B stored MN-major (rows = K)
__device__ __forceinline__ void wgmma_rs_tb(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\n"
      "setp.ne.b32 p, %37, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 1;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d));
}

// ---- adaptive average pooling (F.interpolate mode='area') ----
// output index o of out_size averages the input window [floor(o * in / out), ceil((o + 1) * in / out)); windows of
// neighbouring outputs overlap when in_size is not a multiple of out_size
__device__ __forceinline__ int64_t area_start(int64_t o, int64_t out_size, int64_t in_size) {
  return (o * in_size) / out_size;
}
__device__ __forceinline__ int64_t area_end(int64_t o, int64_t out_size, int64_t in_size) {
  return ((o + 1) * in_size + out_size - 1) / out_size;
}

// ---- misc math ----
// MUFU.EX2 / MUFU.RCP with flush-to-zero: the non-ftz forms (__expf, __fdividef) wrap every MUFU in denormal
// range fix-ups (FSETP + predicated FMULs: ~8 extra instructions per GELU), which matters in the GEMM epilogues that
// are issue-bound.  <= 2 ulp; results that would be denormal flush to zero (|x| > 87 for SiLU, > 13 for GELU tails).
__device__ __forceinline__ float ex2_ftz(float x) {
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float rcp_ftz(float x) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
// x * sigmoid(x): x -> -inf gives x * rcp(inf) = -0, x -> +inf gives x * rcp(1) = x
__device__ __forceinline__ float silu_f(float x) { return x * rcp_ftz(1.0f + ex2_ftz(-1.4426950408889634f * x)); }
// SiLU of two values with ONE reciprocal: 1 / d0 = d1 * (1 / (d0 d1)).  3 MUFU per pair instead of 4 — the GroupNorm+SiLU
// apply pass is a streaming kernel whose XU pipe (MUFU + the fp16 pack) is busy enough to limit it.
// The exponent argument is clamped to 60 so that d0 d1 stays finite (x < -41.6: sigmoid ~ 8.7e-19 either way).
__device__ __forceinline__ void silu2_f(float& a, float& b) {
  const float d0 = 1.0f + ex2_ftz(fminf(-1.4426950408889634f * a, 60.0f));
  const float d1 = 1.0f + ex2_ftz(fminf(-1.4426950408889634f * b, 60.0f));
  const float r = rcp_ftz(d0 * d1);
  a *= r * d1;
  b *= r * d0;
}
// exact-GELU x * Phi(x) with ONE MUFU: Phi(-|x|) = 2^p(|x|), p = degree-8 polynomial fit of log2(erfc(|x| / sqrt 2) / 2)
// on [0, 6] (Chebyshev least squares weighted by Phi, converted to monomials in t = |x| / 3 - 1; tools/fit_gelu.py), then
// gelu(x) = max(x, 0) - |x| * Phi(-|x|) (x >= 0: x (1 - Phi(-x)); x < 0: x Phi(x)).  |x| is clamped to 6 where
// |x| Phi(-|x|) < 6e-9.  11 FP32 instructions + 1 MUFU.EX2 instead of 12 + 2 MUFU (Abramowitz-Stegun erfc with a
// reciprocal, round 1): the GEGLU epilogue is MUFU-throughput bound (16 lanes / clk / SM).  Absolute error of the result
// <= 4.8e-7 in fp32 evaluation (the rounding of x - r near |x| = 8; fit error 1.6e-7), same as the fp32
// 0.5 x (1 + erff(x / sqrt 2)) formula against float64.
__device__ __forceinline__ float gelu_erf_f(float x) {
  const float ax = fminf(fabsf(x), 6.0f);
  const float t = fmaf(ax, 0.3333333333333333f, -1.0f);
  float p = -0.005517261102795601f;
  p = fmaf(p, t, -0.012404678389430046f);
  p = fmaf(p, t, 0.020884426310658455f);
  p = fmaf(p, t, -0.02991572767496109f);
  p = fmaf(p, t, 0.09405267238616943f);
  p = fmaf(p, t, -0.2069002389907837f);
  p = fmaf(p, t, -6.035426616668701f);
  p = fmaf(p, t, -14.20971965789795f);
  p = fmaf(p, t, -9.532933235168457f);
  return fmaf(-ax, ex2_ftz(p), fmaxf(x, 0.0f));
}

// fp32 pair -> packed fp16 with saturation to +-65504 (one F2FP.SATFINITE): an activation that leaves the fp16 range
// clamps instead of becoming inf (which the next GroupNorm would turn into NaN for the whole group)
__device__ __forceinline__ uint32_t pack_half2_sat(float a, float b) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}

// 16-byte global access
__device__ __forceinline__ uint4 ldg16(const void* p) {
  return *reinterpret_cast<const uint4*>(p);
}
__device__ __forceinline__ void stg16(void* p, const uint4& v) {
  *reinterpret_cast<uint4*>(p) = v;
}
// 16-byte streaming load of data read once (weight streams): non-coherent, no L1 allocation, 256-byte L2 prefetch
__device__ __forceinline__ uint4 ldg16_stream(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::256B.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

// fp32 pair -> packed fp16, round to nearest
__device__ __forceinline__ uint32_t pack_half2_rn(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// ---- cp.async / ldmatrix / mma.sync m16n8k16 (warp-level MMA) ----
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool valid) {
  const uint32_t s = smem_u32(smem);
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(gmem), "r"(sz)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() {
  asm volatile("cp.async.commit_group;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(p)));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(p)));
}
// c += a b: a is the 16 x 16 A fragment, (b0, b1) the 16 x 8 B fragment, c the fp32 16 x 8 accumulator (c[0..1] row
// lane / 4, c[2..3] row lane / 4 + 8, columns 2 (lane % 4) + {0, 1})
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0,
                                         uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
      "{%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// smem tile: rows of DT halfs, 16-byte chunks XOR-swizzled by (row & 7)
template <int DT>
__device__ __forceinline__ __half* tile_ptr(__half* base, int row, int chunk) {
  return base + row * DT + ((chunk ^ (row & 7)) << 3);
}

// ---------------------------------------------------------------------------------------
// launch plumbing
// ---------------------------------------------------------------------------------------
// i = every index in [0, n) that this thread owns in a grid-stride loop over a 1-D grid
#define UAV_GRID_STRIDE(i, n)                                                         \
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < (n); \
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)

// gridDim.x of a grid-stride kernel over `items`: one block per `items_per_block`, at most `blocks_per_sm` blocks per SM,
// at least one block
inline unsigned stream_grid(int64_t items, int64_t items_per_block, int blocks_per_sm) {
  int64_t blocks = (items + items_per_block - 1) / items_per_block;
  const int64_t cap = static_cast<int64_t>(num_sms()) * blocks_per_sm;
  if (blocks > cap) blocks = cap;
  return static_cast<unsigned>(blocks < 1 ? 1 : blocks);
}

extern std::atomic<uint64_t> g_launches;  // kernels this library has launched: uav_launch_count()

// follows every kernel launch: a launch error is returned, a launch that went in is counted
#define UAV_LAUNCHED()                                       \
  do {                                                       \
    UAV_CHECK_CUDA(cudaGetLastError());                      \
    uav::g_launches.fetch_add(1, std::memory_order_relaxed); \
  } while (0)

// 16-byte alignment, which ldg16 / stg16, float4 loads, cp.async and TMA need; a null pointer passes
inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
#define UAV_REQUIRE_ALIGNED16(fn, ptr) UAV_REQUIRE(uav::aligned16(ptr), fn ": " #ptr " must be 16-byte aligned")

// Encodes the tensor map of an fp16 tensor of `rank` <= 5 dims (dims and box innermost first, `strides` = the byte
// strides of dims 1..rank-1) with the 128B swizzle that the wgmma operand tiles and the output staging use, unit element
// strides and zero fill out of bounds.  `what` names the map in the error message.
uav_status_t encode_tensor_map(CUtensorMap* map, const void* base, int rank, const cuuint64_t* dims,
                               const cuuint64_t* strides, const cuuint32_t* box, CUtensorMapL2promotion l2,
                               const char* what);

// Lets Kernel use `bytes` of dynamic shared memory, with one cudaFuncSetAttribute per device: the attribute applies to
// the current device only.  Every call for one Kernel passes the same `bytes`.
template <auto Kernel>
uav_status_t opt_in_smem(int bytes) {
  static std::atomic<uint64_t> configured{0};  // bit d: done on device d
  const uint64_t dev_bit = 1ull << (current_device() & 63);
  if (!(configured.load(std::memory_order_relaxed) & dev_bit)) {
    UAV_CHECK_CUDA(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    configured.fetch_or(dev_bit, std::memory_order_relaxed);
  }
  return UAV_OK;
}

// Launches Kernel<<<grid, threads, smem, stream>>>(args...) with `smem` bytes of dynamic shared memory opted in, and
// checks the launch.
template <auto Kernel, class... A>
uav_status_t launch_opted_in(dim3 grid, int threads, int smem, cudaStream_t stream, A&&... args) {
  const uav_status_t st = opt_in_smem<Kernel>(smem);
  if (st != UAV_OK) return st;
  Kernel<<<grid, threads, smem, stream>>>(std::forward<A>(args)...);
  UAV_LAUNCHED();
  return UAV_OK;
}

}  // namespace uav
