// pnx_common.cuh -- shared device helpers for the pillarnext_b200 sm_90a kernels.
// Raw PTX wrappers for mbarrier / TMA (cp.async.bulk.tensor) / cp.async / wgmma.
// The wgmma shared-memory descriptor layout follows the PTX ISA "matrix descriptor" table
// (cross-checked against CUTLASS cute/arch/mma_sm90_desc.hpp).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda.h>
#include <stdint.h>
#include <stdio.h>

#include "wgmma_sm90.cuh"

#define PNX_OK 0
#define PNX_ERR_ARG -1
#define PNX_ERR_CUDA -2
#define PNX_ERR_CAPACITY -3

void pnx_set_error(const char* fmt, ...);

#define PNX_CHECK_ARG(cond, msg)                                        \
  do {                                                                  \
    if (!(cond)) {                                                      \
      pnx_set_error("%s:%d: bad argument: %s", __FILE__, __LINE__, msg); \
      return PNX_ERR_ARG;                                               \
    }                                                                   \
  } while (0)

#define PNX_CHECK_LAUNCH()                                                                   \
  do {                                                                                       \
    cudaError_t e__ = cudaGetLastError();                                                    \
    if (e__ != cudaSuccess) {                                                                \
      pnx_set_error("%s:%d: CUDA launch failed: %s", __FILE__, __LINE__, cudaGetErrorString(e__)); \
      return PNX_ERR_CUDA;                                                                   \
    }                                                                                        \
  } while (0)

#define PNX_CUDA(call)                                                                       \
  do {                                                                                       \
    cudaError_t e__ = (call);                                                                \
    if (e__ != cudaSuccess) {                                                                \
      pnx_set_error("%s:%d: %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__));     \
      return PNX_ERR_CUDA;                                                                   \
    }                                                                                        \
  } while (0)

static inline int pnx_cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

namespace pnx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// ------------------------------------------------------------------ mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  while (!mbar_try_wait(bar, parity)) __nanosleep(32);  // back off: spinning waiters steal issue slots from working warps
}

// ------------------------------------------------------------------ proxy fences
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ------------------------------------------------------------------ TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 2-D tiled load: coordinates (c0 = innermost element index, c1 = row index)
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::
          "r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// 4-D tiled load, coordinates innermost first; out-of-bounds elements (negative coordinates included) are zero-filled
__device__ __forceinline__ void tma_load_4d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::
          "r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// ------------------------------------------------------------------ cp.async (gathered rows)
// 16-byte global -> shared copy; src_bytes = 0 zero-fills the destination (absent neighbour / padding row)
__device__ __forceinline__ void cp_async_16(uint32_t dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
// arrive on `bar` once every cp.async this thread issued so far has landed (counts as one of the barrier's arrivals)
__device__ __forceinline__ void cp_async_mbar_arrive(uint64_t* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// offset of 16-byte chunk `chunk` of row `row` in a 128B-swizzled tile (TMA SWIZZLE_128B / wgmma SW128 layout)
__device__ __forceinline__ uint32_t sw128_offset(uint32_t row, uint32_t chunk) {
  return row * 128u + ((chunk ^ (row & 7u)) << 4);
}

// ------------------------------------------------------------------ wgmma (sm_90a)
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// pins accumulator registers in place around the asynchronous MMAs
template <int R>
__device__ __forceinline__ void fence_acc(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// producer warpgroup hands registers to the accumulator-holding warpgroups
template <uint32_t kRegs>
__device__ __forceinline__ void regs_dealloc() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kRegs)); }
template <uint32_t kRegs>
__device__ __forceinline__ void regs_alloc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kRegs)); }

// wgmma shared-memory descriptor, SWIZZLE_128B: [0,14) start>>4 | [16,30) LBO>>4 | [32,46) SBO>>4 | [49,52) base offset |
// [62,64) layout (1 = SW128).  SBO = stride of 8-row groups; MN-major: LBO = stride of 64-element MN atoms.
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// row / column of accumulator register i of this thread in its warpgroup's 64 x N wgmma tile
__device__ __forceinline__ int acc_row(int i) { return 16 * ((threadIdx.x >> 5) & 3) + ((threadIdx.x & 31) >> 2) + 8 * ((i >> 1) & 1); }
__device__ __forceinline__ int acc_col(int i) { return 8 * (i >> 2) + 2 * (threadIdx.x & 3) + (i & 1); }

// ------------------------------------------------------------------ misc
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

}  // namespace pnx

// host: encode a 2-D bf16 tensor map (rows x cols, row-major), box = box_rows x box_cols, SWIZZLE_128B.
// Resolved through cudaGetDriverEntryPoint so the library links without libcuda.
int pnx_encode_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                            uint64_t row_stride_bytes, uint32_t box_rows, uint32_t box_cols);
// host: 4-D bf16 tensor map, dims / box innermost first, strides of dims 1..3 in bytes, SWIZZLE_128B.
int pnx_encode_tmap_4d_bf16(CUtensorMap* out, const void* base, const uint64_t dims[4], const uint64_t strides_bytes[3],
                            const uint32_t box[4]);
