// tc_prims.cuh -- sm_90a primitives used by the tensor-core path: mbarrier, bulk async
// copies (TMA unit, non-tensor form), warpgroup MMA (wgmma) into the accumulator region,
// shared-memory matrix descriptors and the 128-byte swizzle used by every operand tile.
//
// All operand tiles share ONE physical layout: rows of 64 bf16 (128 bytes), 8-row swizzle
// atoms (1024 bytes), 16-byte chunk index XORed with (row & 7).  Whether a tile is consumed
// K-major (rows = M/N index, columns = K) or MN-major (rows = K index, columns = M/N) is
// chosen per MMA through the descriptor and the wgmma transpose flags, which is what lets
// the same tile feed the forward GEMM, dgrad and wgrad.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include "tc_types.h"
#include "tc_wgmma.cuh"

namespace pinn {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier --------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// bounded spin: a protocol bug traps (kernel error) instead of hanging the GPU
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  for (uint32_t it = 0; it < (1u << 28); ++it)
    if (mbar_try_wait(bar, parity)) return;
  __trap();
}

// ---- bulk async copies (global <-> shared, contiguous bytes; size multiple of 16) ---------------
__device__ __forceinline__ void bulk_load(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void bulk_store(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_load_u(uint32_t smem_dst_addr, const void* gsrc, uint32_t bytes, uint32_t bar_addr) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_dst_addr),
               "l"(gsrc), "r"(bytes), "r"(bar_addr)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// generic-proxy writes to shared memory -> visible to the async proxy (wgmma, bulk copies)
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- accumulator region ------------------------------------------------------------------------------
// The MMA results of a CTA live in an fp32 region of global memory, [kAccCols columns][128 rows] (256 KB per CTA,
// L2-resident: 132 CTAs take 33 MB of the 50 MB L2).  An "accumulator address" packs a row base in the high 16 bits
// and a column in the low 16 bits; acc_ld* read consecutive columns of row (base + lane), so a warp reads whole
// 128-byte lines.  The region pointer of the CTA is kept in shared memory (set once by the kernel).
static __shared__ float* s_acc;

__device__ __forceinline__ const float* acc_row(uint32_t aaddr) {
  return s_acc + (aaddr & 0xffffu) * kAccRows + (aaddr >> 16) + (threadIdx.x & 31);
}
__device__ __forceinline__ void acc_ld16(uint32_t aaddr, float (&v)[16]) {
  const float* r = acc_row(aaddr);
#pragma unroll
  for (int i = 0; i < 16; ++i) v[i] = r[i * kAccRows];
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// One warpgroup computes rows [64 h, 64 h + 64) of D (+)= A * B over nk k-steps of 16 and stores them to the
// accumulator region at column dcol.  Fragment layout of m64nNk16: d[i] is row 16 w + lane/4 + 8 ((i >> 1) & 1),
// column 8 (i >> 2) + 2 (lane & 3) + (i & 1).
template <int N, int TA, int TB>
__device__ __forceinline__ void wg_chain(uint32_t dcol, int h, uint64_t adesc, uint64_t bdesc, uint32_t a_step, uint32_t b_step,
                                         int nk, uint32_t acc_first) {
  float d[N / 2];
  const int w = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  float* base = s_acc + dcol * kAccRows + 64 * h + 16 * w + (lane >> 2) + (size_t)(2 * (lane & 3)) * kAccRows;
#pragma unroll
  for (int i = 0; i < N / 2; ++i)
    d[i] = acc_first ? base[((i >> 2) * 8 + (i & 1)) * kAccRows + 8 * ((i >> 1) & 1)] : 0.f;
  wgmma_fence();
  const uint64_t da = a_step >> 4, db = b_step >> 4;
#pragma unroll 1
  for (int k = 0; k < nk; ++k) {
    const uint32_t sc = (k > 0) ? 1u : acc_first;
    if (N == 16) wgmma_n16<TA, TB>(*reinterpret_cast<float(*)[8]>(d), adesc, bdesc, sc);
    if (N == 32) wgmma_n32<TA, TB>(*reinterpret_cast<float(*)[16]>(d), adesc, bdesc, sc);
    if (N == 48) wgmma_n48<TA, TB>(*reinterpret_cast<float(*)[24]>(d), adesc, bdesc, sc);
    if (N == 64) wgmma_n64<TA, TB>(*reinterpret_cast<float(*)[32]>(d), adesc, bdesc, sc);
    if (N == 128) wgmma_n128<TA, TB>(*reinterpret_cast<float(*)[64]>(d), adesc, bdesc, sc);
    adesc += da;
    bdesc += db;
  }
  wgmma_commit();
  wgmma_wait0();
#pragma unroll
  for (int i = 0; i < N / 2; ++i) base[((i >> 2) * 8 + (i & 1)) * kAccRows + 8 * ((i >> 1) & 1)] = d[i];
}

template <int TA, int TB>
__device__ __forceinline__ void wg_chain_n(int n, uint32_t dcol, int h, uint64_t adesc, uint64_t bdesc, uint32_t a_step,
                                           uint32_t b_step, int nk, uint32_t acc_first) {
  switch (n) {
    case 16: wg_chain<16, TA, TB>(dcol, h, adesc, bdesc, a_step, b_step, nk, acc_first); break;
    case 32: wg_chain<32, TA, TB>(dcol, h, adesc, bdesc, a_step, b_step, nk, acc_first); break;
    case 48: wg_chain<48, TA, TB>(dcol, h, adesc, bdesc, a_step, b_step, nk, acc_first); break;
    case 64: wg_chain<64, TA, TB>(dcol, h, adesc, bdesc, a_step, b_step, nk, acc_first); break;
    case 128: wg_chain<128, TA, TB>(dcol, h, adesc, bdesc, a_step, b_step, nk, acc_first); break;
    default: __trap();   // pinn_create admits only layer widths that give these N
  }
}

__device__ __forceinline__ void prefetch_l1(const void* p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); }
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

// ---- descriptors ---------------------------------------------------------------------------------------
// shared-memory matrix descriptor (wgmma), 128-byte swizzle
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= 1ull << 62;   // SWIZZLE_128B
  return d;
}
// shape of an MMA chain (M = 128): N (16, 32, 48, 64 or 128) and the operand majors (0 = K-major, 1 = MN-major)
__host__ __device__ constexpr uint32_t make_idesc(uint32_t n, uint32_t a_mn_major, uint32_t b_mn_major) {
  return n | (a_mn_major << 8) | (b_mn_major << 9);
}

// byte offset of element (row, col) inside a [rows x 64] bf16 tile with the 128-byte swizzle
__device__ __host__ __forceinline__ uint32_t swz_off(uint32_t row, uint32_t col) {
  return row * 128u + ((((col >> 3) ^ (row & 7u)) & 7u) << 4) + ((col & 7u) << 1);
}
// byte offset of the 16-byte chunk (8 columns starting at chunk*8) of a row
__device__ __host__ __forceinline__ uint32_t swz_chunk(uint32_t row, uint32_t chunk) {
  return row * 128u + (((chunk ^ (row & 7u)) & 7u) << 4);
}

__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

}  // namespace tc
}  // namespace pinn
