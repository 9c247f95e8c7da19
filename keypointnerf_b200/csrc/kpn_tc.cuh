// Thin inline-PTX layer over the sm_90a tensor-core path: warpgroup MMA (wgmma.mma_async, B and usually A in shared memory
// through matrix descriptors, A also from registers, fp32 accumulators in registers), mbarrier and the 1-D bulk (TMA) copy.  Encodings follow the
// PTX ISA wgmma chapter; the bit layout of the shared-memory descriptor is restated below.
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

namespace kpn {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier -----------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// non-blocking probe (try_wait may suspend the thread up to a hardware time limit; a thread that polls several
// barriers must not do that)
__device__ __forceinline__ bool mbar_test_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\tmbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Watchdog.  A barrier wait that has not completed after ~2^20 suspended polls is a protocol bug; instead of hanging the GPU
// the waiter records where it gave up, raises this module's abort flag (every other wait then gives up within 256 polls) and
// returns, so that the kernel terminates (with garbage results) and the host can report the location (kpn_check_health).
static __device__ unsigned int kpn_wd[8];   // [0] flag, [1] block, [2] thread, [3] tag, [4] parity
__device__ __forceinline__ bool wd_give_up(uint32_t spins, uint32_t limit, uint32_t tag, uint32_t parity) {
  const bool aborted = *reinterpret_cast<volatile unsigned int*>(&kpn_wd[0]) != 0u;
  if (!aborted && spins <= limit) return false;
  if (!aborted && atomicCAS(&kpn_wd[0], 0u, 1u) == 0u) {
    kpn_wd[1] = blockIdx.x; kpn_wd[2] = threadIdx.x; kpn_wd[3] = tag; kpn_wd[4] = parity;
    __threadfence();
  }
  return true;
}
// try_wait with a suspend-time hint (ns): the thread sleeps in hardware until the phase completes or the hint elapses, instead of
// re-polling every few hundred cycles (a third of the row warps wait at any time; their polls compete for issue slots).
__device__ __forceinline__ bool mbar_try_wait_hint(uint64_t* bar, uint32_t parity, uint32_t ns) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\tselp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"(ns)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, uint32_t tag = 0) {
  // plain try_wait (the hardware suspends the thread for a short system-defined time per poll); a 20 us suspend hint
  // (mbar_try_wait_hint) measured the same or slightly slower (28.4 vs 28.2 ms/frame)
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 255u) == 0u && wd_give_up(spins, 1u << 20, tag, parity)) return;
  }
}

// ---- 1-D bulk copy global -> shared (TMA unit, SASS UBLKCP), completion on an mbarrier -----------------
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// generic-proxy writes to shared memory -> visible to the async proxy (tensor core operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- descriptors ---------------------------------------------------------------------------------------
// Shared-memory matrix descriptor (64 bit), K-major operand, no swizzle ("interleaved" core matrices of 8 rows x 16 bytes
// stored as 128 contiguous bytes):
//   [0,14)  start address >> 4      [16,30) leading-dimension byte offset >> 4 (distance between core matrices along K)
//   [32,46) stride-dimension byte offset >> 4 (distance between 8-row groups)   [62,64) swizzle mode = 0 (none)
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  return d;
}

// ---- warpgroup MMA ---------------------------------------------------------------------------------------
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// Pins N registers in program order between the volatile wgmma statements: a register-A fragment fenced before wg_fence() is
// complete before the chain starts (the compiler would otherwise sink its last definitions between the chain's MMAs, and ptxas
// then serialises them, C7513), and accumulators fenced after wg_wait0() are not read before the wait.
template <int N>
__device__ __forceinline__ void fence_regs(uint32_t* r) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+r"(r[i])::"memory");
}
template <int N>
__device__ __forceinline__ void fence_regs(float* r) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(r[i])::"memory");
}

}  // namespace tc
}  // namespace kpn
#include "kpn_wgmma.cuh"
namespace kpn {
namespace tc {

// An activation tile of ROWS rows in shared memory, K-major core matrices in the order [k/8][row/8][row%8][k%8] (fp16):
// LBO = (ROWS/8) * 128 bytes, SBO = 128 bytes.  Byte offset of 32-bit word column c (fp16 elements 2c, 2c+1) of row r.
template <int ROWS>
__host__ __device__ constexpr uint32_t a_word_off(int r, int c) {
  return (uint32_t)((((c >> 2) * (ROWS >> 3) + (r >> 3)) * 128) + (r & 7) * 16 + (c & 3) * 4);
}

// D[64 x N] (+)= A[64 x 16*KCH] * B[N x 16*KCH]^T for the warpgroup's 64-row tile at `a_addr` (activation layout above with
// a_lbo = (tile rows / 8) * 128) and a weight tile at `b_addr` ([k/8][n/8][8][8], LBO = (Np/8)*128).  `acc` = 0 overwrites d.
// The caller brackets a chain of these with wg_fence() / wg_commit() + wg_wait0().
template <int N, int KCH>
__device__ __forceinline__ void wg_mma(float* d, uint32_t a_addr, uint32_t a_lbo, uint32_t b_addr, uint32_t b_lbo, uint32_t acc) {
#pragma unroll
  for (int j = 0; j < KCH; ++j)
    Wgmma<N>::mma(d, make_smem_desc(a_addr + 2u * a_lbo * (uint32_t)j, a_lbo, 128u),
                  make_smem_desc(b_addr + 2u * b_lbo * (uint32_t)j, b_lbo, 128u), (acc || j > 0) ? 1u : 0u);
}

// The same product with A from registers: a[4j .. 4j + 3] is k-block j's fragment (WgmmaRA).  The registers must stay unchanged
// until the caller's wg_wait0() after the chain.
template <int N, int KCH>
__device__ __forceinline__ void wg_mma_ra(float* d, const uint32_t* a, uint32_t b_addr, uint32_t b_lbo, uint32_t acc) {
#pragma unroll
  for (int j = 0; j < KCH; ++j)
    WgmmaRA<N>::mma(d, a + 4 * j, make_smem_desc(b_addr + 2u * b_lbo * (uint32_t)j, b_lbo, 128u), (acc || j > 0) ? 1u : 0u);
}

// named barriers (ids 1..15): producer arrives, consumer syncs; `count` = threads of both sides
__device__ __forceinline__ void named_arrive(int id, int count) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory"); }
__device__ __forceinline__ void named_sync(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }

// pack two floats to one register of fp16 pair: low half = a (even K index), high half = b
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// Byte offset of element (row n, col k) of a K-major operand tile stored as interleaved 8x8 core matrices
// in the order [k/8][n/8][n%8][k%8] (fp16): LBO = (rows/8)*128 bytes, SBO = 128 bytes.
__host__ __device__ constexpr uint32_t core_offset_bytes(int n, int k, int rows) {
  return (uint32_t)(((k >> 3) * (rows >> 3) + (n >> 3)) * 128 + (n & 7) * 16 + (k & 7) * 2);
}

}  // namespace tc
}  // namespace kpn
