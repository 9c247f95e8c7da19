// Self-tests of the tensor-core primitive used by the ray-march engine.  One 128 x N x K fp16 GEMM tile with fp32
// accumulation, D[128][N] = A[128][K] * B[N][K]^T, through wgmma.mma_async with the A operand in the activation-tile layout
// the kernels' epilogues write (tc::a_word_off) and the B operand in the interleaved core-matrix layout the weight packer
// emits.  One warpgroup issues the two 64-row halves.  Exercised by tests/test_gpu_umma.py against torch.matmul; it pins
// the descriptor encodings and the accumulator fragment layout independently of the network kernels.
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include "kpn_tc.cuh"

namespace kpn {

template <int N>
__global__ void __launch_bounds__(128, 1)
wgmma_selftest_kernel(int K, const __half* __restrict__ A, const __half* __restrict__ B, float* __restrict__ D) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int t = threadIdx.x, w = t >> 5, l = t & 31;
  uint8_t* sB = smem;
  uint8_t* sA = smem + (size_t)N * K * 2;
  for (int idx = t; idx < N * K; idx += 128) {
    const int n = idx / K, k = idx % K;
    *reinterpret_cast<__half*>(sB + tc::core_offset_bytes(n, k, N)) = B[idx];
  }
  for (int idx = t; idx < 128 * K; idx += 128) {
    const int r = idx / K, k = idx % K;
    *reinterpret_cast<__half*>(sA + tc::a_word_off<128>(r, k >> 1) + (k & 1) * 2) = A[idx];
  }
  tc::fence_proxy_async_smem();
  __syncthreads();
  const uint32_t a_lbo = 16u * 128u, b_lbo = (uint32_t)(N / 8) * 128u;
  for (int half = 0; half < 2; ++half) {
    float d[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; ++i) d[i] = 0.0f;
    tc::wg_fence();
    for (int j = 0; j < K / 16; ++j)
      tc::Wgmma<N>::mma(d, tc::make_smem_desc(tc::smem_u32(sA) + half * 1024u + 2u * a_lbo * j, a_lbo, 128u),
                        tc::make_smem_desc(tc::smem_u32(sB) + 2u * b_lbo * j, b_lbo, 128u), j > 0 ? 1u : 0u);
    tc::wg_commit();
    tc::wg_wait0();
#pragma unroll
    for (int i = 0; i < N / 2; ++i) {
      const int r = 64 * half + 16 * w + (l >> 2) + 8 * ((i >> 1) & 1), c = 8 * (i >> 2) + 2 * (l & 3) + (i & 1);
      D[(size_t)r * N + c] = d[i];
    }
  }
}

template <int N>
static int run_selftest(int K, const void* A, const void* B, float* D, cudaStream_t st) {
  const size_t smem = (size_t)N * K * 2 + (size_t)128 * K * 2;
  if (cudaFuncSetAttribute(wgmma_selftest_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return -2;
  wgmma_selftest_kernel<N><<<1, 128, smem, st>>>(K, (const __half*)A, (const __half*)B, D);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

// The same tile with the A operand in registers (WgmmaRA), as the geometry front kernel feeds layers 1-3: each thread loads its
// warp's fragments of all KCH k-blocks from global memory and the warpgroup issues the KCH MMAs of a 64-row half as one group.
template <int N, int KCH>
__global__ void __launch_bounds__(128, 1)
wgmma_ra_selftest_kernel(const __half* __restrict__ A, const __half* __restrict__ B, float* __restrict__ D) {
  extern __shared__ __align__(128) uint8_t smem[];
  constexpr int K = 16 * KCH;
  const int t = threadIdx.x, w = t >> 5, l = t & 31;
  for (int idx = t; idx < N * K; idx += 128) {
    const int n = idx / K, k = idx % K;
    *reinterpret_cast<__half*>(smem + tc::core_offset_bytes(n, k, N)) = B[idx];
  }
  tc::fence_proxy_async_smem();
  __syncthreads();
  const uint32_t b_lbo = (uint32_t)(N / 8) * 128u;
  for (int half = 0; half < 2; ++half) {
    uint32_t a[4 * KCH];
#pragma unroll
    for (int j = 0; j < KCH; ++j)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int r = 64 * half + 16 * w + (l >> 2) + 8 * (i & 1), k = 16 * j + 8 * (i >> 1) + 2 * (l & 3);
        const __half2 h = __halves2half2(A[(size_t)r * K + k], A[(size_t)r * K + k + 1]);
        a[4 * j + i] = *reinterpret_cast<const uint32_t*>(&h);
      }
    float d[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; ++i) d[i] = 0.0f;
    tc::wg_fence();
    tc::wg_mma_ra<N, KCH>(d, a, tc::smem_u32(smem), b_lbo, 0u);
    tc::wg_commit();
    tc::wg_wait0();
#pragma unroll
    for (int i = 0; i < N / 2; ++i) {
      const int r = 64 * half + 16 * w + (l >> 2) + 8 * ((i >> 1) & 1), c = 8 * (i >> 2) + 2 * (l & 3) + (i & 1);
      D[(size_t)r * N + c] = d[i];
    }
  }
}

template <int N, int KCH>
static int run_ra_selftest(const void* A, const void* B, float* D, cudaStream_t st) {
  const size_t smem = (size_t)N * KCH * 16 * 2;
  if (cudaFuncSetAttribute(wgmma_ra_selftest_kernel<N, KCH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
    return -2;
  wgmma_ra_selftest_kernel<N, KCH><<<1, 128, smem, st>>>((const __half*)A, (const __half*)B, D);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}


// CTA-pair form on a 2-CTA cluster: D[256][N] = A[256][K] * B[N][K]^T.  CTA r holds rows 128r .. 128r+127 of A and keeps rows
// r*N/2 .. (r+1)*N/2-1 of B; the other half of B comes from the peer CTA's shared memory (distributed shared memory), then each
// CTA multiplies its 128 rows by all of B with wgmma.  B is stored as [n/8][k/8] core matrices (LBO = 128 bytes along K,
// SBO = (K/8)*128 bytes), so each CTA's half is one contiguous block at the same offset in both CTAs.  The A tile is a_width
// 32-bit columns wide and A occupies columns [a_col, a_col + K/2) of it.  mode: how the peer's half arrives --
// 0: this CTA reads it through distributed shared memory, 1: the peer pushes it with one bulk copy that completes on this
// CTA's mbarrier, 2: the peer writes it with remote stores.
template <int N>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(128, 1)
wgmma_pair_selftest_kernel(int K, const __half* __restrict__ A, const __half* __restrict__ B, float* __restrict__ D, int a_col,
                           int mode) {
  namespace cg = cooperative_groups;
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ uint64_t bar;
  cg::cluster_group cl = cg::this_cluster();
  const uint32_t rank = cl.block_rank(), peer = rank ^ 1u;
  const int t = threadIdx.x, w = t >> 5, l = t & 31;
  constexpr int NH = N / 2;
  const uint32_t half_bytes = (uint32_t)NH * K * 2;
  uint8_t* sB = smem;
  uint8_t* sA = smem + 2 * half_bytes;
  uint8_t* mine = sB + rank * half_bytes;
  if (t == 0) { tc::mbar_init(&bar, 1); tc::fence_mbar_init(); }
  for (int idx = t; idx < NH * K; idx += 128) {
    const int n = idx / K, k = idx % K;
    *reinterpret_cast<__half*>(mine + ((n >> 3) * (K >> 3) + (k >> 3)) * 128 + (n & 7) * 16 + (k & 7) * 2) =
        B[(size_t)(rank * NH + n) * K + k];
  }
  for (int idx = t; idx < 128 * K; idx += 128) {
    const int r = idx / K, k = idx % K;
    *reinterpret_cast<__half*>(sA + tc::a_word_off<128>(r, a_col + (k >> 1)) + (k & 1) * 2) = A[(size_t)(rank * 128 + r) * K + k];
  }
  __syncthreads();
  if (mode == 1 && t == 0) tc::mbar_expect_tx(&bar, half_bytes);   // the peer's bulk copy completes this phase
  tc::fence_proxy_async_smem();
  cl.sync();   // both CTAs: own halves written, barriers initialised
  if (mode == 0) {
    const uint8_t* theirs = cl.map_shared_rank(sB + peer * half_bytes, peer);
    uint8_t* dst = sB + peer * half_bytes;
    for (uint32_t i = 16u * t; i < half_bytes; i += 16u * 128u)
      *reinterpret_cast<uint4*>(dst + i) = *reinterpret_cast<const uint4*>(theirs + i);
    tc::fence_proxy_async_smem();
    __syncthreads();
  } else if (mode == 1) {
    if (t == 0) {
      uint32_t dst, mb;
      asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(dst) : "r"(tc::smem_u32(mine)), "r"(peer));
      asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(mb) : "r"(tc::smem_u32(&bar)), "r"(peer));
      asm volatile("cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                   ::"r"(dst), "r"(tc::smem_u32(mine)), "r"(half_bytes), "r"(mb) : "memory");
    }
    tc::mbar_wait(&bar, 0, 0x60u);
  } else {
    uint8_t* theirs = cl.map_shared_rank(mine, peer);
    for (uint32_t i = 16u * t; i < half_bytes; i += 16u * 128u)
      *reinterpret_cast<uint4*>(theirs + i) = *reinterpret_cast<const uint4*>(mine + i);
    cl.sync();   // release the remote stores / acquire the peer's
    tc::fence_proxy_async_smem();
    __syncthreads();
  }
  const uint32_t a0 = tc::smem_u32(sA) + tc::a_word_off<128>(0, a_col), b0 = tc::smem_u32(sB), b_sbo = (uint32_t)(K / 8) * 128u;
  for (int half = 0; half < 2; ++half) {
    float d[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; ++i) d[i] = 0.0f;
    tc::wg_fence();
    for (int j = 0; j < K / 16; ++j)
      tc::Wgmma<N>::mma(d, tc::make_smem_desc(a0 + half * 1024u + 4096u * j, 2048u, 128u), tc::make_smem_desc(b0 + 256u * j, 128u, b_sbo),
                        j > 0 ? 1u : 0u);
    tc::wg_commit();
    tc::wg_wait0();
#pragma unroll
    for (int i = 0; i < N / 2; ++i) {
      const int r = 128 * (int)rank + 64 * half + 16 * w + (l >> 2) + 8 * ((i >> 1) & 1), c = 8 * (i >> 2) + 2 * (l & 3) + (i & 1);
      D[(size_t)r * N + c] = d[i];
    }
  }
  cl.sync();   // neither CTA leaves while its peer may still read or write its shared memory
}

template <int N>
static int run_pair_selftest(int K, const void* A, const void* B, float* D, int a_col, int a_width, int mode, cudaStream_t st) {
  const size_t smem = (size_t)N * K * 2 + (size_t)128 * a_width * 4;
  if (cudaFuncSetAttribute(wgmma_pair_selftest_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
    return -2;
  wgmma_pair_selftest_kernel<N><<<2, 128, smem, st>>>(K, (const __half*)A, (const __half*)B, D, a_col, mode);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

}  // namespace kpn

// A (128,K) fp16, B (N,K) fp16, D (128,N) fp32: device pointers.  N in {16, 32, 48, 64, 96, 112, 128, 144, 192} (the widths
// with a wgmma instantiation), K % 16 == 0, K <= 256.  variant 0: A from the activation tile in shared memory; variant 1: A from
// registers, for the shapes of the front kernel's layers 1-3, (N, K) = (128, 144) and (64, 128).
extern "C" int kpn_selftest_umma(int N, int K, const void* A, const void* B, float* D, int variant, void* stream) {
  if (K % 16 || K < 16 || K > 256 || variant < 0 || variant > 1) return -1;
  cudaStream_t st = (cudaStream_t)stream;
  if (variant == 1) {
    if (N == 128 && K == 144) return kpn::run_ra_selftest<128, 9>(A, B, D, st);
    if (N == 64 && K == 128) return kpn::run_ra_selftest<64, 8>(A, B, D, st);
    return -1;
  }
  switch (N) {
    case 16: return kpn::run_selftest<16>(K, A, B, D, st);
    case 32: return kpn::run_selftest<32>(K, A, B, D, st);
    case 48: return kpn::run_selftest<48>(K, A, B, D, st);
    case 64: return kpn::run_selftest<64>(K, A, B, D, st);
    case 96: return kpn::run_selftest<96>(K, A, B, D, st);
    case 112: return kpn::run_selftest<112>(K, A, B, D, st);
    case 128: return kpn::run_selftest<128>(K, A, B, D, st);
    case 144: return kpn::run_selftest<144>(K, A, B, D, st);
    case 192: return kpn::run_selftest<192>(K, A, B, D, st);
    default: return -1;
  }
}

// 2-CTA self-test: A (256,K) fp16, B (N,K) fp16, D (256,N) fp32: device pointers.  N in {32, 64, 96, 128, 192}, K % 16 == 0,
// K <= 256.  The activation tile is d_col 32-bit columns wide with A at columns [a_col, a_col + K/2) (a_col % 8 == 0); mode 0 / 1 / 2:
// the peer's half of B is read through distributed shared memory / pushed by a bulk copy / written by remote stores.
extern "C" int kpn_selftest_umma2(int N, int K, const void* A, const void* B, float* D, int a_col, int d_col, int mode, void* stream) {
  if (N % 32 || N < 32 || N > 256 || K % 16 || K < 16 || K > 256) return -1;
  if (a_col < 0 || a_col % 8 || d_col % 8 || a_col + K / 2 > d_col || d_col + N > 512 || mode < 0 || mode > 2) return -1;
  cudaStream_t st = (cudaStream_t)stream;
  switch (N) {
    case 32: return kpn::run_pair_selftest<32>(K, A, B, D, a_col, d_col, mode, st);
    case 64: return kpn::run_pair_selftest<64>(K, A, B, D, a_col, d_col, mode, st);
    case 96: return kpn::run_pair_selftest<96>(K, A, B, D, a_col, d_col, mode, st);
    case 128: return kpn::run_pair_selftest<128>(K, A, B, D, a_col, d_col, mode, st);
    case 192: return kpn::run_pair_selftest<192>(K, A, B, D, a_col, d_col, mode, st);
    default: return -1;
  }
}
