// The fp32 engine's dense layer over a tile of samples, shared by its forward shading kernel (kpn_kernels.cu) and the
// backward kernels that recompute that forward (kpn_grad.cu), so that both run the same arithmetic.
#pragma once
#include "kpn_device.cuh"

namespace kpn {

constexpr int LDA = 7 * MAXK + 64;  // widest geometry input (7*KPN_MAX_KPT encodings + feat64) = 288 floats, multiple of 4
static_assert(LDA % 4 == 0, "rows are read as float4");
constexpr int LDB = 128;

enum { ACT_NONE = 0, ACT_SP = 1, ACT_ELU = 2 };

template <int ACT>
__device__ __forceinline__ float apply_act(float x) {
  if (ACT == ACT_SP) return softplus100(x);
  if (ACT == ACT_ELU) return elu1(x);
  return x;
}

// out[r][n] = act(bias[n] + sum_k in[r][k] * Wt[k][n]) for the rows of the tile (8 per warp).
// Warp w owns rows 8w..8w+7 (A operand is a warp-wide broadcast), lane owns columns lane+32j.
template <int ACT, int NJ>
__device__ __forceinline__ void dense_tile(const DevWeightsF32& W, int L, const float* sIn, int ldi, float* sOut, int ldo) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int K = W.K[L], N = W.N[L];
  constexpr int ldw = NJ * 32;
  const float* __restrict__ wt = W.wt[L];
  float acc[8][NJ];
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    float b = (lane + 32 * j < N) ? __ldg(W.bias[L] + lane + 32 * j) : 0.0f;
#pragma unroll
    for (int r = 0; r < 8; ++r) acc[r][j] = b;
  }
  const float* a0 = sIn + warp * 8 * ldi;
  int k = 0;
  for (; k + 4 <= K; k += 4) {
    float4 a[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) a[r] = *reinterpret_cast<const float4*>(a0 + r * ldi + k);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      float w[NJ];
#pragma unroll
      for (int j = 0; j < NJ; ++j) w[j] = __ldg(wt + (k + kk) * ldw + lane + 32 * j);
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        float av = kk == 0 ? a[r].x : kk == 1 ? a[r].y : kk == 2 ? a[r].z : a[r].w;
#pragma unroll
        for (int j = 0; j < NJ; ++j) acc[r][j] = fmaf(av, w[j], acc[r][j]);
      }
    }
  }
  for (; k < K; ++k) {
    float w[NJ];
#pragma unroll
    for (int j = 0; j < NJ; ++j) w[j] = __ldg(wt + k * ldw + lane + 32 * j);
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      float av = a0[r * ldi + k];
#pragma unroll
      for (int j = 0; j < NJ; ++j) acc[r][j] = fmaf(av, w[j], acc[r][j]);
    }
  }
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    int col = lane + 32 * j;
    if (col < N) {
#pragma unroll
      for (int r = 0; r < 8; ++r) sOut[(warp * 8 + r) * ldo + col] = apply_act<ACT>(acc[r][j]);
    }
  }
}

}  // namespace kpn
