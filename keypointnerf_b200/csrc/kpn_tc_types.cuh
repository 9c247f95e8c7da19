// Tensor-core engine: stage table (which dense layers run on the tensor cores, their padded shapes and where their
// fp16 weights sit in the weight blob) and the fp32 constants that travel as kernel parameters
// (biases of the tensor-core layers + the tiny layers that stay on the CUDA cores in fp32).
#pragma once
#include <stdint.h>

namespace kpn {

constexpr int TC_NSTAGE = 13;
// stage:            0 L0   1 L1  2 L2  3 L3  4 P0|CMP 5 P1 6 BASE0 7 BASE1 8 VIS1A 9 VIS1B 10 VIS2A 11 OUT0 12 RE1
// Np (padded N):    128    128   128   64    96       64   64      32      32      48      32       16      48
// Kp (padded K):    K0P    144   144   128   144      80   112     64      32      32      32       48      32
// Stage 12 (second ray-encoder layer 16->35 of the colour head, executed FIRST in the colour kernel) also carries its bias row.
// The geometry stages (0..5) carry their bias as one extra K row (the activation tile holds a constant 1 there), so their
// epilogues have no per-column constants.  Stage 0 additionally permutes its inputs (tc_kmap) so that the two threads
// that build a row's input each write one contiguous, 16-byte aligned run of activation-tile columns.

struct TcStage {
  int Kp, Np;
  uint32_t off;  // byte offset of the stage's weight tile in the blob
};

struct TcPlan {
  TcStage st[TC_NSTAGE];
  uint32_t total_bytes;
  int K0P;  // padded input width of layer 0
};

// keypoint pairs of the layer-0 input: keypoints 2j and 2j+1 share the fp16 words of pair j; with an odd count the last
// pair's second slot has no weights (the blob is zero there) and the kernel writes 0 into it
__host__ __device__ constexpr int tc_npair(int n_kpt) { return (n_kpt + 1) / 2; }
// layer-0 input width incl. the bias row, padded to a multiple of 16
__host__ __device__ constexpr int tc_k0p(int n_kpt) { return ((14 * tc_npair(n_kpt) + 64 + 1) + 15) / 16 * 16; }

// Split of the layer-0 input between the two threads of a row: thread 0 builds keypoint pairs [0, pa) and feature channels
// [0, fa) as words [0, 7*pa + fa/2), thread 1 the remaining pairs, the remaining channels and the bias column from there on.
// Both runs start on a 16-byte chunk: 7*pa + fa/2 = 0 (mod 4) with fa a multiple of 4 (float4 groups of feat64), so pa is
// even.  The split depends on the pair count only (an odd count shares its even neighbour's kernel) and balances the two
// runs' words; 17/18 and 23/24 keypoints keep the 4 | 40 split the engine has always used for 18 and 24 (another split
// permutes the K order of layer 0, which changes the last bits of its sums).
struct TcSplit { int pa, fa; };
__host__ __device__ constexpr TcSplit tc_l0_split(int n_kpt) {
  const int np = tc_npair(n_kpt);
  if (np == 9 || np == 12) return TcSplit{4, 40};
  const int half = tc_k0p(n_kpt) / 4;   // words per thread of an even split
  TcSplit best{0, 0};
  int best_d = 1 << 30;
  for (int pa = 0; pa <= np; pa += 2)
    for (int fa = 0; fa <= 64; fa += 4) {
      const int c1 = 7 * pa + fa / 2;
      const int d = c1 > half ? c1 - half : half - c1;
      if (c1 % 4 == 0 && d < best_d) { best = TcSplit{pa, fa}; best_d = d; }
    }
  return best;
}
__host__ __device__ constexpr int tc_l0_pa(int n_kpt) { return tc_l0_split(n_kpt).pa; }
__host__ __device__ constexpr int tc_l0_fa(int n_kpt) { return tc_l0_split(n_kpt).fa; }

// K index (fp16 element of the activation row) that input `i` of geometry stage `stage` is multiplied with.
// Stage 0 inputs: i < 7*n_kpt is encoding element r*n_kpt + k (reference src/spatial.py layout), else feat64 channel.
__host__ __device__ constexpr int tc_kmap(int stage, int n_kpt, int i) {
  if (stage != 0) return i;
  const int NP = tc_npair(n_kpt), PA = tc_l0_pa(n_kpt), FA = tc_l0_fa(n_kpt);
  if (i < 7 * n_kpt) {
    const int r = i / n_kpt, k = i % n_kpt, j = k / 2;
    const int col = j < PA ? 7 * j + r : 7 * PA + FA / 2 + 7 * (j - PA) + r;
    return 2 * col + (k & 1);
  }
  const int c = i - 7 * n_kpt;
  return c < FA ? 2 * 7 * PA + c : 2 * (7 * PA + FA / 2 + 7 * (NP - PA)) + (c - FA);
}
// K index of the bias row of a geometry stage (or of stage 12)
__host__ __device__ constexpr int tc_kbias(int stage, int n_kpt) {
  switch (stage) {
    case 0: return 2 * (7 * tc_npair(n_kpt) + 32);
    case 1: return 128;
    case 2: return 136;
    case 3: return 120;
    case 4: return 128;
    case 12: return 16;
    default: return 64;
  }
}

__host__ __device__ constexpr TcPlan make_tc_plan(int n_kpt) {
  TcPlan p{};
  const int Kp[TC_NSTAGE] = {tc_k0p(n_kpt), 144, 144, 128, 144, 80, 112, 64, 32, 32, 32, 48, 32};
  const int Np[TC_NSTAGE] = {128, 128, 128, 64, 96, 64, 64, 32, 32, 48, 32, 16, 48};
  uint32_t off = 0;
  for (int i = 0; i < TC_NSTAGE; ++i) {
    p.st[i].Kp = Kp[i];
    p.st[i].Np = Np[i];
    p.st[i].off = off;
    off += (uint32_t)(Kp[i] * Np[i] * 2);
  }
  p.total_bytes = off;
  p.K0P = Kp[0];
  return p;
}

// fp32 constants, passed by value as a __grid_constant__ kernel parameter so that unrolled epilogues read
// them as constant-bank operands.
struct TcConsts {
  float w_p2[2][64], b_p2[2];          // density head last layer (fp32 on CUDA cores); the geometry-stage biases ride in the MMAs
  float w_re0[16][4], b_re0[16];       // ray-direction encoder, first layer (the second runs on the tensor core, stage 12)
  float b_base0[64], b_base1[32], b_vis1a[32], b_vis1b[48], b_vis2a[32];
  float w_vis2b[32], b_vis2b;
  float b_out0[16];
  float w_out1[8][16], b_out1[8];
  float w_out2[8], b_out2;
  float ani_abs;
};

}  // namespace kpn
