// Ray-march shading, engine 0: Hopper tensor-core MLPs (wgmma, fp16 operands in shared memory, fp32 accumulators in
// registers, weights resident in shared memory through one bulk-TMA load per CTA).  The kernels that depend on the number of
// source views NV live in this header; kpn_shade_tc.cu instantiates them for 3 views (and holds the kernels every view count
// shares), kpn_shade_tc_v4.cu for 4 views.
//
// Three persistent kernels per batch of valid samples:
//   geo_front_kernel  : gather + keypoint encoding + geometry MLP (L0-L3) + view pooling.  A row is one (sample, source view)
//                       pair; the NV views of a sample sit in NV adjacent lanes (32 / NV samples per warp: 10 with 3 views,
//                       8 with 4).  The pooling (reference src/utils.py:722-748) reads the sample's NV rows from shared
//                       memory and writes the pooled [mean | var] (fp32) of every sample to a scratch buffer.
//   geo_tail_kernel   : density tail per sample (P0|compress, P1 with two-term fp16 weights W_hi + W_lo and two-term
//                       activations, 64->2 head in fp32).  Writes alpha/sdf and, where a colour is needed, the 24-wide
//                       compressed latent (fp16).  The tail is a kernel of its own because the geometry stages' W_hi tiles and
//                       the tail's W_hi + W_lo tiles do not fit in one SM's 227 KB of shared memory together with the tiles.
//   shade_color_kernel: IBR colour head (RE1, BASE0, BASE1, VIS1A, VIS1B, VIS2A, OUT0 on tensor cores; first ray-encoder layer,
//                       32->1, 16->8->1 in fp32 on CUDA cores) for the samples with density > 0 (colour_list_kernel's list).
// Common structure: a warpgroup (4 warps) owns a tile of rows.  Row threads build a layer input as packed fp16 pairs in an
// activation tile in shared memory (tc::a_word_off layout), the warpgroup multiplies it with the resident weights
// (wgmma.mma_async, M = 64 per instruction), and the epilogue either runs on the accumulator fragments directly (elementwise
// activations, written straight into the next layer's activation tile) or stores them to shared memory for the row threads
// (cross-view reductions).  Biases ride in the MMAs as one extra K row multiplied by a constant 1 in the activation tile.
// Stage table:
//   geo    0 L0 190->128 | 1 L1 128->128 | 2 L2 136->120 | 3 L3 120->64 | 4 P0|CMP 128->64|24 | 5 P1 64->64
//   colour 12 RE1 16->35 | 6 BASE0 105->64 | 7 BASE1 64->32 | 8 VIS1A 32->32 | 9 VIS1B 32->33 | 10 VIS2A 32->32 | 11 OUT0 37->16
#pragma once
#include <array>
#include <atomic>
#include <cstdlib>
#include <type_traits>
#include <utility>
#include "kpn_device.cuh"
#include "kpn_launch.h"
#include "kpn_tc.cuh"
#include "kpn_tc_types.cuh"

namespace kpn {
namespace {

constexpr int ROW_WARPS = 4;                              // warps of a warpgroup
constexpr int GEO_NSTAGE = 6;                             // colour stages start at plan.st[6]
// samples per warp (NV views each): 10 with 3 views (lanes 30, 31 idle), 8 with 4
__host__ __device__ constexpr int spw(int nv) { return 32 / nv; }
__host__ __device__ constexpr int spt(int nv) { return spw(nv) * ROW_WARPS; }   // samples per colour tile (128 rows)
constexpr float LOG2E = 1.4426950408889634f;
constexpr unsigned FULL = 0xffffffffu;

__device__ __forceinline__ float ex2f(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float lg2f(float x) { float y; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float rcpf(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

// Softplus(beta=100): max(x,0) + log1p(exp(-100|x|))/100  (reference src/utils.py:523-524; beyond the
// reference's threshold the correction term is < 2e-11).
__device__ __forceinline__ float sp_fast(float x) {
  float e = ex2f(-100.0f * LOG2E * fabsf(x));
  return fmaf(0.0069314718056f, lg2f(1.0f + e), fmaxf(x, 0.0f));
}
__device__ __forceinline__ float elu_fast(float x) { return x > 0.0f ? x : ex2f(x * LOG2E) - 1.0f; }
__device__ __forceinline__ float sig_fast(float x) { return rcpf(1.0f + ex2f(-x * LOG2E)); }
__device__ __forceinline__ float u2f(uint32_t u) { return __uint_as_float(u); }

// two-term fp16 split of a pair of activations: hi = fp16(x), lo = fp16(x - hi)
__device__ __forceinline__ void split_h2(float a, float b, uint32_t& hi, uint32_t& lo) {
  __half2 h = __floats2half2_rn(a, b);
  float2 f = __half22float2(h);
  __half2 l = __floats2half2_rn(a - f.x, b - f.y);
  hi = *reinterpret_cast<uint32_t*>(&h);
  lo = *reinterpret_cast<uint32_t*>(&l);
}

// Scene constants the row threads need, staged once per CTA in shared memory (the per-view index differs per lane).
template <int NV>
struct SceneS {
  float P[NV][12];   // KRT rows
  float E[NV][12];   // extrinsic rows
  float C[NV][4];    // source camera centres
  float4 kc[NV][KPN_MAX_KPT];   // keypoints in camera space
  float wm1, hm1, znear, inv_zrange, sp_scale, inv2sig2, inv_wm1, inv_hm1;
  MapDesc f64, f8, ftex, img;
};

template <int NV>
__device__ __forceinline__ Proj project_s(const SceneS<NV>& S, int v, const float p[3]) {
  const float* P = S.P[v];
  float hx = P[0] * p[0] + P[1] * p[1] + P[2] * p[2] + P[3];
  float hy = P[4] * p[0] + P[5] * p[1] + P[6] * p[2] + P[7];
  float hz = P[8] * p[0] + P[9] * p[1] + P[10] * p[2] + P[11];
  Proj r;
  r.u = 2.0f * ((hx / hz) / S.wm1) - 1.0f;
  r.v = 2.0f * ((hy / hz) / S.hm1) - 1.0f;
  r.zn = 2.0f * (hz - S.znear) * S.inv_zrange - 1.0f;
  return r;
}
__device__ __forceinline__ float boundary_weight_fast(const Proj& q) {
  float c[3] = {q.u, q.v, q.zn};
  float w = 1.0f;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    float x = 0.5f * c[i] + 0.5f;
    float db = fminf(x, 1.0f - x);
    w *= sig_fast(fmaf(50.0f, db, -5.0f));   // sigmoid(5*(db/0.1 - 1)), reference src/model.py:755
  }
  return w;
}

// Keypoint encoding of one keypoint with sp_level == 3: sin/cos(pi*2^l*dz) from one sincos + double angles.
template <int NV>
__device__ __forceinline__ void encode_fast(const SceneS<NV>& S, int v, int k, const float c[3], float e[7]) {
  const float4 kc = S.kc[v][k];
  float dx = c[0] - kc.x, dy = c[1] - kc.y, dzc = c[2] - kc.z;
  float dz = S.sp_scale * dzc;
  float w = __expf(-(dx * dx + dy * dy + dzc * dzc) * S.inv2sig2);
  // sin/cos(pi * dz) have period 2 in dz: reduce to [-1, 1] first, so that the fast intrinsic stays accurate for any scale of the
  // scene (sp_args.sigma = 150 / millimetre scenes make |dz| large; with metres and sigma = 0.1 the reduction is the identity)
  const float dr = fmaf(-2.0f, rintf(0.5f * dz), dz);
  float s, co;
  __sincosf(dr * 3.14159265358979f, &s, &co);
  float s2 = 2.0f * s * co, c2 = 1.0f - 2.0f * s * s;
  float s4 = 2.0f * s2 * c2, c4 = 1.0f - 2.0f * s2 * s2;
  e[0] = dz * w; e[1] = s * w; e[2] = co * w; e[3] = s2 * w; e[4] = c2 * w; e[5] = s4 * w; e[6] = c4 * w;
}

constexpr uint32_t H2_ONE = 0x00003C00u;   // fp16 pair (1.0, 0.0): the activation column that multiplies the bias row

// softplus(beta=100) of two accumulators -> packed fp16 pair, on packed halves and WITHOUT the special-function unit: x is
// rounded to fp16 first (the result is an fp16 activation anyway), y = max(x,0) + c(|x|) with the correction
// c(t) = log1p(exp(-100 t))/100 ~ q^3 (a0 + a1 q + a2 q^2), q = sat(1 - t/0.08)  (minimax fit, fp16 coefficients): 8 instructions
// per pair (F2FP, HFMA2.SAT, 2 HMUL2, 3 HFMA2, HMNMX2).  Against the exact softplus over every fp16 input the error is
// <= 2.8e-5 (rms 9e-6; rounding the exact result to fp16 alone: 1.9e-5 / 2.5e-6), and the rendered RGB error is unchanged
// (tools/err_budget.py: 7.6e-4 vs 7.7e-4 max on the bench-scene tile).  The previous form took one MUFU.EX2 per ELEMENT; at 4
// lanes/clk/quarter the three 128-wide epilogues of a tile kept the XU pipe busy for 1.5k cycles per warp and throttled MIO.
__device__ __forceinline__ uint32_t sp_pair(uint32_t a0, uint32_t a1) {
  const __half2 xh = __floats2half2_rn(u2f(a0), u2f(a1));
  const uint32_t k_it = 0xca40ca40u;   // -12.5 = -1 / 0.08
  const uint32_t k_one = 0x3c003c00u;
  const uint32_t a2 = 0x24c724c7u, a1c = 0xa459a459u, a0c = 0x1d631d63u;   // 0.018666, -0.016988, 0.00526 (fp16)
  const uint32_t xa = *reinterpret_cast<const uint32_t*>(&xh) & 0x7fff7fffu;   // |x| (folds into the HFMA2 as an operand modifier)
  uint32_t q;
  asm("fma.rn.sat.f16x2 %0, %1, %2, %3;" : "=r"(q) : "r"(xa), "r"(k_it), "r"(k_one));
  const __half2 qh = *reinterpret_cast<const __half2*>(&q);
  const __half2 q2 = __hmul2(qh, qh);
  const __half2 q3 = __hmul2(q2, qh);
  __half2 p = __hfma2(*reinterpret_cast<const __half2*>(&a2), qh, *reinterpret_cast<const __half2*>(&a1c));
  p = __hfma2(p, qh, *reinterpret_cast<const __half2*>(&a0c));
  const uint32_t zero = 0u;
  const __half2 y = __hfma2(p, q3, __hmax2(xh, *reinterpret_cast<const __half2*>(&zero)));
  return *reinterpret_cast<const uint32_t*>(&y);
}

template <int NV>
__device__ __forceinline__ void stage_scene(SceneS<NV>& scs, const DevScene& g, int NK, int t, int nthreads) {
  for (int i = t; i < NV * 12; i += nthreads) { scs.P[i / 12][i % 12] = g.P[i / 12][i % 12]; scs.E[i / 12][i % 12] = g.E[i / 12][i % 12]; }
  for (int i = t; i < NV * 3; i += nthreads) scs.C[i / 3][i % 3] = g.C[i / 3][i % 3];
  for (int i = t; i < NV * NK; i += nthreads)
    scs.kc[i / NK][i % NK] = make_float4(g.kc[i / NK][i % NK][0], g.kc[i / NK][i % NK][1], g.kc[i / NK][i % NK][2], 0.0f);
  if (t == 0) {
    scs.wm1 = g.wm1; scs.hm1 = g.hm1; scs.znear = g.znear; scs.inv_zrange = 1.0f / (g.zfar - g.znear);
    scs.sp_scale = g.sp_scale; scs.inv2sig2 = g.inv2sig2; scs.inv_wm1 = 1.0f / g.wm1; scs.inv_hm1 = 1.0f / g.hm1;
    scs.f64 = g.f64; scs.f8 = g.f8; scs.ftex = g.ftex; scs.img = g.img;
  }
}

__device__ __forceinline__ void load_weights(uint8_t* dst, const uint8_t* src, uint32_t bytes, uint64_t* wbar) {
  tc::mbar_expect_tx(wbar, bytes);
  for (uint32_t off = 0; off < bytes; off += 32768u) {
    uint32_t n = bytes - off < 32768u ? bytes - off : 32768u;
    tc::bulk_g2s(dst + off, src + off, n, wbar);
  }
  tc::mbar_wait(wbar, 0, 0x30u);
}

// =====================================================================================================================
// activation tiles, warpgroup synchronisation
// =====================================================================================================================
// store N words (packed fp16 pairs) of row r at word columns [c0, c0 + N) of an activation tile; c0 % 4 == 0
template <int ROWS, int N>
__device__ __forceinline__ void a_put(uint8_t* tile, int r, int c0, const uint32_t* w) {
  static_assert(N % 4 == 0, "runs are whole 16-byte chunks");
#pragma unroll
  for (int i = 0; i < N; i += 4)
    *reinterpret_cast<uint4*>(tile + tc::a_word_off<ROWS>(r, c0 + i)) = make_uint4(w[i], w[i + 1], w[i + 2], w[i + 3]);
}
__device__ __forceinline__ void a_word(uint8_t* tile64, int r, int c, uint32_t w) {
  *reinterpret_cast<uint32_t*>(tile64 + tc::a_word_off<64>(r, c)) = w;
}
// store words [C0, C0 + N) of row r of a 64-row tile: whole 16-byte chunks as one store, the words of a chunk the run shares with
// another writer one at a time
template <int C0, int N>
__device__ __forceinline__ void a_put_span(uint8_t* tile64, int r, const uint32_t* w) {
#pragma unroll
  for (int ch = C0 / 4; ch < (C0 + N + 3) / 4; ++ch) {
    if (4 * ch >= C0 && 4 * ch + 4 <= C0 + N) {
      const int i = 4 * ch - C0;
      *reinterpret_cast<uint4*>(tile64 + tc::a_word_off<64>(r, 4 * ch)) = make_uint4(w[i], w[i + 1], w[i + 2], w[i + 3]);
    } else {
#pragma unroll
      for (int c = 4 * ch; c < 4 * ch + 4; ++c)
        if (c >= C0 && c < C0 + N) a_word(tile64, r, c, w[c - C0]);
    }
  }
}
// the activation tile written by this warpgroup's threads becomes visible to its MMAs
__device__ __forceinline__ void wg_publish(int bar_id) {
  tc::fence_proxy_async_smem();
  tc::named_sync(bar_id, 128);
}

// The NV lanes of this lane's sample: sums, minima and maxima over the views.  Every lane of the group gets the same sum, in
// the reference's order v0 + v1 + ... (torch.sum over the view dimension).
template <int NV>
struct Group {
  int gb;   // lane of view 0
  __device__ explicit Group(int lane) : gb(NV * (lane / NV)) {}
  __device__ float sum(float x) const {
    float s = __shfl_sync(FULL, x, gb & 31);
#pragma unroll
    for (int i = 1; i < NV; ++i) s += __shfl_sync(FULL, x, (gb + i) & 31);
    return s;
  }
  __device__ float vmin(float x) const {
    float m = x;
#pragma unroll
    for (int i = 0; i < NV; ++i) m = fminf(m, __shfl_sync(FULL, x, (gb + i) & 31));
    return m;
  }
  __device__ float vmax(float x) const {
    float m = x;
#pragma unroll
    for (int i = 0; i < NV; ++i) m = fmaxf(m, __shfl_sync(FULL, x, (gb + i) & 31));
    return m;
  }
};
// 3 views: each lane adds the other two lanes' values in the order of its own view (unchanged since the first 3-view kernels, so
// that their results stay bit-identical)
template <>
struct Group<3> {
  int l1, l2;
  __device__ explicit Group(int lane) {
    const int gb = 3 * (lane / 3);
    l1 = (gb + (lane - gb + 1) % 3) & 31;
    l2 = (gb + (lane - gb + 2) % 3) & 31;
  }
  __device__ float sum(float x) const { return x + __shfl_sync(FULL, x, l1) + __shfl_sync(FULL, x, l2); }
  __device__ float vmin(float x) const { return fminf(x, fminf(__shfl_sync(FULL, x, l1), __shfl_sync(FULL, x, l2))); }
  __device__ float vmax(float x) const { return fmaxf(x, fmaxf(__shfl_sync(FULL, x, l1), __shfl_sync(FULL, x, l2))); }
};

// Weighted mean and variance over the NV views of four feature columns (x[u]: view u's columns, w[u]: its weight), with the
// roundings Group<NV>::sum gives the lane of view 0: mean = sum_u w_u x_u, var = sum_u (w_u dl_u) dl_u with dl_u = x_u - mean_u,
// where mean_u is the mean as view u's lane sums it (with 3 views that lane starts at its own view, so the three means may
// differ in the last bit).  The explicit _rn intrinsics keep ptxas from contracting any of it into an FFMA.
template <int NV>
__device__ __forceinline__ float pool_sum(const float* a, int u0) {
  float s = a[u0];
#pragma unroll
  for (int i = 1; i < NV; ++i) s = __fadd_rn(s, a[(u0 + i) % NV]);
  return s;
}
template <int NV>
__device__ __forceinline__ void pool_views(const float* w, const float4* x, float4& mn, float4& vr) {
  float m[4], q[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float xs[NV], p[NV], e[NV];
#pragma unroll
    for (int u = 0; u < NV; ++u) {
      xs[u] = i == 0 ? x[u].x : i == 1 ? x[u].y : i == 2 ? x[u].z : x[u].w;
      p[u] = __fmul_rn(w[u], xs[u]);
    }
    m[i] = pool_sum<NV>(p, 0);
#pragma unroll
    for (int u = 0; u < NV; ++u) {
      const float dl = __fsub_rn(xs[u], NV == 3 ? pool_sum<NV>(p, u) : m[i]);
      e[u] = __fmul_rn(__fmul_rn(w[u], dl), dl);
    }
    q[i] = pool_sum<NV>(e, 0);
  }
  mn = make_float4(m[0], m[1], m[2], m[3]);
  vr = make_float4(q[0], q[1], q[2], q[3]);
}

// =====================================================================================================================
// geometry front: stages L0-L3 + view pooling.  Warpgroup tile = 64 rows: row warps 0/1 hold rows 0-31 with column half
// h = 0 / 1, row warps 2/3 rows 32-63 (the two threads of a row split the layer-0 input build, as tc_kmap's runs are laid
// out), so that each warp's wgmma fragment rows are rows of its own lanes.  2 * spw(NV) samples per tile: 20 with 3 views, 16 with 4.
// =====================================================================================================================
constexpr int GWG = 2;                        // warpgroups per CTA of the tail kernel (the front kernel's: front_wgs)
__host__ __device__ constexpr int fspt(int nv) { return 2 * spw(nv); }   // samples per front tile
constexpr int D3S = 68;                       // row stride (floats) of the L3 accumulator rows staged for the pooling
constexpr int POOL_W = 128;                   // pooled [mean 64 | var 64] fp32 per sample
constexpr long long POOL_SLICE = 1ll << 22;   // samples per front/tail launch pair (bounds the pooled scratch to 2 GiB)
// activation tile of a front warpgroup: 64 rows of the layer-0 input, which is at least as wide as the 144-wide inputs of
// L1 / L2 for 9 keypoints and more; fewer keypoints get the L1 / L2 width
__host__ __device__ constexpr uint32_t front_tile_bytes(int n_kpt) {
  return 64u * (uint32_t)(tc_k0p(n_kpt) > 144 ? tc_k0p(n_kpt) : 144) * 2u;
}
static_assert(64 * D3S * 4 + 64 * 4 <= 64 * 144 * 2, "the L3 rows and the rows' view weights fit in the activation tile");
// Warpgroups per front CTA: as many tiles as fit beside the resident W_hi of stages 0..3 in the 227 KB an SM gives a block,
// up to three.  The row threads' gathers are latency bound, so a third warpgroup helps hide them; the register file caps the
// CTA at three (168 registers per thread at 384 threads).  Three tiles fit up to K0P 208 (20 keypoints: 223 232 B dynamic +
// the static scene block), two up to 28 keypoints (229 376 B), one above (29..32 keypoints: K0P 288 / 304).
// Three warpgroups also need K0P >= 192 (15..20 keypoints): when the feat64 taps were loaded by the row's own threads, narrower
// layer-0 inputs put up to all 64 channels (64 LDG.128) on one thread of a row, and built for 168 registers ptxas spilled or
// serialised the wgmma chain of some of those pair counts, so 1..14 keypoints keep two.  gather_feat64 now spreads the taps
// evenly over both warps of a row; three warpgroups for 1..14 keypoints have not been compiled and measured since.
constexpr uint32_t SMEM_OPTIN = 227u * 1024u;
// static shared memory of the front kernel (SceneS<NV> + mbarrier, ptxas): 2 000 B with 3 views, 2 624 B with 4
constexpr uint32_t FRONT_STATIC_V3 = 2048u;
constexpr uint32_t FRONT_STATIC_V4 = 3072u;
__host__ __device__ constexpr uint32_t front_static(int nv) { return nv <= 3 ? FRONT_STATIC_V3 : FRONT_STATIC_V4; }
static_assert(sizeof(SceneS<3>) + sizeof(uint64_t) <= FRONT_STATIC_V3, "static shared memory of the 3-view front kernel");
static_assert(sizeof(SceneS<4>) + sizeof(uint64_t) <= FRONT_STATIC_V4, "static shared memory of the 4-view front kernel");
__host__ __device__ constexpr uint32_t front_smem_bytes(int n_kpt, int wgs) {
  return make_tc_plan(n_kpt).st[4].off + (uint32_t)wgs * front_tile_bytes(n_kpt);
}
__host__ __device__ constexpr int front_wgs(int n_kpt, int nv) {
  return tc_k0p(n_kpt) >= 192 && front_smem_bytes(n_kpt, 3) + front_static(nv) <= SMEM_OPTIN ? 3
         : front_smem_bytes(n_kpt, 2) + front_static(nv) <= SMEM_OPTIN                       ? 2
                                                                                              : 1;
}
static_assert(front_wgs(1, 3) == 2 && front_wgs(14, 3) == 2 && front_wgs(15, 3) == 3 && front_wgs(18, 3) == 3 &&
                  front_wgs(20, 3) == 3 && front_wgs(21, 3) == 2 && front_wgs(24, 3) == 2 && front_wgs(28, 3) == 2 &&
                  front_wgs(29, 3) == 1, "front CTA layouts");
static_assert(front_wgs(1, 4) == 2 && front_wgs(14, 4) == 2 && front_wgs(15, 4) == 3 && front_wgs(18, 4) == 3 &&
                  front_wgs(20, 4) == 3 && front_wgs(21, 4) == 2 && front_wgs(24, 4) == 2 && front_wgs(28, 4) == 2 &&
                  front_wgs(29, 4) == 1,
              "4-view front CTA layouts: the larger scene block keeps three warpgroups up to 20 keypoints, two up to 28");
static_assert(front_smem_bytes(KPN_MAX_KPT, 1) + FRONT_STATIC_V4 <= SMEM_OPTIN, "one warpgroup fits at the maximum count");
// offsets of the tail's (4, 5) and the colour head's (6..12) tiles relative to the first of them; the tiles past stage 0 have
// the same size for every keypoint count, so any count's plan gives them
constexpr TcPlan REL_PLAN = make_tc_plan(KPN_MAX_KPT);

// one geometry stage of the warpgroup: A (64 rows at `a`) x resident W tile at `b` -> d (N = 128 or 64 fp32 per row)
template <int N, int KCH>
__device__ __forceinline__ void front_mma(float* d, const uint8_t* a, uint32_t b, int bar_id) {
  wg_publish(bar_id);
  tc::wg_fence();
  tc::wg_mma<N, KCH>(d, tc::smem_u32(a), 1024u, b, (uint32_t)(N / 8) * 128u, 0u);
  tc::wg_commit();
  tc::wg_wait0();
  tc::named_sync(bar_id, 128);   // every warp's MMAs are complete: the tile may be overwritten
}
// softplus epilogue of a 128-wide stage on the fragments: next layer's input words [0, 64); bias_tail: words 60..63 become
// (1,0),0,0,0 (layer-3 input: bias column + K padding)
__device__ __forceinline__ void front_epi_sp(const float* d, uint8_t* a, int wq, int lane, bool bias_tail) {
#pragma unroll
  for (int m = 0; m < 32; ++m) {
    const int r = 16 * wq + (lane >> 2) + 8 * (m & 1), c = 4 * (m >> 1) + (lane & 3);
    uint32_t w = sp_pair(__float_as_uint(d[2 * m]), __float_as_uint(d[2 * m + 1]));
    if (bias_tail && m >= 30) w = (lane & 3) == 0 ? H2_ONE : 0u;
    a_word(a, r, c, w);
  }
}

// keypoint encodings of pair j (keypoints 2j, 2j+1) as 7 packed fp16 words; the second slot of an odd count's last pair is 0
template <int NP, int NV>
__device__ __forceinline__ void encode_pair(const SceneS<NV>& S, int v, int j, int nk, const float c[3], uint32_t* a) {
  float e0[7], e1[7];
  encode_fast(S, v, 2 * j, c, e0);
  if (j < NP - 1 || 2 * j + 1 < nk) {
    encode_fast(S, v, 2 * j + 1, c, e1);
  } else {
#pragma unroll
    for (int r = 0; r < 7; ++r) e1[r] = 0.0f;
  }
#pragma unroll
  for (int r = 0; r < 7; ++r) a[r] = tc::pack_h2(e0[r], e1[r]);
}

// feat64 channels of the layer-0 input (reference src/utils.py:74-89), loaded a whole 128-byte line per row at a time.  The row
// warps 2 rh and 2 rh + 1 hold the same 32 rows (lane = row); warp h gathers all 64 channels of its lanes 16h .. 16h + 15, four rows
// per step: lanes 8g .. 8g + 7 take row 16h + 4k + g of step k, and lane l8 = lane & 7 loads float4 groups l8 and l8 + 8 of that
// row's four taps (each load instruction reads four whole lines, one per row; with a lane per row it read ~30 lines of 16 bytes
// each).  The row's tap offsets and weights come from its lane by shuffles.  Each channel is blended with gather_f32's
// expression and packed with the same pairs, and each word goes to the column tc_kmap gives it: channel c < FA to word
// 7 PA + c/2 (thread 0's run), c >= FA to word C1 + NE + (c - FA)/2 (thread 1's run, after its NE encoding words).
template <int NV, int NP>
__device__ __forceinline__ void gather_feat64(const MapDesc& m, const Taps& t, uint8_t* A, int row0, int h, int lane) {
  constexpr int NK = 2 * NP, PA = tc_l0_pa(NK), FA = tc_l0_fa(NK), C1 = 7 * PA + FA / 2, NE = 7 * (NP - PA);
  static_assert(PA % 2 == 0 && FA % 4 == 0 && C1 % 2 == 0, "thread 0's feature words start on an even column");
  const int o[4] = {t.o00, t.o01, t.o10, t.o11};   // texel offsets within the view's plane
  const size_t plane = (size_t)m.H * m.W;
  const float4* base = reinterpret_cast<const float4*>(m.ptr);
  const int l8 = lane & 7;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int src = 16 * h + 4 * k + (lane >> 3);
    const float4* vb = base + (size_t)(src % NV) * plane * 16;   // the row's view (lane = NV g + v); 16 float4 per texel
    const float4* p[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) p[i] = vb + (size_t)__shfl_sync(FULL, o[i], src) * 16;
    const float w00 = __shfl_sync(FULL, t.w00, src), w01 = __shfl_sync(FULL, t.w01, src);
    const float w10 = __shfl_sync(FULL, t.w10, src), w11 = __shfl_sync(FULL, t.w11, src);
    const int r = row0 + src;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int c4 = l8 + 8 * i;
      const float4 a = __ldg(p[0] + c4), b = __ldg(p[1] + c4), c = __ldg(p[2] + c4), d = __ldg(p[3] + c4);
      const uint32_t x0 = tc::pack_h2(a.x * w00 + b.x * w01 + c.x * w10 + d.x * w11, a.y * w00 + b.y * w01 + c.y * w10 + d.y * w11);
      const uint32_t x1 = tc::pack_h2(a.z * w00 + b.z * w01 + c.z * w10 + d.z * w11, a.w * w00 + b.w * w01 + c.w * w10 + d.w * w11);
      const int col = 4 * c4 < FA ? 7 * PA + 2 * c4 : C1 + NE + 2 * (c4 - FA / 4);
      if (NE % 2 == 1 && (col & 1)) {
        a_word(A, r, col, x0);
        a_word(A, r, col + 1, x1);
      } else {
        *reinterpret_cast<uint2*>(A + tc::a_word_off<64>(r, col)) = make_uint2(x0, x1);
      }
    }
  }
}

// feat8 channels [4h, 4h + 4) of the layer-2 input as two packed words (gather_f32's blend, same pairs as the 8-channel gather)
template <int NV>
__device__ __forceinline__ void gather_feat8(const SceneS<NV>& S, int v, const Proj& q, int h, uint32_t w[2]) {
  const Taps t8 = make_taps(q.u, q.v, S.f8.W, S.f8.H);
  float g8[4];
  gather_f32<1>(S.f8, v, t8, h, g8);
  w[0] = tc::pack_h2(g8[0], g8[1]);
  w[1] = tc::pack_h2(g8[2], g8[3]);
}

// Layer-0 input of one tile, this thread's part (reference src/spatial.py:63-118 encoding | src/utils.py:74-89 feat64 gather),
// column order tc_kmap: thread h of row `row` writes the keypoint encodings of its run (and thread 1 the bias column and K
// padding); the feat64 words of both runs come from gather_feat64.
template <int NV, int NP>
__device__ __forceinline__ void front_l0_encode(const SceneS<NV>& scs, int v, int nk, const float p[3], uint8_t* A, int row, int h) {
  constexpr int NK = 2 * NP, PA = tc_l0_pa(NK), FA = tc_l0_fa(NK);
  float c[3];
  const float* E = scs.E[v];
  c[0] = E[0] * p[0] + E[1] * p[1] + E[2] * p[2] + E[3];
  c[1] = E[4] * p[0] + E[5] * p[1] + E[6] * p[2] + E[7];
  c[2] = E[8] * p[0] + E[9] * p[1] + E[10] * p[2] + E[11];
  constexpr int C1 = 7 * PA + FA / 2;             // thread 0's run: words [0, C1); thread 1's: [C1, K0P / 2)
  static_assert(C1 % 4 == 0 && C1 > 0, "both runs start on a 16-byte chunk");
  if (h == 0) {
    if constexpr (PA > 0) {
      uint32_t a[7 * PA];
#pragma unroll
      for (int j = 0; j < PA; ++j) encode_pair<NP, NV>(scs, v, j, nk, c, a + 7 * j);
      a_put_span<0, 7 * PA>(A, row, a);
    }
  } else {
    constexpr int NE = 7 * (NP - PA), NF = (64 - FA) / 2;
    constexpr int N1 = tc_k0p(NK) / 2 - C1;
    static_assert(NE + NF + 1 <= N1, "the bias column is in thread 1's run");
    uint32_t a[NE > 0 ? NE : 1];
#pragma unroll
    for (int j = PA; j < NP; ++j) encode_pair<NP, NV>(scs, v, j, nk, c, a + 7 * (j - PA));
    if constexpr (NE > 0) a_put_span<C1, NE>(A, row, a);
    uint32_t b[N1 - NE - NF];
    b[0] = H2_ONE;
#pragma unroll
    for (int i = 1; i < N1 - NE - NF; ++i) b[i] = 0u;
    a_put_span<C1 + NE + NF, N1 - NE - NF>(A, row, b);
  }
}

// L3 rows (d3: the m64n64 accumulator fragment) and the rows' view weights to shared memory over the warpgroup's activation tile,
// then the view pooling: weighted mean || variance over the NV rows of a sample (src/utils.py:722-748), one (sample, 4 columns)
// item per thread at a time.  The caller has retired every MMA that reads the tile; on return the tile is free again.
template <int NV>
__device__ __forceinline__ void front_pool(const float* d3, float pw, float* D3, int wq, int lane, int row, int h, long long base,
                                           long long end, int tile, float* __restrict__ pool, int bar_id) {
  constexpr int SPW = spw(NV), FSPT = fspt(NV);
#pragma unroll
  for (int m = 0; m < 16; ++m) {
    const int r = 16 * wq + (lane >> 2) + 8 * (m & 1), c = 8 * (m >> 1) + 2 * (lane & 3);
    *reinterpret_cast<float2*>(D3 + r * D3S + c) = make_float2(d3[2 * m], d3[2 * m + 1]);
  }
  if (h == 0) D3[64 * D3S + row] = pw;
  tc::named_sync(bar_id, 128);
  for (int it = 32 * wq + lane; it < FSPT * 16; it += 128) {
    const int s = it >> 4, c = 4 * (it & 15);
    const int r0 = (s / SPW) * 32 + NV * (s % SPW);   // row of the sample's view 0
    float4 x[NV];
    float w[NV];
#pragma unroll
    for (int u = 0; u < NV; ++u) {
      x[u] = *reinterpret_cast<const float4*>(D3 + (r0 + u) * D3S + c);
      w[u] = D3[64 * D3S + r0 + u];
    }
    float4 mn, vr;
    pool_views<NV>(w, x, mn, vr);
    const long long sj = base + (long long)tile * FSPT + s;
    if (sj < end) {
      float* out = pool + (sj - base) * POOL_W + c;
      *reinterpret_cast<float4*>(out) = mn;
      *reinterpret_cast<float4*>(out + 64) = vr;
    }
  }
  tc::named_sync(bar_id, 128);   // the L3 rows are read: the next tile's input may overwrite them
}

// Softplus epilogue of a 128-wide stage into the next layer's A fragments (pipelined form): a[m] is the word front_epi_sp stores at
// row 16 wq + (lane >> 2) + 8 (m & 1), word column 4 (m >> 1) + (lane & 3), so a[4j .. 4j + 3] is k-block j (WgmmaRA).
__device__ __forceinline__ void front_sp_frag(const float* d, uint32_t* a) {
#pragma unroll
  for (int m = 0; m < 32; ++m) a[m] = sp_pair(__float_as_uint(d[2 * m]), __float_as_uint(d[2 * m + 1]));
}

// One register-A stage of the pipelined form: front_ra_issue starts it, front_ra_wait retires it.  The fences keep the fragment's
// definitions before the chain and the accumulators' reads after the wait (ptxas keeps the fragment's registers until the wait).
template <int N, int KCH>
__device__ __forceinline__ void front_ra_issue(float* d, uint32_t* a, uint32_t b) {
  tc::fence_regs<4 * KCH>(a);
  tc::fence_regs<N / 2>(d);
  tc::wg_fence();
  tc::wg_mma_ra<N, KCH>(d, a, b, (uint32_t)(N / 8) * 128u, 0u);
  tc::wg_commit();
}
template <int N>
__device__ __forceinline__ void front_ra_wait(float* d) {
  tc::wg_wait0();
  tc::fence_regs<N / 2>(d);
}

// feat8 words 64..67 of the layer-2 input as the first two registers of k-block 8's A fragment (rows 16 wq + (lane >> 2) and + 8,
// word 64 + (lane & 3)).  A warp's 16 fragment rows are the rows of its lanes 16 (wq & 1) .. + 15 (the row threads' mapping in
// geo_front_kernel): lane l gathers channels [4 (l >> 4), + 4) of fragment row l & 15 from that row thread's projection (the
// same taps and blend as gather_feat8 in the row thread), and the fragment lanes take their words by shuffles.
template <int NV>
__device__ __forceinline__ void gather_feat8_frag(const SceneS<NV>& S, const Proj& q, int wq, int lane, uint32_t f8[2]) {
  const int rl = 16 * (wq & 1) + (lane & 15);
  Proj qr;
  qr.u = __shfl_sync(FULL, q.u, rl);
  qr.v = __shfl_sync(FULL, q.v, rl);
  qr.zn = 0.0f;
  uint32_t w[2];
  gather_feat8(S, rl % NV, qr, lane >> 4, w);
  const int t = lane & 3, s0 = (lane >> 2) + 16 * (t >> 1);
  const uint32_t x0 = __shfl_sync(FULL, w[0], s0), x1 = __shfl_sync(FULL, w[1], s0);
  const uint32_t y0 = __shfl_sync(FULL, w[0], s0 + 8), y1 = __shfl_sync(FULL, w[1], s0 + 8);
  f8[0] = (t & 1) ? x1 : x0;
  f8[1] = (t & 1) ? y1 : y0;
}

// Latency options of a front instantiation's tile chain:
//   FO_F8_EARLY     the feat8 words are gathered at the start of the tile, beside the feat64 gather, and held until the layer-2
//                   input is built (otherwise they are gathered there, and the chain waits on a global load between L1 and L2);
//   FO_NEXT_ID      the next tile's work-list entry is loaded at the start of the tile, so the tile after it starts on one global
//                   load (the sample) instead of two dependent ones;
//   FO_NEXT_SAMPLE  (with FO_NEXT_ID) the next tile's sample is also fetched, after L3, so a tile starts on no global load;
//   FO_PIPE         two tiles in flight per warpgroup (the other bits do not apply): layers 1-3 take their A operand from
//                   registers, so the activation tile is free from the end of L0 until the L3 rows are staged, and the row threads
//                   build the next tile's layer-0 input there while the tensor cores run this tile's L1-L3.
// Each holds registers across the wgmma chain, and for some instantiations that makes ptxas serialise the chain's wgmma
// instructions (warnings C7511 / C7513 / C7520).  The table gives each instantiation the first of 8, 7, 3, 6, 1, 2, 0 with which ptxas
// (CUDA 12.9, -Xptxas -v) builds it without C7511, C7513, C7520 or spills; every front instantiation compiles without them.  One digit
// per pair count NP = 1 .. 16.
constexpr int FO_F8_EARLY = 1, FO_NEXT_ID = 2, FO_NEXT_SAMPLE = 4, FO_PIPE = 8;
__host__ __device__ constexpr int front_opts(int nv, int np, bool grid) {
  const char* t = nv <= 3 ? (grid ? "8888888387888887" : "8888888783888887") : (grid ? "8888888787888886" : "8888888787888887");
  return t[np - 1] - '0';
}

// One instantiation per view count NV and keypoint pair count NP (nk = 2 NP - 1 or 2 NP keypoints); GRID: for grid sources
// (kpn_query_grid), the others take rays and explicit points.
template <int NV, int NP, bool GRID>
__global__ void __launch_bounds__(front_wgs(2 * NP, NV) * 128, 1)
geo_front_kernel(const DevScene* __restrict__ scp, int nk, const uint8_t* __restrict__ wblob, SampleSrc src,
                 const int* __restrict__ list, const int* __restrict__ count_ptr, long long base, long long len,
                 float* __restrict__ pool) {
  extern __shared__ __align__(1024) uint8_t wsm[];
  __shared__ uint64_t wbar;
  __shared__ SceneS<NV> scs;
  constexpr int NK = 2 * NP, FWG = front_wgs(NK, NV), SPW = spw(NV), FSPT = fspt(NV);
  constexpr TcPlan plan = make_tc_plan(NK);
  constexpr uint32_t WBYTES = plan.st[4].off;        // W_hi of stages 0..3
  const long long end = min((long long)*count_ptr, base + len);
  if (end <= base) return;
  const int ntiles = (int)((end - base + FSPT - 1) / FSPT);
  const int t = threadIdx.x, wg = t >> 7, wq = (t >> 5) & 3, lane = t & 31;
  stage_scene(scs, *scp, nk, t, FWG * 128);
  if (t == 0) { tc::mbar_init(&wbar, 1); tc::fence_mbar_init(); }
  __syncthreads();
  if (t == 0) load_weights(wsm, wblob, WBYTES, &wbar);
  __syncthreads();
  uint8_t* A = wsm + WBYTES + (size_t)wg * front_tile_bytes(NK);
  float* D3 = reinterpret_cast<float*>(A);
  const uint32_t W = tc::smem_u32(wsm);
  const int bar_id = 1 + wg;
  // row warps 2 rh and 2 rh + 1 hold rows 32 rh .. 32 rh + 31 (lane = row) with column half h = 0 and 1, so that the 16 rows of a
  // warp's wgmma fragments (16 wq .. 16 wq + 15) are rows of its own lanes
  const int rh = wq >> 1, h = wq & 1;
  const int row = rh * 32 + lane;
  const int g = lane / NV, v = lane - NV * g;         // 3 views: lanes 30, 31 replay views 0, 1 of the warp's last sample (unused)
  const Group<NV> grp(lane);
  const int tile0 = blockIdx.x * FWG + wg, tstride = gridDim.x * FWG;
  const long long srow = rh * SPW + min(g, SPW - 1);   // this lane's sample within a tile
  constexpr int OPT = front_opts(NV, NP, GRID);
  if constexpr ((OPT & FO_PIPE) != 0) {
    // ---- two tiles in flight.  Per tile: L0 from the activation tile (then free); the previous tile's L3 rows staged there and
    //      pooled; L1 -> L2 -> L3 from registers, each issued before the row threads build a part of the next tile's layer-0 input
    //      in the free tile (sample | view weight and feat8 words | encodings and feat64) and retired after it.  The work-list
    //      entry of the tile after next is loaded beside L3, so the sample fetch beside L1 is one global load.  The tile's L3
    //      accumulators and view weight wait in registers across the next tile's L0.
    int tile = tile0;
    if (tile >= ntiles) return;
    float p[3];
    Proj q;
    float pw;
    uint32_t f8[2];
    {
      float dd[3];
      fetch_sample<GRID>(src, list[min(base + (long long)tile * FSPT + srow, end - 1)], p, dd);
      q = project_s(scs, v, p);
      const float bw = boundary_weight_fast(q);
      pw = bw / (grp.sum(bw) + 1e-6f);   // reference src/model.py:750-759 (mask == 1 for shaded samples)
      gather_feat8_frag(scs, q, wq, lane, f8);
      gather_feat64<NV, NP>(scs.f64, make_taps(q.u, q.v, scs.f64.W, scs.f64.H), A, rh * 32, h, lane);
      front_l0_encode<NV, NP>(scs, v, nk, p, A, row, h);
    }
    const uint32_t k8_bias = (lane & 3) == 0 ? H2_ONE : 0u;   // bias word at column 0 of a k-block's word group, K padding after
    float d[64];
    uint32_t a[36];
    front_mma<128, tc_k0p(NK) / 16>(d, A, W + plan.st[0].off, bar_id);
    front_sp_frag(d, a);
    float d3[32];
    int idn = list[min(base + (long long)(tile + tstride) * FSPT + srow, end - 1)];
    for (;;) {
      // the next tile's input is built whether or not there is one (past the end the work-list index is clamped), so that no
      // branch separates a wgmma chain from its wait
      const int next = tile + tstride;
      a[32] = k8_bias; a[33] = k8_bias; a[34] = 0u; a[35] = 0u;   // layer-1 input words 64..71: bias column, K padding
      front_ra_issue<128, 9>(d, a, W + plan.st[1].off);
      float pwn;
      uint32_t f8n[2];
      {
        float dd[3];
        fetch_sample<GRID>(src, idn, p, dd);
      }
      front_ra_wait<128>(d);
      front_sp_frag(d, a);
      a[32] = f8[0]; a[33] = f8[1]; a[34] = k8_bias; a[35] = k8_bias;   // layer-2 input words 64..71: feat8 | bias, K padding
      front_ra_issue<128, 9>(d, a, W + plan.st[2].off);
      {
        q = project_s(scs, v, p);
        const float bw = boundary_weight_fast(q);
        pwn = bw / (grp.sum(bw) + 1e-6f);
        gather_feat8_frag(scs, q, wq, lane, f8n);
      }
      front_ra_wait<128>(d);
      front_sp_frag(d, a);
      a[30] = k8_bias; a[31] = k8_bias;   // layer-3 input words 60..63: bias column, K padding
      front_ra_issue<64, 8>(d3, a, W + plan.st[3].off);
      front_l0_encode<NV, NP>(scs, v, nk, p, A, row, h);
      gather_feat64<NV, NP>(scs.f64, make_taps(q.u, q.v, scs.f64.W, scs.f64.H), A, rh * 32, h, lane);
      idn = list[min(base + (long long)(next + tstride) * FSPT + srow, end - 1)];
      front_ra_wait<64>(d3);
      if (next >= ntiles) break;
      front_mma<128, tc_k0p(NK) / 16>(d, A, W + plan.st[0].off, bar_id);
      front_sp_frag(d, a);
      front_pool<NV>(d3, pw, D3, wq, lane, row, h, base, end, tile, pool, bar_id);
      tile = next; pw = pwn; f8[0] = f8n[0]; f8[1] = f8n[1];
    }
    tc::named_sync(bar_id, 128);   // every thread's writes of the unused input are done before the L3 rows go over them
    front_pool<NV>(d3, pw, D3, wq, lane, row, h, base, end, tile, pool, bar_id);
  } else {
    constexpr bool F8_EARLY = (OPT & FO_F8_EARLY) != 0, NEXT_ID = (OPT & FO_NEXT_ID) != 0;
    constexpr bool NEXT_SAMPLE = NEXT_ID && (OPT & FO_NEXT_SAMPLE) != 0;
    // the tile ahead's work-list entry (and sample) are fetched while the current tile runs; past the end the fetch is clamped to
    // the last entry and not used
    int idn = 0;
    float pn[3] = {0.0f, 0.0f, 0.0f};
    if constexpr (NEXT_ID) {
      idn = list[min(base + (long long)tile0 * FSPT + srow, end - 1)];
      if constexpr (NEXT_SAMPLE) {
        float dd[3];
        fetch_sample<GRID>(src, idn, pn, dd);
      }
    }
    for (int tile = tile0; tile < ntiles; tile += tstride) {
      const long long si = base + (long long)tile * FSPT + srow;
      float p[3];
      if constexpr (NEXT_SAMPLE) {
        p[0] = pn[0]; p[1] = pn[1]; p[2] = pn[2];
      } else {
        float dd[3];
        fetch_sample<GRID>(src, NEXT_ID ? idn : list[min(si, end - 1)], p, dd);
      }
      if constexpr (NEXT_ID) idn = list[min(si + (long long)tstride * FSPT, end - 1)];
      const Proj q = project_s(scs, v, p);
      const float bw = boundary_weight_fast(q);
      const float pw = bw / (grp.sum(bw) + 1e-6f);   // reference src/model.py:750-759 (mask == 1 for shaded samples)
      uint32_t f8w[2];
      if constexpr (F8_EARLY) gather_feat8(scs, v, q, h, f8w);
      gather_feat64<NV, NP>(scs.f64, make_taps(q.u, q.v, scs.f64.W, scs.f64.H), A, rh * 32, h, lane);
      front_l0_encode<NV, NP>(scs, v, nk, p, A, row, h);
      // ---- L0 -> L1 -> L2 -> L3 (reference src/utils.py:691-720)
      float d[64];
      front_mma<128, tc_k0p(NK) / 16>(d, A, W + plan.st[0].off, bar_id);
      front_epi_sp(d, A, wq, lane, false);
      if (h == 0) {   // layer-1 input: bias chunk
        const uint32_t b[8] = {H2_ONE, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
        a_put<64, 8>(A, row, 64, b);
      }
      front_mma<128, 9>(d, A, W + plan.st[1].off, bar_id);
      front_epi_sp(d, A, wq, lane, false);
      {   // layer-2 input: feat8 (words 64 + 2h, 65 + 2h from this thread) | bias chunk (thread 1)
        if constexpr (!F8_EARLY) gather_feat8(scs, v, q, h, f8w);
        const uint32_t b[6] = {f8w[0], f8w[1], H2_ONE, 0u, 0u, 0u};
        if (h == 0) a_put_span<64, 2>(A, row, b);
        else a_put_span<66, 6>(A, row, b);
      }
      front_mma<128, 9>(d, A, W + plan.st[2].off, bar_id);
      front_epi_sp(d, A, wq, lane, true);
      front_mma<64, 8>(d, A, W + plan.st[3].off, bar_id);
      if constexpr (NEXT_SAMPLE) {   // the next tile's sample (its work-list entry was loaded above)
        float dd[3];
        fetch_sample<GRID>(src, idn, pn, dd);
      }
      front_pool<NV>(d, pw, D3, wq, lane, row, h, base, end, tile, pool, bar_id);
    }
  }
}


// =====================================================================================================================
// colour head.  Warpgroup tile = 128 rows (4 row warps x spw(NV) samples x NV views: 40 samples with 3 views, 32 with 4).  Each
// stage issues its two 64-row MMAs back to back and retires them with one wait.  BASE0 and VIS1A, whose epilogues are elementwise,
// write the next stage's activation tile straight from their fragments; the other stages stage their accumulators in shared
// memory (D) for the row threads, which do the cross-view work of the reference.  Two tiles are in flight per warpgroup: while a
// tile runs its stages, the row threads fetch the next tile's inputs (work-list entry beside RE1, sample and latent beside BASE0,
// projection and ray difference beside BASE1, img / feat_tex taps beside OUT0), so a tile starts on no global load.
// =====================================================================================================================
constexpr int CWG = 3;                                   // warpgroups per CTA (168 registers per thread)
constexpr int CDS = 68;                                  // row stride (floats) of the staged accumulators
constexpr uint32_t CA_BYTES = 128 * 112 * 2;             // activation tile (widest colour input: BASE0, K = 112)
constexpr uint32_t CD_BYTES = 128 * CDS * 4;

template <int NV>
struct ColCtx {
  uint8_t* A;
  float* D;
  uint32_t wbase;   // shared address of the colour stages' weights (plan offset of stage 6 at 0)
  int bar_id, row, wq, lane;
  Group<NV> grp;
};

// accumulator registers of a colour stage per thread: Np / 2 for each 64-row half
template <int STAGE>
__host__ __device__ constexpr int col_acc() { return REL_PLAN.st[STAGE].Np; }

// publish the activation tile and issue both halves of stage STAGE as one committed group; d: half 0's accumulators, then half 1's
template <int STAGE, int NV>
__device__ __forceinline__ void col_issue(const ColCtx<NV>& c, float* d) {
  constexpr TcPlan plan = REL_PLAN;
  constexpr int Kp = plan.st[STAGE].Kp, Np = plan.st[STAGE].Np;
  const uint32_t b = c.wbase + (plan.st[STAGE].off - plan.st[GEO_NSTAGE].off);
  wg_publish(c.bar_id);
  tc::wg_fence();
  tc::wg_mma<Np, Kp / 16>(d, tc::smem_u32(c.A), 2048u, b, (uint32_t)(Np / 8) * 128u, 0u);
  tc::wg_mma<Np, Kp / 16>(d + Np / 2, tc::smem_u32(c.A) + 1024u, 2048u, b, (uint32_t)(Np / 8) * 128u, 0u);
  tc::wg_commit();
}
// retire the stage: the fence keeps the accumulators' reads after the wait
template <int N>
__device__ __forceinline__ void col_retire(float* d) {
  tc::wg_wait0();
  tc::fence_regs<N>(d);
}
// stage the retired accumulators (N columns) in D for the row threads
template <int N, int NV>
__device__ __forceinline__ void col_stage(const ColCtx<NV>& c, const float* d) {
#pragma unroll
  for (int half = 0; half < 2; ++half) {
#pragma unroll
    for (int m = 0; m < N / 4; ++m) {
      const int r = 64 * half + 16 * c.wq + (c.lane >> 2) + 8 * (m & 1), col = 8 * (m >> 1) + 2 * (c.lane & 3);
      *reinterpret_cast<float2*>(c.D + r * CDS + col) = make_float2(d[half * N / 2 + 2 * m], d[half * N / 2 + 2 * m + 1]);
    }
  }
  tc::named_sync(c.bar_id, 128);   // accumulators staged, every MMA has read the activation tile
}
template <int N, int NV>
__device__ __forceinline__ void d_get(const ColCtx<NV>& c, int c0, float* x) {
#pragma unroll
  for (int i = 0; i < N; i += 4) {
    const float4 f = *reinterpret_cast<const float4*>(c.D + c.row * CDS + c0 + i);
    x[i] = f.x; x[i + 1] = f.y; x[i + 2] = f.z; x[i + 3] = f.w;
  }
}
// ELU(acc + bias) of the retired accumulators (N columns) as the next input's words [0, N / 2), written from the fragments: the word
// of columns 2w, 2w + 1 of a row is the pair the row thread packed from the staged row before
template <int N, int NV>
__device__ __forceinline__ void col_epi_elu(const ColCtx<NV>& c, const float* d, const float* __restrict__ bias) {
  tc::named_sync(c.bar_id, 128);   // every warp's MMAs have read the activation tile
#pragma unroll
  for (int half = 0; half < 2; ++half) {
#pragma unroll
    for (int m = 0; m < N / 4; ++m) {
      const int r = 64 * half + 16 * c.wq + (c.lane >> 2) + 8 * (m & 1), col = 8 * (m >> 1) + 2 * (c.lane & 3);
      const float x0 = d[half * N / 2 + 2 * m] + bias[col], x1 = d[half * N / 2 + 2 * m + 1] + bias[col + 1];
      *reinterpret_cast<uint32_t*>(c.A + tc::a_word_off<128>(r, col >> 1)) = tc::pack_h2(elu_fast(x0), elu_fast(x1));
    }
  }
}

// The four bilinear taps of NC4 float4 groups of one view (gather_f32's addresses), loaded now and blended later with gather_f32's
// expression, so that the loads are in flight while the tile before runs its last stage.
template <int NC4>
struct TapLoads {
  float4 x[4][NC4];
  float w00, w01, w10, w11;
  __device__ __forceinline__ void issue(const MapDesc& m, int v, float u, float vv) {
    const Taps t = make_taps(u, vv, m.W, m.H);
    const int c4 = m.C >> 2;
    const float4* base = (const float4*)m.ptr + (size_t)v * m.H * m.W * c4;
    const int o[4] = {t.o00, t.o01, t.o10, t.o11};
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
      for (int i = 0; i < NC4; ++i) x[k][i] = __ldg(base + (size_t)o[k] * c4 + i);
    w00 = t.w00; w01 = t.w01; w10 = t.w10; w11 = t.w11;
  }
  __device__ __forceinline__ void blend(float* out) const {
#pragma unroll
    for (int i = 0; i < NC4; ++i) {
      const float4 a = x[0][i], b = x[1][i], c = x[2][i], d = x[3][i];
      out[4 * i + 0] = a.x * w00 + b.x * w01 + c.x * w10 + d.x * w11;
      out[4 * i + 1] = a.y * w00 + b.y * w01 + c.y * w10 + d.y * w11;
      out[4 * i + 2] = a.z * w00 + b.z * w01 + c.z * w10 + d.z * w11;
      out[4 * i + 3] = a.w * w00 + b.w * w01 + c.w * w10 + d.w * w11;
    }
  }
};

// A colour tile's inputs that do not depend on the MLPs, per row (sample, view)
struct ColIn {
  int slot, id;          // work-list entry: index into the first work list (latent slot), sample id
  float rd[4];           // [unit(dir - dir_src), dir . dir_src], reference src/model.py:825-832
  float rgb[3], t8[8];   // img and feat_tex taps, blended
  uint32_t lat[12];      // compressed latent, fp16 pairs
};

// Work-list entry of tile sample si (x = index into the first work list, where the latent sits and, + list_base, where the colour
// goes; y = sample id).  Query mode shades every valid sample: the first list itself is the work list.  Past the end the index is
// clamped to the last entry (the row computes and writes nothing).
__device__ __forceinline__ int2 col_entry(const int2* __restrict__ list2, const int* __restrict__ list1, int count, int si) {
  const int e = min(si, count - 1);
  return list2 ? list2[e] : make_int2(e, list1[e]);
}
// the ray difference and the projection (u, vv) of sample p seen from view v
template <int NV>
__device__ __forceinline__ void col_ray(const SceneS<NV>& sc, int v, const float p[3], const float d[3], float rd[4], float& u,
                                        float& vv) {
  const Proj q = project_s(sc, v, p);
  u = q.u; vv = q.v;
  float r[3] = {p[0] - sc.C[v][0], p[1] - sc.C[v][1], p[2] - sc.C[v][2]};
  float n = fmaxf(sqrtf(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]), 1e-12f);
  r[0] /= n; r[1] /= n; r[2] /= n;
  float e[3] = {d[0] - r[0], d[1] - r[1], d[2] - r[2]};
  float en = fmaxf(sqrtf(e[0] * e[0] + e[1] * e[1] + e[2] * e[2]), 1e-6f);
  rd[0] = e[0] / en; rd[1] = e[1] / en; rd[2] = e[2] / en;
  rd[3] = r[0] * d[0] + r[1] * d[1] + r[2] * d[2];
}
__device__ __forceinline__ void col_lat_issue(const uint4* __restrict__ lat_in, int slot, uint4 w[3]) {
  w[0] = __ldg(lat_in + 3ll * slot + 0); w[1] = __ldg(lat_in + 3ll * slot + 1); w[2] = __ldg(lat_in + 3ll * slot + 2);
}
__device__ __forceinline__ void col_in_finish(const TapLoads<1>& li, const TapLoads<2>& lt, const uint4 w[3], ColIn& in) {
  float c4[4];
  li.blend(c4);
  in.rgb[0] = c4[0]; in.rgb[1] = c4[1]; in.rgb[2] = c4[2];
  lt.blend(in.t8);
  const uint32_t* wl = reinterpret_cast<const uint32_t*>(w);
#pragma unroll
  for (int i = 0; i < 12; ++i) in.lat[i] = wl[i];
}

// Colour pass of one tile (reference src/model.py:806-832, 1279-1301) from its prefetched inputs `in`; beside its stages the row
// threads fetch the inputs of tile sample sn of the next tile into `nx`.  The next tile's inputs are fetched whether or not there is
// one (col_entry clamps the index), so that no branch separates a wgmma chain from its wait.
template <int NV>
__device__ __forceinline__ void color_tile(const SceneS<NV>& sc, const TcConsts& C, const SampleSrc& src,
                                           const int2* __restrict__ list2, const int* __restrict__ list1, int count, int si,
                                           const ColIn& in, int sn, ColIn& nx, const ColCtx<NV>& cx,
                                           const uint4* __restrict__ lat_in, int query_mode, const ShadeOut& so) {
  constexpr int SPW = spw(NV);
  const int lane = cx.lane;
  const int g = lane / NV;
  const int v = lane - NV * g;
  const bool writer = (lane < NV * SPW) && (v == 0) && (si < count);
  float f[35];
  f[0] = in.rgb[0]; f[1] = in.rgb[1]; f[2] = in.rgb[2];
#pragma unroll
  for (int i = 0; i < 8; ++i) f[3 + i] = in.t8[i];
#pragma unroll
  for (int i = 0; i < 12; ++i) {
    const float2 t2 = __half22float2(*reinterpret_cast<const __half2*>(&in.lat[i]));
    f[11 + 2 * i] = t2.x; f[12 + 2 * i] = t2.y;
  }
  int2 en;
  {  // ray-direction encoder 4->16->35, ELU, added onto the features (src/model.py:1279-1284): first layer in fp32 on the CUDA
     // cores, second layer (stage 12, bias as K row 16) on the tensor core
    uint32_t a[16];
#pragma unroll
    for (int o = 0; o < 16; o += 2) {
      float acc0 = C.b_re0[o], acc1 = C.b_re0[o + 1];
#pragma unroll
      for (int i = 0; i < 4; ++i) { acc0 = fmaf(C.w_re0[o][i], in.rd[i], acc0); acc1 = fmaf(C.w_re0[o + 1][i], in.rd[i], acc1); }
      a[o / 2] = tc::pack_h2(elu_fast(acc0), elu_fast(acc1));
    }
    a[8] = H2_ONE;   // bias column
#pragma unroll
    for (int i = 9; i < 16; ++i) a[i] = 0u;
    a_put<128, 16>(cx.A, cx.row, 0, a);
    float d[col_acc<12>()];
    col_issue<12>(cx, d);
    en = col_entry(list2, list1, count, sn);
    col_retire<col_acc<12>()>(d);
    col_stage<col_acc<12>()>(cx, d);
    float r[36];
    d_get<36>(cx, 0, r);
#pragma unroll
    for (int o = 0; o < 35; ++o) f[o] += elu_fast(r[o]);
  }
  float om;  // blending weight (src/model.py:1286-1289), mask == 1
  {
    float ex = ex2f(C.ani_abs * LOG2E * (in.rd[3] - 1.0f));
    float e = ex - cx.grp.vmin(ex);
    om = e / (cx.grp.sum(e) + 1e-8f);
  }
  {  // BASE0 input [mean35 | var35 | f35 | 0-pad] (src/model.py:1291-1292)
    float mean[35], var[35];
#pragma unroll
    for (int c = 0; c < 35; ++c) {
      mean[c] = cx.grp.sum(om * f[c]);
      float dl = f[c] - mean[c];
      var[c] = cx.grp.sum(om * dl * dl);
    }
    uint32_t a[56];
#pragma unroll
    for (int j = 0; j < 56; ++j) {
      const int e0 = 2 * j, e1 = 2 * j + 1;
      float x0 = e0 < 35 ? mean[e0 < 35 ? e0 : 0] : e0 < 70 ? var[e0 < 70 ? (e0 >= 35 ? e0 - 35 : 0) : 0]
                 : e0 < 105 ? f[e0 >= 70 ? (e0 < 105 ? e0 - 70 : 0) : 0] : 0.0f;
      float x1 = e1 < 35 ? mean[e1 < 35 ? e1 : 0] : e1 < 70 ? var[e1 < 70 ? (e1 >= 35 ? e1 - 35 : 0) : 0]
                 : e1 < 105 ? f[e1 >= 70 ? (e1 < 105 ? e1 - 70 : 0) : 0] : 0.0f;
      a[j] = tc::pack_h2(x0, x1);
    }
    a_put<128, 56>(cx.A, cx.row, 0, a);
  }
  // ---- BASE0 -> BASE1
  float pn[3], dn[3];
  uint4 lw[3];
  {
    float d[col_acc<6>()];
    col_issue<6>(cx, d);
    fetch_sample(src, en.y, pn, dn);
    col_lat_issue(lat_in, en.x, lw);
    col_retire<col_acc<6>()>(d);
    col_epi_elu<col_acc<6>()>(cx, d, C.b_base0);
  }
  float un, vn;
  float x[32];
  {
    float d[col_acc<7>()];
    col_issue<7>(cx, d);
    col_ray(sc, v, pn, dn, nx.rd, un, vn);
    col_retire<col_acc<7>()>(d);
    col_stage<col_acc<7>()>(cx, d);
    float r[32];
    d_get<32>(cx, 0, r);
    uint32_t o[16];
#pragma unroll
    for (int i = 0; i < 32; ++i) x[i] = elu_fast(r[i] + C.b_base1[i]);
#pragma unroll
    for (int i = 0; i < 16; ++i) o[i] = tc::pack_h2(x[2 * i] * om, x[2 * i + 1] * om);  // vis_layer1(x * weight)
    a_put<128, 16>(cx.A, cx.row, 0, o);
  }
  // ---- VIS1A -> VIS1B (src/model.py:1294-1296)
  {
    float d[col_acc<8>()];
    col_issue<8>(cx, d);
    col_retire<col_acc<8>()>(d);
    col_epi_elu<col_acc<8>()>(cx, d, C.b_vis1a);
  }
  {
    float d[col_acc<9>()];
    col_issue<9>(cx, d);
    col_retire<col_acc<9>()>(d);
    col_stage<col_acc<9>()>(cx, d);
    float r[36];
    d_get<36>(cx, 0, r);
    float sg = sig_fast(elu_fast(r[32] + C.b_vis1b[32]));
    uint32_t o[16];
#pragma unroll
    for (int i = 0; i < 32; ++i) x[i] += elu_fast(r[i] + C.b_vis1b[i]);
#pragma unroll
    for (int i = 0; i < 16; ++i) o[i] = tc::pack_h2(x[2 * i] * sg, x[2 * i + 1] * sg);  // x * sigmoid(vis) * mask
    a_put<128, 16>(cx.A, cx.row, 0, o);
  }
  // ---- VIS2A (+ 32->1 sigmoid on CUDA cores) -> OUT0 input [x32 | vis | ray_diff4 | 0-pad] (src/model.py:1297-1300)
  {
    float d[col_acc<10>()];
    col_issue<10>(cx, d);
    col_retire<col_acc<10>()>(d);
    col_stage<col_acc<10>()>(cx, d);
    float r[32];
    d_get<32>(cx, 0, r);
    float dot = C.b_vis2b;
#pragma unroll
    for (int i = 0; i < 32; ++i) dot = fmaf(C.w_vis2b[i], elu_fast(r[i] + C.b_vis2a[i]), dot);
    float vis2 = sig_fast(dot);
    uint32_t o[24];
#pragma unroll
    for (int i = 0; i < 16; ++i) o[i] = tc::pack_h2(x[2 * i], x[2 * i + 1]);
    o[16] = tc::pack_h2(vis2, in.rd[0]);
    o[17] = tc::pack_h2(in.rd[1], in.rd[2]);
    o[18] = tc::pack_h2(in.rd[3], 0.0f);
#pragma unroll
    for (int i = 19; i < 24; ++i) o[i] = 0u;
    a_put<128, 24>(cx.A, cx.row, 0, o);
  }
  // ---- OUT0 -> 16->8->1 on CUDA cores -> softmax over the views -> blended colour (src/model.py:1300-1301)
  TapLoads<1> li;
  TapLoads<2> lt;
  float logit;
  {
    float d[col_acc<11>()];
    col_issue<11>(cx, d);
    li.issue(sc.img, v, un, vn);
    lt.issue(sc.ftex, v, un, vn);
    col_retire<col_acc<11>()>(d);
    col_stage<col_acc<11>()>(cx, d);
    float r[16];
    d_get<16>(cx, 0, r);
    float h16[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) h16[i] = elu_fast(r[i] + C.b_out0[i]);
    logit = C.b_out2;
#pragma unroll
    for (int o = 0; o < 8; ++o) {
      float acc = C.b_out1[o];
#pragma unroll
      for (int i = 0; i < 16; ++i) acc = fmaf(C.w_out1[o][i], h16[i], acc);
      logit = fmaf(C.w_out2[o], elu_fast(acc), logit);
    }
  }
  {
    float e = ex2f((logit - cx.grp.vmax(logit)) * LOG2E);
    float inv = 1.0f / cx.grp.sum(e);
    float r0 = cx.grp.sum(e * in.rgb[0]) * inv, r1 = cx.grp.sum(e * in.rgb[1]) * inv, r2 = cx.grp.sum(e * in.rgb[2]) * inv;
    if (writer) {
      float* o = query_mode ? so.out5 + 5ll * in.id + 2 : so.rgb + 3ll * (so.list_base + in.slot);
      o[0] = r0; o[1] = r1; o[2] = r2;
    }
  }
  nx.slot = en.x; nx.id = en.y;
  col_in_finish(li, lt, lw, nx);
}

// wcol: the blob's tile of stage 6 (the colour stages' tiles follow it)
template <int NV>
__global__ void __launch_bounds__(CWG * 128, 1)
shade_color_kernel(const DevScene* __restrict__ scp, const __grid_constant__ TcConsts C, const uint8_t* __restrict__ wcol,
                   SampleSrc src, const int2* __restrict__ list2, const int* __restrict__ list1,
                   const int* __restrict__ count_ptr, const uint4* __restrict__ lat_in, int query_mode, ShadeOut so) {
  extern __shared__ __align__(1024) uint8_t wsm[];
  __shared__ uint64_t wbar;
  __shared__ SceneS<NV> scs;
  constexpr TcPlan plan = REL_PLAN;
  constexpr int SPW = spw(NV), SPT = spt(NV);
  constexpr uint32_t WBYTES = plan.total_bytes - plan.st[GEO_NSTAGE].off;
  constexpr uint32_t WPAD = (WBYTES + 1023u) / 1024u * 1024u;
  const int t = threadIdx.x, wg = t >> 7;
  const int count = *count_ptr;
  const int ntiles = (count + SPT - 1) / SPT;
  if (blockIdx.x * CWG >= ntiles) return;
  stage_scene(scs, *scp, 0, t, CWG * 128);   // the colour head reads no keypoints
  if (t == 0) { tc::mbar_init(&wbar, 1); tc::fence_mbar_init(); }
  __syncthreads();
  if (t == 0) load_weights(wsm, wcol, WBYTES, &wbar);   // the colour stages' weight tiles, once per CTA
  __syncthreads();
  const int lane = t & 31;
  ColCtx<NV> cx{wsm + WPAD + (size_t)wg * (CA_BYTES + CD_BYTES), nullptr, tc::smem_u32(wsm), 1 + wg, t & 127, (t >> 5) & 3, lane,
                Group<NV>(lane)};
  cx.D = reinterpret_cast<float*>(cx.A + CA_BYTES);
  const int g = lane / NV, v = lane - NV * g;
  const int srow = cx.wq * SPW + min(g, SPW - 1);   // this lane's sample within a tile
  const int tstride = gridDim.x * CWG;
  int tile = blockIdx.x * CWG + wg;
  if (tile >= ntiles) return;
  ColIn in;
  {  // the first tile's inputs
    const int2 e = col_entry(list2, list1, count, tile * SPT + srow);
    in.slot = e.x; in.id = e.y;
    float p[3], d[3], u, vv;
    fetch_sample(src, e.y, p, d);
    col_ray(scs, v, p, d, in.rd, u, vv);
    TapLoads<1> li;
    TapLoads<2> lt;
    uint4 lw[3];
    col_lat_issue(lat_in, e.x, lw);
    li.issue(scs.img, v, u, vv);
    lt.issue(scs.ftex, v, u, vv);
    col_in_finish(li, lt, lw, in);
  }
  for (;;) {
    const int next = tile + tstride;
    ColIn nx;
    color_tile(scs, C, src, list2, list1, count, tile * SPT + srow, in, next * SPT + srow, nx, cx, lat_in, query_mode, so);
    if (next >= ntiles) break;
    tile = next;
    in = nx;
  }
}

}  // namespace

// kernels every view count shares (kpn_shade_tc.cu): the density tail of the samples [base, base + len) of the work list, and
// the colour work list of a render
cudaError_t launch_geo_tail(const TcConsts& C, const uint8_t* wtail, const uint8_t* wlo, int lo_mask, const int* list,
                            const int* counter, long long base, long long len, const float* pool, int query_mode, const ShadeOut& so,
                            uint4* lat, int num_sms, cudaStream_t st);
cudaError_t launch_colour_list(const int* list, const int* counter, const float2* ao, int list_base, int2* list2, int* count2,
                               long long n_max, int num_sms, cudaStream_t st);

namespace {

constexpr uint32_t COL_SMEM = (REL_PLAN.total_bytes - REL_PLAN.st[GEO_NSTAGE].off + 1023) / 1024 * 1024 + CWG * (CA_BYTES + CD_BYTES);
static_assert(COL_SMEM + sizeof(SceneS<4>) + sizeof(uint64_t) <= SMEM_OPTIN, "colour CTA with the 4-view scene block");

inline int tc_grid(long long tiles, int per_cta, int num_sms) {
  const long long g = (tiles + per_cta - 1) / per_cta;
  return (int)(g < 1 ? 1 : (g > num_sms ? num_sms : g));
}

template <int NV, int NP>
cudaError_t launch_tc_impl(const ShadeBatch& b) {
  constexpr int NK = 2 * NP, FWG = front_wgs(NK, NV), FSPT = fspt(NV), SPT = spt(NV);
  constexpr TcPlan plan = make_tc_plan(NK);
  const size_t smem_front = front_smem_bytes(NK, FWG);
  static std::atomic<bool> attr[64];   // function attributes are per device (zero-initialised; setting them twice is harmless)
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !attr[dev].load(std::memory_order_acquire)) {
    cudaError_t e = cudaFuncSetAttribute(geo_front_kernel<NV, NP, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_front);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(geo_front_kernel<NV, NP, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_front);
    if (e != cudaSuccess) return e;
    e = cudaFuncSetAttribute(shade_color_kernel<NV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)COL_SMEM);
    if (e != cudaSuccess) return e;
    if (dev >= 0 && dev < 64) attr[dev].store(true, std::memory_order_release);
  }
  const uint8_t* wtail = b.wblob + plan.st[4].off;
  const uint8_t* wcol = b.wblob + plan.st[GEO_NSTAGE].off;
  cudaError_t e = cudaSuccess;
  // the device-side count is not known here: every slice of [0, n_max) is launched, slices past the count exit at once
  const long long nslices = b.n_max > POOL_SLICE ? (b.n_max + POOL_SLICE - 1) / POOL_SLICE : 1;
  for (long long s = 0; s < nslices; ++s) {
    const long long base = s * POOL_SLICE, len = b.n_max - base < POOL_SLICE ? b.n_max - base : POOL_SLICE;
    auto front = b.src.mode == 2 ? geo_front_kernel<NV, NP, true> : geo_front_kernel<NV, NP, false>;
    front<<<tc_grid((len + FSPT - 1) / FSPT, FWG, b.num_sms), FWG * 128, smem_front, b.st>>>(b.sc, b.n_kpt, b.wblob, b.src, b.list,
                                                                                             b.counter, base, len, b.pool);
    e = launch_geo_tail(*b.tcc, wtail, b.wlo, b.lo_mask, b.list, b.counter, base, len, b.pool, b.query_mode, b.so, b.lat, b.num_sms,
                        b.st);
    if (e != cudaSuccess) return e;
    *b.launches += 2;
  }
  if (b.after_geo) { e = cudaEventRecord(b.after_geo, b.st); if (e != cudaSuccess) return e; }
  if (b.query_mode == 2) return cudaSuccess;   // geometry only: no colour work list, no colour kernel
  const int grid = tc_grid((b.n_max + SPT - 1) / SPT, CWG, b.num_sms);
  if (b.query_mode) {   // every valid sample gets a colour: the first list is the colour work list
    shade_color_kernel<NV><<<grid, CWG * 128, COL_SMEM, b.st>>>(b.sc, *b.tcc, wcol, b.src, nullptr, b.list, b.counter, b.lat,
                                                                b.query_mode, b.so);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    *b.launches += 1;
    // statistics: every valid sample was coloured
    return cudaMemcpyAsync(b.count2, b.counter, sizeof(int), cudaMemcpyDeviceToDevice, b.st);
  }
  e = launch_colour_list(b.list, b.counter, b.so.ao, b.so.list_base, b.list2, b.count2, b.n_max, b.num_sms, b.st);
  if (e != cudaSuccess) return e;
  shade_color_kernel<NV><<<grid, CWG * 128, COL_SMEM, b.st>>>(b.sc, *b.tcc, wcol, b.src, b.list2, nullptr, b.count2, b.lat,
                                                              b.query_mode, b.so);
  *b.launches += 2;
  return cudaGetLastError();
}

using LaunchTc = decltype(&launch_tc_impl<3, 1>);
template <int NV, int... I>
constexpr std::array<LaunchTc, sizeof...(I)> launch_table(std::integer_sequence<int, I...>) {
  return {&launch_tc_impl<NV, I + 1>...};
}

// The tensor-core engine for NV source views: launch_tc_impl<NV, NP> for NP = 1 .. KPN_MAX_KPT / 2 keypoint pairs.
template <int NV>
cudaError_t launch_tc_views(const ShadeBatch& b) {
  static constexpr std::array<LaunchTc, KPN_MAX_KPT / 2> table =
      launch_table<NV>(std::make_integer_sequence<int, KPN_MAX_KPT / 2>{});
  if (b.n_kpt < 1 || b.n_kpt > KPN_MAX_KPT) return cudaErrorInvalidValue;
  return table[tc_npair(b.n_kpt) - 1](b);
}

}  // namespace

}  // namespace kpn
