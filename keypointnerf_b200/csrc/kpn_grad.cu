// Backward of the fp32 engine's render pass (reference src/model.py:978-1096, 1150-1176, eval branch, uniform=True, differentiated
// with torch autograd's semantics): the gradient of a loss of one pass' per-ray outputs with respect to every hot-path layer,
// mlp_tex.ani_al and the three gathered feature maps.
//
//   composite_backward   one warp per ray, on composite_kernel's list_entry / composite_weight (kpn_device.cuh): dL/d(colour,
//                        alpha, depth, sdf) of the ray -> per list position d rad, d sdf_raw, d rgb
//   shade_simt_backward  tiles of GTS valid samples: recomputes shade_simt_kernel's forward by calling its phases (kpn_simt.cuh),
//                        then backpropagates colour head -> density head -> view pooling -> per-view geometry MLP (each view's
//                        activations rebuilt in turn); dW / db into the CTA's own slice, feature-map taps scattered with atomics
//   grad_reduce          the CTA slices summed in CTA order (deterministic)
//   canonical_list       the front kernel's work list rewritten in ray order, so that the tiles above (and with them the
//                        summation order of dW, db and d ani_al) depend on the rays alone
#include <cub/device/device_scan.cuh>

#include "kpn_launch.h"
#include "kpn_simt.cuh"

namespace kpn {

// ------------------------------------------------------------------------------------------------
// compositing backward
// ------------------------------------------------------------------------------------------------
// Forward (composite_kernel): a_k = 1 - exp(-sigma_k dist_k), T_k = prod_{j<k} (1 - a_j), c_k = a_k T_k; acc = sum c_k,
// colour = sum c_k rgb_k, depth = sum c_k z_k / (acc + 1e-8), sdf = sum c_k s_k / (acc + 1e-8).  With g_k = dL/dc_k,
// dL/da_k = T_k (g_k - U_k), U_k = sum_{m>k} g_m a_m prod_{k<j<m} (1 - a_j), i.e. U_{k-1} = g_k a_k + (1 - a_k) U_k: a suffix scan
// of affine maps, carried from one group of 32 entries to the one before it.  Nothing is divided by 1 - a_k (exactly 0 on a
// ray's last sample, whose dist is 1e10).
__global__ void __launch_bounds__(128)
composite_backward_kernel(const int* __restrict__ list, const float2* __restrict__ ao, const float* __restrict__ rgb,
                          const int* __restrict__ start_, const int* __restrict__ cnt_, const float* __restrict__ zbuf,
                          const float* __restrict__ ray_nf, int r0, int nr, int S, long long plane, RayGrad gin,
                          float2* __restrict__ d_ao, float* __restrict__ d_rgb, float2* __restrict__ at) {
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  const unsigned FULL = 0xffffffffu;
  for (int i = blockIdx.x * wpb + (threadIdx.x >> 5); i < nr; i += gridDim.x * wpb) {
    const long long r = r0 + i;
    const float gC0 = gin.color ? gin.color[r] : 0.0f, gC1 = gin.color ? gin.color[plane + r] : 0.0f,
                gC2 = gin.color ? gin.color[2 * plane + r] : 0.0f;
    const float gA = gin.alpha ? gin.alpha[r] : 0.0f, gD = gin.depth ? gin.depth[r] : 0.0f, gS = gin.sdf ? gin.sdf[r] : 0.0f;
    const float* zz = zbuf ? zbuf + (long long)i * S : nullptr;
    const float n_r = zbuf ? 0.0f : ray_nf[2 * i], f_r = zbuf ? 0.0f : ray_nf[2 * i + 1];
    const int start = start_[i], cnt = cnt_[i];
    // ---- sweep 1 (composite_kernel's arithmetic): the ray's sums; a_k and T_k of every entry go to `at`
    float Tc = 1.0f, acc = 0.0f, cd = 0.0f, cs = 0.0f;
    for (int e0 = 0; e0 < cnt; e0 += 32) {
      const int e = start + e0 + lane;
      const bool live = e0 + lane < cnt;
      float a = 0.0f, zk = 0.0f, q1 = 0.0f;
      if (live) {
        const int k = list[e] - i * S;
        const float2 as = ao[e];
        const ListEntry en = list_entry(zz, n_r, f_r, k, S, as.x);
        zk = en.z; a = en.alpha;
        q1 = as.y;
      }
      float T;
      const float c = composite_weight(a, lane, Tc, T);
      if (live) { acc += c; cd += c * zk; cs += c * q1; at[e] = make_float2(a, T); }
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      acc += __shfl_xor_sync(FULL, acc, d); cd += __shfl_xor_sync(FULL, cd, d); cs += __shfl_xor_sync(FULL, cs, d);
    }
    const float inv = 1.0f / (acc + 1e-8f);
    const float gDn = gD * inv, gSn = gS * inv;
    const float gAe = gA - gDn * (cd * inv) - gSn * (cs * inv);   // alpha's own gradient + the normalisation of depth and sdf
    __syncwarp();
    // ---- sweep 2, last group first
    float carry = 0.0f;   // U of the last entry of the current group
    for (int e0 = (cnt - 1) & ~31; e0 >= 0; e0 -= 32) {
      const int e = start + e0 + lane;
      const bool live = e0 + lane < cnt;
      float b = 0.0f, m = 1.0f, gc = 0.0f, a = 0.0f, T = 0.0f, zk = 0.0f, dist = 0.0f, q2 = 0.0f, q3 = 0.0f, q4 = 0.0f;
      float2 as = make_float2(0.0f, 0.0f);
      if (live) {
        const int k = list[e] - i * S;
        as = ao[e];
        const ListEntry en = list_entry(zz, n_r, f_r, k, S, as.x);   // a_k and T_k as sweep 1 stored them, below
        zk = en.z; dist = en.dist;
        const float2 aT = at[e];
        a = aT.x; T = aT.y;
        if (as.x > 0.0f) { q2 = rgb[3ll * e]; q3 = rgb[3ll * e + 1]; q4 = rgb[3ll * e + 2]; }
        gc = gAe + gC0 * q2 + gC1 * q3 + gC2 * q4 + gDn * zk + gSn * as.y;
        b = gc * a; m = 1.0f - a;
      }
      float B = b, M = m;   // inclusive suffix composition f_lane o ... o f_31 as U -> B + M U
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const float Bn = __shfl_down_sync(FULL, B, d), Mn = __shfl_down_sync(FULL, M, d);
        if (lane + d < 32) { B = fmaf(M, Bn, B); M *= Mn; }
      }
      const float Bx = __shfl_down_sync(FULL, B, 1), Mx = __shfl_down_sync(FULL, M, 1);
      const float U = lane == 31 ? carry : fmaf(Mx, carry, Bx);
      carry = fmaf(__shfl_sync(FULL, M, 0), carry, __shfl_sync(FULL, B, 0));
      if (live) {
        const float c = a * T;
        const float da = T * (gc - U);
        const float dsig = da * dist * expf(-as.x * dist);
        const bool on = as.x > 0.0f;   // alpha = relu(rad): no gradient where rad <= 0
        d_ao[e] = make_float2(on ? dsig : 0.0f, gSn * c);
        d_rgb[3ll * e + 0] = on ? gC0 * c : 0.0f;
        d_rgb[3ll * e + 1] = on ? gC1 * c : 0.0f;
        d_rgb[3ll * e + 2] = on ? gC2 * c : 0.0f;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// shading backward (fp32 SIMT)
// ------------------------------------------------------------------------------------------------
constexpr int GTS = 32;         // samples per tile: 4 warps x 8 rows (dense_tile's row mapping)
constexpr int GNT = 4 * GTS;

// Shared memory of one tile, offsets in floats (every array starts on a 16-byte boundary).  The persistent arrays live for the
// whole tile; the geometry, density and colour phases share the region at U.
template <int NV>
struct GradSmem {
  static constexpr int r4(int x) { return (x + 3) & ~3; }
  static constexpr int Pd = 0;                         // [TS][8] p xyz, d xyz
  static constexpr int UV = Pd + GTS * 8;              // [NV][TS][4] u, v, zn, boundary weight
  static constexpr int PW = UV + NV * GTS * 4;         // [NV][TS]
  static constexpr int Y = r4(PW + NV * GTS);          // [NV][TS][64] geometry MLP outputs, later their gradients
  static constexpr int Pool = Y + NV * GTS * 64;       // [TS][128] mean || var
  static constexpr int dPool = Pool + GTS * 128;
  static constexpr int Lat = dPool + GTS * 128;        // [TS][24]
  static constexpr int dLat = Lat + GTS * 24;
  static constexpr int G = dLat + GTS * 24;            // [TS][8] d sdf_raw, d rad, d rgb[3]
  static constexpr int Misc = G + GTS * 8;             // [4] d |ani_al|
  static constexpr int Id = Misc + 4;                  // int [TS]
  static constexpr int U = r4(Id + GTS);
  // geometry phase
  static constexpr int X0 = U;                         // [TS][LDA] layer-0 input (encoding || feat64)
  static constexpr int H1 = X0 + GTS * LDA;            // [TS][128]
  static constexpr int X2 = H1 + GTS * 128;            // [TS][136] layer-1 output || feat8
  static constexpr int H3 = X2 + GTS * 136;            // [TS][120]
  static constexpr int GA = H3 + GTS * 120;            // [TS][136]
  static constexpr int GB = GA + GTS * 136;            // [TS][136]
  static constexpr int geo_end = GB + GTS * 136;
  // density phase
  static constexpr int D1 = U, D2 = U + GTS * 64, gA = D2 + GTS * 64, gB = gA + GTS * 64;
  // colour phase
  static constexpr int F = U;                          // [NV][TS][36] rgb || tex || latent, + ray encoding
  static constexpr int dF = F + NV * GTS * 36;
  static constexpr int MV = dF + NV * GTS * 36;        // [TS][72]
  static constexpr int dMV = MV + GTS * 72;
  static constexpr int RD = dMV + GTS * 72;            // [NV][TS][4]
  static constexpr int RGB = RD + NV * GTS * 4;        // [NV][TS][4]
  static constexpr int Om = RGB + NV * GTS * 4;        // [NV][TS]
  static constexpr int dOm = Om + NV * GTS;
  static constexpr int Logit = dOm + NV * GTS;
  static constexpr int dLogit = Logit + NV * GTS;
  static constexpr int Xv = r4(dLogit + NV * GTS);     // [TS][108] base_layer input (mean || var || f)
  static constexpr int Hb1 = Xv + GTS * 108;           // [TS][64]
  static constexpr int Hx = Hb1 + GTS * 64;            // [TS][32] base_layer output x
  static constexpr int Hs2 = Hx + GTS * 32;            // x * w
  static constexpr int Ht1 = Hs2 + GTS * 32;
  static constexpr int Hpv = Ht1 + GTS * 32;           // [TS][36] vis_layer1 output (res || vis)
  static constexpr int Hxx = Hpv + GTS * 36;           // x + res
  static constexpr int Hs3 = Hxx + GTS * 32;           // (x + res) * sigmoid(vis)
  static constexpr int Hu1 = Hs3 + GTS * 32;
  static constexpr int Hv2 = Hu1 + GTS * 32;           // [TS]
  static constexpr int Hoin = r4(Hv2 + GTS);           // [TS][40] out_layer input (x + res || vis2 || ray diff)
  static constexpr int Ho1 = Hoin + GTS * 40;          // [TS][16]
  static constexpr int Ho2 = Ho1 + GTS * 16;           // [TS][8]
  static constexpr int GA2 = Ho2 + GTS * 8;            // [TS][108]
  static constexpr int GB2 = GA2 + GTS * 108;          // [TS][108]
  static constexpr int GC = GB2 + GTS * 108;           // [TS][40]
  static constexpr int col_end = GC + GTS * 40;
  static constexpr int total = geo_end > col_end ? geo_end : col_end;
};
template <int NV>
constexpr size_t GRAD_SMEM_BYTES = (size_t)GradSmem<NV>::total * sizeof(float);
static_assert(GRAD_SMEM_BYTES<4> <= 227u * 1024u, "the backward tile of 4 views fits in shared memory");

// derivatives from the activations' outputs
__device__ __forceinline__ float dsoftplus100(float y) { return -expm1f(-100.0f * y); }   // sigmoid(100 x) = 1 - exp(-100 y)
__device__ __forceinline__ float delu(float y) { return y > 0.0f ? 1.0f : y + 1.0f; }

// dX[r][k] (+)= sum_n dY[r][n] W[n][k0 + k] for k < Kc, W row-major (n_out, n_in) = (N, K).  Warp w owns rows 8w..8w+7.
template <int NJ, bool ADD = false>
__device__ __forceinline__ void dense_bwd_x(const float* __restrict__ w, int N, int K, int k0, int Kc, const float* dY, int ldy,
                                            float* dX, int ldx) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float acc[8][NJ];
#pragma unroll
  for (int r = 0; r < 8; ++r)
#pragma unroll
    for (int j = 0; j < NJ; ++j) acc[r][j] = 0.0f;
  const float* y0 = dY + warp * 8 * ldy;
  for (int n = 0; n < N; ++n) {
    float wv[NJ];
#pragma unroll
    for (int j = 0; j < NJ; ++j) wv[j] = lane + 32 * j < Kc ? __ldg(w + (size_t)n * K + k0 + lane + 32 * j) : 0.0f;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const float dy = y0[r * ldy + n];
#pragma unroll
      for (int j = 0; j < NJ; ++j) acc[r][j] = fmaf(dy, wv[j], acc[r][j]);
    }
  }
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int k = lane + 32 * j;
    if (k < Kc) {
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        float* o = dX + (warp * 8 + r) * ldx + k;
        *o = ADD ? *o + acc[r][j] : acc[r][j];
      }
    }
  }
}

// dW[n][k] += sum_r dY[r][n] X[r][k], db[n] += sum_r dY[r][n] over the tile's rows, into this CTA's slice.
__device__ __forceinline__ void accum_dw(float* __restrict__ slice, const GradLayout& lay, const DevWeightsF32& W, int L,
                                         const float* dY, int ldy, const float* X, int ldx) {
  const int N = W.N[L], K = W.K[L];
  float* dw = slice + lay.wo[L];
  for (int idx = threadIdx.x; idx < N * K; idx += GNT) {
    const int n = idx / K, k = idx - n * K;
    float s = 0.0f;
#pragma unroll 8
    for (int r = 0; r < GTS; ++r) s = fmaf(dY[r * ldy + n], X[r * ldx + k], s);
    dw[idx] += s;
  }
  float* db = slice + lay.bo[L];
  for (int n = threadIdx.x; n < N; n += GNT) {
    float s = 0.0f;
    for (int r = 0; r < GTS; ++r) s += dY[r * ldy + n];
    db[n] += s;
  }
}

// g[r][c] *= act'(y[r][c]) for c < C
template <int ACT>
__device__ __forceinline__ void act_bwd(float* g, int ldg, const float* y, int ldy, int C) {
  for (int idx = threadIdx.x; idx < GTS * C; idx += GNT) {
    const int r = idx / C, c = idx - r * C;
    const float v = y[r * ldy + c];
    g[r * ldg + c] *= ACT == ACT_SP ? dsoftplus100(v) : delu(v);
  }
}

// Bilinear taps of (u, v) on a [V][H][W][C] gradient map: g (C floats, C % 4 == 0, channel group c4 of 4) scattered with the
// weights grid_sample's backward uses (border padding, align_corners=True: make_taps' clamping).
__device__ __forceinline__ void scatter4(float* map, const MapDesc& m, int C, int v, float u, float vv, int c4, float4 g) {
  const Taps t = make_taps(u, vv, m.W, m.H);
  float4* base = reinterpret_cast<float4*>(map + (size_t)v * m.H * m.W * C) + c4;
  const int c4n = C >> 2;
  const int o[4] = {t.o00, t.o01, t.o10, t.o11};
  const float w[4] = {t.w00, t.w01, t.w10, t.w11};
#pragma unroll
  for (int q = 0; q < 4; ++q)
    if (w[q] != 0.0f) atomicAdd(base + (size_t)o[q] * c4n, make_float4(g.x * w[q], g.y * w[q], g.z * w[q], g.w * w[q]));
}

template <int NV>
__global__ void __launch_bounds__(GNT, 1)
shade_simt_backward_kernel(const DevScene* __restrict__ scp, const DevWeightsF32* __restrict__ Wp, SampleSrc src,
                           const int* __restrict__ list, const int* __restrict__ count_ptr, int list_base, ShadeGrad gr) {
  using SM = GradSmem<NV>;
  extern __shared__ float4 smem4[];
  float* sm = reinterpret_cast<float*>(smem4);
  float *sPd = sm + SM::Pd, *sUV = sm + SM::UV, *sPW = sm + SM::PW, *sY = sm + SM::Y, *sPool = sm + SM::Pool;
  float *sdPool = sm + SM::dPool, *sLat = sm + SM::Lat, *sdLat = sm + SM::dLat, *sG = sm + SM::G, *sMisc = sm + SM::Misc;
  int* sId = reinterpret_cast<int*>(sm + SM::Id);
  const DevScene& sc = *scp;
  const DevWeightsF32& W = *Wp;
  const GradLayout& lay = gr.lay;
  float* slice = gr.slices + (size_t)blockIdx.x * lay.total;
  const float* wr = gr.wr;
  auto wrow = [&](int L) { return wr + lay.wo[L]; };
  const int t = threadIdx.x;
  const int V = sc.V, K = sc.K;
  const int encd = (1 + 2 * sc.sp_level) * K;
  const int count = *count_ptr;
  if (t == 0) sMisc[0] = 0.0f;

  // the per-view geometry MLP up to layer 2 (layer 3's input) for view v: X0, H1, X2 (|| feat8), H3
  auto geo_front = [&](int v) {
    float *X0 = sm + SM::X0, *H1 = sm + SM::H1, *X2 = sm + SM::X2, *H3 = sm + SM::H3;
    geo_input<GTS>(sc, v, K, encd, sUV, sPd, {X0, LDA}, {X2 + 128, 136});
    __syncthreads();
    dense_tile<ACT_SP, 4>(W, L_GEO0, X0, LDA, H1, 128);
    __syncthreads();
    dense_tile<ACT_SP, 4>(W, L_GEO1, H1, 128, X2, 136);
    __syncthreads();
    dense_tile<ACT_SP, 4>(W, L_GEO2, X2, 136, H3, 120);
    __syncthreads();
  };

  // the colour head of view v with every activation kept
  const HeadBufs head = {{sm + SM::Xv, 108}, {sm + SM::Hb1, 64}, {sm + SM::Hx, 32},  {sm + SM::Hs2, 32}, {sm + SM::Ht1, 32},
                         {sm + SM::Hpv, 36}, {sm + SM::Hxx, 32}, {sm + SM::Hs3, 32}, {sm + SM::Hu1, 32}, {sm + SM::Hv2, 1},
                         {sm + SM::Hoin, 40}, {sm + SM::Ho1, 16}, {sm + SM::Ho2, 8}};
  // the ray encoder of view v: E1 = elu(RE0 rd) (Hb1, ld 16), E = elu(RE1 E1) (Xv, ld 36)
  const Buf E1 = {sm + SM::Hb1, 16}, E = {sm + SM::Xv, 36};

  for (int tile = blockIdx.x; tile * GTS < count; tile += gridDim.x) {
    const int base = tile * GTS;
    const int nrows = min(GTS, count - base);
    // ---- 1-2. the tile's samples, projections and view weights; upstream gradients (zero on rows past the end, which replicate
    // the last one)
    load_tile<GTS>(sc, V, src, list, base, nrows, sId, sPd, sUV, sPW);
    if (t < GTS) {
      float* g = sG + t * 8;
      if (t < nrows) {
        const long long pos = (long long)list_base + base + t;
        const float2 da = gr.d_ao[pos];
        g[0] = da.y; g[1] = da.x;
        g[2] = gr.d_rgb[3 * pos]; g[3] = gr.d_rgb[3 * pos + 1]; g[4] = gr.d_rgb[3 * pos + 2];
      } else {
        g[0] = g[1] = g[2] = g[3] = g[4] = 0.0f;
      }
    }
    // ---- 3. per-view geometry MLP outputs
    for (int v = 0; v < V; ++v) {
      geo_front(v);
      dense_tile<ACT_NONE, 2>(W, L_GEO3, sm + SM::H3, 120, sY + v * GTS * 64, 64);
      __syncthreads();
    }
    // ---- 4. pooling, latent, density head forward and backward
    pool_geometry<GTS>(V, sPW, sY, {sPool, 128});
    __syncthreads();
    {
      float *D1 = sm + SM::D1, *D2 = sm + SM::D2, *gA = sm + SM::gA, *gB = sm + SM::gB;
      dense_tile<ACT_NONE, 1>(W, L_CMP, sPool, 128, sLat, 24);
      density_hidden<GTS>(W, {sPool, 128}, {D1, 64}, {D2, 64});
      // d [sdf_raw, rad] = sG[:, 0:2]
      accum_dw(slice, lay, W, L_DEN2, sG, 8, D2, 64);
      dense_bwd_x<2>(wrow(L_DEN2), 2, 64, 0, 64, sG, 8, gA, 64);
      __syncthreads();
      act_bwd<ACT_SP>(gA, 64, D2, 64, 64);
      __syncthreads();
      accum_dw(slice, lay, W, L_DEN1, gA, 64, D1, 64);
      dense_bwd_x<2>(wrow(L_DEN1), 64, 64, 0, 64, gA, 64, gB, 64);
      __syncthreads();
      act_bwd<ACT_SP>(gB, 64, D1, 64, 64);
      __syncthreads();
      accum_dw(slice, lay, W, L_DEN0, gB, 64, sPool, 128);
      dense_bwd_x<4>(wrow(L_DEN0), 64, 128, 0, 128, gB, 64, sdPool, 128);
      __syncthreads();
    }
    // ---- 5. colour branch forward (reference src/model.py:806-832, 1279-1289)
    float *F = sm + SM::F, *dF = sm + SM::dF, *MV = sm + SM::MV, *dMV = sm + SM::dMV, *RD = sm + SM::RD, *RGB = sm + SM::RGB;
    float *Om = sm + SM::Om, *dOm = sm + SM::dOm, *Logit = sm + SM::Logit, *dLogit = sm + SM::dLogit;
    for (int idx = t; idx < V * GTS; idx += GNT) dOm[idx] = 0.0f;
    for (int idx = t; idx < GTS * 72; idx += GNT) dMV[idx] = 0.0f;
    colour_inputs<GTS>(sc, V, sUV, sPd, sLat, F, RGB, RD);
    add_ray_encoding<GTS>(W, V, RD, E1, E, F);
    blend_weights<GTS>(W, V, RD, Om);
    __syncthreads();
    pool_colour<GTS>(V, F, Om, MV);
    __syncthreads();
    for (int v = 0; v < V; ++v) {
      colour_head<GTS>(W, v, MV, F, Om, RD, head);
      dense_tile<ACT_NONE, 1>(W, L_OUT2, sm + SM::Ho2, 8, Logit + v * GTS, 1);
      __syncthreads();
    }
    // ---- 6. softmax blend backward: d logit_v = sm_v (rgb_v - rgb) . d rgb
    if (t < GTS) {
      float e[MAXV], rgb[3];
      const float den = blend_colours<GTS>(V, Logit, RGB, t, e, rgb);
      const float* g = sG + t * 8 + 2;
      for (int v = 0; v < V; ++v) {
        float s = 0.0f;
        for (int c = 0; c < 3; ++c) s += (RGB[(v * GTS + t) * 4 + c] - rgb[c] / den) * g[c];
        dLogit[v * GTS + t] = e[v] / den * s;
      }
    }
    __syncthreads();
    // ---- 7. per-view colour head backward, activations rebuilt view by view
    for (int v = 0; v < V; ++v) {
      colour_head<GTS>(W, v, MV, F, Om, RD, head);
      float *Xv = sm + SM::Xv, *Hb1 = sm + SM::Hb1, *Hx = sm + SM::Hx, *Hs2 = sm + SM::Hs2, *Ht1 = sm + SM::Ht1;
      float *Hpv = sm + SM::Hpv, *Hxx = sm + SM::Hxx, *Hs3 = sm + SM::Hs3, *Hu1 = sm + SM::Hu1, *Hoin = sm + SM::Hoin;
      float *Ho1 = sm + SM::Ho1, *Ho2 = sm + SM::Ho2, *GA2 = sm + SM::GA2, *GB2 = sm + SM::GB2, *GC = sm + SM::GC;
      float* dL = dLogit + v * GTS;
      // out_layer (37 -> 16 -> 8 -> 1)
      accum_dw(slice, lay, W, L_OUT2, dL, 1, Ho2, 8);
      dense_bwd_x<1>(wrow(L_OUT2), 1, 8, 0, 8, dL, 1, GB2, 108);
      __syncthreads();
      act_bwd<ACT_ELU>(GB2, 108, Ho2, 8, 8);
      __syncthreads();
      accum_dw(slice, lay, W, L_OUT1, GB2, 108, Ho1, 16);
      dense_bwd_x<1>(wrow(L_OUT1), 8, 16, 0, 16, GB2, 108, GA2, 108);
      __syncthreads();
      act_bwd<ACT_ELU>(GA2, 108, Ho1, 16, 16);
      __syncthreads();
      accum_dw(slice, lay, W, L_OUT0, GA2, 108, Hoin, 40);
      dense_bwd_x<2>(wrow(L_OUT0), 16, 37, 0, 33, GA2, 108, GB2, 108);   // d (x + res) | d vis2; the ray diff is data
      __syncthreads();
      // vis_layer2 (32 -> 32 -> 1, sigmoid)
      if (t < GTS) {
        const float s = Hoin[t * 40 + 32];
        GC[t * 40 + 36] = GB2[t * 108 + 32] * s * (1.0f - s);   // d v2
      }
      __syncthreads();
      accum_dw(slice, lay, W, L_VIS2B, GC + 36, 40, Hu1, 32);
      dense_bwd_x<1>(wrow(L_VIS2B), 1, 32, 0, 32, GC + 36, 40, GA2, 108);
      __syncthreads();
      act_bwd<ACT_ELU>(GA2, 108, Hu1, 32, 32);
      __syncthreads();
      accum_dw(slice, lay, W, L_VIS2A, GA2, 108, Hs3, 32);
      dense_bwd_x<1>(wrow(L_VIS2A), 32, 32, 0, 32, GA2, 108, GC, 40);   // d s3
      __syncthreads();
      // s3 = xx * sigmoid(vis): d xx += d s3 * g (kept in GB2[:, 0:32]); d vis = sum_c d s3 xx * g (1 - g)
      for (int idx = t; idx < GTS * 32; idx += GNT) {
        int r = idx >> 5, c = idx & 31;
        const float g = sigmoidf(Hpv[r * 36 + 32]);
        GB2[r * 108 + c] += GC[r * 40 + c] * g;
      }
      if (t < GTS) {
        const float g = sigmoidf(Hpv[t * 36 + 32]);
        float s = 0.0f;
        for (int c = 0; c < 32; ++c) s += GC[t * 40 + c] * Hxx[t * 32 + c];
        GA2[t * 108 + 32] = s * g * (1.0f - g);
      }
      __syncthreads();
      // vis_layer1 (32 -> 32 -> 33): d pv = d res (= d xx) || d vis
      for (int idx = t; idx < GTS * 32; idx += GNT) {
        int r = idx >> 5, c = idx & 31;
        GA2[r * 108 + c] = GB2[r * 108 + c];
      }
      __syncthreads();
      act_bwd<ACT_ELU>(GA2, 108, Hpv, 36, 33);
      __syncthreads();
      accum_dw(slice, lay, W, L_VIS1B, GA2, 108, Ht1, 32);
      dense_bwd_x<1>(wrow(L_VIS1B), 33, 32, 0, 32, GA2, 108, GC, 40);
      __syncthreads();
      act_bwd<ACT_ELU>(GC, 40, Ht1, 32, 32);
      __syncthreads();
      accum_dw(slice, lay, W, L_VIS1A, GC, 40, Hs2, 32);
      dense_bwd_x<1>(wrow(L_VIS1A), 32, 32, 0, 32, GC, 40, GA2, 108);   // d s2, s2 = x * w_v
      __syncthreads();
      // d x = d xx + d s2 * w_v;  d w_v += sum_c d s2 * x
      for (int idx = t; idx < GTS * 32; idx += GNT) {
        int r = idx >> 5, c = idx & 31;
        GC[r * 40 + c] = GB2[r * 108 + c] + GA2[r * 108 + c] * Om[v * GTS + r];
      }
      if (t < GTS) {
        float s = 0.0f;
        for (int c = 0; c < 32; ++c) s += GA2[t * 108 + c] * Hx[t * 32 + c];
        dOm[v * GTS + t] += s;
      }
      __syncthreads();
      // base_layer (105 -> 64 -> 32)
      act_bwd<ACT_ELU>(GC, 40, Hx, 32, 32);
      __syncthreads();
      accum_dw(slice, lay, W, L_BASE1, GC, 40, Hb1, 64);
      dense_bwd_x<2>(wrow(L_BASE1), 32, 64, 0, 64, GC, 40, GA2, 108);
      __syncthreads();
      act_bwd<ACT_ELU>(GA2, 108, Hb1, 64, 64);
      __syncthreads();
      accum_dw(slice, lay, W, L_BASE0, GA2, 108, Xv, 108);
      dense_bwd_x<4>(wrow(L_BASE0), 64, 105, 0, 105, GA2, 108, GB2, 108);
      __syncthreads();
      for (int idx = t; idx < GTS * 105; idx += GNT) {
        int r = idx / 105, c = idx % 105;
        if (c < 70) dMV[r * 72 + c] += GB2[r * 108 + c];
        else dF[(v * GTS + r) * 36 + (c - 70)] = GB2[r * 108 + c];
      }
      __syncthreads();
    }
    // ---- 8. weighted mean || variance over views backward (reference src/model.py:1289-1291)
    for (int idx = t; idx < GTS * 35; idx += GNT) {
      int r = idx / 35, c = idx % 35;
      float mean = 0.0f;
      for (int v = 0; v < V; ++v) mean += F[(v * GTS + r) * 36 + c] * Om[v * GTS + r];
      float dl = 0.0f;
      for (int v = 0; v < V; ++v) dl += Om[v * GTS + r] * (F[(v * GTS + r) * 36 + c] - mean);
      const float dvar = dMV[r * 72 + 35 + c];
      const float dmean = dMV[r * 72 + c] - 2.0f * dl * dvar;   // the variance's own dependence on the mean
      for (int v = 0; v < V; ++v) {
        const float f = F[(v * GTS + r) * 36 + c], dlt = f - mean, w = Om[v * GTS + r];
        dF[(v * GTS + r) * 36 + c] += w * (dmean + 2.0f * dlt * dvar);
      }
      float* mdv = sm + SM::GA2 + r * 108;   // mean, dmean, dvar of (r, c) for the blend-weight gradient below
      mdv[c] = mean; mdv[35 + c] = dmean; mdv[70 + c] = dvar;
    }
    __syncthreads();
    // d Om_v += sum_c dmean f + dvar (f - mean)^2, one thread per (view, row) summing the channels in order (reproducible)
    for (int idx = t; idx < V * GTS; idx += GNT) {
      const int r = idx % GTS;
      const float* f = F + idx * 36;
      const float* mdv = sm + SM::GA2 + r * 108;
      float s = 0.0f;
      for (int c = 0; c < 35; ++c) {
        const float dlt = f[c] - mdv[c];
        s += mdv[35 + c] * f[c] + mdv[70 + c] * dlt * dlt;
      }
      dOm[idx] += s;
    }
    __syncthreads();
    // ---- 9. ray encoder backward per view; d tex -> feature map; d latent
    for (int idx = t; idx < GTS * 24; idx += GNT) {
      int r = idx / 24, c = idx % 24;
      float s = 0.0f;
      for (int v = 0; v < V; ++v) s += dF[(v * GTS + r) * 36 + 11 + c];
      sdLat[idx] = s;
    }
    for (int v = 0; v < V; ++v) {
      __syncthreads();
      ray_encoder<GTS>(W, v, RD, E1, E);
      float *GA2 = sm + SM::GA2, *GB2 = sm + SM::GB2;
      float* dFv = dF + v * GTS * 36;
      for (int idx = t; idx < GTS * 35; idx += GNT) {
        int r = idx / 35, c = idx % 35;
        GA2[r * 108 + c] = dFv[r * 36 + c] * delu(E.p[r * 36 + c]);
      }
      for (int idx = t; idx < nrows * 2; idx += GNT) {   // d feat_tex of view v (channels 3..10 of f)
        const int r = idx >> 1, c4 = idx & 1;
        const float* g = dFv + r * 36 + 3 + 4 * c4;
        scatter4(gr.d_ftex, sc.ftex, 8, v, sUV[(v * GTS + r) * 4], sUV[(v * GTS + r) * 4 + 1], c4, make_float4(g[0], g[1], g[2], g[3]));
      }
      __syncthreads();
      accum_dw(slice, lay, W, L_RE1, GA2, 108, E1.p, 16);
      dense_bwd_x<1>(wrow(L_RE1), 35, 16, 0, 16, GA2, 108, GB2, 108);
      __syncthreads();
      act_bwd<ACT_ELU>(GB2, 108, E1.p, 16, 16);
      __syncthreads();
      accum_dw(slice, lay, W, L_RE0, GB2, 108, RD + v * GTS * 4, 4);
    }
    // ---- 10. colour blending weights -> ani_al: w_v = ex_v - min_u ex_u, Om_v = w_v / (sum w + 1e-8), ex_v = exp(a (dot_v - 1))
    if (t < GTS) {
      // w_v = ex_v - ex_min is rebuilt as ex_min expm1(a (dot_v - dot_min)): the difference of two nearly equal exponentials
      // loses ~1e-7 / w of relative accuracy in fp32, and the gradient of Om weighs that error with 1 / w
      const float a = W.ani_al_abs;
      float dot[MAXV], mn = 3.0e38f;
      int amin = 0;
      for (int v = 0; v < V; ++v) {
        dot[v] = RD[(v * GTS + t) * 4 + 3];
        const float ex = expf(a * (dot[v] - 1.0f));
        if (ex < mn) { mn = ex; amin = v; }
      }
      float w[MAXV], dwda[MAXV], sum = 0.0f;
      for (int v = 0; v < V; ++v) {
        const float dl = dot[v] - dot[amin];
        w[v] = mn * expm1f(a * dl);
        dwda[v] = (dot[amin] - 1.0f) * w[v] + mn * dl * expf(a * dl);   // d w_v / d a
        sum += w[v];
      }
      const float inv = 1.0f / (sum + 1e-8f);
      // d w_u = inv^2 (sum_v (dOm_u - dOm_v) w_v + 1e-8 dOm_u): dOm_u inv - sum_v dOm_v w_v inv^2 without the cancellation of
      // 1 - Om when one weight carries nearly all of the sum
      float da = 0.0f;
      for (int u = 0; u < V; ++u) {
        const float du = dOm[u * GTS + t];
        float s = 1e-8f * du;
        for (int v = 0; v < V; ++v) s += (du - dOm[v * GTS + t]) * w[v];
        da += s * inv * inv * dwda[u];
      }
      // the tile's sum over its rows by a fixed butterfly (warp 0 holds the GTS = 32 rows), added by one thread (reproducible)
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) da += __shfl_xor_sync(0xffffffffu, da, d);
      if (t == 0) sMisc[0] += da;
    }
    __syncthreads();
    // ---- 11. latent backward (ibr_compress_gfeat): dPool += Wc^T dLat
    accum_dw(slice, lay, W, L_CMP, sdLat, 24, sPool, 128);
    dense_bwd_x<4, true>(wrow(L_CMP), 24, 128, 0, 128, sdLat, 24, sdPool, 128);
    __syncthreads();
    // ---- 12. pooled mean || variance backward -> d y_v (in place of y_v)
    {
      const int r = t >> 2, q4 = t & 3;
      for (int c = q4 * 16; c < q4 * 16 + 16; ++c) {
        float y[MAXV], mean = 0.0f;
        for (int v = 0; v < V; ++v) { y[v] = sY[(v * GTS + r) * 64 + c]; mean += sPW[v * GTS + r] * y[v]; }
        float dl = 0.0f;
        for (int v = 0; v < V; ++v) dl += sPW[v * GTS + r] * (y[v] - mean);
        const float dvar = sdPool[r * 128 + 64 + c];
        const float dmean = sdPool[r * 128 + c] - 2.0f * dl * dvar;
        for (int v = 0; v < V; ++v) sY[(v * GTS + r) * 64 + c] = sPW[v * GTS + r] * (dmean + 2.0f * (y[v] - mean) * dvar);
      }
    }
    __syncthreads();
    // ---- 13. per-view geometry MLP backward, layers rebuilt view by view
    for (int v = 0; v < V; ++v) {
      geo_front(v);
      float *X0 = sm + SM::X0, *H1 = sm + SM::H1, *X2 = sm + SM::X2, *H3 = sm + SM::H3, *GA = sm + SM::GA, *GB = sm + SM::GB;
      float* dY = sY + v * GTS * 64;
      accum_dw(slice, lay, W, L_GEO3, dY, 64, H3, 120);
      dense_bwd_x<4>(wrow(L_GEO3), 64, 120, 0, 120, dY, 64, GA, 136);
      __syncthreads();
      act_bwd<ACT_SP>(GA, 136, H3, 120, 120);
      __syncthreads();
      accum_dw(slice, lay, W, L_GEO2, GA, 136, X2, 136);
      dense_bwd_x<5>(wrow(L_GEO2), 120, 136, 0, 136, GA, 136, GB, 136);
      __syncthreads();
      act_bwd<ACT_SP>(GB, 136, X2, 136, 128);
      for (int idx = t; idx < nrows * 2; idx += GNT) {   // d feat8 (columns 128..135)
        const int r = idx >> 1, c4 = idx & 1;
        const float* g = GB + r * 136 + 128 + 4 * c4;
        scatter4(gr.d_f8, sc.f8, 8, v, sUV[(v * GTS + r) * 4], sUV[(v * GTS + r) * 4 + 1], c4, make_float4(g[0], g[1], g[2], g[3]));
      }
      __syncthreads();
      accum_dw(slice, lay, W, L_GEO1, GB, 136, H1, 128);
      dense_bwd_x<4>(wrow(L_GEO1), 128, 128, 0, 128, GB, 136, GA, 136);
      __syncthreads();
      act_bwd<ACT_SP>(GA, 136, H1, 128, 128);
      __syncthreads();
      accum_dw(slice, lay, W, L_GEO0, GA, 136, X0, LDA);
      dense_bwd_x<2>(wrow(L_GEO0), 128, encd + 64, encd, 64, GA, 136, GB, 136);   // d feat64 (the encoding is data)
      __syncthreads();
      for (int idx = t; idx < nrows * 16; idx += GNT) {
        const int r = idx >> 4, c4 = idx & 15;
        const float* g = GB + r * 136 + 4 * c4;
        scatter4(gr.d_f64, sc.f64, 64, v, sUV[(v * GTS + r) * 4], sUV[(v * GTS + r) * 4 + 1], c4, make_float4(g[0], g[1], g[2], g[3]));
      }
      __syncthreads();
    }
  }
  __syncthreads();
  if (t == 0) slice[lay.ani] += sMisc[0] * gr.ani_sign;
}

// ------------------------------------------------------------------------------------------------
// weights and reduction
// ------------------------------------------------------------------------------------------------
// wr[wo[l] + n K + k] = W_l[n][k] from the fp32 engine's transposed, padded copy; grid.y = layer
__global__ void weights_rowmajor_kernel(const DevWeightsF32* __restrict__ Wp, float* __restrict__ wr, GradLayout lay) {
  const DevWeightsF32& W = *Wp;
  const int l = blockIdx.y;
  const int N = W.N[l], K = W.K[l], ldw = W.ldw[l];
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < N * K; idx += gridDim.x * blockDim.x) {
    const int n = idx / K, k = idx - n * K;
    wr[lay.wo[l] + idx] = W.wt[l][k * ldw + n];
  }
}

__global__ void grad_reduce_kernel(const float* __restrict__ slices, int n, int total, float* __restrict__ out) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    float s = 0.0f;
    for (int b = 0; b < n; ++b) s += slices[(size_t)b * total + i];
    out[i] = s;
  }
}

// ------------------------------------------------------------------------------------------------
// canonical work list
// ------------------------------------------------------------------------------------------------
// The front kernel's blocks reserve their ranges of the work list with an atomicAdd each, so the order of the rays in its list
// changes from call to call.  Rewritten with every ray's entries (in sample order, as the front wrote them) at the exclusive
// scan of the counts in ray order, the list is a function of the rays alone.  One warp per ray.
__global__ void canonical_list_kernel(const int* __restrict__ list_in, const int* __restrict__ start_in, const int* __restrict__ cnt,
                                      const int* __restrict__ start_out, int nr, int* __restrict__ list_out) {
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  for (int i = blockIdx.x * wpb + (threadIdx.x >> 5); i < nr; i += gridDim.x * wpb) {
    const int a = start_in[i], b = start_out[i], n = cnt[i];
    for (int j = lane; j < n; j += 32) list_out[b + j] = list_in[a + j];
  }
}

size_t canonical_list_temp_bytes(int nr) {
  size_t bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, bytes, (const int*)nullptr, (int*)nullptr, nr);
  return bytes;
}

cudaError_t launch_canonical_list(const int* list_in, const int* start_in, const int* cnt, int nr, int* list_out, int* start_out,
                                  void* scan_tmp, size_t scan_bytes, int num_sms, cudaStream_t st) {
  if (nr < 1) return cudaSuccess;
  cudaError_t e = cub::DeviceScan::ExclusiveSum(scan_tmp, scan_bytes, cnt, start_out, nr, st);   // deterministic
  if (e != cudaSuccess) return e;
  long long blocks = ((long long)nr * 32 + 255) / 256;
  if (blocks > (long long)num_sms * 16) blocks = (long long)num_sms * 16;
  canonical_list_kernel<<<(unsigned)blocks, 256, 0, st>>>(list_in, start_in, cnt, start_out, nr, list_out);
  return cudaGetLastError();
}

cudaError_t launch_composite_backward(const int* list, const float2* ao, const float* rgb, const int* start, const int* cnt,
                                      const float* zbuf, const float* ray_nf, int r0, int nr, int S, long long plane, const RayGrad& g,
                                      float2* d_ao, float* d_rgb, float2* at, int num_sms, cudaStream_t st) {
  if (nr < 1) return cudaSuccess;
  long long blocks = ((long long)nr * 32 + 127) / 128;
  if (blocks > (long long)num_sms * 64) blocks = (long long)num_sms * 64;
  composite_backward_kernel<<<(unsigned)blocks, 128, 0, st>>>(list, ao, rgb, start, cnt, zbuf, ray_nf, r0, nr, S, plane, g, d_ao, d_rgb, at);
  return cudaGetLastError();
}

template <int NV>
static cudaError_t launch_shade_backward_nv(const ShadeBatch& b, const ShadeGrad& g) {
  constexpr size_t smem = GRAD_SMEM_BYTES<NV>;
  cudaError_t e = cudaFuncSetAttribute(shade_simt_backward_kernel<NV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  shade_simt_backward_kernel<NV><<<b.num_sms, GNT, smem, b.st>>>(b.sc, b.wf32, b.src, b.list, b.counter, b.so.list_base, g);
  e = cudaGetLastError();
  if (e == cudaSuccess) *b.launches += 1;
  return e;
}

cudaError_t launch_shade_simt_backward(const ShadeBatch& b, const ShadeGrad& g) {
  switch (b.n_views) {
    case 1: return launch_shade_backward_nv<1>(b, g);
    case 2: return launch_shade_backward_nv<2>(b, g);
    case 3: return launch_shade_backward_nv<3>(b, g);
    case 4: return launch_shade_backward_nv<4>(b, g);
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t launch_weights_rowmajor(const DevWeightsF32* w, float* wr, const GradLayout& lay, cudaStream_t st) {
  weights_rowmajor_kernel<<<dim3(16, NLAYER), 256, 0, st>>>(w, wr, lay);
  return cudaGetLastError();
}

cudaError_t launch_grad_reduce(const float* slices, int n, int total, float* out, cudaStream_t st) {
  grad_reduce_kernel<<<(total + 255) / 256, 256, 0, st>>>(slices, n, total, out);
  return cudaGetLastError();
}

}  // namespace kpn
