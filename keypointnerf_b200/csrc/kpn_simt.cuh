// The fp32 engine's forward over a tile of TS samples with 4 TS threads: its dense layer and the phases of shading around it.
// Its forward shading kernel (shade_simt_kernel, kpn_kernels.cu) and the backward kernel that recomputes that forward
// (shade_simt_backward_kernel, kpn_grad.cu) both call these, so that the gradient is taken at the forward's own values.  Each
// kernel keeps its own shared-memory layout and passes the buffers in; the forward reuses buffers in place, so a phase's
// elementwise steps read only the elements they write or another buffer.
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

// A tile's rows in shared memory: row r at p + r * ld.
struct Buf {
  float* p;
  int ld;
};

// ---- 1. the tile's samples list[base, base + nrows) into Id and P ([TS][8]: p xyz, d xyz; rows past nrows replicate the last
// one), their projections into UV ([NV][TS][4]: u, v, zn, boundary weight) and the view weights into PW ([NV][TS])
// (reference src/model.py:713-723, 750-759; mask == 1 here)
template <int TS>
__device__ __forceinline__ void load_tile(const DevScene& sc, int V, const SampleSrc& src, const int* list, int base, int nrows,
                                          int* Id, float* P, float* UV, float* PW) {
  constexpr int NT = 4 * TS;
  const int t = threadIdx.x;
  if (t < TS) {
    int id = list[base + min(t, nrows - 1)];
    Id[t] = id;
    float p[3], d[3];
    fetch_sample<true>(src, id, p, d);
    float* o = P + t * 8;
    o[0] = p[0]; o[1] = p[1]; o[2] = p[2]; o[3] = d[0]; o[4] = d[1]; o[5] = d[2];
  }
  __syncthreads();
  for (int idx = t; idx < V * TS; idx += NT) {
    int v = idx / TS, r = idx % TS;
    Proj q = project_view(sc, v, P + r * 8);
    float* o = UV + idx * 4;
    o[0] = q.u; o[1] = q.v; o[2] = q.zn; o[3] = boundary_weight(q);
  }
  __syncthreads();
  if (t < TS) {
    float sum = 0.0f;
    for (int v = 0; v < V; ++v) sum += UV[(v * TS + t) * 4 + 3];
    for (int v = 0; v < V; ++v) PW[v * TS + t] = UV[(v * TS + t) * 4 + 3] / (sum + 1e-6f);
  }
}

// ---- 2. view v's geometry MLP input (reference src/utils.py:691-720): keypoint encoding (encd floats) || feat64 taps into
// x0, and the feat8 taps (the last 8 inputs of layer 2) into f8.  Four threads per row.
template <int TS>
__device__ __forceinline__ void geo_input(const DevScene& sc, int v, int K, int encd, const float* UV, const float* P, Buf x0,
                                          Buf f8) {
  const int t = threadIdx.x;
  const int r = t >> 2, q4 = t & 3;
  const float* uv = UV + (v * TS + r) * 4;
  float* row = x0.p + r * x0.ld;
  Taps t64 = make_taps(uv[0], uv[1], sc.f64.W, sc.f64.H);
  float f[16];
  gather_f32<4>(sc.f64, v, t64, q4 * 4, f);
#pragma unroll
  for (int i = 0; i < 16; ++i) row[encd + q4 * 16 + i] = f[i];
  float c[3];
  to_camera(sc, v, P + r * 8, c);
  for (int k = q4; k < K; k += 4) encode_kpt(sc, v, k, c, row);
  if (q4 < 2) {
    Taps t8 = make_taps(uv[0], uv[1], sc.f8.W, sc.f8.H);
    float g[4];
    gather_f32<1>(sc.f8, v, t8, q4, g);
#pragma unroll
    for (int i = 0; i < 4; ++i) f8.p[r * f8.ld + q4 * 4 + i] = g[i];
  }
}

// ---- 3. weighted mean || variance over the views of the geometry features Y ([NV][TS][64]) into 128 columns of out
// (reference src/utils.py:722-748)
template <int TS>
__device__ __forceinline__ void pool_geometry(int V, const float* PW, const float* Y, Buf out) {
  const int t = threadIdx.x;
  const int r = t >> 2, q4 = t & 3;
  for (int c = q4 * 16; c < q4 * 16 + 16; ++c) {
    float mean = 0.0f;
    for (int v = 0; v < V; ++v) mean += PW[v * TS + r] * Y[(v * TS + r) * 64 + c];
    float var = 0.0f;
    for (int v = 0; v < V; ++v) {
      float dlt = Y[(v * TS + r) * 64 + c] - mean;
      var += PW[v * TS + r] * dlt * dlt;
    }
    out.p[r * out.ld + c] = mean;
    out.p[r * out.ld + 64 + c] = var;
  }
}

// ---- 4. the density head's hidden layers: pool -> h1 -> h2
template <int TS>
__device__ __forceinline__ void density_hidden(const DevWeightsF32& W, Buf pool, Buf h1, Buf h2) {
  dense_tile<ACT_SP, 2>(W, L_DEN0, pool.p, pool.ld, h1.p, h1.ld);
  __syncthreads();
  dense_tile<ACT_SP, 2>(W, L_DEN1, h1.p, h1.ld, h2.p, h2.ld);
  __syncthreads();
}

// ---- 5. colour branch inputs of every view (reference src/model.py:806-832): F ([NV][TS][36]) = rgb || feat_tex taps ||
// latent (Lat, [TS][24]), the source colours into RGB and the ray differences into RD ([NV][TS][4])
template <int TS>
__device__ __forceinline__ void colour_inputs(const DevScene& sc, int V, const float* UV, const float* P, const float* Lat,
                                              float* F, float* RGB, float* RD) {
  constexpr int NT = 4 * TS;
  const int t = threadIdx.x;
  for (int idx = t; idx < V * TS; idx += NT) {
    int v = idx / TS, r = idx % TS;
    const float* uv = UV + idx * 4;
    float* f = F + idx * 36;
    Taps ti = make_taps(uv[0], uv[1], sc.img.W, sc.img.H);
    float c4[4];
    gather_f32<1>(sc.img, v, ti, 0, c4);
    RGB[idx * 4 + 0] = c4[0]; RGB[idx * 4 + 1] = c4[1]; RGB[idx * 4 + 2] = c4[2];
    f[0] = c4[0]; f[1] = c4[1]; f[2] = c4[2];
    Taps tt = make_taps(uv[0], uv[1], sc.ftex.W, sc.ftex.H);
    float g[8];
    gather_f32<2>(sc.ftex, v, tt, 0, g);
#pragma unroll
    for (int i = 0; i < 8; ++i) f[3 + i] = g[i];
    ray_diff(sc, v, P + r * 8, P + r * 8 + 3, RD + idx * 4);
  }
  __syncthreads();
  for (int idx = t; idx < V * TS * 24; idx += NT) {
    int c = idx % 24, vr = idx / 24;
    F[vr * 36 + 11 + c] = Lat[(vr % TS) * 24 + c];
  }
}

// ---- 6. ray-direction encoder 4->16->35 (ELU) of view v (src/model.py:1279-1284): e1 = elu(RE0 rd_v), e = elu(RE1 e1)
template <int TS>
__device__ __forceinline__ void ray_encoder(const DevWeightsF32& W, int v, const float* RD, Buf e1, Buf e) {
  dense_tile<ACT_ELU, 1>(W, L_RE0, RD + v * TS * 4, 4, e1.p, e1.ld);
  __syncthreads();
  dense_tile<ACT_ELU, 2>(W, L_RE1, e1.p, e1.ld, e.p, e.ld);
  __syncthreads();
}

// ... added onto the first 35 features of every view
template <int TS>
__device__ __forceinline__ void add_ray_encoding(const DevWeightsF32& W, int V, const float* RD, Buf e1, Buf e, float* F) {
  constexpr int NT = 4 * TS;
  const int t = threadIdx.x;
  for (int v = 0; v < V; ++v) {
    __syncthreads();
    ray_encoder<TS>(W, v, RD, e1, e);
    for (int idx = t; idx < TS * 35; idx += NT) {
      int r = idx / 35, c = idx % 35;
      F[(v * TS + r) * 36 + c] += e.p[r * e.ld + c];
    }
  }
}

// ---- 7. blending weights Om ([NV][TS]) from the ray differences (src/model.py:1286-1289), mask == 1
template <int TS>
__device__ __forceinline__ void blend_weights(const DevWeightsF32& W, int V, const float* RD, float* Om) {
  const int t = threadIdx.x;
  if (t < TS) {
    float ex[MAXV], mn = 3.0e38f;
    for (int v = 0; v < V; ++v) {
      ex[v] = expf(W.ani_al_abs * (RD[(v * TS + t) * 4 + 3] - 1.0f));
      mn = fminf(mn, ex[v]);
    }
    float sum = 0.0f;
    for (int v = 0; v < V; ++v) { ex[v] -= mn; sum += ex[v]; }
    for (int v = 0; v < V; ++v) Om[v * TS + t] = ex[v] / (sum + 1e-8f);
  }
}

// ---- 8. Om-weighted mean || variance of the 35 features over the views into MV ([TS][72])
template <int TS>
__device__ __forceinline__ void pool_colour(int V, const float* F, const float* Om, float* MV) {
  constexpr int NT = 4 * TS;
  for (int idx = threadIdx.x; idx < TS * 35; idx += NT) {
    int r = idx / 35, c = idx % 35;
    float mean = 0.0f;
    for (int v = 0; v < V; ++v) mean += F[(v * TS + r) * 36 + c] * Om[v * TS + r];
    float var = 0.0f;
    for (int v = 0; v < V; ++v) {
      float dlt = F[(v * TS + r) * 36 + c] - mean;
      var += Om[v * TS + r] * dlt * dlt;
    }
    MV[r * 72 + c] = mean;
    MV[r * 72 + 35 + c] = var;
  }
}

// ---- 9. view v's IBR head (src/model.py:1292-1300) up to out_layer's last hidden layer (ho2, 8 columns).  Activations:
// xv = mean || var || f_v (105), base_layer hb1 (64) -> hx (32); vis_layer1 on hs2 = hx w_v: ht1 -> hpv (res || vis, 33);
// hxx = hx + res; vis_layer2 on hs3 = hxx sigmoid(vis): hu1 -> hv2 (1); out_layer on hoin = hxx || sigmoid(hv2) || rd_v (37):
// ho1 (16) -> ho2 (8).
struct HeadBufs {
  Buf xv, hb1, hx, hs2, ht1, hpv, hxx, hs3, hu1, hv2, hoin, ho1, ho2;
};

template <int TS>
__device__ __forceinline__ void colour_head(const DevWeightsF32& W, int v, const float* MV, const float* F, const float* Om,
                                            const float* RD, const HeadBufs& h) {
  constexpr int NT = 4 * TS;
  const int t = threadIdx.x;
  for (int idx = t; idx < TS * 105; idx += NT) {
    int r = idx / 105, c = idx % 105;
    h.xv.p[r * h.xv.ld + c] = c < 70 ? MV[r * 72 + c] : F[(v * TS + r) * 36 + (c - 70)];
  }
  __syncthreads();
  dense_tile<ACT_ELU, 2>(W, L_BASE0, h.xv.p, h.xv.ld, h.hb1.p, h.hb1.ld);
  __syncthreads();
  dense_tile<ACT_ELU, 1>(W, L_BASE1, h.hb1.p, h.hb1.ld, h.hx.p, h.hx.ld);
  __syncthreads();
  for (int idx = t; idx < TS * 32; idx += NT) {
    int r = idx >> 5, c = idx & 31;
    h.hs2.p[r * h.hs2.ld + c] = h.hx.p[r * h.hx.ld + c] * Om[v * TS + r];
  }
  __syncthreads();
  dense_tile<ACT_ELU, 1>(W, L_VIS1A, h.hs2.p, h.hs2.ld, h.ht1.p, h.ht1.ld);
  __syncthreads();
  dense_tile<ACT_ELU, 2>(W, L_VIS1B, h.ht1.p, h.ht1.ld, h.hpv.p, h.hpv.ld);
  __syncthreads();
  for (int idx = t; idx < TS * 32; idx += NT) {
    int r = idx >> 5, c = idx & 31;
    float x = h.hx.p[r * h.hx.ld + c] + h.hpv.p[r * h.hpv.ld + c];
    h.hxx.p[r * h.hxx.ld + c] = x;
    h.hs3.p[r * h.hs3.ld + c] = x * sigmoidf(h.hpv.p[r * h.hpv.ld + 32]);
  }
  __syncthreads();
  dense_tile<ACT_ELU, 1>(W, L_VIS2A, h.hs3.p, h.hs3.ld, h.hu1.p, h.hu1.ld);
  __syncthreads();
  dense_tile<ACT_NONE, 1>(W, L_VIS2B, h.hu1.p, h.hu1.ld, h.hv2.p, h.hv2.ld);
  __syncthreads();
  for (int idx = t; idx < TS * 37; idx += NT) {
    int r = idx / 37, c = idx % 37;
    float val = c < 32 ? h.hxx.p[r * h.hxx.ld + c]
                       : (c == 32 ? sigmoidf(h.hv2.p[r * h.hv2.ld]) : RD[(v * TS + r) * 4 + (c - 33)]);
    h.hoin.p[r * h.hoin.ld + c] = val;
  }
  __syncthreads();
  dense_tile<ACT_ELU, 1>(W, L_OUT0, h.hoin.p, h.hoin.ld, h.ho1.p, h.ho1.ld);
  __syncthreads();
  dense_tile<ACT_ELU, 1>(W, L_OUT1, h.ho1.p, h.ho1.ld, h.ho2.p, h.ho2.ld);
  __syncthreads();
}

// ---- 10. softmax over the views' logits (Logit, [NV][TS]) of row r (src/model.py:1300-1301): e[v] = exp(logit_v - max),
// rgb = sum_v e[v] rgb_v of the source colours RGB; returns sum_v e[v]
template <int TS>
__device__ __forceinline__ float blend_colours(int V, const float* Logit, const float* RGB, int r, float e[MAXV], float rgb[3]) {
  float m = -3.0e38f;
  for (int v = 0; v < V; ++v) m = fmaxf(m, Logit[v * TS + r]);
  float den = 0.0f;
  rgb[0] = rgb[1] = rgb[2] = 0.0f;
  for (int v = 0; v < V; ++v) {
    e[v] = expf(Logit[v * TS + r] - m);
    den += e[v];
    for (int c = 0; c < 3; ++c) rgb[c] += e[v] * RGB[(v * TS + r) * 4 + c];
  }
  return den;
}

}  // namespace kpn
