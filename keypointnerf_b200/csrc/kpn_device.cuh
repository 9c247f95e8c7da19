// Device helpers shared by the ray-march kernels: sample fetch, projection + validity,
// border-clamped bilinear taps on channel-last atlases, keypoint encoding, activations.
#pragma once
#include "kpn_types.cuh"

namespace kpn {

__device__ __forceinline__ float softplus100(float x) {
  // torch.nn.Softplus(beta=100, threshold=20): reference src/utils.py:523-524
  float bx = 100.0f * x;
  return bx > 20.0f ? x : log1pf(expf(bx)) * 0.01f;
}
__device__ __forceinline__ float elu1(float x) { return x > 0.0f ? x : expm1f(x); }
__device__ __forceinline__ float sigmoidf(float x) { return 1.0f / (1.0f + expf(-x)); }

// torch.linspace(0, 1, S) in fp32: symmetric evaluation from both ends (reference src/model.py:1045).
__device__ __forceinline__ float linspace01(int i, int S) {
  if (S <= 1) return 0.0f;
  float step = 1.0f / (float)(S - 1);
  return i < S / 2 ? step * (float)i : 1.0f - step * (float)(S - 1 - i);
}
// depth of coarse sample s of a ray: z = near + (far - near) * linspace(0,1,S)[s]  (reference src/model.py:1045-1055)
__device__ __forceinline__ float coarse_depth(float n_r, float f_r, int s, int S) { return n_r + (f_r - n_r) * linspace01(s, S); }

// Compositing (reference src/model.py:1150-1176), shared by composite_kernel and its backward.  The list entry at sample k of a
// ray of S samples: its depth (zz: the ray's depths, else the coarse depths between n_r and f_r), the distance to the next
// sample (1e10 on the ray's last, reference src/model.py:1166) and its alpha 1 - exp(-sigma dist).
struct ListEntry { float z, dist, alpha; };
__device__ __forceinline__ ListEntry list_entry(const float* zz, float n_r, float f_r, int k, int S, float sigma) {
  ListEntry en;
  float znext;
  if (zz) { en.z = zz[k]; znext = k + 1 < S ? zz[k + 1] : 0.0f; }
  else { en.z = coarse_depth(n_r, f_r, k, S); znext = k + 1 < S ? coarse_depth(n_r, f_r, k + 1, S) : 0.0f; }
  en.dist = k + 1 < S ? znext - en.z : 1e10f;
  en.alpha = 1.0f - expf(-sigma * en.dist);
  return en;
}
// Compositing weights of a group of 32 list entries (lane l: entry l, alpha a): c_l = a T_l with the transmittance
// T_l = Tc prod_{j<l} (1 - a_j), an exclusive product scan across the lanes.  Tc is carried on to the next group.
__device__ __forceinline__ float composite_weight(float a, int lane, float& Tc, float& T) {
  float p = 1.0f - a;   // inclusive product scan of (1 - a)
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const float t = __shfl_up_sync(0xffffffffu, p, d);
    if (lane >= d) p *= t;
  }
  float ex = __shfl_up_sync(0xffffffffu, p, 1);
  if (lane == 0) ex = 1.0f;
  T = Tc * ex;
  const float c = a * T;
  Tc *= __shfl_sync(0xffffffffu, p, 31);
  return c;
}

__device__ __forceinline__ float sample_depth(const SampleSrc& src, long long id, long long r) {
  if (src.z) return src.z[id];
  return coarse_depth(src.ray_nf[2 * r], src.ray_nf[2 * r + 1], (int)(id - r * src.S), src.S);
}

// ---- sample fetch -----------------------------------------------------------------------------
// GRID: the kernel may see grid sources (mode 2).  The render kernels are compiled without that branch, so that their code is
// what it is without the grid source.
template <bool GRID = false>
__device__ __forceinline__ void fetch_sample(const SampleSrc& src, long long id, float p[3], float d[3]) {
  if (GRID && src.mode == 2) {
    const long long g = src.g_id0 + id;
    const long long r = g / src.g_nx;
    const int idx[3] = {(int)(g - r * src.g_nx), (int)(r % src.g_ny), (int)(r / src.g_ny)};
#pragma unroll
    for (int a = 0; a < 3; ++a) p[a] = __fadd_rn(src.g_org[a], __fmul_rn(src.g_sp[a], (float)idx[a]));
    d[0] = 0.0f; d[1] = 0.0f; d[2] = 0.0f;
  } else if (src.mode == 0) {
    long long r = id / src.S;
    float z = sample_depth(src, id, r);
    d[0] = src.ray_d[3 * r + 0]; d[1] = src.ray_d[3 * r + 1]; d[2] = src.ray_d[3 * r + 2];
    // eval_pts = cam_pos + cam_rays * z  (reference src/model.py:1057)
    const float* o = src.o + 3 * r;
    p[0] = o[0] + d[0] * z; p[1] = o[1] + d[1] * z; p[2] = o[2] + d[2] * z;
  } else {
    p[0] = src.pts[3 * id + 0]; p[1] = src.pts[3 * id + 1]; p[2] = src.pts[3 * id + 2];
    d[0] = src.view[3 * id + 0]; d[1] = src.view[3 * id + 1]; d[2] = src.view[3 * id + 2];
  }
}

// ---- projection (reference src/model.py:713-723) ------------------------------------------------
struct Proj { float u, v, zn; };  // normalised [-1,1] image coords and normalised depth

__device__ __forceinline__ Proj project_view(const DevScene& sc, int v, const float p[3]) {
  const float* P = sc.P[v];
  float hx = P[0] * p[0] + P[1] * p[1] + P[2] * p[2] + P[3];
  float hy = P[4] * p[0] + P[5] * p[1] + P[6] * p[2] + P[7];
  float hz = P[8] * p[0] + P[9] * p[1] + P[10] * p[2] + P[11];
  Proj r;
  r.u = 2.0f * ((hx / hz) / sc.wm1) - 1.0f;
  r.v = 2.0f * ((hy / hz) / sc.hm1) - 1.0f;
  r.zn = 2.0f * (hz - sc.znear) / (sc.zfar - sc.znear) - 1.0f;
  return r;
}

__device__ __forceinline__ bool in_frustum(const Proj& q) {
  // reference src/model.py:725-729 (epsilon = 1e-2, no far bound on z)
  const float lo = -1.0f - 1e-2f, hi = 1.0f + 1e-2f;
  return q.u >= lo && q.u <= hi && q.v >= lo && q.v <= hi && q.zn >= -1.0f;
}

// ---- bilinear taps, grid_sample(bilinear, border, align_corners=True): reference src/utils.py:74-89 ---
struct Taps {
  int o00, o01, o10, o11;   // texel offsets (in texels) within one view's HxW plane
  float w00, w01, w10, w11; // nw, ne, sw, se
};

__device__ __forceinline__ Taps make_taps(float u, float v, int W, int H) {
  float ix = (u + 1.0f) * 0.5f * (float)(W - 1);
  float iy = (v + 1.0f) * 0.5f * (float)(H - 1);
  ix = fminf(fmaxf(ix, 0.0f), (float)(W - 1));
  iy = fminf(fmaxf(iy, 0.0f), (float)(H - 1));
  float x0f = floorf(ix), y0f = floorf(iy);
  int x0 = (int)x0f, y0 = (int)y0f;
  int x1 = min(x0 + 1, W - 1), y1 = min(y0 + 1, H - 1);  // weight is exactly 0 when the clamp bites
  float wx1 = ix - x0f, wy1 = iy - y0f;
  float wx0 = (x0f + 1.0f) - ix, wy0 = (y0f + 1.0f) - iy;
  Taps t;
  t.o00 = y0 * W + x0; t.o01 = y0 * W + x1; t.o10 = y1 * W + x0; t.o11 = y1 * W + x1;
  t.w00 = wx0 * wy0; t.w01 = wx1 * wy0; t.w10 = wx0 * wy1; t.w11 = wx1 * wy1;
  return t;
}

// Foreground mask atlas: uint8 [V][H][W].
__device__ __forceinline__ float sample_fg(const DevScene& sc, int v, const Proj& q) {
  const MapDesc& m = sc.fg;
  Taps t = make_taps(q.u, q.v, m.W, m.H);
  const uint8_t* b = (const uint8_t*)m.ptr + (size_t)v * m.H * m.W;
  return t.w00 * (float)b[t.o00] + t.w01 * (float)b[t.o01] + t.w10 * (float)b[t.o10] + t.w11 * (float)b[t.o11];
}

// A sample is valid iff it is inside EVERY view's frustum and foreground in EVERY view
// (reference src/model.py:729-739).  Also returns the per-view projections.
__device__ __forceinline__ bool sample_valid(const DevScene& sc, const float p[3], Proj q[MAXV]) {
  bool ok = true;
  for (int v = 0; v < sc.V && ok; ++v) {   // the first view that rejects the sample ends the test (q of the later views is unset)
    q[v] = project_view(sc, v, p);
    ok = in_frustum(q[v]);
  }
  if (ok && sc.use_fg) {
    for (int v = 0; v < sc.V; ++v) ok = ok && (sample_fg(sc, v, q[v]) > 0.1f);
  }
  return ok;
}

// Boundary-smooth (unnormalised) view weight, reference src/model.py:750-756.
__device__ __forceinline__ float boundary_weight(const Proj& q) {
  float c[3] = {q.u, q.v, q.zn};
  float w = 1.0f;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    float x = 0.5f * c[i] + 0.5f;
    float db = fminf(x, 1.0f - x);
    w *= sigmoidf(5.0f * (db / 0.1f - 1.0f));
  }
  return w;
}

// fp32 channel-last gather of NC4 float4 groups starting at float4-group g0:  out[4*i..] for i<NC4.
template <int NC4>
__device__ __forceinline__ void gather_f32(const MapDesc& m, int v, const Taps& t, int g0, float* out) {
  const int c4 = m.C >> 2;
  const float4* base = (const float4*)m.ptr + (size_t)v * m.H * m.W * c4 + g0;
  const float4* p00 = base + (size_t)t.o00 * c4;
  const float4* p01 = base + (size_t)t.o01 * c4;
  const float4* p10 = base + (size_t)t.o10 * c4;
  const float4* p11 = base + (size_t)t.o11 * c4;
#pragma unroll
  for (int i = 0; i < NC4; ++i) {
    float4 a = __ldg(p00 + i), b = __ldg(p01 + i), c = __ldg(p10 + i), d = __ldg(p11 + i);
    out[4 * i + 0] = a.x * t.w00 + b.x * t.w01 + c.x * t.w10 + d.x * t.w11;
    out[4 * i + 1] = a.y * t.w00 + b.y * t.w01 + c.y * t.w10 + d.y * t.w11;
    out[4 * i + 2] = a.z * t.w00 + b.z * t.w01 + c.z * t.w10 + d.z * t.w11;
    out[4 * i + 3] = a.w * t.w00 + b.w * t.w01 + c.w * t.w10 + d.w * t.w11;
  }
}

// Relative spatial keypoint encoding of one keypoint (sp_type "rel_z_decay"):
// reference src/spatial.py:76,81-85,110-118 with position_embedding 23-39.
// Writes row[r*K + k], r = 0: dz*w, 1+2l: sin(pi 2^l dz)*w, 2+2l: cos(pi 2^l dz)*w.
__device__ __forceinline__ void encode_kpt(const DevScene& sc, int v, int k, const float c[3], float* row) {
  const float* kc = sc.kc[v][k];
  float dx = c[0] - kc[0], dy = c[1] - kc[1], dzc = c[2] - kc[2];
  float dz = sc.sp_scale * dzc;
  float w = expf(-(dx * dx + dy * dy + dzc * dzc) * sc.inv2sig2);
  const int K = sc.K;
  row[k] = dz * w;
  for (int l = 0; l < sc.sp_level; ++l) {
    float s, co;
    sincosf(dz * sc.freq[l], &s, &co);
    row[(1 + 2 * l) * K + k] = s * w;
    row[(2 + 2 * l) * K + k] = co * w;
  }
}

__device__ __forceinline__ void to_camera(const DevScene& sc, int v, const float p[3], float c[3]) {
  const float* E = sc.E[v];
  c[0] = E[0] * p[0] + E[1] * p[1] + E[2] * p[2] + E[3];
  c[1] = E[4] * p[0] + E[5] * p[1] + E[6] * p[2] + E[7];
  c[2] = E[8] * p[0] + E[9] * p[1] + E[10] * p[2] + E[11];
}

// [unit(dir - dir_src), dir . dir_src], reference src/model.py:825-832.
__device__ __forceinline__ void ray_diff(const DevScene& sc, int v, const float p[3], const float d[3], float rd[4]) {
  float r[3] = {p[0] - sc.C[v][0], p[1] - sc.C[v][1], p[2] - sc.C[v][2]};
  float n = fmaxf(sqrtf(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]), 1e-12f);
  r[0] /= n; r[1] /= n; r[2] /= n;
  float e[3] = {d[0] - r[0], d[1] - r[1], d[2] - r[2]};
  float en = fmaxf(sqrtf(e[0] * e[0] + e[1] * e[1] + e[2] * e[2]), 1e-6f);
  rd[0] = e[0] / en; rd[1] = e[1] / en; rd[2] = e[2] / en;
  rd[3] = r[0] * d[0] + r[1] * d[1] + r[2] * d[2];
}

}  // namespace kpn
