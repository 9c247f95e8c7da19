// Ray-march kernels, engine 1: fp32 SIMT ("parity anchor").
//
// Stages (reference src/model.py:1018-1096 for the eval branch of batch_render_pifu_nerf):
//   pack_nhwc      feature maps NCHW -> channel-last atlases (once per scene)
//   prep_*         derived camera constants on device (no host sync)
//   camera_rays    pixel lattice -> rays (origin, direction, near/far before the bbox clip)
//   front          one kernel per pass: rays -> bbox clip, depths, per-sample validity (frustum + foreground in every view),
//                  ray-ordered compacted work list
//   compact        the same validity test + compaction for explicit points (KeypointNeRF.query)
//   shade_simt     per-sample gather + keypoint encoding + MLPs for tiles of 64 valid samples
//   composite      alpha compositing along the ray over the compact per-sample records
//   resample       inverse-CDF resampling + merge with the coarse depths (warp per ray)
#include <algorithm>
#include <atomic>
#include "kpn_launch.h"
#include "kpn_simt.cuh"

namespace kpn {

// ------------------------------------------------------------------------------------------------
// scene packing
// ------------------------------------------------------------------------------------------------
// in (V,C,H,W) fp32 -> out [V][H][W][Cp] fp32, Cp >= C zero padded.
__global__ void pack_nhwc_f32_kernel(const float* __restrict__ in, float* __restrict__ out, int V, int C, int H, int W, int Cp) {
  long long n = (long long)V * H * W * Cp;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % Cp);
    long long t = i / Cp;
    int x = (int)(t % W); t /= W;
    int y = (int)(t % H);
    int v = (int)(t / H);
    out[i] = c < C ? in[(((long long)v * C + c) * H + y) * W + x] : 0.0f;
  }
}

__device__ void invert_n(double* a, double* inv, int n) {
  // Gauss-Jordan with partial pivoting on an n x n (n <= 4) row-major matrix.
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < n; ++j) inv[i * n + j] = (i == j) ? 1.0 : 0.0;
  for (int c = 0; c < n; ++c) {
    int piv = c;
    double best = fabs(a[c * n + c]);
    for (int r = c + 1; r < n; ++r)
      if (fabs(a[r * n + c]) > best) { best = fabs(a[r * n + c]); piv = r; }
    if (piv != c)
      for (int j = 0; j < n; ++j) {
        double t = a[c * n + j]; a[c * n + j] = a[piv * n + j]; a[piv * n + j] = t;
        t = inv[c * n + j]; inv[c * n + j] = inv[piv * n + j]; inv[piv * n + j] = t;
      }
    double d = 1.0 / a[c * n + c];
    for (int j = 0; j < n; ++j) { a[c * n + j] *= d; inv[c * n + j] *= d; }
    for (int r = 0; r < n; ++r)
      if (r != c) {
        double f = a[r * n + c];
        for (int j = 0; j < n; ++j) { a[r * n + j] -= f * a[c * n + j]; inv[r * n + j] -= f * inv[c * n + j]; }
      }
  }
}

__global__ void prep_scene_kernel(const RawScene* __restrict__ raw, DevScene* sc) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  for (int v = 0; v < sc->V; ++v) {
    for (int i = 0; i < 12; ++i) { sc->P[v][i] = raw->KRT[v * 16 + i]; sc->E[v][i] = raw->extrin[v * 16 + i]; }
    double a[16], inv[16];
    for (int i = 0; i < 16; ++i) a[i] = (double)raw->KRT[v * 16 + i];
    invert_n(a, inv, 4);
    for (int i = 0; i < 3; ++i) sc->C[v][i] = (float)inv[i * 4 + 3];
    for (int k = 0; k < sc->K; ++k) {
      const float* p = raw->kpt3d + 3 * k;
      const float* E = sc->E[v];
      for (int i = 0; i < 3; ++i) sc->kc[v][k][i] = E[4 * i] * p[0] + E[4 * i + 1] * p[1] + E[4 * i + 2] * p[2] + E[4 * i + 3];
    }
  }
  for (int i = 0; i < 3; ++i) { sc->bounds[i] = raw->bounds[i] - 0.01f; sc->bounds[3 + i] = raw->bounds[3 + i] + 0.01f; }
  for (int v = 0; v < MAXV; ++v) { sc->fgbox[v][0] = 1 << 30; sc->fgbox[v][1] = -1; sc->fgbox[v][2] = 1 << 30; sc->fgbox[v][3] = -1; }
}

// Bounding box of the non-zero foreground texels of every view (grid: 64 row slices x V views; block reduce, 4 global atomics).
__global__ void __launch_bounds__(256)
fg_box_kernel(DevScene* sc) {
  const int v = blockIdx.y;
  const int W = sc->fg.W, H = sc->fg.H;
  const uint8_t* b = (const uint8_t*)sc->fg.ptr + (size_t)v * W * H;
  int x0 = 1 << 30, x1 = -1, y0 = 1 << 30, y1 = -1;
  for (int y = blockIdx.x; y < H; y += gridDim.x) {
    const uint8_t* row = b + (size_t)y * W;
    bool any = false;
    for (int x = threadIdx.x; x < W; x += blockDim.x)
      if (row[x]) { x0 = min(x0, x); x1 = max(x1, x); any = true; }
    if (any) { y0 = min(y0, y); y1 = max(y1, y); }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    x0 = min(x0, __shfl_xor_sync(0xffffffffu, x0, d)); x1 = max(x1, __shfl_xor_sync(0xffffffffu, x1, d));
    y0 = min(y0, __shfl_xor_sync(0xffffffffu, y0, d)); y1 = max(y1, __shfl_xor_sync(0xffffffffu, y1, d));
  }
  if ((threadIdx.x & 31) == 0 && x1 >= 0) {
    atomicMin(&sc->fgbox[v][0], x0); atomicMax(&sc->fgbox[v][1], x1); atomicMin(&sc->fgbox[v][2], y0); atomicMax(&sc->fgbox[v][3], y1);
  }
}

// Per-view window of normalised image coordinates outside of which no sample can be valid: the frustum test's +-1.01
// (reference src/model.py:725-729) intersected with the foreground bounding box dilated by the bilinear footprint (a look-up
// > 0.1 needs a non-zero texel among its 4 taps, reference src/model.py:737-739) plus 1.5 texels of slack for round-off.  A box
// that touches a border stays open on that side: border padding clamps the look-up onto the border texel.
__device__ void fg_windows(const DevScene& sc, float win[MAXV][4]) {
  const float lo = -1.0f - 1e-2f, hi = 1.0f + 1e-2f;
  for (int v = 0; v < sc.V; ++v) {
    float* w = win[v];
    w[0] = lo; w[1] = hi; w[2] = lo; w[3] = hi;
    if (!sc.use_fg) continue;
    const int W = sc.fg.W, H = sc.fg.H;
    const int* bx = sc.fgbox[v];
    if (bx[1] < 0) { w[0] = 2.0f; w[1] = -2.0f; w[2] = 2.0f; w[3] = -2.0f; continue; }   // empty mask: nothing is valid
    const float slack = 2.5f;   // 1 texel of bilinear footprint + 1.5 of round-off slack
    if (bx[0] > 0 && W > 1) w[0] = fmaxf(lo, 2.0f * ((float)bx[0] - slack) / (float)(W - 1) - 1.0f);
    if (bx[1] < W - 1 && W > 1) w[1] = fminf(hi, 2.0f * ((float)bx[1] + slack) / (float)(W - 1) - 1.0f);
    if (bx[2] > 0 && H > 1) w[2] = fmaxf(lo, 2.0f * ((float)bx[2] - slack) / (float)(H - 1) - 1.0f);
    if (bx[3] < H - 1 && H > 1) w[3] = fminf(hi, 2.0f * ((float)bx[3] + slack) / (float)(H - 1) - 1.0f);
  }
}

// raw: the target camera (nullptr: leave the camera fields alone); sc: the bound scene whose foreground windows ray_interval
// reads (nullptr: no scene, the windows are left alone).
__global__ void prep_target_kernel(const RawTarget* __restrict__ raw, DevTarget* tg, const DevScene* __restrict__ sc) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  if (sc) fg_windows(*sc, tg->win);
  if (!raw) return;
  double a[9], inv[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) a[i * 3 + j] = (double)raw->K[i * 4 + j];
  invert_n(a, inv, 3);
  for (int i = 0; i < 9; ++i) tg->invK[i] = (float)inv[i];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) tg->R[i * 3 + j] = raw->RT[i * 4 + j];
  for (int j = 0; j < 3; ++j) {
    float s = 0.0f;
    for (int i = 0; i < 3; ++i) s += raw->RT[i * 4 + 3] * raw->RT[i * 4 + j];
    tg->o[j] = -s;
  }
}

// ------------------------------------------------------------------------------------------------
// rays (reference src/model.py:1018-1043, 1178-1237)
// ------------------------------------------------------------------------------------------------
// The ray of lattice pixel (px, py): origin, unit direction and the near/far distances of the znear / zfar planes along it,
// before the bounding-box clip (reference src/model.py:1026-1036).
__device__ __forceinline__ void camera_ray(const DevTarget& tg, float px, float py, float o[3], float d[3], float& n_r, float& f_r) {
  const float* iK = tg.invK;
  float dc[3], gn[3], gf[3];
  for (int i = 0; i < 3; ++i) {
    dc[i] = iK[i * 3 + 0] * px + iK[i * 3 + 1] * py + iK[i * 3 + 2];
    gn[i] = iK[i * 3 + 0] * (tg.znear * px) + iK[i * 3 + 1] * (tg.znear * py) + iK[i * 3 + 2] * tg.znear;
    gf[i] = iK[i * 3 + 0] * (tg.zfar * px) + iK[i * 3 + 1] * (tg.zfar * py) + iK[i * 3 + 2] * tg.zfar;
  }
  n_r = sqrtf(gn[0] * gn[0] + gn[1] * gn[1] + gn[2] * gn[2]);
  f_r = sqrtf(gf[0] * gf[0] + gf[1] * gf[1] + gf[2] * gf[2]);
  float w[3];
  for (int j = 0; j < 3; ++j) w[j] = dc[0] * tg.R[j] + dc[1] * tg.R[3 + j] + dc[2] * tg.R[6 + j];
  float nn = fmaxf(sqrtf(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]), 1e-12f);
  d[0] = w[0] / nn; d[1] = w[1] / nn; d[2] = w[2] / nn;
  o[0] = tg.o[0]; o[1] = tg.o[1]; o[2] = tg.o[2];
}

// Tightens a ray's near/far to its bounding-box interval: slab test with the "exactly two face hits" rule, from the ray's own
// origin (reference src/model.py:1039-1043, 1178-1237).
__device__ __forceinline__ void bbox_clip(const DevScene& sc, const float o[3], const float d[3], float& n_r, float& f_r) {
  float dd[3];
  for (int i = 0; i < 3; ++i) dd[i] = fabsf(d[i]) < 1e-5f ? 1e-5f : d[i];
  float ddn = sqrtf(dd[0] * dd[0] + dd[1] * dd[1] + dd[2] * dd[2]);
  const float* b = sc.bounds;
  const float eps = 1e-6f;
  int cnt = 0;
  float tn = 3.0e38f, tf = -3.0e38f;
  for (int f = 0; f < 6; ++f) {
    int ax = f % 3;
    float t = (b[f] - o[ax]) / dd[ax];
    float p[3] = {t * dd[0] + o[0], t * dd[1] + o[1], t * dd[2] + o[2]};
    bool in = p[0] >= b[0] - eps && p[0] <= b[3] + eps && p[1] >= b[1] - eps && p[1] <= b[4] + eps &&
              p[2] >= b[2] - eps && p[2] <= b[5] + eps;
    if (in) {
      float e[3] = {p[0] - o[0], p[1] - o[1], p[2] - o[2]};
      float dist = sqrtf(e[0] * e[0] + e[1] * e[1] + e[2] * e[2]) / ddn;
      tn = fminf(tn, dist); tf = fmaxf(tf, dist);
      ++cnt;
    }
  }
  bool hit = cnt == 2;
  if (hit && tn > n_r) n_r = tn;
  if (hit && tf < f_r) f_r = tf;
}

// Rays of lattice pixels r0 .. r0 + n - 1 (pixel r = j*nx + i): o, d (n,3), near/far (n,2) before the bounding-box clip.  One
// thread per ray and no loop: a grid-stride loop lets the compiler hoist the loop-invariant products (iK[.][2] * znear, ...) out of
// it, and a product hoisted out of the block of its sum is no longer fused into an FMA, which changes the rays' last bits.
__global__ void camera_rays_kernel(const DevTarget* __restrict__ tgp, long long r0, long long n, float* __restrict__ o,
                                   float* __restrict__ d, float* __restrict__ nf) {
  const DevTarget& tg = *tgp;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long r = r0 + i;
  const int ix = (int)(r % tg.nx), iy = (int)(r / tg.nx);
  float oo[3], dd[3], n_r, f_r;
  camera_ray(tg, (float)(tg.x0 + tg.step * ix), (float)(tg.y0 + tg.step_y * iy), oo, dd, n_r, f_r);
  o[3 * i + 0] = oo[0]; o[3 * i + 1] = oo[1]; o[3 * i + 2] = oo[2];
  d[3 * i + 0] = dd[0]; d[3 * i + 1] = dd[1]; d[3 * i + 2] = dd[2];
  nf[2 * i + 0] = n_r; nf[2 * i + 1] = f_r;
}

// ------------------------------------------------------------------------------------------------
// front end of a render pass: rays + depths + validity + ray-ordered compaction in ONE kernel
// ------------------------------------------------------------------------------------------------
// One warp per ray, 8 rays per block iteration.  The chunk's rays come in as origins / directions (ray_o, ray_d) and, for the
// coarse pass (zbuf == nullptr), near/far before the bounding-box clip (nf_in): the warp clips them with the ray's own origin
// and stores the clipped near/far in ray_nf; the coarse depths are the uniform ones and are never stored (every consumer
// recomputes them with coarse_depth()).  Fine pass: the depths come from zbuf (R, S).  Lane l tests samples l, l+32, ..
// (3 projections + frustum + foreground lookups, reference src/model.py:713-739); the ballots give the ray's valid samples in
// order.  The 8 rays of a block iteration reserve ONE contiguous range of the work list with one atomicAdd; inside it the
// entries are ordered by (ray, sample), so that ray r owns list[ray_start[r] .. +ray_cnt[r]) -- the compositing pass walks
// exactly that range, and nothing is ever written for the invalid samples.
// Early-ray termination (ert.s_hi > 0): only samples s_lo <= s < s_hi are looked at; a ray whose accumulated alpha of the
// earlier segment leaves a transmittance < ert.eps contributes no entries (what it could still add is < eps per channel).
// Depth interval [zlo, zhi] of a ray outside of which no sample can be valid: every view contributes the half-lines
// c0 + z c1 >= 0 of "depth >= znear" and of its window's four sides (h = P (o + z d) is linear in z; h_z > 0 wherever the
// first one holds, so the sides multiply through).  Conservative: the windows carry slack, znear a margin; samples inside the
// interval still take the exact test.
__device__ __forceinline__ void ray_interval(const DevScene& sc, const DevTarget& tg, const float o[3], const float d[3], float& zlo,
                                             float& zhi) {
  zlo = -3.0e38f; zhi = 3.0e38f;
  if (sc.znear - 1e-3f <= 0.0f) return;   // the sides below assume a positive camera depth wherever "depth >= znear" holds
  bool empty = false;
  auto side = [&](float c0, float c1) {
    if (c1 > 0.0f) zlo = fmaxf(zlo, -c0 / c1);
    else if (c1 < 0.0f) zhi = fminf(zhi, -c0 / c1);
    else if (c0 < 0.0f) empty = true;
  };
  for (int v = 0; v < sc.V; ++v) {
    const float* P = sc.P[v];
    float a[3], b[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      a[i] = P[4 * i] * o[0] + P[4 * i + 1] * o[1] + P[4 * i + 2] * o[2] + P[4 * i + 3];
      b[i] = P[4 * i] * d[0] + P[4 * i + 1] * d[1] + P[4 * i + 2] * d[2];
    }
    const float sl = 1e-3f * (fabsf(a[2]) + fabsf(b[2]) * 8.0f + 1.0f);   // absolute slack on the linear forms
    side(a[2] - (sc.znear - 1e-3f), b[2]);
    const float xl = (tg.win[v][0] + 1.0f) * 0.5f * sc.wm1, xh = (tg.win[v][1] + 1.0f) * 0.5f * sc.wm1;
    const float yl = (tg.win[v][2] + 1.0f) * 0.5f * sc.hm1, yh = (tg.win[v][3] + 1.0f) * 0.5f * sc.hm1;
    if (xl > xh || yl > yh) empty = true;
    side(a[0] - xl * a[2] + sl * fmaxf(1.0f, fabsf(xl)), b[0] - xl * b[2]);
    side(xh * a[2] - a[0] + sl * fmaxf(1.0f, fabsf(xh)), xh * b[2] - b[0]);
    side(a[1] - yl * a[2] + sl * fmaxf(1.0f, fabsf(yl)), b[1] - yl * b[2]);
    side(yh * a[2] - a[1] + sl * fmaxf(1.0f, fabsf(yh)), yh * b[2] - b[1]);
  }
  if (empty) { zlo = 3.0e38f; zhi = -3.0e38f; }
  else { const float m = 1e-4f * (1.0f + fabsf(zlo) + fabsf(zhi)); zlo -= m; zhi += m; }   // round-off of the divisions
}

constexpr int FRONT_WARPS = 8;
constexpr int FRONT_THREADS = FRONT_WARPS * 32;
constexpr int FRONT_MASKW = 2048;   // ballot words of one batch of rays held in shared memory (8 KB)
constexpr int FRONT_MAXW = 40;      // ballot words per ray: up to 1280 samples (256 coarse + 1024 fine)

struct FrontRay { float o[3], d[3], n, f, zlo, zhi; int wa, wb; };   // per ray of a batch: origin, direction, near/far, interval, word range

__global__ void __launch_bounds__(FRONT_THREADS, 4)
front_kernel(const DevScene* __restrict__ scp, const DevTarget* __restrict__ tgp, int nr, int S, const float* __restrict__ zbuf,
             const float* __restrict__ ray_o, const float* __restrict__ ray_d, const float* __restrict__ nf_in, float* __restrict__ ray_nf,
             int* __restrict__ list, int list_base, int* __restrict__ counter, int* __restrict__ ray_start,
             int* __restrict__ ray_cnt, ErtSegment ert) {
  const DevScene& sc = *scp;
  const DevTarget& tg = *tgp;
  __shared__ FrontRay s_ray[FRONT_THREADS];
  __shared__ unsigned s_mask[FRONT_MASKW];
  __shared__ int s_cnt[FRONT_THREADS];     // per ray: valid samples, then (after the scan) exclusive offset inside the batch
  __shared__ int s_wsum[FRONT_WARPS];
  __shared__ int s_base;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int nwords = (S + 31) >> 5;
  // rays per batch: as many as a block has threads, fewer when their ballot words would not fit (very long rays)
  const int batch = min(FRONT_THREADS, (FRONT_MASKW / nwords) & ~31);
  const int s_lo = ert.s_hi > 0 ? ert.s_lo : 0, s_hi = ert.s_hi > 0 ? ert.s_hi : S;
  for (int base = blockIdx.x * batch; base < nr; base += gridDim.x * batch) {   // block-uniform trip count
    // ---- phase A, one THREAD per ray: the ray, its clipped near/far, the depth interval outside of which nothing can be valid, and the
    //      range of 32-sample words that can intersect it (uniform depths are monotone in the sample index)
    if (threadIdx.x < batch) {
      const int i = base + threadIdx.x;
      FrontRay fr;
      fr.wa = 0; fr.wb = 0;
      if (i < nr) {
        fr.o[0] = ray_o[3 * i + 0]; fr.o[1] = ray_o[3 * i + 1]; fr.o[2] = ray_o[3 * i + 2];
        fr.d[0] = ray_d[3 * i + 0]; fr.d[1] = ray_d[3 * i + 1]; fr.d[2] = ray_d[3 * i + 2];
        if (zbuf == nullptr) {
          fr.n = nf_in[2 * i + 0]; fr.f = nf_in[2 * i + 1];
          bbox_clip(sc, fr.o, fr.d, fr.n, fr.f);
          ray_nf[2 * i + 0] = fr.n; ray_nf[2 * i + 1] = fr.f;
        } else {
          fr.n = 0.0f; fr.f = 0.0f;
        }
        ray_interval(sc, tg, fr.o, fr.d, fr.zlo, fr.zhi);
        const bool dead = ert.ray_alpha != nullptr && 1.0f - ert.ray_alpha[i] < ert.eps;   // ray already opaque
        if (!dead && fr.zlo <= fr.zhi) {
          int sa = s_lo, sb = s_hi;
          if (zbuf == nullptr && S > 1 && fr.f != fr.n) {
            // z(s) = n + (f - n) s / (S - 1): samples with z in [zlo, zhi] have s in [ta, tb] (one sample of slack either side)
            const float k = (float)(S - 1) / (fr.f - fr.n);
            float ta = (fr.zlo - fr.n) * k, tb = (fr.zhi - fr.n) * k;
            if (ta > tb) { const float t = ta; ta = tb; tb = t; }
            if (ta == ta && tb == tb) {   // (NaN: a degenerate near == far up to round-off; keep the whole ray)
              sa = max(sa, (int)fminf(fmaxf(floorf(ta) - 1.0f, 0.0f), (float)S));
              sb = min(sb, (int)fminf(fmaxf(ceilf(tb) + 2.0f, 0.0f), (float)S));
            }
          }
          if (sa < sb) { fr.wa = sa >> 5; fr.wb = (sb + 31) >> 5; }
        }
      }
      s_ray[threadIdx.x] = fr;
      s_cnt[threadIdx.x] = 0;
    }
    __syncthreads();
    // ---- phase B, one WARP per ray (round robin over the batch): the exact validity test of the samples in the word range,
    //      lane l takes samples l, l+32, ..; ballots -> the ray's valid samples in order
    for (int t = wid; t < batch; t += FRONT_WARPS) {
      const FrontRay& fr = s_ray[t];
      const int i = base + t;
      unsigned* mw = s_mask + t * nwords;
      int cnt = 0;
      for (int w = 0; w < nwords; ++w) {
        unsigned m = 0u;
        if (w >= fr.wa && w < fr.wb) {
          const int s = 32 * w + lane;
          bool ok = false;
          if (s < S && s >= s_lo && s < s_hi) {
            const float z = zbuf ? zbuf[(long long)i * S + s] : coarse_depth(fr.n, fr.f, s, S);
            if (z >= fr.zlo && z <= fr.zhi) {   // outside the ray's interval no view can accept the sample
              const float p[3] = {fr.o[0] + fr.d[0] * z, fr.o[1] + fr.d[1] * z, fr.o[2] + fr.d[2] * z};   // reference src/model.py:1057
              Proj q[MAXV];
              ok = sample_valid(sc, p, q);
            }
          }
          m = __ballot_sync(0xffffffffu, ok);
          cnt += __popc(m);
        }
        if (lane == 0) mw[w] = m;
      }
      if (lane == 0) s_cnt[t] = cnt;
    }
    __syncthreads();
    // ---- block scan of the batch's per-ray counts, ONE atomic reserves the batch's contiguous range of the work list
    {
      const int c = threadIdx.x < batch ? s_cnt[threadIdx.x] : 0;
      int v = c;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, v, d);
        if (lane >= d) v += u;
      }
      if (lane == 31) s_wsum[wid] = v;
      __syncthreads();
      if (threadIdx.x == 0) {
        int tot = 0;
#pragma unroll
        for (int w = 0; w < FRONT_WARPS; ++w) { const int x = s_wsum[w]; s_wsum[w] = tot; tot += x; }
        s_base = tot ? atomicAdd(counter, tot) : 0;
      }
      __syncthreads();
      if (threadIdx.x < batch) {
        const int off = s_wsum[wid] + v - c;   // exclusive offset of this ray inside the batch
        s_cnt[threadIdx.x] = off;
        const int i = base + threadIdx.x;
        if (i < nr) { ray_start[i] = list_base + s_base + off; ray_cnt[i] = c; }
      }
    }
    __syncthreads();
    // ---- the entries, ordered by (ray, sample)
    for (int t = wid; t < batch; t += FRONT_WARPS) {
      const int i = base + t;
      if (i >= nr) break;
      const FrontRay& fr = s_ray[t];
      const unsigned* mw = s_mask + t * nwords;
      int pos = list_base + s_base + s_cnt[t];
      for (int w = fr.wa; w < fr.wb; ++w) {
        const unsigned m = mw[w];
        if ((m >> lane) & 1u) list[pos + __popc(m & ((1u << lane) - 1u))] = i * S + 32 * w + lane;
        pos += __popc(m);
      }
    }
    __syncthreads();   // the shared arrays are rewritten by the next batch
  }
}

// ------------------------------------------------------------------------------------------------
// validity + compaction of explicit points (KeypointNeRF.query)
// ------------------------------------------------------------------------------------------------
// out: out_w floats per point (5: query, 2: geometry-only query), zeroed on invalid rows
__global__ void compact_kernel(const DevScene* __restrict__ sc, SampleSrc src, long long n, int* __restrict__ list,
                               int* __restrict__ counter, float* __restrict__ out, int out_w, uint8_t* __restrict__ valid_out) {
  const DevScene& S = *sc;
  __shared__ int s_cnt[8];
  __shared__ int s_base;
  for (long long base = (blockIdx.x * (long long)blockDim.x) ; base < n; base += (long long)gridDim.x * blockDim.x) {   // block-uniform trip count
    long long i = base + threadIdx.x;
    bool ok = false;
    if (i < n) {
      float p[3], d[3];
      Proj q[MAXV];
      fetch_sample<true>(src, i, p, d);
      ok = sample_valid(S, p, q);
      if (!ok) {   // rows with valid == 0 carry zeros (the reference multiplies them by a zero mask downstream)
        float* o = out + out_w * i;
        for (int c = 0; c < out_w; ++c) o[c] = 0.f;
      }
      if (valid_out) valid_out[i] = ok ? 1 : 0;
    }
    // block-aggregated append: one atomic per 256 samples instead of one per warp (the single counter serialises in L2)
    const unsigned m = __ballot_sync(0xffffffffu, ok);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (lane == 0) s_cnt[wid] = __popc(m);
    __syncthreads();
    if (threadIdx.x == 0) {
      int tot = 0;
#pragma unroll
      for (int w = 0; w < 8; ++w) { int c = s_cnt[w]; s_cnt[w] = tot; tot += c; }
      s_base = tot ? atomicAdd(counter, tot) : 0;
    }
    __syncthreads();
    if (ok) list[s_base + s_cnt[wid] + __popc(m & ((1u << lane) - 1u))] = (int)i;
    __syncthreads();   // s_cnt / s_base are rewritten by the next iteration
  }
}

// ------------------------------------------------------------------------------------------------
// shade (fp32 SIMT): tiles of TS valid samples, 4 TS threads.  The view-indexed shared arrays hold NV views: up to 3 views in
// tiles of 64 samples, 4 views in tiles of 56 (64 samples x 4 views would need 253 952 B of shared memory).  A sample's
// arithmetic does not depend on the tile it sits in.
// ------------------------------------------------------------------------------------------------
struct ShadeSmem {
  float* A;     // [TS][LDA]
  float* B;     // [TS][LDB]
  float* XV;    // [NV][TS][64]   (later scratch S1,S2,S3)
  float* F;     // [NV][TS][36]
  float* MV;    // [TS][72]
  float* Lat;   // [TS][24]
  float* RD;    // [NV][TS][4]
  float* RGB;   // [NV][TS][4]
  float* UV;    // [NV][TS][4]  u, v, zn, boundary weight
  float* PW;    // [NV][TS]
  float* Om;    // [NV][TS]
  float* P;     // [TS][8]  p xyz, d xyz
  float* F8;    // [TS][8]
  float* Geo;   // [TS][2]
  float* Vis;   // [TS]
  float* Logit; // [NV][TS]
  int* Id;      // [TS]
};

__host__ __device__ constexpr int shade_smem_floats(int NV, int TS) {
  return TS * LDA + TS * LDB + NV * TS * 64 + NV * TS * 36 + TS * 72 + TS * 24 + NV * TS * 4 * 3 + NV * TS * 2 + TS * 8 * 2 +
         TS * 2 + TS + NV * TS + TS;
}
template <int NV, int TS>
constexpr size_t SHADE_SMEM_BYTES = shade_smem_floats(NV, TS) * sizeof(float);
static_assert(SHADE_SMEM_BYTES<3, 64> <= 227u * 1024u && SHADE_SMEM_BYTES<4, 56> <= 227u * 1024u, "fp32 engine tiles");
static_assert(MAXV == 4, "the fp32 engine's tiles cover up to 4 views");

template <int NV, int TS>
__global__ void __launch_bounds__(4 * TS, 1)
shade_simt_kernel(const DevScene* __restrict__ scp, const DevWeightsF32* __restrict__ Wp, SampleSrc src,
                  const int* __restrict__ list, const int* __restrict__ count_ptr, int query_mode, ShadeOut so) {
  constexpr int NT = 4 * TS;
  extern __shared__ float4 smem4[];
  float* sm = reinterpret_cast<float*>(smem4);
  ShadeSmem s;
  s.A = sm; sm += TS * LDA;
  s.B = sm; sm += TS * LDB;
  s.XV = sm; sm += NV * TS * 64;
  s.F = sm; sm += NV * TS * 36;
  s.MV = sm; sm += TS * 72;
  s.Lat = sm; sm += TS * 24;
  s.RD = sm; sm += NV * TS * 4;
  s.RGB = sm; sm += NV * TS * 4;
  s.UV = sm; sm += NV * TS * 4;
  s.PW = sm; sm += NV * TS;
  s.Om = sm; sm += NV * TS;
  s.P = sm; sm += TS * 8;
  s.F8 = sm; sm += TS * 8;
  s.Geo = sm; sm += TS * 2;
  s.Vis = sm; sm += TS;
  s.Logit = sm; sm += NV * TS;
  s.Id = reinterpret_cast<int*>(sm);
  float* S1 = s.XV;
  float* S2 = s.XV + TS * 64;
  float* S3 = s.XV + 2 * TS * 64;

  const DevScene& sc = *scp;
  const DevWeightsF32& W = *Wp;
  const int t = threadIdx.x;
  const int V = sc.V, K = sc.K;
  const int encd = (1 + 2 * sc.sp_level) * K;
  const int count = *count_ptr;

  for (int tile = blockIdx.x; tile * TS < count; tile += gridDim.x) {
    const int base = tile * TS;
    const int nrows = min(TS, count - base);
    // ---- 1. fetch the tile's samples, projections and view weights
    load_tile<TS>(sc, V, src, list, base, nrows, s.Id, s.P, s.UV, s.PW);
    // ---- 2. per-view geometry MLP; layer 0's input is still live in A after layer 1, so the feat8 taps wait in F8
    for (int v = 0; v < V; ++v) {
      geo_input<TS>(sc, v, K, encd, s.UV, s.P, {s.A, LDA}, {s.F8, 8});
      __syncthreads();
      dense_tile<ACT_SP, 4>(W, L_GEO0, s.A, LDA, s.B, LDB);
      __syncthreads();
      dense_tile<ACT_SP, 4>(W, L_GEO1, s.B, LDB, s.A, LDA);
      for (int idx = t; idx < TS * 8; idx += NT) s.A[(idx >> 3) * LDA + 128 + (idx & 7)] = s.F8[idx];
      __syncthreads();
      dense_tile<ACT_SP, 4>(W, L_GEO2, s.A, LDA, s.B, LDB);
      __syncthreads();
      dense_tile<ACT_NONE, 2>(W, L_GEO3, s.B, LDB, s.XV + v * TS * 64, 64);
      __syncthreads();
    }
    // ---- 3. pooling over views, density head
    pool_geometry<TS>(V, s.PW, s.XV, {s.A, LDA});
    __syncthreads();
    if (query_mode != 2) dense_tile<ACT_NONE, 1>(W, L_CMP, s.A, LDA, s.Lat, 24);   // ibr_compress_gfeat (src/model.py:819)
    density_hidden<TS>(W, {s.A, LDA}, {s.B, LDB}, {s.A, LDA});
    dense_tile<ACT_NONE, 1>(W, L_DEN2, s.A, LDA, s.Geo, 2);
    if (query_mode == 2) {   // geometry only: [sdf_raw, rad], no colour stages
      __syncthreads();
      if (t < nrows) reinterpret_cast<float2*>(so.out2)[s.Id[t]] = make_float2(s.Geo[t * 2], s.Geo[t * 2 + 1]);
      __syncthreads();
      continue;
    }
    // ---- 4. colour branch inputs, ray encoding, blending weights, pooling over views
    colour_inputs<TS>(sc, V, s.UV, s.P, s.Lat, s.F, s.RGB, s.RD);
    add_ray_encoding<TS>(W, V, s.RD, {s.B, LDB}, {s.A, LDA}, s.F);
    blend_weights<TS>(W, V, s.RD, s.Om);
    __syncthreads();
    pool_colour<TS>(V, s.F, s.Om, s.MV);
    __syncthreads();
    // ---- 5. per-view IBR head
    for (int v = 0; v < V; ++v) {
      // the activations in place in S1-S3 (see colour_head)
      colour_head<TS>(W, v, s.MV, s.F, s.Om, s.RD,
                      {{s.A, LDA}, {s.B, LDB}, {S1, 64}, {S2, 64}, {S3, 64}, {S2, 64}, {S1, 64}, {S3, 64}, {S2, 64}, {s.Vis, 1},
                       {S3, 64}, {S2, 64}, {S3, 64}});
      dense_tile<ACT_NONE, 1>(W, L_OUT2, S3, 64, s.Logit + v * TS, 1);
      __syncthreads();
    }
    // ---- 6. softmax blend of the source colours and output (src/model.py:1300-1301, 978-997)
    if (t < nrows) {
      float e[MAXV], rgb[3];
      const float den = blend_colours<TS>(V, s.Logit, s.RGB, t, e, rgb);
      float g0 = s.Geo[t * 2], rad = s.Geo[t * 2 + 1];
      if (query_mode) {
        float* o = so.out5 + 5ll * s.Id[t];
        o[0] = g0; o[1] = rad; o[2] = rgb[0] / den; o[3] = rgb[1] / den; o[4] = rgb[2] / den;
      } else {   // eval_func (reference src/model.py:978-997): alpha = relu(rad), compact record at the sample's list position
        const long long pos = (long long)so.list_base + base + t;
        so.ao[pos] = make_float2(fmaxf(rad, 0.0f), g0);
        float* o = so.rgb + 3 * pos;
        o[0] = rgb[0] / den; o[1] = rgb[1] / den; o[2] = rgb[2] / den;
      }
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------
// compositing (reference src/model.py:1150-1176) over the compact per-ray records
// ------------------------------------------------------------------------------------------------
// One WARP per ray walks the ray's range(s) of the work list in sample order: lane l takes entries l, l+32, ... (coalesced),
// the transmittance T_k = prod_{j<k} (1 - a_j) is an exclusive product scan across the lanes carried from one group of 32
// entries to the next (invalid samples have a = 0, i.e. a factor of exactly 1, and are simply not there), the ray sums are
// warp reductions.  Depths: zbuf (fine pass) or recomputed uniform depths (coarse pass).  dist of the ray's last sample is
// 1e10 (reference src/model.py:1166).  Optional outputs: cw[e] = compositing weight of list entry e (input of the
// resampling pass), ray_alpha = accumulated alpha of the segments walked (early-ray termination).
struct RaySeg { const int* start; const int* cnt; };

__global__ void __launch_bounds__(128)
composite_kernel(const int* __restrict__ list, const float2* __restrict__ ao, const float* __restrict__ rgb, RaySeg seg0,
                 RaySeg seg1, int nseg, const float* __restrict__ zbuf, const float* __restrict__ ray_nf, int r0, int nr, int S,
                 long long plane, float* __restrict__ color, float* __restrict__ depth, float* __restrict__ alpha,
                 float* __restrict__ sdf, float* __restrict__ ray_alpha, float* __restrict__ cw) {
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  for (int i = blockIdx.x * wpb + (threadIdx.x >> 5); i < nr; i += gridDim.x * wpb) {
    const float* zz = zbuf ? zbuf + (long long)i * S : nullptr;
    const float n_r = zbuf ? 0.0f : ray_nf[2 * i], f_r = zbuf ? 0.0f : ray_nf[2 * i + 1];
    float Tc = 1.0f;   // transmittance in front of this group of 32 entries
    float acc = 0.0f, cr = 0.0f, cg = 0.0f, cb = 0.0f, cd = 0.0f, cs = 0.0f;
    for (int sg = 0; sg < nseg; ++sg) {
      const RaySeg& sgm = sg == 0 ? seg0 : seg1;
      const int start = sgm.start[i], cnt = sgm.cnt[i];
      for (int e0 = 0; e0 < cnt; e0 += 32) {
        const int e = start + e0 + lane;
        const bool live = e0 + lane < cnt;
        float a = 0.0f, zk = 0.0f, q1 = 0.0f, q2 = 0.0f, q3 = 0.0f, q4 = 0.0f;
        if (live) {
          const int k = list[e] - i * S;
          const float2 as = ao[e];
          const ListEntry en = list_entry(zz, n_r, f_r, k, S, as.x);
          zk = en.z; a = en.alpha;
          q1 = as.y;
          if (as.x > 0.0f) { q2 = rgb[3ll * e]; q3 = rgb[3ll * e + 1]; q4 = rgb[3ll * e + 2]; }   // colour exists iff alpha > 0
        }
        float T;
        const float c = composite_weight(a, lane, Tc, T);
        if (live) {
          acc += c; cr += c * q2; cg += c * q3; cb += c * q4; cd += c * zk; cs += c * q1;
          if (cw) cw[e] = c;
        }
      }
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      acc += __shfl_xor_sync(0xffffffffu, acc, d); cr += __shfl_xor_sync(0xffffffffu, cr, d); cg += __shfl_xor_sync(0xffffffffu, cg, d);
      cb += __shfl_xor_sync(0xffffffffu, cb, d); cd += __shfl_xor_sync(0xffffffffu, cd, d); cs += __shfl_xor_sync(0xffffffffu, cs, d);
    }
    if (lane == 0) {
      const long long r = r0 + i;
      if (color) { color[r] = cr; color[plane + r] = cg; color[2 * plane + r] = cb; }
      if (alpha) alpha[r] = acc;
      if (depth) depth[r] = cd / (acc + 1e-8f);
      if (sdf) sdf[r] = cs / (acc + 1e-8f);
      if (ray_alpha) ray_alpha[i] = acc;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// hierarchical resampling (reference src/model.py:1110-1148, 1072-1076), uniform=True
// ------------------------------------------------------------------------------------------------
// One WARP per ray, everything in shared memory: the ray's compositing weights are scattered from the compact records into a
// dense array (invalid samples: 0), pdf = (contrib[1:-1] + 1e-5) / sum, cdf by a warp scan, the S_f inverse-CDF samples
// (searchsorted right=True by binary search, the reference's clamp / den<1e-5 rules), then z_all = sort(cat[z, z_fine]) as a
// merge by rank (both sequences are monotone; coarse samples come first on ties).  Optional: the dense weights (debug output).
constexpr int MAX_SC = 256, MAX_SF = 1024, RES_WARPS = 4;

__device__ __forceinline__ int count_le(const float* a, int n, float x, bool rev) {   // # of a[i] <= x, a ascending (rev: descending storage)
  int lo = 0, hi = n;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (a[rev ? n - 1 - mid : mid] <= x) lo = mid + 1; else hi = mid; }
  return lo;
}
__device__ __forceinline__ int count_lt(const float* a, int n, float x, bool rev) {
  int lo = 0, hi = n;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (a[rev ? n - 1 - mid : mid] < x) lo = mid + 1; else hi = mid; }
  return lo;
}

__global__ void __launch_bounds__(RES_WARPS * 32)
resample_kernel(const int* __restrict__ list, const float* __restrict__ cw, RaySeg seg0, RaySeg seg1, int nseg,
                const float* __restrict__ ray_nf, int nr, int Sc, int Sf, float* __restrict__ zout,
                float* __restrict__ contrib_out) {
  extern __shared__ float rsm[];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int per_warp = 4 * Sc + 2 * Sf;   // cd | cdf | zc | zf | zo
  float* cd = rsm + wid * per_warp;   // dense weights [Sc]
  float* cdf = cd + Sc;               // [Sc - 1]
  float* zc = cdf + Sc;               // coarse depths [Sc]
  float* zf = zc + Sc;                // fine depths [Sf]
  float* zo = zf + Sf;                // merged [Sc + Sf]
  const unsigned FULLM = 0xffffffffu;
  for (int i = blockIdx.x * RES_WARPS + wid; i < nr; i += gridDim.x * RES_WARPS) {
    const float n_r = ray_nf[2 * i], f_r = ray_nf[2 * i + 1];
    for (int k = lane; k < Sc; k += 32) { cd[k] = 0.0f; zc[k] = coarse_depth(n_r, f_r, k, Sc); }
    __syncwarp();
    for (int sg = 0; sg < nseg; ++sg) {
      const RaySeg& sgm = sg == 0 ? seg0 : seg1;
      const int start = sgm.start[i], cnt = sgm.cnt[i];
      for (int e = lane; e < cnt; e += 32) cd[list[start + e] - i * Sc] = cw[start + e];
    }
    __syncwarp();
    if (contrib_out) for (int k = lane; k < Sc; k += 32) contrib_out[(long long)i * Sc + k] = cd[k];
    if (Sf > 0) {
      const int nb = Sc - 2;   // pdf bins = contrib[1:-1]
      const int nc = Sc - 1;   // cdf entries == z_mid entries
      float sum = 0.0f;
      for (int k = lane; k < nb; k += 32) sum += cd[k + 1] + 1e-5f;
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) sum += __shfl_xor_sync(FULLM, sum, d);
      float carry = 0.0f;
      if (lane == 0) cdf[0] = 0.0f;
      for (int k0 = 0; k0 < nb; k0 += 32) {
        const int k = k0 + lane;
        float v = k < nb ? (cd[k + 1] + 1e-5f) / sum : 0.0f;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          const float t = __shfl_up_sync(FULLM, v, d);
          if (lane >= d) v += t;
        }
        if (k < nb) cdf[k + 1] = carry + v;
        carry += __shfl_sync(FULLM, v, 31);
      }
      __syncwarp();
      for (int j = lane; j < Sf; j += 32) {
        const float u = linspace01(j, Sf);
        const int idx = count_le(cdf, nc, u, false);   // searchsorted(cdf, u, right=True)
        const int lo = max(idx - 1, 0), hi = min(idx, nc - 1);
        const float clo = cdf[lo], chi = cdf[hi];
        const float zlo = 0.5f * (zc[lo + 1] + zc[lo]), zhi = 0.5f * (zc[hi + 1] + zc[hi]);
        float den = chi - clo;
        if (den < 1e-5f) den = 1.0f;
        zf[j] = zlo + ((u - clo) / den) * (zhi - zlo);
      }
      __syncwarp();
      // merge by rank; near > far (depths running backwards, as the reference allows) flips both sequences
      const bool rev = f_r < n_r;
      for (int t = lane; t < Sc; t += 32) {
        const int tt = rev ? Sc - 1 - t : t;
        zo[t + count_lt(zf, Sf, zc[tt], rev)] = zc[tt];
      }
      for (int j = lane; j < Sf; j += 32) {
        const int jj = rev ? Sf - 1 - j : j;
        zo[j + count_le(zc, Sc, zf[jj], rev)] = zf[jj];
      }
      __syncwarp();
      for (int k = lane; k < Sc + Sf; k += 32) zout[(long long)i * (Sc + Sf) + k] = zo[k];
    }
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------------
// host launchers
// ------------------------------------------------------------------------------------------------
static inline int grid_for(long long n, int block, int cap) {
  long long g = (n + block - 1) / block;
  if (g < 1) g = 1;
  if (g > cap) g = cap;
  return (int)g;
}

cudaError_t launch_pack_nhwc_f32(const float* in, float* out, int V, int C, int H, int W, int Cp, cudaStream_t st) {
  long long n = (long long)V * H * W * Cp;
  pack_nhwc_f32_kernel<<<grid_for(n, 256, 132 * 16), 256, 0, st>>>(in, out, V, C, H, W, Cp);
  return cudaGetLastError();
}
cudaError_t launch_prep_scene(const RawScene* raw, DevScene* sc, cudaStream_t st) {
  prep_scene_kernel<<<1, 32, 0, st>>>(raw, sc);
  return cudaGetLastError();
}
cudaError_t launch_fg_box(DevScene* sc, int n_views, cudaStream_t st) {
  fg_box_kernel<<<dim3(64, n_views), 256, 0, st>>>(sc);
  return cudaGetLastError();
}
cudaError_t launch_prep_target(const RawTarget* raw, DevTarget* tg, const DevScene* sc, cudaStream_t st) {
  prep_target_kernel<<<1, 32, 0, st>>>(raw, tg, sc);
  return cudaGetLastError();
}
cudaError_t launch_camera_rays(const DevTarget* tg, long long r0, long long n, float* o, float* d, float* nf, cudaStream_t st) {
  if (n < 1) return cudaSuccess;
  camera_rays_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(tg, r0, n, o, d, nf);
  return cudaGetLastError();
}
cudaError_t launch_front(const DevScene* sc, const DevTarget* tg, int nr, int S, const float* zbuf, const float* ray_o,
                         const float* ray_d, const float* nf_in, float* ray_nf, int* list, int list_base, int* counter, int* ray_start,
                         int* ray_cnt, const ErtSegment& ert, cudaStream_t st) {
  // persistent grid: as many blocks as are resident at once (no partial second wave)
  static std::atomic<int> per_sm{0};
  int bps = per_sm.load(std::memory_order_acquire);
  if (bps == 0) {
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, front_kernel, FRONT_THREADS, 0) != cudaSuccess || bps < 1) bps = 4;
    per_sm.store(bps, std::memory_order_release);
  }
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int nwords = (S + 31) / 32;
  const int batch = std::min(FRONT_THREADS, (FRONT_MASKW / nwords) & ~31);
  front_kernel<<<grid_for(nr, batch, sms * bps), FRONT_THREADS, 0, st>>>(sc, tg, nr, S, zbuf, ray_o, ray_d, nf_in, ray_nf, list,
                                                                            list_base, counter, ray_start, ray_cnt, ert);
  return cudaGetLastError();
}
cudaError_t launch_compact(const DevScene* sc, const SampleSrc& src, long long n, int* list, int* counter, float* out, int out_w,
                           uint8_t* valid_out, cudaStream_t st) {
  compact_kernel<<<grid_for(n, 256, 132 * 16), 256, 0, st>>>(sc, src, n, list, counter, out, out_w, valid_out);
  return cudaGetLastError();
}
template <int NV, int TS>
static cudaError_t launch_shade_simt_tile(const ShadeBatch& b) {
  constexpr size_t smem = SHADE_SMEM_BYTES<NV, TS>;
  static std::atomic<bool> attr_set[64];   // function attributes are per device (setting them twice is harmless)
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !attr_set[dev].load(std::memory_order_acquire)) {
    cudaError_t e = cudaFuncSetAttribute(shade_simt_kernel<NV, TS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    if (dev >= 0 && dev < 64) attr_set[dev].store(true, std::memory_order_release);
  }
  int grid = grid_for(b.n_max, TS, b.num_sms);
  shade_simt_kernel<NV, TS><<<grid, 4 * TS, smem, b.st>>>(b.sc, b.wf32, b.src, b.list, b.counter, b.query_mode, b.so);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  *b.launches += 1;
  return b.after_geo ? cudaEventRecord(b.after_geo, b.st) : cudaSuccess;
}
cudaError_t launch_shade_simt(const ShadeBatch& b) {
  if (b.n_views < 1 || b.n_views > MAXV) return cudaErrorInvalidValue;
  return b.n_views <= 3 ? launch_shade_simt_tile<3, 64>(b) : launch_shade_simt_tile<4, 56>(b);
}
cudaError_t launch_composite(const int* list, const float2* ao, const float* rgb, const int* start0, const int* cnt0,
                             const int* start1, const int* cnt1, const float* zbuf, const float* ray_nf, int r0, int nr, int S,
                             long long plane, float* color, float* depth, float* alpha, float* sdf, float* ray_alpha, float* cw,
                             cudaStream_t st) {
  const RaySeg s0{start0, cnt0}, s1{start1, cnt1};
  composite_kernel<<<grid_for((long long)nr * 32, 128, 132 * 64), 128, 0, st>>>(list, ao, rgb, s0, s1, start1 ? 2 : 1, zbuf, ray_nf, r0, nr,
                                                                               S, plane, color, depth, alpha, sdf, ray_alpha, cw);
  return cudaGetLastError();
}
cudaError_t launch_resample(const int* list, const float* cw, const int* start0, const int* cnt0, const int* start1, const int* cnt1,
                            const float* ray_nf, int nr, int Sc, int Sf, float* zout, float* contrib_out, cudaStream_t st) {
  const RaySeg s0{start0, cnt0}, s1{start1, cnt1};
  const size_t smem = (size_t)RES_WARPS * (4 * Sc + 2 * Sf) * sizeof(float);
  static std::atomic<bool> attr_set[64];
  int dev = 0;
  cudaGetDevice(&dev);
  if (smem > 48 * 1024 && (dev < 0 || dev >= 64 || !attr_set[dev].load(std::memory_order_acquire))) {
    cudaError_t e = cudaFuncSetAttribute(resample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(RES_WARPS * (4 * MAX_SC + 2 * MAX_SF) * sizeof(float)));
    if (e != cudaSuccess) return e;
    if (dev >= 0 && dev < 64) attr_set[dev].store(true, std::memory_order_release);
  }
  resample_kernel<<<grid_for(nr, RES_WARPS, 132 * 16), RES_WARPS * 32, smem, st>>>(list, cw, s0, s1, start1 ? 2 : 1, ray_nf, nr, Sc, Sf, zout,
                                                                               contrib_out);
  return cudaGetLastError();
}
int max_coarse_samples() { return MAX_SC; }
int simt_max_kpt() { return (LDA - 64) / 7; }
int simt_max_geo_input() { return LDA; }

}  // namespace kpn
