// Marching cubes on an fp32 volume f[nz][ny][nx] (x fastest), the device half of kpn_mesh_begin / kpn_mesh_emit.
//
// A corner is inside when f > level (NaN: outside).  Each crossing grid edge gets one vertex, owned by its lower corner; the
// vertices are numbered by (owner's linear index, axis x < y < z), the faces by (cell linear index, table order), both through
// exclusive scans of per-point / per-cell counts, so the output does not depend on the order the threads run in.  The case
// table (kpn_mc_table.cuh, tools/gen_mc_table.py) cuts every cube face the same way from both cells that share it, which makes
// the mesh closed and edge-manifold when f <= level on the grid boundary.
#include <cub/device/device_scan.cuh>

#include "kpn_launch.h"
#include "kpn_mc_table.cuh"

namespace kpn {
namespace {

struct Grid3 {
  int nx, ny, nz;
};

__device__ __forceinline__ bool mc_inside(float v, float level) { return v > level; }

// point id -> (i, j, k)
__device__ __forceinline__ void mc_ijk(const Grid3& g, int p, int& i, int& j, int& k) {
  i = p % g.nx;
  const int r = p / g.nx;
  j = r % g.ny;
  k = r / g.ny;
}

__device__ __forceinline__ int mc_stride(const Grid3& g, int ax) { return ax == 0 ? 1 : ax == 1 ? g.nx : g.nx * g.ny; }
__device__ __forceinline__ int mc_extent(const Grid3& g, int ax) { return ax == 0 ? g.nx : ax == 1 ? g.ny : g.nz; }

// the edge from point p (at index idx along ax) to its +ax neighbour crosses the level
__device__ __forceinline__ bool mc_crossing(const float* __restrict__ f, const Grid3& g, int p, int idx, int ax, float level) {
  if (idx + 1 >= mc_extent(g, ax)) return false;
  return mc_inside(__ldg(f + p), level) != mc_inside(__ldg(f + p + mc_stride(g, ax)), level);
}

// grid point coordinate: origin + spacing * idx, both roundings explicit (no FMA contraction)
__device__ __forceinline__ float mc_coord(float origin, float spacing, int idx) { return __fadd_rn(origin, __fmul_rn(spacing, (float)idx)); }

// Per point: owned crossings (vcnt) and, for the cell whose lower corner it is, the case byte and triangle count; the 64-bit
// totals [vertices, faces] (integer sums: the same whatever the order of the atomics).
__global__ void __launch_bounds__(256)
mc_classify_kernel(const float* __restrict__ f, Grid3 g, float level, unsigned int* __restrict__ vcnt, uint8_t* __restrict__ cases,
                   unsigned int* __restrict__ tcnt, unsigned long long* __restrict__ totals) {
  const int n = g.nx * g.ny * g.nz;
  unsigned int my_v = 0, my_t = 0;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) {
    int i, j, k;
    mc_ijk(g, p, i, j, k);
    const unsigned int nv = (unsigned int)mc_crossing(f, g, p, i, 0, level) + (unsigned int)mc_crossing(f, g, p, j, 1, level) +
                            (unsigned int)mc_crossing(f, g, p, k, 2, level);
    vcnt[p] = nv;
    my_v += nv;
    if (i + 1 < g.nx && j + 1 < g.ny && k + 1 < g.nz) {
      unsigned int cs = 0;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const int q = p + (c & 1) + ((c >> 1) & 1) * g.nx + ((c >> 2) & 1) * g.nx * g.ny;
        cs |= (unsigned int)mc_inside(__ldg(f + q), level) << c;
      }
      const int cell = (k * (g.ny - 1) + j) * (g.nx - 1) + i;
      cases[cell] = (uint8_t)cs;
      tcnt[cell] = c_mc_ntri[cs];
      my_t += c_mc_ntri[cs];
    }
  }
  my_v = __reduce_add_sync(0xffffffffu, my_v);
  my_t = __reduce_add_sync(0xffffffffu, my_t);
  if ((threadIdx.x & 31) == 0 && (my_v | my_t)) {
    atomicAdd(totals, (unsigned long long)my_v);
    atomicAdd(totals + 1, (unsigned long long)my_t);
  }
}

// central differences inside the grid, one-sided at its border, zero along an axis of extent 1
__device__ __forceinline__ void mc_gradient(const float* __restrict__ f, const Grid3& g, const float h[3], int p, const int idx[3],
                                            float out[3]) {
#pragma unroll
  for (int ax = 0; ax < 3; ++ax) {
    const int n = mc_extent(g, ax), s = mc_stride(g, ax);
    const int lo = idx[ax] > 0 ? p - s : p, hi = idx[ax] + 1 < n ? p + s : p;
    const int span = (idx[ax] > 0) + (idx[ax] + 1 < n);
    out[ax] = span ? (__ldg(f + hi) - __ldg(f + lo)) / (h[ax] * (float)span) : 0.0f;
  }
}

// One thread per point: its owned crossings, in axis order, at vofs[p] ...
__global__ void __launch_bounds__(256)
mc_vertices_kernel(const float* __restrict__ f, Grid3 g, float level, float3 origin, float3 spacing, const unsigned int* __restrict__ vofs,
                   float* __restrict__ verts, float* __restrict__ normals) {
  const int n = g.nx * g.ny * g.nz;
  const float o[3] = {origin.x, origin.y, origin.z}, h[3] = {spacing.x, spacing.y, spacing.z};
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) {
    int idx[3];
    mc_ijk(g, p, idx[0], idx[1], idx[2]);
    unsigned int v = vofs[p];
    float ga[3];
    bool have_ga = false;
#pragma unroll
    for (int ax = 0; ax < 3; ++ax) {
      if (!mc_crossing(f, g, p, idx[ax], ax, level)) continue;
      const int q = p + mc_stride(g, ax);
      const float fa = __ldg(f + p), fb = __ldg(f + q);
      float t = __fdiv_rn(__fsub_rn(level, fa), __fsub_rn(fb, fa));
      if (!isfinite(t)) t = 0.5f;   // a NaN or infinite endpoint: the edge's midpoint
      float pa[3];
#pragma unroll
      for (int a = 0; a < 3; ++a) pa[a] = mc_coord(o[a], h[a], idx[a]);
      const float pb = mc_coord(o[ax], h[ax], idx[ax] + 1);
      float* vo = verts + 3ll * v;
#pragma unroll
      for (int a = 0; a < 3; ++a) vo[a] = a == ax ? __fadd_rn(pa[a], __fmul_rn(t, __fsub_rn(pb, pa[a]))) : pa[a];
      if (normals) {
        if (!have_ga) { mc_gradient(f, g, h, p, idx, ga); have_ga = true; }
        int jdx[3] = {idx[0], idx[1], idx[2]};
        jdx[ax] += 1;
        float gb[3];
        mc_gradient(f, g, h, q, jdx, gb);
        float nn[3];
#pragma unroll
        for (int a = 0; a < 3; ++a) nn[a] = -(ga[a] + t * (gb[a] - ga[a]));
        const float l2 = nn[0] * nn[0] + nn[1] * nn[1] + nn[2] * nn[2];
        const bool ok = l2 > 0.0f && isfinite(l2);   // false for a zero gradient and for one a NaN / infinite sample touches
        const float inv = ok ? rsqrtf(l2) : 0.0f;
        float* no = normals + 3ll * v;
#pragma unroll
        for (int a = 0; a < 3; ++a) no[a] = ok ? nn[a] * inv : 0.0f;
      }
      ++v;
    }
  }
}

// One thread per cell: its triangles at tofs[cell] ...; a cell edge's vertex is vofs[owner] + (crossings of the owner on the
// lower axes).
__global__ void __launch_bounds__(256)
mc_faces_kernel(const float* __restrict__ f, Grid3 g, float level, const uint8_t* __restrict__ cases, const unsigned int* __restrict__ tofs,
                const unsigned int* __restrict__ vofs, int* __restrict__ faces) {
  const int cx = g.nx - 1, cy = g.ny - 1, ncell = cx * cy * (g.nz - 1);
  for (int cell = blockIdx.x * blockDim.x + threadIdx.x; cell < ncell; cell += gridDim.x * blockDim.x) {
    const int cs = cases[cell];
    const int nt = c_mc_ntri[cs];
    if (nt == 0) continue;
    const int ci = cell % cx, cj = (cell / cx) % cy, ck = cell / (cx * cy);
    int* out = faces + 3ll * tofs[cell];
    for (int m = 0; m < 3 * nt; ++m) {
      const int e = c_mc_tri[cs][m];
      const int ax = e >> 2, r = e & 3;
      const int o0 = r & 1, o1 = r >> 1;   // offsets along the two other axes, lower axis first
      const int di = ax == 0 ? 0 : o0, dj = ax == 1 ? 0 : (ax == 0 ? o0 : o1), dk = ax == 2 ? 0 : o1;
      const int pi = ci + di, pj = cj + dj, pk = ck + dk;
      const int p = (pk * g.ny + pj) * g.nx + pi;
      int rank = 0;
      if (ax > 0) rank += mc_crossing(f, g, p, pi, 0, level);
      if (ax > 1) rank += mc_crossing(f, g, p, pj, 1, level);
      out[m] = (int)(vofs[p] + (unsigned int)rank);
    }
  }
}

inline int mc_grid(long long n) {
  const long long b = (n + 255) / 256;
  return (int)(b < 1 ? 1 : (b > 132 * 32 ? 132 * 32 : b));
}

}  // namespace

size_t mc_scan_temp_bytes(int n) {
  size_t bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, bytes, (unsigned int*)nullptr, n);
  return bytes;
}

cudaError_t launch_mc_classify(const float* f, int nx, int ny, int nz, float level, unsigned int* vcnt, uint8_t* cases, unsigned int* tcnt,
                               unsigned long long* totals, void* scan_tmp, size_t scan_bytes, cudaStream_t st) {
  const Grid3 g{nx, ny, nz};
  const int n = nx * ny * nz;
  const int ncell = (nx - 1) * (ny - 1) * (nz - 1);
  cudaError_t e = cudaMemsetAsync(totals, 0, 2 * sizeof(unsigned long long), st);
  if (e != cudaSuccess) return e;
  mc_classify_kernel<<<mc_grid(n), 256, 0, st>>>(f, g, level, vcnt, cases, tcnt, totals);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  size_t bytes = scan_bytes;
  if ((e = cub::DeviceScan::ExclusiveSum(scan_tmp, bytes, vcnt, n, st)) != cudaSuccess) return e;
  if (ncell > 0) {
    bytes = scan_bytes;
    e = cub::DeviceScan::ExclusiveSum(scan_tmp, bytes, tcnt, ncell, st);
  }
  return e;
}

cudaError_t launch_mc_emit(const float* f, int nx, int ny, int nz, float level, const float origin[3], const float spacing[3],
                           const unsigned int* vofs, const uint8_t* cases, const unsigned int* tofs, float* verts, float* normals,
                           int* faces, long long n_faces, cudaStream_t st) {
  const Grid3 g{nx, ny, nz};
  const int n = nx * ny * nz;
  mc_vertices_kernel<<<mc_grid(n), 256, 0, st>>>(f, g, level, make_float3(origin[0], origin[1], origin[2]),
                                                   make_float3(spacing[0], spacing[1], spacing[2]), vofs, verts, normals);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess || n_faces == 0) return e;
  mc_faces_kernel<<<mc_grid((long long)(nx - 1) * (ny - 1) * (nz - 1)), 256, 0, st>>>(f, g, level, cases, tofs, vofs, faces);
  return cudaGetLastError();
}

}  // namespace kpn
