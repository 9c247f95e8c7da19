// Tensor-core engine (kpn_shade_tc.cuh): the 3-view instantiations of the view-dependent kernels, the kernels every view count
// shares (density tail, colour work list) and the host entry points.  The 4-view kernels are in kpn_shade_tc_v4.cu, a translation
// unit of their own so that the two sets of 16 front-kernel variants compile in parallel.
#include "kpn_shade_tc.cuh"

namespace kpn {
namespace {

// Colour work list: the entries of the first list whose sample needs a colour (alpha > 0), in list order, as (index into the
// first list, sample id).  Block-aggregated append (one atomic per 1024 entries).
__global__ void __launch_bounds__(256)
colour_list_kernel(const int* __restrict__ list, const int* __restrict__ count_ptr, const float2* __restrict__ ao, int list_base,
                   int2* __restrict__ list2, int* __restrict__ count2) {
  __shared__ int s_cnt[8];
  __shared__ int s_base;
  const int count = *count_ptr;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int base = blockIdx.x * 1024; base < count; base += gridDim.x * 1024) {   // block-uniform trip count
    bool ok[4];
    unsigned m[4];
    int mine = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int i = base + j * 256 + threadIdx.x;
      ok[j] = i < count && ao[list_base + i].x > 0.0f;
      m[j] = __ballot_sync(FULL, ok[j]);
      mine += __popc(m[j]);
    }
    if (lane == 0) s_cnt[wid] = mine;
    __syncthreads();
    if (threadIdx.x == 0) {
      int tot = 0;
#pragma unroll
      for (int w = 0; w < 8; ++w) { const int c = s_cnt[w]; s_cnt[w] = tot; tot += c; }
      s_base = tot ? atomicAdd(count2, tot) : 0;
    }
    __syncthreads();
    int pos = s_base + s_cnt[wid];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int i = base + j * 256 + threadIdx.x;
      if (ok[j]) list2[pos + __popc(m[j] & ((1u << lane) - 1u))] = make_int2(i, list[i]);
      pos += __popc(m[j]);
    }
    __syncthreads();
  }
}

// =====================================================================================================================
// geometry tail: P0|compress and P1 per sample (64 samples per warpgroup tile, two threads per row for the input build),
// two-term weights and activations: D = A_hi W_hi [+ A_hi W_lo] [+ A_lo W_hi] (lo_mask bits 4/5: W_lo of stage 4/5,
// bits 6/7: A_lo of stage 4/5).  Everything after the input build runs on the accumulator fragments.
// =====================================================================================================================
constexpr uint32_t T4H = 64 * 144 * 2, T4L = 64 * 128 * 2, T5H = 64 * 80 * 2, T5L = 64 * 64 * 2;   // activation tiles
constexpr uint32_t TAIL_TILE_BYTES = T4H + T4L + T5H + T5L;

template <int N, int KH, int KL>
__device__ __forceinline__ void tail_mma(float* d, const uint8_t* ahi, const uint8_t* alo, uint32_t whi, uint32_t wlo, bool w_lo,
                                         bool a_lo, int bar_id) {
  constexpr uint32_t lbo = (uint32_t)(N / 8) * 128u;
  wg_publish(bar_id);
  tc::wg_fence();
  tc::wg_mma<N, KH>(d, tc::smem_u32(ahi), 1024u, whi, lbo, 0u);
  if (w_lo) tc::wg_mma<N, KH>(d, tc::smem_u32(ahi), 1024u, wlo, lbo, 1u);
  if (a_lo) tc::wg_mma<N, KL>(d, tc::smem_u32(alo), 1024u, whi, lbo, 1u);
  tc::wg_commit();
  tc::wg_wait0();
  tc::named_sync(bar_id, 128);
}

// whi: the blob's W_hi tile of stage 4 (stage 5's follows it).  GEO_ONLY: the geometry-only query (query_mode 2), which writes
// so.out2 and keeps no latent; a template parameter, so that the render / query instantiation is unchanged.
template <bool GEO_ONLY>
__global__ void __launch_bounds__(GWG * 128, 1)
geo_tail_kernel(const __grid_constant__ TcConsts C, const uint8_t* __restrict__ whi, const uint8_t* __restrict__ wlo, int lo_mask,
                const int* __restrict__ list, const int* __restrict__ count_ptr, long long base, long long len,
                const float* __restrict__ pool, int query_mode, ShadeOut so, uint4* __restrict__ lat_out) {
  extern __shared__ __align__(1024) uint8_t wsm[];
  __shared__ uint64_t wbar;
  __shared__ __align__(16) float wp2[132];                 // density head: w[0][64] | w[1][64] | b[2]
  constexpr TcPlan plan = REL_PLAN;
  constexpr uint32_t HOFF = plan.st[4].off, WH = plan.st[GEO_NSTAGE].off - plan.st[4].off;   // W_hi of stages 4, 5
  const long long end = min((long long)*count_ptr, base + len);
  if (end <= base) return;
  const int ntiles = (int)((end - base + 63) / 64);
  const int t = threadIdx.x, wg = t >> 7, wt = t & 127, wq = wt >> 5, lane = t & 31;
  for (int i = t; i < 130; i += GWG * 128) wp2[i] = i < 64 ? C.w_p2[0][i] : i < 128 ? C.w_p2[1][i - 64] : C.b_p2[i - 128];
  if (t == 0) { tc::mbar_init(&wbar, 1); tc::fence_mbar_init(); }
  __syncthreads();
  if (t == 0) {   // [W_hi 4 | W_hi 5 | W_lo 4 | W_lo 5]
    tc::mbar_expect_tx(&wbar, 2 * WH);
    tc::bulk_g2s(wsm, whi, WH, &wbar);
    tc::bulk_g2s(wsm + WH, wlo, WH, &wbar);
    tc::mbar_wait(&wbar, 0, 0x31u);
  }
  __syncthreads();
  uint8_t* A4h = wsm + 2 * WH + (size_t)wg * TAIL_TILE_BYTES;
  uint8_t* A4l = A4h + T4H;
  uint8_t* A5h = A4l + T4L;
  uint8_t* A5l = A5h + T5H;
  const uint32_t W4h = tc::smem_u32(wsm), W5h = W4h + (plan.st[5].off - HOFF), W4l = W4h + WH, W5l = W5h + WH;
  const int bar_id = 1 + wg;
  const int row = wt & 63, h = wt >> 6;
  if (h == 0) {   // bias chunks of the two stages' inputs (never overwritten)
    const uint32_t b[8] = {H2_ONE, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
    a_put<64, 8>(A4h, row, 64, b);
    a_put<64, 8>(A5h, row, 32, b);
  }
  for (int tile = blockIdx.x * GWG + wg; tile < ntiles; tile += gridDim.x * GWG) {
    const long long t0 = base + (long long)tile * 64;
    {   // P0|compress input: [mean hi | var hi | bias chunk], [mean lo | var lo]
      const long long si = min(t0 + row, end - 1);
      const float* in = pool + (si - base) * POOL_W + 32 * h;
      uint32_t mh[16], ml[16], vh[16], vl[16];
#pragma unroll
      for (int c4 = 0; c4 < 8; ++c4) {
        const float4 m = __ldg(reinterpret_cast<const float4*>(in) + c4);
        const float4 s = __ldg(reinterpret_cast<const float4*>(in + 64) + c4);
        split_h2(m.x, m.y, mh[2 * c4], ml[2 * c4]);
        split_h2(m.z, m.w, mh[2 * c4 + 1], ml[2 * c4 + 1]);
        split_h2(s.x, s.y, vh[2 * c4], vl[2 * c4]);
        split_h2(s.z, s.w, vh[2 * c4 + 1], vl[2 * c4 + 1]);
      }
      a_put<64, 16>(A4h, row, 16 * h, mh);
      a_put<64, 16>(A4h, row, 32 + 16 * h, vh);
      a_put<64, 16>(A4l, row, 16 * h, ml);
      a_put<64, 16>(A4l, row, 32 + 16 * h, vl);
    }
    // ---- P0 (softplus, two fp16 terms out) | compress (linear, fp16 latent kept in registers until the density is known)
    uint32_t lat[2][3];
    {
      float d[48];
      tail_mma<96, 9, 8>(d, A4h, A4l, W4h, W4l, (lo_mask >> 4) & 1, (lo_mask >> 6) & 1, bar_id);
#pragma unroll
      for (int m = 0; m < 24; ++m) {
        const int r = 16 * wq + (lane >> 2) + 8 * (m & 1), c = 4 * (m >> 1) + (lane & 3);
        if (m < 16) {
          uint32_t hi, lo;
          split_h2(sp_fast(d[2 * m]), sp_fast(d[2 * m + 1]), hi, lo);
          a_word(A5h, r, c, hi);
          a_word(A5l, r, c, lo);
        } else if (m < 22) {
          lat[m & 1][(m >> 1) - 8] = tc::pack_h2(d[2 * m], d[2 * m + 1]);
        }
      }
    }
    // ---- P1 (softplus) then the 64->2 density head in fp32: partial dots over this lane's 16 columns, summed over the quad
    float gs[2] = {0.0f, 0.0f}, rs[2] = {0.0f, 0.0f};
    {
      float d[32];
      tail_mma<64, 5, 4>(d, A5h, A5l, W5h, W5l, (lo_mask >> 5) & 1, (lo_mask >> 7) & 1, bar_id);
#pragma unroll
      for (int m = 0; m < 16; ++m) {
        const int c = 8 * (m >> 1) + 2 * (lane & 3);
        const float h0 = sp_fast(d[2 * m]), h1 = sp_fast(d[2 * m + 1]);
        gs[m & 1] = fmaf(wp2[c], h0, fmaf(wp2[c + 1], h1, gs[m & 1]));
        rs[m & 1] = fmaf(wp2[64 + c], h0, fmaf(wp2[65 + c], h1, rs[m & 1]));
      }
    }
    // ---- outputs (eval_func, src/model.py:978-997): alpha / sdf and, where a colour will be needed (density > 0: a sample with
    //      alpha == 0 composites with weight exactly 0, skipping its colour is exact; every valid sample in query mode; none in
    //      geometry-only mode), the compressed latent at the sample's own list index
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      float g0 = gs[k], rad = rs[k];
      g0 += __shfl_xor_sync(FULL, g0, 1); g0 += __shfl_xor_sync(FULL, g0, 2);
      rad += __shfl_xor_sync(FULL, rad, 1); rad += __shfl_xor_sync(FULL, rad, 2);
      g0 += wp2[128];
      rad += wp2[129];
      const long long si = t0 + 16 * wq + (lane >> 2) + 8 * k;
      if (si < end) {
        if (GEO_ONLY) {
          if ((lane & 3) == 0) reinterpret_cast<float2*>(so.out2)[list[si]] = make_float2(g0, rad);
          continue;
        }
        if ((lane & 3) == 0) {
          if (query_mode) {
            float* o = so.out5 + 5ll * list[si];
            o[0] = g0; o[1] = rad; o[2] = 0.0f; o[3] = 0.0f; o[4] = 0.0f;
          } else {
            so.ao[so.list_base + si] = make_float2(fmaxf(rad, 0.0f), g0);
          }
        }
        if (query_mode != 0 || rad > 0.0f) {
          uint32_t* lw = reinterpret_cast<uint32_t*>(lat_out + 3ll * si);
#pragma unroll
          for (int j = 0; j < 3; ++j) lw[4 * j + (lane & 3)] = lat[k][j];
        }
      }
    }
  }
}

}  // namespace

size_t tc_weight_blob_bytes(int n_kpt) { return make_tc_plan(n_kpt).total_bytes; }
size_t tc_weight_lo_bytes(int n_kpt) {
  const TcPlan p = make_tc_plan(n_kpt);
  return p.st[GEO_NSTAGE].off - p.st[4].off;
}
size_t tc_pool_bytes(long long n_max) { return (size_t)(n_max < POOL_SLICE ? n_max : POOL_SLICE) * POOL_W * sizeof(float); }
bool tc_supported(int n_views, int n_kpt, int sp_level) {
  return (n_views == 3 || n_views == 4) && n_kpt >= 1 && n_kpt <= KPN_MAX_KPT && sp_level == 3;
}

cudaError_t launch_geo_tail(const TcConsts& C, const uint8_t* wtail, const uint8_t* wlo, int lo_mask, const int* list,
                            const int* counter, long long base, long long len, const float* pool, int query_mode, const ShadeOut& so,
                            uint4* lat, int num_sms, cudaStream_t st) {
  constexpr TcPlan rel = REL_PLAN;
  constexpr uint32_t smem_tail = 2 * (rel.st[GEO_NSTAGE].off - rel.st[4].off) + GWG * TAIL_TILE_BYTES;
  static std::atomic<bool> attr[64];   // function attributes are per device (zero-initialised; setting them twice is harmless)
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !attr[dev].load(std::memory_order_acquire)) {
    cudaError_t e = cudaFuncSetAttribute(geo_tail_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_tail);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(geo_tail_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_tail);
    if (e != cudaSuccess) return e;
    if (dev >= 0 && dev < 64) attr[dev].store(true, std::memory_order_release);
  }
  auto kernel = query_mode == 2 ? geo_tail_kernel<true> : geo_tail_kernel<false>;
  kernel<<<tc_grid((len + 63) / 64, GWG, num_sms), GWG * 128, smem_tail, st>>>(C, wtail, wlo, lo_mask, list, counter, base, len, pool,
                                                                              query_mode, so, lat);
  return cudaGetLastError();
}

cudaError_t launch_colour_list(const int* list, const int* counter, const float2* ao, int list_base, int2* list2, int* count2,
                               long long n_max, int num_sms, cudaStream_t st) {
  const long long lb = (n_max + 1023) / 1024;
  colour_list_kernel<<<(int)(lb < 1 ? 1 : (lb > num_sms * 8 ? num_sms * 8 : lb)), 256, 0, st>>>(list, counter, ao, list_base, list2,
                                                                                                 count2);
  return cudaGetLastError();
}

cudaError_t launch_shade_tc(const ShadeBatch& b) {
  if (b.n_views == 3) return launch_tc_views<3>(b);
  if (b.n_views == 4) return launch_shade_tc_v4(b);
  return cudaErrorInvalidValue;
}

// Watchdog state of the tensor-core kernels.  Every translation unit has its own copy of the words (kpn_tc.cuh): the 3-view
// module's (with the shared tail kernel) and the 4-view module's.
static_assert(TC_WD_MODULES == 2, "the 3-view and the 4-view module");
cudaError_t tc_watchdog_words(void* w[TC_WD_MODULES]) {
  cudaError_t e = cudaGetSymbolAddress(&w[0], tc::kpn_wd);
  return e != cudaSuccess ? e : tc_watchdog_addr_v4(&w[1]);
}

}  // namespace kpn
