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
// two-term weights and activations: D = A_hi W_hi [+ A_hi W_lo] [+ A_lo W_hi] (LO_MASK bits 4/5: W_lo of stage 4/5, bits 6/7:
// A_lo of stage 4/5).  A tile's pooled rows arrive in the warpgroup's staging slot by one bulk copy, issued while the tile before
// it runs its MMAs; P0|compress reads its input tiles from shared memory, P1 takes its A operand from registers (P0's
// accumulator fragments after the softplus).  Everything after the input build runs on the accumulator fragments.
// =====================================================================================================================
constexpr uint32_t T4H = 64 * 144 * 2, T4L = 64 * 128 * 2;   // P0|compress input tiles: [mean hi | var hi | bias chunk], [mean lo | var lo]
constexpr uint32_t TAIL_SLOT = 64 * POOL_W * 4;              // staging slot: the pooled rows of one tile
constexpr uint32_t TAIL_WG_BYTES = T4H + T4L + TAIL_SLOT;
constexpr uint32_t tail_smem_bytes() {
  return 2 * (REL_PLAN.st[GEO_NSTAGE].off - REL_PLAN.st[4].off) + GWG * TAIL_WG_BYTES;
}
static_assert(tail_smem_bytes() == 210944u && tail_smem_bytes() + 1024u <= SMEM_OPTIN,
              "W_hi + W_lo of stages 4-5 and two warpgroups' input tiles and staging slots fit beside the static block");

// One sub-chain sequence of a tail stage, committed once: A_hi W_hi (KH k-blocks), then A_hi W_lo, then A_lo W_hi (KL k-blocks),
// into the same accumulators.  A from shared memory (the activation tiles ahi / alo).
template <int N, int KH, int KL, bool W_LO, bool A_LO>
__device__ __forceinline__ void tail_mma(float* d, const uint8_t* ahi, const uint8_t* alo, uint32_t whi, uint32_t wlo) {
  constexpr uint32_t lbo = (uint32_t)(N / 8) * 128u;
  tc::wg_fence();
  tc::wg_mma<N, KH>(d, tc::smem_u32(ahi), 1024u, whi, lbo, 0u);
  if constexpr (W_LO) tc::wg_mma<N, KH>(d, tc::smem_u32(ahi), 1024u, wlo, lbo, 1u);
  if constexpr (A_LO) tc::wg_mma<N, KL>(d, tc::smem_u32(alo), 1024u, whi, lbo, 1u);
  tc::wg_commit();
  tc::wg_wait0();
  tc::fence_regs<N / 2>(d);
}
// The same with A from registers: ahi[4 KH], alo[4 KL] (the k-block fragments of WgmmaRA).
template <int N, int KH, int KL, bool W_LO, bool A_LO>
__device__ __forceinline__ void tail_mma_ra(float* d, uint32_t* ahi, uint32_t* alo, uint32_t whi, uint32_t wlo) {
  constexpr uint32_t lbo = (uint32_t)(N / 8) * 128u;
  tc::fence_regs<4 * KH>(ahi);
  if constexpr (A_LO) tc::fence_regs<4 * KL>(alo);
  tc::fence_regs<N / 2>(d);
  tc::wg_fence();
  tc::wg_mma_ra<N, KH>(d, ahi, whi, lbo, 0u);
  if constexpr (W_LO) tc::wg_mma_ra<N, KH>(d, ahi, wlo, lbo, 1u);
  if constexpr (A_LO) tc::wg_mma_ra<N, KL>(d, alo, whi, lbo, 1u);
  tc::wg_commit();
  tc::wg_wait0();
  tc::fence_regs<N / 2>(d);
}

// whi: the blob's W_hi tile of stage 4 (stage 5's follows it).  GEO_ONLY: the geometry-only query (query_mode 2), which writes
// so.out2 and keeps no latent.  LO_MASK: the W_lo / A_lo sub-chains (0xF0 two-term weights, 0xC0 single-term: kpn_api.cu); a
// template parameter, so that each stage's chain is one branch-free wgmma sequence.
template <bool GEO_ONLY, int LO_MASK>
__global__ void __launch_bounds__(GWG * 128, 1)
geo_tail_kernel(const __grid_constant__ TcConsts C, const uint8_t* __restrict__ whi, const uint8_t* __restrict__ wlo,
                const int* __restrict__ list, const int* __restrict__ count_ptr, long long base, long long len,
                const float* __restrict__ pool, int query_mode, ShadeOut so, uint4* __restrict__ lat_out) {
  extern __shared__ __align__(1024) uint8_t wsm[];
  __shared__ uint64_t wbar, sbar[GWG];                     // weights; each warpgroup's staging slot
  __shared__ __align__(16) float wp2[132];                 // density head: w[0][64] | w[1][64] | b[2]
  constexpr TcPlan plan = REL_PLAN;
  constexpr uint32_t HOFF = plan.st[4].off, WH = plan.st[GEO_NSTAGE].off - plan.st[4].off;   // W_hi of stages 4, 5
  constexpr bool W_LO4 = (LO_MASK >> 4) & 1, W_LO5 = (LO_MASK >> 5) & 1, A_LO4 = (LO_MASK >> 6) & 1, A_LO5 = (LO_MASK >> 7) & 1;
  const long long end = min((long long)*count_ptr, base + len);
  if (end <= base) return;
  const int ntiles = (int)((end - base + 63) / 64);
  const int t = threadIdx.x, wg = t >> 7, wt = t & 127, wq = wt >> 5, lane = t & 31;
  const int tstride = gridDim.x * GWG;
  auto slot_of = [&](int w) { return reinterpret_cast<float*>(wsm + 2 * WH + (size_t)w * TAIL_WG_BYTES + T4H + T4L); };
  // the pooled rows of a tile are contiguous in the scratch: one bulk copy of its valid rows into warpgroup w's slot
  auto stage_rows = [&](int w, int tile) {
    const long long s0 = (long long)tile * 64;
    const uint32_t bytes = (uint32_t)min(64ll, end - base - s0) * (POOL_W * 4u);
    tc::mbar_expect_tx(&sbar[w], bytes);
    tc::bulk_g2s(slot_of(w), pool + s0 * POOL_W, bytes, &sbar[w]);
  };
  for (int i = t; i < 130; i += GWG * 128) wp2[i] = i < 64 ? C.w_p2[0][i] : i < 128 ? C.w_p2[1][i - 64] : C.b_p2[i - 128];
  if (t == 0) {
    tc::mbar_init(&wbar, 1);
    for (int w = 0; w < GWG; ++w) tc::mbar_init(&sbar[w], 1);
    tc::fence_mbar_init();
  }
  __syncthreads();
  if (t == 0) {   // [W_hi 4 | W_hi 5 | W_lo 4 | W_lo 5], then each warpgroup's first tile
    tc::mbar_expect_tx(&wbar, 2 * WH);
    tc::bulk_g2s(wsm, whi, WH, &wbar);
    tc::bulk_g2s(wsm + WH, wlo, WH, &wbar);
    for (int w = 0; w < GWG; ++w)
      if (blockIdx.x * GWG + w < ntiles) stage_rows(w, blockIdx.x * GWG + w);
    tc::mbar_wait(&wbar, 0, 0x31u);
  }
  __syncthreads();
  uint8_t* A4h = wsm + 2 * WH + (size_t)wg * TAIL_WG_BYTES;
  uint8_t* A4l = A4h + T4H;
  const float* slot = slot_of(wg);
  const uint32_t W4h = tc::smem_u32(wsm), W5h = W4h + (plan.st[5].off - HOFF), W4l = W4h + WH, W5l = W5h + WH;
  const int bar_id = 1 + wg;
  const int row = wt & 63, h = wt >> 6;
  if (h == 0) {   // bias chunk of P0's input (never overwritten)
    const uint32_t b[8] = {H2_ONE, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
    a_put<64, 8>(A4h, row, 64, b);
  }
  // P1's input words 64..71 (k-block 4): bias column, K padding
  const uint32_t k_bias = (lane & 3) == 0 ? H2_ONE : 0u;
  // the 8 threads of a quarter warp hold 8 consecutive rows, 512 bytes apart in the slot: each reads the 32-byte pairs of its
  // half-row rotated by its row (pair p + row, first or second 16 bytes first), so that the 8 reads of a quarter warp fall in
  // 8 different 16-byte bank groups
  const int rot = row & 3, sw = (row >> 2) & 1;
  int phase = 0;
  for (int tile = blockIdx.x * GWG + wg; tile < ntiles; tile += tstride, phase ^= 1) {
    const long long t0 = base + (long long)tile * 64;
    tc::mbar_wait(&sbar[wg], (uint32_t)phase, 0x32u);
    {   // P0|compress input: [mean hi | var hi | bias chunk], [mean lo | var lo]; the ghost rows of a partial tile repeat the
        // last valid row (they are never written)
      const float4* in = reinterpret_cast<const float4*>(slot + (size_t)min((long long)row, end - 1 - t0) * POOL_W + 32 * h);
#pragma unroll
      for (int half = 0; half < 2; ++half) {   // mean, var
#pragma unroll
        for (int p = 0; p < 4; ++p) {
          const int q = (p + rot) & 3;
          const float4 u = in[16 * half + 2 * q + sw], v = in[16 * half + 2 * q + 1 - sw];
          const float4 x0 = sw ? v : u, x1 = sw ? u : v;   // floats 8q .. 8q + 7 of the half-row
          uint32_t hi[4], lo[4];
          split_h2(x0.x, x0.y, hi[0], lo[0]);
          split_h2(x0.z, x0.w, hi[1], lo[1]);
          split_h2(x1.x, x1.y, hi[2], lo[2]);
          split_h2(x1.z, x1.w, hi[3], lo[3]);
          a_put<64, 4>(A4h, row, 32 * half + 16 * h + 4 * q, hi);
          a_put<64, 4>(A4l, row, 32 * half + 16 * h + 4 * q, lo);
        }
      }
    }
    wg_publish(bar_id);   // the input tiles are visible to the MMAs, and every thread of the warpgroup is done with the slot
    if (wt == 0 && tile + tstride < ntiles) stage_rows(wg, tile + tstride);
    // ---- P0 (softplus, two fp16 terms out: P1's A fragments) | compress (linear, fp16 latent kept in registers until the
    //      density is known).  a*[m] is the word at row 16 wq + (lane >> 2) + 8 (m & 1), word column 4 (m >> 1) + (lane & 3), so
    //      a*[4j .. 4j + 3] is k-block j of P1's input.
    uint32_t ahi[20], alo[16], lat[2][3];
    {
      float d[48];
      tail_mma<96, 9, 8, W_LO4, A_LO4>(d, A4h, A4l, W4h, W4l);
      tc::named_sync(bar_id, 128);   // the input tiles are read: the next tile's may overwrite them
#pragma unroll
      for (int m = 0; m < 24; ++m) {
        if (m < 16) split_h2(sp_fast(d[2 * m]), sp_fast(d[2 * m + 1]), ahi[m], alo[m]);
        else if (m < 22) lat[m & 1][(m >> 1) - 8] = tc::pack_h2(d[2 * m], d[2 * m + 1]);
      }
    }
    ahi[16] = k_bias; ahi[17] = k_bias; ahi[18] = 0u; ahi[19] = 0u;
    // ---- P1 (softplus) then the 64->2 density head in fp32: partial dots over this lane's 16 columns, summed over the quad
    float gs[2] = {0.0f, 0.0f}, rs[2] = {0.0f, 0.0f};
    {
      float d[32];
      tail_mma_ra<64, 5, 4, W_LO5, A_LO5>(d, ahi, alo, W5h, W5l);
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
    for (int m = 0; m < 2; ++m) {   // the quad's rows: fragment pairs 0 and 1, row r, word column c (the latent word of the lane)
      const int r = 16 * wq + (lane >> 2) + 8 * (m & 1), c = 4 * (m >> 1) + (lane & 3);
      float g0 = gs[m], rad = rs[m];
      g0 += __shfl_xor_sync(FULL, g0, 1); g0 += __shfl_xor_sync(FULL, g0, 2);
      rad += __shfl_xor_sync(FULL, rad, 1); rad += __shfl_xor_sync(FULL, rad, 2);
      g0 += wp2[128];
      rad += wp2[129];
      const long long si = t0 + r;
      if (si < end) {
        if (GEO_ONLY) {
          if (c == 0) reinterpret_cast<float2*>(so.out2)[list[si]] = make_float2(g0, rad);
          continue;
        }
        if (c == 0) {
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
          for (int j = 0; j < 3; ++j) lw[4 * j + c] = lat[m][j];
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
  using TailFn = decltype(&geo_tail_kernel<false, 0xF0>);
  // [two-term | single-term weights][render / query | geometry-only]
  static constexpr TailFn kernels[2][2] = {{geo_tail_kernel<false, 0xF0>, geo_tail_kernel<true, 0xF0>},
                                           {geo_tail_kernel<false, 0xC0>, geo_tail_kernel<true, 0xC0>}};
  if (lo_mask != 0xF0 && lo_mask != 0xC0) return cudaErrorInvalidValue;
  constexpr uint32_t smem_tail = tail_smem_bytes();
  static std::atomic<bool> attr[64];   // function attributes are per device (zero-initialised; setting them twice is harmless)
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !attr[dev].load(std::memory_order_acquire)) {
    for (const auto& row : kernels)
      for (TailFn k : row) {
        const cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_tail);
        if (e != cudaSuccess) return e;
      }
    if (dev >= 0 && dev < 64) attr[dev].store(true, std::memory_order_release);
  }
  const TailFn kernel = kernels[lo_mask == 0xC0][query_mode == 2];
  kernel<<<tc_grid((len + 63) / 64, GWG, num_sms), GWG * 128, smem_tail, st>>>(C, wtail, wlo, list, counter, base, len, pool, query_mode,
                                                                              so, lat);
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
