// Tensor-core engine, 4 source views: the 4-view instantiations of the view-dependent kernels of kpn_shade_tc.cuh (8 samples per
// warp, 16 per front tile, 32 per colour tile).  The density tail and the colour work list are shared with the 3-view path
// (kpn_shade_tc.cu).
#include "kpn_shade_tc.cuh"

namespace kpn {

cudaError_t launch_shade_tc_v4(const DevScene* sc, const TcConsts& C, const uint8_t* wblob, const uint8_t* wlo, int lo_mask, int n_kpt,
                               const SampleSrc& src, const int* list, const int* counter, long long n_max, int query_mode,
                               const ShadeOut& so, void* lat_scratch, void* pool_scratch, void* list2, int* count2, int num_sms,
                               cudaEvent_t after_geo, int* launches, cudaStream_t st) {
  return launch_tc_views<4>(sc, C, wblob, wlo, lo_mask, n_kpt, src, list, counter, n_max, query_mode, so, lat_scratch, pool_scratch,
                            list2, count2, num_sms, after_geo, launches, st);
}

// device address of this module's watchdog words (kpn_tc.cuh)
cudaError_t tc_watchdog_addr_v4(void** p) { return cudaGetSymbolAddress(p, tc::kpn_wd); }

}  // namespace kpn
