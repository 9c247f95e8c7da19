// Tensor-core engine, 4 source views: the 4-view instantiations of the view-dependent kernels of kpn_shade_tc.cuh (8 samples per
// warp, 16 per front tile, 32 per colour tile).  The density tail and the colour work list are shared with the 3-view path
// (kpn_shade_tc.cu).
#include "kpn_shade_tc.cuh"

namespace kpn {

cudaError_t launch_shade_tc_v4(const ShadeBatch& b) { return launch_tc_views<4>(b); }

// device address of this module's watchdog words (kpn_tc.cuh)
cudaError_t tc_watchdog_addr_v4(void** p) { return cudaGetSymbolAddress(p, tc::kpn_wd); }

}  // namespace kpn
