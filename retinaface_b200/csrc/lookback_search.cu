// lookback_search.cu -- f17 k_lookback_search (lookback.cuh, rf_b200.h rf_tracker_set_lookback_search).  Built with -fmad=false: the
// steps are f16's template search (tsearch.cuh) and f15's motion undo, every FP64 step one rounding as oracle/lookback_search.py
// restates it.
#include <algorithm>

#include "lookback.cuh"
#include "search_kernels.cuh"

namespace rf {
namespace {

static_assert(sizeof(LookbackArgs) + sizeof(LookbackSearchTable) + 32 <= 4096, "k_lookback_search exceeds the classic 4 KB parameter space");

// One CTA per (frame of the table, birth rank): the chain of the birth (rf_b200.h rf_tracker_set_lookback_search).  The template is
// cut once into shared memory; each step then runs f16's Windows, Match, Box and Status from the previous step's box, moved back by
// frame e + 1's camera motion when it is OK.
__global__ void __launch_bounds__(FOLLOW_THREADS) k_lookback_search(const LookbackArgs a, const __grid_constant__ LookbackSearchTable t) {
    lookback_search<false>(a, t);
}

}  // namespace

cudaError_t launch_lookback_search(const LookbackArgs &a, const LookbackSearchTable &t, cudaStream_t s, bool oriented) {
    if (oriented) return launch_lookback_search_oriented(a, t, s);
    k_lookback_search<<<dim3(std::min(a.max_faces, a.max_tracks), t.n), FOLLOW_THREADS, 0, s>>>(a, t);
    return cudaGetLastError();
}

}  // namespace rf
