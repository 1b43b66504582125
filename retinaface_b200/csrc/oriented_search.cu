// oriented_search.cu -- f20's oriented twins of the kernels that search luma (search_kernels.cuh): k_follow_cut, k_follow_search and
// k_lookback_search on frames read as their videos display them.  Built with -fmad=false, as follow.cu and lookback_search.cu are: the
// FP64 steps are the same, and only the byte each luma tap reads moves.
#include <algorithm>

#include "search_kernels.cuh"

namespace rf {
namespace {

__global__ void __launch_bounds__(FOLLOW_THREADS) k_follow_cut_oriented(const FollowArgs a, const __grid_constant__ FollowTable t) {
    follow_cut<true>(a, t);
}

__global__ void __launch_bounds__(FOLLOW_THREADS) k_follow_search_oriented(const FollowArgs a, const __grid_constant__ FollowTable t) {
    follow_search<true>(a, t);
}

__global__ void __launch_bounds__(FOLLOW_THREADS) k_lookback_search_oriented(const LookbackArgs a,
                                                                               const __grid_constant__ LookbackSearchTable t) {
    lookback_search<true>(a, t);
}

}  // namespace

cudaError_t launch_follow_cut_oriented(const FollowArgs &a, const FollowTable &t, cudaStream_t s) {
    k_follow_cut_oriented<<<dim3(a.p.max_tracks, t.n), FOLLOW_THREADS, 0, s>>>(a, t);
    return cudaGetLastError();
}

cudaError_t launch_follow_search_oriented(const FollowArgs &a, const FollowTable &t, cudaStream_t s) {
    k_follow_search_oriented<<<dim3(a.p.max_tracks, t.n), FOLLOW_THREADS, 0, s>>>(a, t);
    return cudaGetLastError();
}

cudaError_t launch_lookback_search_oriented(const LookbackArgs &a, const LookbackSearchTable &t, cudaStream_t s) {
    k_lookback_search_oriented<<<dim3(std::min(a.max_faces, a.max_tracks), t.n), FOLLOW_THREADS, 0, s>>>(a, t);
    return cudaGetLastError();
}

}  // namespace rf
