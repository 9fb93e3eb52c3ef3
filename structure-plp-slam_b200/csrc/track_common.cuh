// track_common.cuh -- block-level device code shared by the trackers that end in pose_optimizer::optimize +
// frame_tracker::discard_outliers: motion_based_track (pipeline.cu) and bow_match_based_track
// (keyframe_track_kernels.cuh).  They differ only in where a matched keypoint's landmark position comes from.
// Free of host-side CUDA runtime dependencies so that tests/cta_emu can compile the same text for the host.
#pragma once
#include <stdint.h>

#include "../../include/plpslam_b200.h"

namespace plp {

// pose_optimizer.cc:126-151: the observation of one matched keypoint (monocular)
__device__ __forceinline__ plp_pt_obs point_obs(const double *X, float x, float y, float inv_sigma_sq) {
    plp_pt_obs o;
    o.pos_w[0] = X[0];
    o.pos_w[1] = X[1];
    o.pos_w[2] = X[2];
    o.obs_x = x;
    o.obs_y = y;
    o.x_right = -1.0f;
    o.inv_sigma_sq = inv_sigma_sq;
    return o;
}

// Ordered compaction over i < n by a block of kThreads: emit(i, k) for the k-th i (in ascending i) with take(i).
// Returns the count, in every thread.
template <int kThreads, class Take, class Emit>
__device__ __forceinline__ int compact_in_order(int n, Take take, Emit emit) {
    __shared__ int warp_sums[kThreads / 32];
    __shared__ int s_base;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_base = 0;
    __syncthreads();
    for (int start = 0; start < n; start += kThreads) {
        const int i = start + tid;
        const int flag = i < n && take(i);
        const unsigned bal = __ballot_sync(0xffffffffu, flag);
        if (lane == 0) warp_sums[warp] = __popc(bal);
        __syncthreads();
        int off = s_base;
        for (int w = 0; w < warp; ++w) off += warp_sums[w];
        off += __popc(bal & ((1u << lane) - 1));
        if (flag) emit(i, off);
        __syncthreads();
        if (tid == 0) {
            int tot = 0;
            for (int w = 0; w < kThreads / 32; ++w) tot += warp_sums[w];
            s_base += tot;
        }
        __syncthreads();
    }
    return s_base;
}

// frame_tracker::discard_outliers (frame_tracker.cc:253-283) by a block of kThreads: with enough matches an outlier of
// the pose optimisation loses its landmark; without, every keypoint does.  Returns the valid matches, in every thread.
template <int kThreads>
__device__ __forceinline__ int discard_outliers(int n, int n_obs, bool enough, const uint8_t *obs_outlier,
                                                const int32_t *obs_kp, int32_t *matched) {
    __shared__ int s_cnt;
    const int tid = threadIdx.x;
    if (tid == 0) s_cnt = 0;
    __syncthreads();
    int valid = 0;
    if (enough) {
        for (int k = tid; k < n_obs; k += kThreads) {
            if (obs_outlier[k])
                matched[obs_kp[k]] = -1;
            else
                ++valid;
        }
    } else {
        for (int i = tid; i < n; i += kThreads) matched[i] = -1;
    }
    atomicAdd(&s_cnt, valid);
    __syncthreads();
    return s_cnt;
}

}  // namespace plp
