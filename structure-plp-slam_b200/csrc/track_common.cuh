// track_common.cuh -- device code shared by the stages of the batched tracker.  The motion (pipeline.cu), keyframe
// (keyframe_track.cu) and robust (robust_track.cu) stages end alike: pose_optimizer::optimize over the matched
// keypoints, then frame_tracker::discard_outliers.  That tail is the two kernels below around the pose optimiser, over
// one TrackTail job per stage; the stages differ only in its data (gate, rows, starting pose).
// Free of host-side CUDA runtime dependencies so that tests/cta_emu can compile the same text for the host.
#pragma once
#include <stdint.h>

#include "../../include/plpslam_b200.h"
#include "track_record.h"

namespace plp {

constexpr int kNumMatchesThr = 20;  // frame_tracker::num_matches_thr_ (module/frame_tracker.h)
constexpr int kTailThreads = 256;   // gather / finish: one CTA per frame

// frame b's block of rows
__device__ __forceinline__ int row_block(const TrackRows &R, int b) { return R.of_frame ? R.of_frame[b] : b; }

struct TrackTail {
    int cap;
    // the current frames' keypoints (undistorted, SoA: batch x cap)
    const int32_t *n_kp;
    const float *x, *y;
    const int32_t *octave;
    float inv_level_sigma_sq[16];
    // the gate: count[b] >= kNumMatchesThr, and stage[b] != 0 / status[b] == 0 where those are not null
    const int32_t *count, *stage, *status;
    TrackRows rows;                    // the rows the matches index
    const double *pose_in;             // batch x 16: where the optimisation starts
    int32_t *matched;                  // batch x cap: the stage's matches (rows), then discard_outliers' result
    // scratch
    PoseJob *posejobs;                 // batch
    plp_pt_obs *obs;                   // batch x cap
    int32_t *obs_kp, *obs_row;         // batch x cap: keypoint and row of each observation
    uint8_t *obs_outlier;              // batch x cap
    // outputs
    double *pose;                      // batch x 16
    int32_t *num_valid, *n_inliers, *lm_iters;  // batch
};

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
// It begins with a block barrier, so take() sees what the block wrote before the call.  The thread that calls take(i)
// calls emit(i, k) right after it, in the same round.  Returns the count, in every thread.
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

// frame_tracker.cc:75 / :140 / :203: the frame ran the stage and found enough matches
__device__ __forceinline__ bool tail_enough(const TrackTail &J, int b) {
    return (!J.stage || J.stage[b] != 0) && (!J.status || J.status[b] == 0) && J.count[b] >= kNumMatchesThr;
}

// Internal linkage, as in the other kernel headers, so that several translation units can include this one;
// launch_track_tail (pipeline.cu) launches them.
namespace {

// pose_optimizer.cc:126-151: one observation per matched keypoint, in keypoint order; a frame below the gate has none
// (the optimiser then copies pose_in and reports 0 / 0)
__global__ void __launch_bounds__(kTailThreads) track_gather_kernel(TrackTail J) {
    const int b = blockIdx.x;
    const size_t base = (size_t)b * J.cap;
    const bool enough = tail_enough(J, b);
    const int r0 = enough ? J.rows.offsets[row_block(J.rows, b)] : 0;
    const int32_t *matched = J.matched + base;
    const int n_obs = compact_in_order<kTailThreads>(
        enough ? J.n_kp[b] : 0, [&](int i) { return matched[i] >= 0; },
        [&](int i, int off) {
            const int q = matched[i];
            J.obs[base + off] = point_obs(J.rows.pos_w + 3 * (size_t)(r0 + q), J.x[base + i], J.y[base + i],
                                          J.inv_level_sigma_sq[J.octave[base + i]]);
            J.obs_kp[base + off] = i;
            J.obs_row[base + off] = q;
        });
    if (threadIdx.x == 0) {
        PoseJob P;
        P.T_in = J.pose_in + 16 * (size_t)b;
        P.pts = J.obs + base;
        P.n_pts = n_obs;
        P.lines = nullptr;
        P.n_lines = 0;
        P.T_out = J.pose + 16 * (size_t)b;
        P.pt_outlier = J.obs_outlier + base;
        P.line_outlier = nullptr;
        P.n_inliers = J.n_inliers + b;
        P.lm_iters = J.lm_iters + b;
        J.posejobs[b] = P;
    }
}

// frame_tracker::discard_outliers (frame_tracker.cc:253-283); a frame below the gate keeps no match
__global__ void __launch_bounds__(kTailThreads) track_finish_kernel(TrackTail J) {
    const int b = blockIdx.x;
    const size_t base = (size_t)b * J.cap;
    const int valid = discard_outliers<kTailThreads>(J.n_kp[b], J.posejobs[b].n_pts, tail_enough(J, b),
                                                     J.obs_outlier + base, J.obs_kp + base, J.matched + base);
    if (threadIdx.x == 0) J.num_valid[b] = valid;
}

}  // namespace

}  // namespace plp
