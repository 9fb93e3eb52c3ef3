// sim3_kernels.cuh -- device code of the batched Sim3 RANSAC (sim3.cu launches it).  Free of host-side CUDA runtime
// dependencies so that tests/cta_emu can compile the same text for the host (see essential_kernels.cuh).
#pragma once
#include <stddef.h>
#include <stdint.h>

#include "sim3math.h"

namespace plp {

namespace {

constexpr int kSim3Threads = 32;     // one warp per CTA in every kernel: one hypothesis / one problem
constexpr int kSim3PrepThreads = 128;
constexpr int kSim3MinSet = 3;       // sim3_solver.cc:130, :149

// P independent problems; problem p owns correspondences [offsets[p], offsets[p + 1]).  Every pointer is a device
// pointer, so a caller that already holds the correspondences on the device can fill the job directly.
struct Sim3Job {
    const int32_t *offsets;     // P + 1
    const double *cams;         // P x 4: fx, fy, cx, cy
    const double *pts_1;        // N x 3, keyframe-1 camera frame
    const double *pts_2;        // N x 3, keyframe-2 camera frame
    const float *chi_sq_1;      // N: chi_sq_2D * sigma_sq in keyframe 1
    const float *chi_sq_2;      // N
    const int32_t *samples;     // P x num_iter x 3, problem-local indices
    int num_problems, num_iter, fix_scale, min_num_inliers;
    double *reproj_1, *reproj_2;  // N x 2: reprojected_1_ / reprojected_2_ (:117-118)
    // per hypothesis
    double *hyp_Rt;             // P x num_iter x 12: rot_12 row-major, trans_12
    float *hyp_scale;           // P x num_iter: scale_12
    int32_t *hyp_count;         // P x num_iter: count_inliers
    // results
    int32_t *valid, *num_inliers;  // P
    double *rot_12, *trans_12;     // P x 9, P x 3
    float *scale_12;               // P
};

// find_via_ransac's early exit (:130-134)
__device__ __forceinline__ bool sim3_runs(const Sim3Job &J, int p, int *off, int *n) {
    *off = J.offsets[p];
    *n = J.offsets[p + 1] - *off;
    return *n >= kSim3MinSet && *n >= J.min_num_inliers;
}

// One CTA per problem: the constructor's reproject_to_same_image of both keyframes' points (:117-118), once.
__global__ void __launch_bounds__(kSim3PrepThreads) sim3_reproject_kernel(Sim3Job J) {
    const int p = blockIdx.x;
    int off, n;
    if (!sim3_runs(J, p, &off, &n)) return;
    const double *cam = J.cams + 4 * (size_t)p;
    for (int i = threadIdx.x; i < n; i += kSim3PrepThreads) {
        const size_t c = (size_t)(off + i);
        sim3_reproject_same(cam, J.pts_1 + 3 * c, J.reproj_1 + 2 * c);
        sim3_reproject_same(cam, J.pts_2 + 3 * c, J.reproj_2 + 2 * c);
    }
}

// One warp-sized CTA per (problem, hypothesis), grid (P, num_iter): thread 0 solves Horn's method on the three sampled
// points (:147-159), every lane tests a strided share of the problem's correspondences (:163, count_inliers), and the
// count is an integer warp sum.
__global__ void __launch_bounds__(kSim3Threads) sim3_hypothesis_kernel(Sim3Job J) {
    __shared__ sim3_model s_m;
    const int p = blockIdx.x, iter = blockIdx.y, lane = threadIdx.x;
    int off, n;
    if (!sim3_runs(J, p, &off, &n)) return;
    const size_t h = (size_t)p * J.num_iter + iter;
    if (lane == 0) {
        double pts_1[3 * kSim3MinSet], pts_2[3 * kSim3MinSet];
        const int32_t *s = J.samples + h * kSim3MinSet;
        for (int k = 0; k < kSim3MinSet; ++k) {
            const size_t c = (size_t)(off + s[k]);
            for (int r = 0; r < 3; ++r) {
                pts_1[3 * k + r] = J.pts_1[3 * c + r];
                pts_2[3 * k + r] = J.pts_2[3 * c + r];
            }
        }
        sim3_model m;
        sim3_compute(pts_1, pts_2, J.fix_scale, &m);
        s_m = m;
        for (int k = 0; k < 9; ++k) J.hyp_Rt[h * 12 + k] = m.rot_12[k];
        for (int k = 0; k < 3; ++k) J.hyp_Rt[h * 12 + 9 + k] = m.trans_12[k];
        J.hyp_scale[h] = m.scale_12;
    }
    __syncthreads();
    const double *cam = J.cams + 4 * (size_t)p;
    int local = 0;
    for (int i = lane; i < n; i += kSim3Threads) {
        const size_t c = (size_t)(off + i);
        local += sim3_is_inlier(&s_m, cam, J.pts_1 + 3 * c, J.pts_2 + 3 * c, J.reproj_1 + 2 * c, J.reproj_2 + 2 * c,
                                J.chi_sq_1[c], J.chi_sq_2[c]);
    }
    for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
    if (lane == 0) J.hyp_count[h] = local;
}

// One warp per problem: the ordered "max_num_inliers < num_inliers" replay (:145-175), the validity test
// max_num_inliers >= min_num_inliers (:177), and the winner's rot_12 / trans_12 / scale_12, or the reference's zeros
// (:126-128, :181-183) for a problem that is invalid or does not run.
__global__ void __launch_bounds__(kSim3Threads) sim3_select_kernel(Sim3Job J) {
    __shared__ int s_best, s_valid;
    const int p = blockIdx.x, lane = threadIdx.x;
    int off, n;
    const bool runs = sim3_runs(J, p, &off, &n);
    if (lane == 0) {
        int best = -1, max_num_inliers = 0;
        for (int it = 0; runs && it < J.num_iter; ++it) {
            const int num = J.hyp_count[(size_t)p * J.num_iter + it];
            if (max_num_inliers < num) {
                max_num_inliers = num;
                best = it;
            }
        }
        s_best = best;
        s_valid = runs && max_num_inliers >= J.min_num_inliers;
        J.valid[p] = s_valid;
        J.num_inliers[p] = max_num_inliers;
    }
    __syncthreads();
    // a valid problem without a winner (every count 0, min_num_inliers 0) keeps the zero-initialised best model
    const bool take = s_valid && s_best >= 0;
    const double *Rt = J.hyp_Rt + ((size_t)p * J.num_iter + (take ? s_best : 0)) * 12;
    if (lane < 9) J.rot_12[9 * (size_t)p + lane] = take ? Rt[lane] : 0.0;
    else if (lane < 12) J.trans_12[3 * (size_t)p + lane - 9] = take ? Rt[lane] : 0.0;
    else if (lane == 12) J.scale_12[p] = take ? J.hyp_scale[(size_t)p * J.num_iter + s_best] : 0.0f;
}

}  // namespace

}  // namespace plp
