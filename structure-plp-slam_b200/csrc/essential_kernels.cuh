// essential_kernels.cuh -- device code of the essential-matrix RANSAC (essential.cu launches it).  Free of host-side CUDA
// runtime dependencies so that tests/cta_emu can compile the same text for the host (see plane_kernels.cuh).
#pragma once
#include <stddef.h>
#include <stdint.h>

#include "essential_common.cuh"

namespace plp {

namespace {

constexpr int kEssThreads = 128;

struct EssJob {
    const double *b1, *b2;
    const int32_t *matches;  // num_matches x 2
    const int32_t *samples;  // num_iter x 8
    int num_matches, num_iter, recompute;
    // per hypothesis
    double *E;          // num_iter x 9
    float *score;       // num_iter
    uint8_t *inlier;    // num_iter x num_matches
    float *res;         // num_iter x num_matches x 2 (s2, s1) scratch
    // result
    uint8_t *best_inlier;  // num_matches
    double *best_E;        // 9
    double *best_score;    // 1
    int32_t *valid;        // 1
};

// inlier test of every match against E (all threads), then the ordered float sum (thread 0); returns the score to thread 0
__device__ float check_inliers_cta(const EssJob &J, const double *E, uint8_t *inlier, float *res) {
    return ess_score_cta<kEssThreads>(J.b1, J.b2, J.matches, J.num_matches, E, inlier, res);
}

__global__ void __launch_bounds__(kEssThreads) essential_hypothesis_kernel(EssJob J) {
    __shared__ double sE[9];
    const int iter = blockIdx.x, tid = threadIdx.x;
    if (tid == 0) {
        double E[9];
        ess_hypothesis(J.b1, J.b2, J.matches, J.samples + iter * 8, E);  // :72-81
        for (int k = 0; k < 9; ++k) {
            sE[k] = E[k];
            J.E[iter * 9 + k] = E[k];
        }
    }
    __syncthreads();
    const float score = check_inliers_cta(J, sE, J.inlier + (size_t)iter * J.num_matches,
                                          J.res + (size_t)iter * J.num_matches * 2);  // :84
    if (tid == 0) J.score[iter] = score;
}

__global__ void __launch_bounds__(kEssThreads) essential_select_kernel(EssJob J) {
    __shared__ int s_best, s_valid, s_cnt;
    __shared__ double sE[9];
    const int tid = threadIdx.x;
    if (tid == 0) {
        s_cnt = 0;
        double best_score;
        const int best = ess_first_best(J.score, J.num_iter, &best_score);  // :87-92
        s_best = best;
        *J.best_score = best_score;
        for (int k = 0; k < 9; ++k) J.best_E[k] = best >= 0 ? J.E[best * 9 + k] : 0.0;
    }
    __syncthreads();
    const int best = s_best;
    int local = 0;
    for (int i = tid; i < J.num_matches; i += kEssThreads) {
        const uint8_t v = best >= 0 ? J.inlier[(size_t)best * J.num_matches + i] : 0;
        J.best_inlier[i] = v;
        local += v;
    }
    atomicAdd(&s_cnt, local);
    __syncthreads();
    if (tid == 0) {
        s_valid = (*J.best_score > 0.0) && (s_cnt >= 8);  // :95-96
        *J.valid = s_valid;
    }
    __syncthreads();
    if (!J.recompute || !s_valid) return;
    // :99-120 recompute from all inliers (accumulated in match order), then re-score
    if (tid == 0) {
        double ata[81];
        for (int k = 0; k < 81; ++k) ata[k] = 0.0;
        for (int i = 0; i < J.num_matches; ++i)
            if (J.best_inlier[i])
                ess_accumulate(ata, J.b1 + 3 * (size_t)J.matches[2 * i], J.b2 + 3 * (size_t)J.matches[2 * i + 1]);
        double E[9];
        ess_solve(ata, E);
        for (int k = 0; k < 9; ++k) {
            sE[k] = E[k];
            J.best_E[k] = E[k];
        }
    }
    __syncthreads();
    const float score = check_inliers_cta(J, sE, J.best_inlier, J.res);
    if (tid == 0) *J.best_score = (double)score;
}

}  // namespace

}  // namespace plp
