// essential_common.cuh -- block-level device code of solve::essential_solver::find_via_ransac (solve/essential_solver.cc:
// 37-121) shared by the single-call RANSAC (essential_kernels.cuh) and the batched robust tracker
// (robust_track_kernels.cuh): the eight-point hypothesis, the inlier score and the first-best replay.  Both callers give
// the same bits for the same sample sets.  Free of host-side CUDA runtime dependencies so that tests/cta_emu can compile
// the same text for the host.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include "essmath.h"

namespace plp {

// :72-81 (one thread): E_21 of the sample set `sample` (8 indices into the match list; matches[2 k] indexes b1,
// matches[2 k + 1] indexes b2), accumulated in sample order
__device__ __forceinline__ void ess_hypothesis(const double *b1, const double *b2, const int32_t *matches,
                                               const int32_t *sample, double *E) {
    double ata[81];
    for (int k = 0; k < 81; ++k) ata[k] = 0.0;
    for (int i = 0; i < 8; ++i) {
        const int idx = sample[i];
        ess_accumulate(ata, b1 + 3 * (size_t)matches[2 * idx], b2 + 3 * (size_t)matches[2 * idx + 1]);
    }
    ess_solve(ata, E);
}

// :84 (essential_solver.cc:200-254) by a block of kThreads: the inlier test of every match against E, then the
// reference's sequential float sum in match order (thread 0, over the residuals staged in res: n x 2).  inlier may be
// null.  Returns the score to thread 0.
template <int kThreads>
__device__ __forceinline__ float ess_score_cta(const double *b1, const double *b2, const int32_t *matches, int n,
                                               const double *E, uint8_t *inlier, float *res) {
    const int tid = threadIdx.x;
    for (int i = tid; i < n; i += kThreads) {
        float s2, s1;
        int add1;
        const int ok = ess_check_match(E, b1 + 3 * (size_t)matches[2 * i], b2 + 3 * (size_t)matches[2 * i + 1], &s2,
                                       &add1, &s1);
        if (inlier) inlier[i] = (uint8_t)ok;
        res[2 * i] = s2;
        res[2 * i + 1] = add1 ? s1 : -1.0f;  // -1 marks "not added" (residuals are absolute values, never negative)
    }
    __syncthreads();
    float score = 0;
    if (tid == 0) {
        for (int i = 0; i < n; ++i) {
            score += res[2 * i];
            const float s1 = res[2 * i + 1];
            if (!(s1 == -1.0f)) score += s1;
        }
    }
    return score;
}

// :87-92 (one thread): "if (best_score_ < score_in_sac)" over the hypotheses in iteration order; the first best wins.
// Returns its index, or -1 when no score exceeds 0 (best_score_ stays 0).
__device__ __forceinline__ int ess_first_best(const float *score, int num_iter, double *best_score) {
    double best_sc = 0.0;
    int best = -1;
    for (int it = 0; it < num_iter; ++it) {
        const float sc = score[it];
        if (best_sc < (double)sc) {
            best_sc = (double)sc;
            best = it;
        }
    }
    *best_score = best_sc;
    return best;
}

}  // namespace plp
