// robust_track_kernels.cuh -- device code of the batched robust tracker (robust_track.cu launches it):
// frame_tracker::robust_match_based_track (module/frame_tracker.cc:192-245) against each frame's reference keyframe, for
// the frames whose keyframe track (keyframe_track_kernels.cuh) ran and failed:
//   robust::match_frame_and_keyframe (match/robust.cc:218-255) = brute_force_match (Lowe 0.8, no orientation check)
//   -> essential_solver(frm.bearings_, keyfrm->bearings_, matches).find_via_ransac(50, false) -> the inlier matches
//   -> below 20 the frame fails; else pose_optimizer::optimize from last_frm.cam_pose_cw_ -> discard_outliers.
// Free of host-side CUDA runtime dependencies so that tests/cta_emu can compile the same text for the host.
//
// Kernels, in launch order (brute_match_kernel in between is the existing one):
//   rt_prep_kernel        one thread per frame: stage flag, status, the BruteJob (empty for a frame that does not run)
//   rt_list_kernel        one CTA per frame: the brute-force match list in frame keypoint order, the frame's bearings
//                         (undistorted tracker), the 50 x 8 sample sets (ransac_sample.h)
//   rt_hypothesis_kernel  grid (50, frames): the eight-point solve and the inlier score of one hypothesis; the residuals
//                         are staged in shared memory, only E and the score are kept
//   rt_select_kernel      one CTA per frame: the first-best replay, validity, the winner's inlier flags (recomputed)
//                         and the robust matches
// then the tail of track_common.cuh: count = the robust matches, rows = the keyframes', from last_frm.cam_pose_cw_.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include "../../include/plpslam_b200.h"
#include "cammath.h"
#include "devmath.cuh"
#include "essential_common.cuh"
#include "match_jobs.h"
#include "ransac_sample.h"
#include "track_common.cuh"

namespace plp {

namespace rt {

constexpr int kThreads = 256;         // list: one CTA per frame
constexpr int kEssThreads = 128;      // hypothesis / select
constexpr int kPrepThreads = 128;
constexpr float kLoweRatio = 0.8f;    // frame_tracker.cc:196: robust robust_matcher(0.8, false)
constexpr int kNumIter = 50;          // robust.cc:233: find_via_ransac(50, false)
constexpr int kMinSet = 8;            // essential_solver.cc:44

struct RtDev {
    int batch, cap, max_kf_points;
    uint64_t seed;
    // the motion track of the same batch (tracker state)
    const int32_t *n_kp;
    const float *x, *y;                // undistorted keypoints, SoA (batch x cap)
    const uint8_t *desc;               // batch x cap x 32
    double K_cfg[4];                   // the camera's fx, fy, cx, cy (convert_keypoints_to_bearings)
    // the keyframe track of the same batch
    const int32_t *kf_stage, *kf_status, *kf_num_valid;  // batch
    // the reference keyframes (the keyframe call's plp_track_keyframe) and their bearings
    const int32_t *kf_of_frame, *row_offsets;
    const uint8_t *kf_desc;
    const uint8_t *kf_valid;           // may be null
    const double *kf_bearings;         // keyframe rows x 3
    // the frames' bearings (batch x cap x 3): the undistortion's output on a distorted tracker, else written here
    double *bearings;
    int write_bearings;
    // scratch
    BruteJob *bjobs;                   // batch
    int32_t *choice;                   // batch x max_kf_points
    int32_t *pairs;                    // batch x cap x 2: (frame keypoint, keyframe row) in keypoint order
    int32_t *samples;                  // batch x kNumIter x 8
    double *E;                         // batch x kNumIter x 9
    float *score;                      // batch x kNumIter
    uint8_t *inlier;                   // batch x cap: the winner's flag per match-list entry
    double *best_score;                // batch
    int32_t *valid;                    // batch: solution_is_valid_
    // outputs
    int32_t *stage, *status;           // batch
    int32_t *matched;                  // batch x cap: brute-force matches, then the robust ones (keyframe rows)
    int32_t *num_bf, *num_robust;      // batch
};

// the frame runs robust_match_based_track: it needs it and its inputs are in range
__device__ __forceinline__ bool frame_active(const RtDev &D, int b) {
    return D.stage[b] != 0 && D.status[b] == 0;
}

// tracking_module.cc:636-647: the frames whose bow_match_based_track ran and failed.  A keyframe status (1: rows over
// the reservation, 2: kf_of_frame out of range) carries over and the frame fails like a track with no match.
__global__ void __launch_bounds__(kPrepThreads) rt_prep_kernel(RtDev D) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= D.batch) return;
    const int stage = D.kf_stage[b] != 0 && D.kf_num_valid[b] < kNumMatchesThr;
    const int status = D.kf_status[b];
    D.stage[b] = stage;
    D.status[b] = status;
    const bool active = stage && status == 0;
    const int r0 = active ? D.row_offsets[D.kf_of_frame[b]] : 0;
    const size_t base = (size_t)b * D.cap;
    BruteJob J;  // frame = side 1 (robust.cc:280: matched_indices_2_in_1 over the frame's keypoints)
    J.n_frm = active ? D.n_kp[b] : 0;
    J.frm_desc = D.desc + 32 * base;
    J.frm_angle = nullptr;  // no orientation check
    J.n_kf = active ? D.row_offsets[D.kf_of_frame[b] + 1] - r0 : 0;
    J.kf_desc = D.kf_desc + 32 * (size_t)r0;
    J.kf_angle = nullptr;
    J.kf_valid = D.kf_valid ? D.kf_valid + r0 : nullptr;  // robust.cc:288-296
    J.choice = D.choice + (size_t)b * D.max_kf_points;
    J.matched_out = D.matched + base;
    J.num_matches = nullptr;  // rt_list_kernel counts the list
    D.bjobs[b] = J;
}

// robust.cc:371-382: the match list in ascending frame keypoint order; the frame's bearings (frame.cc:79) where the
// undistortion did not write them; create_random_array(8, 0, M - 1) for each of the 50 hypotheses (-1: none drawn).
__global__ void __launch_bounds__(kThreads) rt_list_kernel(RtDev D) {
    const int b = blockIdx.x, tid = threadIdx.x;
    const size_t base = (size_t)b * D.cap;
    const bool active = frame_active(D, b);
    const int n = active ? D.n_kp[b] : 0;
    const int32_t *matched = D.matched + base;
    int32_t *pairs = D.pairs + 2 * base;
    const int M = compact_in_order<kThreads>(n, [&](int i) { return matched[i] >= 0; },
                                             [&](int i, int off) {
                                                 pairs[2 * off] = i;
                                                 pairs[2 * off + 1] = matched[i];
                                             });
    if (D.write_bearings)
        for (int i = tid; i < n; i += kThreads) cam_bearing(D.K_cfg, D.x[base + i], D.y[base + i], D.bearings + 3 * (base + i));
    for (int it = tid; it < kNumIter; it += kThreads) {
        int32_t *s = D.samples + ((size_t)b * kNumIter + it) * 8;
        if (M >= kMinSet) {
            rs_sample8(D.seed, (uint32_t)b, (uint32_t)it, (uint32_t)M, s);
        } else {
            for (int k = 0; k < 8; ++k) s[k] = -1;
        }
    }
    if (tid == 0) D.num_bf[b] = M;
}

// Dynamic shared memory: cap x 2 floats (the residuals of one hypothesis).
// essential_solver.cc:69-85 for hypothesis blockIdx.x of frame blockIdx.y; below 8 matches the solver returns at once.
__global__ void __launch_bounds__(kEssThreads) rt_hypothesis_kernel(RtDev D) {
    PLP_DYNAMIC_SMEM(smem_raw);
    __shared__ double sE[9];
    float *s_res = (float *)smem_raw;
    const int it = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    if (!frame_active(D, b)) return;  // uniform over the block
    const int M = D.num_bf[b];
    if (M < kMinSet) return;
    const size_t base = (size_t)b * D.cap, h = (size_t)b * kNumIter + it;
    const double *b1 = D.bearings + 3 * base;
    const double *b2 = D.kf_bearings + 3 * (size_t)D.row_offsets[D.kf_of_frame[b]];
    const int32_t *pairs = D.pairs + 2 * base;
    if (tid == 0) {
        double E[9];
        ess_hypothesis(b1, b2, pairs, D.samples + h * 8, E);
        for (int k = 0; k < 9; ++k) {
            sE[k] = E[k];
            D.E[h * 9 + k] = E[k];
        }
    }
    __syncthreads();
    const float score = ess_score_cta<kEssThreads>(b1, b2, pairs, M, sE, nullptr, s_res);
    if (tid == 0) D.score[h] = score;
}

// essential_solver.cc:87-96 + robust.cc:234-252: the first best hypothesis, its inlier flags (recomputed from its E, the
// same test as the hypothesis kernel's), validity; the inlier matches keep their keyframe row, the others lose it.
__global__ void __launch_bounds__(kEssThreads) rt_select_kernel(RtDev D) {
    __shared__ int s_best, s_cnt;
    __shared__ double s_score, sE[9];
    const int b = blockIdx.x, tid = threadIdx.x;
    const bool active = frame_active(D, b);
    const int M = active ? D.num_bf[b] : 0;
    const size_t base = (size_t)b * D.cap;
    const bool run = M >= kMinSet;
    if (tid == 0) {
        s_cnt = 0;
        double best_score = 0.0;
        s_best = run ? ess_first_best(D.score + (size_t)b * kNumIter, kNumIter, &best_score) : -1;
        s_score = best_score;
        D.best_score[b] = best_score;
        for (int k = 0; k < 9; ++k) sE[k] = s_best >= 0 ? D.E[((size_t)b * kNumIter + s_best) * 9 + k] : 0.0;
    }
    __syncthreads();
    const int best = s_best;
    const double *b1 = D.bearings + 3 * base;
    const double *b2 = D.kf_bearings + 3 * (size_t)(active ? D.row_offsets[D.kf_of_frame[b]] : 0);
    const int32_t *pairs = D.pairs + 2 * base;
    int local = 0;
    for (int k = tid; k < M; k += kEssThreads) {
        uint8_t v = 0;
        if (best >= 0) {
            float s2, s1;
            int add1;
            v = (uint8_t)ess_check_match(sE, b1 + 3 * (size_t)pairs[2 * k], b2 + 3 * (size_t)pairs[2 * k + 1], &s2,
                                         &add1, &s1);
        }
        D.inlier[base + k] = v;
        local += v;
    }
    atomicAdd(&s_cnt, local);
    __syncthreads();
    const int cnt = s_cnt;
    const bool valid = run && s_score > 0.0 && cnt >= kMinSet;
    for (int k = tid; k < M; k += kEssThreads)
        if (!(valid && D.inlier[base + k])) D.matched[base + pairs[2 * k]] = -1;
    if (tid == 0) {
        D.valid[b] = valid;
        D.num_robust[b] = valid ? cnt : 0;
    }
}

}  // namespace rt

}  // namespace plp
