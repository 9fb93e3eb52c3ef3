// match_jobs.h -- device job descriptors of the matchers (plain structs; shared by match.cu, pipeline.cu and the
// device-code headers that tests/cta_emu also compiles for the host).
#pragma once
#include <stdint.h>

namespace plp {

// Per-frame keypoint capacities of the shared-memory matchers.  A job over its launch's capacity matches nothing and
// reports the count 0xffffffff.
constexpr int kMatchMaxPoints = 3072;  // the window matcher (point_match_kernel)
constexpr int kBruteMaxPoints = 4096;  // the brute-force matcher (brute_match_kernel)

// One CTA per job.  All pointers are device pointers.
struct PointMatchJob {
    // current frame (candidates)
    int n;
    const float *x, *y;
    const int32_t *octave;
    const float *angle;    // may be null
    const float *x_right;  // may be null (== all monocular)
    const uint8_t *desc;
    const uint8_t *claimed;  // may be null
    // queries, in the reference's iteration order
    int m;
    const float *qx, *qy;
    const float *qxr;      // predicted x_right, may be null
    const float *qradius;  // margin * scale_factors[level]
    const int32_t *qmin, *qmax;
    const float *qangle;  // may be null
    const uint8_t *qdesc;
    const uint8_t *qvalid;  // may be null
    int32_t *choice;        // scratch, m entries
    // outputs
    int32_t *best_idx_out;  // m entries (match_frame_and_landmarks) or null
    int32_t *matched_out;   // n entries (match_current_and_last_frames) or null
    uint32_t *num_matches;  // 1 entry
    // acceptance threshold of the no-ratio path + 1; 0 = HAMMING_DIST_THR_HIGH (match_frame_and_keyframe passes its own)
    unsigned hamm_thr_p1;
};

struct LineMatchJob {
    int n;
    const float *sx, *sy, *ex, *ey;
    const int32_t *octave;
    const int32_t *ratio_level;  // may be null (=> octave)
    const float *xr_sp, *xr_ep;  // may be null
    const uint8_t *desc;
    const uint8_t *claimed;  // may be null
    int m;
    const float *q_spx, *q_spy, *q_epx, *q_epy;
    const float *q_xr_sp, *q_xr_ep;  // may be null
    const float *qradius;
    const int32_t *qmin, *qmax;
    const uint8_t *qdesc;
    const uint8_t *qvalid;
    int32_t *choice;
    int32_t *best_idx_out;
    int32_t *matched_out;
    uint32_t *num_matches;
    unsigned hamm_thr_p1;  // acceptance threshold + 1; 0 = HAMMING_DIST_THR_HIGH
};

struct BruteJob {
    int n_frm;
    const uint8_t *frm_desc;
    const float *frm_angle;
    int n_kf;
    const uint8_t *kf_desc;
    const float *kf_angle;
    const uint8_t *kf_valid;  // may be null
    int32_t *choice;          // scratch n_kf
    int32_t *matched_out;     // n_frm
    uint32_t *num_matches;
};

// inputs of the reprojection pre-pass of match_current_and_last_frames[_line]
struct ProjectJob {
    int n_last;
    const double *pos_w;     // n x 3 (points) or n x 6 (lines)
    const int32_t *octave;   // last-frame octave
    const uint8_t *valid;    // may be null
    double pose_cw[12];      // rows of [R|t] of the current frame
    int assume_forward, assume_backward;
    // outputs (queries)
    float *qx, *qy, *qxr;          // points: reproj + x_right ; lines: start point
    float *qx2, *qy2, *qxr2;       // lines: end point
    float *qradius;
    int32_t *qmin, *qmax;
    uint8_t *qvalid;
};

}  // namespace plp
