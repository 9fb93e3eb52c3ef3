// keyframe_track.h -- internal: what plp_tracker_keyframe_track_batch_dev leaves on the device for the local-map stage
// of the same batch (plain struct; shared by tracker.h and local_map_kernels.cuh, which tests/cta_emu also compiles).
#pragma once
#include <stdint.h>

#include "pose_jobs.h"

namespace plp {

struct KeyframeTrack {
    const int32_t *stage;              // batch: 1 = bow_match_based_track ran (the motion result does not stand)
    const int32_t *status;             // batch: 0, or the frame was skipped
    const int32_t *matched;            // batch x cap: keyframe row per keypoint after discard_outliers, or -1
    const double *pose;                // batch x 16
    const int32_t *num_valid;          // batch
    const PoseJob *posejobs;           // batch: n_pts = observations of the keyframe stage's pose optimisation
    const int32_t *obs_row;            // batch x cap: keyframe row of each of those observations
    const double *kf_pos_w;            // keyframe rows x 3
    const int32_t *kf_row_offsets;     // keyframes + 1
    const int32_t *kf_of_frame;        // batch
    const int32_t *local_idx;          // per frame, one entry per row of its keyframe (may be null)
    const int32_t *local_idx_offsets;  // batch + 1 (may be null)
};

}  // namespace plp
