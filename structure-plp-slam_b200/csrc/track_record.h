// track_record.h -- internal: what a tracking stage of the batched tracker (motion, keyframe, robust) leaves on the
// device for the later stages of the same batch (plain structs; shared by tracker.h and track_common.cuh, which
// tests/cta_emu also compiles).
#pragma once
#include <stdint.h>

#include "pose_jobs.h"

namespace plp {

// The rows a stage's matches index: frame b's rows begin at offsets[of_frame ? of_frame[b] : b].  The motion stage
// matches the last frames' rows (one block per frame), the keyframe and robust stages the reference keyframes' rows.
struct TrackRows {
    const double *pos_w;               // rows x 3
    const int32_t *offsets;            // blocks + 1
    const int32_t *of_frame;           // batch: the frame's block, or null (block b)
};

struct TrackRecord {
    const int32_t *stage;              // batch: 1 = the stage ran (an earlier result does not stand); null: every frame
    const int32_t *status;             // batch: 0, or the frame was skipped; null: all 0
    const int32_t *matched;            // batch x cap: row per keypoint after discard_outliers, or -1
    const double *pose;                // batch x 16
    const int32_t *num_valid;          // batch
    const PoseJob *posejobs;           // batch: n_pts = observations of the stage's pose optimisation
    const int32_t *obs_row;            // batch x cap: row of each of those observations
    TrackRows rows;
    const int32_t *local_idx;          // per frame, one entry per row of its block (may be null)
    const int32_t *local_idx_offsets;  // batch + 1 (may be null)
};

}  // namespace plp
