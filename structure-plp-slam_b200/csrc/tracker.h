// tracker.h -- internal: the state of a plp_tracker, shared by its stages, which run in order on a batch:
// pipeline.cu (motion_based_track), keyframe_track.cu (bow_match_based_track), robust_track.cu
// (robust_match_based_track), local_map_update.cu (update_local_map) and local_map.cu
// (optimize_current_frame_with_local_map).  Each of the first three ends in
// the same tail (track_common.cuh) and leaves a TrackRecord (track_record.h) that the later stages of the batch read.
#pragma once
#include <memory>

#include "common.cuh"
#include "camera_jobs.h"
#include "match_jobs.h"
#include "pose_jobs.h"
#include "track_common.cuh"

namespace plp {

namespace lm {
struct LocalDev;  // local_map_kernels.cuh
}
namespace kt {
struct KfDev;  // keyframe_track_kernels.cuh
}
namespace rt {
struct RtDev;  // robust_track_kernels.cuh
}
namespace lu {
struct UpdDev;  // local_map_update_kernels.cuh
}

struct TrackDev {
    int batch, cap, num_levels;
    // current frames (ORB output)
    const plp_keypoint *kp;
    const uint8_t *desc;
    const int32_t *n_kp;
    // last frames
    const double *last_pos_w;
    const int32_t *last_octave;
    const float *last_angle;
    const uint8_t *last_desc;
    const uint8_t *last_valid;
    const int32_t *last_offsets;
    const double *pose_pred, *pose_last;
    // scratch (SoA copies of the current keypoints, queries, jobs)
    float *x, *y, *angle;
    int32_t *octave;
    float *qx, *qy, *qxr, *qradius;
    int32_t *qmin, *qmax;
    uint8_t *qvalid;
    int32_t *choice;
    uint32_t *num_matches;
    ProjectJob *pjobs;       // 2 x batch (first attempt, retry)
    PointMatchJob *mjobs;    // 2 x batch
    // output
    int32_t *matched;        // batch x cap : last-frame index per keypoint (-1: none)
    int max_last;
};

// the stages that end in the tail, in the order they run on a batch
enum TrackStage : int { kStageMotion, kStageKeyframe, kStageRobust, kNumStages };

// gather -> pose_optimizer::optimize -> discard_outliers over the first `batch` frames (pipeline.cu)
plp_status launch_track_tail(plp_ctx *ctx, const TrackTail &J, int batch, const plp_camera &cam);

}  // namespace plp

struct plp_tracker {
    plp_ctx *ctx = nullptr;
    int max_batch = 0, cap = 0, max_last = 0, num_levels = 0;
    plp_camera cam;
    plp_grid grid;
    float scale_factors[16];
    float inv_level_sigma_sq[16];
    float *d_scale_factors = nullptr;
    uint8_t *d_block = nullptr;  // one allocation carved into the scratch arrays
    plp::TrackDev dev;
    bool distorted = false;
    plp::UndistJob undist;             // camera and coefficients; kp / n_kp / batch set per call
    plp_keypoint *d_undist = nullptr;  // max_batch x cap (inside d_block)
    double *d_bearings = nullptr;      // max_batch x cap x 3
    // the most recent motion_track_batch_dev: its inputs and scratch, which the later stages read
    plp::TrackDev motion;
    // per stage: its tail job with the scratch bound (at create or reserve), and the record its most recent call left;
    // record_batch[s] is that call's batch, or 0 once the record no longer stands
    plp::TrackTail tail[plp::kNumStages];
    plp::TrackRecord record[plp::kNumStages];
    int record_batch[plp::kNumStages] = {};
    // a call of stage s, or a new reservation for it, ends the records of s and of every later stage, and the local-map
    // update built on them
    void invalidate_from(int s) {
        for (; s < plp::kNumStages; ++s) record_batch[s] = 0;
        update_batch = 0;
    }
    // stage s left a record that covers the first `batch` (>= 1) frames
    bool covers(int s, int batch) const { return batch <= record_batch[s]; }
    // the call of stage s over `batch` frames ended in tail J
    void set_record(int s, int batch, const plp::TrackTail &J, const int32_t *local_idx,
                    const int32_t *local_idx_offsets) {
        record[s] = plp::TrackRecord{J.stage,   J.status,  J.matched, J.pose,    J.num_valid,
                                     J.posejobs, J.obs_row, J.rows,    local_idx, local_idx_offsets};
        record_batch[s] = batch;
    }
    // local-map tracking (plp_tracker_reserve_local_map); d_local == nullptr until reserved
    int max_local = 0;
    uint8_t *d_local = nullptr;      // one allocation, carved by local_map.cu
    // the job with that scratch bound and the predict_scale_level thresholds set; every call adds its own inputs
    std::shared_ptr<plp::lm::LocalDev> local;
    // keyframe tracking (plp_tracker_reserve_keyframe_track); d_kf == nullptr until reserved
    int max_keyframes = 0, max_kf_points = 0;
    uint8_t *d_kf = nullptr;         // one allocation, carved by keyframe_track.cu
    std::shared_ptr<plp::kt::KfDev> kf;
    int32_t *kf_choice = nullptr;    // the BoW matcher's scratch (max_batch x max_kf_points), reused by the robust stage
    plp_track_keyframe kf_table;     // the keyframe table of the keyframe record
    // robust tracking (plp_tracker_reserve_robust_track); d_rb == nullptr until reserved
    uint8_t *d_rb = nullptr;         // one allocation, carved by robust_track.cu
    std::shared_ptr<plp::rt::RtDev> rb;
    // local-map update (plp_tracker_reserve_local_map_update); d_upd == nullptr until reserved
    uint8_t *d_upd = nullptr;        // one allocation, carved by local_map_update.cu
    std::shared_ptr<plp::lu::UpdDev> upd;
    int upd_max_kf_points = 0;       // the keyframe rows its local_idx blocks hold
    // the update's list (pointers fixed by the reservation) and its keyframe local_idx blocks, which a local-map call
    // given that list reads in place of plp_track_keyframe.local_idx; the records themselves are never changed
    plp_track_local updated{};
    const int32_t *upd_local_idx = nullptr, *upd_local_idx_offsets = nullptr;
    // the batch of the most recent update, 0 once none stands (a tracking call or a new reservation ends it)
    int update_batch = 0;
};
