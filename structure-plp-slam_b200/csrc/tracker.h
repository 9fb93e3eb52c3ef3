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
    const float *x_right;    // batch x cap: stereo_x_right_ (stereo trackers; null for monocular)
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

// the keyframe job's BoW matcher scratch (max_batch x max_kf_points), which the robust stage reuses once the keyframe
// call is done with it (keyframe_track.cu, where KfDev is complete)
int32_t *keyframe_choice(const plp_tracker *t);

// lays out the scratch of a tail job for B frames of C keypoints
inline void tail_scratch(DevLayout &L, TrackTail &J, size_t B, size_t C) {
    L.out(J.posejobs, B);
    L.out(J.obs, B * C);
    L.out(J.obs_kp, B * C);
    L.out(J.obs_row, B * C);
    L.out(J.obs_outlier, B * C);
}

// A stage's reservation: one device block carved into the scratch of the stage's job, which binds it.  The two are made
// and released together, so the job never outlives its block.
template <class Dev>
struct Reservation {
    uint8_t *block = nullptr;
    std::shared_ptr<Dev> job;  // null until reserved; a shared_ptr can be destroyed where Dev is only declared

    explicit operator bool() const { return job != nullptr; }
    Dev *operator->() const { return job.get(); }
    // frees the block once the stream has stopped using it; the reservation then no longer stands
    cudaError_t release(cudaStream_t stream) {
        if (!block) return cudaSuccess;
        const cudaError_t e = cudaStreamSynchronize(stream);
        if (e != cudaSuccess) return e;
        cudaFree(block);
        block = nullptr;
        job.reset();
        return cudaSuccess;
    }
    // replaces the reservation with one block laid out by L, whose pointers bind job D; `what` names the stage
    plp_status reserve(plp_ctx *ctx, DevLayout &L, std::shared_ptr<Dev> D, const char *what) {
        PLP_CUDA_TRY(release(ctx->stream));
        if (alloc(ctx, L, &block, false) != cudaSuccess) {
            set_error("tracker: cudaMalloc(%zu) for %s failed", L.bytes(), what);
            return PLP_ERR_CUDA;
        }
        job = std::move(D);
        return PLP_OK;
    }
};

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
    // a stereo tracker's current-frame stereo_x_right_ (plp_tracker_bind_stereo): max_batch x cap, caller-owned
    const float *d_x_right = nullptr;
    bool stereo() const { return cam.setup_type == 1; }
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
    // stage s's record if it stands, else one whose stage is null
    plp::TrackRecord standing(int s) const { return record_batch[s] ? record[s] : plp::TrackRecord{}; }
    // The order of a batch's calls, for a call of stage s over `batch` frames; s == kNumStages stands for the local-map
    // update and local-map calls.  The keyframe call follows a motion call and the robust call a keyframe call, of at
    // least as many frames.  The local-map calls follow a motion call and start each frame from the last record that
    // ran on it, so a keyframe or robust record that stands must cover the batch too.
    plp_status check_order(int s, int batch) const {
        PLP_REQUIRE(batch >= 1 && batch <= max_batch, "batch exceeds the tracker's max_batch");
        PLP_REQUIRE(!stereo() || d_x_right, "a stereo tracker needs plp_tracker_bind_stereo first");
        if (s == plp::kStageRobust)
            PLP_REQUIRE(covers(plp::kStageKeyframe, batch),
                        "the batch must follow a plp_tracker_keyframe_track_batch_dev of at least as many frames");
        else if (s != plp::kStageMotion)
            PLP_REQUIRE(covers(plp::kStageMotion, batch),
                        "the batch must follow a plp_tracker_motion_track_batch_dev of at least as many frames");
        if (s == plp::kNumStages) {
            PLP_REQUIRE(!record_batch[plp::kStageKeyframe] || covers(plp::kStageKeyframe, batch),
                        "the batch must not exceed that of the plp_tracker_keyframe_track_batch_dev that followed the "
                        "motion track");
            PLP_REQUIRE(!record_batch[plp::kStageRobust] || covers(plp::kStageRobust, batch),
                        "the batch must not exceed that of the plp_tracker_robust_track_batch_dev that followed the "
                        "keyframe track");
        }
        return PLP_OK;
    }
    // stage s's tail job over the current frames of the motion call, writing the caller's outputs; the stage adds its
    // gate (count, stage, status), its rows and its starting pose
    plp::TrackTail tail_job(int s, int32_t *matched, double *pose, int32_t *num_valid, int32_t *n_inliers,
                            int32_t *lm_iters) const {
        plp::TrackTail J = tail[s];
        J.n_kp = motion.n_kp;
        J.x = motion.x;
        J.y = motion.y;
        J.octave = motion.octave;
        J.x_right = motion.x_right;
        J.matched = matched;
        J.pose = pose;
        J.num_valid = num_valid;
        J.n_inliers = n_inliers;
        J.lm_iters = lm_iters;
        return J;
    }
    // the call of stage s over `batch` frames ended in tail J
    void set_record(int s, int batch, const plp::TrackTail &J, const int32_t *local_idx,
                    const int32_t *local_idx_offsets) {
        record[s] = plp::TrackRecord{J.stage,   J.status,  J.matched, J.pose,    J.num_valid,
                                     J.posejobs, J.obs_row, J.rows,    local_idx, local_idx_offsets};
        record_batch[s] = batch;
    }
    // local-map tracking (plp_tracker_reserve_local_map): the job with its scratch bound and the predict_scale_level
    // thresholds set; every call adds its own inputs
    int max_local = 0;
    plp::Reservation<plp::lm::LocalDev> local;
    // keyframe tracking (plp_tracker_reserve_keyframe_track)
    int max_keyframes = 0, max_kf_points = 0;
    plp::Reservation<plp::kt::KfDev> kf;
    plp_track_keyframe kf_table;     // the keyframe table of the keyframe record
    // robust tracking (plp_tracker_reserve_robust_track)
    plp::Reservation<plp::rt::RtDev> rb;
    // local-map update (plp_tracker_reserve_local_map_update)
    plp::Reservation<plp::lu::UpdDev> upd;
    int upd_max_kf_points = 0;       // the keyframe rows its local_idx blocks hold
    // the update's list (pointers fixed by the reservation) and its keyframe local_idx blocks, which a local-map call
    // given that list reads in place of plp_track_keyframe.local_idx; the records themselves are never changed
    plp_track_local updated{};
    const int32_t *upd_local_idx = nullptr, *upd_local_idx_offsets = nullptr;
    // the batch of the most recent update, 0 once none stands (a tracking call or a new reservation ends it)
    int update_batch = 0;
};
