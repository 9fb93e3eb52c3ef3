// local_map.cu -- device-resident, frame-batched local-map tracking:
//   tracking_module::optimize_current_frame_with_local_map (tracking_module.cc:732-835) =
//       search_local_landmarks (frame::can_observe + projection::match_frame_and_landmarks, Lowe ratio 0.8)
//     + pose_optimizer::optimize + the outlier drop and tracked-landmark count
// for the batch of the tracker's most recent plp_tracker_motion_track_batch_dev, on the same stream and without leaving
// HBM.  Each frame starts from the last tracking stage that ran on it: the records of the motion call and of the
// keyframe and robust calls that followed it (tracker.h).  It reads those calls' inputs, outputs and scratch and writes
// separate outputs, so theirs stay as they wrote them.  Device code: local_map_kernels.cuh.  The window matcher (ratio path) and the
// pose optimiser are the existing launchers, and the predict_scale_level table is plp_fuse_level_thresholds'.
//
// This file is compiled with -fmad=false (build.py FILE_FLAGS): can_observe's double / float mix rounds like the oracle.
#include "common.cuh"
#include "local_map_kernels.cuh"
#include "match_kernels.cuh"
#include "pose_kernels.cuh"
#include "tracker.h"

namespace plp {

namespace {

using lm::LocalDev;
using lm::local_finish_kernel;
using lm::local_gather_kernel;
using lm::local_observe_kernel;
using lm::local_prep_kernel;

}  // namespace

}  // namespace plp

using namespace plp;

extern "C" {

plp_status plp_tracker_reserve_local_map(plp_tracker *t, float log_scale_factor, int max_local_points) {
    PLP_REQUIRE(t, "null pointer");
    PLP_REQUIRE(max_local_points >= 1, "max_local_points");
    float thr[16];
    PLP_TRY(plp_fuse_level_thresholds(log_scale_factor, t->num_levels, thr));
    PLP_CUDA_TRY(cudaSetDevice(t->ctx->device));
    if (t->d_local) {  // a second reservation replaces the first once the stream has stopped using it
        PLP_CUDA_TRY(cudaStreamSynchronize(t->ctx->stream));
        cudaFree(t->d_local);
        t->d_local = nullptr;
        t->max_local = 0;
    }
    // the scratch of every later call, bound once (B frames, C keypoints, ML local rows)
    const size_t B = t->max_batch, C = t->cap, ML = max_local_points;
    auto D = std::make_shared<LocalDev>();
    memset(D.get(), 0, sizeof(LocalDev));
    DevLayout L;
    L.out(D->excl, B * ML);
    L.out(D->center, B * 3);
    L.out(D->qx, B * ML);
    L.out(D->qy, B * ML);
    L.out(D->qradius, B * ML);
    L.out(D->qmin, B * ML);
    L.out(D->qmax, B * ML);
    L.out(D->qvalid, B * ML);
    L.out(D->choice, B * ML);
    L.out(D->best, B * ML);
    L.out(D->num_matches, B);
    L.out(D->claimed, B * C);
    L.out(D->mjobs, B);
    L.out(D->posejobs, B);
    L.out(D->obs, B * C);
    L.out(D->obs_kp, B * C);
    L.out(D->obs_outlier, B * C);
    if (alloc(t->ctx, L, &t->d_local, false) != cudaSuccess) {
        set_error("tracker: cudaMalloc(%zu) for the local map failed", L.bytes());
        return PLP_ERR_CUDA;
    }
    t->max_local = max_local_points;
    D->cap = t->cap;
    D->max_local = t->max_local;
    D->cam = t->cam;
    for (int l = 0; l < 16; ++l) {
        D->scale_factors[l] = l < t->num_levels ? t->scale_factors[l] : 1.0f;
        D->level_thr[l] = l < t->num_levels ? thr[l] : INFINITY;
    }
    D->num_levels = t->num_levels;
    t->local = D;
    return PLP_OK;
}

plp_status plp_tracker_local_map_track_batch_dev(plp_tracker *t, int batch, const plp_track_local *local, float margin,
                                                 int32_t *d_matched_out, int32_t *d_local_out, uint8_t *d_observable_out,
                                                 double *d_pose_out, int32_t *d_num_tracked_out, int32_t *d_n_inliers_out,
                                                 int32_t *d_lm_iters_out, int32_t *d_status_out) {
    PLP_REQUIRE(t && local && d_matched_out && d_local_out && d_observable_out && d_pose_out && d_num_tracked_out &&
                    d_n_inliers_out && d_lm_iters_out && d_status_out,
                "null pointer");
    PLP_REQUIRE(local->pos_w && local->obs_mean_normal && local->min_valid_dist && local->max_valid_dist &&
                    local->max_valid_dist_raw && local->desc && local->offsets && local->last_local_idx,
                "local-map arrays");
    PLP_REQUIRE(t->d_local, "plp_tracker_reserve_local_map has not been called");
    PLP_REQUIRE(batch >= 1 && batch <= t->max_batch, "batch exceeds the tracker's max_batch");
    PLP_REQUIRE(t->covers(kStageMotion, batch),
                "the batch must follow a plp_tracker_motion_track_batch_dev of at least as many frames");
    PLP_REQUIRE(!t->record_batch[kStageKeyframe] || t->covers(kStageKeyframe, batch),
                "the batch must not exceed that of the plp_tracker_keyframe_track_batch_dev that followed the motion track");
    PLP_REQUIRE(!t->record_batch[kStageRobust] || t->covers(kStageRobust, batch),
                "the batch must not exceed that of the plp_tracker_robust_track_batch_dev that followed the keyframe track");
    PLP_REQUIRE(margin > 0.0f, "margin");
    plp_ctx *ctx = t->ctx;
    PLP_CUDA_TRY(cudaSetDevice(ctx->device));
    const TrackDev &M = t->motion;
    LocalDev D = *t->local;
    D.batch = batch;
    D.n_kp = M.n_kp;
    D.x = M.x;
    D.y = M.y;
    D.octave = M.octave;
    D.desc = M.desc;
    for (int l = 0; l < 16; ++l) D.inv_level_sigma_sq[l] = t->tail[kStageMotion].inv_level_sigma_sq[l];
    D.motion = t->record[kStageMotion];
    D.motion.local_idx = local->last_local_idx;  // one entry per last-frame row
    D.motion.local_idx_offsets = M.last_offsets;
    if (t->record_batch[kStageKeyframe]) D.kf = t->record[kStageKeyframe];  // else D.kf.stage stays null
    if (t->record_batch[kStageRobust]) D.rb = t->record[kStageRobust];      // else D.rb.stage stays null
    D.pos_w = local->pos_w;
    D.normal = local->obs_mean_normal;
    D.min_d = local->min_valid_dist;
    D.max_d = local->max_valid_dist;
    D.max_raw = local->max_valid_dist_raw;
    D.lm_desc = local->desc;
    D.valid = local->valid;
    D.offsets = local->offsets;
    D.margin = margin;
    D.matched = d_matched_out;
    D.local = d_local_out;
    D.observable = d_observable_out;
    D.pose = d_pose_out;
    D.num_tracked = d_num_tracked_out;
    D.n_inliers = d_n_inliers_out;
    D.lm_iters = d_lm_iters_out;
    D.status = d_status_out;

    PLP_LAUNCH(ctx, local_prep_kernel, batch, lm::kThreads, 0, D);
    PLP_CHECK_LAUNCH();
    const dim3 ogrid(div_up(t->max_local, lm::kObserveThreads), batch);
    PLP_LAUNCH(ctx, local_observe_kernel, ogrid, lm::kObserveThreads, 0, D);
    PLP_CHECK_LAUNCH();
    // projection::match_frame_and_landmarks: ratio test, no orientation check, claims resolved in local-list order
    PLP_TRY(launch_point_match(ctx, D.mjobs, batch, t->cap > kMatchMaxPoints ? kMatchMaxPoints : t->cap, t->grid, 1,
                               lm::kLoweRatio, 0));
    PLP_LAUNCH(ctx, local_gather_kernel, batch, lm::kThreads, 0, D);
    PLP_CHECK_LAUNCH();
    plp_pose_opt_cfg cfg{4, 10};
    PLP_TRY(launch_pose_opt(ctx, D.posejobs, batch, t->cam, cfg));
    PLP_LAUNCH(ctx, local_finish_kernel, batch, lm::kThreads, 0, D);
    PLP_CHECK_LAUNCH();
    return PLP_OK;
}

}  // extern "C"
