// robust_track.cu -- device-resident, frame-batched robust tracking:
//   frame_tracker::robust_match_based_track (module/frame_tracker.cc:192-245) =
//       robust::brute_force_match (Lowe 0.8, no orientation check) + essential_solver::find_via_ransac(50, false)
//     + pose_optimizer::optimize from the last frame's pose + discard_outliers
// for the frames of the tracker's most recent plp_tracker_keyframe_track_batch_dev that ran that stage and failed, on
// the same stream and without leaving HBM.  It reads the motion and keyframe calls' inputs, outputs and scratch
// (tracker.h) and writes separate outputs.  Device code: robust_track_kernels.cuh; the brute-force matcher
// (brute_match_kernel) and the tail (track_common.cuh) are the existing ones, and the eight-point solve and the score
// are plp_essential_ransac's (essential_common.cuh).
#include "common.cuh"
#include "match_kernels.cuh"
#include "robust_track_kernels.cuh"
#include "tracker.h"

namespace plp {

namespace {

size_t hypothesis_smem(int cap) { return (size_t)cap * 2 * sizeof(float); }

}  // namespace

}  // namespace plp

using namespace plp;

extern "C" {

plp_status plp_tracker_reserve_robust_track(plp_tracker *t) {
    PLP_REQUIRE(t, "null pointer");
    PLP_REQUIRE(t->cap <= kBruteMaxPoints, "kp_capacity exceeds the brute-force matcher's capacity (4096)");
    PLP_CUDA_TRY(cudaSetDevice(t->ctx->device));
    PLP_SMEM_OPTIN(rt::rt_hypothesis_kernel, hypothesis_smem(t->cap));  // one hypothesis' residuals
    if (t->d_rb) {  // a second reservation replaces the first once the stream has stopped using it
        PLP_CUDA_TRY(cudaStreamSynchronize(t->ctx->stream));
        cudaFree(t->d_rb);
        t->d_rb = nullptr;
        t->invalidate_from(kStageRobust);
    }
    // the scratch of every later call, bound once (B frames, C keypoints, K hypotheses)
    const size_t B = t->max_batch, C = t->cap, K = rt::kNumIter;
    auto D = std::make_shared<rt::RtDev>();
    memset(D.get(), 0, sizeof(rt::RtDev));
    DevLayout L;
    L.out(D->bjobs, B);
    L.out(D->pairs, B * C * 2);
    L.out(D->samples, B * K * 8);
    L.out(D->E, B * K * 9);
    L.out(D->score, B * K);
    L.out(D->inlier, B * C);
    L.out(D->best_score, B);
    L.out(D->valid, B);
    if (!t->distorted) L.out(D->bearings, B * C * 3);  // a distorted tracker's undistortion writes them
    TrackTail J = t->tail[kStageMotion];  // the tracker's cap and inv_level_sigma_sq; this stage's scratch
    L.out(J.posejobs, B);
    L.out(J.obs, B * C);
    L.out(J.obs_kp, B * C);
    L.out(J.obs_row, B * C);
    L.out(J.obs_outlier, B * C);
    if (alloc(t->ctx, L, &t->d_rb, false) != cudaSuccess) {
        set_error("tracker: cudaMalloc(%zu) for robust tracking failed", L.bytes());
        return PLP_ERR_CUDA;
    }
    D->cap = t->cap;
    if (t->distorted) {
        D->bearings = t->d_bearings;
    } else {  // convert_keypoints_to_bearings of the (undistorted) keypoints, with the camera's double parameters
        D->write_bearings = 1;
        D->K_cfg[0] = t->cam.fx;
        D->K_cfg[1] = t->cam.fy;
        D->K_cfg[2] = t->cam.cx;
        D->K_cfg[3] = t->cam.cy;
    }
    t->rb = D;
    t->tail[kStageRobust] = J;
    return PLP_OK;
}

plp_status plp_tracker_robust_track_batch_dev(plp_tracker *t, int batch, const double *d_kf_bearings, uint64_t seed,
                                              int32_t *d_stage_out, int32_t *d_kf_matched_out,
                                              int32_t *d_num_bf_matches_out, int32_t *d_num_robust_matches_out,
                                              double *d_pose_out, int32_t *d_num_valid_out, int32_t *d_n_inliers_out,
                                              int32_t *d_lm_iters_out, int32_t *d_status_out) {
    PLP_REQUIRE(t && d_kf_bearings && d_stage_out && d_kf_matched_out && d_num_bf_matches_out &&
                    d_num_robust_matches_out && d_pose_out && d_num_valid_out && d_n_inliers_out && d_lm_iters_out &&
                    d_status_out,
                "null pointer");
    PLP_REQUIRE(t->d_rb, "plp_tracker_reserve_robust_track has not been called");
    PLP_REQUIRE(batch >= 1 && batch <= t->max_batch, "batch exceeds the tracker's max_batch");
    PLP_REQUIRE(t->covers(kStageKeyframe, batch),
                "the batch must follow a plp_tracker_keyframe_track_batch_dev of at least as many frames");
    plp_ctx *ctx = t->ctx;
    PLP_CUDA_TRY(cudaSetDevice(ctx->device));
    t->invalidate_from(kStageRobust);
    const TrackDev &M = t->motion;
    const TrackRecord &KT = t->record[kStageKeyframe];
    const plp_track_keyframe &tab = t->kf_table;
    rt::RtDev D = *t->rb;
    D.batch = batch;
    D.seed = seed;
    D.max_kf_points = t->max_kf_points;
    D.n_kp = M.n_kp;
    D.x = M.x;
    D.y = M.y;
    D.desc = M.desc;
    D.kf_stage = KT.stage;
    D.kf_status = KT.status;
    D.kf_num_valid = KT.num_valid;
    D.kf_of_frame = tab.kf_of_frame;
    D.row_offsets = tab.row_offsets;
    D.kf_desc = tab.desc;
    D.kf_valid = tab.valid;
    D.kf_bearings = d_kf_bearings;
    D.choice = t->kf_choice;  // the keyframe call's matcher scratch (max_batch x max_keyframe_points), free again now
    D.stage = d_stage_out;
    D.status = d_status_out;
    D.matched = d_kf_matched_out;
    D.num_bf = d_num_bf_matches_out;
    D.num_robust = d_num_robust_matches_out;
    // pose-opt from last_frm.cam_pose_cw_ over the frames with 20 robust matches (frame_tracker.cc:203-245)
    TrackTail J = t->tail[kStageRobust];
    J.n_kp = M.n_kp;
    J.x = M.x;
    J.y = M.y;
    J.octave = M.octave;
    J.count = d_num_robust_matches_out;
    J.stage = d_stage_out;
    J.status = d_status_out;
    J.rows = KT.rows;  // the keyframe call's rows and kf_of_frame
    J.pose_in = M.pose_last;
    J.matched = d_kf_matched_out;
    J.pose = d_pose_out;
    J.num_valid = d_num_valid_out;
    J.n_inliers = d_n_inliers_out;
    J.lm_iters = d_lm_iters_out;

    PLP_LAUNCH(ctx, rt::rt_prep_kernel, div_up(batch, rt::kPrepThreads), rt::kPrepThreads, 0, D);
    PLP_CHECK_LAUNCH();
    PLP_TRY(launch_brute_match(ctx, D.bjobs, batch, t->cap, rt::kLoweRatio, 0));
    PLP_LAUNCH(ctx, rt::rt_list_kernel, batch, rt::kThreads, 0, D);
    PLP_CHECK_LAUNCH();
    PLP_LAUNCH(ctx, rt::rt_hypothesis_kernel, dim3(rt::kNumIter, batch), rt::kEssThreads, hypothesis_smem(t->cap), D);
    PLP_CHECK_LAUNCH();
    PLP_LAUNCH(ctx, rt::rt_select_kernel, batch, rt::kEssThreads, 0, D);
    PLP_CHECK_LAUNCH();
    PLP_TRY(launch_track_tail(ctx, J, batch, t->cam));
    t->set_record(kStageRobust, batch, J, KT.local_idx, KT.local_idx_offsets);  // the keyframe record's mapping
    return PLP_OK;
}

plp_status plp_tracker_robust_samples(const plp_tracker *t, const int32_t **d_samples) {
    PLP_REQUIRE(t && d_samples, "null pointer");
    PLP_REQUIRE(t->d_rb, "plp_tracker_reserve_robust_track has not been called");
    *d_samples = t->rb->samples;
    return PLP_OK;
}

}  // extern "C"
