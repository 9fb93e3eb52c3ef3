// robust_track.cu -- device-resident, frame-batched robust tracking:
//   frame_tracker::robust_match_based_track (module/frame_tracker.cc:192-245) =
//       robust::brute_force_match (Lowe 0.8, no orientation check) + essential_solver::find_via_ransac(50, false)
//     + pose_optimizer::optimize from the last frame's pose + discard_outliers
// for the frames of the tracker's most recent plp_tracker_keyframe_track_batch_dev that ran that stage and failed, on
// the same stream and without leaving HBM.  It reads the motion and keyframe calls' inputs, outputs and scratch
// (tracker.h) and writes separate outputs.  Device code: robust_track_kernels.cuh; the brute-force matcher
// (brute_match_kernel), the keyframe tracker's gather and finish kernels and the pose optimiser are the existing ones,
// and the eight-point solve and the score are plp_essential_ransac's (essential_common.cuh).
#include "common.cuh"
#include "keyframe_track_kernels.cuh"
#include "match_kernels.cuh"
#include "pose_kernels.cuh"
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
    // the hypothesis kernel's residuals in dynamic shared memory, next to its static shared memory, within the opt-in
    // limit (the attribute is per kernel: it allows the most any tracker can ask for)
    int optin = 0;
    cudaFuncAttributes fa;
    PLP_CUDA_TRY(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, t->ctx->device));
    PLP_CUDA_TRY(cudaFuncGetAttributes(&fa, rt::rt_hypothesis_kernel));
    PLP_REQUIRE(hypothesis_smem(t->cap) + fa.sharedSizeBytes <= (size_t)optin,
                "kp_capacity too large for the hypothesis kernel's shared memory");
    PLP_CUDA_TRY(cudaFuncSetAttribute(rt::rt_hypothesis_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      optin - (int)fa.sharedSizeBytes));
    if (t->d_rb) {  // a second reservation replaces the first once the stream has stopped using it
        PLP_CUDA_TRY(cudaStreamSynchronize(t->ctx->stream));
        cudaFree(t->d_rb);
        t->d_rb = nullptr;
        t->has_rb = false;
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
    L.out(D->posejobs, B);
    L.out(D->obs, B * C);
    L.out(D->obs_kp, B * C);
    L.out(D->obs_row, B * C);
    L.out(D->obs_outlier, B * C);
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
    PLP_REQUIRE(t->has_kf && batch <= t->kf_batch,
                "the batch must follow a plp_tracker_keyframe_track_batch_dev of at least as many frames");
    plp_ctx *ctx = t->ctx;
    PLP_CUDA_TRY(cudaSetDevice(ctx->device));
    t->has_rb = false;
    const TrackDev &M = t->motion;
    const KeyframeTrack &KT = t->kf_track;
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
    D.choice = t->kf->choice;  // the keyframe call's matcher scratch (max_batch x max_keyframe_points), free again now
    D.stage = d_stage_out;
    D.status = d_status_out;
    D.matched = d_kf_matched_out;
    D.num_bf = d_num_bf_matches_out;
    D.num_robust = d_num_robust_matches_out;
    // the keyframe tracker's gather and finish over this stage's matches: the robust count stands for the BoW count
    kt::KfDev G;
    memset(&G, 0, sizeof(G));
    G.batch = batch;
    G.cap = t->cap;
    G.n_kp = M.n_kp;
    G.x = M.x;
    G.y = M.y;
    G.octave = M.octave;
    G.pose_last = M.pose_last;
    for (int l = 0; l < kt::kMaxLevels; ++l) G.inv_level_sigma_sq[l] = M.inv_level_sigma_sq[l];
    G.kf_of_frame = tab.kf_of_frame;
    G.row_offsets = tab.row_offsets;
    G.kf_pos_w = tab.pos_w;
    G.posejobs = D.posejobs;
    G.obs = D.obs;
    G.obs_kp = D.obs_kp;
    G.obs_row = D.obs_row;
    G.obs_outlier = D.obs_outlier;
    G.stage = d_stage_out;
    G.status = d_status_out;
    G.matched = d_kf_matched_out;
    G.num_bow = (uint32_t *)d_num_robust_matches_out;
    G.pose = d_pose_out;
    G.num_valid = d_num_valid_out;
    G.n_inliers = d_n_inliers_out;
    G.lm_iters = d_lm_iters_out;

    PLP_LAUNCH(ctx, rt::rt_prep_kernel, div_up(batch, rt::kPrepThreads), rt::kPrepThreads, 0, D);
    PLP_CHECK_LAUNCH();
    PLP_TRY(launch_brute_match(ctx, D.bjobs, batch, t->cap, rt::kLoweRatio, 0));
    PLP_LAUNCH(ctx, rt::rt_list_kernel, batch, rt::kThreads, 0, D);
    PLP_CHECK_LAUNCH();
    PLP_LAUNCH(ctx, rt::rt_hypothesis_kernel, dim3(rt::kNumIter, batch), rt::kEssThreads, hypothesis_smem(t->cap), D);
    PLP_CHECK_LAUNCH();
    PLP_LAUNCH(ctx, rt::rt_select_kernel, batch, rt::kEssThreads, 0, D);
    PLP_CHECK_LAUNCH();
    PLP_LAUNCH(ctx, kt::kf_gather_kernel, batch, kt::kThreads, 0, G);
    PLP_CHECK_LAUNCH();
    plp_pose_opt_cfg cfg{4, 10};
    PLP_TRY(launch_pose_opt(ctx, D.posejobs, batch, t->cap, t->cam, cfg));
    PLP_LAUNCH(ctx, kt::kf_finish_kernel, batch, kt::kThreads, 0, G);
    PLP_CHECK_LAUNCH();

    KeyframeTrack &R = t->rb_track;
    R = KT;  // the same keyframe rows, kf_of_frame and local_idx mapping
    R.stage = d_stage_out;
    R.status = d_status_out;
    R.matched = d_kf_matched_out;
    R.pose = d_pose_out;
    R.num_valid = d_num_valid_out;
    R.posejobs = D.posejobs;
    R.obs_row = D.obs_row;
    t->rb_batch = batch;
    t->has_rb = true;
    return PLP_OK;
}

plp_status plp_tracker_robust_samples(const plp_tracker *t, const int32_t **d_samples) {
    PLP_REQUIRE(t && d_samples, "null pointer");
    PLP_REQUIRE(t->d_rb, "plp_tracker_reserve_robust_track has not been called");
    *d_samples = t->rb->samples;
    return PLP_OK;
}

}  // extern "C"
