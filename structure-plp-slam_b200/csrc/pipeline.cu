// pipeline.cu -- device-resident, frame-batched tracking front-end:
//   frame_tracker::motion_based_track (module/frame_tracker.cc:52-124) =
//       projection::match_current_and_last_frames (margin, retry with 2*margin below 20 matches)
//     + pose_optimizer::optimize + discard_outliers (frame_tracker.cc:253-283)
// chained after orb_extractor::extract without leaving HBM.  This is the "extract + match + pose-opt" hot loop
// of BASELINE.json for a batch of independent (frame, last-frame-landmarks, predicted pose) triples -- SURVEY.md
// section 8(e): a live sequence is sequential, so the batch is made of independent tracking problems (offline /
// multi-sequence mode); each CTA handles one frame.
//
// The keypoints of the current frames are taken from the ORB handle's most recent extraction.  A tracker made with a
// distortion (plp_tracker_create_ex) first undistorts them (camera::*::undistort_keypoints, camera_kernels.cuh) into
// arrays of its own, so that the grid, the window queries and the pose optimiser's observations read undist_keypts_ as
// the reference's do (frame.cc:68-86); the octave and angle are those of the ORB keypoints.  Without distortion
// (plp_tracker_create, or a perspective model with all coefficients 0) undistortion returns every keypoint coordinate
// bit for bit, so the ORB keypoints are used as they are and no kernel is added.
#include "common.cuh"
#include "camera_kernels.cuh"
#include "match_kernels.cuh"
#include "pose_kernels.cuh"
#include "track_common.cuh"
#include "tracker.h"

namespace plp {

namespace {

__global__ void track_prep_kernel(TrackDev T, float margin, int check_orientation) {
    const int b = blockIdx.x, tid = threadIdx.x;
    const int n = T.n_kp[b];
    const size_t base = (size_t)b * T.cap;
    for (int i = tid; i < n; i += blockDim.x) {
        const plp_keypoint k = T.kp[base + i];
        T.x[base + i] = k.x;
        T.y[base + i] = k.y;
        T.angle[base + i] = k.angle;
        T.octave[base + i] = k.octave;
    }
    if (tid == 0) {
        const int l0 = T.last_offsets[b], m = T.last_offsets[b + 1] - l0;
        for (int attempt = 0; attempt < 2; ++attempt) {
            ProjectJob P;
            P.n_last = m;
            P.pos_w = T.last_pos_w + 3 * (size_t)l0;
            P.octave = T.last_octave + l0;
            P.valid = T.last_valid ? T.last_valid + l0 : nullptr;
            for (int k = 0; k < 12; ++k) P.pose_cw[k] = T.pose_pred[16 * (size_t)b + k];
            P.assume_forward = 0;  // monocular (projection.cc:231-238)
            P.assume_backward = 0;
            const size_t qb = (size_t)b * T.max_last;
            P.qx = T.qx + qb;
            P.qy = T.qy + qb;
            P.qxr = T.qxr + qb;
            P.qx2 = P.qy2 = P.qxr2 = nullptr;
            P.qradius = T.qradius + qb;
            P.qmin = T.qmin + qb;
            P.qmax = T.qmax + qb;
            P.qvalid = T.qvalid + qb;
            PointMatchJob J;
            J.n = n;
            J.x = T.x + base;
            J.y = T.y + base;
            J.octave = T.octave + base;
            J.angle = T.angle + base;
            J.x_right = nullptr;
            J.desc = T.desc + base * 32;
            J.claimed = nullptr;  // curr_frm.landmarks_ was just cleared (frame_tracker.cc:61)
            J.hamm_thr_p1 = 0;
            J.m = m;
            J.qx = P.qx;
            J.qy = P.qy;
            J.qxr = P.qxr;
            J.qradius = P.qradius;
            J.qmin = P.qmin;
            J.qmax = P.qmax;
            J.qangle = T.last_angle + l0;
            J.qdesc = T.last_desc + (size_t)l0 * 32;
            J.qvalid = P.qvalid;
            J.choice = T.choice + qb;
            J.best_idx_out = nullptr;
            J.matched_out = T.matched + base;
            J.num_matches = T.num_matches + b;
            T.pjobs[attempt * T.batch + b] = P;
            T.mjobs[attempt * T.batch + b] = J;
        }
    }
}

// disable the widened-margin retry for frames whose first attempt reached the threshold (frame_tracker.cc:66-71)
__global__ void track_retry_gate_kernel(TrackDev T) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= T.batch) return;
    if (T.num_matches[b] >= (uint32_t)kNumMatchesThr) {
        T.pjobs[T.batch + b].n_last = -1;
        T.mjobs[T.batch + b].m = -1;
    }
}

}  // namespace

plp_status launch_track_tail(plp_ctx *ctx, const TrackTail &J, int batch, const plp_camera &cam) {
    PLP_LAUNCH(ctx, track_gather_kernel, batch, kTailThreads, 0, J);
    PLP_CHECK_LAUNCH();
    plp_pose_opt_cfg cfg{4, 10};
    PLP_TRY(launch_pose_opt(ctx, J.posejobs, batch, cam, cfg));
    PLP_LAUNCH(ctx, track_finish_kernel, batch, kTailThreads, 0, J);
    PLP_CHECK_LAUNCH();
    return PLP_OK;
}

}  // namespace plp

using namespace plp;

namespace plp {
plp_status make_undist_job(const plp_camera *cam, const plp_distortion *dist, UndistJob *J);  // camera.cu
bool distortion_is_identity(const plp_distortion *dist);
plp_status launch_undistort(plp_ctx *ctx, const UndistJob &J);
}  // namespace plp

extern "C" {

plp_status plp_tracker_create(plp_ctx *ctx, const plp_camera *cam, const plp_grid *grid, const float *scale_factors,
                              const float *inv_level_sigma_sq, int num_levels, int max_batch, int kp_capacity,
                              int max_last_points, plp_tracker **out) {
    return plp_tracker_create_ex(ctx, cam, grid, scale_factors, inv_level_sigma_sq, num_levels, max_batch, kp_capacity,
                                 max_last_points, nullptr, out);
}

plp_status plp_tracker_create_ex(plp_ctx *ctx, const plp_camera *cam, const plp_grid *grid, const float *scale_factors,
                                 const float *inv_level_sigma_sq, int num_levels, int max_batch, int kp_capacity,
                                 int max_last_points, const plp_distortion *dist, plp_tracker **out) {
    PLP_REQUIRE(ctx && cam && grid && scale_factors && inv_level_sigma_sq && out, "null pointer");
    const bool distorted = !distortion_is_identity(dist);
    UndistJob uj;
    if (distorted) PLP_TRY(make_undist_job(cam, dist, &uj));
    PLP_REQUIRE(num_levels >= 1 && num_levels <= 16 && max_batch >= 1 && kp_capacity >= 1 && max_last_points >= 1, "sizes");
    PLP_REQUIRE(cam->setup_type == 0, "the batched tracker implements the monocular path");
    *out = nullptr;
    PLP_CUDA_TRY(cudaSetDevice(ctx->device));
    plp_tracker *t = new plp_tracker();
    t->ctx = ctx;
    t->max_batch = max_batch;
    t->cap = kp_capacity;
    t->max_last = max_last_points;
    t->num_levels = num_levels;
    t->cam = *cam;
    t->grid = *grid;
    for (int l = 0; l < num_levels; ++l) {
        t->scale_factors[l] = scale_factors[l];
        t->inv_level_sigma_sq[l] = inv_level_sigma_sq[l];
    }
    const size_t B = max_batch, C = kp_capacity, M = max_last_points;
    DevLayout L;
    L.in(t->d_scale_factors, t->scale_factors, num_levels, 16);
    TrackDev &T = t->dev;
    memset(&T, 0, sizeof(T));
    T.cap = kp_capacity;
    T.num_levels = num_levels;
    T.max_last = max_last_points;
    L.out(T.x, B * C);
    L.out(T.y, B * C);
    L.out(T.angle, B * C);
    L.out(T.octave, B * C);
    L.out(T.qx, B * M);
    L.out(T.qy, B * M);
    L.out(T.qxr, B * M);
    L.out(T.qradius, B * M);
    L.out(T.qmin, B * M);
    L.out(T.qmax, B * M);
    L.out(T.qvalid, B * M);
    L.out(T.choice, B * M);
    L.out(T.num_matches, B);
    L.out(T.pjobs, 2 * B);
    L.out(T.mjobs, 2 * B);
    TrackTail &J = t->tail[kStageMotion];
    memset(&J, 0, sizeof(J));
    J.cap = kp_capacity;
    for (int l = 0; l < 16; ++l) J.inv_level_sigma_sq[l] = l < num_levels ? inv_level_sigma_sq[l] : 1.0f;
    L.out(J.posejobs, B);
    L.out(J.obs, B * C);
    L.out(J.obs_kp, B * C);
    L.out(J.obs_outlier, B * C);
    L.out(J.obs_row, B * C);
    if (distorted) {
        t->distorted = true;
        t->undist = uj;
        L.out(t->d_undist, B * C);
        L.out(t->d_bearings, B * C * 3);
    }
    const cudaError_t e = alloc(ctx, L, &t->d_block, false);
    if (!t->d_block) {
        set_error("tracker: cudaMalloc(%zu) failed", L.bytes());
        delete t;
        return PLP_ERR_CUDA;
    }
    if (e != cudaSuccess) {
        set_error("tracker: upload failed: %s", cudaGetErrorString(e));
        plp_tracker_destroy(t);
        return PLP_ERR_CUDA;
    }
    *out = t;
    return PLP_OK;
}

plp_status plp_tracker_undistorted(const plp_tracker *t, const plp_keypoint **d_undist_kp, const double **d_bearings) {
    PLP_REQUIRE(t && d_undist_kp && d_bearings, "null pointer");
    PLP_REQUIRE(t->distorted, "the tracker has no distortion: its undistorted keypoints are the ORB keypoints");
    *d_undist_kp = t->d_undist;
    *d_bearings = t->d_bearings;
    return PLP_OK;
}

void plp_tracker_destroy(plp_tracker *t) {
    if (!t) return;
    cudaSetDevice(t->ctx->device);
    cudaStreamSynchronize(t->ctx->stream);
    if (t->d_block) cudaFree(t->d_block);
    if (t->d_local) cudaFree(t->d_local);
    if (t->d_kf) cudaFree(t->d_kf);
    if (t->d_rb) cudaFree(t->d_rb);
    delete t;
}

plp_status plp_tracker_motion_track_batch_dev(plp_tracker *t, int batch, const plp_keypoint *d_kp, const uint8_t *d_desc,
                                              const int32_t *d_n_kp, const plp_track_last *last, float margin,
                                              int32_t *d_matched_out, double *d_pose_out, int32_t *d_num_valid_out,
                                              int32_t *d_n_inliers_out, int32_t *d_lm_iters_out) {
    PLP_REQUIRE(t && d_kp && d_desc && d_n_kp && last && d_matched_out && d_pose_out && d_num_valid_out &&
                    d_n_inliers_out && d_lm_iters_out,
                "null pointer");
    PLP_REQUIRE(batch >= 1 && batch <= t->max_batch, "batch exceeds the tracker's max_batch");
    PLP_REQUIRE(last->pos_w && last->octave && last->angle && last->desc && last->offsets && last->pose_pred &&
                    last->pose_last,
                "last-frame arrays");
    plp_ctx *ctx = t->ctx;
    t->invalidate_from(kStageMotion);
    PLP_CUDA_TRY(cudaSetDevice(ctx->device));
    TrackDev T = t->dev;
    T.batch = batch;
    T.kp = d_kp;
    T.desc = d_desc;
    T.n_kp = d_n_kp;
    T.last_pos_w = last->pos_w;
    T.last_octave = last->octave;
    T.last_angle = last->angle;
    T.last_desc = last->desc;
    T.last_valid = last->valid;
    T.last_offsets = last->offsets;
    T.pose_pred = last->pose_pred;
    T.pose_last = last->pose_last;
    T.matched = d_matched_out;
    if (t->distorted) {  // frame.cc:68,79: undist_keypts_ and bearings_ of the current frames
        UndistJob J = t->undist;
        J.batch = batch;
        J.cap = t->cap;
        J.kp = d_kp;
        J.n_kp = d_n_kp;
        J.out = t->d_undist;
        J.bearings = t->d_bearings;
        PLP_TRY(launch_undistort(ctx, J));
        T.kp = t->d_undist;
    }
    PLP_LAUNCH(ctx, track_prep_kernel, batch, 256, 0, T, margin, 1);
    PLP_CHECK_LAUNCH();
    // first attempt (projection.cc:214-358 with `margin`)
    PLP_TRY(launch_project_points(ctx, T.pjobs, batch, t->max_last, t->cam, t->d_scale_factors, t->num_levels, margin));
    PLP_TRY(launch_point_match(ctx, T.mjobs, batch, t->cap > kMatchMaxPoints ? kMatchMaxPoints : t->cap, t->grid, 0, 0.0f, 1));
    // widened retry for the frames that found fewer than 20 matches (frame_tracker.cc:66-71)
    PLP_LAUNCH(ctx, track_retry_gate_kernel, div_up(batch, 128), 128, 0, T);
    PLP_CHECK_LAUNCH();
    PLP_TRY(launch_project_points(ctx, T.pjobs + batch, batch, t->max_last, t->cam, t->d_scale_factors, t->num_levels,
                                  2 * margin));
    PLP_TRY(launch_point_match(ctx, T.mjobs + batch, batch, t->cap > kMatchMaxPoints ? kMatchMaxPoints : t->cap, t->grid,
                               0, 0.0f, 1));
    // pose-opt from the predicted pose over the frames with 20 matches (frame_tracker.cc:73-108)
    TrackTail J = t->tail[kStageMotion];
    J.n_kp = d_n_kp;
    J.x = T.x;
    J.y = T.y;
    J.octave = T.octave;
    J.count = (const int32_t *)T.num_matches;  // the matcher's count (uint32_t), far below 2^31
    J.rows = TrackRows{T.last_pos_w, T.last_offsets, nullptr};
    J.pose_in = T.pose_pred;
    J.matched = d_matched_out;
    J.pose = d_pose_out;
    J.num_valid = d_num_valid_out;
    J.n_inliers = d_n_inliers_out;
    J.lm_iters = d_lm_iters_out;
    PLP_TRY(launch_track_tail(ctx, J, batch, t->cam));
    t->motion = T;
    t->set_record(kStageMotion, batch, J, nullptr, nullptr);  // local_map.cu binds last_local_idx
    return PLP_OK;
}

}  // extern "C"
