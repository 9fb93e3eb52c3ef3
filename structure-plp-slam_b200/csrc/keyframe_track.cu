// keyframe_track.cu -- device-resident, frame-batched keyframe tracking:
//   frame_tracker::bow_match_based_track (module/frame_tracker.cc:126-189) =
//       frame::compute_bow + bow_tree::match_frame_and_keyframe (Lowe 0.7, orientation check)
//     + pose_optimizer::optimize from the last frame's pose + discard_outliers
// for the frames of the tracker's most recent plp_tracker_motion_track_batch_dev that the reference hands to it (motion
// model unusable, or motion track failed), on the same stream and without leaving HBM.  It reads that call's inputs and
// scratch (tracker.h) and writes separate outputs.  Device code: keyframe_track_kernels.cuh; the BoW matcher
// (bow_match_kernel) and the pose optimiser are the existing ones, the vocabulary descent is bow_transform_kernel's.
#include "common.cuh"
#include "bow_vocab.h"
#include "keyframe_track_kernels.cuh"
#include "pose_kernels.cuh"
#include "tracker.h"

namespace plp {

namespace {

using kt::KfDev;

plp_status launch_kf_transform(plp_ctx *ctx, const plp_bow_vocab *v, const KfDev &D, int batch) {
    const VocabDev V = vocab_dev(v);
    const int nid_level = v->L - kt::kLevelsUp;
    const int G = transform_group(v);
    const dim3 grid(div_up(D.cap, 256 / G), batch);
    switch (G) {
        case 4:
            PLP_LAUNCH(ctx, kt::kf_transform_kernel<4>, grid, 256, 0, D, V, nid_level);
            break;
        case 8:
            PLP_LAUNCH(ctx, kt::kf_transform_kernel<8>, grid, 256, 0, D, V, nid_level);
            break;
        case 16:
            PLP_LAUNCH(ctx, kt::kf_transform_kernel<16>, grid, 256, 0, D, V, nid_level);
            break;
        default:
            PLP_LAUNCH(ctx, kt::kf_transform_kernel<32>, grid, 256, 0, D, V, nid_level);
            break;
    }
    PLP_CHECK_LAUNCH();
    return PLP_OK;
}

size_t job_smem(int cap) { return (size_t)cap * (sizeof(unsigned long long) + sizeof(uint32_t)); }

}  // namespace

}  // namespace plp

using namespace plp;

extern "C" {

plp_status plp_tracker_reserve_keyframe_track(plp_tracker *t, int max_keyframes, int max_keyframe_points) {
    PLP_REQUIRE(t, "null pointer");
    PLP_REQUIRE(max_keyframes >= 1 && max_keyframe_points >= 1, "max_keyframes / max_keyframe_points");
    PLP_CUDA_TRY(cudaSetDevice(t->ctx->device));
    // The feature-vector kernel's dynamic shared memory, next to its static shared memory, within the opt-in limit.  The
    // attribute is per kernel, not per tracker: it allows the most any tracker can ask for.
    const size_t smem = job_smem(t->cap);
    int optin = 0;
    cudaFuncAttributes fa;
    PLP_CUDA_TRY(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, t->ctx->device));
    PLP_CUDA_TRY(cudaFuncGetAttributes(&fa, kt::kf_job_kernel));
    PLP_REQUIRE(smem + fa.sharedSizeBytes <= (size_t)optin,
                "kp_capacity too large for the feature-vector kernel's shared memory");
    PLP_CUDA_TRY(cudaFuncSetAttribute(kt::kf_job_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      optin - (int)fa.sharedSizeBytes));
    if (t->d_kf) {  // a second reservation replaces the first once the stream has stopped using it
        PLP_CUDA_TRY(cudaStreamSynchronize(t->ctx->stream));
        cudaFree(t->d_kf);
        t->d_kf = nullptr;
        t->max_keyframes = t->max_kf_points = 0;
        t->has_kf = false;
    }
    // the scratch of every later call, bound once (B frames, C keypoints, R keyframe rows)
    const size_t B = t->max_batch, C = t->cap, R = max_keyframe_points;
    auto D = std::make_shared<KfDev>();
    memset(D.get(), 0, sizeof(KfDev));
    DevLayout L;
    L.out(D->word, B * C);
    L.out(D->node, B * C);
    L.out(D->weight, B * C);
    L.out(D->fidx, B * C);
    L.out(D->nb1, B * C);
    L.out(D->ne1, B * C);
    L.out(D->nb2, B * C);
    L.out(D->ne2, B * C);
    L.out(D->claimed, B * C);
    L.out(D->choice, B * R);
    L.out(D->m21, B * R);
    L.out(D->bjobs, B);
    L.out(D->posejobs, B);
    L.out(D->obs, B * C);
    L.out(D->obs_kp, B * C);
    L.out(D->obs_row, B * C);
    L.out(D->obs_outlier, B * C);
    if (alloc(t->ctx, L, &t->d_kf, false) != cudaSuccess) {
        set_error("tracker: cudaMalloc(%zu) for keyframe tracking failed", L.bytes());
        return PLP_ERR_CUDA;
    }
    t->max_keyframes = max_keyframes;
    t->max_kf_points = max_keyframe_points;
    D->cap = t->cap;
    D->max_kf_points = max_keyframe_points;
    t->kf = D;
    return PLP_OK;
}

plp_status plp_tracker_keyframe_track_batch_dev(plp_tracker *t, plp_bow_vocab *vocab, int batch,
                                                const plp_track_keyframe *kf, const uint8_t *d_motion_valid,
                                                int32_t *d_stage_out, int32_t *d_kf_matched_out,
                                                int32_t *d_num_bow_matches_out, double *d_pose_out,
                                                int32_t *d_num_valid_out, int32_t *d_n_inliers_out,
                                                int32_t *d_lm_iters_out, int32_t *d_status_out) {
    PLP_REQUIRE(t && vocab && kf && d_stage_out && d_kf_matched_out && d_num_bow_matches_out && d_pose_out &&
                    d_num_valid_out && d_n_inliers_out && d_lm_iters_out && d_status_out,
                "null pointer");
    PLP_REQUIRE(kf->kf_of_frame && kf->row_offsets && kf->desc && kf->angle && kf->pos_w && kf->fv_offsets &&
                    kf->node_ids && kf->node_begin && kf->indices,
                "keyframe arrays");
    PLP_REQUIRE(!kf->local_idx == !kf->local_idx_offsets, "local_idx and local_idx_offsets go together");
    PLP_REQUIRE(t->d_kf, "plp_tracker_reserve_keyframe_track has not been called");
    PLP_REQUIRE(kf->num_keyframes >= 0 && kf->num_keyframes <= t->max_keyframes,
                "num_keyframes exceeds the reserved max_keyframes");
    PLP_REQUIRE(batch >= 1 && batch <= t->max_batch, "batch exceeds the tracker's max_batch");
    PLP_REQUIRE(t->has_motion && batch <= t->motion.batch,
                "the batch must follow a plp_tracker_motion_track_batch_dev of at least as many frames");
    PLP_REQUIRE(vocab->ctx->device == t->ctx->device, "the vocabulary lives on another device");
    plp_ctx *ctx = t->ctx;
    PLP_CUDA_TRY(cudaSetDevice(ctx->device));
    t->has_kf = false;
    t->has_rb = false;
    const TrackDev &M = t->motion;
    KfDev D = *t->kf;
    D.batch = batch;
    D.num_keyframes = kf->num_keyframes;
    D.n_kp = M.n_kp;
    D.x = M.x;
    D.y = M.y;
    D.angle = M.angle;
    D.octave = M.octave;
    D.desc = M.desc;
    D.motion_num_valid = M.num_valid;
    D.pose_last = M.pose_last;
    for (int l = 0; l < kt::kMaxLevels; ++l) D.inv_level_sigma_sq[l] = M.inv_level_sigma_sq[l];
    D.motion_valid = d_motion_valid;
    D.kf_of_frame = kf->kf_of_frame;
    D.row_offsets = kf->row_offsets;
    D.kf_desc = kf->desc;
    D.kf_angle = kf->angle;
    D.kf_valid = kf->valid;
    D.kf_pos_w = kf->pos_w;
    D.fv_offsets = kf->fv_offsets;
    D.node_ids = kf->node_ids;
    D.node_begin = kf->node_begin;
    D.indices = kf->indices;
    D.stage = d_stage_out;
    D.status = d_status_out;
    D.matched = d_kf_matched_out;
    D.num_bow = (uint32_t *)d_num_bow_matches_out;
    D.pose = d_pose_out;
    D.num_valid = d_num_valid_out;
    D.n_inliers = d_n_inliers_out;
    D.lm_iters = d_lm_iters_out;

    PLP_LAUNCH(ctx, kt::kf_prep_kernel, div_up(batch, kt::kPrepThreads), kt::kPrepThreads, 0, D);
    PLP_CHECK_LAUNCH();
    PLP_TRY(launch_kf_transform(ctx, vocab, D, batch));
    PLP_LAUNCH(ctx, kt::kf_job_kernel, batch, kt::kThreads, job_smem(t->cap), D);
    PLP_CHECK_LAUNCH();
    PLP_LAUNCH(ctx, bow_match_kernel, batch, kMatchThreads, 0, D.bjobs, kt::kLoweRatio, 1);
    PLP_CHECK_LAUNCH();
    PLP_LAUNCH(ctx, kt::kf_gather_kernel, batch, kt::kThreads, 0, D);
    PLP_CHECK_LAUNCH();
    plp_pose_opt_cfg cfg{4, 10};
    PLP_TRY(launch_pose_opt(ctx, D.posejobs, batch, t->cap, t->cam, cfg));
    PLP_LAUNCH(ctx, kt::kf_finish_kernel, batch, kt::kThreads, 0, D);
    PLP_CHECK_LAUNCH();

    KeyframeTrack &K = t->kf_track;
    K.stage = d_stage_out;
    K.status = d_status_out;
    K.matched = d_kf_matched_out;
    K.pose = d_pose_out;
    K.num_valid = d_num_valid_out;
    K.posejobs = D.posejobs;
    K.obs_row = D.obs_row;
    K.kf_pos_w = kf->pos_w;
    K.kf_row_offsets = kf->row_offsets;
    K.kf_of_frame = kf->kf_of_frame;
    K.local_idx = kf->local_idx;
    K.local_idx_offsets = kf->local_idx_offsets;
    t->kf_table = *kf;
    t->kf_batch = batch;
    t->has_kf = true;
    return PLP_OK;
}

plp_status plp_tracker_keyframe_bow(const plp_tracker *t, const int32_t **d_word_id, const int32_t **d_node_id,
                                    const float **d_weight) {
    PLP_REQUIRE(t && d_word_id && d_node_id && d_weight, "null pointer");
    PLP_REQUIRE(t->d_kf, "plp_tracker_reserve_keyframe_track has not been called");
    *d_word_id = t->kf->word;
    *d_node_id = t->kf->node;
    *d_weight = t->kf->weight;
    return PLP_OK;
}

}  // extern "C"
