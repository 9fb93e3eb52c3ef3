// keyframe_track.cu -- device-resident, frame-batched keyframe tracking:
//   frame_tracker::bow_match_based_track (module/frame_tracker.cc:126-189) =
//       frame::compute_bow + bow_tree::match_frame_and_keyframe (Lowe 0.7, orientation check)
//     + pose_optimizer::optimize from the last frame's pose + discard_outliers
// for the frames of the tracker's most recent plp_tracker_motion_track_batch_dev that the reference hands to it (motion
// model unusable, or motion track failed), on the same stream and without leaving HBM.  It reads that call's inputs and
// scratch (tracker.h) and writes separate outputs.  Device code: keyframe_track_kernels.cuh; the BoW matcher
// (bow_match_kernel) and the tail (track_common.cuh) are the existing ones, the vocabulary descent is
// bow_transform_kernel's.
#include "common.cuh"
#include "bow_vocab.h"
#include "keyframe_track_kernels.cuh"
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

int32_t *keyframe_choice(const plp_tracker *t) { return t->kf->choice; }

}  // namespace plp

using namespace plp;

extern "C" {

plp_status plp_tracker_reserve_keyframe_track(plp_tracker *t, int max_keyframes, int max_keyframe_points) {
    PLP_REQUIRE(t, "null pointer");
    PLP_REQUIRE(max_keyframes >= 1 && max_keyframe_points >= 1, "max_keyframes / max_keyframe_points");
    PLP_CUDA_TRY(cudaSetDevice(t->ctx->device));
    PLP_SMEM_OPTIN(kt::kf_job_kernel, job_smem(t->cap));  // the feature-vector kernel's cap x 12 bytes
    if (t->kf) {  // a second reservation ends the first, and what was tracked with it
        t->max_keyframes = t->max_kf_points = 0;
        t->invalidate_from(kStageKeyframe);
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
    TrackTail J = t->tail[kStageMotion];  // the tracker's cap and inv_level_sigma_sq; this stage's scratch
    tail_scratch(L, J, B, C);
    D->cap = t->cap;
    D->max_kf_points = max_keyframe_points;
    PLP_TRY(t->kf.reserve(t->ctx, L, D, "keyframe tracking"));
    t->max_keyframes = max_keyframes;
    t->max_kf_points = max_keyframe_points;
    t->tail[kStageKeyframe] = J;
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
    PLP_REQUIRE(t->kf, "plp_tracker_reserve_keyframe_track has not been called");
    PLP_REQUIRE(kf->num_keyframes >= 0 && kf->num_keyframes <= t->max_keyframes,
                "num_keyframes exceeds the reserved max_keyframes");
    PLP_TRY(t->check_order(kStageKeyframe, batch));
    PLP_REQUIRE(vocab->ctx->device == t->ctx->device, "the vocabulary lives on another device");
    plp_ctx *ctx = t->ctx;
    PLP_CUDA_TRY(cudaSetDevice(ctx->device));
    t->invalidate_from(kStageKeyframe);
    const TrackDev &M = t->motion;
    KfDev D = *t->kf.job;
    D.batch = batch;
    D.num_keyframes = kf->num_keyframes;
    D.n_kp = M.n_kp;
    D.angle = M.angle;
    D.desc = M.desc;
    D.motion_num_valid = t->record[kStageMotion].num_valid;
    D.motion_valid = d_motion_valid;
    D.kf_of_frame = kf->kf_of_frame;
    D.row_offsets = kf->row_offsets;
    D.kf_desc = kf->desc;
    D.kf_angle = kf->angle;
    D.kf_valid = kf->valid;
    D.fv_offsets = kf->fv_offsets;
    D.node_ids = kf->node_ids;
    D.node_begin = kf->node_begin;
    D.indices = kf->indices;
    D.stage = d_stage_out;
    D.status = d_status_out;
    D.matched = d_kf_matched_out;
    D.num_bow = (uint32_t *)d_num_bow_matches_out;
    // pose-opt from last_frm.cam_pose_cw_ over the frames with 20 BoW matches (frame_tracker.cc:138-169)
    TrackTail J = t->tail_job(kStageKeyframe, d_kf_matched_out, d_pose_out, d_num_valid_out, d_n_inliers_out,
                              d_lm_iters_out);
    J.count = d_num_bow_matches_out;
    J.stage = d_stage_out;
    J.status = d_status_out;
    J.rows = TrackRows{kf->pos_w, kf->row_offsets, kf->kf_of_frame};
    J.pose_in = M.pose_last;

    PLP_LAUNCH(ctx, kt::kf_prep_kernel, div_up(batch, kt::kPrepThreads), kt::kPrepThreads, 0, D);
    PLP_CHECK_LAUNCH();
    PLP_TRY(launch_kf_transform(ctx, vocab, D, batch));
    PLP_LAUNCH(ctx, kt::kf_job_kernel, batch, kt::kThreads, job_smem(t->cap), D);
    PLP_CHECK_LAUNCH();
    PLP_LAUNCH(ctx, bow_match_kernel, batch, kMatchThreads, 0, D.bjobs, kt::kLoweRatio, 1);
    PLP_CHECK_LAUNCH();
    PLP_TRY(launch_track_tail(ctx, J, batch, t->cam));
    t->kf_table = *kf;
    t->set_record(kStageKeyframe, batch, J, kf->local_idx, kf->local_idx_offsets);
    return PLP_OK;
}

plp_status plp_tracker_keyframe_bow(const plp_tracker *t, const int32_t **d_word_id, const int32_t **d_node_id,
                                    const float **d_weight) {
    PLP_REQUIRE(t && d_word_id && d_node_id && d_weight, "null pointer");
    PLP_REQUIRE(t->kf, "plp_tracker_reserve_keyframe_track has not been called");
    *d_word_id = t->kf->word;
    *d_node_id = t->kf->node;
    *d_weight = t->kf->weight;
    return PLP_OK;
}

}  // extern "C"
