// local_map_update.cu -- device-resident, frame-batched local-map update:
//   tracking_module::update_local_map (tracking_module.cc:837-906) = the clean-up of erased tracked landmarks
//     + local_map_updater::acquire_local_map (find_local_keyframes, find_local_landmarks)
// for the batch of the tracker's most recent tracking calls, on the same stream and without leaving HBM, between the last
// tracking call (motion, keyframe or robust) and the local-map stage.  It reads the tracking records (tracker.h) and a
// caller-owned map snapshot (plp_track_map) and writes the plp_track_local the local-map stage takes, tracker-owned, plus
// the caller's per-frame outputs.  Device code: local_map_update_kernels.cuh.
#include "common.cuh"
#include "local_map_update_kernels.cuh"
#include "tracker.h"

namespace plp {

namespace {

using lu::UpdDev;

int pow2_at_least(long long n) {
    int p = 1;
    while (p < n) p <<= 1;
    return p;
}

}  // namespace

}  // namespace plp

using namespace plp;

extern "C" {

plp_status plp_tracker_reserve_local_map_update(plp_tracker *t, int max_local_keyframes) {
    PLP_REQUIRE(t, "null pointer");
    PLP_REQUIRE(t->local, "plp_tracker_reserve_local_map has not been called");
    PLP_REQUIRE(max_local_keyframes >= lu::kMinReservedKeyframes && max_local_keyframes <= (1 << 20),
                "max_local_keyframes must be at least 64");
    PLP_CUDA_TRY(cudaSetDevice(t->ctx->device));
    const int vote_slots = pow2_at_least(2LL * max_local_keyframes);
    PLP_SMEM_OPTIN(lu::lmu_vote_kernel, lu::vote_smem_bytes(vote_slots, max_local_keyframes));
    // a second reservation ends the first's list
    t->update_batch = 0;
    t->updated = plp_track_local{};
    t->upd_local_idx = t->upd_local_idx_offsets = nullptr;
    // the scratch and tracker-owned outputs of every later call, bound once (B frames, ML local rows, LK local
    // keyframes, S landmark slots, M last rows, R keyframe rows)
    const size_t B = t->max_batch, ML = t->max_local, LK = max_local_keyframes, M = t->max_last, R = t->max_kf_points;
    const int lm_slots = pow2_at_least(2LL * t->max_local);
    const size_t S = lm_slots;
    auto D = std::make_shared<UpdDev>();
    memset(D.get(), 0, sizeof(UpdDev));
    DevLayout L;
    L.out(D->cand_off, B * (LK + 1));
    L.out(D->hkey, B * S);
    L.out(D->hpos, B * S);
    L.out(D->hidx, B * S);
    L.out(D->uniq, B);
    L.out(D->first_lm, B * ML);
    L.out(D->count, B);
    L.out(D->lidx_len, B);
    L.out(D->pos_w, B * ML * 3);
    L.out(D->normal, B * ML * 3);
    L.out(D->min_d, B * ML);
    L.out(D->max_d, B * ML);
    L.out(D->max_raw, B * ML);
    L.out(D->desc, B * ML * 32);
    L.out(D->valid, B * ML);
    L.out(D->offsets, B + 1);
    L.out(D->last_local_idx, B * M);
    L.out(D->local_idx, R ? B * R : 1);
    L.out(D->local_idx_offsets, B + 1);
    D->cap = t->cap;
    D->max_local = t->max_local;
    D->max_lkf = max_local_keyframes;
    D->vote_slots = vote_slots;
    D->lm_slots = lm_slots;
    PLP_TRY(t->upd.reserve(t->ctx, L, D, "the local-map update"));
    t->upd_max_kf_points = t->max_kf_points;
    plp_track_local &out = t->updated;  // the list every later call writes
    out.pos_w = D->pos_w;
    out.obs_mean_normal = D->normal;
    out.min_valid_dist = D->min_d;
    out.max_valid_dist = D->max_d;
    out.max_valid_dist_raw = D->max_raw;
    out.desc = D->desc;
    out.valid = D->valid;
    out.offsets = D->offsets;
    out.last_local_idx = D->last_local_idx;
    t->upd_local_idx = D->local_idx;
    t->upd_local_idx_offsets = D->local_idx_offsets;
    return PLP_OK;
}

plp_status plp_tracker_update_local_map_batch_dev(plp_tracker *t, int batch, const plp_track_map *map,
                                                  int32_t *d_nearest_out, int32_t *d_local_kf_out,
                                                  int32_t *d_num_local_kf_out, int32_t *d_local_lm_out,
                                                  int32_t *d_status_out) {
    PLP_REQUIRE(t && map && d_nearest_out && d_local_kf_out && d_num_local_kf_out && d_local_lm_out && d_status_out,
                "null pointer");
    PLP_REQUIRE(map->pos_w && map->obs_mean_normal && map->min_valid_dist && map->max_valid_dist &&
                    map->max_valid_dist_raw && map->desc && map->lm_erased && map->obs_offsets && map->obs_kf &&
                    map->kf_erased && map->row_offsets && map->row_lm && map->cov_offsets && map->cov_kf &&
                    map->child_offsets && map->child_kf && map->parent && map->last_row_lm,
                "map arrays");
    PLP_REQUIRE(((uintptr_t)map->desc & 3) == 0, "map desc must be 4-byte aligned");
    PLP_REQUIRE(t->upd, "plp_tracker_reserve_local_map_update has not been called");
    PLP_REQUIRE(t->upd->max_local == t->max_local,
                "plp_tracker_reserve_local_map was called again after plp_tracker_reserve_local_map_update");
    PLP_TRY(t->check_order(kNumStages, batch));
    const bool kf = t->record_batch[kStageKeyframe] != 0;
    PLP_REQUIRE(!kf || map->kf_row_lm, "kf_row_lm is required after a plp_tracker_keyframe_track_batch_dev");
    PLP_REQUIRE(!kf || t->max_kf_points <= t->upd_max_kf_points,
                "plp_tracker_reserve_keyframe_track was called with more points after plp_tracker_reserve_local_map_update");
    plp_ctx *ctx = t->ctx;
    PLP_CUDA_TRY(cudaSetDevice(ctx->device));
    UpdDev D = *t->upd.job;
    D.batch = batch;
    D.n_kp = t->motion.n_kp;
    D.last_offsets = t->motion.last_offsets;
    D.motion = t->record[kStageMotion];
    D.kf = t->standing(kStageKeyframe);
    D.rb = t->standing(kStageRobust);
    if (kf) {
        D.kf_of_frame = t->kf_table.kf_of_frame;
        D.kf_row_offsets = t->kf_table.row_offsets;
    }
    D.map = *map;
    D.nearest = d_nearest_out;
    D.local_kf = d_local_kf_out;
    D.num_local_kf = d_num_local_kf_out;
    D.local_lm = d_local_lm_out;
    D.status = d_status_out;

    PLP_LAUNCH(ctx, lu::lmu_vote_kernel, batch, lu::kThreads, lu::vote_smem_bytes(D.vote_slots, D.max_lkf), D);
    PLP_CHECK_LAUNCH();
    // enough chunks per frame to fill the device at small batches; a chunk strides over the rest
    const int want = div_up(4 * (ctx->sm_count > 0 ? ctx->sm_count : 1), batch);
    const int chunks = want < 16 ? want : 16;
    PLP_LAUNCH(ctx, lu::lmu_dedup_kernel, dim3(chunks, batch), lu::kChunkThreads, 0, D);
    PLP_CHECK_LAUNCH();
    PLP_LAUNCH(ctx, lu::lmu_compact_kernel, batch, lu::kThreads, 0, D);
    PLP_CHECK_LAUNCH();
    PLP_LAUNCH(ctx, lu::lmu_scan_kernel, 1, lu::kThreads, 0, D);
    PLP_CHECK_LAUNCH();
    PLP_LAUNCH(ctx, lu::lmu_fill_kernel, dim3(chunks, batch), lu::kChunkThreads, 0, D);
    PLP_CHECK_LAUNCH();

    // The records are left as the tracking calls made them: a local-map call given this list maps the keyframe rows
    // through this call's local_idx blocks instead (local_map.cu), so nothing has to be restored when the list ends.
    t->update_batch = batch;
    return PLP_OK;
}

plp_status plp_tracker_updated_local_map(const plp_tracker *t, plp_track_local *out) {
    PLP_REQUIRE(t && out, "null pointer");
    PLP_REQUIRE(t->update_batch, "no plp_tracker_update_local_map_batch_dev since the last tracking call");
    *out = t->updated;
    return PLP_OK;
}

plp_status plp_tracker_updated_local_idx(const plp_tracker *t, const int32_t **d_local_idx,
                                        const int32_t **d_local_idx_offsets) {
    PLP_REQUIRE(t && d_local_idx && d_local_idx_offsets, "null pointer");
    PLP_REQUIRE(t->update_batch, "no plp_tracker_update_local_map_batch_dev since the last tracking call");
    *d_local_idx = t->upd_local_idx;
    *d_local_idx_offsets = t->upd_local_idx_offsets;
    return PLP_OK;
}

}  // extern "C"
