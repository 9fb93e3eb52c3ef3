// lmupdate_emu.cc -- csrc/local_map_update_kernels.cuh (the local-map update of tracking) executed on the host: vote ->
// dedup -> compact -> scan -> fill, with the scratch local_map_update.cu reserves.  The motion, keyframe and robust
// records come as EmuRecords (the layout of local_map_emu.cc; only stage, status, matched, num_valid, offsets and
// of_frame are read).
#include "cta_emu.h"

#include <string.h>

#include <vector>

#include "local_map_update_kernels.cuh"

using namespace plp;

struct EmuRecord {
    const int32_t *stage, *status, *matched;
    const double *pose;
    const int32_t *num_valid, *n_obs, *obs_row;
    const double *pos_w;
    const int32_t *offsets, *of_frame, *local_idx, *local_idx_offsets;
};

namespace {

std::vector<int32_t> g_cand_off, g_hkey, g_hpos, g_hidx, g_uniq, g_first, g_count, g_lidx_len;

int pow2_at_least(long long n) {
    int p = 1;
    while (p < n) p <<= 1;
    return p;
}

}  // namespace

// Every output is caller-allocated at the reservation's sizes: local_kf batch x max_lkf; the rows batch x max_local;
// last_local_idx the batch's last rows; local_idx batch x (largest keyframe); offsets batch + 1.
extern "C" void emu_lmu_run(int batch, int cap, int max_local, int max_lkf, const int32_t *n_kp, const EmuRecord *records,
                            const int32_t *last_offsets, const int32_t *kf_of_frame, const int32_t *kf_row_offsets,
                            const plp_track_map *map, int32_t *nearest, int32_t *local_kf, int32_t *num_local_kf,
                            int32_t *local_lm, int32_t *status, double *pos_w, double *normal, float *min_d,
                            float *max_d, float *max_raw, uint8_t *desc, uint8_t *valid, int32_t *offsets,
                            int32_t *last_local_idx, int32_t *local_idx, int32_t *local_idx_offsets) {
    lu::UpdDev D;
    memset(&D, 0, sizeof(D));
    D.batch = batch;
    D.cap = cap;
    D.max_local = max_local;
    D.max_lkf = max_lkf;
    D.vote_slots = pow2_at_least(2LL * max_lkf);
    D.lm_slots = pow2_at_least(2LL * max_local);
    TrackRecord rec[3] = {};
    for (int s = 0; s < 3; ++s) {
        const EmuRecord &E = records[s];
        if (s > 0 && !E.stage) continue;
        rec[s].stage = E.stage;
        rec[s].status = E.status;
        rec[s].matched = E.matched;
        rec[s].num_valid = E.num_valid;
        rec[s].rows = TrackRows{nullptr, E.offsets, E.of_frame};
    }
    D.motion = rec[0];
    D.kf = rec[1];
    D.rb = rec[2];
    D.n_kp = n_kp;
    D.last_offsets = last_offsets;
    D.kf_of_frame = kf_of_frame;
    D.kf_row_offsets = kf_row_offsets;
    D.map = *map;
    const size_t B = batch, S = D.lm_slots;
    // scratch with leftovers of an earlier call, as device scratch has
    g_cand_off.assign(B * (max_lkf + 1), 77);
    g_hkey.assign(B * S, 5);
    g_hpos.assign(B * S, 3);
    g_hidx.assign(B * S, 9);
    g_uniq.assign(B, 1234);
    g_first.assign(B * max_local, -7);
    g_count.assign(B, 99);
    g_lidx_len.assign(B, 99);
    D.cand_off = g_cand_off.data();
    D.hkey = g_hkey.data();
    D.hpos = g_hpos.data();
    D.hidx = g_hidx.data();
    D.uniq = g_uniq.data();
    D.first_lm = g_first.data();
    D.count = g_count.data();
    D.lidx_len = g_lidx_len.data();
    D.nearest = nearest;
    D.local_kf = local_kf;
    D.num_local_kf = num_local_kf;
    D.local_lm = local_lm;
    D.status = status;
    D.pos_w = pos_w;
    D.normal = normal;
    D.min_d = min_d;
    D.max_d = max_d;
    D.max_raw = max_raw;
    D.desc = desc;
    D.valid = valid;
    D.offsets = offsets;
    D.last_local_idx = last_local_idx;
    D.local_idx = local_idx;
    D.local_idx_offsets = local_idx_offsets;

    emu_launch2(lu::lmu_vote_kernel, (unsigned)batch, 1u, (unsigned)lu::kThreads,
                lu::vote_smem_bytes(D.vote_slots, max_lkf), D);
    emu_launch2(lu::lmu_dedup_kernel, 3u, (unsigned)batch, (unsigned)lu::kChunkThreads, (size_t)0, D);
    emu_launch(lu::lmu_compact_kernel, (unsigned)batch, (unsigned)lu::kThreads, D);
    emu_launch(lu::lmu_scan_kernel, 1u, (unsigned)lu::kThreads, D);
    emu_launch2(lu::lmu_fill_kernel, 2u, (unsigned)batch, (unsigned)lu::kChunkThreads, (size_t)0, D);
}
