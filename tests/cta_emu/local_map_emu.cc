// local_map_emu.cc -- csrc/local_map_kernels.cuh (the local-map stage of tracking) executed on the host, with the window
// matcher of point_match_kernels.cuh between observe and gather.  The pose optimiser is not emulated: emu_local_begin
// runs prep -> observe -> match -> gather and returns the gathered observations; the caller optimises them and hands
// the outlier flags to emu_local_finish.  The motion, keyframe and robust records come as EmuRecords.
#include "cta_emu.h"

#include <string.h>

#include <vector>

#include "local_map_kernels.cuh"
#include "point_match_kernels.cuh"

using namespace plp;

namespace {

lm::LocalDev g_D;
std::vector<uint8_t> g_excl, g_qvalid, g_claimed, g_outlier;
std::vector<double> g_center;
std::vector<float> g_qx, g_qy, g_qr;
std::vector<int32_t> g_qmin, g_qmax, g_choice, g_best, g_obs_kp, g_n_inl, g_iters;
std::vector<uint32_t> g_nm;
std::vector<PointMatchJob> g_mjobs;
std::vector<PoseJob> g_posejobs, g_record_jobs[3];
std::vector<plp_pt_obs> g_obs;
std::vector<double> g_pose;

}  // namespace

// one TrackRecord as the caller's arrays, n_obs[b] standing for posejobs[b].n_pts; a keyframe or robust record with
// stage == nullptr is left out
struct EmuRecord {
    const int32_t *stage, *status, *matched;
    const double *pose;
    const int32_t *num_valid, *n_obs, *obs_row;
    const double *pos_w;
    const int32_t *offsets, *of_frame, *local_idx, *local_idx_offsets;
};

// records: motion, keyframe, robust.  As local_map.cu does, the motion record's local_idx is last_local_idx over its
// row offsets.
extern "C" void emu_local_begin(const plp_grid *grid, const plp_camera *cam, int batch, int cap, int max_local,
                                const int32_t *n_kp, const float *x, const float *y, const int32_t *octave,
                                const uint8_t *desc, const EmuRecord *records, const float *inv_level_sigma_sq,
                                const double *pos_w, const double *normal, const float *min_d, const float *max_d,
                                const float *max_raw, const uint8_t *lm_desc, const uint8_t *valid,
                                const int32_t *offsets, const int32_t *last_local_idx, const float *scale_factors,
                                const float *level_thr, int num_levels, float margin, int32_t *matched, int32_t *local,
                                uint8_t *observable, int32_t *status, plp_pt_obs *obs_out, int32_t *obs_kp_out,
                                int32_t *n_obs_out) {
    const size_t B = batch, C = cap, ML = max_local;
    g_excl.assign(B * ML, 0);
    g_qvalid.assign(B * ML, 0);
    g_claimed.assign(B * C, 0);
    g_outlier.assign(B * C, 0);
    g_center.assign(B * 3, 0.0);
    g_qx.assign(B * ML, 0.0f);
    g_qy.assign(B * ML, 0.0f);
    g_qr.assign(B * ML, 0.0f);
    g_qmin.assign(B * ML, 0);
    g_qmax.assign(B * ML, 0);
    // the matcher's choice scratch starts with leftovers of an earlier call, as device scratch does
    g_choice.resize(B * ML);
    for (size_t i = 0; i < g_choice.size(); ++i) g_choice[i] = (int32_t)((i * 7919u) % 97u);
    g_best.assign(B * ML, -1);
    g_obs_kp.assign(B * C, -1);
    g_n_inl.assign(B, 0);
    g_iters.assign(B, 0);
    g_nm.assign(B, 0);
    g_mjobs.assign(B, PointMatchJob{});
    g_posejobs.assign(B, PoseJob{});
    g_obs.assign(B * C, plp_pt_obs{});
    g_pose.assign(B * 16, 0.0);
    TrackRecord rec[3] = {};
    for (int s = 0; s < 3; ++s) {
        const EmuRecord &E = records[s];
        if (s > 0 && !E.stage) continue;
        g_record_jobs[s].assign(B, PoseJob{});
        for (size_t b = 0; b < B; ++b) g_record_jobs[s][b].n_pts = E.n_obs[b];
        rec[s] = TrackRecord{E.stage,    E.status,     E.matched, E.pose,         E.num_valid, g_record_jobs[s].data(),
                             E.obs_row, TrackRows{E.pos_w, E.offsets, E.of_frame}, E.local_idx, E.local_idx_offsets};
    }
    rec[0].local_idx = last_local_idx;
    rec[0].local_idx_offsets = records[0].offsets;
    lm::LocalDev &D = g_D;
    memset(&D, 0, sizeof(D));
    D.batch = batch;
    D.cap = cap;
    D.max_local = max_local;
    D.n_kp = n_kp;
    D.x = x;
    D.y = y;
    D.octave = octave;
    D.desc = desc;
    D.motion = rec[0];
    D.kf = rec[1];
    D.rb = rec[2];
    for (int l = 0; l < lm::kMaxLevels; ++l) {
        D.inv_level_sigma_sq[l] = l < num_levels ? inv_level_sigma_sq[l] : 1.0f;
        D.scale_factors[l] = l < num_levels ? scale_factors[l] : 1.0f;
        D.level_thr[l] = l < num_levels ? level_thr[l] : INFINITY;
    }
    D.pos_w = pos_w;
    D.normal = normal;
    D.min_d = min_d;
    D.max_d = max_d;
    D.max_raw = max_raw;
    D.lm_desc = lm_desc;
    D.valid = valid;
    D.offsets = offsets;
    D.cam = *cam;
    D.num_levels = num_levels;
    D.margin = margin;
    D.excl = g_excl.data();
    D.center = g_center.data();
    D.qx = g_qx.data();
    D.qy = g_qy.data();
    D.qradius = g_qr.data();
    D.qmin = g_qmin.data();
    D.qmax = g_qmax.data();
    D.qvalid = g_qvalid.data();
    D.choice = g_choice.data();
    D.best = g_best.data();
    D.num_matches = g_nm.data();
    D.claimed = g_claimed.data();
    D.mjobs = g_mjobs.data();
    D.posejobs = g_posejobs.data();
    D.obs = g_obs.data();
    D.obs_kp = g_obs_kp.data();
    D.obs_outlier = g_outlier.data();
    D.matched = matched;
    D.local = local;
    D.observable = observable;
    D.pose = g_pose.data();
    D.num_tracked = nullptr;  // set by emu_local_finish
    D.n_inliers = g_n_inl.data();
    D.lm_iters = g_iters.data();
    D.status = status;

    emu_launch(lm::local_prep_kernel, (unsigned)batch, (unsigned)lm::kThreads, D);
    emu_launch2(lm::local_observe_kernel, (unsigned)((max_local + lm::kObserveThreads - 1) / lm::kObserveThreads),
                (unsigned)batch, (unsigned)lm::kObserveThreads, (size_t)0, D);
    const PointMatchJob *jobs = g_mjobs.data();
    const size_t smem = pm::point_smem_bytes(cap, grid->num_cols, grid->num_rows);
    emu_launch2(pm::point_match_kernel, (unsigned)batch, 1u, (unsigned)pm::kThreads, smem, jobs, *grid, cap, 1,
                lm::kLoweRatio, 0);
    emu_launch(lm::local_gather_kernel, (unsigned)batch, (unsigned)lm::kThreads, D);
    for (size_t b = 0; b < B; ++b) {
        n_obs_out[b] = g_posejobs[b].n_pts;
        memcpy(obs_out + b * C, g_obs.data() + b * C, C * sizeof(plp_pt_obs));
        memcpy(obs_kp_out + b * C, g_obs_kp.data() + b * C, C * 4);
    }
}

extern "C" void emu_local_finish(const uint8_t *outlier, int32_t *num_tracked) {
    memcpy(g_outlier.data(), outlier, g_outlier.size());
    g_D.num_tracked = num_tracked;
    emu_launch(lm::local_finish_kernel, (unsigned)g_D.batch, (unsigned)lm::kThreads, g_D);
}
