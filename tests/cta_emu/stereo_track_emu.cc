// stereo_track_emu.cc -- the stereo rows of the batched tracker's device code executed on the host: motion_assumption
// (match_common.cuh), the shared tail's gather (track_common.cuh) with the current frames' x_right, and the local-map
// stage (local_map_kernels.cuh: prep -> observe -> window matcher -> gather) with x_right and the qxr scratch row.
// The pose optimiser is not emulated: the callers compare the gathered observations and the matches.
#include "cta_emu.h"

#include <string.h>

#include <vector>

#include "local_map_kernels.cuh"
#include "point_match_kernels.cuh"

using namespace plp;

namespace {

std::vector<uint8_t> g_excl, g_qvalid, g_claimed, g_outlier, g_observable;
std::vector<double> g_center, g_pose;
std::vector<float> g_qx, g_qy, g_qr;
std::vector<int32_t> g_qmin, g_qmax, g_choice, g_best, g_local, g_n_inl, g_iters, g_status, g_obs_row;
std::vector<uint32_t> g_nm;
std::vector<PointMatchJob> g_mjobs;
std::vector<PoseJob> g_posejobs, g_record_jobs;

}  // namespace

extern "C" void emu_motion_assumption(const plp_camera *cam, const double *Tc, const double *Tl, int *fwd, int *bwd) {
    motion_assumption(*cam, Tc, Tl, fwd, bwd);
}

// track_gather_kernel over a tail job whose gate is count alone, the rows one block per frame
extern "C" void emu_tail_gather_stereo(int batch, int cap, const int32_t *n_kp, const float *x, const float *y,
                                       const int32_t *octave, const float *x_right, const float *inv_level_sigma_sq,
                                       int num_levels, const int32_t *count, const double *pos_w,
                                       const int32_t *offsets, const double *pose_in, int32_t *matched,
                                       plp_pt_obs *obs, int32_t *obs_kp, int32_t *n_obs) {
    const size_t B = batch, C = cap;
    g_outlier.assign(B * C, 0);
    g_obs_row.assign(B * C, 0);
    g_posejobs.assign(B, PoseJob{});
    g_pose.assign(B * 16, 0.0);
    g_n_inl.assign(B, 0);
    g_iters.assign(B, 0);
    TrackTail J;
    memset(&J, 0, sizeof(J));
    J.cap = cap;
    J.n_kp = n_kp;
    J.x = x;
    J.y = y;
    J.octave = octave;
    J.x_right = x_right;
    for (int l = 0; l < 16; ++l) J.inv_level_sigma_sq[l] = l < num_levels ? inv_level_sigma_sq[l] : 1.0f;
    J.count = count;
    J.rows = TrackRows{pos_w, offsets, nullptr};
    J.pose_in = pose_in;
    J.matched = matched;
    J.posejobs = g_posejobs.data();
    J.obs = obs;
    J.obs_kp = obs_kp;
    J.obs_row = g_obs_row.data();
    J.obs_outlier = g_outlier.data();
    J.pose = g_pose.data();
    J.n_inliers = g_n_inl.data();
    J.lm_iters = g_iters.data();
    emu_launch(track_gather_kernel, (unsigned)batch, (unsigned)kTailThreads, J);
    for (int b = 0; b < batch; ++b) n_obs[b] = g_posejobs[b].n_pts;
}

// The local-map stage of one batch whose frames start from their motion record (matched: after discard_outliers;
// n_obs / obs_row: the rows of its pose optimisation), up to the gather.  x_right == nullptr runs the monocular stage
// (no qxr row, as a monocular tracker reserves none).  Outputs: the matcher's best keypoint per local row, the qxr row
// (rows the observe kernel left alone keep the caller's values), the local row per keypoint and the gathered
// observations.
extern "C" void emu_local_stereo(const plp_grid *grid, const plp_camera *cam, int batch, int cap, int max_local,
                                 const int32_t *n_kp, const float *x, const float *y, const int32_t *octave,
                                 const uint8_t *desc, const float *x_right, const float *inv_level_sigma_sq,
                                 const int32_t *m_matched, const double *m_pose, const int32_t *m_num_valid,
                                 const int32_t *m_n_obs, const int32_t *m_obs_row, const double *last_pos_w,
                                 const int32_t *last_offsets, const double *pos_w, const double *normal,
                                 const float *min_d, const float *max_d, const float *max_raw, const uint8_t *lm_desc,
                                 const int32_t *offsets, const int32_t *last_local_idx, const float *scale_factors,
                                 const float *level_thr, int num_levels, float margin, float *qxr_inout,
                                 int32_t *best_out, int32_t *matched, int32_t *local, plp_pt_obs *obs_out,
                                 int32_t *obs_kp_out, int32_t *n_obs_out) {
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
    g_choice.assign(B * ML, 0);
    g_best.assign(B * ML, -1);
    g_n_inl.assign(B, 0);
    g_iters.assign(B, 0);
    g_status.assign(B, -1);
    g_nm.assign(B, 0);
    g_mjobs.assign(B, PointMatchJob{});
    g_posejobs.assign(B, PoseJob{});
    g_pose.assign(B * 16, 0.0);
    g_observable.assign(offsets[batch] > 0 ? offsets[batch] : 1, 0);
    g_record_jobs.assign(B, PoseJob{});
    for (size_t b = 0; b < B; ++b) g_record_jobs[b].n_pts = m_n_obs[b];
    lm::LocalDev D;
    memset(&D, 0, sizeof(D));
    D.batch = batch;
    D.cap = cap;
    D.max_local = max_local;
    D.n_kp = n_kp;
    D.x = x;
    D.y = y;
    D.octave = octave;
    D.x_right = x_right;
    D.desc = desc;
    D.motion = TrackRecord{nullptr, nullptr, m_matched, m_pose, m_num_valid, g_record_jobs.data(), m_obs_row,
                           TrackRows{last_pos_w, last_offsets, nullptr}, last_local_idx, last_offsets};
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
    D.offsets = offsets;
    D.cam = *cam;
    D.num_levels = num_levels;
    D.margin = margin;
    D.excl = g_excl.data();
    D.center = g_center.data();
    D.qx = g_qx.data();
    D.qy = g_qy.data();
    D.qxr = x_right ? qxr_inout : nullptr;
    D.qradius = g_qr.data();
    D.qmin = g_qmin.data();
    D.qmax = g_qmax.data();
    D.qvalid = g_qvalid.data();
    D.choice = g_choice.data();
    D.best = best_out;
    D.num_matches = g_nm.data();
    D.claimed = g_claimed.data();
    D.mjobs = g_mjobs.data();
    D.posejobs = g_posejobs.data();
    D.obs = obs_out;
    D.obs_kp = obs_kp_out;
    D.obs_outlier = g_outlier.data();
    D.matched = matched;
    D.local = local;
    D.observable = g_observable.data();
    D.pose = g_pose.data();
    D.n_inliers = g_n_inl.data();
    D.lm_iters = g_iters.data();
    D.status = g_status.data();
    emu_launch(lm::local_prep_kernel, (unsigned)batch, (unsigned)lm::kThreads, D);
    emu_launch2(lm::local_observe_kernel, (unsigned)((max_local + lm::kObserveThreads - 1) / lm::kObserveThreads),
                (unsigned)batch, (unsigned)lm::kObserveThreads, (size_t)0, D);
    const size_t smem = pm::point_smem_bytes(cap, grid->num_cols, grid->num_rows);
    emu_launch2(pm::point_match_kernel, (unsigned)batch, 1u, (unsigned)pm::kThreads, smem,
                (const PointMatchJob *)g_mjobs.data(), *grid, cap, 1, lm::kLoweRatio, 0);
    emu_launch(lm::local_gather_kernel, (unsigned)batch, (unsigned)lm::kThreads, D);
    for (size_t b = 0; b < B; ++b) n_obs_out[b] = g_posejobs[b].n_pts;
}
