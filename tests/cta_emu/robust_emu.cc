// robust_emu.cc -- csrc/robust_track_kernels.cuh (the batched robust tracker) executed on the host, with the keyframe
// tracker's gather and finish kernels (keyframe_track_kernels.cuh) after it.  Neither the brute-force matcher nor the
// pose optimiser is emulated: the caller hands in the brute-force matches of every frame (as brute_match_kernel leaves
// them in matched_out), emu_rt_begin runs prep -> list -> hypotheses -> select -> gather and returns what they wrote,
// and the caller hands the optimiser's outlier flags to emu_rt_finish.
#include "cta_emu.h"

#include <string.h>

#include <vector>

#include "keyframe_track_kernels.cuh"
#include "robust_track_kernels.cuh"

using namespace plp;

namespace {

rt::RtDev g_D;
kt::KfDev g_G;
std::vector<BruteJob> g_bjobs;
std::vector<PoseJob> g_posejobs;
std::vector<uint8_t> g_outlier;
std::vector<double> g_pose;
std::vector<int32_t> g_n_inl, g_iters;

}  // namespace

// ransac_sample.h's create_random_array(8, 0, n - 1) of hypothesis `iter` of frame `b`
extern "C" void emu_rs_sample8(uint64_t seed, uint32_t b, uint32_t iter, uint32_t n, int32_t *out) {
    rs_sample8(seed, b, iter, n, out);
}

// prep only: stage, status and the BruteJob sizes of every frame
extern "C" void emu_rt_prep(int batch, int cap, const int32_t *kf_stage, const int32_t *kf_status,
                            const int32_t *kf_num_valid, const int32_t *n_kp, const int32_t *kf_of_frame,
                            const int32_t *row_offsets, int32_t *stage, int32_t *status, int32_t *n_frm,
                            int32_t *n_kf) {
    std::vector<BruteJob> jobs(batch);
    std::vector<int32_t> matched((size_t)batch * cap);
    rt::RtDev D;
    memset(&D, 0, sizeof(D));
    D.batch = batch;
    D.cap = cap;
    D.n_kp = n_kp;
    D.kf_stage = kf_stage;
    D.kf_status = kf_status;
    D.kf_num_valid = kf_num_valid;
    D.kf_of_frame = kf_of_frame;
    D.row_offsets = row_offsets;
    D.bjobs = jobs.data();
    D.matched = matched.data();
    D.stage = stage;
    D.status = status;
    emu_launch(rt::rt_prep_kernel, (unsigned)((batch + rt::kPrepThreads - 1) / rt::kPrepThreads),
               (unsigned)rt::kPrepThreads, D);
    for (int b = 0; b < batch; ++b) {
        n_frm[b] = jobs[b].n_frm;
        n_kf[b] = jobs[b].n_kf;
    }
}

extern "C" void emu_rt_begin(int batch, int cap, uint64_t seed, const int32_t *n_kp, const float *x, const float *y,
                             const int32_t *octave, const double *pose_last, const float *inv_level_sigma_sq,
                             int num_levels, const double *K_cfg, const int32_t *kf_stage, const int32_t *kf_status,
                             const int32_t *kf_num_valid, const int32_t *kf_of_frame, const int32_t *row_offsets,
                             const double *kf_pos_w, const double *kf_bearings, double *bearings, int write_bearings,
                             const int32_t *bf_matched, int32_t *stage, int32_t *status, int32_t *matched,
                             int32_t *num_bf, int32_t *pairs, int32_t *samples, double *E, float *score,
                             uint8_t *inlier, double *best_score, int32_t *valid, int32_t *num_robust, plp_pt_obs *obs,
                             int32_t *obs_kp, int32_t *obs_row, int32_t *n_obs) {
    const size_t B = batch, C = cap;
    g_bjobs.assign(B, BruteJob{});
    g_posejobs.assign(B, PoseJob{});
    g_outlier.assign(B * C, 0);
    g_pose.assign(B * 16, 0.0);
    g_n_inl.assign(B, 0);
    g_iters.assign(B, 0);
    rt::RtDev &D = g_D;
    memset(&D, 0, sizeof(D));
    D.batch = batch;
    D.cap = cap;
    D.seed = seed;
    D.n_kp = n_kp;
    D.x = x;
    D.y = y;
    for (int i = 0; i < 4; ++i) D.K_cfg[i] = K_cfg[i];
    D.kf_stage = kf_stage;
    D.kf_status = kf_status;
    D.kf_num_valid = kf_num_valid;
    D.kf_of_frame = kf_of_frame;
    D.row_offsets = row_offsets;
    D.kf_bearings = kf_bearings;
    D.bearings = bearings;
    D.write_bearings = write_bearings;
    D.bjobs = g_bjobs.data();
    D.pairs = pairs;
    D.samples = samples;
    D.E = E;
    D.score = score;
    D.inlier = inlier;
    D.best_score = best_score;
    D.valid = valid;
    D.posejobs = g_posejobs.data();
    D.obs = obs;
    D.obs_kp = obs_kp;
    D.obs_row = obs_row;
    D.obs_outlier = g_outlier.data();
    D.stage = stage;
    D.status = status;
    D.matched = matched;
    D.num_bf = num_bf;
    D.num_robust = num_robust;

    emu_launch(rt::rt_prep_kernel, (unsigned)((batch + rt::kPrepThreads - 1) / rt::kPrepThreads),
               (unsigned)rt::kPrepThreads, D);
    // brute_match_kernel's matched_out for the frames it ran on (an empty job writes nothing)
    for (size_t b = 0; b < B; ++b)
        for (int i = 0; i < g_bjobs[b].n_frm; ++i) matched[b * C + i] = bf_matched[b * C + i];
    emu_launch(rt::rt_list_kernel, (unsigned)batch, (unsigned)rt::kThreads, D);
    emu_launch2(rt::rt_hypothesis_kernel, (unsigned)rt::kNumIter, (unsigned)batch, (unsigned)rt::kEssThreads,
                (size_t)cap * 2 * sizeof(float), D);
    emu_launch(rt::rt_select_kernel, (unsigned)batch, (unsigned)rt::kEssThreads, D);

    kt::KfDev &G = g_G;
    memset(&G, 0, sizeof(G));
    G.batch = batch;
    G.cap = cap;
    G.n_kp = n_kp;
    G.x = x;
    G.y = y;
    G.octave = octave;
    G.pose_last = pose_last;
    for (int l = 0; l < kt::kMaxLevels; ++l) G.inv_level_sigma_sq[l] = l < num_levels ? inv_level_sigma_sq[l] : 1.0f;
    G.kf_of_frame = kf_of_frame;
    G.row_offsets = row_offsets;
    G.kf_pos_w = kf_pos_w;
    G.posejobs = g_posejobs.data();
    G.obs = obs;
    G.obs_kp = obs_kp;
    G.obs_row = obs_row;
    G.obs_outlier = g_outlier.data();
    G.stage = stage;
    G.status = status;
    G.matched = matched;
    G.num_bow = (uint32_t *)num_robust;
    G.pose = g_pose.data();
    G.n_inliers = g_n_inl.data();
    G.lm_iters = g_iters.data();
    emu_launch(kt::kf_gather_kernel, (unsigned)batch, (unsigned)kt::kThreads, G);
    for (size_t b = 0; b < B; ++b) n_obs[b] = g_posejobs[b].n_pts;
}

extern "C" void emu_rt_finish(const uint8_t *outlier, int32_t *num_valid) {
    memcpy(g_outlier.data(), outlier, g_outlier.size());
    g_G.num_valid = num_valid;
    emu_launch(kt::kf_finish_kernel, (unsigned)g_G.batch, (unsigned)kt::kThreads, g_G);
}
