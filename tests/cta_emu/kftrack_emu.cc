// kftrack_emu.cc -- csrc/keyframe_track_kernels.cuh (the batched keyframe tracker) executed on the host, with
// bow_match_kernel (bow_kernels.cuh) between the job and gather kernels.  The pose optimiser is not emulated:
// emu_kf_begin runs prep -> transform -> job -> bow match -> gather and returns what they wrote; the caller optimises
// the gathered observations and hands the outlier flags to emu_kf_finish.  With node_desc == nullptr the transform is
// skipped and the caller's word / node / weight rows stand for it, so that a test can pick the feature vectors.
#include "cta_emu.h"

#include <string.h>

#include <vector>

#include "keyframe_track_kernels.cuh"

using namespace plp;

namespace {

kt::KfDev g_D;
std::vector<int32_t> g_nb1, g_ne1, g_nb2, g_ne2, g_choice, g_m21, g_n_inl, g_iters, g_obs_kp;
std::vector<uint8_t> g_claimed, g_outlier;
std::vector<BowJob> g_bjobs;
std::vector<PoseJob> g_posejobs;
std::vector<double> g_pose;

}  // namespace

extern "C" void emu_kf_begin(int batch, int cap, int num_keyframes, int max_kf_points, const int32_t *n_kp,
                             const float *x, const float *y, const float *angle, const int32_t *octave,
                             const uint8_t *desc, const int32_t *motion_num_valid, const double *pose_last,
                             const float *inv_level_sigma_sq, int num_levels, const uint8_t *motion_valid,
                             const int32_t *kf_of_frame, const int32_t *row_offsets, const uint8_t *kf_desc,
                             const float *kf_angle, const uint8_t *kf_valid, const double *kf_pos_w,
                             const int32_t *fv_offsets, const uint32_t *node_ids, const int32_t *node_begin,
                             const uint32_t *indices, int G, const uint8_t *node_desc, const uint32_t *child_begin,
                             const uint32_t *children, const float *vweight, const int32_t *vword, int nid_level,
                             int32_t *word, int32_t *node, float *weight, int32_t *stage, int32_t *status,
                             uint32_t *fidx, int32_t *num_nodes, int32_t *nb2, int32_t *ne2, int32_t *nb1,
                             int32_t *ne1, int32_t *matched, uint32_t *num_bow, plp_pt_obs *obs, int32_t *obs_kp,
                             int32_t *obs_row, int32_t *n_obs) {
    const size_t B = batch, C = cap, R = max_kf_points;
    g_nb1.assign(B * C, -7);
    g_ne1.assign(B * C, -7);
    g_nb2.assign(B * C, -7);
    g_ne2.assign(B * C, -7);
    g_choice.assign(B * R, 0);
    g_m21.assign(B * R, 0);
    g_n_inl.assign(B, 0);
    g_iters.assign(B, 0);
    g_claimed.assign(B * C, 1);
    g_outlier.assign(B * C, 0);
    g_bjobs.assign(B, BowJob{});
    g_posejobs.assign(B, PoseJob{});
    g_pose.assign(B * 16, 0.0);
    kt::KfDev &D = g_D;
    memset(&D, 0, sizeof(D));
    D.batch = batch;
    D.cap = cap;
    D.num_keyframes = num_keyframes;
    D.max_kf_points = max_kf_points;
    D.n_kp = n_kp;
    D.x = x;
    D.y = y;
    D.angle = angle;
    D.octave = octave;
    D.desc = desc;
    D.motion_num_valid = motion_num_valid;
    D.pose_last = pose_last;
    for (int l = 0; l < kt::kMaxLevels; ++l) D.inv_level_sigma_sq[l] = l < num_levels ? inv_level_sigma_sq[l] : 1.0f;
    D.motion_valid = motion_valid;
    D.kf_of_frame = kf_of_frame;
    D.row_offsets = row_offsets;
    D.kf_desc = kf_desc;
    D.kf_angle = kf_angle;
    D.kf_valid = kf_valid;
    D.kf_pos_w = kf_pos_w;
    D.fv_offsets = fv_offsets;
    D.node_ids = node_ids;
    D.node_begin = node_begin;
    D.indices = indices;
    D.word = word;
    D.node = node;
    D.weight = weight;
    D.fidx = fidx;
    D.nb1 = g_nb1.data();
    D.ne1 = g_ne1.data();
    D.nb2 = g_nb2.data();
    D.ne2 = g_ne2.data();
    D.claimed = g_claimed.data();
    D.choice = g_choice.data();
    D.m21 = g_m21.data();
    D.bjobs = g_bjobs.data();
    D.posejobs = g_posejobs.data();
    D.obs = obs;
    D.obs_kp = obs_kp;
    D.obs_row = obs_row;
    D.obs_outlier = g_outlier.data();
    D.stage = stage;
    D.status = status;
    D.matched = matched;
    D.num_bow = num_bow;
    D.pose = g_pose.data();
    D.num_valid = nullptr;  // set by emu_kf_finish
    D.n_inliers = g_n_inl.data();
    D.lm_iters = g_iters.data();

    emu_launch(kt::kf_prep_kernel, (unsigned)((batch + kt::kPrepThreads - 1) / kt::kPrepThreads),
               (unsigned)kt::kPrepThreads, D);
    if (node_desc) {
        VocabDev V;
        V.desc = node_desc;
        V.child_begin = child_begin;
        V.children = children;
        V.weight = vweight;
        V.word_id = vword;
        const unsigned gx = (unsigned)((cap + 256 / G - 1) / (256 / G));
        if (G == 4) emu_launch2(kt::kf_transform_kernel<4>, gx, (unsigned)batch, 256u, (size_t)0, D, V, nid_level);
        else if (G == 8) emu_launch2(kt::kf_transform_kernel<8>, gx, (unsigned)batch, 256u, (size_t)0, D, V, nid_level);
        else if (G == 16) emu_launch2(kt::kf_transform_kernel<16>, gx, (unsigned)batch, 256u, (size_t)0, D, V, nid_level);
        else emu_launch2(kt::kf_transform_kernel<32>, gx, (unsigned)batch, 256u, (size_t)0, D, V, nid_level);
    }
    emu_launch2(kt::kf_job_kernel, (unsigned)batch, 1u, (unsigned)kt::kThreads,
                (size_t)cap * (sizeof(unsigned long long) + sizeof(uint32_t)), D);
    for (size_t b = 0; b < B; ++b) num_nodes[b] = g_bjobs[b].num_nodes;
    memcpy(nb1, g_nb1.data(), B * C * 4);
    memcpy(ne1, g_ne1.data(), B * C * 4);
    memcpy(nb2, g_nb2.data(), B * C * 4);
    memcpy(ne2, g_ne2.data(), B * C * 4);
    emu_launch(bow_match_kernel, (unsigned)batch, (unsigned)kMatchThreads, (const BowJob *)g_bjobs.data(),
               kt::kLoweRatio, 1);
    emu_launch(kt::kf_gather_kernel, (unsigned)batch, (unsigned)kt::kThreads, D);
    for (size_t b = 0; b < B; ++b) n_obs[b] = g_posejobs[b].n_pts;
}

extern "C" void emu_kf_finish(const uint8_t *outlier, int32_t *num_valid) {
    memcpy(g_outlier.data(), outlier, g_outlier.size());
    g_D.num_valid = num_valid;
    emu_launch(kt::kf_finish_kernel, (unsigned)g_D.batch, (unsigned)kt::kThreads, g_D);
}
