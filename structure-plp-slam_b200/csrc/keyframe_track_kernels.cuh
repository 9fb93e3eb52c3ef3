// keyframe_track_kernels.cuh -- device code of the batched keyframe tracker (keyframe_track.cu launches it):
// frame_tracker::bow_match_based_track (module/frame_tracker.cc:126-189) against each frame's reference keyframe, for
// the frames of a motion-track batch whose motion model was unusable or whose motion track failed:
//   frame::compute_bow (data/frame.cc:785-795, levelsup 4) -> bow_tree::match_frame_and_keyframe (match/bow_tree.cc:41-165,
//   Lowe 0.7, orientation check) -> pose_optimizer::optimize from last_frm.cam_pose_cw_ -> discard_outliers.
// Free of host-side CUDA runtime dependencies so that tests/cta_emu can compile the same text for the host.
//
// Kernels, in launch order (bow_match_kernel and the pose optimiser in between are the existing ones):
//   kf_prep_kernel       one thread per frame: stage flag and status
//   kf_transform_kernel  grid (row blocks, frames): the vocabulary descent of the active frames' keypoints only; the
//                        blocks of the other frames return at once
//   kf_job_kernel        one CTA per frame: the frame's bow_feat_vec_, the merge-join with the keyframe's node list,
//                        the BowJob (side 1 = keyframe, side 2 = frame)
//   kf_gather_kernel     one CTA per frame: the observations of the pose optimisation in keypoint order
//   kf_finish_kernel     one CTA per frame: discard_outliers
#pragma once
#include <stddef.h>
#include <stdint.h>

#include "../../include/plpslam_b200.h"
#include "bow_kernels.cuh"
#include "pose_jobs.h"
#include "track_common.cuh"

namespace plp {

namespace kt {

constexpr int kThreads = 256;         // job / gather / finish: one CTA per frame
constexpr int kPrepThreads = 128;
constexpr int kNumMatchesThr = 20;    // frame_tracker::num_matches_thr_
constexpr float kLoweRatio = 0.7f;    // frame_tracker.cc:130: bow_tree bow_matcher(0.7, true)
constexpr int kLevelsUp = 4;          // frame::compute_bow: transform(..., 4)
constexpr int kMaxLevels = 16;

enum : int32_t { kStatusOk = 0, kStatusCapacity = 1, kStatusKeyframe = 2 };

struct KfDev {
    int batch, cap, num_keyframes, max_kf_points;
    // the motion track of the same batch (tracker state)
    const int32_t *n_kp;
    const float *x, *y, *angle;        // undistorted keypoints, SoA (batch x cap)
    const int32_t *octave;
    const uint8_t *desc;               // batch x cap x 32
    const int32_t *motion_num_valid;   // batch
    const double *pose_last;           // batch x 16: last_frm.cam_pose_cw_
    float inv_level_sigma_sq[kMaxLevels];
    const uint8_t *motion_valid;       // batch, may be null (all 1)
    // the reference keyframes (plp_track_keyframe)
    const int32_t *kf_of_frame, *row_offsets;
    const uint8_t *kf_desc;
    const float *kf_angle;
    const uint8_t *kf_valid;           // may be null
    const double *kf_pos_w;
    const int32_t *fv_offsets;
    const uint32_t *node_ids;
    const int32_t *node_begin;
    const uint32_t *indices;
    // scratch
    int32_t *word, *node;              // batch x cap: the frames' BoW rows
    float *weight;
    uint32_t *fidx;                    // batch x cap: the frame's bow_feat_vec_ indices, node by node
    int32_t *nb1, *ne1, *nb2, *ne2;    // batch x cap: spans of the shared nodes
    uint8_t *claimed;                  // batch x cap
    int32_t *choice, *m21;             // batch x max_kf_points
    BowJob *bjobs;                     // batch
    PoseJob *posejobs;                 // batch
    plp_pt_obs *obs;                   // batch x cap
    int32_t *obs_kp, *obs_row;
    uint8_t *obs_outlier;
    // outputs
    int32_t *stage, *status;           // batch
    int32_t *matched;                  // batch x cap: matched_lms_in_frm as keyframe rows
    uint32_t *num_bow;                 // batch
    double *pose;                      // batch x 16
    int32_t *num_valid, *n_inliers, *lm_iters;  // batch
};

// the frame runs bow_match_based_track: it needs it and its inputs are in range
__device__ __forceinline__ bool frame_active(const KfDev &D, int b) {
    return D.stage[b] != 0 && D.status[b] == kStatusOk;
}

// The kernels have internal linkage, as essential_kernels.cuh's do: robust_track.cu launches the gather and finish
// kernels as well, over its own matches.
namespace {

// tracking_module.cc:608-637: the frames the reference hands to bow_match_based_track
__global__ void __launch_bounds__(kPrepThreads) kf_prep_kernel(KfDev D) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= D.batch) return;
    const bool motion_usable = !D.motion_valid || D.motion_valid[b] != 0;
    const int stage = !motion_usable || D.motion_num_valid[b] < kNumMatchesThr;
    int status = kStatusOk;
    if (stage) {
        const int k = D.kf_of_frame[b];
        if (k < 0 || k >= D.num_keyframes) {
            status = kStatusKeyframe;
        } else {
            const int rows = D.row_offsets[k + 1] - D.row_offsets[k];
            if (rows < 0 || rows > D.max_kf_points) status = kStatusCapacity;
        }
    }
    D.stage[b] = stage;
    D.status[b] = status;
}

// frame::compute_bow's per-row transform for the active frames: the descent is bow_transform_kernel's (bow_descend)
template <int G>
__global__ void __launch_bounds__(256) kf_transform_kernel(KfDev D, VocabDev V, int nid_level) {
    const int b = blockIdx.y;
    const int n = D.n_kp[b];
    const int first = blockIdx.x * (256 / G);
    if (!frame_active(D, b) || first >= n) return;  // uniform over the block
    const int gid = first + (int)(threadIdx.x / G), gl = (int)(threadIdx.x % G);
    const size_t base = (size_t)b * D.cap;
    const int row = min(gid, n - 1);  // surplus groups shadow the last row and do not store
    const BowWord w = bow_descend<G>(V, D.desc + 32 * (base + row), nid_level, gl);
    if (gl == 0 && gid < n) {
        D.word[base + gid] = w.word;
        D.node[base + gid] = w.node;
        D.weight[base + gid] = w.weight;
    }
}

// keyframe k's node holding node id `id`, or -1 (its node ids ascend)
__device__ __forceinline__ int find_node(const KfDev &D, int k, uint32_t id) {
    int lo = D.fv_offsets[k], hi = D.fv_offsets[k + 1];
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (D.node_ids[mid] < id)
            lo = mid + 1;
        else
            hi = mid;
    }
    return lo < D.fv_offsets[k + 1] && D.node_ids[lo] == id ? lo : -1;
}

// Dynamic shared memory: cap x (8 + 4) bytes.
// The frame's bow_feat_vec_ as TemplatedVocabulary::transform builds it: the rows with weight > 0, grouped by ascending
// node id, in row order inside a node (a row's place is the number of (node, row) keys below its own).  Then the nodes
// it shares with the keyframe's feature vector (the merge-join of bow_tree.cc:63-152, one binary search per frame node)
// and the BowJob.  A frame that does not run the stage gets an empty job.
__global__ void __launch_bounds__(kThreads) kf_job_kernel(KfDev D) {
    PLP_DYNAMIC_SMEM(smem_raw);
    __shared__ int s_kept;
    unsigned long long *s_key = (unsigned long long *)smem_raw;  // cap: (node id, row), ~0 for a row with weight 0
    uint32_t *s_node = (uint32_t *)(s_key + D.cap);              // cap: node id of the r-th feature-vector entry
    const int b = blockIdx.x, tid = threadIdx.x;
    const size_t base = (size_t)b * D.cap;
    const bool active = frame_active(D, b);
    const int n = active ? D.n_kp[b] : 0;
    const int k = active ? D.kf_of_frame[b] : 0;
    if (tid == 0) s_kept = 0;
    for (int i = tid; i < n; i += kThreads)
        s_key[i] = D.weight[base + i] > 0.0f ? ((unsigned long long)(uint32_t)D.node[base + i] << 32) | (unsigned)i
                                             : ~0ull;
    __syncthreads();
    int kept = 0;
    for (int i = tid; i < n; i += kThreads) {
        const unsigned long long key = s_key[i];
        if (key == ~0ull) continue;
        int r = 0;
        for (int j = 0; j < n; ++j) r += s_key[j] < key;
        D.fidx[base + r] = (uint32_t)i;
        s_node[r] = (uint32_t)(key >> 32);
        ++kept;
    }
    atomicAdd(&s_kept, kept);
    __syncthreads();
    const int nk = s_kept;
    // one shared node per first entry of a frame node that the keyframe also holds
    const auto kf_node = [&](int r) { return (r == 0 || s_node[r] != s_node[r - 1]) ? find_node(D, k, s_node[r]) : -1; };
    const int num_nodes = compact_in_order<kThreads>(
        nk, [&](int r) { return kf_node(r) >= 0; },
        [&](int r, int off) {
            const int a = kf_node(r);
            int e = r + 1;
            while (e < nk && s_node[e] == s_node[r]) ++e;
            D.nb1[base + off] = D.node_begin[a];
            D.ne1[base + off] = D.node_begin[a + 1];
            D.nb2[base + off] = r;
            D.ne2[base + off] = e;
        });
    if (tid == 0) {
        const int r0 = active ? D.row_offsets[k] : 0;
        BowJob J;
        J.n1 = active ? D.row_offsets[k + 1] - r0 : 0;
        J.n2 = n;
        J.num_nodes = num_nodes;
        J.desc1 = D.kf_desc + 32 * (size_t)r0;
        J.desc2 = D.desc + 32 * base;
        J.angle1 = D.kf_angle + r0;
        J.angle2 = D.angle + base;
        J.valid1 = D.kf_valid ? D.kf_valid + r0 : nullptr;  // bow_tree.cc:77-86
        J.valid2 = nullptr;
        J.idx1 = D.indices;
        J.idx2 = D.fidx + base;
        J.nb1 = D.nb1 + base;
        J.ne1 = D.ne1 + base;
        J.nb2 = D.nb2 + base;
        J.ne2 = D.ne2 + base;
        J.claimed = D.claimed + base;
        J.choice = D.choice + (size_t)b * D.max_kf_points;
        J.matched_2_of_1 = D.m21 + (size_t)b * D.max_kf_points;
        J.matched_1_of_2 = D.matched + base;
        J.num_matches = D.num_bow + b;
        D.bjobs[b] = J;
    }
}

// frame_tracker.cc:138-163 + pose_optimizer.cc:126-151: below 20 BoW matches the frame fails; otherwise one observation
// per keypoint holding a keyframe landmark, in keypoint order, and the optimisation starts from last_frm.cam_pose_cw_
__device__ __forceinline__ bool enough_matches(const KfDev &D, int b) {
    return frame_active(D, b) && D.num_bow[b] >= (uint32_t)kNumMatchesThr;
}

__global__ void __launch_bounds__(kThreads) kf_gather_kernel(KfDev D) {
    const int b = blockIdx.x;
    const size_t base = (size_t)b * D.cap;
    const bool enough = enough_matches(D, b);
    const int r0 = enough ? D.row_offsets[D.kf_of_frame[b]] : 0;
    const int32_t *matched = D.matched + base;
    const int n_obs = compact_in_order<kThreads>(
        enough ? D.n_kp[b] : 0, [&](int i) { return matched[i] >= 0; },
        [&](int i, int off) {
            const int q = matched[i];
            D.obs[base + off] = point_obs(D.kf_pos_w + 3 * (size_t)(r0 + q), D.x[base + i], D.y[base + i],
                                          D.inv_level_sigma_sq[D.octave[base + i]]);
            D.obs_kp[base + off] = i;
            D.obs_row[base + off] = q;
        });
    if (threadIdx.x == 0) {  // no observation: the optimiser copies pose_last and reports 0 / 0
        PoseJob J;
        J.T_in = D.pose_last + 16 * (size_t)b;
        J.pts = D.obs + base;
        J.n_pts = n_obs;
        J.lines = nullptr;
        J.n_lines = 0;
        J.T_out = D.pose + 16 * (size_t)b;
        J.pt_outlier = D.obs_outlier + base;
        J.line_outlier = nullptr;
        J.n_inliers = D.n_inliers + b;
        J.lm_iters = D.lm_iters + b;
        D.posejobs[b] = J;
    }
}

// frame_tracker::discard_outliers (frame_tracker.cc:166); a frame that failed or did not run keeps no match
__global__ void __launch_bounds__(kThreads) kf_finish_kernel(KfDev D) {
    const int b = blockIdx.x;
    const size_t base = (size_t)b * D.cap;
    const int valid = discard_outliers<kThreads>(D.n_kp[b], D.posejobs[b].n_pts, enough_matches(D, b),
                                                 D.obs_outlier + base, D.obs_kp + base, D.matched + base);
    if (threadIdx.x == 0) D.num_valid[b] = valid;
}

}  // namespace

}  // namespace kt

}  // namespace plp
