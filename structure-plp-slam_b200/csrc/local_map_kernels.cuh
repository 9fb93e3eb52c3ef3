// local_map_kernels.cuh -- device code of the batched local-map stage of tracking (local_map.cu launches it):
// tracking_module::optimize_current_frame_with_local_map (tracking_module.cc:732-835) for the frames whose
// motion_based_track succeeded, or, after a keyframe-track call of the same batch (keyframe_track.cu), whose
// bow_match_based_track did, or, after a robust-track call of the same batch (robust_track.cu), whose
// robust_match_based_track did; monocular points:
//   search_local_landmarks (:908-984) = exclusion of the landmarks the motion track matched, frame::can_observe
//   (data/frame.cc:797-824) and projection::match_frame_and_landmarks (margin, Lowe ratio 0.8)
//   -> pose_optimizer::optimize -> drop the outliers and count the tracked landmarks (:762-784).
// Free of host-side CUDA runtime dependencies so that tests/cta_emu can compile the same text for the host.
//
// Kernels, in launch order (the window matcher and the pose optimiser in between are the existing launchers):
//   local_prep_kernel     one CTA per frame: status, per-keypoint outputs, claimed flags, exclusions, camera centre,
//                         match job
//   local_observe_kernel  one thread per local row, grid (row chunks, frames): can_observe and the matcher's query
//   local_gather_kernel   one CTA per frame: keypoint -> local row, the observations of pose-opt #2 in keypoint order
//   local_finish_kernel   one CTA per frame: drop the outliers, count the tracked landmarks
//
// Exactness: the reprojection, the distance and the viewing-angle gates run in the reference's double / float mix and
// round like the oracle only when compiled with -fmad=false (build.py FILE_FLAGS: local_map.cu); predict_scale_level's
// logf is a comparison of the float ratio against the host-derived table of plp_fuse_level_thresholds.
#pragma once
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/plpslam_b200.h"
#include "devmath.cuh"
#include "keyframe_track.h"
#include "match_common.cuh"
#include "match_jobs.h"
#include "pose_jobs.h"

namespace plp {

namespace lm {

constexpr int kThreads = 256;          // prep / gather / finish: one CTA per frame
constexpr int kObserveThreads = 128;   // observe: one thread per local row
constexpr int kNumMatchesThr = 20;     // frame_tracker::num_matches_thr_: the motion track succeeded
constexpr int kMinPoseObs = 5;         // pose_optimizer.cc:153-156: fewer observations leave the frame untouched
constexpr int kMaxLevels = 16;
constexpr float kLoweRatio = 0.8f;     // tracking_module.cc:975
constexpr double kRayCosThr = 0.5;     // tracking_module.cc:944: can_observe(lm, 0.5, ...)

// kStatusLastLocalIdx also flags a keyframe-tracked frame without a valid local_idx block
enum : int32_t { kStatusOk = 0, kStatusCapacity = 1, kStatusLastLocalIdx = 2 };

struct LocalDev {
    int batch, cap, max_local;
    // the motion track of the same batch (tracker state)
    const int32_t *n_kp;
    const float *x, *y;                // undistorted keypoints, SoA (batch x cap)
    const int32_t *octave;
    const uint8_t *desc;               // batch x cap x 32
    const double *last_pos_w;
    const int32_t *last_offsets;
    const int32_t *motion_matched;     // batch x cap, after discard_outliers
    const double *motion_pose;         // batch x 16
    const int32_t *motion_num_valid;   // batch
    const PoseJob *motion_jobs;        // batch: n_pts = observations of pose-opt #1
    const int32_t *obs_last;           // batch x cap: last-frame row of each observation of pose-opt #1
    float inv_level_sigma_sq[kMaxLevels];
    // the keyframe and robust tracks of the same batch; kf.stage / rb.stage == nullptr without one
    KeyframeTrack kf, rb;
    // the local maps (rows of frame b: [offsets[b], offsets[b + 1]))
    const double *pos_w, *normal;
    const float *min_d, *max_d, *max_raw;
    const uint8_t *lm_desc;
    const uint8_t *valid;              // may be null
    const int32_t *offsets;
    const int32_t *last_local_idx;     // one per last-frame row
    // parameters
    plp_camera cam;
    float scale_factors[kMaxLevels];
    float level_thr[kMaxLevels];       // level_thr[k], 1 <= k < num_levels: smallest ratio whose level is >= k
    int num_levels;
    float margin;
    // scratch
    uint8_t *excl;                     // batch x max_local
    double *center;                    // batch x 3
    float *qx, *qy, *qradius;          // batch x max_local
    int32_t *qmin, *qmax;
    uint8_t *qvalid;
    int32_t *choice, *best;
    uint32_t *num_matches;             // batch
    uint8_t *claimed;                  // batch x cap
    PointMatchJob *mjobs;              // batch
    PoseJob *posejobs;                 // batch
    plp_pt_obs *obs;                   // batch x cap
    int32_t *obs_kp;
    uint8_t *obs_outlier;
    // outputs
    int32_t *matched, *local;          // batch x cap
    uint8_t *observable;               // rows of the local maps
    double *pose;                      // batch x 16
    int32_t *num_tracked, *n_inliers, *lm_iters, *status;  // batch
};

// The tracker whose result the frame starts from: the robust track where it ran, else the keyframe track where it ran
// (stage 1), else the motion track.  The robust track runs only where the keyframe track ran, and both match against
// rows of the same keyframe; the motion track's matches are rows of the last frame.
__device__ __forceinline__ bool kf_tracked(const LocalDev &D, int b) { return D.kf.stage && D.kf.stage[b]; }
__device__ __forceinline__ const KeyframeTrack &kf_record(const LocalDev &D, int b) {
    return D.rb.stage && D.rb.stage[b] ? D.rb : D.kf;
}
__device__ __forceinline__ int tracked_num_valid(const LocalDev &D, int b) {
    return kf_tracked(D, b) ? kf_record(D, b).num_valid[b] : D.motion_num_valid[b];
}
__device__ __forceinline__ const double *tracked_pose(const LocalDev &D, int b) {
    return (kf_tracked(D, b) ? kf_record(D, b).pose : D.motion_pose) + 16 * (size_t)b;
}

// the frame runs the stage: its tracker succeeded and its inputs are in range
__device__ __forceinline__ bool frame_active(const LocalDev &D, int b) {
    return tracked_num_valid(D, b) >= kNumMatchesThr && D.status[b] == kStatusOk;
}

// data/landmark.cc:341-362 through the host-derived threshold table
__device__ __forceinline__ int predict_level(float ratio, const LocalDev &D) {
    int lvl = 0;
    for (int k = 1; k < D.num_levels; ++k) lvl += (ratio >= D.level_thr[k]) ? 1 : 0;
    return lvl;
}

__global__ void __launch_bounds__(kThreads) local_prep_kernel(LocalDev D) {
    __shared__ int s_bad;
    const int b = blockIdx.x, tid = threadIdx.x;
    const int l0 = D.offsets[b], m = D.offsets[b + 1] - l0;
    const bool kf = kf_tracked(D, b);
    const KeyframeTrack &K = kf_record(D, b);
    const bool kf_ok = kf && K.status[b] == 0;
    // the rows the tracker matched against, and their local-list indices: the keyframe's or the last frame's
    const int32_t *row_local = D.last_local_idx;
    int r0 = D.last_offsets[b], r1 = D.last_offsets[b + 1];
    bool rows_ok = true;
    if (kf) {
        r0 = r1 = 0;
        row_local = K.local_idx;
        if (kf_ok) {  // frame b's local_idx block has one entry per row of its keyframe
            const int k = K.kf_of_frame[b];
            rows_ok = K.local_idx && K.local_idx_offsets[b + 1] - K.local_idx_offsets[b] ==
                                         K.kf_row_offsets[k + 1] - K.kf_row_offsets[k];
            if (rows_ok) {
                r0 = K.local_idx_offsets[b];
                r1 = K.local_idx_offsets[b + 1];
            }
        }
    }
    const int n = D.n_kp[b];
    const size_t base = (size_t)b * D.cap, lbase = (size_t)b * D.max_local;
    const bool fits = m >= 0 && m <= D.max_local;
    if (tid == 0) s_bad = rows_ok ? 0 : 1;
    __syncthreads();
    if (fits) {  // every matched-against row names a landmark of this frame's list, or none
        int bad = 0;
        for (int r = r0 + tid; r < r1; r += kThreads) {
            const int li = row_local[r];
            if (li < -1 || li >= m) bad = 1;
        }
        if (bad) atomicOr(&s_bad, 1);
        for (int j = tid; j < m; j += kThreads) D.excl[lbase + j] = 0;
    }
    __syncthreads();
    const int status = !fits ? kStatusCapacity : (s_bad ? kStatusLastLocalIdx : kStatusOk);
    const bool active = tracked_num_valid(D, b) >= kNumMatchesThr && status == kStatusOk;
    // the landmarks the frame keeps from its tracker; they are the matcher's claimed keypoints
    const int32_t *tracked_matched = kf ? K.matched : D.motion_matched;
    for (int i = tid; i < n; i += kThreads) {
        const int q = active ? tracked_matched[base + i] : -1;
        D.matched[base + i] = q;
        D.local[base + i] = -1;
        D.claimed[base + i] = q >= 0;
    }
    // Every landmark the tracker matched is excluded, the outliers of pose-opt #1 included: discard_outliers stamps
    // identifier_in_local_lm_search_ on those (frame_tracker.cc:273-278), search_local_landmarks on the rest (:910-926).
    if (active) {
        const int n1 = (kf ? K.posejobs : D.motion_jobs)[b].n_pts;
        const int32_t *obs_row = (kf ? K.obs_row : D.obs_last) + base;
        for (int k = tid; k < n1; k += kThreads) {
            const int li = row_local[r0 + obs_row[k]];
            if (li >= 0) D.excl[lbase + li] = 1;
        }
    }
    if (tid == 0) {
        D.status[b] = status;
        // cam_center_ = -R^T t (frame.cc:750)
        const double *P = tracked_pose(D, b);
        for (int r = 0; r < 3; ++r)
            D.center[3 * (size_t)b + r] = -(P[0 * 4 + r] * P[3] + P[1 * 4 + r] * P[7] + P[2 * 4 + r] * P[11]);
        PointMatchJob J;
        J.n = n;
        J.x = D.x + base;
        J.y = D.y + base;
        J.octave = D.octave + base;
        J.angle = nullptr;  // match_frame_and_landmarks has no orientation check
        J.x_right = nullptr;
        J.desc = D.desc + base * 32;
        J.claimed = D.claimed + base;
        J.m = active ? m : -1;  // -1: the matcher skips the frame
        J.qx = D.qx + lbase;
        J.qy = D.qy + lbase;
        J.qxr = nullptr;
        J.qradius = D.qradius + lbase;
        J.qmin = D.qmin + lbase;
        J.qmax = D.qmax + lbase;
        J.qangle = nullptr;
        J.qdesc = D.lm_desc + 32 * (size_t)(fits ? l0 : 0);
        J.qvalid = D.qvalid + lbase;
        J.choice = D.choice + lbase;
        J.best_idx_out = D.best + lbase;
        J.matched_out = nullptr;
        J.num_matches = D.num_matches + b;
        J.hamm_thr_p1 = 0;
        D.mjobs[b] = J;
    }
}

// search_local_landmarks (tracking_module.cc:928-962) for one local row: skip the excluded and erased landmarks, then
// frame::can_observe at the tracked pose; the observable ones become the matcher's queries (projection.cc:54-58).
__global__ void __launch_bounds__(kObserveThreads) local_observe_kernel(LocalDev D) {
    const int b = blockIdx.y;
    const int l0 = D.offsets[b], m = D.offsets[b + 1] - l0;
    const bool active = frame_active(D, b);
    const size_t lbase = (size_t)b * D.max_local;
    const double *P = tracked_pose(D, b);
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < m; j += gridDim.x * blockDim.x) {
        const size_t row = (size_t)l0 + j;
        uint8_t ok = 0;
        if (active) {
            if (!D.excl[lbase + j] && (!D.valid || D.valid[row])) {
                const double *X = D.pos_w + 3 * row;
                const Reproj r = reproject(D.cam, P, X);  // camera::reproject_to_image (perspective.cc:190-209)
                if (r.in_image) {
                    const double *c = D.center + 3 * (size_t)b;
                    const double d0 = X[0] - c[0], d1 = X[1] - c[1], d2 = X[2] - c[2];
                    const double dist = sqrt(d0 * d0 + d1 * d1 + d2 * d2);
                    const float fdist = (float)dist;  // landmark::is_inside_in_orb_scale(const float) (landmark.h:91-96)
                    if (D.min_d[row] <= fdist && fdist <= D.max_d[row]) {
                        const double *nm = D.normal + 3 * row;
                        const double ray_cos = (d0 * nm[0] + d1 * nm[1] + d2 * nm[2]) / dist;
                        if (!(ray_cos < kRayCosThr)) {
                            const int pred = predict_level(D.max_raw[row] / fdist, D);
                            D.qx[lbase + j] = (float)r.u;
                            D.qy[lbase + j] = (float)r.v;
                            D.qradius[lbase + j] = D.margin * D.scale_factors[pred];
                            D.qmin[lbase + j] = pred - 1;
                            D.qmax[lbase + j] = pred;
                            ok = 1;
                        }
                    }
                }
            }
            D.qvalid[lbase + j] = ok;
        }
        D.observable[row] = ok;
    }
}

// pose_optimizer.cc:126-151: one observation per keypoint holding a landmark, in keypoint order
__global__ void __launch_bounds__(kThreads) local_gather_kernel(LocalDev D) {
    __shared__ int warp_sums[kThreads / 32];
    __shared__ int s_base;
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n = D.n_kp[b];
    const size_t base = (size_t)b * D.cap, lbase = (size_t)b * D.max_local;
    const bool active = frame_active(D, b);
    const int l0 = D.offsets[b];
    // the positions of the tracker's matches: keyframe rows or last-frame rows
    const bool kf = kf_tracked(D, b);
    const KeyframeTrack &K = kf_record(D, b);
    const double *row_pos_w =
        kf ? K.kf_pos_w + 3 * (size_t)(active ? K.kf_row_offsets[K.kf_of_frame[b]] : 0)
           : D.last_pos_w + 3 * (size_t)D.last_offsets[b];
    if (active) {  // the local row each keypoint matched (projection.cc:115: frm.landmarks_.at(best_idx) = local_lm)
        const int m = D.offsets[b + 1] - l0;
        for (int q = tid; q < m; q += kThreads) {
            const int p = D.best[lbase + q];
            if (p >= 0) D.local[base + p] = q;
        }
    }
    if (tid == 0) s_base = 0;
    __syncthreads();
    for (int start = 0; start < n; start += kThreads) {
        const int i = start + tid;
        int qm = -1, ql = -1;
        if (i < n && active) {
            qm = D.matched[base + i];
            ql = D.local[base + i];
        }
        const int flag = qm >= 0 || ql >= 0;
        // ordered compaction
        const unsigned bal = __ballot_sync(0xffffffffu, flag);
        if (lane == 0) warp_sums[warp] = __popc(bal);
        __syncthreads();
        int off = s_base;
        for (int w = 0; w < warp; ++w) off += warp_sums[w];
        off += __popc(bal & ((1u << lane) - 1));
        if (flag) {
            const double *X = qm >= 0 ? row_pos_w + 3 * (size_t)qm : D.pos_w + 3 * (size_t)(l0 + ql);
            plp_pt_obs o;
            o.pos_w[0] = X[0];
            o.pos_w[1] = X[1];
            o.pos_w[2] = X[2];
            o.obs_x = D.x[base + i];
            o.obs_y = D.y[base + i];
            o.x_right = -1.0f;
            o.inv_sigma_sq = D.inv_level_sigma_sq[D.octave[base + i]];
            D.obs[base + off] = o;
            D.obs_kp[base + off] = i;
        }
        __syncthreads();
        if (tid == 0) {
            int tot = 0;
            for (int w = 0; w < kThreads / 32; ++w) tot += warp_sums[w];
            s_base += tot;
        }
        __syncthreads();
    }
    if (tid == 0) {  // an inactive frame has no observation: the optimiser copies the tracked pose and reports 0 / 0
        PoseJob J;
        J.T_in = tracked_pose(D, b);
        J.pts = D.obs + base;
        J.n_pts = s_base;
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

// tracking_module.cc:762-784: an outlier of pose-opt #2 loses its landmark; the inliers are num_tracked_lms_
__global__ void __launch_bounds__(kThreads) local_finish_kernel(LocalDev D) {
    __shared__ int s_cnt;
    const int b = blockIdx.x, tid = threadIdx.x;
    const size_t base = (size_t)b * D.cap;
    const int n_obs = D.posejobs[b].n_pts;
    // below kMinPoseObs the optimiser writes no outlier flag; an active frame holds >= kNumMatchesThr observations
    const bool flagged = frame_active(D, b) && n_obs >= kMinPoseObs;
    if (tid == 0) s_cnt = 0;
    __syncthreads();
    int cnt = 0;
    for (int k = tid; k < n_obs; k += kThreads) {
        if (flagged && D.obs_outlier[base + k]) {
            const int i = D.obs_kp[base + k];
            D.matched[base + i] = -1;
            D.local[base + i] = -1;
        } else {
            ++cnt;
        }
    }
    atomicAdd(&s_cnt, cnt);
    __syncthreads();
    if (tid == 0) D.num_tracked[b] = s_cnt;
}

}  // namespace lm

}  // namespace plp
