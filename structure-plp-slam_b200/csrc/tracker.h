// tracker.h -- internal: the state of a plp_tracker, shared by pipeline.cu (motion_based_track), keyframe_track.cu
// (bow_match_based_track), robust_track.cu (robust_match_based_track) and local_map.cu
// (optimize_current_frame_with_local_map), which read what the earlier calls of the batch left on the device.
#pragma once
#include <memory>

#include "common.cuh"
#include "camera_jobs.h"
#include "keyframe_track.h"
#include "match_jobs.h"
#include "pose_jobs.h"

namespace plp {

namespace lm {
struct LocalDev;  // local_map_kernels.cuh
}
namespace kt {
struct KfDev;  // keyframe_track_kernels.cuh
}
namespace rt {
struct RtDev;  // robust_track_kernels.cuh
}

struct TrackDev {
    int batch, cap, num_levels;
    // current frames (ORB output)
    const plp_keypoint *kp;
    const uint8_t *desc;
    const int32_t *n_kp;
    // last frames
    const double *last_pos_w;
    const int32_t *last_octave;
    const float *last_angle;
    const uint8_t *last_desc;
    const uint8_t *last_valid;
    const int32_t *last_offsets;
    const double *pose_pred, *pose_last;
    // scratch (SoA copies of the current keypoints, queries, jobs)
    float *x, *y, *angle;
    int32_t *octave;
    float *qx, *qy, *qxr, *qradius;
    int32_t *qmin, *qmax;
    uint8_t *qvalid;
    int32_t *choice;
    uint32_t *num_matches;
    ProjectJob *pjobs;       // 2 x batch (first attempt, retry)
    PointMatchJob *mjobs;    // 2 x batch
    PoseJob *posejobs;       // batch
    plp_pt_obs *obs;         // batch x cap
    int32_t *obs_kp;         // batch x cap : keypoint index of each observation
    int32_t *obs_last;       // batch x cap : last-frame row of each observation (before discard_outliers)
    uint8_t *obs_outlier;    // batch x cap
    float inv_level_sigma_sq[16];
    // outputs
    int32_t *matched;        // batch x cap : last-frame index per keypoint (-1: none) after discard_outliers
    double *pose_out;        // batch x 16
    int32_t *num_valid;      // batch
    int32_t *n_inliers;      // batch (pose optimiser return value)
    int32_t *lm_iters;       // batch
    int max_last;
};

}  // namespace plp

struct plp_tracker {
    plp_ctx *ctx = nullptr;
    int max_batch = 0, cap = 0, max_last = 0, num_levels = 0;
    plp_camera cam;
    plp_grid grid;
    float scale_factors[16];
    float inv_level_sigma_sq[16];
    float *d_scale_factors = nullptr;
    uint8_t *d_block = nullptr;  // one allocation carved into the scratch arrays
    plp::TrackDev dev;
    bool distorted = false;
    plp::UndistJob undist;             // camera and coefficients; kp / n_kp / batch set per call
    plp_keypoint *d_undist = nullptr;  // max_batch x cap (inside d_block)
    double *d_bearings = nullptr;      // max_batch x cap x 3
    // the most recent motion_track_batch_dev: its inputs, outputs and scratch, which local_map_track_batch_dev reads
    plp::TrackDev motion;
    bool has_motion = false;
    // local-map tracking (plp_tracker_reserve_local_map); d_local == nullptr until reserved
    int max_local = 0;
    uint8_t *d_local = nullptr;      // one allocation, carved by local_map.cu
    // the job with that scratch bound and the predict_scale_level thresholds set; every call adds its own inputs
    std::shared_ptr<plp::lm::LocalDev> local;
    // keyframe tracking (plp_tracker_reserve_keyframe_track); d_kf == nullptr until reserved
    int max_keyframes = 0, max_kf_points = 0;
    uint8_t *d_kf = nullptr;         // one allocation, carved by keyframe_track.cu
    std::shared_ptr<plp::kt::KfDev> kf;
    // the keyframe_track_batch_dev that followed the most recent motion track, for the robust and local-map stages
    plp::KeyframeTrack kf_track;
    plp_track_keyframe kf_table;     // the keyframe table that call was given
    int kf_batch = 0;
    bool has_kf = false;
    // robust tracking (plp_tracker_reserve_robust_track); d_rb == nullptr until reserved
    uint8_t *d_rb = nullptr;         // one allocation, carved by robust_track.cu
    std::shared_ptr<plp::rt::RtDev> rb;
    // the robust_track_batch_dev that followed the most recent keyframe track, for the local-map stage
    plp::KeyframeTrack rb_track;
    int rb_batch = 0;
    bool has_rb = false;
};
