// plpslam_b200_adapter.hpp -- reference-side adapters: marshal the reference's own types (cv::Mat,
// cv::KeyPoint, data::frame, data::landmark, g2o-free PODs) into the C ABI of include/plpslam_b200.h.
//
// This header is compiled INSIDE the reference tree (it needs OpenCV / Eigen / the PLPSLAM headers, none of which
// exist in the authoring environment) and is what the patched bodies of
//   src/PLPSLAM/feature/orb_extractor.cc        (orb_extractor::extract)
//   src/PLPSLAM/match/projection.cc             (match_frame_and_landmarks, match_current_and_last_frames, *_line)
//   src/PLPSLAM/match/robust.cc                 (brute_force_match)
//   src/PLPSLAM/optimize/pose_optimizer*.cc     (optimize)
//   src/PLPSLAM/feature/line_extractor.cc       (LineFeatureTracker::extract_LSD_LBD)
//   src/PLPSLAM/data/frame.cc                   (match::stereo::compute call site)
//   src/PLPSLAM/match/projection.cc / robust.cc (match_frame_and_keyframe, match_for_triangulation)
//   src/PLPSLAM/mapping_module.cc               (fuse_landmark_duplication -> match::fuse::replace_duplication)
//   src/PLPSLAM/data/frame.cc / keyframe.cc     (compute_bow), src/PLPSLAM/module/relocalizer.cc (bow_tree matcher)
//   src/PLPSLAM/planar_mapping_module.cc        (estimate_plane_sequential_RANSAC, update_plane_via_RANSAC)
//   src/PLPSLAM/optimize/local_bundle_adjuster*.cc (optimize: gather, plp_local_ba, outlier erase + write-back, trimming)
// call.  Public signatures, PLPSLAM::system, the YAML configs and the map database stay unchanged.
// See INTEGRATION.md for the patch of each call site.
#pragma once
#ifdef PLPSLAM_B200_WITH_REFERENCE_TYPES

#include <cmath>
#include <cstring>
#include <set>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <vector>

#include <opencv2/core.hpp>
#include <opencv2/core/mat.hpp>

#include "PLPSLAM/camera/perspective.h"
#include "PLPSLAM/data/frame.h"
#include "PLPSLAM/data/keyframe.h"
#include "PLPSLAM/feature/line_descriptor/descriptor_custom.hpp"
#include "PLPSLAM/data/landmark.h"
#include "PLPSLAM/data/landmark_line.h"
#include "PLPSLAM/data/landmark_plane.h"
#include <functional>
#include <map>
#include <mutex>
#include <random>
#include "PLPSLAM/data/map_database.h"
#include "PLPSLAM/data/graph_node.h"
#include "PLPSLAM/util/trigonometric.h"
#include "plpslam_b200.h"
#include "plpslam_b200_line_trimming.h"

namespace plpslam_b200 {

inline void check(plp_status s) {
    // the reference's operators do not return errors; a failing GPU call is a hard error, never a CPU fallback
    if (s != PLP_OK) throw std::runtime_error(std::string("plpslam_b200: ") + plp_last_error());
}

// one context per calling thread (tracking thread, mapping thread), like the reference's per-thread objects
inline plp_ctx *thread_ctx(int device = 0) {
    thread_local plp_ctx *ctx = nullptr;
    if (!ctx) check(plp_ctx_create(device, &ctx));
    return ctx;
}

inline plp_grid grid_of(const PLPSLAM::camera::base *c) {
    return plp_grid{c->img_bounds_.min_x_, c->img_bounds_.min_y_, c->inv_cell_width_, c->inv_cell_height_,
                    (int32_t)c->num_grid_cols_, (int32_t)c->num_grid_rows_};
}

inline plp_camera camera_of(const PLPSLAM::camera::base *b) {
    const auto *c = static_cast<const PLPSLAM::camera::perspective *>(b);
    return plp_camera{c->fx_, c->fy_, c->cx_, c->cy_, b->focal_x_baseline_, b->true_baseline_,
                      b->img_bounds_.min_x_, b->img_bounds_.max_x_, b->img_bounds_.min_y_, b->img_bounds_.max_y_,
                      (int32_t)b->setup_type_};
}

// ---- camera::{perspective,fisheye}::undistort_keypoints + convert_keypoints_to_bearings (data/frame.cc:68, :79) ----------
// Replaces the two calls of every data::frame constructor.  cam: the camera's fx_, fy_, cx_, cy_ (camera_of() for a
// perspective camera; for a fisheye camera its own fx_ .. cy_) and img_bounds_; dist: Camera.model and the coefficients
// as the camera holds them (perspective {0, {k1_, k2_, p1_, p2_, k3_}}, fisheye {1, {k1_, k2_, k3_, k4_, 0}}) -- see
// INTEGRATION.md for the call site.
inline void undistort_keypoints(const plp_camera &cam, const plp_distortion &dist, const std::vector<cv::KeyPoint> &keypts,
                                std::vector<cv::KeyPoint> &undist_keypts,
                                PLPSLAM::eigen_alloc_vector<PLPSLAM::Vec3_t> &bearings) {
    const int n = (int)keypts.size();
    undist_keypts.resize(n);
    std::vector<double> b(3 * (size_t)n);
    check(plp_undistort_keypoints(thread_ctx(), &cam, &dist, reinterpret_cast<const plp_keypoint *>(keypts.data()), n,
                                  reinterpret_cast<plp_keypoint *>(undist_keypts.data()), b.data()));
    bearings.resize(n);
    for (int i = 0; i < n; ++i) bearings[i] = PLPSLAM::Vec3_t{b[3 * i], b[3 * i + 1], b[3 * i + 2]};
}

// ---- util::stereo_rectifier (util/stereo_rectifier.cc:39-92) ----------------------------------------------
// The constructor fills plp_stereo_rectifier_params from the StereoRectifier.* keys and the camera's fx_, fy_, cx_, cy_
// (see INTEGRATION.md) and calls create(); rectify() replaces the two cv::remap calls.  The GPU rectifies 8-bit
// single-channel images of the camera's size.  cv::remap would take any type and size, so anything else (a BGR frame of
// cv::VideoCapture, an image of another size) is rejected here instead of being read as a gray image of the camera's size.
struct stereo_rectifier_backend {
    plp_stereo_rectifier *h = nullptr;
    int rows = 0, cols = 0;
    stereo_rectifier_backend() = default;
    stereo_rectifier_backend(const stereo_rectifier_backend &) = delete;
    stereo_rectifier_backend &operator=(const stereo_rectifier_backend &) = delete;
    ~stereo_rectifier_backend() { plp_stereo_rectifier_destroy(h); }
    void create(const plp_stereo_rectifier_params &p, int r, int c) {
        check(plp_stereo_rectifier_create(thread_ctx(), &p, r, c, &h));
        rows = r;
        cols = c;
    }
    void require_gray_of_camera_size(const cv::Mat &m, const char *side) const {
        if (m.empty() || cv::_InputArray(m).type() != CV_8UC1 || m.rows != rows || m.cols != cols)
            throw std::runtime_error(std::string("plpslam_b200: stereo_rectifier::rectify: the ") + side +
                                     " image must be 8-bit single-channel (CV_8UC1) of " + std::to_string(rows) + " x " +
                                     std::to_string(cols) + " (convert colour frames to gray before rectifying)");
    }
    void rectify(const cv::Mat &in_l, const cv::Mat &in_r, cv::Mat &out_l, cv::Mat &out_r) const {
        require_gray_of_camera_size(in_l, "left");
        require_gray_of_camera_size(in_r, "right");
        if (in_l.step != in_r.step) throw std::runtime_error("plpslam_b200: left and right images differ in row stride");
        out_l.create(rows, cols, CV_8UC1);
        out_r.create(rows, cols, CV_8UC1);
        if (out_l.step != out_r.step) throw std::runtime_error("plpslam_b200: output images differ in row stride");
        check(plp_stereo_rectify(thread_ctx(), h, in_l.data, in_r.data, in_l.step, out_l.data, out_r.data, out_l.step));
    }
};

// ---- feature::orb_extractor::extract (feature/orb_extractor.cc:73-160) -------------------------------------
struct orb_backend {
    plp_orb *h = nullptr;
    int rows = 0, cols = 0;
    std::vector<plp_keypoint> kp;
    void ensure(const PLPSLAM::feature::orb_params &p, int r, int c) {
        if (h && r == rows && c == cols) return;
        if (h) plp_orb_destroy(h);
        plp_orb_params q{p.max_num_keypts_, p.scale_factor_, p.num_levels_, p.ini_fast_thr_, p.min_fast_thr};
        check(plp_orb_create(thread_ctx(), &q, r, c, 1, &h));
        rows = r;
        cols = c;
        kp.resize(plp_orb_capacity(h));
    }
    void extract(const cv::Mat &image, const cv::Mat &mask, std::vector<cv::KeyPoint> &keypts,
                 const cv::_OutputArray &out_descriptors) {
        cv::Mat desc(plp_orb_capacity(h), 32, CV_8U);
        int n = 0;
        check(plp_orb_extract(h, image.data, image.rows, image.cols, image.step, mask.empty() ? nullptr : mask.data,
                              mask.empty() ? 0 : mask.step, kp.data(), desc.data, &n));
        static_assert(sizeof(plp_keypoint) == sizeof(cv::KeyPoint), "plp_keypoint mirrors cv::KeyPoint");
        keypts.assign(reinterpret_cast<cv::KeyPoint *>(kp.data()), reinterpret_cast<cv::KeyPoint *>(kp.data()) + n);
        if (n == 0)
            out_descriptors.release();
        else
            desc.rowRange(0, n).copyTo(out_descriptors);
    }
};

// ---- match::projection::match_frame_and_landmarks (match/projection.cc:37-121) -------------------------------
inline unsigned match_frame_and_landmarks(PLPSLAM::data::frame &frm,
                                          const std::vector<PLPSLAM::data::landmark *> &local_landmarks, float margin,
                                          float lowe_ratio) {
    const int n = frm.num_keypts_, m = (int)local_landmarks.size();
    std::vector<float> x(n), y(n), xr(n), qx(m), qy(m), qxr(m);
    std::vector<int32_t> oct(n), lvl(m), best(m);
    std::vector<uint8_t> claimed(n), valid(m), qdesc((size_t)m * 32);
    for (int i = 0; i < n; ++i) {
        x[i] = frm.undist_keypts_[i].pt.x;
        y[i] = frm.undist_keypts_[i].pt.y;
        oct[i] = frm.undist_keypts_[i].octave;
        xr[i] = frm.stereo_x_right_[i];
        claimed[i] = frm.landmarks_[i] && frm.landmarks_[i]->has_observation();
    }
    for (int q = 0; q < m; ++q) {
        auto *lm = local_landmarks[q];
        valid[q] = lm->is_observable_in_tracking_ && !lm->will_be_erased();
        qx[q] = lm->reproj_in_tracking_(0);
        qy[q] = lm->reproj_in_tracking_(1);
        qxr[q] = lm->x_right_in_tracking_;
        lvl[q] = lm->scale_level_in_tracking_;
        const cv::Mat d = lm->get_descriptor();
        std::copy(d.data, d.data + 32, qdesc.begin() + (size_t)q * 32);
    }
    plp_frame_points fp{n, x.data(), y.data(), oct.data(), nullptr, xr.data(), frm.descriptors_.data, claimed.data()};
    plp_landmark_queries lq{m, qx.data(), qy.data(), qxr.data(), lvl.data(), qdesc.data(), valid.data()};
    const plp_grid g = grid_of(frm.camera_);
    uint32_t num = 0;
    check(plp_match_frame_and_landmarks(thread_ctx(), &fp, &g, frm.scale_factors_.data(), (int)frm.scale_factors_.size(),
                                        &lq, margin, lowe_ratio, best.data(), &num));
    for (int q = 0; q < m; ++q)  // re-apply the pointer writes in landmark order
        if (best[q] >= 0) frm.landmarks_[best[q]] = local_landmarks[q];
    return num;
}

// ---- optimize::pose_optimizer::optimize (optimize/pose_optimizer.cc:53-229) ----------------------------------
inline unsigned pose_optimize(PLPSLAM::data::frame &frm, bool with_lines, int num_trials = 4, int num_each_iter = 10) {
    std::vector<plp_pt_obs> pts;
    std::vector<unsigned> pt_idx;
    for (unsigned idx = 0; idx < frm.num_keypts_; ++idx) {
        auto lm = frm.landmarks_[idx];
        if (!lm || lm->will_be_erased()) continue;
        frm.outlier_flags_[idx] = false;
        const PLPSLAM::Vec3_t X = lm->get_pos_in_world();
        const auto &kp = frm.undist_keypts_[idx];
        pts.push_back(plp_pt_obs{{X(0), X(1), X(2)}, kp.pt.x, kp.pt.y, frm.stereo_x_right_[idx],
                                 frm.inv_level_sigma_sq_[kp.octave]});
        pt_idx.push_back(idx);
    }
    std::vector<plp_line_obs> lines;
    std::vector<unsigned> line_idx;
    if (with_lines && pts.size() >= 5) {
        for (unsigned idx = 0; idx < frm._num_keylines; ++idx) {
            auto ll = frm._landmarks_line[idx];
            if (!ll || ll->will_be_erased()) continue;
            frm._outlier_flags_line[idx] = false;
            const PLPSLAM::Vec6_t L = ll->get_PlueckerCoord();
            const auto &kl = frm._keylsd[idx];
            lines.push_back(plp_line_obs{{L(0), L(1), L(2), L(3), L(4), L(5)}, kl.getStartPoint().x, kl.getStartPoint().y,
                                         kl.getEndPoint().x, kl.getEndPoint().y, frm._inv_level_sigma_sq_lsd[kl.octave], 0.f});
            line_idx.push_back(idx);
        }
    }
    const plp_camera cam = camera_of(frm.camera_);
    const plp_pose_opt_cfg cfg{num_trials, num_each_iter};
    double T_in[16], T_out[16];
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) T_in[r * 4 + c] = frm.cam_pose_cw_(r, c);
    std::vector<uint8_t> pout(pts.size() + 1), lout(lines.size() + 1);
    int32_t n_inliers = 0;
    check(plp_pose_optimize(thread_ctx(), &cam, T_in, pts.data(), (int)pts.size(), lines.data(), (int)lines.size(), &cfg,
                            T_out, pout.data(), lout.data(), &n_inliers));
    if (pts.size() < 5) return 0;  // pose_optimizer.cc:153-156
    for (size_t k = 0; k < pt_idx.size(); ++k) frm.outlier_flags_[pt_idx[k]] = pout[k];
    for (size_t k = 0; k < line_idx.size(); ++k) frm._outlier_flags_line[line_idx[k]] = lout[k];
    PLPSLAM::Mat44_t T;
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) T(r, c) = T_out[r * 4 + c];
    frm.set_cam_pose(T);
    return (unsigned)n_inliers;
}

// ---- feature::LineFeatureTracker::extract_LSD_LBD (feature/line_extractor.cc:88-160) -------------------------
struct line_backend {
    plp_line *h = nullptr;
    int rows = 0, cols = 0;
    std::vector<plp_keyline> kl;
    std::vector<double> fn;
    void ensure(int r, int c) {
        if (h && r == rows && c == cols) return;
        if (h) plp_line_destroy(h);
        check(plp_line_create(thread_ctx(), r, c, 1, &h));
        rows = r;
        cols = c;
        kl.resize(plp_line_capacity(h));
        fn.resize((size_t)plp_line_capacity(h) * 3);
    }
    void extract(const cv::Mat &img, std::vector<cv::line_descriptor::KeyLine> &frame_keylsd, cv::Mat &frame_lbd_descr,
                 std::vector<PLPSLAM::Vec3_t> &keyline_functions) {
        static_assert(sizeof(plp_keyline) == sizeof(cv::line_descriptor::KeyLine), "plp_keyline mirrors KeyLine");
        cv::Mat lbd(plp_line_capacity(h), 32, CV_8U);
        int n = 0;
        check(plp_line_extract(h, img.data, img.rows, img.cols, img.step, kl.data(), lbd.data, fn.data(), &n));
        auto *k = reinterpret_cast<cv::line_descriptor::KeyLine *>(kl.data());
        frame_keylsd.assign(k, k + n);                                  // line_extractor.cc:143
        frame_lbd_descr = n ? lbd.rowRange(0, n).clone() : cv::Mat();   // :144
        for (int i = 0; i < n; ++i)                                      // :147-159 (appended, like the reference)
            keyline_functions.emplace_back(fn[3 * i], fn[3 * i + 1], fn[3 * i + 2]);
    }
};

// ---- match::stereo::compute (match/stereo.cc:45-150), called from data::frame (frame.cc:470-480) -------------
// `left` / `right` are the backends of the two extractors that just produced keypts_ / keypts_right_.
inline void stereo_compute(const orb_backend &left, const orb_backend &right, const std::vector<cv::KeyPoint> &keypts_left,
                           const std::vector<cv::KeyPoint> &keypts_right, const cv::Mat &descs_left,
                           const cv::Mat &descs_right, float focal_x_baseline, float true_baseline,
                           std::vector<float> &stereo_x_right, std::vector<float> &depths) {
    stereo_x_right.assign(keypts_left.size(), -1.0f);
    depths.assign(keypts_left.size(), -1.0f);
    check(plp_stereo_compute(thread_ctx(), left.h, right.h, reinterpret_cast<const plp_keypoint *>(keypts_left.data()),
                             descs_left.data, (int)keypts_left.size(),
                             reinterpret_cast<const plp_keypoint *>(keypts_right.data()), descs_right.data,
                             (int)keypts_right.size(), focal_x_baseline, true_baseline, stereo_x_right.data(),
                             depths.data(), nullptr));
}

// ---- match::projection::match_frame_and_keyframe (match/projection.cc:529-645) --------------------------------
inline unsigned match_frame_and_keyframe(PLPSLAM::data::frame &curr_frm, PLPSLAM::data::keyframe *keyfrm,
                                         const std::set<PLPSLAM::data::landmark *> &already_matched_lms, float margin,
                                         unsigned hamm_dist_thr, bool check_orientation) {
    const PLPSLAM::Mat33_t rot_cw = curr_frm.cam_pose_cw_.block<3, 3>(0, 0);
    const PLPSLAM::Vec3_t trans_cw = curr_frm.cam_pose_cw_.block<3, 1>(0, 3);
    const PLPSLAM::Vec3_t cam_center = -rot_cw.transpose() * trans_cw;
    const auto landmarks = keyfrm->get_landmarks();
    const int n = curr_frm.num_keypts_, m = (int)landmarks.size();
    std::vector<float> x(n), y(n), ang(n), qx(m), qy(m), qang(m);
    std::vector<int32_t> oct(n), lvl(m, 0), matched(n);
    std::vector<uint8_t> claimed(n), valid(m, 0), qdesc((size_t)m * 32, 0);
    for (int i = 0; i < n; ++i) {
        x[i] = curr_frm.undist_keypts_[i].pt.x;
        y[i] = curr_frm.undist_keypts_[i].pt.y;
        oct[i] = curr_frm.undist_keypts_[i].octave;
        ang[i] = curr_frm.undist_keypts_[i].angle;
        claimed[i] = curr_frm.landmarks_[i] != nullptr;  // :604
    }
    for (int idx = 0; idx < m; ++idx) {  // the gates of :543-582 stay on the host (they read landmark state)
        auto *lm = landmarks[idx];
        if (!lm || lm->will_be_erased() || already_matched_lms.count(lm)) continue;
        const PLPSLAM::Vec3_t pos_w = lm->get_pos_in_world();
        PLPSLAM::Vec2_t reproj;
        float x_right;
        if (!curr_frm.camera_->reproject_to_image(rot_cw, trans_cw, pos_w, reproj, x_right)) continue;
        const auto dist = (pos_w - cam_center).norm();
        if (dist < lm->get_min_valid_distance() || lm->get_max_valid_distance() < dist) continue;
        valid[idx] = 1;
        qx[idx] = reproj(0);
        qy[idx] = reproj(1);
        lvl[idx] = lm->predict_scale_level(dist, &curr_frm);
        qang[idx] = keyfrm->undist_keypts_[idx].angle;
        std::memcpy(&qdesc[(size_t)idx * 32], lm->get_descriptor().data, 32);
    }
    const plp_frame_points fp{n, x.data(), y.data(), oct.data(), ang.data(), nullptr, curr_frm.descriptors_.data,
                              claimed.data()};
    const plp_landmark_queries q{m, qx.data(), qy.data(), nullptr, lvl.data(), qdesc.data(), valid.data()};
    const plp_grid grid = grid_of(curr_frm.camera_);
    uint32_t num = 0;
    check(plp_match_frame_and_keyframe(thread_ctx(), &fp, &grid, curr_frm.scale_factors_.data(),
                                       (int)curr_frm.scale_factors_.size(), &q, qang.data(), margin, hamm_dist_thr,
                                       check_orientation, matched.data(), &num));
    for (int i = 0; i < n; ++i)
        if (matched[i] >= 0) curr_frm.landmarks_[i] = landmarks[matched[i]];
    return num;
}

// ---- match::robust::match_for_triangulation (match/robust.cc:43-216) ------------------------------------------
template <class FeatureVector>  // DBoW2::FeatureVector or fbow::BoWFeatVector: ordered map node id -> index list
inline unsigned match_for_triangulation(PLPSLAM::data::keyframe *kf1, PLPSLAM::data::keyframe *kf2,
                                        const FeatureVector &fv1, const FeatureVector &fv2, const PLPSLAM::Mat33_t &E_12,
                                        bool check_orientation,
                                        std::vector<std::pair<unsigned, unsigned>> &matched_idx_pairs) {
    auto flatten_fv = [](const FeatureVector &fv, std::vector<uint32_t> &ids, std::vector<int32_t> &off,
                         std::vector<uint32_t> &idx) {
        off.push_back(0);
        for (const auto &node : fv) {
            ids.push_back(node.first);
            idx.insert(idx.end(), node.second.begin(), node.second.end());
            off.push_back((int32_t)idx.size());
        }
    };
    auto flatten_kf = [](PLPSLAM::data::keyframe *kf, std::vector<float> &ang, std::vector<int32_t> &oct,
                         std::vector<double> &bear, std::vector<uint8_t> &has) {
        const auto lms = kf->get_landmarks();
        for (unsigned i = 0; i < kf->num_keypts_; ++i) {
            ang.push_back(kf->undist_keypts_[i].angle);
            oct.push_back(kf->undist_keypts_[i].octave);
            for (int k = 0; k < 3; ++k) bear.push_back(kf->bearings_[i](k));
            has.push_back(lms[i] != nullptr);
        }
    };
    std::vector<uint32_t> ids1, ids2, idx1, idx2;
    std::vector<int32_t> off1, off2, oct1, oct2;
    std::vector<float> ang1, ang2;
    std::vector<double> b1, b2;
    std::vector<uint8_t> has1, has2;
    flatten_fv(fv1, ids1, off1, idx1);
    flatten_fv(fv2, ids2, off2, idx2);
    flatten_kf(kf1, ang1, oct1, b1, has1);
    flatten_kf(kf2, ang2, oct2, b2, has2);
    PLPSLAM::Vec3_t epi;
    kf2->camera_->reproject_to_bearing(kf2->get_rotation(), kf2->get_translation(), kf1->get_cam_center(), epi);  // :54-57
    double E[9];
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) E[r * 3 + c] = E_12(r, c);
    const plp_keyframe_points p1{(int32_t)kf1->num_keypts_, kf1->descriptors_.data, ang1.data(), oct1.data(), b1.data(),
                                 has1.data(), kf1->stereo_x_right_.data()};
    const plp_keyframe_points p2{(int32_t)kf2->num_keypts_, kf2->descriptors_.data, ang2.data(), oct2.data(), b2.data(),
                                 has2.data(), kf2->stereo_x_right_.data()};
    const plp_bow_feature_vector v1{(int32_t)ids1.size(), ids1.data(), off1.data(), idx1.data()};
    const plp_bow_feature_vector v2{(int32_t)ids2.size(), ids2.data(), off2.data(), idx2.data()};
    std::vector<int32_t> m21(kf1->num_keypts_);
    uint32_t num = 0;
    check(plp_match_for_triangulation(thread_ctx(), &p1, &p2, &v1, &v2, E, epi.data(), kf1->scale_factors_.data(),
                                      (int)kf1->scale_factors_.size(), check_orientation, m21.data(), &num));
    matched_idx_pairs.clear();
    for (unsigned i = 0; i < m21.size(); ++i)   // :201-213
        if (m21[i] >= 0) matched_idx_pairs.emplace_back(i, (unsigned)m21[i]);
    return num;
}

// ---- match::robust::brute_force_match + match_frame_and_keyframe (match/robust.cc:218-385) -------------------------
inline unsigned brute_force_match(PLPSLAM::data::frame &frm, PLPSLAM::data::keyframe *keyfrm, float lowe_ratio,
                                  bool check_orientation, std::vector<std::pair<int, int>> &matches) {
    const auto keyfrm_lms = keyfrm->get_landmarks();
    const int n_frm = frm.num_keypts_, n_kf = (int)keyfrm->num_keypts_;
    std::vector<float> a_frm(n_frm), a_kf(n_kf);
    std::vector<uint8_t> kf_valid(n_kf);
    for (int i = 0; i < n_frm; ++i) a_frm[i] = frm.keypts_[i].angle;
    for (int j = 0; j < n_kf; ++j) {
        a_kf[j] = keyfrm->keypts_[j].angle;
        kf_valid[j] = keyfrm_lms[j] && !keyfrm_lms[j]->will_be_erased();  // robust.cc:283-291
    }
    std::vector<int32_t> matched(n_frm);
    uint32_t num = 0;
    check(plp_match_brute_force(thread_ctx(), frm.descriptors_.data, a_frm.data(), n_frm, keyfrm->descriptors_.data,
                                a_kf.data(), kf_valid.data(), n_kf, lowe_ratio, check_orientation, matched.data(), &num));
    matches.clear();
    for (int i = 0; i < n_frm; ++i)  // robust.cc:372-382: pairs (idx_1 in frame, idx_2 in keyframe), ascending idx_1
        if (matched[i] >= 0) matches.emplace_back(i, matched[i]);
    return num;
}

// robust::match_frame_and_keyframe (:218-255): brute force, then the eight-point RANSAC keeps the inliers.  The sample
// sets are drawn here with the reference's own util::create_random_array, so the random stream is the reference's.
inline unsigned robust_match_frame_and_keyframe(PLPSLAM::data::frame &frm, PLPSLAM::data::keyframe *keyfrm, float lowe_ratio,
                                                bool check_orientation,
                                                std::vector<PLPSLAM::data::landmark *> &matched_lms_in_frm) {
    const auto keyfrm_lms = keyfrm->get_landmarks();
    matched_lms_in_frm.assign(frm.num_keypts_, nullptr);
    std::vector<std::pair<int, int>> matches;
    brute_force_match(frm, keyfrm, lowe_ratio, check_orientation, matches);
    const int M = (int)matches.size();
    if (M < 8) return 0;  // essential_solver.cc:45-49 -> solution invalid -> robust.cc:233-236
    constexpr int num_iter = 50;
    std::vector<int32_t> samples((size_t)num_iter * 8), m12((size_t)M * 2);
    for (int it = 0; it < num_iter; ++it) {
        const auto idx = PLPSLAM::util::create_random_array(8, 0U, (unsigned)(M - 1));
        for (int k = 0; k < 8; ++k) samples[(size_t)it * 8 + k] = (int32_t)idx[k];
    }
    for (int i = 0; i < M; ++i) m12[2 * i] = matches[i].first, m12[2 * i + 1] = matches[i].second;
    std::vector<double> b1((size_t)frm.num_keypts_ * 3), b2((size_t)keyfrm->num_keypts_ * 3);
    for (unsigned i = 0; i < frm.num_keypts_; ++i)
        for (int k = 0; k < 3; ++k) b1[3 * i + k] = frm.bearings_[i](k);
    for (unsigned i = 0; i < keyfrm->num_keypts_; ++i)
        for (int k = 0; k < 3; ++k) b2[3 * i + k] = keyfrm->bearings_[i](k);
    std::vector<uint8_t> inlier(M);
    double E[9], score = 0;
    int32_t valid = 0;
    check(plp_essential_ransac(thread_ctx(), b1.data(), (int)frm.num_keypts_, b2.data(), (int)keyfrm->num_keypts_, m12.data(),
                               M, samples.data(), num_iter, /*recompute=*/0, inlier.data(), E, &score, &valid));
    if (!valid) return 0;
    unsigned num_inlier_matches = 0;
    for (int i = 0; i < M; ++i) {  // :240-252
        if (!inlier[i]) continue;
        matched_lms_in_frm[matches[i].first] = keyfrm_lms[matches[i].second];
        ++num_inlier_matches;
    }
    return num_inlier_matches;
}

// ---- relocalizer::relocalize's EPnP (module/relocalizer.cc:86-100) for every candidate keyframe in one call ----------
// run[i]: the candidate reached the loop's pnp_solver (not will_be_erased(), >= min_num_bow_matches_ BoW matches).  The
// correspondences are extract_valid_indices / setup_pnp_solver's (:254-291); max_cos_error and the 4-point samples are
// computed with the reference's own util::cos and util::create_random_array, and samples are drawn only for candidates
// that run.  Result i stands in for pnp_solver i: valid, get_best_cam_pose(), and
// resample_by_indices(valid_indices, get_inlier_flags()) (frame keypoint indices).
struct pnp_candidate_result {
    bool valid = false;
    PLPSLAM::Mat44_t pose_cw;
    std::vector<unsigned> inlier_indices;
};

inline std::vector<pnp_candidate_result> pnp_ransac_candidates(const PLPSLAM::data::frame &curr_frm,
                                                               const std::vector<std::vector<PLPSLAM::data::landmark *>> &matched_landmarks,
                                                               const std::vector<bool> &run, unsigned num_iter = 30,
                                                               unsigned min_num_inliers = 10) {
    const size_t K = matched_landmarks.size();
    if (run.size() != K) throw std::invalid_argument("plpslam_b200::pnp_ransac_candidates: run and matched_landmarks differ in size");
    constexpr double max_rad_error = 1.0 * M_PI / 180.0;  // pnp_solver.cc:47
    std::vector<int32_t> off(K + 1, 0), samples;
    std::vector<std::vector<unsigned>> valid_indices(K);
    std::vector<double> bearings, pos_w;
    std::vector<float> max_cos;
    for (size_t k = 0; k < K; ++k) {
        if (run[k]) {
            for (unsigned idx = 0; idx < matched_landmarks[k].size(); ++idx) {
                auto *lm = matched_landmarks[k][idx];
                if (!lm || lm->will_be_erased()) continue;
                valid_indices[k].push_back(idx);
                const PLPSLAM::Vec3_t pw = lm->get_pos_in_world();
                for (int c = 0; c < 3; ++c) bearings.push_back(curr_frm.bearings_[idx](c)), pos_w.push_back(pw(c));
                max_cos.push_back(PLPSLAM::util::cos(curr_frm.scale_factors_.at(curr_frm.keypts_[idx].octave) * max_rad_error));
            }
        }
        const unsigned n = (unsigned)valid_indices[k].size();
        off[k + 1] = off[k] + (int32_t)n;
        for (unsigned it = 0; it < num_iter; ++it) {
            if (n >= 4 && n >= min_num_inliers) {
                const auto idx = PLPSLAM::util::create_random_array(4, 0U, n - 1);
                samples.insert(samples.end(), idx.begin(), idx.end());
            } else {
                samples.insert(samples.end(), 4, 0);  // not read: the problem does not run
            }
        }
    }
    const size_t N = (size_t)off[K];
    std::vector<int32_t> valid(K), num_inliers(K);
    std::vector<double> pose(K * 16);
    std::vector<uint8_t> flags(N + 1);
    check(plp_pnp_ransac(thread_ctx(), (int)K, off.data(), bearings.data(), pos_w.data(), max_cos.data(), samples.data(),
                         (int)num_iter, (int)min_num_inliers, /*recompute=*/1, valid.data(), num_inliers.data(), pose.data(),
                         flags.data()));
    std::vector<pnp_candidate_result> out(K);
    for (size_t k = 0; k < K; ++k) {
        out[k].valid = run[k] && valid[k];
        if (!out[k].valid) continue;
        for (int r = 0; r < 4; ++r)
            for (int c = 0; c < 4; ++c) out[k].pose_cw(r, c) = pose[16 * k + 4 * r + c];
        for (size_t i = 0; i < valid_indices[k].size(); ++i)
            if (flags[off[k] + i]) out[k].inlier_indices.push_back(valid_indices[k][i]);
    }
    return out;
}

// ---- loop_detector::select_loop_candidate_via_Sim3's linear Sim3 (module/loop_detector.cc:368-374) for every candidate in
// one call ----
// run[i]: candidate i reached the loop's sim3_solver (not will_be_erased(), >= 20 BoW matches); matched_lms[i] is its
// curr_match_lms_observed_in_cand (indexed by cur_keyfrm's keypoints).  Each candidate's correspondences are the
// sim3_solver constructor's (solve/sim3_solver.cc:46-115): camera-frame points of both keyframes and the float
// chi_sq_2D * level_sigma_sq_[octave] of each undistorted keypoint (level_sigma_sq_ read as the bit-identical square of
// scale_factors_, and get_index_in_keyframe as a lookup in get_observations(), so the header needs no other members).  The 3-point samples are drawn with the reference's
// util::create_random_array, only for candidates that run.  cam: undistort_keypoints' convention (camera_of() for a
// perspective camera, the fisheye camera's own fx_ .. cy_); fix_scale: setup_type_ != Monocular (system.cc:140).
// Result i stands in for sim3_solver i after find_via_ransac(num_iter): solution_is_valid(), get_best_rotation_12(),
// get_best_translation_12(), get_best_scale_12().
struct sim3_candidate_result {
    bool valid = false;
    PLPSLAM::Mat33_t rot_12;
    PLPSLAM::Vec3_t trans_12;
    float scale_12 = 0.0f;
};

inline std::vector<sim3_candidate_result> sim3_ransac_candidates(PLPSLAM::data::keyframe *cur_keyfrm,
                                                                 const std::vector<PLPSLAM::data::keyframe *> &candidates,
                                                                 const std::vector<std::vector<PLPSLAM::data::landmark *>> &matched_lms,
                                                                 const std::vector<bool> &run, bool fix_scale,
                                                                 const plp_camera &cam, unsigned num_iter = 200,
                                                                 unsigned min_num_inliers = 20) {
    const size_t K = candidates.size();
    if (matched_lms.size() != K || run.size() != K)
        throw std::invalid_argument("plpslam_b200::sim3_ransac_candidates: candidates, matched_lms and run differ in size");
    constexpr float chi_sq_2D = 9.21034;  // sim3_solver.cc:67
    const auto keyfrm_1_lms = cur_keyfrm->get_landmarks();
    const PLPSLAM::Mat33_t rot_1w = cur_keyfrm->get_rotation();
    const PLPSLAM::Vec3_t trans_1w = cur_keyfrm->get_translation();
    std::vector<int32_t> off(K + 1, 0), samples;
    std::vector<double> pts_1, pts_2;
    std::vector<float> chi_sq_1, chi_sq_2;
    for (size_t k = 0; k < K; ++k) {
        unsigned n = 0;
        if (run[k]) {
            auto *keyfrm_2 = candidates[k];
            const PLPSLAM::Mat33_t rot_2w = keyfrm_2->get_rotation();
            const PLPSLAM::Vec3_t trans_2w = keyfrm_2->get_translation();
            for (unsigned idx1 = 0; idx1 < keyfrm_1_lms.size(); ++idx1) {  // :70-115
                auto *lm_2 = matched_lms[k].at(idx1);
                auto *lm_1 = keyfrm_1_lms.at(idx1);
                if (!lm_1 || !lm_2) continue;
                if (lm_1->will_be_erased() || lm_2->will_be_erased()) continue;
                // get_index_in_keyframe(keyfrm_2) (data/landmark.cc:156-167): the observation index, or -1
                const auto obs_2 = lm_2->get_observations();
                const auto found = obs_2.find(keyfrm_2);
                if (found == obs_2.end()) continue;
                const auto &keypt_1 = cur_keyfrm->undist_keypts_.at(idx1);
                const auto &keypt_2 = keyfrm_2->undist_keypts_.at(found->second);
                // level_sigma_sq_[octave] == scale_factors_[octave]^2 in float: calc_level_sigma_sq squares the same
                // float recurrence calc_scale_factors stores (feature/orb_params.cc:86-116)
                const float sf_1 = cur_keyfrm->scale_factors_.at(keypt_1.octave);
                const float sf_2 = keyfrm_2->scale_factors_.at(keypt_2.octave);
                chi_sq_1.push_back(chi_sq_2D * (sf_1 * sf_1));
                chi_sq_2.push_back(chi_sq_2D * (sf_2 * sf_2));
                const PLPSLAM::Vec3_t p1 = rot_1w * lm_1->get_pos_in_world(), p2 = rot_2w * lm_2->get_pos_in_world();
                for (int c = 0; c < 3; ++c) pts_1.push_back(p1(c) + trans_1w(c)), pts_2.push_back(p2(c) + trans_2w(c));
                ++n;
            }
        }
        off[k + 1] = off[k] + (int32_t)n;
        for (unsigned it = 0; it < num_iter; ++it) {
            if (n >= 3 && n >= min_num_inliers) {  // :130, :149
                const auto idx = PLPSLAM::util::create_random_array(3, 0, static_cast<int>(n - 1));
                samples.insert(samples.end(), idx.begin(), idx.end());
            } else {
                samples.insert(samples.end(), 3, 0);  // not read: the problem does not run
            }
        }
    }
    const std::vector<plp_camera> cams(K, cam);
    std::vector<int32_t> valid(K), num_inliers(K);
    std::vector<double> rot(K * 9), trans(K * 3);
    std::vector<float> scale(K);
    check(plp_sim3_ransac(thread_ctx(), (int)K, off.data(), cams.data(), pts_1.data(), pts_2.data(), chi_sq_1.data(),
                          chi_sq_2.data(), samples.data(), (int)num_iter, fix_scale ? 1 : 0, (int)min_num_inliers,
                          valid.data(), num_inliers.data(), rot.data(), trans.data(), scale.data()));
    std::vector<sim3_candidate_result> out(K);
    for (size_t k = 0; k < K; ++k) {
        out[k].valid = run[k] && valid[k];
        for (int r = 0; r < 3; ++r) {
            for (int c = 0; c < 3; ++c) out[k].rot_12(r, c) = rot[9 * k + 3 * r + c];
            out[k].trans_12(r) = trans[3 * k + r];
        }
        out[k].scale_12 = scale[k];
    }
    return out;
}

// camera::base::model_type_ == Equirectangular (camera/base.h); a camera type without that member has no such model
template <class Camera>
inline auto is_equirectangular(const Camera *c, int) -> decltype((void)c->model_type_, bool()) {
    return c->model_type_ == std::remove_cv_t<decltype(c->model_type_)>::Equirectangular;
}
template <class Camera>
inline bool is_equirectangular(const Camera *, long) { return false; }

// ---- loop_detector::select_loop_candidate_via_Sim3's Sim3 optimisation (module/loop_detector.cc:394-397) for every
// candidate in one call ----
// run[i]: candidate i reached the optimiser (not will_be_erased(), >= 20 BoW matches, a valid RANSAC Sim3) and
// match_keyframes_mutually has filled matched_lms[i].  sim3s[i] is the candidate's g2o::Sim3(rot_12, trans_12, scale_12)
// built from the RANSAC result (scale widened from float); on return it is the optimised Sim3 -- or unchanged where the
// reference returns 0 before writing it.  Each candidate's matches are transform_optimizer::optimize's
// (optimize/transform_optimizer.cc:91-126): idx1 in order, skipping null and will_be_erased() landmarks and landmarks
// that keyframe 2 does not observe (get_index_in_keyframe as a lookup in get_observations()), with both keyframes'
// undist_keypts_ and inv_level_sigma_sq_.  Outliers are set to nullptr in matched_lms[i], as the reference does.
// cam: the camera of both keyframes (camera_of() for a perspective camera, the fisheye camera's own fx_ .. cy_);
// fix_scale: fix_scale_in_Sim3_estimation_.  Returns num_optimized_inliers per candidate (0 where run[i] is false).
// Throws on size mismatches, on keyframes with different cameras, and on equirectangular keyframes (not supported).
struct sim3_estimate {
    PLPSLAM::Mat33_t rot_12;
    PLPSLAM::Vec3_t trans_12;
    double scale_12 = 1.0;
};

inline std::vector<unsigned> sim3_optimize_candidates(PLPSLAM::data::keyframe *cur_keyfrm,
                                                      const std::vector<PLPSLAM::data::keyframe *> &candidates,
                                                      std::vector<std::vector<PLPSLAM::data::landmark *>> &matched_lms,
                                                      std::vector<sim3_estimate> &sim3s, const std::vector<bool> &run,
                                                      bool fix_scale, const plp_camera &cam, float chi_sq = 10,
                                                      unsigned num_iter = 10) {
    const size_t K = candidates.size();
    if (matched_lms.size() != K || sim3s.size() != K || run.size() != K)
        throw std::invalid_argument("plpslam_b200::sim3_optimize_candidates: candidates, matched_lms, sim3s and run differ in size");
    if (is_equirectangular(cur_keyfrm->camera_, 0))
        throw std::invalid_argument("plpslam_b200::sim3_optimize_candidates: equirectangular keyframes are not supported");
    const auto keyfrm_1_lms = cur_keyfrm->get_landmarks();
    const PLPSLAM::Mat33_t rot_1w = cur_keyfrm->get_rotation();
    const PLPSLAM::Vec3_t trans_1w = cur_keyfrm->get_translation();
    std::vector<size_t> cand;  // problem -> candidate
    std::vector<std::vector<unsigned>> idx1s;  // problem -> idx1 of each valid match
    std::vector<int32_t> off(1, 0);
    std::vector<plp_camera> cams;
    std::vector<double> r1, t1, r2, t2, r12, t12, s12, pos_1, pos_2;
    std::vector<float> obs_1, obs_2, w_1, w_2;
    for (size_t k = 0; k < K; ++k) {
        if (!run[k]) continue;
        auto *keyfrm_2 = candidates[k];
        if (keyfrm_2->camera_ != cur_keyfrm->camera_)
            throw std::invalid_argument("plpslam_b200::sim3_optimize_candidates: the keyframes' cameras differ");
        const PLPSLAM::Mat33_t rot_2w = keyfrm_2->get_rotation();
        const PLPSLAM::Vec3_t trans_2w = keyfrm_2->get_translation();
        for (int r = 0; r < 3; ++r) {
            for (int c = 0; c < 3; ++c) {
                r1.push_back(rot_1w(r, c));
                r2.push_back(rot_2w(r, c));
                r12.push_back(sim3s[k].rot_12(r, c));
            }
            t1.push_back(trans_1w(r));
            t2.push_back(trans_2w(r));
            t12.push_back(sim3s[k].trans_12(r));
        }
        s12.push_back(sim3s[k].scale_12);
        cams.push_back(cam);
        std::vector<unsigned> idx;
        for (unsigned idx1 = 0; idx1 < matched_lms[k].size(); ++idx1) {  // :91-126
            auto *lm_2 = matched_lms[k][idx1];
            if (!lm_2) continue;
            auto *lm_1 = keyfrm_1_lms.at(idx1);
            if (!lm_1 || !lm_2) continue;
            if (lm_1->will_be_erased() || lm_2->will_be_erased()) continue;
            // get_index_in_keyframe(keyfrm_2) (data/landmark.cc:156-167): the observation index, or -1
            const auto obs = lm_2->get_observations();
            const auto found = obs.find(keyfrm_2);
            if (found == obs.end()) continue;
            const auto &kp_1 = cur_keyfrm->undist_keypts_.at(idx1);
            const auto &kp_2 = keyfrm_2->undist_keypts_.at(found->second);
            const PLPSLAM::Vec3_t p1 = lm_1->get_pos_in_world(), p2 = lm_2->get_pos_in_world();
            for (int c = 0; c < 3; ++c) pos_1.push_back(p1(c)), pos_2.push_back(p2(c));
            obs_1.push_back(kp_1.pt.x), obs_1.push_back(kp_1.pt.y);
            obs_2.push_back(kp_2.pt.x), obs_2.push_back(kp_2.pt.y);
            w_1.push_back(cur_keyfrm->inv_level_sigma_sq_.at(kp_1.octave));
            w_2.push_back(keyfrm_2->inv_level_sigma_sq_.at(kp_2.octave));
            idx.push_back(idx1);
        }
        off.push_back(off.back() + (int32_t)idx.size());
        cand.push_back(k);
        idx1s.push_back(std::move(idx));
    }
    const size_t P = cand.size(), N = (size_t)off.back();
    std::vector<int32_t> num_inliers(P + 1);
    std::vector<double> rot(P * 9 + 1), trans(P * 3 + 1), scale(P + 1);
    std::vector<uint8_t> inlier(N + 1);
    check(plp_sim3_optimize(thread_ctx(), (int)P, off.data(), cams.data(), r1.data(), t1.data(), r2.data(), t2.data(),
                            r12.data(), t12.data(), s12.data(), pos_1.data(), pos_2.data(), obs_1.data(), obs_2.data(),
                            w_1.data(), w_2.data(), chi_sq, (int)num_iter, fix_scale ? 1 : 0, num_inliers.data(), rot.data(),
                            trans.data(), scale.data(), inlier.data()));
    std::vector<unsigned> out(K, 0);
    for (size_t p = 0; p < P; ++p) {
        const size_t k = cand[p];
        for (size_t i = 0; i < idx1s[p].size(); ++i)
            if (!inlier[off[p] + i]) matched_lms[k][idx1s[p][i]] = nullptr;
        for (int r = 0; r < 3; ++r) {
            for (int c = 0; c < 3; ++c) sim3s[k].rot_12(r, c) = rot[9 * p + 3 * r + c];
            sim3s[k].trans_12(r) = trans[3 * p + r];
        }
        sim3s[k].scale_12 = scale[p];
        out[k] = (unsigned)num_inliers[p];
    }
    return out;
}

// ---- match::fuse::replace_duplication (match/fuse.cc:153-300) over the loop of mapping_module.cc:711-714 / :749 ---
// One batched search for (targets x landmarks); the effects are applied in the reference's order.  landmark::replace
// recomputes the surviving landmark's descriptor (data/landmark.cc:429), so a landmark whose descriptor changed is
// searched again against the remaining targets before its next use -- results are identical to the sequential loop
// (tests/test_fuse_oracle.py::test_adapter_protocol_equals_sequential_reference checks the protocol on a map model).
// NOTE: needs read access to landmark::max_valid_dist_ (predict_scale_level's numerator, landmark.cc:346); add
// `friend struct plpslam_b200::landmark_access;` to data/landmark.h (no public signature changes).
struct landmark_access {
    static float max_valid_dist_raw(const PLPSLAM::data::landmark *lm) { return lm->max_valid_dist_; }
};

struct fuse_batch {
    std::vector<double> pos, normal;
    std::vector<float> min_d, max_d, max_raw;
    std::vector<uint8_t> desc, valid;
    void gather(const std::vector<PLPSLAM::data::landmark *> &lms, const std::vector<size_t> &which) {
        const size_t m = which.size();
        pos.resize(3 * m), normal.resize(3 * m), min_d.resize(m), max_d.resize(m), max_raw.resize(m);
        desc.resize(32 * m), valid.resize(m);
        for (size_t q = 0; q < m; ++q) {
            auto *lm = lms[which[q]];
            valid[q] = lm && !lm->will_be_erased();
            if (!valid[q]) continue;
            const PLPSLAM::Vec3_t p = lm->get_pos_in_world(), nrm = lm->get_obs_mean_normal();
            for (int k = 0; k < 3; ++k) pos[3 * q + k] = p(k), normal[3 * q + k] = nrm(k);
            min_d[q] = lm->get_min_valid_distance();
            max_d[q] = lm->get_max_valid_distance();
            max_raw[q] = landmark_access::max_valid_dist_raw(lm);
            const cv::Mat d = lm->get_descriptor();
            std::copy(d.data, d.data + 32, desc.begin() + 32 * q);
        }
    }
    plp_fuse_landmarks view() const {
        return plp_fuse_landmarks{(int32_t)valid.size(), pos.data(), normal.data(), min_d.data(), max_d.data(),
                                  max_raw.data(), desc.data(), valid.data()};
    }
};

struct fuse_target {
    std::vector<float> x, y;
    std::vector<int32_t> oct;
    plp_fuse_target_points t;
    explicit fuse_target(PLPSLAM::data::keyframe *kf) {
        const int n = kf->num_keypts_;
        x.resize(n), y.resize(n), oct.resize(n);
        for (int i = 0; i < n; ++i) x[i] = kf->undist_keypts_[i].pt.x, y[i] = kf->undist_keypts_[i].pt.y, oct[i] = kf->undist_keypts_[i].octave;
        t.pts = plp_frame_points{n, x.data(), y.data(), oct.data(), nullptr, kf->stereo_x_right_.data(), kf->descriptors_.data, nullptr};
        const PLPSLAM::Mat33_t R = kf->get_rotation();
        const PLPSLAM::Vec3_t tr = kf->get_translation(), c = kf->get_cam_center();
        for (int r = 0; r < 3; ++r) {
            for (int k = 0; k < 3; ++k) t.rot_cw[3 * r + k] = R(r, k);
            t.trans_cw[r] = tr(r), t.cam_center[r] = c(r);
        }
        t.skip = nullptr;  // is_observed_in_keyframe is re-checked when the effect is applied
    }
};

// fuse.cc:284-318 for one landmark with a search hit
inline void fuse_apply(PLPSLAM::data::keyframe *keyfrm, PLPSLAM::data::landmark *lm, int best_idx) {
    auto *lm_in_keyfrm = keyfrm->get_landmark(best_idx);
    if (lm_in_keyfrm) {
        if (!lm_in_keyfrm->will_be_erased()) {
            if (lm->num_observations() < lm_in_keyfrm->num_observations())
                lm->replace(lm_in_keyfrm);
            else
                lm_in_keyfrm->replace(lm);
        }
    } else {
        lm->add_observation(keyfrm, best_idx);
        keyfrm->add_landmark(lm, best_idx);
    }
}

// body of `for (fuse_tgt_keyfrm : fuse_tgt_keyfrms) matcher.replace_duplication(fuse_tgt_keyfrm, cur_landmarks)` and of
// the single-target call at mapping_module.cc:749 (targets.size() == 1); returns num_fused per target
inline std::vector<unsigned> replace_duplication(const std::vector<PLPSLAM::data::keyframe *> &targets,
                                                 const std::vector<PLPSLAM::data::landmark *> &lms, float margin = 3.0f) {
    const size_t K = targets.size(), M = lms.size();
    std::vector<unsigned> num_fused(K, 0);
    if (!K || !M) return num_fused;
    auto *kf0 = targets[0];
    const plp_grid g = grid_of(kf0->camera_);
    const plp_camera cam = camera_of(kf0->camera_);
    std::vector<fuse_target> tg;
    tg.reserve(K);
    for (auto *kf : targets) tg.emplace_back(kf);
    auto search = [&](size_t first_target, const std::vector<size_t> &which, std::vector<int32_t> &best) {
        fuse_batch fb;
        fb.gather(lms, which);
        std::vector<plp_fuse_target_points> tv;
        for (size_t k = first_target; k < K; ++k) tv.push_back(tg[k].t);
        const plp_fuse_landmarks lv = fb.view();
        best.resize(tv.size() * which.size());
        check(plp_fuse_search_points(thread_ctx(), tv.data(), (int)tv.size(), &g, &cam, kf0->scale_factors_.data(),
                                     kf0->inv_level_sigma_sq_.data(), (int)kf0->num_scale_levels_, kf0->log_scale_factor_,
                                     &lv, margin, PLP_FUSE_REPLACE, best.data(), nullptr));
    };
    std::vector<size_t> all(M);
    for (size_t i = 0; i < M; ++i) all[i] = i;
    std::vector<int32_t> best;
    search(0, all, best);  // best[k * M + i]
    std::vector<std::vector<uint8_t>> desc_seen(M);
    for (size_t i = 0; i < M; ++i)
        if (lms[i]) { const cv::Mat d = lms[i]->get_descriptor(); desc_seen[i].assign(d.data, d.data + 32); }
    for (size_t k = 0; k < K; ++k) {
        for (size_t i = 0; i < M; ++i) {
            auto *lm = lms[i];
            if (!lm || lm->will_be_erased() || lm->is_observed_in_keyframe(targets[k])) continue;  // fuse.cc:163-174
            const cv::Mat d = lm->get_descriptor();
            if (!std::equal(d.data, d.data + 32, desc_seen[i].begin())) {  // recomputed by an earlier replace()
                std::vector<int32_t> again;
                search(k, {i}, again);
                for (size_t kk = k; kk < K; ++kk) best[kk * M + i] = again[kk - k];
                desc_seen[i].assign(d.data, d.data + 32);
            }
            const int b = best[k * M + i];
            if (b < 0) continue;
            fuse_apply(targets[k], lm, b);
            ++num_fused[k];
        }
    }
    return num_fused;
}

// ---- Planar_Mapping_module::estimate_plane_sequential_RANSAC / update_plane_via_RANSAC (planar_mapping_module.cc:412-733)
// `update` = false: estimate (POINTS_PER_RANSAC samples, ratio gate, early exit); true: update (0.8 n samples).
inline bool plane_ransac(PLPSLAM::data::Plane *plane, bool update, unsigned iterations_count, unsigned points_per_ransac,
                         double planar_distance_thresh, double final_error_thresh, double inliers_ratio_thr) {
    std::vector<PLPSLAM::data::landmark *> lms = plane->get_landmarks();
    const int n = (int)lms.size();
    if (n == 0) return false;                                   // :423-426 / :597-600
    if (n < (int)points_per_ransac) {                           // :428-436 / :602-606
        if (update) plane->set_invalid();
        return false;
    }
    std::vector<double> pos((size_t)n * 3);
    std::vector<uint8_t> valid(n), inlier(n);
    for (int j = 0; j < n; ++j) {
        valid[j] = !lms[j]->will_be_erased();
        const PLPSLAM::Vec3_t p = lms[j]->get_pos_in_world();
        for (int k = 0; k < 3; ++k) pos[3 * (size_t)j + k] = p(k);
    }
    // the reference's own index draws (:444-457 / :613-632): uniform indices, erased landmarks rejected
    const int sample_size = update ? (int)std::ceil(n * 0.8) : (int)points_per_ransac;
    std::function<int()> rnd = std::bind(std::uniform_int_distribution<>(0, n - 1), std::mt19937(std::random_device()()));
    std::vector<int32_t> samples((size_t)iterations_count * sample_size);
    for (auto &s : samples) {
        int index = rnd();
        while (!valid[index] || (update && !lms[index]->get_Owning_Plane())) index = rnd();  // :623-631
        s = index;
    }
    double eq[4], best_error = plane->get_best_error();
    plane->get_equation(eq[0], eq[1], eq[2], eq[3]);
    const plp_plane_ransac_cfg cfg{update ? 1 : 0, (int32_t)points_per_ransac, planar_distance_thresh, final_error_thresh,
                                   inliers_ratio_thr, best_error};
    int32_t status = 0;
    check(plp_plane_ransac(thread_ctx(), pos.data(), valid.data(), n, samples.data(), (int)iterations_count, sample_size, &cfg,
                           eq, &best_error, inlier.data(), &status));
    plane->set_equation(eq[0], eq[1], eq[2], eq[3]);  // the Plane is mutated every iteration, also on failure (:465-467)
    plane->set_best_error(best_error);
    if (status == 2) plane->set_invalid();                      // :713-717
    if (status == 0 && update) plane->set_need_refinement();    // :691-695
    if (status != 1) return false;
    std::vector<PLPSLAM::data::landmark *> kept;
    for (int j = 0; j < n; ++j)
        if (inlier[j]) kept.push_back(lms[j]);
    plane->remove_landmarks_ownership();                        // :586-588 / :719-721
    plane->set_landmarks(kept);
    plane->set_landmarks_ownership();
    return true;
}

// ---- frame::compute_bow / keyframe::compute_bow (data/frame.cc:785-795) ----------------------------------------
// One device vocabulary per process (loaded from the same file as bow_vocab_->loadFromBinaryFile, system.cc:82).
#ifdef USE_DBOW2
inline void compute_bow(plp_bow_vocab *vocab, const cv::Mat &descriptors, DBoW2::BowVector &bow_vec,
                        DBoW2::FeatureVector &bow_feat_vec, int levelsup = 4) {
    const int n = descriptors.rows;
    std::vector<int32_t> word(n), node(n);
    std::vector<float> weight(n);
    check(plp_bow_transform(vocab, descriptors.data, n, levelsup, word.data(), node.data(), weight.data()));
    bow_vec.clear();
    bow_feat_vec.clear();
    for (int i = 0; i < n; ++i) {  // TemplatedVocabulary::transform(features, v, fv, levelsup), TF_IDF branch
        if (!(weight[i] > 0)) continue;
        bow_vec.addWeight((DBoW2::WordId)word[i], (DBoW2::WordValue)weight[i]);
        bow_feat_vec.addFeature((DBoW2::NodeId)node[i], (unsigned)i);
    }
    bow_vec.normalize(DBoW2::L1);  // L1_NORM scoring: mustNormalize
}

// ---- match::bow_tree::match_frame_and_keyframe (match/bow_tree.cc:41-165) for a batch of candidate keyframes -----
struct bow_side_view {
    std::vector<uint32_t> ids, idx;
    std::vector<int32_t> off;
    std::vector<float> angle;
    std::vector<uint8_t> valid;
    plp_bow_side s;
    template <class KP>
    void fill(const DBoW2::FeatureVector &fv, const KP &keypts, const cv::Mat &desc, bool with_valid) {
        off.push_back(0);
        for (const auto &kv : fv) {
            ids.push_back(kv.first);
            idx.insert(idx.end(), kv.second.begin(), kv.second.end());
            off.push_back((int32_t)idx.size());
        }
        angle.resize(keypts.size());
        for (size_t i = 0; i < keypts.size(); ++i) angle[i] = keypts[i].angle;
        s = plp_bow_side{(int32_t)keypts.size(), desc.data, angle.data(), with_valid ? valid.data() : nullptr,
                         plp_bow_feature_vector{(int32_t)ids.size(), ids.data(), off.data(), idx.data()}};
    }
};

inline std::vector<unsigned> match_frame_and_keyframes(const std::vector<PLPSLAM::data::keyframe *> &keyfrms,
                                                       PLPSLAM::data::frame &frm, float lowe_ratio, bool check_orientation,
                                                       std::vector<std::vector<PLPSLAM::data::landmark *>> &matched_lms_in_frm) {
    const size_t K = keyfrms.size();
    bow_side_view fs;
    fs.fill(frm.bow_feat_vec_, frm.keypts_, frm.descriptors_, false);
    std::vector<bow_side_view> ks(K);
    std::vector<std::vector<PLPSLAM::data::landmark *>> kf_lms(K);
    std::vector<std::vector<int32_t>> m12(K, std::vector<int32_t>(frm.num_keypts_));
    std::vector<plp_bow_pair> pairs(K);
    for (size_t k = 0; k < K; ++k) {
        kf_lms[k] = keyfrms[k]->get_landmarks();
        ks[k].valid.resize(kf_lms[k].size());
        for (size_t i = 0; i < kf_lms[k].size(); ++i) ks[k].valid[i] = kf_lms[k][i] && !kf_lms[k][i]->will_be_erased();
        ks[k].fill(keyfrms[k]->bow_feat_vec_, keyfrms[k]->keypts_, keyfrms[k]->descriptors_, true);
        pairs[k] = plp_bow_pair{&ks[k].s, &fs.s, nullptr, m12[k].data(), 0};
    }
    check(plp_match_bow_tree(thread_ctx(), pairs.data(), (int)K, lowe_ratio, check_orientation));
    std::vector<unsigned> num(K);
    matched_lms_in_frm.assign(K, std::vector<PLPSLAM::data::landmark *>(frm.num_keypts_, nullptr));
    for (size_t k = 0; k < K; ++k) {
        for (unsigned i = 0; i < frm.num_keypts_; ++i)
            if (m12[k][i] >= 0) matched_lms_in_frm[k][i] = kf_lms[k][m12[k][i]];
        num[k] = pairs[k].num_matches;
    }
    return num;
}
#endif  // USE_DBOW2


// ---- match::projection::match_current_and_last_frames (match/projection.cc:214-358) ----------------------------------
// The per-frame call of frame_tracker::motion_based_track (module/frame_tracker.cc:63-71).  The reprojection of the last
// frame's landmarks, the window query, the claimed-keypoint rule and the orientation histogram all run on the device;
// the adapter flattens the last frame's (landmark, keypoint) pairs and re-applies the pointer writes.
inline unsigned match_current_and_last_frames(PLPSLAM::data::frame &curr_frm, const PLPSLAM::data::frame &last_frm, float margin,
                                              bool check_orientation = true) {
    const int n = curr_frm.num_keypts_;
    std::vector<float> x(n), y(n), ang(n);
    std::vector<int32_t> oct(n), matched(n);
    std::vector<uint8_t> claimed(n);
    for (int i = 0; i < n; ++i) {
        x[i] = curr_frm.undist_keypts_[i].pt.x;
        y[i] = curr_frm.undist_keypts_[i].pt.y;
        oct[i] = curr_frm.undist_keypts_[i].octave;
        ang[i] = curr_frm.undist_keypts_[i].angle;
        claimed[i] = curr_frm.landmarks_[i] && curr_frm.landmarks_[i]->has_observation();  // :303-306
    }
    std::vector<PLPSLAM::data::landmark *> lms;
    std::vector<double> pos;
    std::vector<int32_t> l_oct;
    std::vector<float> l_ang;
    std::vector<uint8_t> l_desc;
    for (unsigned idx = 0; idx < last_frm.num_keypts_; ++idx) {  // :240-253
        auto *lm = last_frm.landmarks_[idx];
        if (!lm || last_frm.outlier_flags_[idx]) continue;
        const PLPSLAM::Vec3_t X = lm->get_pos_in_world();
        lms.push_back(lm);
        pos.insert(pos.end(), {X(0), X(1), X(2)});
        l_oct.push_back(last_frm.keypts_[idx].octave);           // :268
        l_ang.push_back(last_frm.undist_keypts_[idx].angle);     // :329
        const cv::Mat d = lm->get_descriptor();
        l_desc.insert(l_desc.end(), d.data, d.data + 32);
    }
    double Tc[16], Tl[16];
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) {
            Tc[r * 4 + c] = curr_frm.cam_pose_cw_(r, c);
            Tl[r * 4 + c] = last_frm.cam_pose_cw_(r, c);
        }
    const plp_frame_points fp{n, x.data(), y.data(), oct.data(), ang.data(), curr_frm.stereo_x_right_.data(),
                              curr_frm.descriptors_.data, claimed.data()};
    const plp_last_frame_points lp{(int32_t)lms.size(), pos.data(), l_oct.data(), l_ang.data(), l_desc.data(), nullptr};
    const plp_grid grid = grid_of(curr_frm.camera_);
    const plp_camera cam = camera_of(curr_frm.camera_);
    uint32_t num = 0;
    check(plp_match_current_and_last_frames(thread_ctx(), &fp, &grid, curr_frm.scale_factors_.data(),
                                            (int)curr_frm.scale_factors_.size(), &cam, Tc, Tl, &lp, margin, check_orientation,
                                            matched.data(), &num));
    for (int i = 0; i < n; ++i)  // curr_frm.landmarks_.at(best_idx) = lm (:325), minus the orientation rejects (:337-354)
        if (matched[i] >= 0) curr_frm.landmarks_[i] = lms[matched[i]];
    return num;
}

// keylines of a frame as the C ABI sees them; ratio_level reproduces the reference reading a POINT octave at a line index
// (match/projection.cc:170,175) so that the behaviour is unchanged
struct frame_lines_view {
    std::vector<float> sx, sy, ex, ey;
    std::vector<int32_t> oct, ratio_level;
    std::vector<uint8_t> claimed;
    plp_frame_lines v;
    explicit frame_lines_view(PLPSLAM::data::frame &frm) {
        const int n = frm._num_keylines;
        sx.resize(n), sy.resize(n), ex.resize(n), ey.resize(n), oct.resize(n), ratio_level.resize(n), claimed.resize(n);
        for (int i = 0; i < n; ++i) {
            const auto &kl = frm._keylsd[i];
            sx[i] = kl.getStartPoint().x;
            sy[i] = kl.getStartPoint().y;
            ex[i] = kl.getEndPoint().x;
            ey[i] = kl.getEndPoint().y;
            oct[i] = kl.octave;
            ratio_level[i] = i < (int)frm.undist_keypts_.size() ? frm.undist_keypts_[i].octave : kl.octave;
            claimed[i] = frm._landmarks_line[i] && frm._landmarks_line[i]->has_observation();
        }
        v = plp_frame_lines{n, sx.data(), sy.data(), ex.data(), ey.data(), oct.data(), ratio_level.data(), nullptr, nullptr,
                            frm._lbd_descr.data, claimed.data()};
    }
};

// ---- match::projection::match_current_and_last_frames_line (match/projection.cc:361-527) --------------------------------
inline unsigned match_current_and_last_frames_line(PLPSLAM::data::frame &curr_frm, const PLPSLAM::data::frame &last_frm,
                                                   float margin) {
    frame_lines_view cv_(curr_frm);
    std::vector<PLPSLAM::data::Line *> lms;
    std::vector<double> pos;
    std::vector<int32_t> l_oct;
    std::vector<uint8_t> l_desc;
    for (unsigned idx = 0; idx < last_frm._num_keylines; ++idx) {  // :392-405
        auto *ll = last_frm._landmarks_line[idx];
        if (!ll || last_frm._outlier_flags_line[idx]) continue;
        const PLPSLAM::Vec6_t X = ll->get_pos_in_world();
        lms.push_back(ll);
        for (int k = 0; k < 6; ++k) pos.push_back(X(k));
        l_oct.push_back(last_frm._keylsd[idx].octave);
        const cv::Mat d = ll->get_descriptor();
        l_desc.insert(l_desc.end(), d.data, d.data + 32);
    }
    double Tc[16], Tl[16];
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) {
            Tc[r * 4 + c] = curr_frm.cam_pose_cw_(r, c);
            Tl[r * 4 + c] = last_frm.cam_pose_cw_(r, c);
        }
    const plp_last_frame_lines lp{(int32_t)lms.size(), pos.data(), l_oct.data(), l_desc.data(), nullptr};
    const plp_camera cam = camera_of(curr_frm.camera_);
    std::vector<int32_t> matched(curr_frm._num_keylines);
    uint32_t num = 0;
    check(plp_match_current_and_last_frames_line(thread_ctx(), &cv_.v, curr_frm._scale_factors_lsd.data(),
                                                 (int)curr_frm._scale_factors_lsd.size(), &cam, Tc, Tl, &lp, margin,
                                                 matched.data(), &num));
    for (unsigned i = 0; i < curr_frm._num_keylines; ++i)
        if (matched[i] >= 0) curr_frm._landmarks_line[i] = lms[matched[i]];
    return num;
}

// ---- match::projection::match_frame_and_landmarks_line (match/projection.cc:124-212) -------------------------------------
// called beside the point matcher in tracking_module::search_local_landmarks_line (tracking_module.cc:986-1060)
inline unsigned match_frame_and_landmarks_line(PLPSLAM::data::frame &frm, const std::vector<PLPSLAM::data::Line *> &local_lines,
                                               float margin, float lowe_ratio) {
    const int m = (int)local_lines.size();
    if (m == 0) return 0;  // :130-133
    frame_lines_view fv(frm);
    std::vector<float> spx(m), spy(m), epx(m), epy(m);
    std::vector<int32_t> lvl(m), best(m);
    std::vector<uint8_t> valid(m), qdesc((size_t)m * 32);
    for (int q = 0; q < m; ++q) {
        auto *ll = local_lines[q];
        valid[q] = ll->_is_observable_in_tracking && !ll->will_be_erased();
        spx[q] = ll->_reproj_in_tracking_sp(0);
        spy[q] = ll->_reproj_in_tracking_sp(1);
        epx[q] = ll->_reproj_in_tracking_ep(0);
        epy[q] = ll->_reproj_in_tracking_ep(1);
        lvl[q] = ll->_scale_level_in_tracking;
        const cv::Mat d = ll->get_descriptor();
        std::copy(d.data, d.data + 32, qdesc.begin() + (size_t)q * 32);
    }
    const plp_line_queries lq{m, spx.data(), spy.data(), epx.data(), epy.data(), lvl.data(), qdesc.data(), valid.data()};
    uint32_t num = 0;
    check(plp_match_frame_and_landmarks_line(thread_ctx(), &fv.v, frm._scale_factors_lsd.data(), (int)frm._scale_factors_lsd.size(),
                                             &lq, margin, lowe_ratio, best.data(), &num));
    for (int q = 0; q < m; ++q)
        if (best[q] >= 0) frm._landmarks_line[best[q]] = local_lines[q];
    return num;
}

// ---- optimize::local_bundle_adjuster[_extended_line|_extended_plane]::optimize ------------------------------------------
// (optimize/local_bundle_adjuster.cc:62-410, local_bundle_adjuster_extended_line.cc:69-674,
//  local_bundle_adjuster_extended_plane.cc:70-487): the WHOLE method body.  [1] gather local / fixed keyframes and local
// landmarks by walking the covisibility graph and the observation tables (:72-158) -- ordered maps by id instead of the
// reference's unordered_map, which only fixes the summation order; [2-6] the solve on the GPU (plp_local_ba: two LM runs
// with the outlier round in between, force-stop polled between chunks of LM tries); [7-8] outlier observations erased
// and the estimates written back under the map mutex (:342-409), lines re-trimmed on their reference keyframe
// (local_bundle_adjuster_extended_line.cc:642-672, 676-787).  Neither the number of local nor of fixed keyframes is
// bounded: up to 32 NON-FIXED keyframes the reduced camera system is solved in shared memory, beyond that dense in HBM.
struct local_ba_options {
    bool with_lines = false;   // local_bundle_adjuster_extended_line
    bool with_planes = false;  // local_bundle_adjuster_extended_plane: unary point-to-plane edges (:309-345)
    int num_first_iter = 5, num_second_iter = 10;
};

inline void local_bundle_adjust(PLPSLAM::data::keyframe *curr_keyfrm, bool *const force_stop_flag, const local_ba_options &opt) {
    using namespace PLPSLAM;
    // ---- [1] aggregate (local_bundle_adjuster.cc:72-158)
    std::map<unsigned, data::keyframe *> local_keyfrms, fixed_keyfrms;
    local_keyfrms[curr_keyfrm->id_] = curr_keyfrm;
    for (auto *kf : curr_keyfrm->graph_node_->get_covisibilities())
        if (kf && !kf->will_be_erased()) local_keyfrms[kf->id_] = kf;
    std::map<unsigned, data::landmark *> local_lms;
    std::map<unsigned, data::Line *> local_lines;
    for (auto &ikf : local_keyfrms) {
        for (auto *lm : ikf.second->get_landmarks())
            if (lm && !lm->will_be_erased()) local_lms.emplace(lm->id_, lm);
        if (opt.with_lines)
            for (auto *ll : ikf.second->get_landmarks_line())
                if (ll && !ll->will_be_erased()) local_lines.emplace(ll->_id, ll);
    }
    auto add_fixed = [&](data::keyframe *kf) {
        if (kf && !kf->will_be_erased() && !local_keyfrms.count(kf->id_)) fixed_keyfrms.emplace(kf->id_, kf);
    };
    for (auto &ilm : local_lms)
        for (auto &obs : ilm.second->get_observations()) add_fixed(obs.first);
    for (auto &ill : local_lines)
        for (auto &obs : ill.second->get_observations()) add_fixed(obs.first);
    // ---- [3-4] flatten: keyframes (local first, then fixed), landmarks, one edge per observation grouped by landmark
    std::vector<data::keyframe *> kfs;
    std::map<data::keyframe *, int> kf_index;
    std::vector<double> kf_pose;
    std::vector<uint8_t> kf_fixed;
    auto push_kf = [&](data::keyframe *kf, bool fixed) {
        kf_index[kf] = (int)kfs.size();
        kfs.push_back(kf);
        const Mat44_t T = kf->get_cam_pose();
        for (int r = 0; r < 4; ++r)
            for (int c = 0; c < 4; ++c) kf_pose.push_back(T(r, c));
        kf_fixed.push_back(fixed ? 1 : 0);
    };
    for (auto &ikf : local_keyfrms) push_kf(ikf.second, ikf.second->id_ == 0);  // :197-202
    for (auto &ikf : fixed_keyfrms) push_kf(ikf.second, true);                  // :205-213
    std::vector<data::landmark *> lms;
    std::vector<double> pt_pos, plane_fn;
    std::vector<int32_t> pe_kf, pe_lm, plane_lm;
    std::vector<float> pe_obs, pe_info;
    std::vector<std::pair<data::keyframe *, data::landmark *>> pe_owner;
    for (auto &ilm : local_lms) {  // :226-272
        auto *lm = ilm.second;
        const int li = (int)lms.size();
        lms.push_back(lm);
        const Vec3_t X = lm->get_pos_in_world();
        pt_pos.insert(pt_pos.end(), {X(0), X(1), X(2)});
        for (auto &obs : lm->get_observations()) {
            auto *kf = obs.first;
            if (!kf || kf->will_be_erased()) continue;
            const auto &kp = kf->undist_keypts_.at(obs.second);
            pe_kf.push_back(kf_index.at(kf));
            pe_lm.push_back(li);
            pe_obs.insert(pe_obs.end(), {kp.pt.x, kp.pt.y, kf->stereo_x_right_.at(obs.second)});
            pe_info.push_back(kf->inv_level_sigma_sq_.at(kp.octave));
            pe_owner.emplace_back(kf, lm);
        }
        if (opt.with_planes) {  // local_bundle_adjuster_extended_plane.cc:309-345: constants, not vertices
            auto *pl = lm->get_Owning_Plane();
            if (pl && pl->is_valid() && !pl->need_refinement()) {
                const Vec3_t nrm = pl->get_normal();
                plane_lm.push_back(li);
                plane_fn.insert(plane_fn.end(), {nrm(0), nrm(1), nrm(2), pl->get_offset()});
            }
        }
    }
    std::vector<data::Line *> lines;
    std::vector<double> ln_plucker;
    std::vector<int32_t> le_kf, le_lm;
    std::vector<float> le_obs, le_info;
    std::vector<std::pair<data::keyframe *, data::Line *>> le_owner;
    for (auto &ill : local_lines) {  // local_bundle_adjuster_extended_line.cc:365-417
        auto *ll = ill.second;
        const int li = (int)lines.size();
        lines.push_back(ll);
        const Vec6_t L = ll->get_PlueckerCoord();
        for (int k = 0; k < 6; ++k) ln_plucker.push_back(L(k));
        for (auto &obs : ll->get_observations()) {
            auto *kf = obs.first;
            if (!kf || kf->will_be_erased()) continue;
            const auto &kl = kf->_keylsd.at(obs.second);
            le_kf.push_back(kf_index.at(kf));
            le_lm.push_back(li);
            le_obs.insert(le_obs.end(), {kl.getStartPoint().x, kl.getStartPoint().y, kl.getEndPoint().x, kl.getEndPoint().y});
            le_info.push_back(kf->_inv_level_sigma_sq_lsd.at(kl.octave));
            le_owner.emplace_back(kf, ll);
        }
    }
    if (force_stop_flag && *force_stop_flag) return;  // :276-282
    const auto *pc = static_cast<const camera::perspective *>(curr_keyfrm->camera_);
    plp_ba_problem P{};
    P.fx = pc->fx_, P.fy = pc->fy_, P.cx = pc->cx_, P.cy = pc->cy_;
    P.focal_x_baseline = curr_keyfrm->camera_->focal_x_baseline_;
    P.setup_type = (int32_t)curr_keyfrm->camera_->setup_type_;
    P.n_kf = (int32_t)kfs.size(), P.kf_pose_cw = kf_pose.data(), P.kf_fixed = kf_fixed.data();
    P.n_pts = (int32_t)lms.size(), P.pt_pos_w = pt_pos.data();
    P.n_pt_edges = (int32_t)pe_kf.size(), P.pt_edge_kf = pe_kf.data(), P.pt_edge_lm = pe_lm.data();
    P.pt_edge_obs = pe_obs.data(), P.pt_edge_inv_sigma_sq = pe_info.data();
    P.n_lines = (int32_t)lines.size(), P.line_plucker = ln_plucker.data();
    P.n_line_edges = (int32_t)le_kf.size(), P.line_edge_kf = le_kf.data(), P.line_edge_lm = le_lm.data();
    P.line_edge_obs = le_obs.data(), P.line_edge_inv_sigma_sq = le_info.data();
    P.n_plane_edges = (int32_t)plane_lm.size(), P.plane_edge_lm = plane_lm.data(), P.plane_edge_fn = plane_fn.data();
    std::vector<double> out_pose(kf_pose.size()), out_pts(pt_pos.size() + 3), out_lines(ln_plucker.size() + 6);
    std::vector<uint8_t> pt_out(pe_kf.size() + 1), ln_out(le_kf.size() + 1);
    plp_ba_result R{out_pose.data(), out_pts.data(), out_lines.data(), pt_out.data(), ln_out.data(), 0, 0, 0, 0.0};
    const plp_ba_cfg cfg{opt.num_first_iter, opt.num_second_iter, 0};
    // the reference hands g2o a plain bool that the tracking thread writes (mapping_module.cc:159-164)
    check(plp_local_ba(thread_ctx(), &P, &cfg, reinterpret_cast<volatile const uint8_t *>(force_stop_flag), &R));
    // ---- [7-8] write-back under the map mutex (:375-409)
    std::lock_guard<std::mutex> lock(data::map_database::mtx_database_);
    for (size_t e = 0; e < pe_owner.size(); ++e) {
        if (!pt_out[e] || pe_owner[e].second->will_be_erased()) continue;  // :346-372
        pe_owner[e].first->erase_landmark(pe_owner[e].second);
        pe_owner[e].second->erase_observation(pe_owner[e].first);
    }
    for (size_t e = 0; e < le_owner.size(); ++e) {
        if (!ln_out[e] || le_owner[e].second->will_be_erased()) continue;
        le_owner[e].first->erase_landmark_line(le_owner[e].second);
        le_owner[e].second->erase_observation(le_owner[e].first);
    }
    for (auto &ikf : local_keyfrms) {
        const int k = kf_index.at(ikf.second);
        Mat44_t T;
        for (int r = 0; r < 4; ++r)
            for (int c = 0; c < 4; ++c) T(r, c) = out_pose[16 * (size_t)k + r * 4 + c];
        ikf.second->set_cam_pose(T);
    }
    for (size_t l = 0; l < lms.size(); ++l) {
        lms[l]->set_pos_in_world(Vec3_t(out_pts[3 * l], out_pts[3 * l + 1], out_pts[3 * l + 2]));
        lms[l]->update_normal_and_depth();
    }
    for (size_t l = 0; l < lines.size(); ++l) {  // local_bundle_adjuster_extended_line.cc:642-672
        auto *ll = lines[l];
        Vec6_t L;
        for (int k = 0; k < 6; ++k) L(k) = out_lines[6 * l + k];
        ll->set_PlueckerCoord_without_update_endpoints(L);
        auto *ref_kf = ll->get_ref_keyframe();
        const int idx = ll->get_index_in_keyframe(ref_kf);
        bool keep = idx != -1;  // :688-691
        Vec6_t updated;
        if (keep) {
            const auto &kl = ref_kf->_keylsd.at(idx);
            const auto *rc = static_cast<const camera::perspective *>(ref_kf->camera_);
            const Mat44_t T = ref_kf->get_cam_pose();
            double Tm[16], old_ep[6], new_ep[6];
            for (int r = 0; r < 4; ++r)
                for (int c = 0; c < 4; ++c) Tm[r * 4 + c] = T(r, c);
            const Vec6_t old = ll->get_pos_in_world();
            for (int k = 0; k < 6; ++k) old_ep[k] = old(k);
            keep = endpoint_trimming(trimming_camera{rc->fx_, rc->fy_, rc->cx_, rc->cy_}, Tm, &out_lines[6 * l],
                                     kl.getStartPoint().x, kl.getStartPoint().y, kl.getEndPoint().x, kl.getEndPoint().y, old_ep,
                                     ref_kf->compute_median_depth(true), new_ep);
            for (int k = 0; k < 6; ++k) updated(k) = new_ep[k];
        }
        if (keep) {
            ll->set_pos_in_world_without_update_pluecker(updated);
            ll->update_information();
        } else {
            ll->prepare_for_erasing();  // outlier found by trimming
        }
    }
}

}  // namespace plpslam_b200

#endif  // PLPSLAM_B200_WITH_REFERENCE_TYPES
