// oracle/sim3.cc -- solve::sim3_solver (TEST INFRASTRUCTURE ONLY).  Follows
// the reference's src/PLPSLAM/solve/sim3_solver.cc; compute_Sim3, reproject_to_image and the inlier test are restated in
// sim3math.h (see its header).
#include "sim3math.h"

#include <stdint.h>

#include <cstring>
#include <vector>

namespace {

// the constructor's reproject_to_same_image (:117-118)
void reproject_to_same_image(const double *cam, const double *pts, int n, std::vector<double> &reprojected) {
    reprojected.assign(2 * (size_t)n, 0.0);
    for (int i = 0; i < n; ++i) sim3_reproject_same(cam, pts + 3 * (size_t)i, reprojected.data() + 2 * (size_t)i);
}

// count_inliers (:290-325)
int count_inliers(const sim3_model &m, const double *cam, const double *pts_1, const double *pts_2,
                  const std::vector<double> &reprojected_1, const std::vector<double> &reprojected_2,
                  const float *chi_sq_1, const float *chi_sq_2, int n) {
    int num_inliers = 0;
    for (int i = 0; i < n; ++i)
        num_inliers += sim3_is_inlier(&m, cam, pts_1 + 3 * (size_t)i, pts_2 + 3 * (size_t)i,
                                      reprojected_1.data() + 2 * (size_t)i, reprojected_2.data() + 2 * (size_t)i,
                                      chi_sq_1[i], chi_sq_2[i]);
    return num_inliers;
}

}  // namespace

extern "C" {

/* compute_Sim3 (:193-288) of one hypothesis; pts: 3 points x 3 coordinates.  rot row-major. */
void orc_sim3_compute(const double *pts_1, const double *pts_2, int fix_scale, double *rot_12, double *trans_12,
                      float *scale_12, double *rot_21, double *trans_21, float *scale_21) {
    sim3_model m;
    sim3_compute(pts_1, pts_2, fix_scale, &m);
    std::memcpy(rot_12, m.rot_12, sizeof(m.rot_12));
    std::memcpy(trans_12, m.trans_12, sizeof(m.trans_12));
    std::memcpy(rot_21, m.rot_21, sizeof(m.rot_21));
    std::memcpy(trans_21, m.trans_21, sizeof(m.trans_21));
    *scale_12 = m.scale_12;
    *scale_21 = m.scale_21;
}

/* find_via_ransac(num_iter) (:121-191) of P independent problems, as plp_sim3_ransac (include/plpslam_b200.h); cams:
 * P x 4 (fx, fy, cx, cy).  hyp_num_inliers_out (optional, P x num_iter) receives count_inliers of every hypothesis of a
 * problem that ran. */
void orc_sim3_ransac(int num_problems, const int32_t *corr_offsets, const double *cams, const double *pts_1,
                     const double *pts_2, const float *chi_sq_1, const float *chi_sq_2, const int32_t *samples,
                     int num_iter, int fix_scale, int min_num_inliers, int32_t *valid_out, int32_t *num_inliers_out,
                     double *rot_12_out, double *trans_12_out, float *scale_12_out, int32_t *hyp_num_inliers_out) {
    constexpr int min_set_size = 3;
    for (int p = 0; p < num_problems; ++p) {
        const int off = corr_offsets[p], n = corr_offsets[p + 1] - off;
        const double *cam = cams + 4 * (size_t)p;
        const double *x1 = pts_1 + 3 * (size_t)off, *x2 = pts_2 + 3 * (size_t)off;
        // :124-128
        int max_num_inliers = 0;
        int valid = 0;
        double best_rot_12[9] = {0}, best_trans_12[3] = {0};
        float best_scale_12 = 0.0f;
        if (n >= min_set_size && n >= min_num_inliers) {  // :130-134
            std::vector<double> reprojected_1, reprojected_2;
            reproject_to_same_image(cam, x1, n, reprojected_1);
            reproject_to_same_image(cam, x2, n, reprojected_2);
            for (int iter = 0; iter < num_iter; ++iter) {  // :145-175
                const int32_t *s = samples + ((size_t)p * num_iter + iter) * min_set_size;
                double sp1[9], sp2[9];
                for (int k = 0; k < min_set_size; ++k)
                    for (int r = 0; r < 3; ++r) {
                        sp1[3 * k + r] = x1[3 * (size_t)s[k] + r];
                        sp2[3 * k + r] = x2[3 * (size_t)s[k] + r];
                    }
                sim3_model m;
                sim3_compute(sp1, sp2, fix_scale, &m);
                const int num = count_inliers(m, cam, x1, x2, reprojected_1, reprojected_2, chi_sq_1 + off, chi_sq_2 + off, n);
                if (hyp_num_inliers_out) hyp_num_inliers_out[(size_t)p * num_iter + iter] = num;
                if (max_num_inliers < num) {
                    max_num_inliers = num;
                    std::memcpy(best_rot_12, m.rot_12, sizeof(best_rot_12));
                    std::memcpy(best_trans_12, m.trans_12, sizeof(best_trans_12));
                    best_scale_12 = m.scale_12;
                }
            }
            valid = !(max_num_inliers < min_num_inliers);  // :177-190
            if (!valid) {
                std::memset(best_rot_12, 0, sizeof(best_rot_12));
                std::memset(best_trans_12, 0, sizeof(best_trans_12));
                best_scale_12 = 0.0f;
            }
        }
        valid_out[p] = valid;
        num_inliers_out[p] = max_num_inliers;
        std::memcpy(rot_12_out + 9 * (size_t)p, best_rot_12, sizeof(best_rot_12));
        std::memcpy(trans_12_out + 3 * (size_t)p, best_trans_12, sizeof(best_trans_12));
        scale_12_out[p] = best_scale_12;
    }
}

}  // extern "C"
