// oracle/pnp.cc -- solve::pnp_solver (TEST INFRASTRUCTURE ONLY).  Follows
// /root/reference/src/PLPSLAM/solve/pnp_solver.cc; EPnP itself is restated in pnpmath.h (see its header).
#include "pnpmath.h"

#include <stdint.h>

#include <cstring>
#include <vector>

namespace {

// the reference's pws_ / us_ / alphas_ / pcs_ / signs_ for up to `cap` correspondences (set_max_num_correspondences,
// :188-202; reset_correspondences, :183-186)
struct Corr {
    std::vector<double> pws, us, alphas, pcs;
    std::vector<int> signs;
    pnp_work w;
    explicit Corr(size_t cap) : pws(3 * cap + 3), us(2 * cap + 2), alphas(4 * cap + 4), pcs(3 * cap + 3), signs(cap + 1) {
        w = pnp_work{pws.data(), us.data(), alphas.data(), pcs.data(), signs.data(), 0};
    }
};

// check_inliers (:155-181)
int check_inliers(const double *R, const double *t, const double *bearings, const double *pos_w, const float *max_cos,
                  int n, uint8_t *flags) {
    int num = 0;
    for (int i = 0; i < n; ++i) {
        flags[i] = (uint8_t)pnp_is_inlier(R, t, pos_w + 3 * (size_t)i, bearings + 3 * (size_t)i, max_cos[i]);
        num += flags[i];
    }
    return num;
}

}  // namespace

extern "C" {

/* compute_pose (:230-290) over the correspondences (pos_w[i], bearing[i]), i < n, added by add_correspondence (:204-228,
 * z == 0 skipped).  Returns the reprojection error; *num_used = correspondences kept. */
double orc_pnp_compute_pose(const double *bearings, const double *pos_w, int n, double *R_out, double *t_out, int *num_used) {
    Corr c((size_t)n);
    for (int i = 0; i < n; ++i) pnp_add_correspondence(&c.w, pos_w + 3 * (size_t)i, bearings + 3 * (size_t)i);
    if (num_used) *num_used = c.w.n;
    return pnp_compute_pose(&c.w, R_out, t_out);
}

/* JacobiSVD(L_6xk).solve(rho), k in {3, 4, 5} (find_betas_approx_1/2/3) */
void orc_pnp_min_norm_solve(int k, const double *L, const double *rho, double *x) {
    if (k == 3) pnp_min_norm_solve<3>(L, rho, x);
    if (k == 4) pnp_min_norm_solve<4>(L, rho, x);
    if (k == 5) pnp_min_norm_solve<5>(L, rho, x);
}

/* estimate_R_and_t (:440-519) from camera-frame points pcs and world points pws (n x 3 each) */
void orc_pnp_estimate_R_and_t(const double *pcs, const double *pws, int n, double *R_out, double *t_out) {
    Corr c((size_t)n);
    std::memcpy(c.pcs.data(), pcs, sizeof(double) * 3 * (size_t)n);
    std::memcpy(c.pws.data(), pws, sizeof(double) * 3 * (size_t)n);
    c.w.n = n;
    double R[3][3];
    pnp_estimate_R_and_t(&c.w, R, t_out);
    for (int r = 0; r < 3; ++r)
        for (int k = 0; k < 3; ++k) R_out[r * 3 + k] = R[r][k];
}

/* qr_solve (:748-866), A 6 x 4 row-major */
void orc_pnp_qr_solve(const double *A, const double *b, double *X) {
    double a[24], bb[6];
    std::memcpy(a, A, sizeof(a));
    std::memcpy(bb, b, sizeof(bb));
    pnp_qr_solve(a, bb, X);
}

/* find_via_ransac(num_iter, recompute) (:70-153) of P independent problems, as plp_pnp_ransac (include/plpslam_b200.h).
 * hyp_num_inliers_out (optional, P x num_iter) receives check_inliers' count of every hypothesis of a problem that ran. */
void orc_pnp_ransac(int num_problems, const int32_t *corr_offsets, const double *bearings, const double *pos_w,
                    const float *max_cos_error, const int32_t *samples, int num_iter, int min_num_inliers, int recompute,
                    int32_t *valid_out, int32_t *num_inliers_out, double *pose_cw_out, uint8_t *is_inlier_out,
                    int32_t *hyp_num_inliers_out) {
    constexpr int min_set_size = 4;
    for (int p = 0; p < num_problems; ++p) {
        const int off = corr_offsets[p], n = corr_offsets[p + 1] - off;
        valid_out[p] = 0;
        num_inliers_out[p] = 0;
        if (n < min_set_size || n < min_num_inliers) continue;  // :76-80
        const double *b = bearings + 3 * (size_t)off, *x = pos_w + 3 * (size_t)off;
        const float *mc = max_cos_error + off;
        uint8_t *best = is_inlier_out + off;
        std::vector<uint8_t> in_sac((size_t)n);
        std::memset(best, 0, (size_t)n);
        int max_num_inliers = 0;
        double best_R[9] = {0}, best_t[3] = {0};
        Corr c(min_set_size);
        for (int iter = 0; iter < num_iter; ++iter) {  // :96-124
            const int32_t *s = samples + ((size_t)p * num_iter + iter) * min_set_size;
            c.w.n = 0;
            for (int k = 0; k < min_set_size; ++k) pnp_add_correspondence(&c.w, x + 3 * (size_t)s[k], b + 3 * (size_t)s[k]);
            double R[9], t[3];
            pnp_compute_pose(&c.w, R, t);
            const int num = check_inliers(R, t, b, x, mc, n, in_sac.data());
            if (hyp_num_inliers_out) hyp_num_inliers_out[(size_t)p * num_iter + iter] = num;
            if (max_num_inliers < num) {
                max_num_inliers = num;
                std::memcpy(best_R, R, sizeof(R));
                std::memcpy(best_t, t, sizeof(t));
                std::memcpy(best, in_sac.data(), (size_t)n);
            }
        }
        num_inliers_out[p] = max_num_inliers;
        const int valid = max_num_inliers > min_num_inliers;  // :126-129
        valid_out[p] = valid;
        if (!valid) continue;
        if (recompute) {  // :136-152, the inlier flags are not re-tested
            Corr all((size_t)n);
            for (int i = 0; i < n; ++i)
                if (best[i]) pnp_add_correspondence(&all.w, x + 3 * (size_t)i, b + 3 * (size_t)i);
            pnp_compute_pose(&all.w, best_R, best_t);
        }
        pnp_cam_pose(best_R, best_t, pose_cw_out + 16 * (size_t)p);
    }
}

}  // extern "C"
