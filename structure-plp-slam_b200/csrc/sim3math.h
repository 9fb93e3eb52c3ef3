/* sim3math.h -- Horn's closed-form Sim3 and the two-image inlier test of solve::sim3_solver (solve/sim3_solver.cc:193-358)
 * in plain IEEE-754 double / float arithmetic (+, -, *, /, sqrt only; no FMA, no library calls), so that a host build
 * (-ffp-contract=off) and a device build (-fmad=false) return bit-identical results.
 *
 * Types and operation order are the reference's.  Where it calls Eigen, the restatement fixes one order:
 *   - rowwise().mean() (:201-202): ((p0 + p1) + p2) / 3.0 per row;
 *   - every 3 x 3 product (M = A1 A2^T :213, rot_21 * ave_pts_1 :270, matrix x vector :282, :287, the reprojection's
 *     rot_cw * pos_w) sums its three terms left to right, (a0 b0 + a1 b1) + a2 b2;
 *   - squaredNorm() (:253, :259, :273) and cwiseProduct().sum() (:275) sum left to right over Eigen's storage order:
 *     column-major for a 3 x 3 matrix, (x, y, z, w) for a quaternion's coefficients;
 *   - Eigen::EigenSolver<Mat44_t> of the symmetric N (:234): cyclic Jacobi rotations (ess_jacobi_eig<4>, essmath.h); the
 *     eigenvalues are the rotated diagonal, scanned in index order with the reference's `max_eigenvalue <= lambda`;
 *   - normalize() / normalized() divide by sqrt(squaredNorm()) when it is positive; toRotationMatrix() is Eigen's
 *     published formula (Quaternion.h).  q and -q give bit-identical rotations in it (negation is exact and every term is
 *     a product of two coefficients), so the eigenvector's sign does not reach the result.
 * A float times a double matrix (scale_21 * rot_21, -scale_12 * rot_12) promotes the float and multiplies element-wise
 * first, as Eigen's scalar product does; the scales are stored as float (:277, :286) exactly as the reference stores them.
 * These orders are Eigen's where Eigen's own is plain and may differ from its unrolled reductions elsewhere: PARITY
 * UNPINNED against Eigen (absent).
 *
 * TWO INTENDED DEVIATIONS:
 *   1. reproject_to_image (camera/perspective.cc:190-209, camera/fisheye.cc:231-250) returns early for z <= 0, and the
 *      reference's reproject_to_other_image / reproject_to_same_image then store an uninitialised Vec2_t.  Here that
 *      reprojection is NaN: the correspondence is never an inlier of that hypothesis (other image) or of any hypothesis
 *      (same image), since every comparison against NaN is false.
 *   2. For exactly tied largest eigenvalues the last one in Jacobi's diagonal order wins, not the last in Eigen's order.
 *      Ties need degenerate samples (coincident or collinear points).
 * With NaN in N no eigenvalue passes the scan and the reference reads column -1; here column 0 (NaN input only).
 *
 * The library (nvcc -fmad=false), the oracle (g++ -ffp-contract=off) and the CPU emulators of tests/cta_emu compile
 * this one text, so the device and the oracle evaluate the same expressions.
 */
#ifndef PLP_SIM3MATH_H
#define PLP_SIM3MATH_H

#include "essmath.h"

#if defined(__CUDACC__)
#define SIM3_HD __host__ __device__ __forceinline__
#else
#define SIM3_HD static inline
#endif

/* sim3_solver.cc:67, chi-square at 1 % significance with 2 degrees of freedom */
#define SIM3_CHI_SQ_2D 9.21034f

/* One hypothesis: both directions, rotations row-major. */
struct sim3_model {
    double rot_12[9], trans_12[3];
    double rot_21[9], trans_21[3];
    float scale_12, scale_21;
};

/* compute_Sim3 (:193-288).  pts_1 / pts_2: the three sampled points of each keyframe, point k at [3 k .. 3 k + 2]
 * (the reference's column k). */
SIM3_HD void sim3_compute(const double *pts_1, const double *pts_2, int fix_scale, sim3_model *m) {
    /* :201-208 centroids and centred points; a1[3 k + r] = ave_pts_1(r, k) */
    double c1[3], c2[3], a1[9], a2[9];
    for (int r = 0; r < 3; ++r) {
        c1[r] = ((pts_1[r] + pts_1[3 + r]) + pts_1[6 + r]) / 3.0;
        c2[r] = ((pts_2[r] + pts_2[3 + r]) + pts_2[6 + r]) / 3.0;
    }
    for (int k = 0; k < 3; ++k)
        for (int r = 0; r < 3; ++r) {
            a1[3 * k + r] = pts_1[3 * k + r] - c1[r];
            a2[3 * k + r] = pts_2[3 * k + r] - c2[r];
        }
    /* :213 M = A1 A2^T: M(i, j) = sum_k A1(i, k) A2(j, k) */
    double M[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) M[3 * i + j] = (a1[i] * a2[j] + a1[3 + i] * a2[3 + j]) + a1[6 + i] * a2[6 + j];
    const double Sxx = M[0], Sxy = M[1], Sxz = M[2];
    const double Syx = M[3], Syy = M[4], Syz = M[5];
    const double Szx = M[6], Szy = M[7], Szz = M[8];
    /* :225-229, row-major and symmetric as written */
    double N[16] = {(Sxx + Syy) + Szz, Syz - Szy,         Szx - Sxz,          Sxy - Syx,
                    Syz - Szy,         (Sxx - Syy) - Szz, Sxy + Syx,          Szx + Sxz,
                    Szx - Sxz,         Sxy + Syx,         (-Sxx + Syy) - Szz, Syz + Szy,
                    Sxy - Syx,         Szx + Sxz,         Syz + Szy,          (-Sxx - Syy) + Szz};
    /* :234-248 */
    double V[16];
    ess_jacobi_eig<4>(N, V);
    int max_idx = -1;
    double max_eigenvalue = -(1.0 / 0.0);
    for (int idx = 0; idx < 4; ++idx)
        if (max_eigenvalue <= N[5 * idx]) {
            max_eigenvalue = N[5 * idx];
            max_idx = idx;
        }
    if (max_idx < 0) max_idx = 0;
    /* :251-253 normalize() */
    double e[4] = {V[max_idx], V[4 + max_idx], V[8 + max_idx], V[12 + max_idx]};
    double z = ((e[0] * e[0] + e[1] * e[1]) + e[2] * e[2]) + e[3] * e[3];
    if (z > 0.0) {
        const double s = sqrt(z);
        for (int k = 0; k < 4; ++k) e[k] = e[k] / s;
    }
    /* :256-259 Quaterniond(w, x, y, z).normalized(): coefficients stored (x, y, z, w) */
    double qw = e[0], qx = e[1], qy = e[2], qz = e[3];
    z = ((qx * qx + qy * qy) + qz * qz) + qw * qw;
    if (z > 0.0) {
        const double s = sqrt(z);
        qx = qx / s;
        qy = qy / s;
        qz = qz / s;
        qw = qw / s;
    }
    /* toRotationMatrix() */
    const double tx = 2.0 * qx, ty = 2.0 * qy, tz = 2.0 * qz;
    const double twx = tx * qw, twy = ty * qw, twz = tz * qw;
    const double txx = tx * qx, txy = ty * qx, txz = tz * qx;
    const double tyy = ty * qy, tyz = tz * qy, tzz = tz * qz;
    double *R = m->rot_21;
    R[0] = 1.0 - (tyy + tzz);
    R[1] = txy - twz;
    R[2] = txz + twy;
    R[3] = txy + twz;
    R[4] = 1.0 - (txx + tzz);
    R[5] = tyz - twx;
    R[6] = txz - twy;
    R[7] = tyz + twx;
    R[8] = 1.0 - (txx + tyy);
    /* :263-278 */
    if (fix_scale) {
        m->scale_21 = 1.0f;
    } else {
        /* b[3 k + r] = (rot_21 * ave_pts_1)(r, k); column-major sums */
        double denom = 0.0, numer = 0.0;
        for (int k = 0; k < 3; ++k)
            for (int r = 0; r < 3; ++r) {
                const double b = (R[3 * r] * a1[3 * k] + R[3 * r + 1] * a1[3 * k + 1]) + R[3 * r + 2] * a1[3 * k + 2];
                denom = denom + a1[3 * k + r] * a1[3 * k + r];
                numer = numer + a2[3 * k + r] * b;
            }
        m->scale_21 = (float)(numer / denom);
    }
    /* :282 trans_21 = centroid_2 - (scale_21 * rot_21) * centroid_1 */
    const double s21 = (double)m->scale_21;
    for (int r = 0; r < 3; ++r)
        m->trans_21[r] = c2[r] - (((s21 * R[3 * r]) * c1[0] + (s21 * R[3 * r + 1]) * c1[1]) + (s21 * R[3 * r + 2]) * c1[2]);
    /* :285-287 */
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) m->rot_12[3 * r + c] = R[3 * c + r];
    m->scale_12 = (float)(1.0 / (double)m->scale_21);
    const double ns12 = (double)(-m->scale_12);
    const double *R12 = m->rot_12;
    for (int r = 0; r < 3; ++r)
        m->trans_12[r] = ((ns12 * R12[3 * r]) * m->trans_21[0] + (ns12 * R12[3 * r + 1]) * m->trans_21[1]) +
                         (ns12 * R12[3 * r + 2]) * m->trans_21[2];
}

/* camera::{perspective,fisheye}::reproject_to_image(scale * rot, trans, pos) (perspective.cc:190-209, fisheye.cc:231-250;
 * the same formula) as sim3_solver calls it; rot row-major.  z <= 0: NaN (deviation 1 above). */
SIM3_HD void sim3_reproject(const double *rot, const double *trans, float scale, const double *cam /* fx fy cx cy */,
                            const double *pos, double *reproj) {
    const double s = (double)scale;
    double pc[3];
    for (int r = 0; r < 3; ++r)
        pc[r] = (((s * rot[3 * r]) * pos[0] + (s * rot[3 * r + 1]) * pos[1]) + (s * rot[3 * r + 2]) * pos[2]) + trans[r];
    if (pc[2] <= 0.0) {
        reproj[0] = reproj[1] = NAN;
        return;
    }
    const double z_inv = 1.0 / pc[2];
    reproj[0] = (cam[0] * pc[0]) * z_inv + cam[2];
    reproj[1] = (cam[1] * pc[1]) * z_inv + cam[3];
}

/* reproject_to_same_image (:344-358): rotation Identity, translation Zero (the product is still evaluated) */
SIM3_HD void sim3_reproject_same(const double *cam, const double *pos, double *reproj) {
    const double I[9] = {1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0}, Z[3] = {0.0, 0.0, 0.0};
    sim3_reproject(I, Z, 1.0f, cam, pos, reproj);
}

/* count_inliers (:290-325) for correspondence i: the two reprojections of this hypothesis against the same-image ones;
 * double squared errors, strict `<` against the float thresholds chi_sq_2D * sigma_sq (promoted). */
SIM3_HD int sim3_is_inlier(const sim3_model *m, const double *cam, const double *pt_1, const double *pt_2,
                           const double *reproj_1, const double *reproj_2, float chi_sq_1, float chi_sq_2) {
    double r12[2], r21[2];
    sim3_reproject(m->rot_21, m->trans_21, m->scale_21, cam, pt_1, r12);  /* points 1 into image 2 */
    sim3_reproject(m->rot_12, m->trans_12, m->scale_12, cam, pt_2, r21);  /* points 2 into image 1 */
    const double d2x = r12[0] - reproj_2[0], d2y = r12[1] - reproj_2[1];
    const double d1x = r21[0] - reproj_1[0], d1y = r21[1] - reproj_1[1];
    const double error_in_2 = d2x * d2x + d2y * d2y;
    const double error_in_1 = d1x * d1x + d1y * d1y;
    return (error_in_2 < (double)chi_sq_2 && error_in_1 < (double)chi_sq_1) ? 1 : 0;
}

#endif
