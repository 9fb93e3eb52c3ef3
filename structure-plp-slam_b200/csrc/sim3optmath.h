/* sim3optmath.h -- the g2o pieces of optimize::transform_optimizer (optimize/transform_optimizer.cc:47-197) that are not
 * already restated for the pose optimiser: the 7-DoF g2o::Sim3, transform_vertex::oplusImpl, the two mutual reprojection
 * edges (optimize/g2o/sim3/{forward,backward}_reproj_edge.h) and BaseUnaryEdge's central-difference Jacobian, in plain
 * IEEE-754 double arithmetic with no FMA (host: -ffp-contract=off; device: -fmad=false).
 *
 * g2o is NOT under the reference tree and is not installed.  PARITY UNPINNED: everything below is restated from g2o's
 * published types/sim3/sim3.h and core/base_unary_edge.hpp, as g2o_lite.hpp does for SE3Quat.  Restated, branch by branch:
 *   - Sim3(const Vector7 &update), update = (omega, upsilon, sigma): s = exp(sigma), theta = |omega|, eps = 1e-5;
 *       |sigma| <  eps, theta <  eps: A = 1/2, B = 1/6, C = 1, R = I + Omega + Omega^2 (g2o's own second-order term);
 *       |sigma| <  eps, theta >= eps: A = (1 - cos theta) / theta^2, B = (theta - sin theta) / (theta^2 theta), C = 1,
 *                                     R = I + sin theta / theta Omega + (1 - cos theta) / theta^2 Omega^2;
 *       |sigma| >= eps, theta <  eps: C = (s - 1) / sigma, A = ((sigma - 1) s + 1) / sigma^2,
 *                                     B = ((sigma^2 / 2 - sigma + 1) s - 1) / (sigma^2 sigma), R = I + Omega + Omega^2
 *                                     (the theta -> 0 limit; some older g2o copies omit the "- 1", which makes B ~ 1 /
 *                                     sigma^3 -- tests/test_sim3_opt_oracle.py pins this branch against expm);
 *       |sigma| >= eps, theta >= eps: C = (s - 1) / sigma, a = s sin theta, b = s cos theta, c = theta^2 + sigma^2,
 *                                     A = (a sigma + (1 - b) theta) / (theta c), B = (C - ((b - 1) sigma + a theta) / c) / theta^2,
 *                                     R as in the second case;
 *     then r = Quaternion(R) (not normalised) and t = (A Omega + B Omega^2 + C I) upsilon;
 *   - Sim3(R, t, s) and Sim3(q, t, s) normalise the rotation: q -> -q when w < 0, then q / |q| (normalizeRotation);
 *   - map(x) = s (r x) + t, with Eigen's quaternion-vector product uv = 2 (v x x), r x = x + w uv + v x uv;
 *   - inverse() = Sim3(conj(r), conj(r) ((-1 / s) t), 1 / s);
 *   - (a * b): r = a.r b.r (Eigen's quaternion product, not normalised), t = a.s (a.r b.t) + a.t, s = a.s b.s;
 *   - transform_vertex::oplusImpl: update(6) = 0 when fix_scale_ -- IN PLACE, so the caller's step vector loses its scale
 *     component too (g2o's Levenberg scale dx^T (lambda dx + b) then reads the zeroed dx) -- and estimate = Sim3(update) *
 *     estimate;
 *   - BaseUnaryEdge::linearizeOplus: delta = 1e-9, column d = (e(oplus(+delta e_d)) - e(oplus(-delta e_d))) / (2 delta),
 *     the scalar 1 / (2 delta) multiplied in; with fix_scale both perturbations of column 6 are the estimate itself, so the
 *     column is exactly 0.
 * Eigen's fixed-size 3 x 3 products sum their terms left to right, (a0 b0 + a1 b1) + a2 b2, and its quaternion norm sums
 * (x, y, z, w) in storage order.  Eigen(Quaternion(Matrix3)) and toRotationMatrix() are the helpers the pose optimiser
 * already restates (se3.cuh R_to_quat / quat_to_R on the device, g2o_lite.hpp quat_from_matrix / quat_to_matrix in the
 * oracle; the same arithmetic), reached through s3o_R_to_quat / s3o_quat_to_R below.
 *
 * This file exists twice with identical text (oracle/sim3optmath.h and structure-plp-slam_b200/csrc/sim3optmath.h); the
 * oracle defines SIM3OPT_WITH_G2O_LITE before including it and never includes product code, and vice versa.
 * tests/test_sim3_opt_oracle.py checks that the copies stay identical.
 */
#ifndef PLP_SIM3OPTMATH_H
#define PLP_SIM3OPTMATH_H

#include <math.h>

#if defined(__CUDACC__)
#define SIM3O_HD __host__ __device__ __forceinline__
#else
#define SIM3O_HD static inline
#endif

#if defined(SIM3OPT_WITH_G2O_LITE)
#include "g2o_lite.hpp"
/* Eigen::Quaternion(Matrix3) of a row-major R; q = (w, x, y, z) */
SIM3O_HD void s3o_R_to_quat(const double *R, double *q) {
    g2o_lite::Mat3 M;
    for (int i = 0; i < 9; ++i) M.m[i] = R[i];
    const g2o_lite::Quat Q = g2o_lite::quat_from_matrix(M);
    q[0] = Q.w;
    q[1] = Q.x;
    q[2] = Q.y;
    q[3] = Q.z;
}
/* Quaternion::toRotationMatrix(), row-major */
SIM3O_HD void s3o_quat_to_R(const double *q, double *R) {
    const g2o_lite::Mat3 M = g2o_lite::quat_to_matrix(g2o_lite::Quat{q[0], q[1], q[2], q[3]});
    for (int i = 0; i < 9; ++i) R[i] = M.m[i];
}
#else
#include "se3.cuh"
SIM3O_HD void s3o_R_to_quat(const double *R, double *q) { plp::se3::R_to_quat(R, q[0], q[1], q[2], q[3]); }
SIM3O_HD void s3o_quat_to_R(const double *q, double *R) { plp::se3::quat_to_R(q[0], q[1], q[2], q[3], R); }
#endif

/* g2o::Sim3: rotation r as a quaternion (w, x, y, z), translation t, scale s */
struct s3o_sim3 {
    double q[4];
    double t[3];
    double s;
};

#define SIM3O_NUMERIC_DELTA 1e-9 /* BaseUnaryEdge::linearizeOplus */

/* Sim3::normalizeRotation */
SIM3O_HD void s3o_normalize_rotation(double *q) {
    if (q[0] < 0) {
        q[0] = -q[0];
        q[1] = -q[1];
        q[2] = -q[2];
        q[3] = -q[3];
    }
    const double n = sqrt(((q[1] * q[1] + q[2] * q[2]) + q[3] * q[3]) + q[0] * q[0]);
    q[0] /= n;
    q[1] /= n;
    q[2] /= n;
    q[3] /= n;
}

/* Sim3(const Matrix3 &R, const Vector3 &t, number_t s); R row-major */
SIM3O_HD s3o_sim3 s3o_from_Rts(const double *R, const double *t, double s) {
    s3o_sim3 S;
    s3o_R_to_quat(R, S.q);
    s3o_normalize_rotation(S.q);
    S.t[0] = t[0];
    S.t[1] = t[1];
    S.t[2] = t[2];
    S.s = s;
    return S;
}

/* Eigen's Quaternion * Vector3 (_transformVector) */
SIM3O_HD void s3o_rotate(const double *q, const double *v, double *out) {
    double uv[3] = {q[2] * v[2] - q[3] * v[1], q[3] * v[0] - q[1] * v[2], q[1] * v[1] - q[2] * v[0]};
    uv[0] += uv[0];
    uv[1] += uv[1];
    uv[2] += uv[2];
    const double c[3] = {q[2] * uv[2] - q[3] * uv[1], q[3] * uv[0] - q[1] * uv[2], q[1] * uv[1] - q[2] * uv[0]};
    out[0] = (v[0] + q[0] * uv[0]) + c[0];
    out[1] = (v[1] + q[0] * uv[1]) + c[1];
    out[2] = (v[2] + q[0] * uv[2]) + c[2];
}

/* Sim3::map: s (r x) + t */
SIM3O_HD void s3o_map(const s3o_sim3 &S, const double *x, double *out) {
    double rx[3];
    s3o_rotate(S.q, x, rx);
    out[0] = S.s * rx[0] + S.t[0];
    out[1] = S.s * rx[1] + S.t[1];
    out[2] = S.s * rx[2] + S.t[2];
}

/* Sim3::operator*: a * b */
SIM3O_HD s3o_sim3 s3o_mul(const s3o_sim3 &a, const s3o_sim3 &b) {
    s3o_sim3 o;
    o.q[0] = a.q[0] * b.q[0] - a.q[1] * b.q[1] - a.q[2] * b.q[2] - a.q[3] * b.q[3];
    o.q[1] = a.q[0] * b.q[1] + a.q[1] * b.q[0] + a.q[2] * b.q[3] - a.q[3] * b.q[2];
    o.q[2] = a.q[0] * b.q[2] + a.q[2] * b.q[0] + a.q[3] * b.q[1] - a.q[1] * b.q[3];
    o.q[3] = a.q[0] * b.q[3] + a.q[3] * b.q[0] + a.q[1] * b.q[2] - a.q[2] * b.q[1];
    double rt[3];
    s3o_rotate(a.q, b.t, rt);
    o.t[0] = a.s * rt[0] + a.t[0];
    o.t[1] = a.s * rt[1] + a.t[1];
    o.t[2] = a.s * rt[2] + a.t[2];
    o.s = a.s * b.s;
    return o;
}

/* Sim3::inverse: Sim3(conj(r), conj(r) ((-1 / s) t), 1 / s) */
SIM3O_HD s3o_sim3 s3o_inverse(const s3o_sim3 &a) {
    s3o_sim3 o;
    o.q[0] = a.q[0];
    o.q[1] = -a.q[1];
    o.q[2] = -a.q[2];
    o.q[3] = -a.q[3];
    const double k = -1 / a.s;
    const double kt[3] = {k * a.t[0], k * a.t[1], k * a.t[2]};
    s3o_rotate(o.q, kt, o.t);
    o.s = 1 / a.s;
    s3o_normalize_rotation(o.q);
    return o;
}

/* Sim3(const Vector7 &update), update = (omega, upsilon, sigma) */
SIM3O_HD s3o_sim3 s3o_exp(const double *u) {
    const double wx = u[0], wy = u[1], wz = u[2];
    const double sigma = u[6];
    const double theta = sqrt((wx * wx + wy * wy) + wz * wz);
    const double O[9] = {0, -wz, wy, wz, 0, -wx, -wy, wx, 0};
    double O2[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) O2[i * 3 + j] = (O[i * 3] * O[j] + O[i * 3 + 1] * O[3 + j]) + O[i * 3 + 2] * O[6 + j];
    const double s = exp(sigma);
    const double eps = 0.00001;
    double A, B, C, ra, rb;  // R = I + ra Omega + rb Omega^2
    if (fabs(sigma) < eps) {
        C = 1;
        if (theta < eps) {
            A = 1. / 2.;
            B = 1. / 6.;
            ra = 1.0;
            rb = 1.0;
        } else {
            const double theta2 = theta * theta;
            A = (1 - cos(theta)) / theta2;
            B = (theta - sin(theta)) / (theta2 * theta);
            ra = sin(theta) / theta;
            rb = (1 - cos(theta)) / (theta * theta);
        }
    } else {
        C = (s - 1) / sigma;
        if (theta < eps) {
            const double sigma2 = sigma * sigma;
            A = ((sigma - 1) * s + 1) / sigma2;
            B = ((0.5 * sigma2 - sigma + 1) * s - 1) / (sigma2 * sigma);
            ra = 1.0;
            rb = 1.0;
        } else {
            ra = sin(theta) / theta;
            rb = (1 - cos(theta)) / (theta * theta);
            const double a = s * sin(theta), b = s * cos(theta);
            const double theta2 = theta * theta, sigma2 = sigma * sigma;
            const double c = theta2 + sigma2;
            A = (a * sigma + (1 - b) * theta) / (theta * c);
            B = (C - ((b - 1) * sigma + a * theta) / c) * 1. / theta2;
        }
    }
    /* the small-angle branches' I + Omega + Omega^2 is ra = rb = 1: multiplying by 1.0 is exact */
    double R[9], W[9];
    for (int i = 0; i < 9; ++i) {
        const double I = (i == 0 || i == 4 || i == 8) ? 1.0 : 0.0;
        R[i] = (I + ra * O[i]) + rb * O2[i];
        W[i] = (A * O[i] + B * O2[i]) + C * I;
    }
    s3o_sim3 S;
    s3o_R_to_quat(R, S.q);
    for (int r = 0; r < 3; ++r) S.t[r] = (W[r * 3] * u[3] + W[r * 3 + 1] * u[4]) + W[r * 3 + 2] * u[5];
    S.s = s;
    return S;
}

/* transform_vertex::oplusImpl; zeroes u[6] in place when fix_scale, as the reference does through its Eigen::Map */
SIM3O_HD s3o_sim3 s3o_oplus(const s3o_sim3 &est, double *u, int fix_scale) {
    if (fix_scale) u[6] = 0;
    return s3o_mul(s3o_exp(u), est);
}

/* rot_kw * pos_w + trans_kw (the edges' first line); R row-major */
SIM3O_HD void s3o_to_cam(const double *R, const double *t, const double *X, double *pc) {
    pc[0] = ((R[0] * X[0] + R[1] * X[1]) + R[2] * X[2]) + t[0];
    pc[1] = ((R[3] * X[0] + R[4] * X[1]) + R[5] * X[2]) + t[1];
    pc[2] = ((R[6] * X[0] + R[7] * X[1]) + R[8] * X[2]) + t[2];
}

/* computeError of both edges: obs - cam_project(S.map(pc)), cam_project = perspective_{forward,backward}_reproj_edge's
 * (fx x / z + cx, fy y / z + cy); cam = (fx, fy, cx, cy).  Forward: S = Sim3_12, pc = rot_2w pos_w_2 + trans_2w.  Backward:
 * S = Sim3_12.inverse(), pc = rot_1w pos_w_1 + trans_1w. */
SIM3O_HD void s3o_error(const double *cam, const s3o_sim3 &S, const double *pc, const double *obs, double *e) {
    double p[3];
    s3o_map(S, pc, p);
    e[0] = obs[0] - (cam[0] * p[0] / p[2] + cam[2]);
    e[1] = obs[1] - (cam[1] * p[1] / p[2] + cam[3]);
}

/* _error.dot(information() * _error) with information = inv_sigma_sq I */
SIM3O_HD double s3o_chi2(const double *e, double w) { return e[0] * (w * e[0]) + e[1] * (w * e[1]); }

/* The 14 estimates linearizeOplus visits: pert[2 d] = oplus(+delta e_d), pert[2 d + 1] = oplus(-delta e_d). */
SIM3O_HD s3o_sim3 s3o_perturbed(const s3o_sim3 &est, int k, int fix_scale) {
    double u[7];
    for (int d = 0; d < 7; ++d) u[d] = d == (k >> 1) ? ((k & 1) ? -SIM3O_NUMERIC_DELTA : SIM3O_NUMERIC_DELTA) : 0.0;
    return s3o_oplus(est, u, fix_scale);
}

/* One edge's numeric Jacobian, J row-major 2 x 7, from the 14 visited estimates as this edge's computeError sees them
 * (the estimates themselves for the forward edge, their inverses for the backward one). */
SIM3O_HD void s3o_numeric_jacobian(const double *cam, const s3o_sim3 *visited, const double *pc, const double *obs,
                                   double *J) {
    const double scalar = 1 / (2 * SIM3O_NUMERIC_DELTA);
    for (int d = 0; d < 7; ++d) {
        double ep[2], em[2];
        s3o_error(cam, visited[2 * d], pc, obs, ep);
        s3o_error(cam, visited[2 * d + 1], pc, obs, em);
        J[d] = scalar * (ep[0] - em[0]);
        J[7 + d] = scalar * (ep[1] - em[1]);
    }
}

#endif /* PLP_SIM3OPTMATH_H */
