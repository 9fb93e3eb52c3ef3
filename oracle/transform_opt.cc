// oracle/transform_opt.cc -- CPU restatement of optimize::transform_optimizer::optimize (TEST INFRASTRUCTURE ONLY).
// Follows optimize/transform_optimizer.cc:47-197 step by step; the Sim3 vertex, the mutual edges and the numeric
// Jacobian are restated in sim3optmath.h, the Huber kernel and the SPD solve in g2o_lite.hpp, and the Levenberg driver
// is the one of pose_opt.cc at dimension 7 (PARITY UNPINNED, see both headers).
#define SIM3OPT_WITH_G2O_LITE
#include "sim3optmath.h"

#include <stdint.h>

#include <algorithm>
#include <cstring>
#include <limits>
#include <vector>

namespace {

// Summation order.  g2o sums H, b and chi2 over its active-edge container, whose order follows heap addresses, so no
// restatement can reproduce it; this oracle fixes one: match i goes into partial sum i mod 128 (in match order), each
// group of 32 partials is combined by the pairwise butterfly (o = 16, 8, 4, 2, 1: v[l] + v[l ^ o]) and the 4 group totals
// are added left to right -- the order in which sim3_opt_kernels.cuh's 128 threads reduce.
constexpr int kLanes = 128;

double ordered_total(const std::vector<double> &part, int stride, int k) {
    double total = 0;
    for (int w = 0; w < kLanes / 32; ++w) {
        double v[32], nv[32];
        for (int l = 0; l < 32; ++l) v[l] = part[(size_t)(32 * w + l) * stride + k];
        for (int o = 16; o > 0; o >>= 1) {
            for (int l = 0; l < 32; ++l) nv[l] = v[l] + v[l ^ o];
            std::memcpy(v, nv, sizeof(v));
        }
        total = w == 0 ? v[0] : total + v[0];
    }
    return total;
}

// one mutual_reproj_edge_wapper: edge_12_ (forward, keyframe-1 camera) and edge_21_ (backward, keyframe-2 camera)
struct Mutual {
    double pc_2[3];         // rot_2w pos_w_2 + trans_2w (the forward edge's first line; the same every evaluation)
    double pc_1[3];         // rot_1w pos_w_1 + trans_1w (the backward edge's)
    double obs_1[2], obs_2[2];
    double info_1, info_2;  // information = inv_sigma_sq I
    int level = 0;          // both edges share it (set_as_outlier)
    double err_12[2] = {0, 0}, err_21[2] = {0, 0};  // _error as left by the last computeError()
    double chi2_12() const { return s3o_chi2(err_12, info_1); }
    double chi2_21() const { return s3o_chi2(err_21, info_2); }
};

struct Problem {
    double cam[4];
    int fix_scale = 0;
    double delta = 0;  // Huber delta: sqrt_chi_sq (float) as number_t
    s3o_sim3 est;
    std::vector<Mutual> edges;

    void compute_error(Mutual &m, const s3o_sim3 &S12) const {
        s3o_error(cam, S12, m.pc_2, m.obs_1, m.err_12);
        s3o_error(cam, s3o_inverse(S12), m.pc_1, m.obs_2, m.err_21);
    }
    void compute_active_errors(const std::vector<int> &active) {
        for (int i : active) compute_error(edges[i], est);
    }
    // robust chi2 of both edges of match i, as the kernel's trial pass adds it
    double robust_pair(const Mutual &m) const {
        double rho[3];
        g2o_lite::huber(m.chi2_12(), delta, rho);
        const double chi = rho[0];
        g2o_lite::huber(m.chi2_21(), delta, rho);
        return chi + rho[0];
    }
    double active_robust_chi2(const std::vector<int> &active) const {
        std::vector<double> part(kLanes, 0.0);
        for (int i : active) part[i % kLanes] += robust_pair(edges[i]);
        return ordered_total(part, 1, 0);
    }
    // BaseUnaryEdge::linearizeOplus for one edge: the vertex is pushed, oplus'ed by +-delta e_d and popped, per edge
    void jacobian(const Mutual &m, bool backward, double *J /*2 x 7*/) const {
        s3o_sim3 visited[14];
        for (int k = 0; k < 14; ++k) {
            visited[k] = s3o_perturbed(est, k, fix_scale);
            if (backward) visited[k] = s3o_inverse(visited[k]);
        }
        if (backward)
            s3o_numeric_jacobian(cam, visited, m.pc_1, m.obs_2, J);
        else
            s3o_numeric_jacobian(cam, visited, m.pc_2, m.obs_1, J);
    }
    // constructQuadraticForm with the Huber weight rho'(chi2): acc[0..27] += upper(J^T w J) row-wise, acc[28..34] -=
    // J^T w e, acc[35] += rho(chi2)
    static void add_edge(const double *J, const double *e, double info, double chi2, double delta, double *acc) {
        double rho[3];
        g2o_lite::huber(chi2, delta, rho);
        acc[35] += rho[0];
        const double ww = info * rho[1];
        int k = 0;
        for (int a = 0; a < 7; ++a) {
            const double wa = ww * J[a], wb = ww * J[7 + a];
            for (int c = a; c < 7; ++c) {
                acc[k] += wa * J[c] + wb * J[7 + c];
                ++k;
            }
            acc[28 + a] -= wa * e[0] + wb * e[1];
        }
    }
    // H (7 x 7), b and the robust chi2 of computeActiveErrors at the current estimate
    double build_system(const std::vector<int> &active, double *H /*49*/, double *b /*7*/) const {
        std::vector<double> part(kLanes * 36, 0.0);
        for (int i : active) {
            const Mutual &m = edges[i];
            double *acc = part.data() + 36 * (size_t)(i % kLanes);
            double J[14];
            jacobian(m, false, J);
            add_edge(J, m.err_12, m.info_1, m.chi2_12(), delta, acc);
            jacobian(m, true, J);
            add_edge(J, m.err_21, m.info_2, m.chi2_21(), delta, acc);
        }
        int k = 0;
        for (int a = 0; a < 7; ++a)
            for (int c = a; c < 7; ++c) {
                H[a * 7 + c] = H[c * 7 + a] = ordered_total(part, 36, k);
                ++k;
            }
        for (int a = 0; a < 7; ++a) b[a] = ordered_total(part, 36, 28 + a);
        return ordered_total(part, 36, 35);
    }

    // SparseOptimizer::optimize(iterations) with OptimizationAlgorithmLevenberg (pose_opt.cc's driver at dimension 7)
    void optimize(const std::vector<int> &active, int iterations) {
        double lambda = 0, ni = 2;
        for (int it = 0; it < iterations; ++it) {
            compute_active_errors(active);
            double H[49], b[7];
            double current_chi = build_system(active, H, b);  // activeRobustChi2, summed with the system
            double temp_chi = current_chi;
            if (it == 0) {  // computeLambdaInit
                double max_diag = 0;
                for (int j = 0; j < 7; ++j) max_diag = std::max(std::fabs(H[j * 7 + j]), max_diag);
                lambda = 1e-5 * max_diag;
                ni = 2;
            }
            double rho = 0;
            int qmax = 0;
            bool lambda_finite = true;
            do {
                const s3o_sim3 backup = est;  // push
                std::vector<double> Hl(H, H + 49);
                for (int j = 0; j < 7; ++j) Hl[j * 7 + j] += lambda;
                double x[7] = {0, 0, 0, 0, 0, 0, 0};
                const bool ok2 = g2o_lite::cholesky_solve(Hl, b, x, 7);
                est = s3o_oplus(est, x, fix_scale);  // zeroes x[6] when fix_scale: the scale below reads that
                compute_active_errors(active);
                temp_chi = active_robust_chi2(active);
                if (!ok2) temp_chi = std::numeric_limits<double>::max();
                rho = current_chi - temp_chi;
                double scale = 0;
                for (int j = 0; j < 7; ++j) scale += x[j] * (lambda * x[j] + b[j]);
                scale += 1e-3;
                rho /= scale;
                if (rho > 0 && std::isfinite(temp_chi)) {
                    double alpha = 1. - std::pow((2 * rho - 1), 3);
                    alpha = std::min(alpha, 2. / 3.);
                    const double scale_factor = std::max(1. / 3., alpha);
                    lambda *= scale_factor;
                    ni = 2;
                    current_chi = temp_chi;
                } else {
                    lambda *= ni;
                    ni *= 2;
                    est = backup;  // pop (the edge errors are NOT recomputed, as in g2o)
                    if (!std::isfinite(lambda)) {
                        lambda_finite = false;
                        break;
                    }
                }
                qmax++;
            } while (rho < 0 && qmax < 10);
            if (qmax == 10 || rho == 0 || !lambda_finite) break;  // Terminate
        }
    }
};

}  // namespace

extern "C" {

/* Sim3 algebra of sim3optmath.h for the tests; a Sim3 is 8 doubles (q w, x, y, z, t, s); rotations row-major. */
void orc_sim3o_exp(const double *u7, double *out) {
    const s3o_sim3 S = s3o_exp(u7);
    std::memcpy(out, &S, sizeof(S));
}
void orc_sim3o_from_Rts(const double *R, const double *t, double s, double *out) {
    const s3o_sim3 S = s3o_from_Rts(R, t, s);
    std::memcpy(out, &S, sizeof(S));
}
void orc_sim3o_rotation(const double *S, double *R) { s3o_quat_to_R(S, R); }
void orc_sim3o_mul(const double *a, const double *b, double *out) {
    s3o_sim3 A, B;
    std::memcpy(&A, a, sizeof(A));
    std::memcpy(&B, b, sizeof(B));
    const s3o_sim3 O = s3o_mul(A, B);
    std::memcpy(out, &O, sizeof(O));
}
void orc_sim3o_inverse(const double *a, double *out) {
    s3o_sim3 A;
    std::memcpy(&A, a, sizeof(A));
    const s3o_sim3 O = s3o_inverse(A);
    std::memcpy(out, &O, sizeof(O));
}
void orc_sim3o_map(const double *a, const double *x, double *out) {
    s3o_sim3 A;
    std::memcpy(&A, a, sizeof(A));
    s3o_map(A, x, out);
}
/* One edge at estimate S12 = (q, t, s): backward 0 is edge_12_ (pos_w of keyframe 2's landmark, keyframe-2 pose
 * (rot_kw, trans_kw)), 1 is edge_21_ (keyframe 1's).  e: 2; J: 2 x 7 row-major (linearizeOplus). */
void orc_sim3o_edge(int backward, const double *cam, const double *S12, const double *rot_kw, const double *trans_kw,
                    const double *pos_w, const double *obs, int fix_scale, double *e, double *J) {
    s3o_sim3 est;
    std::memcpy(&est, S12, sizeof(est));
    double pc[3];
    s3o_to_cam(rot_kw, trans_kw, pos_w, pc);
    s3o_error(cam, backward ? s3o_inverse(est) : est, pc, obs, e);
    s3o_sim3 visited[14];
    for (int k = 0; k < 14; ++k) {
        visited[k] = s3o_perturbed(est, k, fix_scale);
        if (backward) visited[k] = s3o_inverse(visited[k]);
    }
    s3o_numeric_jacobian(cam, visited, pc, obs, J);
}

/* transform_optimizer(fix_scale, num_iter).optimize(keyfrm_1, keyfrm_2, matches, Sim3_12, chi_sq) of P independent
 * problems, as plp_sim3_optimize (include/plpslam_b200.h).  cams: P x 4 (fx, fy, cx, cy); poses: P x 12 (rot row-major,
 * trans) per keyframe.  round1_inlier_out (optional, N) receives the flags after step 4 for every problem. */
void orc_sim3_optimize(int num_problems, const int32_t *match_offsets, const double *cams, const double *pose_1w,
                       const double *pose_2w, const double *rot_12_in, const double *trans_12_in, const double *scale_12_in,
                       const double *pos_w_1, const double *pos_w_2, const float *obs_1, const float *obs_2,
                       const float *inv_sigma_sq_1, const float *inv_sigma_sq_2, float chi_sq, int num_iter,
                       int fix_scale, int32_t *num_inliers_out, double *rot_12_out, double *trans_12_out,
                       double *scale_12_out, uint8_t *inlier_out, uint8_t *round1_inlier_out) {
    const float sqrt_chi_sq = std::sqrt(chi_sq);
    for (int p = 0; p < num_problems; ++p) {
        const int off = match_offsets[p], n = match_offsets[p + 1] - off;
        Problem P;
        std::memcpy(P.cam, cams + 4 * (size_t)p, sizeof(P.cam));
        P.fix_scale = fix_scale;
        P.delta = sqrt_chi_sq;
        P.est = s3o_from_Rts(rot_12_in + 9 * (size_t)p, trans_12_in + 3 * (size_t)p, scale_12_in[p]);
        const double *R1 = pose_1w + 12 * (size_t)p, *R2 = pose_2w + 12 * (size_t)p;
        // 2. one mutual edge per valid match
        P.edges.resize(n);
        for (int i = 0; i < n; ++i) {
            const size_t g = (size_t)off + i;
            Mutual &m = P.edges[i];
            s3o_to_cam(R2, R2 + 9, pos_w_2 + 3 * g, m.pc_2);
            s3o_to_cam(R1, R1 + 9, pos_w_1 + 3 * g, m.pc_1);
            m.obs_1[0] = obs_1[2 * g];
            m.obs_1[1] = obs_1[2 * g + 1];
            m.obs_2[0] = obs_2[2 * g];
            m.obs_2[1] = obs_2[2 * g + 1];
            m.info_1 = inv_sigma_sq_1[g];
            m.info_2 = inv_sigma_sq_2[g];
        }
        uint8_t *inl = inlier_out + off;
        for (int i = 0; i < n; ++i) inl[i] = 1;
        // 3. initializeOptimization(); optimize(5)
        std::vector<int> active;
        for (int i = 0; i < n; ++i) active.push_back(i);
        P.optimize(active, 5);
        // 4. outliers: either edge fails chi2 < chi_sq (the errors of the last evaluated estimate)
        int num_outliers = 0;
        for (int i = 0; i < n; ++i) {
            const Mutual &m = P.edges[i];
            if (m.chi2_12() < chi_sq && m.chi2_21() < chi_sq) continue;
            inl[i] = 0;
            P.edges[i].level = 1;
            ++num_outliers;
        }
        if (round1_inlier_out) std::memcpy(round1_inlier_out + off, inl, (size_t)n);
        if (n - num_outliers < 10) {  // return 0: the caller's Sim3 is untouched
            num_inliers_out[p] = 0;
            std::memcpy(rot_12_out + 9 * (size_t)p, rot_12_in + 9 * (size_t)p, 9 * sizeof(double));
            std::memcpy(trans_12_out + 3 * (size_t)p, trans_12_in + 3 * (size_t)p, 3 * sizeof(double));
            scale_12_out[p] = scale_12_in[p];
            continue;
        }
        // 5. initializeOptimization() (level-0 edges); optimize(num_iter)
        active.clear();
        for (int i = 0; i < n; ++i)
            if (P.edges[i].level == 0) active.push_back(i);
        P.optimize(active, num_iter);
        // 6. count inliers
        int num_inliers = 0;
        for (int i = 0; i < n; ++i) {
            const Mutual &m = P.edges[i];
            if (m.level != 0) continue;
            if (chi_sq < m.chi2_12() || chi_sq < m.chi2_21()) {
                inl[i] = 0;
                continue;
            }
            ++num_inliers;
        }
        // 7. the estimate
        num_inliers_out[p] = num_inliers;
        s3o_quat_to_R(P.est.q, rot_12_out + 9 * (size_t)p);
        std::memcpy(trans_12_out + 3 * (size_t)p, P.est.t, 3 * sizeof(double));
        scale_12_out[p] = P.est.s;
    }
}

}  // extern "C"
