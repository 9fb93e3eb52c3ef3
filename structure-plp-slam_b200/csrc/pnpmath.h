/* pnpmath.h -- EPnP of solve::pnp_solver (solve/pnp_solver.cc:183-866) in plain IEEE-754 double arithmetic (+, -, *, /,
 * sqrt only; no FMA, no library calls), so that a host build (-ffp-contract=off) and a device build (-fmad=false) return
 * bit-identical results.
 *
 * The reference calls Eigen five times; Eigen is not installed here, so each call is restated:
 *   - choose_control_points (:320-323): JacobiSVD of the symmetric 3 x 3 PW0^T PW0 -> cyclic Jacobi eigen-decomposition
 *     (ess_jacobi_eig, essmath.h); singular values = |eigenvalues| in descending order, ties broken by index.
 *   - compute_pose (:242-244): JacobiSVD of the 12 x 12 M^T M -> the same; row 11 - i of Ut is the eigenvector of the
 *     (i + 1)-th smallest singular value.
 *   - find_betas_approx_1/2/3 (:570-572, :604-606, :644-646): JacobiSVD(L_6xk).solve(Rho), the minimum-norm least-squares
 *     solution -> a one-sided (Hestenes) Jacobi SVD of the 6 x k matrix, singular values below sigma_max * k * eps
 *     dropped as Eigen's default threshold does (SVDBase::rank()).  Rank-deficient systems occur (coplanar samples).
 *   - estimate_R_and_t (:487-514): full 3 x 3 SVD of Abt with "change 1" (a negative determinant flips V's third
 *     column) -> one-sided Jacobi SVD; the third left singular vector is u0 x u1.  The result U diag(1, 1, d) V^T with
 *     det = +1 does not depend on that choice, so R is unique whenever rank(Abt) >= 2.
 *   - CC.inverse() (:347): the cofactor formula with the determinant taken along the first column, as Eigen's fixed-size
 *     3 x 3 inverse computes it.
 * These are the same mathematical objects as Eigen's up to the sign of each singular vector.  That sign is a convention,
 * and for PW0^T PW0 it is not invisible: choose_control_points puts control point i at c0 + k u_i, so flipping u_i
 * mirrors that control point, which changes M^T M and hence the EPnP estimate on noisy data (not on exact data).  This
 * restatement fixes the convention (pnp_sign_convention: each eigenvector's largest-magnitude component, the first on
 * ties, is positive); Eigen's JacobiSVD makes its own choice, so poses differ from the reference's Eigen path at noise
 * level, not by rounding.  The signs of M^T M's singular vectors, of the 6 x k and of the 3 x 3 SVDs do not reach the
 * pose (the betas and the determinant fix-up absorb them).  PARITY UNPINNED against Eigen (absent).
 *
 * Everything else is kept as written: qr_solve's Householder QR (without its function-local static buffers; note its
 * pivot scan never looks at the last row), 5 Gauss-Newton iterations, solve_for_sign on the first correspondence, the
 * reprojection error and its sum order, the float literals (1.0f - a[1] ..., 2.0f * dot(...)), fx = fy = 1, cx = cy = 0.
 * Sums over correspondences run in correspondence order (centroids, PW0^T PW0, M^T M, Abt, the reprojection error).
 *
 * ONE INTENDED DEVIATION: when qr_solve meets a zero column (eta == 0, :786-790) the reference returns without writing X,
 * so gauss_newton adds an uninitialised (or the previous iteration's) step; here X = 0.
 *
 * The library (nvcc -fmad=false), the oracle (g++ -ffp-contract=off) and the CPU emulators of tests/cta_emu compile
 * this one text, so the device and the oracle evaluate the same expressions.
 */
#ifndef PLP_PNPMATH_H
#define PLP_PNPMATH_H

#include "essmath.h"

#if defined(__CUDACC__)
#define PNP_HD __host__ __device__ __forceinline__
#define PNP_NOUNROLL _Pragma("unroll 1") /* keeps the device code's register footprint spill-free */
#else
#define PNP_HD static inline
#define PNP_NOUNROLL
#endif

#define PNP_DBL_EPSILON 2.220446049250313080847e-16
#define PNP_DBL_MIN 2.2250738585072013830902e-308

/* pnp_solver.h:166 */
#define PNP_FX 1.0f
#define PNP_FY 1.0f
#define PNP_CX 0.0f
#define PNP_CY 0.0f

/* The per-problem working set of the reference's pws_ / us_ / alphas_ / pcs_ / signs_ (caller-owned storage). */
struct pnp_work {
    double *pws;    /* 3 n */
    double *us;     /* 2 n */
    double *alphas; /* 4 n */
    double *pcs;    /* 3 n */
    int *signs;     /* n */
    int n;
};

/* add_correspondence (:204-228): a bearing with z == 0 is skipped silently */
PNP_HD void pnp_add_correspondence(pnp_work *w, const double *pos_w, const double *bearing) {
    if (bearing[2] == 0) return;
    const int i = w->n;
    w->pws[3 * i] = pos_w[0];
    w->pws[3 * i + 1] = pos_w[1];
    w->pws[3 * i + 2] = pos_w[2];
    w->us[2 * i] = bearing[0] / bearing[2];
    w->us[2 * i + 1] = bearing[1] / bearing[2];
    w->signs[i] = (0.0 < bearing[2]) ? 1 : -1;
    w->n = i + 1;
}

PNP_HD double pnp_dot(const double *v1, const double *v2) { return v1[0] * v2[0] + v1[1] * v2[1] + v1[2] * v2[2]; }

PNP_HD double pnp_dist2(const double *p1, const double *p2) {
    return (p1[0] - p2[0]) * (p1[0] - p2[0]) + (p1[1] - p2[1]) * (p1[1] - p2[1]) + (p1[2] - p2[2]) * (p1[2] - p2[2]);
}

/* Symmetric N x N a (row-major, destroyed) -> sv[k] = k-th largest |eigenvalue| (ties by index), row k of ut = its
 * eigenvector: JacobiSVD's singular values and U^T of a symmetric matrix. */
template <int N>
PNP_HD void pnp_sym_svd(double *a, double *ut, double *sv) {
    double v[N * N];
    ess_jacobi_eig<N>(a, v);
    int idx[N];
    double key[N];
    for (int k = 0; k < N; ++k) {
        idx[k] = k;
        key[k] = a[k * N + k] < 0.0 ? -a[k * N + k] : a[k * N + k];
    }
    PNP_NOUNROLL
    for (int i = 1; i < N; ++i)  // stable insertion sort, descending
        for (int j = i; j > 0 && key[idx[j - 1]] < key[idx[j]]; --j) {
            const int s = idx[j - 1];
            idx[j - 1] = idx[j];
            idx[j] = s;
        }
    PNP_NOUNROLL
    for (int k = 0; k < N; ++k) {
        sv[k] = key[idx[k]];
        for (int j = 0; j < N; ++j) ut[k * N + j] = v[j * N + idx[k]];
    }
}

/* One-sided (Hestenes) Jacobi on the R x C matrix w (row-major): on return the columns of w are sigma_k u_k and v (C x C,
 * row-major) holds the right singular vectors as columns.  Fixed pair order (p < q ascending); a pair is rotated when
 * |w_p . w_q| > 1e-15 sqrt(|w_p|^2 |w_q|^2); at most 30 sweeps, stopping after a sweep without rotations. */
template <int R, int C>
PNP_HD void pnp_onesided_jacobi(double *w, double *v) {
    for (int i = 0; i < C; ++i)
        for (int j = 0; j < C; ++j) v[i * C + j] = (i == j) ? 1.0 : 0.0;
    PNP_NOUNROLL
    for (int sweep = 0; sweep < 30; ++sweep) {
        int rotated = 0;
        PNP_NOUNROLL
        for (int p = 0; p < C; ++p) {
            PNP_NOUNROLL
            for (int q = p + 1; q < C; ++q) {
                double al = 0.0, be = 0.0, ga = 0.0;
                for (int r = 0; r < R; ++r) {
                    al = al + w[r * C + p] * w[r * C + p];
                    be = be + w[r * C + q] * w[r * C + q];
                    ga = ga + w[r * C + p] * w[r * C + q];
                }
                const double aga = ga < 0.0 ? -ga : ga;
                if (!(aga > 1e-15 * ESS_SQRT(al * be))) continue;
                const double zeta = (be - al) / (2.0 * ga);
                const double az = zeta < 0.0 ? -zeta : zeta;
                double t = 1.0 / (az + ESS_SQRT(zeta * zeta + 1.0));
                if (zeta < 0.0) t = -t;
                const double c = 1.0 / ESS_SQRT(t * t + 1.0);
                const double s = t * c;
                for (int r = 0; r < R; ++r) {
                    const double wp = w[r * C + p], wq = w[r * C + q];
                    w[r * C + p] = c * wp - s * wq;
                    w[r * C + q] = s * wp + c * wq;
                }
                for (int r = 0; r < C; ++r) {
                    const double vp = v[r * C + p], vq = v[r * C + q];
                    v[r * C + p] = c * vp - s * vq;
                    v[r * C + q] = s * vp + c * vq;
                }
                rotated = 1;
            }
        }
        if (!rotated) break;
    }
}

/* column norms of w (the singular values) and their order: descending, ties by index */
template <int R, int C>
PNP_HD void pnp_sigma_order(const double *w, double *sigma, int *idx) {
    for (int k = 0; k < C; ++k) {
        double s = 0.0;
        for (int r = 0; r < R; ++r) s = s + w[r * C + k] * w[r * C + k];
        sigma[k] = ESS_SQRT(s);
        idx[k] = k;
    }
    for (int i = 1; i < C; ++i)
        for (int j = i; j > 0 && sigma[idx[j - 1]] < sigma[idx[j]]; --j) {
            const int s = idx[j - 1];
            idx[j - 1] = idx[j];
            idx[j] = s;
        }
}

/* JacobiSVD<MatX_t>(L, ComputeFullU | ComputeFullV).solve(rho) for the 6 x K matrix L (row-major): the minimum-norm
 * least-squares x = sum_k v_k (u_k . rho) / sigma_k over the singular values >= max(sigma_max K eps, DBL_MIN)
 * (SVDBase::rank() and _solve_impl, in descending order of sigma). */
template <int K>
PNP_HD void pnp_min_norm_solve(const double *L, const double *rho, double *x) {
    double w[6 * K], v[K * K], sigma[K];
    int idx[K];
    for (int i = 0; i < 6 * K; ++i) w[i] = L[i];
    pnp_onesided_jacobi<6, K>(w, v);
    pnp_sigma_order<6, K>(w, sigma, idx);
    double thr = sigma[idx[0]] * (K * PNP_DBL_EPSILON);
    if (thr < PNP_DBL_MIN) thr = PNP_DBL_MIN;
    for (int k = 0; k < K; ++k) x[k] = 0.0;
    PNP_NOUNROLL
    for (int kk = 0; kk < K; ++kk) {
        const int k = idx[kk];
        if (sigma[k] < thr) break;
        double ub = 0.0;
        for (int r = 0; r < 6; ++r) ub = ub + (w[r * K + k] / sigma[k]) * rho[r];
        const double tmp = ub / sigma[k];
        for (int j = 0; j < K; ++j) x[j] = x[j] + v[j * K + k] * tmp;
    }
}

/* the sign convention of the control-point directions (see the file header): the component of largest magnitude of each
 * row of the N x N ut, the first one on ties, is made positive */
template <int N>
PNP_HD void pnp_sign_convention(double *ut) {
    for (int i = 0; i < N; ++i) {
        int jm = 0;
        double am = ut[i * N] < 0.0 ? -ut[i * N] : ut[i * N];
        for (int j = 1; j < N; ++j) {
            const double a = ut[i * N + j] < 0.0 ? -ut[i * N + j] : ut[i * N + j];
            if (am < a) {
                am = a;
                jm = j;
            }
        }
        if (ut[i * N + jm] < 0.0)
            for (int j = 0; j < N; ++j) ut[i * N + j] = -ut[i * N + j];
    }
}

/* choose_control_points (:292-333) and compute_barycentric_coordinates (:335-361) */
PNP_HD void pnp_control_points(pnp_work *w, double cws[4][3]) {
    const int n = w->n;
    cws[0][0] = cws[0][1] = cws[0][2] = 0;
    for (int i = 0; i < n; ++i)
        for (int j = 0; j < 3; ++j) cws[0][j] += w->pws[3 * i + j];
    for (int j = 0; j < 3; ++j) cws[0][j] /= (double)(unsigned)n;
    double a[9], ut[9], d[3];
    for (int k = 0; k < 9; ++k) a[k] = 0.0;
    for (int i = 0; i < n; ++i) {
        double p[3];
        for (int j = 0; j < 3; ++j) p[j] = w->pws[3 * i + j] - cws[0][j];
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) a[r * 3 + c] = a[r * 3 + c] + p[r] * p[c];
    }
    pnp_sym_svd<3>(a, ut, d);
    pnp_sign_convention<3>(ut);
    for (int i = 1; i < 4; ++i) {
        const double k = ESS_SQRT(d[i - 1] / (double)(unsigned)n);
        for (int j = 0; j < 3; ++j) cws[i][j] = cws[0][j] + k * ut[(i - 1) * 3 + j];
    }
    /* CC(i, j - 1) = cws[j][i] - cws[0][i]; CC.inverse() as Eigen's compute_inverse<.., 3> */
    double m[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 1; j < 4; ++j) m[i][j - 1] = cws[j][i] - cws[0][i];
    double cof[3][3];  // cof[i][j] = m(i1, j1) m(i2, j2) - m(i1, j2) m(i2, j1), i1 = (i + 1) % 3, ...
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
            cof[i][j] = m[i1][j1] * m[i2][j2] - m[i1][j2] * m[i2][j1];
        }
    const double det = cof[0][0] * m[0][0] + cof[1][0] * m[1][0] + cof[2][0] * m[2][0];
    const double invdet = 1.0 / det;
    double inv[3][3];
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) inv[r][c] = cof[c][r] * invdet;
    for (int i = 0; i < n; ++i) {
        const double *pi = w->pws + 3 * i;
        double *al = w->alphas + 4 * i;
        for (int j = 0; j < 3; ++j)
            al[1 + j] = inv[j][0] * (pi[0] - cws[0][0]) + inv[j][1] * (pi[1] - cws[0][1]) + inv[j][2] * (pi[2] - cws[0][2]);
        al[0] = 1.0f - al[1] - al[2] - al[3];
    }
}

/* fill_M (:363-375) row pair of correspondence i, element (row, col) */
PNP_HD double pnp_M(const pnp_work *w, int i, int row, int col) {
    const double a = w->alphas[4 * i + col / 3];
    const int c = col % 3;
    if (row == 0) return c == 0 ? a * PNP_FX : (c == 1 ? 0.0 : a * (PNP_CX - w->us[2 * i]));
    return c == 0 ? 0.0 : (c == 1 ? a * PNP_FY : a * (PNP_CY - w->us[2 * i + 1]));
}

/* (M^T M)(a, b) (:242): the sum over the rows 2 i, 2 i + 1 in correspondence order */
PNP_HD double pnp_mtm_entry(const pnp_work *w, int a, int b) {
    double s = 0.0;
    for (int i = 0; i < w->n; ++i) {
        s = s + pnp_M(w, i, 0, a) * pnp_M(w, i, 0, b);
        s = s + pnp_M(w, i, 1, a) * pnp_M(w, i, 1, b);
    }
    return s;
}

/* qr_solve (:748-866) on the 6 x 4 system A X = b (A row-major, both destroyed) */
PNP_HD void pnp_qr_solve(double *A, double *b, double *X) {
    const int nr = 6, nc = 4;
    double A1[4], A2[4];
    PNP_NOUNROLL
    for (int k = 0; k < nc; ++k) {
        double eta = A[k * nc + k] < 0.0 ? -A[k * nc + k] : A[k * nc + k];
        for (int i = k + 1; i < nr; ++i) {  // as written: rows k .. nr - 2
            const double e = A[(i - 1) * nc + k];
            const double elt = e < 0.0 ? -e : e;
            if (eta < elt) eta = elt;
        }
        if (eta == 0) {  // the reference returns leaving X unset; here X = 0 (see the file header)
            for (int j = 0; j < nc; ++j) X[j] = 0.0;
            return;
        }
        double sum = 0.0;
        const double inv_eta = 1.0 / eta;
        for (int i = k; i < nr; ++i) {
            A[i * nc + k] *= inv_eta;
            sum += A[i * nc + k] * A[i * nc + k];
        }
        double sigma = ESS_SQRT(sum);
        if (A[k * nc + k] < 0) sigma = -sigma;
        A[k * nc + k] += sigma;
        A1[k] = sigma * A[k * nc + k];
        A2[k] = -eta * sigma;
        for (int j = k + 1; j < nc; ++j) {
            double s = 0.0;
            for (int i = k; i < nr; i++) s += A[i * nc + k] * A[i * nc + j];
            const double tau = s / A1[k];
            for (int i = k; i < nr; ++i) A[i * nc + j] -= tau * A[i * nc + k];
        }
    }
    for (int j = 0; j < nc; ++j) {  // b <- Q^T b
        double tau = 0;
        for (int i = j; i < nr; i++) tau += A[i * nc + j] * b[i];
        tau /= A1[j];
        for (int i = j; i < nr; ++i) b[i] -= tau * A[i * nc + j];
    }
    X[nc - 1] = b[nc - 1] / A2[nc - 1];  // X = R^-1 b
    for (int i = nc - 2; i >= 0; --i) {
        double sum = 0;
        for (int j = i + 1; j < nc; ++j) sum += A[i * nc + j] * X[j];
        X[i] = (b[i] - sum) / A2[i];
    }
}

/* gauss_newton (:728-746) with compute_A_and_b_gauss_newton (:714-726) */
PNP_HD void pnp_gauss_newton(const double L[6][10], const double *Rho, double betas[4]) {
    PNP_NOUNROLL
    for (int k = 0; k < 5; ++k) {
        double A[24], B[6], X[4];
        for (int i = 0; i < 6; ++i) {
            const double *l = L[i];
            A[i * 4 + 0] = 2 * l[0] * betas[0] + l[1] * betas[1] + l[3] * betas[2] + l[6] * betas[3];
            A[i * 4 + 1] = l[1] * betas[0] + 2 * l[2] * betas[1] + l[4] * betas[2] + l[7] * betas[3];
            A[i * 4 + 2] = l[3] * betas[0] + l[4] * betas[1] + 2 * l[5] * betas[2] + l[8] * betas[3];
            A[i * 4 + 3] = l[6] * betas[0] + l[7] * betas[1] + l[8] * betas[2] + 2 * l[9] * betas[3];
            B[i] = Rho[i] - (l[0] * betas[0] * betas[0] + l[1] * betas[0] * betas[1] + l[2] * betas[1] * betas[1] +
                             l[3] * betas[0] * betas[2] + l[4] * betas[1] * betas[2] + l[5] * betas[2] * betas[2] +
                             l[6] * betas[0] * betas[3] + l[7] * betas[1] * betas[3] + l[8] * betas[2] * betas[3] +
                             l[9] * betas[3] * betas[3]);
        }
        pnp_qr_solve(A, B, X);
        for (int i = 0; i < 4; ++i) betas[i] += X[i];
    }
}

/* find_betas_approx_1 (:558-588): columns 0, 1, 3, 6 */
PNP_HD void pnp_betas_approx_1(const double L[6][10], const double *Rho, double *betas) {
    double l[24], b4[4];
    for (int i = 0; i < 6; ++i) {
        l[i * 4 + 0] = L[i][0];
        l[i * 4 + 1] = L[i][1];
        l[i * 4 + 2] = L[i][3];
        l[i * 4 + 3] = L[i][6];
    }
    pnp_min_norm_solve<4>(l, Rho, b4);
    if (b4[0] < 0) {
        betas[0] = ESS_SQRT(-b4[0]);
        betas[1] = -b4[1] / betas[0];
        betas[2] = -b4[2] / betas[0];
        betas[3] = -b4[3] / betas[0];
    } else {
        betas[0] = ESS_SQRT(b4[0]);
        betas[1] = b4[1] / betas[0];
        betas[2] = b4[2] / betas[0];
        betas[3] = b4[3] / betas[0];
    }
}

/* find_betas_approx_2 (:593-626): columns 0, 1, 2 */
PNP_HD void pnp_betas_approx_2(const double L[6][10], const double *Rho, double *betas) {
    double l[18], b3[3];
    for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 3; ++j) l[i * 3 + j] = L[i][j];
    pnp_min_norm_solve<3>(l, Rho, b3);
    if (b3[0] < 0) {
        betas[0] = ESS_SQRT(-b3[0]);
        betas[1] = (b3[2] < 0) ? ESS_SQRT(-b3[2]) : 0.0;
    } else {
        betas[0] = ESS_SQRT(b3[0]);
        betas[1] = (b3[2] > 0) ? ESS_SQRT(b3[2]) : 0.0;
    }
    if (b3[1] < 0) betas[0] = -betas[0];
    betas[2] = 0.0;
    betas[3] = 0.0;
}

/* find_betas_approx_3 (:631-665): columns 0 .. 4 */
PNP_HD void pnp_betas_approx_3(const double L[6][10], const double *Rho, double *betas) {
    double l[30], b5[5];
    for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 5; ++j) l[i * 5 + j] = L[i][j];
    pnp_min_norm_solve<5>(l, Rho, b5);
    if (b5[0] < 0) {
        betas[0] = ESS_SQRT(-b5[0]);
        betas[1] = (b5[2] < 0) ? ESS_SQRT(-b5[2]) : 0.0;
    } else {
        betas[0] = ESS_SQRT(b5[0]);
        betas[1] = (b5[2] > 0) ? ESS_SQRT(b5[2]) : 0.0;
    }
    if (b5[1] < 0) betas[0] = -betas[0];
    betas[2] = b5[3] / betas[0];
    betas[3] = 0.0;
}

/* estimate_R_and_t (:440-519) */
PNP_HD void pnp_estimate_R_and_t(const pnp_work *w, double R[3][3], double t[3]) {
    const int n = w->n;
    double pc0[3], pw0[3];
    pc0[0] = pc0[1] = pc0[2] = 0.0;
    pw0[0] = pw0[1] = pw0[2] = 0.0;
    for (int i = 0; i < n; ++i)
        for (int j = 0; j < 3; ++j) {
            pc0[j] += w->pcs[3 * i + j];
            pw0[j] += w->pws[3 * i + j];
        }
    for (int j = 0; j < 3; ++j) {
        pc0[j] /= (double)(unsigned)n;
        pw0[j] /= (double)(unsigned)n;
    }
    double abt[9];
    for (int k = 0; k < 9; ++k) abt[k] = 0.0;
    for (int i = 0; i < n; ++i) {
        const double *pc = w->pcs + 3 * i;
        const double *pw = w->pws + 3 * i;
        for (int j = 0; j < 3; ++j) {
            abt[j * 3 + 0] += (pc[j] - pc0[j]) * (pw[0] - pw0[0]);
            abt[j * 3 + 1] += (pc[j] - pc0[j]) * (pw[1] - pw0[1]);
            abt[j * 3 + 2] += (pc[j] - pc0[j]) * (pw[2] - pw0[2]);
        }
    }
    /* Abt = U S V^T: columns sigma_k u_k of abt, V, ordered by descending sigma; u2 = u0 x u1 */
    double v[9], sigma[3], U[3][3], V[3][3];
    int idx[3];
    pnp_onesided_jacobi<3, 3>(abt, v);
    pnp_sigma_order<3, 3>(abt, sigma, idx);
    for (int c = 0; c < 2; ++c)
        for (int r = 0; r < 3; ++r) U[r][c] = abt[r * 3 + idx[c]] / sigma[idx[c]];
    U[0][2] = U[1][0] * U[2][1] - U[2][0] * U[1][1];
    U[1][2] = U[2][0] * U[0][1] - U[0][0] * U[2][1];
    U[2][2] = U[0][0] * U[1][1] - U[1][0] * U[0][1];
    for (int c = 0; c < 3; ++c)
        for (int r = 0; r < 3; ++r) V[r][c] = v[r * 3 + idx[c]];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) R[i][j] = U[i][0] * V[j][0] + U[i][1] * V[j][1] + U[i][2] * V[j][2];
    const double det = R[0][0] * R[1][1] * R[2][2] + R[0][1] * R[1][2] * R[2][0] + R[0][2] * R[1][0] * R[2][1] -
                       R[0][2] * R[1][1] * R[2][0] - R[0][1] * R[1][0] * R[2][2] - R[0][0] * R[1][2] * R[2][1];
    if (det < 0) {  // change 1: flip V's third column, not R
        for (int r = 0; r < 3; ++r) V[r][2] = -V[r][2];
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) R[i][j] = U[i][0] * V[j][0] + U[i][1] * V[j][1] + U[i][2] * V[j][2];
    }
    t[0] = pc0[0] - pnp_dot(R[0], pw0);
    t[1] = pc0[1] - pnp_dot(R[1], pw0);
    t[2] = pc0[2] - pnp_dot(R[2], pw0);
}

/* reprojection_error (:420-438) */
PNP_HD double pnp_reprojection_error(const pnp_work *w, const double R[3][3], const double t[3]) {
    double sum2 = 0.0;
    for (int i = 0; i < w->n; ++i) {
        const double *pw = w->pws + 3 * i;
        const double Xc = pnp_dot(R[0], pw) + t[0];
        const double Yc = pnp_dot(R[1], pw) + t[1];
        const double inv_Zc = 1.0 / (pnp_dot(R[2], pw) + t[2]);
        const double ue = PNP_CX + PNP_FX * Xc * inv_Zc;
        const double ve = PNP_CY + PNP_FY * Yc * inv_Zc;
        const double u = w->us[2 * i], vv = w->us[2 * i + 1];
        sum2 += ESS_SQRT((u - ue) * (u - ue) + (vv - ve) * (vv - ve));
    }
    return sum2 / (double)(unsigned)w->n;
}

/* compute_R_and_t (:543-553) with compute_ccs (:377-394), compute_pcs (:396-408) and solve_for_sign (:521-541) */
PNP_HD double pnp_compute_R_and_t(pnp_work *w, const double *ut /*144*/, const double *betas, double R[3][3], double t[3]) {
    double ccs[4][3];
    for (int i = 0; i < 4; ++i) ccs[i][0] = ccs[i][1] = ccs[i][2] = 0.0;
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j)
            for (int k = 0; k < 3; ++k) ccs[j][k] += betas[i] * ut[(11 - i) * 12 + 3 * j + k];
    for (int i = 0; i < w->n; ++i) {
        const double *a = w->alphas + 4 * i;
        double *pc = w->pcs + 3 * i;
        for (int j = 0; j < 3; ++j) pc[j] = a[0] * ccs[0][j] + a[1] * ccs[1][j] + a[2] * ccs[2][j] + a[3] * ccs[3][j];
    }
    /* the reference reads pcs_[2] even without correspondences (uninitialised); here no flip then */
    if (w->n > 0 && ((w->pcs[2] < 0.0 && w->signs[0] > 0) || (w->pcs[2] > 0.0 && w->signs[0] < 0))) {
        for (int i = 0; i < w->n; ++i) {
            w->pcs[3 * i] = -w->pcs[3 * i];
            w->pcs[3 * i + 1] = -w->pcs[3 * i + 1];
            w->pcs[3 * i + 2] = -w->pcs[3 * i + 2];
        }
    }
    pnp_estimate_R_and_t(w, R, t);
    return pnp_reprojection_error(w, R, t);
}

/* compute_pose (:230-290) after choose_control_points / compute_barycentric_coordinates (pnp_control_points) and
 * M^T M (pnp_mtm_entry, row-major 144, destroyed): R (row-major 9), t; returns the chosen reprojection error */
PNP_HD double pnp_compute_pose_from_mtm(pnp_work *w, const double cws[4][3], double *mtm, double *R_out, double *t_out) {
    double ut[144], sv[12];
    pnp_sym_svd<12>(mtm, ut, sv);
    double L[6][10], Rho[6];
    double dv[4][6][3];  // compute_L_6x10 (:667-702)
    PNP_NOUNROLL
    for (int i = 0; i < 4; ++i) {
        int a = 0, b = 1;
        for (int j = 0; j < 6; ++j) {
            dv[i][j][0] = ut[(11 - i) * 12 + 3 * a] - ut[(11 - i) * 12 + 3 * b];
            dv[i][j][1] = ut[(11 - i) * 12 + 3 * a + 1] - ut[(11 - i) * 12 + 3 * b + 1];
            dv[i][j][2] = ut[(11 - i) * 12 + 3 * a + 2] - ut[(11 - i) * 12 + 3 * b + 2];
            ++b;
            if (b > 3) {
                ++a;
                b = a + 1;
            }
        }
    }
    PNP_NOUNROLL
    for (int i = 0; i < 6; ++i) {
        L[i][0] = pnp_dot(dv[0][i], dv[0][i]);
        L[i][1] = 2.0f * pnp_dot(dv[0][i], dv[1][i]);
        L[i][2] = pnp_dot(dv[1][i], dv[1][i]);
        L[i][3] = 2.0f * pnp_dot(dv[0][i], dv[2][i]);
        L[i][4] = 2.0f * pnp_dot(dv[1][i], dv[2][i]);
        L[i][5] = pnp_dot(dv[2][i], dv[2][i]);
        L[i][6] = 2.0f * pnp_dot(dv[0][i], dv[3][i]);
        L[i][7] = 2.0f * pnp_dot(dv[1][i], dv[3][i]);
        L[i][8] = 2.0f * pnp_dot(dv[2][i], dv[3][i]);
        L[i][9] = pnp_dot(dv[3][i], dv[3][i]);
    }
    Rho[0] = pnp_dist2(cws[0], cws[1]);  // compute_rho (:704-712)
    Rho[1] = pnp_dist2(cws[0], cws[2]);
    Rho[2] = pnp_dist2(cws[0], cws[3]);
    Rho[3] = pnp_dist2(cws[1], cws[2]);
    Rho[4] = pnp_dist2(cws[1], cws[3]);
    Rho[5] = pnp_dist2(cws[2], cws[3]);
    double Betas[4][4], rep_errors[4], Rs[4][3][3], ts[4][3];
    PNP_NOUNROLL
    for (int k = 1; k <= 3; ++k) {  // :255-265, approximations 1, 2, 3 in this order
        if (k == 1) pnp_betas_approx_1(L, Rho, Betas[k]);
        if (k == 2) pnp_betas_approx_2(L, Rho, Betas[k]);
        if (k == 3) pnp_betas_approx_3(L, Rho, Betas[k]);
        pnp_gauss_newton(L, Rho, Betas[k]);
        rep_errors[k] = pnp_compute_R_and_t(w, ut, Betas[k], Rs[k], ts[k]);
    }
    int N = 1;
    if (rep_errors[2] < rep_errors[1]) N = 2;
    if (rep_errors[3] < rep_errors[N]) N = 3;
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) R_out[r * 3 + c] = Rs[N][r][c];
    t_out[0] = ts[N][0];
    t_out[1] = ts[N][1];
    t_out[2] = ts[N][2];
    return rep_errors[N];
}

/* compute_pose (:230-290) in one thread */
PNP_HD double pnp_compute_pose(pnp_work *w, double *R, double *t) {
    double cws[4][3], mtm[144];
    pnp_control_points(w, cws);
    PNP_NOUNROLL
    for (int a = 0; a < 12; ++a)
        for (int b = 0; b < 12; ++b) mtm[a * 12 + b] = pnp_mtm_entry(w, a, b);
    return pnp_compute_pose_from_mtm(w, cws, mtm, R, t);
}

/* one correspondence of check_inliers (:155-181): cos = pos_c . bearing / |pos_c|, pos_c = R pos_w + t, the norm
 * sqrt((x^2 + y^2) + z^2); an inlier when the float max_cos_error is strictly below cos */
PNP_HD int pnp_is_inlier(const double *R, const double *t, const double *pos_w, const double *bearing, float max_cos_error) {
    double pc[3];
    for (int r = 0; r < 3; ++r) pc[r] = R[r * 3 + 0] * pos_w[0] + R[r * 3 + 1] * pos_w[1] + R[r * 3 + 2] * pos_w[2] + t[r];
    const double cosv = (pc[0] * bearing[0] + pc[1] * bearing[1] + pc[2] * bearing[2]) /
                        ESS_SQRT(pc[0] * pc[0] + pc[1] * pc[1] + pc[2] * pc[2]);
    return (double)max_cos_error < cosv ? 1 : 0;
}

/* util::converter::to_eigen_cam_pose(R, t), row-major 4 x 4 */
PNP_HD void pnp_cam_pose(const double *R, const double *t, double *pose) {
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) pose[r * 4 + c] = R[r * 3 + c];
        pose[r * 4 + 3] = t[r];
    }
    pose[12] = pose[13] = pose[14] = 0.0;
    pose[15] = 1.0;
}

#endif
