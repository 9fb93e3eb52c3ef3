/* essmath.h -- eight-point essential matrix and epipolar inlier test of solve::essential_solver
 * (solve/essential_solver.cc:123-160, 200-254) in plain IEEE-754 double / float arithmetic (+, -, *, /, sqrt only; no FMA,
 * no library calls), so that a host build (-ffp-contract=off) and a device build (-fmad=false) return bit-identical
 * results.
 *
 * The reference calls Eigen::JacobiSVD (3P; Eigen is not installed here) twice: the right singular vector of the n x 9
 * coefficient matrix A with the smallest singular value, then the rank-2 projection of the 3 x 3 estimate.  Restated as:
 *   - v = eigenvector of A^T A (9 x 9, symmetric) with the smallest eigenvalue, by cyclic Jacobi rotations;
 *   - E = U diag(s1, s2, 0) V^T = E0 - (E0 v3) v3^T with v3 = eigenvector of E0^T E0 with the smallest eigenvalue.
 * Both are the same mathematical objects as JacobiSVD's (up to the sign of v, which neither the inlier test nor the
 * score can see); they differ from Eigen's numbers by rounding only.  PARITY UNPINNED against Eigen (absent).
 *
 * The library (nvcc -fmad=false), the oracle (g++ -ffp-contract=off) and the CPU emulators of tests/cta_emu compile
 * this one text, so the device and the oracle evaluate the same expressions.
 */
#ifndef PLP_ESSMATH_H
#define PLP_ESSMATH_H

#if defined(__CUDACC__)
#define ESS_HD __host__ __device__ __forceinline__
#define ESS_SQRT(x) sqrt(x)
#else
#include <math.h>
#define ESS_HD static inline
#define ESS_SQRT(x) sqrt(x)
#endif

/* Cyclic Jacobi eigen-decomposition of the symmetric N x N matrix a (row-major, destroyed: its diagonal ends up holding
 * the eigenvalues); v (row-major) receives the eigenvectors as COLUMNS.  Fixed sweep order (p < q ascending), at most 30
 * sweeps; stops when the off-diagonal sum of squares is below 1e-30 x the diagonal sum of squares (relative off-norm
 * 1e-15) or below 1e-300. */
template <int N>
ESS_HD void ess_jacobi_eig(double *a, double *v) {
    for (int i = 0; i < N; ++i)
        for (int j = 0; j < N; ++j) v[i * N + j] = (i == j) ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 30; ++sweep) {
        double off = 0.0, diag = 0.0;
        for (int p = 0; p < N; ++p) {
            diag = diag + a[p * N + p] * a[p * N + p];
            for (int q = p + 1; q < N; ++q) off = off + a[p * N + q] * a[p * N + q];
        }
        if (!(off > 1e-300) || !(off > 1e-30 * diag)) break;
        for (int p = 0; p < N; ++p) {
            for (int q = p + 1; q < N; ++q) {
                const double apq = a[p * N + q];
                if (apq == 0.0) continue;
                const double theta = (a[q * N + q] - a[p * N + p]) / (2.0 * apq);
                const double at = theta < 0.0 ? -theta : theta;
                double t = 1.0 / (at + ESS_SQRT(theta * theta + 1.0));
                if (theta < 0.0) t = -t;
                const double c = 1.0 / ESS_SQRT(t * t + 1.0);
                const double s = t * c;
                /* A <- J^T A J on rows / columns p and q */
                for (int k = 0; k < N; ++k) {
                    const double akp = a[k * N + p], akq = a[k * N + q];
                    a[k * N + p] = c * akp - s * akq;
                    a[k * N + q] = s * akp + c * akq;
                }
                for (int k = 0; k < N; ++k) {
                    const double apk = a[p * N + k], aqk = a[q * N + k];
                    a[p * N + k] = c * apk - s * aqk;
                    a[q * N + k] = s * apk + c * aqk;
                }
                for (int k = 0; k < N; ++k) {
                    const double vkp = v[k * N + p], vkq = v[k * N + q];
                    v[k * N + p] = c * vkp - s * vkq;
                    v[k * N + q] = s * vkp + c * vkq;
                }
            }
        }
    }
}

/* accumulate one correspondence into the upper triangle of A^T A (essential_solver.cc:132-137: row = b2 (x) b1) */
ESS_HD void ess_accumulate(double *ata /*81*/, const double *b1, const double *b2) {
    double row[9];
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) row[3 * r + c] = b2[r] * b1[c];
    for (int i = 0; i < 9; ++i)
        for (int j = i; j < 9; ++j) ata[i * 9 + j] = ata[i * 9 + j] + row[i] * row[j];
}

/* essential_solver.cc:139-158 from the accumulated upper triangle; E_21 row-major */
ESS_HD void ess_solve(double *ata /*81, destroyed*/, double *E /*9*/) {
    double v[81];
    for (int i = 0; i < 9; ++i)
        for (int j = 0; j < i; ++j) ata[i * 9 + j] = ata[j * 9 + i];
    ess_jacobi_eig<9>(ata, v);
    int kmin = 0;
    for (int k = 1; k < 9; ++k)
        if (ata[k * 9 + k] < ata[kmin * 9 + kmin]) kmin = k;
    double E0[9];
    for (int i = 0; i < 9; ++i) E0[i] = v[i * 9 + kmin]; /* Mat33_t(v.data()).transpose(): E0(r, c) = v[3 r + c] */
    /* rank-2 projection: E = E0 - (E0 v3) v3^T, v3 = eigenvector of E0^T E0 with the smallest eigenvalue */
    double m[9], w[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) m[i * 3 + j] = E0[0 * 3 + i] * E0[0 * 3 + j] + E0[1 * 3 + i] * E0[1 * 3 + j] + E0[2 * 3 + i] * E0[2 * 3 + j];
    ess_jacobi_eig<3>(m, w);
    int k3 = 0;
    for (int k = 1; k < 3; ++k)
        if (m[k * 3 + k] < m[k3 * 3 + k3]) k3 = k;
    const double v3[3] = {w[0 * 3 + k3], w[1 * 3 + k3], w[2 * 3 + k3]};
    for (int r = 0; r < 3; ++r) {
        const double ev = E0[r * 3 + 0] * v3[0] + E0[r * 3 + 1] * v3[1] + E0[r * 3 + 2] * v3[2];
        for (int c = 0; c < 3; ++c) E[r * 3 + c] = E0[r * 3 + c] - ev * v3[c];
    }
}

/* essential_solver.cc:215-251 for one match: returns the inlier flag; *s2 / *s1 are the float residuals the reference
 * adds to the score in this order (s1 only when the first test passed; note that a match failing the SECOND test has
 * already contributed its first residual -- kept as written). */
ESS_HD int ess_check_match(const double *E21, const double *b1, const double *b2, float *s2, int *add1, float *s1) {
    const float residual_cos_thr = 0.01745240643f;
    *add1 = 0;
    *s1 = 0.0f;
    const double p0 = E21[0] * b1[0] + E21[1] * b1[1] + E21[2] * b1[2];
    const double p1 = E21[3] * b1[0] + E21[4] * b1[1] + E21[5] * b1[2];
    const double p2 = E21[6] * b1[0] + E21[7] * b1[1] + E21[8] * b1[2];
    const double d2 = (p0 * b2[0] + p1 * b2[1] + p2 * b2[2]) / ESS_SQRT(p0 * p0 + p1 * p1 + p2 * p2);
    const float r2 = (float)(d2 < 0.0 ? -d2 : d2);
    *s2 = r2;
    if (residual_cos_thr < r2) {
        *s2 = 0.0f;
        return 0;
    }
    /* E_12 = E_21^T */
    const double q0 = E21[0] * b2[0] + E21[3] * b2[1] + E21[6] * b2[2];
    const double q1 = E21[1] * b2[0] + E21[4] * b2[1] + E21[7] * b2[2];
    const double q2 = E21[2] * b2[0] + E21[5] * b2[1] + E21[8] * b2[2];
    const double d1 = (q0 * b1[0] + q1 * b1[1] + q2 * b1[2]) / ESS_SQRT(q0 * q0 + q1 * q1 + q2 * q2);
    const float r1 = (float)(d1 < 0.0 ? -d1 : d1);
    if (residual_cos_thr < r1) return 0;
    *add1 = 1;
    *s1 = r1;
    return 1;
}

#endif
