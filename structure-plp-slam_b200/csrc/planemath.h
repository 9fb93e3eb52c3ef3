/* planemath.h -- least-squares plane through 3-D points as Planar_Mapping_module::estimate_plane_SVD computes it
 * (planar_mapping_module.cc:735-771), in plain IEEE-754 double arithmetic (+, -, *, /, sqrt only; no FMA, no library calls)
 * so that a host build (-ffp-contract=off) and a device build (-fmad=false) return bit-identical results.
 *
 * The reference takes U.col(2) of Eigen::JacobiSVD(centered 3 x n matrix) -- the left singular vector of the smallest
 * singular value = the eigenvector of the smallest eigenvalue of the 3 x 3 scatter matrix Xc Xc^T, which is what this
 * header computes with the cyclic Jacobi kernel of essmath.h.  Sums run in index order.  The SIGN of the normal is
 * arbitrary in both formulations (distances and residuals do not see it).  PARITY UNPINNED against Eigen (absent).
 *
 * The library (nvcc -fmad=false), the oracle (g++ -ffp-contract=off) and the CPU emulators of tests/cta_emu compile
 * this one text.
 */
#ifndef PLP_PLANEMATH_H
#define PLP_PLANEMATH_H
#include "essmath.h"

#if defined(__CUDACC__)
#define PLN_HDM __host__ __device__ __forceinline__
#else
#define PLN_HDM inline
#endif

/* Fit over the points selected by `sel`: sel.count() points, sel.at(k) = index of the k-th one (ascending call order).
 * eq = (a, b, c, d) with (a, b, c) normalised; returns the reference's "residual" = ||X^T n + d|| / count. */
template <class Sel>
ESS_HD double plane_fit(const double *pts, const Sel &sel, double *eq) {
    const int cnt = sel.count();
    double cx = 0.0, cy = 0.0, cz = 0.0;
    for (int k = 0; k < cnt; ++k) {
        const double *p = pts + 3 * (size_t)sel.at(k);
        cx = cx + p[0];
        cy = cy + p[1];
        cz = cz + p[2];
    }
    cx = cx / (double)cnt;
    cy = cy / (double)cnt;
    cz = cz / (double)cnt;
    double m[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, w[9];
    for (int k = 0; k < cnt; ++k) {
        const double *p = pts + 3 * (size_t)sel.at(k);
        const double x = p[0] - cx, y = p[1] - cy, z = p[2] - cz;
        m[0] = m[0] + x * x;
        m[1] = m[1] + x * y;
        m[2] = m[2] + x * z;
        m[4] = m[4] + y * y;
        m[5] = m[5] + y * z;
        m[8] = m[8] + z * z;
    }
    m[3] = m[1];
    m[6] = m[2];
    m[7] = m[5];
    ess_jacobi_eig<3>(m, w);
    int k3 = 0;
    for (int k = 1; k < 3; ++k)
        if (m[k * 3 + k] < m[k3 * 3 + k3]) k3 = k;
    double n0 = w[0 * 3 + k3], n1 = w[1 * 3 + k3], n2 = w[2 * 3 + k3];
    const double nn = ESS_SQRT(n0 * n0 + n1 * n1 + n2 * n2); /* .normalized() */
    n0 = n0 / nn;
    n1 = n1 / nn;
    n2 = n2 / nn;
    const double d = -(n0 * cx + n1 * cy + n2 * cz);
    double ss = 0.0;
    for (int k = 0; k < cnt; ++k) {
        const double *p = pts + 3 * (size_t)sel.at(k);
        const double v = (p[0] * n0 + p[1] * n1 + p[2] * n2) + d;
        ss = ss + v * v;
    }
    eq[0] = n0;
    eq[1] = n1;
    eq[2] = n2;
    eq[3] = d;
    const double r = ESS_SQRT(ss) / (double)cnt;
    return r < 0.0 ? -r : r;
}

/* Plane::calculate_distance (data/landmark_plane.cc:118-123) with _abs_n = ||n|| as set_equation stores it (:101-107) */
ESS_HD double plane_distance(const double *eq, const double *p) {
    const double abs_n = ESS_SQRT(eq[0] * eq[0] + eq[1] * eq[1] + eq[2] * eq[2]);
    const double dist = ((eq[0] * p[0] + eq[1] * p[1] + eq[2] * p[2]) + eq[3]) / abs_n;
    return dist < 0.0 ? -dist : dist;
}

struct PlaneSelIndices { /* an explicit index list (the RANSAC sample) */
    const int *idx;
    int n;
    PLN_HDM int count() const { return n; }
    PLN_HDM int at(int k) const { return idx[k]; }
};

#endif
