"""High-precision reference of ONE Levenberg-Marquardt try's linear algebra (TEST INFRASTRUCTURE): the reduced camera system
S = Hpp - sum_l W_l (Hll_l + lambda I)^-1 W_l^T, g = bp - sum_l W_l (Hll_l + lambda I)^-1 bl_l, formed in np.longdouble from
the FULL normal equations that tests/ba_numpy.py assembles edge by edge, and the checks a downloaded (S, g, dp, lambda) has to
pass.  Used on the GPU read-back (plp_ba_debug_try) and on the same kernels run by tests/cta_emu."""
from __future__ import annotations

import numpy as np

import ba_numpy as bn
import synth

CAM = (synth.FX, synth.FY, synth.CX, synth.CY, synth.BF)
LD = np.longdouble


def _inv_ld(A):
    """Inverse of a small symmetric positive definite matrix in long double (numpy's LAPACK calls stop at double)."""
    n = len(A)
    M = np.concatenate([A.astype(LD), np.eye(n, dtype=LD)], 1)
    for c in range(n):
        piv = c + int(np.argmax(np.abs(M[c:, c])))
        M[[c, piv]] = M[[piv, c]]
        M[c] /= M[c, c]
        for r in range(n):
            if r != c:
                M[r] -= M[r, c] * M[c]
    return M[:, n:]


def reference_try(prob, lam=None):
    """(S [6N x 6N, symmetric, WITHOUT lambda on its diagonal], g, bp, chi2, lambda_init) at the initial state with the Huber
    kernel on.  lam: the damping inside the Schur term (default: lambda_init = 1e-5 max diag H, computeLambdaInit)."""
    g = bn.Graph(prob, CAM)
    g.compute_errors()
    chi2 = g.robust_chi2()
    H, b, off_p, off_l, nf = g.build()
    lam_init = 1e-5 * float(np.abs(np.diag(H)).max())
    lam = LD(lam_init if lam is None else lam)
    n = 6 * nf
    S, gv = H[:n, :n].astype(LD), b[:n].astype(LD)
    for offs, d in ((off_p, 3), (off_l, 4)):
        for o in offs[offs >= 0]:
            rows = np.nonzero(np.abs(H[:n, o:o + d]).sum(1))[0]  # the free observers of this landmark
            Di = _inv_ld(H[o:o + d, o:o + d].astype(LD) + lam * np.eye(d, dtype=LD))
            if len(rows):
                W = H[rows, o:o + d].astype(LD)
                S[np.ix_(rows, rows)] -= W @ Di @ W.T
                gv[rows] -= W @ (Di @ b[o:o + d].astype(LD))
    return S, gv, b[:n].copy(), chi2, lam_init


def dense_from_blocks(S_blocks, n_free):
    """The upper 6 x 6 blocks (i, j), i <= j, row-wise -> the full symmetric matrix."""
    S = np.zeros((6 * n_free, 6 * n_free))
    q = 0
    for i in range(n_free):
        for j in range(i, n_free):
            S[6 * i:6 * i + 6, 6 * j:6 * j + 6] = S_blocks[q]
            if i != j:
                S[6 * j:6 * j + 6, 6 * i:6 * i + 6] = S_blocks[q].T
            q += 1
    return S


def backward_error(S, g, dp, lam):
    """|(S + lambda I) dp - g|_inf / (n (|S|_inf |dp|_inf + |g|_inf)), the residual in long double: how exactly dp solves the
    system it was computed from, whatever that system's conditioning."""
    n = len(g)
    A = S.astype(LD) + LD(lam) * np.eye(n, dtype=LD)
    r = A @ dp.astype(LD) - g.astype(LD)
    return float(np.abs(r).max() / (n * (np.abs(A).sum(1).max() * np.abs(dp).max() + np.abs(g).max())))


def check_system(got, prob, n_free, tol):
    """got: dict(S [n_pairs, 6, 6], g, bp, chi2, dp, lam).  tol: 1e-11 for problems whose Jacobians are all analytic (point
    edges only); line and plane edges are differentiated numerically (delta = 1e-9, ~1e-7 relative noise) by the kernels AND
    by the reference, which is what 1e-5 stands for.  Returns the observed (relative S error, relative g error)."""
    S_ref, g_ref, bp_ref, chi2_ref, lam_ref = reference_try(prob, got["lam"])
    # computeLambdaInit: 1e-5 max diag(H); the largest diagonal entry may belong to a numerically differentiated block
    assert abs(got["lam"] - lam_ref) <= max(1e-12, 1e-2 * tol) * lam_ref, (got["lam"], lam_ref)
    S = dense_from_blocks(got["S"], n_free)
    sS, sg = float(np.abs(S_ref).max()), float(np.abs(g_ref).max())
    err_blocks = np.abs(S - S_ref).astype(float).reshape(n_free, 6, n_free, 6).max(axis=(1, 3)) / sS
    assert err_blocks.max() <= tol, ("S block (i, j) =", np.unravel_index(err_blocks.argmax(), err_blocks.shape), err_blocks.max())
    err_g = float(np.abs(got["g"] - g_ref).max() / sg)
    assert err_g <= tol, err_g
    assert np.abs(got["bp"] - bp_ref).max() <= tol * max(np.abs(bp_ref).max(), 1e-300)
    assert abs(got["chi2"] - chi2_ref) <= 1e-12 * chi2_ref, (got["chi2"], chi2_ref)
    return float(err_blocks.max()), err_g
