"""Pinning the optimiser oracle (oracle/local_ba.cc, oracle/pose_opt.cc, oracle/g2o_lite.hpp).

g2o -- the third-party library behind optimize::pose_optimizer and optimize::local_bundle_adjuster* -- is neither
vendored nor installed, so the C++ oracle cannot be compared with g2o itself.  It is pinned here from four independent
directions instead:
  (i)   tests/ba_numpy.py, a second restatement in another formulation (4x4 matrices, FULL normal equations solved in one
        piece, every Jacobian numeric), must be matched try for try: LM try counts, iteration counts, final state, flags;
  (ii)  every analytic Jacobian the reference ships (perspective_pose_opt_edge.cc:76-101, perspective_reproj_edge.cc:78-125)
        equals the finite difference of the residual through the vertex update (T <- Exp(delta) T, X <- X + delta);
  (iii) the optimum LM reaches equals the optimum scipy.optimize.least_squares finds for the same (Huber) cost;
  (iv)  the line landmarks: which of them move by how much when the only thing that changes is the numeric-Jacobian noise.
"""
import ctypes as C

import numpy as np
import pytest

import ba_data
import ba_numpy as bn
import synth

_P = C.c_void_p
CAM = (synth.FX, synth.FY, synth.CX, synth.CY, synth.BF)


def _dp(a):
    return np.ascontiguousarray(a, np.float64).ctypes.data_as(_P)


def _cam5(stereo):
    return np.array([synth.FX, synth.FY, synth.CX, synth.CY, synth.BF if stereo else -1.0])


def _rand_pose(rng):
    return bn.se3_exp(np.concatenate([rng.normal(0, 0.3, 3), rng.normal(0, 0.5, 3)]))


# ---------------------------------------------------------------------------------------------------------------------
# (ii) edge algebra: update conventions and analytic Jacobians
# ---------------------------------------------------------------------------------------------------------------------
def test_se3_oplus_is_left_multiplication_by_exp(orc):
    rng = np.random.default_rng(0)
    for _ in range(20):
        T = _rand_pose(rng)
        u = np.concatenate([rng.normal(0, 0.2, 3), rng.normal(0, 0.3, 3)]) * rng.choice([1.0, 1e-7])
        out = np.zeros(16)
        orc.lib.orc_debug_se3_oplus(_dp(T), _dp(u), out.ctypes.data_as(_P))
        assert np.allclose(out.reshape(4, 4), bn.pose_oplus(T, u), atol=1e-13)


def test_line_oplus_and_line_error_match_the_numpy_restatement(orc):
    rng = np.random.default_rng(1)
    for _ in range(20):
        P_, Q_ = rng.uniform(-2, 2, 3) + [0, 0, 6], rng.uniform(-2, 2, 3) + [0, 0, 6]
        L = synth.plucker_from_endpoints(P_[None], Q_[None])[0]
        v = rng.normal(0, 0.05, 4)
        out = np.zeros(6)
        orc.lib.orc_debug_line_oplus(_dp(L), _dp(v), out.ctypes.data_as(_P))
        assert np.allclose(out, bn.line_oplus(L, v), rtol=0, atol=1e-13)
        T = _rand_pose(rng) @ np.eye(4)
        T[:3, 3] *= 0.2
        obs = rng.uniform(50, 400, 4)
        e = np.zeros(2)
        orc.lib.orc_debug_line_error(_dp(_cam5(False)), _dp(T), _dp(L), _dp(obs), e.ctypes.data_as(_P))
        assert np.allclose(e, bn.line_residual(CAM, T, L, obs), rtol=1e-12, atol=1e-10)


@pytest.mark.parametrize("stereo", [False, True])
def test_analytic_point_jacobians_equal_finite_differences(orc, stereo):
    """perspective_pose_opt_edge.cc:76-101 / :142-173 and perspective_reproj_edge.cc:78-125 / :166-214 are d e / d delta for
    T <- Exp(delta) T (columns 0-2 rotation, 3-5 translation) and X <- X + delta, with e = obs - projection."""
    rng = np.random.default_rng(2)
    for _ in range(25):
        T = _rand_pose(rng)
        T[:3, 3] *= 0.3
        Xc = np.array([rng.uniform(-2, 2), rng.uniform(-1.5, 1.5), rng.uniform(2, 9)])
        X = T[:3, :3].T @ (Xc - T[:3, 3])
        obs = np.array([rng.uniform(0, 640), rng.uniform(0, 480), rng.uniform(0, 600) if stereo else -1.0])
        e, Jp, Jl = np.zeros(3), np.zeros(18), np.zeros(9)
        orc.lib.orc_debug_point_edge(_dp(_cam5(stereo)), _dp(T), _dp(X), _dp(obs), e.ctypes.data_as(_P),
                                     Jp.ctypes.data_as(_P), Jl.ctypes.data_as(_P))
        D = 3 if stereo else 2
        assert np.allclose(e[:D], bn.point_residual(CAM, T, X, obs), rtol=1e-12, atol=1e-10)
        fd_p = bn.numeric_jacobian(lambda u: bn.point_residual(CAM, bn.pose_oplus(T, u), X, obs), 6, delta=1e-6)
        fd_l = bn.numeric_jacobian(lambda u: bn.point_residual(CAM, T, X + u, obs), 3, delta=1e-6)
        assert np.allclose(Jp.reshape(3, 6)[:D], fd_p, rtol=2e-6, atol=2e-5)
        assert np.allclose(Jl.reshape(3, 3)[:D], fd_l, rtol=2e-6, atol=2e-5)
        # and the numpy transcription used by the restatement below is the same formula
        assert np.allclose(Jp.reshape(3, 6)[:D], bn.point_jac_pose_analytic(CAM, T, X, stereo), rtol=1e-12, atol=1e-10)
        assert np.allclose(Jl.reshape(3, 3)[:D], bn.point_jac_landmark_analytic(CAM, T, X, stereo), rtol=1e-12, atol=1e-10)


def _np_line_depth_positive(g, e):
    """reproj_edge_line3d_orthonormal.h:97-177 restated with numpy matrices."""
    fx, fy, cx, cy, _ = g.cam
    T, L, (sx, sy, ex, ey) = g.T[e["kf"]], g.L[e["lm"]], e["obs"]
    R, t = T[:3, :3], T[:3, 3]
    Kl = np.array([[fy, 0, 0], [0, fx, 0], [-fy * cx, -fx * cy, fx * fy]])
    l1, l2, l3 = Kl @ (R @ L[:3] + bn.skew(t) @ R @ L[3:])
    P = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1.0]]) @ T[:3]
    M = np.zeros((4, 4))
    M[:3, :3], M[:3, 3], M[3, :3] = bn.skew(L[:3]), L[3:], -L[3:]
    ok = True
    for (px, py) in ((sx, sy), (ex, ey)):
        xc = -(py - (l2 / l1) * px + (l3 / l2)) * ((l1 * l2) / (l1 * l1 + l2 * l2))
        yc = -(l1 / l2) * xc - (l3 / l2)
        y0 = py - (l2 / l1) * px
        plane = P.T @ np.cross([xc, yc, 1.0], [0.0, y0, 1.0])
        Xh = M @ plane
        ok = ok and 0 < (T[:3] @ np.append(Xh[:3] / Xh[3], 1.0))[2]
    return ok


def test_line_depth_test_matches_the_numpy_restatement(orc):
    prob = ba_data.make_ba_problem(5, n_local=4, n_fixed=2, n_points=30, n_lines=60, n_plane_pts=0)
    g = bn.Graph(prob, CAM)
    rng = np.random.default_rng(3)
    flips = 0
    for e in g.le:
        if rng.random() < 0.3:   # observations on the far side exercise the negative branch
            e["obs"] = e["obs"] + rng.normal(0, 400, 4)
        want = _np_line_depth_positive(g, e)
        got = orc.lib.orc_debug_line_depth_positive(_dp(_cam5(False)), _dp(g.T[e["kf"]]), _dp(g.L[e["lm"]]), _dp(e["obs"]))
        assert bool(got) == bool(want)
        flips += not want
    assert len(g.le) > 100


# ---------------------------------------------------------------------------------------------------------------------
# (i) try-for-try agreement with the full-system numpy restatement
# ---------------------------------------------------------------------------------------------------------------------
def _oracle_trace(orc):
    tr = np.zeros(3 * 400)
    n = orc.lib.orc_debug_lm_trace(tr.ctypes.data_as(_P), 400)
    return tr[:3 * n].reshape(n, 3)


def _compare(o, g, it1, it2, pt_out, ln_out, prob, tol=1e-7, trace=None, rho_tol=1e-5, lam_tol=1e-6):
    """Try for try: the lambda of every try, its gain ratio rho and the accept / reject decision agree until the solve has
    converged (|rho| < 1e-6: chi2 differences at round-off level, where the SIGN of rho -- and with it one more or one
    fewer try -- is decided by the summation order; g2o itself would differ from either restatement there)."""
    if trace is not None:
        conv = False
        for i, (a, b) in enumerate(zip(trace, g.trace)):
            if abs(a[1]) < 1e-6 or abs(b[1]) < 1e-6:
                conv = True
                break
            assert abs(a[0] - b[0]) <= lam_tol * abs(b[0]), (i, a, b)
            assert abs(a[1] - b[1]) <= rho_tol * max(1.0, abs(b[1])), (i, a, b)
            assert bool(a[2]) == bool(b[2]), (i, a, b)
        assert i >= 6, "the compared LM path is trivial"
        assert abs(len(trace) - len(g.trace)) <= (12 if conv else 0)  # <= 10 noise retries of one iteration
        if not conv:
            assert (o.iters_first, o.iters_second) == (it1, it2) and o.lm_tries == g.lm_tries
    else:
        assert (o.iters_first, o.iters_second) == (it1, it2)
        assert o.lm_tries == g.lm_tries
    Tn = np.stack(g.T)
    assert np.linalg.norm(Tn - o.kf_pose_cw.reshape(-1, 4, 4)) / np.linalg.norm(Tn) < tol
    assert np.abs(g.X - o.pt_pos_w).max() / np.abs(g.X).max() < tol
    assert np.array_equal(pt_out, o.pt_edge_outlier)
    if len(g.L):
        rel = np.linalg.norm(g.L - o.line_plucker, axis=1) / np.linalg.norm(g.L, axis=1)
        assert np.quantile(rel, 0.99) < 1e-4 and rel.max() < 1e-3, (np.quantile(rel, 0.99), rel.max())
        assert (ln_out != o.line_edge_outlier).sum() <= 1


@pytest.mark.parametrize("seed,stereo", [(0, False), (1, True), (2, False)])
def test_local_ba_points_matches_full_system_lm_try_for_try(orc, seed, stereo):
    """Points only: analytic Jacobians on both sides, so the two formulations (Schur complement with per-landmark block
    inverses vs one dense solve of the full system) must walk the same LM path to ~1e-9."""
    prob = ba_data.make_ba_problem(seed, n_local=5, n_fixed=3, n_points=120, n_lines=0, n_plane_pts=0, stereo=stereo,
                                   outlier_frac=0.08)
    o = ba_data.oracle_local_ba(orc, prob)
    trace = _oracle_trace(orc)
    g = bn.Graph(prob, CAM)
    it1, it2, pt_out, ln_out = g.local_ba()
    _compare(o, g, it1, it2, pt_out, ln_out, prob, trace=trace)


def test_local_ba_numeric_point_jacobians_give_the_same_path(orc):
    """The restatement with NUMERIC point Jacobians (central differences through the vertex updates, what g2o would do for
    an edge without linearizeOplus) still follows the oracle: the analytic formulas are the derivative of this residual
    under these update rules, not of something similar."""
    prob = ba_data.make_ba_problem(4, n_local=4, n_fixed=2, n_points=80, n_lines=0, n_plane_pts=0)
    o = ba_data.oracle_local_ba(orc, prob)
    trace = _oracle_trace(orc)
    g = bn.Graph(prob, CAM, numeric_point_jacobians=True)
    it1, it2, pt_out, ln_out = g.local_ba()
    _compare(o, g, it1, it2, pt_out, ln_out, prob, tol=1e-5, trace=trace, rho_tol=1e-3)


@pytest.mark.parametrize("seed", [0, 1])
def test_local_ba_points_lines_planes_matches_full_system_lm(orc, seed):
    prob = ba_data.make_ba_problem(20 + seed, n_local=5, n_fixed=3, n_points=100, n_lines=40, n_plane_pts=12)
    o = ba_data.oracle_local_ba(orc, prob)
    trace = _oracle_trace(orc)
    g = bn.Graph(prob, CAM)
    it1, it2, pt_out, ln_out = g.local_ba(line_depth_positive=_np_line_depth_positive)
    # numeric line Jacobians (delta = 1e-9) carry ~1e-7 relative noise that the lambda recursion (cubic in rho) amplifies:
    # decisions must still agree try for try, lambda to 1 %, rho to 5 %
    _compare(o, g, it1, it2, pt_out, ln_out, prob, tol=1e-5, trace=trace, rho_tol=5e-2, lam_tol=1e-2)


def test_local_ba_with_an_edgeless_keyframe_and_fixed_only_landmarks_matches_full_system_lm(orc):
    """Shapes make_ba_problem cannot draw: a free keyframe without a single edge (zero Hpp block: g2o leaves such a vertex
    out of the active set, here its step is 0 / lambda = 0), landmarks seen by fixed keyframes only, landmarks with two observations, points with 33 edges.  The oracle accepts them
    and walks the path of the full-system restatement."""
    prob = ba_data.make_ba_shape_problem(
        9, 5, 34, empty_free=(4,), outlier_frac=0.05,
        points=[dict(n=3, k=33), dict(n=6, k=4, who="fixed"), dict(n=8, k=2), dict(n=4, k=5, who="one_free"), dict(n=100, k=(3, 9))])
    assert prob.shape["kf_deg"][4] == 0 and (prob.shape["pt_free_deg"][3:9] == 0).all() and (prob.shape["pt_deg"][:3] == 33).all()
    o = ba_data.oracle_local_ba(orc, prob)
    trace = _oracle_trace(orc)
    assert np.allclose(o.kf_pose_cw.reshape(-1, 4, 4)[4], prob.kf_pose_cw[4], atol=1e-12)
    g = bn.Graph(prob, CAM)
    it1, it2, pt_out, ln_out = g.local_ba()
    _compare(o, g, it1, it2, pt_out, ln_out, prob, trace=trace)


def test_make_ba_problem_is_unchanged_by_the_shape_generator():
    """The problems the GPU parity tests and the benchmark were tuned on: one checksum over every field of one seed."""
    import hashlib
    prob = ba_data.make_ba_problem(42, n_local=6, n_fixed=3, n_points=200, n_lines=40, n_plane_pts=10, stereo=True)
    h = hashlib.sha256()
    for a in (prob.kf_pose_cw, prob.kf_fixed, prob.pt_pos_w, prob.pt_edge_kf, prob.pt_edge_lm, prob.pt_edge_obs,
              prob.pt_edge_inv_sigma_sq, prob.line_plucker, prob.line_edge_kf, prob.line_edge_lm, prob.line_edge_obs,
              prob.plane_edge_lm, prob.plane_edge_fn):
        h.update(np.ascontiguousarray(a).tobytes())
    assert h.hexdigest() == "fc4a0df26339f4dfd9333398fd24f86ba771e17dd16b5ece1e033f5a63fe542b"


# ---------------------------------------------------------------------------------------------------------------------
# (iii) the optimum equals scipy's for the same cost
# ---------------------------------------------------------------------------------------------------------------------
def test_pose_optimizer_huber_optimum_equals_scipy(orc, plp):
    """Trial 0 of pose_optimizer = Huber-robustified LM.  With enough iterations it must reach the minimiser of
    sum_e rho_huber(e^T Omega e) -- found independently by scipy's trust-region solver on the whitened edge norms."""
    from scipy.optimize import least_squares
    cam = plp.capi.make_camera(synth.FX, synth.FY, synth.CX, synth.CY, synth.COLS, synth.ROWS)
    for seed in (0, 1, 2):
        T_gt, T_init, pts, _ = synth.make_pose_opt_scene(seed, n_pts=150, n_lines=0, outlier_frac=0.1)
        T, _, _, _, iters = orc.pose_optimize(cam, T_init, pts, None, num_trials=1, num_each_iter=60)
        delta = float(np.sqrt(np.float32(5.99146)))

        def fun(xi):
            Tx = bn.pose_oplus(T, xi)
            Xc = pts["pos_w"] @ Tx[:3, :3].T + Tx[:3, 3]
            ex = pts["obs_x"] - (synth.FX * Xc[:, 0] / Xc[:, 2] + synth.CX)
            ey = pts["obs_y"] - (synth.FY * Xc[:, 1] / Xc[:, 2] + synth.CY)
            return np.sqrt(pts["inv_sigma_sq"] * (ex * ex + ey * ey))   # one scalar per edge: rho acts on e^T Omega e

        sol = least_squares(fun, np.zeros(6), loss="huber", f_scale=delta, xtol=1e-15, ftol=1e-15, gtol=1e-15)
        assert np.linalg.norm(sol.x) < 1e-6, (seed, sol.x)     # scipy cannot improve on the oracle's optimum
        assert 2 * sol.cost <= np.sum([bn.huber(v * v, delta)[0] for v in fun(np.zeros(6))]) + 1e-9


def test_local_ba_optimum_equals_scipy_on_a_noise_free_and_a_noisy_problem(orc):
    from scipy.optimize import least_squares
    for noise_free in (True, False):
        prob = ba_data.make_ba_problem(31, n_local=3, n_fixed=3, n_points=40, n_lines=0, n_plane_pts=0, outlier_frac=0.0)
        if noise_free:   # observations = exact projections of the ground truth
            T, X = prob.gt["poses"], prob.gt["points"]
            Xc = np.einsum("eij,ej->ei", T[prob.pt_edge_kf, :3, :3], X[prob.pt_edge_lm]) + T[prob.pt_edge_kf, :3, 3]
            prob.pt_edge_obs[:, 0] = synth.FX * Xc[:, 0] / Xc[:, 2] + synth.CX
            prob.pt_edge_obs[:, 1] = synth.FY * Xc[:, 1] / Xc[:, 2] + synth.CY
        o = ba_data.oracle_local_ba(orc, prob, num_first=60, num_second=0)
        free = np.nonzero(prob.kf_fixed == 0)[0]
        T0, X0 = o.kf_pose_cw.reshape(-1, 4, 4), o.pt_pos_w
        delta = float(np.sqrt(np.float32(5.99146)))

        def fun(p):
            T = T0.copy()
            for i, k in enumerate(free):
                T[k] = bn.pose_oplus(T0[k], p[6 * i:6 * i + 6])
            X = X0 + p[6 * len(free):].reshape(-1, 3)
            Xc = np.einsum("eij,ej->ei", T[prob.pt_edge_kf, :3, :3], X[prob.pt_edge_lm]) + T[prob.pt_edge_kf, :3, 3]
            ex = prob.pt_edge_obs[:, 0] - (synth.FX * Xc[:, 0] / Xc[:, 2] + synth.CX)
            ey = prob.pt_edge_obs[:, 1] - (synth.FY * Xc[:, 1] / Xc[:, 2] + synth.CY)
            if noise_free:
                return np.concatenate([ex, ey]) * np.sqrt(np.tile(prob.pt_edge_inv_sigma_sq, 2))
            return np.sqrt(prob.pt_edge_inv_sigma_sq * (ex * ex + ey * ey))

        n = 6 * len(free) + 3 * len(X0)
        sol = least_squares(fun, np.zeros(n), loss="linear" if noise_free else "huber", f_scale=delta, xtol=1e-15,
                            ftol=1e-15, gtol=1e-15)
        assert np.abs(sol.x).max() < 1e-6, (noise_free, np.abs(sol.x).max())
        if noise_free:   # and that optimum is the ground truth
            assert np.abs(X0 - prob.gt["points"]).max() < 1e-6
            assert np.abs(T0 - prob.gt["poses"]).max() < 1e-6


# ---------------------------------------------------------------------------------------------------------------------
# (iv) line landmarks under numeric-Jacobian noise
# ---------------------------------------------------------------------------------------------------------------------
def test_line_result_sensitivity_to_numeric_jacobian_noise(orc):
    """Line edges have no linearizeOplus in the reference: g2o differentiates them with delta = 1e-9, i.e. ~1e-7 relative
    Jacobian noise.  Two evaluations of the SAME mathematics (the C++ oracle and the numpy restatement, different
    operation order) agree to 1e-4 -- north_star's tolerance -- on every line landmark that keeps at least two inlier
    observations.  A line whose observations are ALL classified as outliers is not part of the second optimize() at all
    (its vertex keeps whatever the 5 robust iterations left) and the reference erases those observations right after the
    solve (local_bundle_adjuster_extended_line.cc:560-640): such lines are excluded, and counted."""
    n_excluded = 0
    for seed in (25, 26):
        prob = ba_data.make_ba_problem(seed, n_local=5, n_fixed=3, n_points=100, n_lines=60, n_plane_pts=0)
        o = ba_data.oracle_local_ba(orc, prob)
        g = bn.Graph(prob, CAM)
        g.local_ba(line_depth_positive=_np_line_depth_positive)
        rel = np.linalg.norm(g.L - o.line_plucker, axis=1) / np.linalg.norm(g.L, axis=1)
        inl = np.bincount(prob.line_edge_lm, weights=1.0 - o.line_edge_outlier, minlength=len(g.L))
        kept = inl >= 2
        n_excluded += int((~kept).sum())
        assert rel[kept].max() < 1e-4, (seed, rel[kept].max())
        assert kept.sum() >= 0.8 * len(rel)
    assert n_excluded >= 1   # the case exists in these problems: the exclusion rule is exercised
