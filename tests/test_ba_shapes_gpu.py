"""Bundle adjustment on the graph shapes a real map produces, against the oracle with the criteria of tests/test_ba_gpu.py.

ba_data.make_ba_problem gives every landmark 3..9 observers drawn over all keyframes, so the problems of test_ba_gpu.py never
have a landmark with more than 9 edges, a landmark without a free observer or a keyframe without edges, and they sit at 5..20,
40 and 71 free keyframes.  The problems here prescribe the observation structure (ba_data.make_ba_shape_problem):
  * points with more than 32 edges: the second and later rounds of the lane = edge loop of ba_linearize_kernel, the edge
    strides of ba_update_kernel, CTA ranges under the one-round-per-32-edges cost model;
  * free degree up to the number of free keyframes: few landmarks per batch (LB = pool_cap / max_deg < 16: idle warps), the
    slot table and keyframe masks full, the pool bounded by shared memory on the dense path;
  * landmarks whose observers are all fixed (no pool entry), landmarks with two observations, a free keyframe without edges, a
    free keyframe that loses every edge to the outlier round;
  * 31 / 32 / 33 free keyframes around the switch between the shared-memory and the dense-in-HBM reduced system, and 37 / 48 /
    64 where the last 32-column block of the blocked Cholesky (ba_chol.cu) is 30 wide / exactly full / 0 wide plus the
    right-hand-side row.
Every case asserts that the shape it asked for is the shape it got.  Each runs once."""
import numpy as np
import pytest

import ba_data
from test_ba_gpu import _compare, _solve_gpu

pytestmark = pytest.mark.gpu

_BACKGROUND = dict(k=(3, 9))  # what make_ba_problem draws: enough ordinary landmarks to keep every keyframe well constrained


def _long_tracks_12_60():
    prob = ba_data.make_ba_shape_problem(
        101, 12, 60, stereo_frac=0.5,
        points=[dict(n=6, k=33), dict(n=6, k=64), dict(n=6, k=65, plane=True), dict(n=6, k="all"), dict(n=700, **_BACKGROUND)],
        lines=[dict(n=6, k=40), dict(n=120, **_BACKGROUND)])
    assert list(prob.shape["pt_deg"][:24:6]) == [33, 64, 65, 72] and (prob.shape["pt_free_deg"][18:24] == 12).all()
    assert (prob.shape["ln_deg"][:6] == 40).all() and len(prob.plane_edge_lm) == 6
    assert (prob.pt_edge_obs[:, 2] >= 0).any() and (prob.pt_edge_obs[:, 2] < 0).any()   # mixed mono / stereo edges
    return prob


def _all_32_free_see_200_points():
    # Points only.  With lines in this problem (4 seen by all 32 free keyframes + 100 ordinary ones) the ORACLE's own final
    # chi2 moves by 1.4e-6 relative when its finite-difference step changes from 1e-9 to 1.0000001e-9 (orc_debug_set_numeric_delta),
    # more than the 1e-6 the comparison allows, and the GPU differed from it by 1.5e-6 at two of the three CTA counts: that
    # shape is not reproducible in the reference itself.  Without lines every Jacobian is analytic and the probe moves nothing.
    prob = ba_data.make_ba_shape_problem(102, 32, 8, points=[dict(n=200, k="all", who="free"), dict(n=1200, **_BACKGROUND)])
    assert (prob.shape["pt_free_deg"][:200] == 32).all() and (prob.shape["pt_deg"][:200] == 32).all()
    return prob


@pytest.mark.parametrize("num_ctas", [0, 1, 132], ids=lambda c: f"ctas{c}")
@pytest.mark.parametrize("make", [_long_tracks_12_60, _all_32_free_see_200_points],
                         ids=["12free_60fixed_pt33_pt64_pt65_pt72_ln40", "32free_200pts_seen_by_all_32"])
def test_long_tracks_shared_memory_path(ctx, orc, plp, make, num_ctas):
    """num_ctas 0: the automatic grid; 1: one CTA walks every batch; 132: one CTA per SM of an H100, ranges of a few landmarks
    cut by the cost model (a point costs one round per 32 edges)."""
    prob = make()
    _compare(_solve_gpu(ctx, plp, prob, num_ctas=num_ctas), ba_data.oracle_local_ba(orc, prob), prob, orc=orc)


@pytest.mark.parametrize("n_free", [31, 32, 33, 37, 48, 64], ids=lambda n: f"{n}free")
def test_local_window_around_the_representation_switch(ctx, orc, plp, n_free):
    """<= 32 free keyframes: reduced system in shared memory; above: dense in HBM, 32 columns per Cholesky step.  6 n_free =
    198 (33: last block 6 wide), 222 (37: 30 wide), 288 (48: a multiple of 32 -- below the last block only the right-hand-side
    row is left), 384 (64: the same, twelve steps)."""
    n_kf = n_free + 6
    prob = ba_data.make_ba_shape_problem(200 + n_free, n_free, 6,
                                         points=[dict(n=8, k="all"), dict(n=8, k=33), dict(n=45 * n_kf, **_BACKGROUND)],
                                         lines=[dict(n=2, k=40 if n_kf >= 40 else "all"), dict(n=5 * n_kf, **_BACKGROUND)])
    assert (prob.shape["pt_deg"][:8] == n_kf).all() and (prob.shape["pt_free_deg"][:8] == n_free).all()
    assert (prob.shape["pt_deg"][8:16] == 33).all() and int((prob.kf_fixed == 0).sum()) == n_free
    _compare(_solve_gpu(ctx, plp, prob), ba_data.oracle_local_ba(orc, prob), prob, orc=orc)


def _seen_by_all_71(n_fixed, global_ba):
    prob = ba_data.make_ba_shape_problem(103, 71, n_fixed, global_ba=global_ba,
                                         points=[dict(n=100, k="all"), dict(n=2900, **_BACKGROUND)])
    n_kf = len(prob.kf_fixed)
    assert (prob.shape["pt_deg"][:100] == n_kf).all() and (prob.shape["pt_free_deg"][:100] == 71).all()
    return prob


def test_global_ba_71_free_100_points_seen_by_all(ctx, orc, plp):
    """The dense path (ba_linearize_kernel<true>, FP64 atomics) with max_deg = 71: the pool of (keyframe, landmark) blocks is
    bounded by shared memory alone, fewer than 16 landmarks fit a batch, and one landmark adds 71 * 72 / 2 blocks to S.
    One optimize(20); criteria of test_ba_gpu.test_global_ba for more than 32 keyframes (the try counts are not compared
    there: once converged, accept / reject hangs on the sign of a chi2 difference at rounding level)."""
    from plpslam_b200.ba import global_ba
    prob = _seen_by_all_71(0, True)
    assert prob.kf_fixed[0] == 1 and prob.kf_fixed.sum() == 1
    o = ba_data.oracle_global_ba(orc, prob, 20, True)
    g = global_ba(ctx, prob.struct(), (len(prob.kf_fixed), len(prob.pt_pos_w), 0, len(prob.pt_edge_kf), 0), 20, True)
    rel_pose = np.linalg.norm(g["kf_pose_cw"] - o.kf_pose_cw) / np.linalg.norm(o.kf_pose_cw)
    assert rel_pose < 1e-4, rel_pose
    rel_pts = np.linalg.norm(g["pt_pos_w"] - o.pt_pos_w, axis=1) / np.linalg.norm(o.pt_pos_w, axis=1)
    assert np.quantile(rel_pts, 0.999) < 1e-4
    assert g["iters_first"] >= 3 and o.iters_first > 2
    assert abs(g["final_chi2"] - o.final_chi2) <= 1e-5 * abs(o.final_chi2)


@pytest.mark.parametrize("num_ctas", [1, 132], ids=lambda c: f"ctas{c}")
def test_long_tracks_dense_path(ctx, orc, plp, num_ctas):
    """The same 71-keyframe tracks in a local window (4 fixed keyframes, two optimize() phases with the outlier round between
    them), where the number of CTAs can be chosen: 1 and one per SM."""
    prob = _seen_by_all_71(4, False)
    _compare(_solve_gpu(ctx, plp, prob, num_ctas=num_ctas), ba_data.oracle_local_ba(orc, prob), prob, orc=orc)


def _degenerate_corners(with_lines):
    # keyframe 9: free, no edge at all.  Points only: keyframe 8 (free) has every observation 100..200 px off, so all its
    # edges are outliers after optimize(5).  (With lines that keyframe is left alone: a line edge displaced at both ends can
    # still pass the chi2 test, and the lines it drags along are not reproducible in the oracle itself.)
    lines = [dict(n=5, k=3, who="fixed"), dict(n=3, k=2), dict(n=150, **_BACKGROUND)] if with_lines else ()
    prob = ba_data.make_ba_shape_problem(
        104, 10, 6, empty_free=(9,), outlier_free=() if with_lines else (8,), lines=lines,
        points=[dict(n=20, k=4, who="fixed"), dict(n=40, k=2), dict(n=20, k=5, who="one_free"), dict(n=500, **_BACKGROUND)])
    sh = prob.shape
    assert (sh["pt_free_deg"][:20] == 0).all() and (sh["pt_deg"][20:60] == 2).all() and (sh["pt_free_deg"][60:80] == 1).all()
    assert not with_lines or ((sh["ln_free_deg"][:5] == 0).all() and (sh["ln_deg"][5:8] == 2).all())
    assert sh["kf_deg"][9] == 0 and prob.kf_fixed[9] == 0 and sh["kf_deg"][8] > 100
    return prob


@pytest.mark.parametrize("with_lines", [False, True], ids=["points_outlier_keyframe", "points_lines"])
def test_landmarks_without_free_observers_two_observations_and_edgeless_keyframes(ctx, orc, plp, with_lines):
    """pn == 0 (a landmark that adds nothing to S but is still optimised), the minimum degree, a zero Hpp block (the step of
    that keyframe is g / lambda = 0) and a keyframe whose Hpp block becomes zero in the second optimize()."""
    prob = _degenerate_corners(with_lines)
    o = ba_data.oracle_local_ba(orc, prob)
    assert with_lines or o.pt_edge_outlier[prob.pt_edge_kf == 8].all(), "keyframe 8 keeps an edge"
    g = _solve_gpu(ctx, plp, prob)
    _compare(g, o, prob, orc=orc)
    assert np.allclose(g["kf_pose_cw"][9], prob.kf_pose_cw[9], atol=1e-12)   # no edge: the pose does not move
