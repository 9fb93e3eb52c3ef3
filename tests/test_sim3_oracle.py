"""The Sim3 RANSAC oracle (oracle/sim3.cc on sim3math.h) against closed-form truths, independent rotation solvers and
the numpy restatement in tests/sim3_data.py, plus the reference's boundaries and sim3math.h's two deviations."""
from __future__ import annotations

from pathlib import Path

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import sim3_data as sd

ROOT = Path(__file__).resolve().parents[1]


def test_math_header_copies_are_identical():
    a = (ROOT / "oracle" / "sim3math.h").read_bytes()
    b = (ROOT / "structure-plp-slam_b200" / "csrc" / "sim3math.h").read_bytes()
    assert a == b


@pytest.mark.parametrize("fix_scale,scale", [(False, 2.0), (False, 0.5), (True, None)])
def test_noise_free_recovery(orc, fix_scale, scale):
    # powers of two: the float scales and their reciprocals are exact, so R, t and s are recovered to rounding
    for seed in range(20):
        sc = sd.make_scene(seed, 3, noise_px=0.0, fix_scale=fix_scale, scale=scale)
        R12, t12, s12, R21, t21, s21 = sd.oracle_compute(orc, sc["pts_1"], sc["pts_2"], fix_scale)
        assert s21 == np.float32(sc["s"]) and s12 == np.float32(1.0 / sc["s"])
        assert np.abs(R21 - sc["R"]).max() < 1e-9 and np.abs(R12 - sc["R"].T).max() < 1e-9
        assert np.abs(t21 - sc["t"]).max() < 1e-9
        assert np.abs(t12 - (-(1.0 / sc["s"]) * sc["R"].T @ sc["t"])).max() < 1e-9


def test_rotation_agrees_with_svd_and_scipy(orc):
    checked = 0
    for seed in range(200):
        sc = sd.make_scene(seed, 3, noise_px=2.0)
        p1, p2 = sc["pts_1"], sc["pts_2"]
        R21 = sd.oracle_compute(orc, p1, p2)[3]
        # Kabsch / Umeyama: maximise sum_i b_i . R a_i over the centred points
        A, B = p1 - p1.mean(0), p2 - p2.mean(0)
        U, S, Vt = np.linalg.svd(A.T @ B)
        d = np.sign(np.linalg.det(Vt.T @ U.T))
        if S[1] < 1e-6 * S[0]:
            continue
        R_svd = Vt.T @ np.diag([1.0, 1.0, d]) @ U.T
        R_sp = Rotation.align_vectors(B, A)[0].as_matrix()
        assert np.abs(R21 - R_svd).max() < 1e-9
        assert np.abs(R21 - R_sp).max() < 1e-9
        checked += 1
    assert checked > 150


@pytest.mark.parametrize("fix_scale", [False, True])
def test_hypotheses_equal_numpy_restatement(orc, fix_scale):
    sc = sd.make_scene(5, 300, 0.5, fix_scale=fix_scale)
    samples = sd.draw_samples(5, 300, 200)
    off, x1, x2, c1, c2, sm = sd.pack([sc], [samples])
    hyp = sd.oracle_ransac(orc, off, x1, x2, c1, c2, sm, fix_scale=fix_scale, with_hyp=True)[5][0]
    compared = exact_counts = 0
    for it, s in enumerate(samples):
        got = sd.oracle_compute(orc, x1[s], x2[s], fix_scale)
        want = sd.numpy_compute(x1[s], x2[s], fix_scale)
        if want[6] < 1e-6:       # degenerate: tied largest eigenvalues
            continue
        for g, w in zip(got[:6], want[:6]):
            assert np.abs(np.asarray(g, np.float64) - np.asarray(w, np.float64)).max() <= 1e-9 * max(1.0, np.abs(w).max())
        sure, possible = sd.numpy_inliers(want, sc, rtol=1e-6)
        assert sure.sum() <= hyp[it] <= possible.sum()
        exact_counts += sure.sum() == possible.sum()
        compared += 1
    assert compared > 190 and exact_counts > 190


def test_ransac_finds_the_scene(orc):
    for fix_scale in (False, True):
        sc = sd.make_scene(9, 400, 0.5, fix_scale=fix_scale)
        off, x1, x2, c1, c2, sm = sd.pack([sc], [sd.draw_samples(9, 400, 200)])
        valid, num, R12, t12, s12 = sd.oracle_ransac(orc, off, x1, x2, c1, c2, sm, fix_scale=fix_scale)
        assert valid[0] == 1 and num[0] >= 0.4 * 400
        assert np.degrees(np.arccos(np.clip((np.trace(R12[0] @ sc["R"]) - 1) / 2, -1, 1))) < 1.0
        assert abs(float(s12[0]) * sc["s"] - 1.0) < 0.05


def test_min_num_inliers_boundary(orc):
    sc = sd.make_scene(3, 120, 0.5)
    off, x1, x2, c1, c2, sm = sd.pack([sc], [sd.draw_samples(3, 120, 50)])
    best = int(sd.oracle_ransac(orc, off, x1, x2, c1, c2, sm, min_num_inliers=0)[1][0])
    at = sd.oracle_ransac(orc, off, x1, x2, c1, c2, sm, min_num_inliers=best)
    above = sd.oracle_ransac(orc, off, x1, x2, c1, c2, sm, min_num_inliers=best + 1)
    assert at[0][0] == 1 and at[1][0] == best and at[4][0] != 0      # max == min_num_inliers is valid (`>=`)
    assert above[0][0] == 0 and above[1][0] == best                   # one more is not: the reference's zeros
    assert not above[2].any() and not above[3].any() and above[4][0] == 0


def test_small_and_skipped_problems(orc):
    scenes = [sd.make_scene(1, 2, noise_px=0.0), sd.make_scene(2, 3, noise_px=0.0), sd.make_scene(3, 10, noise_px=0.0)]
    samples = [sd.draw_samples(1, 2, 5), np.tile([[0, 1, 2]], (5, 1)).astype(np.int32), sd.draw_samples(3, 10, 5)]
    off, x1, x2, c1, c2, sm = sd.pack(scenes, samples)
    valid, num, R, t, s = sd.oracle_ransac(orc, off, x1, x2, c1, c2, sm, min_num_inliers=3)
    assert list(valid) == [0, 1, 1] and list(num) == [0, 3, 10]     # n = 2 never runs; n = 3 is one exact sample
    assert not R[0].any() and not t[0].any() and s[0] == 0
    valid, num, R, t, s = sd.oracle_ransac(orc, off, x1, x2, c1, c2, sm, min_num_inliers=4)
    assert list(valid) == [0, 0, 1] and list(num) == [0, 0, 10]     # n < min_num_inliers: skipped
    assert not R[1].any() and s[1] == 0


def tie_scene(m=20):
    """Two noise-free groups of m points under two different Sim3s, and a sample of each group: two hypotheses with m
    inliers each and disjoint inlier sets."""
    a, b = sd.make_scene(41, m, noise_px=0.0, scale=2.0), sd.make_scene(42, m, noise_px=0.0, scale=0.5)
    return sd.concat(a, b), np.array([0, 1, 2], np.int32), np.array([m, m + 1, m + 2], np.int32)


def test_first_best_wins_ties(orc):
    sc, sa, sb = tie_scene()
    for first, second in ((sa, sb), (sb, sa)):
        off, x1, x2, c1, c2, sm = sd.pack([sc], [np.stack([first, second])])
        valid, num, R, t, s, hyp = sd.oracle_ransac(orc, off, x1, x2, c1, c2, sm, with_hyp=True)
        assert list(hyp[0]) == [20, 20] and valid[0] == 1
        assert s[0] == sd.oracle_compute(orc, x1[first], x2[first])[2]


def test_point_behind_the_same_image_is_never_an_inlier(orc):
    # t = 0: negating both points keeps every hypothesis' reprojection, so without the z check the pair would be an
    # inlier; its same-image reprojection is NaN instead
    sc = sd.make_scene(7, 30, noise_px=0.0, scale=2.0)
    sc["pts_2"] = sc["pts_2"] - sc["t"]
    sc["pts_1"][5] *= -1
    sc["pts_2"][5] *= -1
    off, x1, x2, c1, c2, sm = sd.pack([sc], [np.array([[0, 1, 2], [3, 4, 6]], np.int32)])
    hyp = sd.oracle_ransac(orc, off, x1, x2, c1, c2, sm, with_hyp=True)[5]
    assert list(hyp[0]) == [29, 29]


def test_point_behind_the_other_image_is_never_an_inlier(orc):
    # t = 0 and a 70 degree turn: keyframe-2 points far to one side lie behind keyframe 1.  For such a point X_2,
    # pts_1 = -inverse(X_2) is in front of keyframe 1 and reprojects onto the same pixels in both images, but each
    # other-image reprojection has z < 0 and is NaN
    rng = np.random.default_rng(3)
    R = sd.rotation(np.array([0.0, np.radians(70.0), 0.0]))
    s = 2.0
    u, v, z = rng.uniform(20, 620, 400), rng.uniform(20, 460, 400), rng.uniform(3, 12, 400)
    X2 = np.stack([(u - sd.CX) / sd.FX * z, (v - sd.CY) / sd.FY * z, z], 1)
    X1 = (X2 @ R) / s
    front, back = np.flatnonzero(X1[:, 2] > 0)[:30], np.flatnonzero(X1[:, 2] < 0)[:1]
    assert len(front) == 30 and len(back) == 1
    p1 = np.concatenate([X1[front], -X1[back]])
    p2 = np.concatenate([X2[front], X2[back]])
    sc = dict(pts_1=p1, pts_2=p2, chi_sq_1=sd.chi_sq(np.zeros(31, np.int32)), chi_sq_2=sd.chi_sq(np.zeros(31, np.int32)))
    off, x1, x2, c1, c2, sm = sd.pack([sc], [np.array([[0, 1, 2]], np.int32)])
    hyp = sd.oracle_ransac(orc, off, x1, x2, c1, c2, sm, with_hyp=True)[5]
    assert hyp[0][0] == 30
    model = sd.numpy_compute(p1[:3], p2[:3])
    e1, e2 = sd.numpy_errors(model, p1, p2)
    assert np.isnan(e1[30]) and np.isnan(e2[30])


def test_coincident_points(orc):
    p = np.tile([[0.25, -0.5, 4.0]], (3, 1))   # exact centroids: the centred points are 0
    q = np.tile([[0.125, 0.375, 5.0]], (3, 1))
    R12, t12, s12, R21, t21, s21 = sd.oracle_compute(orc, p, q)
    assert np.isnan(s21) and np.isnan(s12) and np.isnan(t21).all()    # denom = 0: numer / denom = 0 / 0
    # N = 0: every eigenvalue ties at 0 and the last in Jacobi's order wins, q = (0, 0, 0, 1): a half turn about z
    assert np.array_equal(R21, np.diag([-1.0, -1.0, 1.0]))
    R12, t12, s12, R21, t21, s21 = sd.oracle_compute(orc, p, q, fix_scale=True)
    assert s21 == 1 and s12 == 1 and np.array_equal(R21, np.diag([-1.0, -1.0, 1.0]))
    assert np.abs(t21 - (q[0] - R21 @ p[0])).max() < 1e-12
    # a sample of one repeated point (legal input) counts no inliers
    sc = sd.make_scene(8, 40, noise_px=0.0)
    off, x1, x2, c1, c2, sm = sd.pack([sc], [np.array([[4, 4, 4], [0, 1, 2]], np.int32)])
    hyp = sd.oracle_ransac(orc, off, x1, x2, c1, c2, sm, with_hyp=True)[5]
    assert list(hyp[0]) == [0, 40]
