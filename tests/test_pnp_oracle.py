"""CPU tests of the solve::pnp_solver restatement (oracle/pnp.cc on pnpmath.h): the textual identity of the two
pnpmath.h copies, ground-truth recovery on noise-free data, the numpy restatement (numpy's svd / lstsq / inv), OpenCV's
EPnP frozen in tests/golden/cv2_epnp.npz, the Eigen-replacing helpers, and find_via_ransac's wrapper rules."""
from pathlib import Path

import numpy as np
import pytest

import pnp_data as pd

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden" / "cv2_epnp.npz"


def test_pnpmath_copies_identical():
    a = (ROOT / "oracle" / "pnpmath.h").read_text()
    b = (ROOT / "structure-plp-slam_b200" / "csrc" / "pnpmath.h").read_text()
    assert a == b


@pytest.mark.parametrize("seed", range(4))
def test_noise_free_recovers_ground_truth(orc, seed):
    s = pd.make_scene(seed, 200, 0.0, noise_px=0.0)
    b, x = s["bearings"], s["pos_w"]
    # every non-minimal set (and the recompute over all points): exact up to rounding.  Tolerance 1e-9 on every entry of
    # R and t (scene units, depths 2-10): the solve goes through M^T M, whose conditioning squares that of M.
    for n in (6, 10, 50, 200):
        R, t, err, used = pd.oracle_compute_pose(orc, b[:n], x[:n])
        assert used == n and np.abs(R - s["R"]).max() < 1e-9 and np.abs(t - s["t"]).max() < 1e-9 and err < 1e-9
    # minimal hypotheses: EPnP with exactly four points has a four-dimensional null space and its beta approximations
    # miss the pose on more than half of the samples by the algorithm's nature (OpenCV's EPnP: 325 of 600 such samples
    # off by more than 1e-3 degrees, this restatement 342 of 600).  The others land within 1e-3 degrees (five
    # Gauss-Newton steps leave them ~1e-5 off); RANSAC then finds the whole inlier set and the recompute recovers the
    # truth.  Observed here: 11 to 15 of 30.
    samples = pd.draw_samples(seed, 200, 30)
    hits = 0
    for smp in samples:
        R, t, err, _ = pd.oracle_compute_pose(orc, b[smp], x[smp])
        if pd.rot_angle_deg(R, s["R"]) < 1e-3:
            hits += 1
            assert np.abs(R - s["R"]).max() < 1e-4 and np.abs(t - s["t"]).max() < 1e-3 and err < 1e-4
    assert hits >= 8
    off, bb, xx, mc, sm = pd.pack([s], [samples])
    valid, num, pose, flags = pd.oracle_ransac(orc, off, bb, xx, mc, sm)
    assert valid[0] == 1 and num[0] == 200 and flags.all()
    assert np.abs(pose[0][:3, :3] - s["R"]).max() < 1e-9 and np.abs(pose[0][:3, 3] - s["t"]).max() < 1e-9


@pytest.mark.parametrize("seed", range(3))
def test_against_numpy_restatement(orc, seed):
    """The numpy restatement (numpy's svd, lstsq and inv; the control-point sign convention of pnpmath.h) against the
    oracle on noisy scenes with outliers: each hypothesis' count and the winner's flags through numpy's inlier test, the
    first-best replay, and the recompute over the winner's inliers -- R, t and the reprojection error to 1e-9.  The
    minimal hypotheses themselves depend on the basis a solver picks for M^T M's four-dimensional null space, so they
    are compared through their inlier tests, not pose by pose."""
    for frac in (0.0, 0.5, 0.9):
        s = pd.make_scene(seed * 10 + int(frac * 10), 400, frac)
        samples = pd.draw_samples(seed, 400, 30)
        off, b, x, mc, sm = pd.pack([s], [samples])
        valid, num, pose, flags, hyp = pd.oracle_ransac(orc, off, b, x, mc, sm, with_hyp=True)
        counts = []
        for smp in samples:
            R, t, _, _ = pd.oracle_compute_pose(orc, s["bearings"][smp], s["pos_w"][smp])
            counts.append(int(pd.numpy_check_inliers(R, t, s["bearings"], s["pos_w"], s["max_cos"]).sum()))
        assert counts == list(hyp[0])
        best = int(np.argmax(counts)) if max(counts) > 0 else -1
        assert num[0] == (counts[best] if best >= 0 else 0) and valid[0] == int(num[0] > 10)
        if best >= 0:
            R, t, _, _ = pd.oracle_compute_pose(orc, s["bearings"][samples[best]], s["pos_w"][samples[best]])
            assert np.array_equal(flags, pd.numpy_check_inliers(R, t, s["bearings"], s["pos_w"], s["max_cos"]))
        if valid[0]:
            m = flags.astype(bool)
            Rn, tn, en = pd.numpy_compute_pose(s["bearings"][m], s["pos_w"][m])
            R, t, e, _ = pd.oracle_compute_pose(orc, s["bearings"][m], s["pos_w"][m])
            assert np.array_equal(R, pose[0][:3, :3]) and np.array_equal(t, pose[0][:3, 3])
            # observed: <= 3e-15 in R, 2e-14 in t, 1e-13 relative in the error
            assert np.abs(R - Rn).max() < 1e-9 and np.abs(t - tn).max() < 1e-9 and abs(e - en) < 1e-9 * en


@pytest.mark.parametrize("n", [6, 8, 12, 30, 300])
def test_non_minimal_sets_against_numpy(orc, n):
    """compute_pose over noisy non-minimal sets (a one-dimensional null space for n >= 6): R, t and the reprojection error
    of the oracle and the numpy restatement agree to 1e-9 (observed below that on every case here)."""
    rng = np.random.default_rng(n)
    for seed in range(20):
        s = pd.make_scene(100 + seed, 300, 0.0)
        i = rng.choice(300, n, replace=False)
        R, t, e, _ = pd.oracle_compute_pose(orc, s["bearings"][i], s["pos_w"][i])
        Rn, tn, en = pd.numpy_compute_pose(s["bearings"][i], s["pos_w"][i])
        assert np.abs(R - Rn).max() < 1e-9 and np.abs(t - tn).max() < 1e-9 and abs(e - en) < 1e-9 * en


def test_first_best_wins_ties(orc):
    """Two hypotheses with equal counts and disjoint inlier sets: the first in sample order wins, either way round; a
    mixed sample placed before them (fewer inliers) changes nothing."""
    s, sa, sb = pd.tie_scene(orc, 7)
    mixed = np.array([sa[0], sa[1], sb[0], sb[1]], np.int32)
    want = {}
    for name, smp in (("a", sa), ("b", sb)):
        R, t, _, _ = pd.oracle_compute_pose(orc, s["bearings"][smp], s["pos_w"][smp])
        want[name] = pd.numpy_check_inliers(R, t, s["bearings"], s["pos_w"], s["max_cos"])
    assert want["a"].sum() == want["b"].sum() == 20 and not (want["a"] & want["b"]).any()
    off, b, x, mc, _ = pd.pack([s], [np.zeros((1, 4), np.int32)])
    for order, first in (((sa, sb), "a"), ((sb, sa), "b"), ((mixed, sa, sb), "a"), ((mixed, sb, sa), "b")):
        sm = np.stack(order)[None]
        valid, num, _, flags, hyp = pd.oracle_ransac(orc, off, b, x, mc, sm, recompute=False, with_hyp=True)
        assert num[0] == 20 and valid[0] == 1 and list(hyp[0][-2:]) == [20, 20]
        assert np.array_equal(flags, want[first])
    assert hyp[0][0] < 20


def test_against_opencv_epnp(orc):
    """cv2.solvePnP(SOLVEPNP_EPNP, K = I) frozen by tools/gen_golden.py.  Observed differences on these noisy sets: up to
    0.10 degrees and 0.033 scene units (depths 2-10) at n <= 30, below 0.013 degrees / 0.002 at n >= 100; OpenCV's EPnP
    uses its own SVD and Gauss-Newton, so the estimates agree to the noise-driven spread, not to rounding."""
    g = np.load(GOLDEN)
    for i in range(6):
        R, t, _, _ = pd.oracle_compute_pose(orc, g[f"bearings_{i}"], g[f"pos_w_{i}"])
        n = len(g[f"bearings_{i}"])
        tol_r, tol_t = (0.2, 0.05) if n <= 30 else (0.03, 0.005)
        assert pd.rot_angle_deg(R, g[f"R_{i}"]) < tol_r and np.abs(t - g[f"t_{i}"]).max() < tol_t


@pytest.mark.parametrize("k", [3, 4, 5])
def test_min_norm_solve(orc, k):
    rng = np.random.default_rng(k)
    for rank in range(0, k + 1):
        L = rng.normal(size=(6, rank)) @ rng.normal(size=(rank, k)) if rank else np.zeros((6, k))
        rho = rng.normal(size=6)
        x = pd.oracle_min_norm_solve(orc, L, rho)
        xn = pd.numpy_min_norm_solve(L, rho)
        assert np.allclose(x, xn, atol=1e-10 * max(1.0, np.abs(xn).max()))
    L = rng.normal(size=(6, k))
    L[:, -1] = L[:, 0]                                  # coplanar-like: two equal columns
    rho = rng.normal(size=6)
    assert np.allclose(pd.oracle_min_norm_solve(orc, L, rho), pd.numpy_min_norm_solve(L, rho), atol=1e-10)


def test_estimate_R_and_t(orc):
    rng = np.random.default_rng(0)
    dets = set()
    for trial in range(40):
        pws = rng.normal(size=(8, 3))
        R0, t0 = pd.random_pose(rng)
        pcs = pws @ R0.T + t0 + rng.normal(size=(8, 3)) * (0.0 if trial % 2 else 0.3)
        if trial % 4 == 3:
            pcs = pcs * np.array([1, 1, -1])            # a reflection: SVD gives det(U V^T) < 0, change 1 applies
        R, t = orc_R = pd.oracle_estimate_R_and_t(orc, pcs, pws)
        Rn, tn = pd.numpy_estimate_R_and_t(pcs, pws)
        U, _, Vt = np.linalg.svd((pcs - pcs.mean(0)).T @ (pws - pws.mean(0)))
        dets.add(bool(np.linalg.det(U @ Vt) < 0))
        assert np.allclose(R, Rn, atol=1e-10) and np.allclose(t, tn, atol=1e-10)
        assert abs(np.linalg.det(R) - 1) < 1e-12
        del orc_R
    assert dets == {True, False}


def test_qr_solve(orc):
    rng = np.random.default_rng(1)
    for _ in range(20):
        A, b = rng.normal(size=(6, 4)), rng.normal(size=6)
        assert np.allclose(pd.oracle_qr_solve(orc, A, b), np.linalg.lstsq(A, b, rcond=None)[0], atol=1e-10)
    A = rng.normal(size=(6, 4))
    A[:5, 0] = 0.0                                      # eta == 0 (the pivot scan skips the last row): X = 0
    assert np.array_equal(pd.oracle_qr_solve(orc, A, rng.normal(size=6)), np.zeros(4))


def test_wrapper_rules(orc):
    s = pd.make_scene(5, 60, 0.3)
    samples = pd.draw_samples(5, 60, 30)
    off, b, x, mc, sm = pd.pack([s], [samples])
    num = pd.oracle_ransac(orc, off, b, x, mc, sm)[1]
    m = int(num[0])
    assert pd.oracle_ransac(orc, off, b, x, mc, sm, min_num_inliers=m)[0][0] == 0       # exactly min: invalid
    assert pd.oracle_ransac(orc, off, b, x, mc, sm, min_num_inliers=m - 1)[0][0] == 1   # one more: valid
    # the recompute keeps the RANSAC flags; only the pose changes
    a = pd.oracle_ransac(orc, off, b, x, mc, sm, recompute=True)
    c = pd.oracle_ransac(orc, off, b, x, mc, sm, recompute=False)
    assert np.array_equal(a[3], c[3]) and not np.array_equal(a[2], c[2])
    # num_iter = 0: invalid, no inliers, pose untouched
    z = pd.oracle_ransac(orc, off, b, x, mc, np.zeros((1, 0, 4), np.int32))
    assert z[0][0] == 0 and z[1][0] == 0 and not z[3].any() and np.isnan(z[2]).all()
    # the size gate (:76-80): n < 4 or n < min_num_inliers -> nothing but valid / num_inliers written
    g = pd.oracle_ransac(orc, off, b, x, mc, sm, min_num_inliers=61)
    assert g[0][0] == 0 and g[1][0] == 0 and (g[3] == 255).all() and np.isnan(g[2]).all()
    s3 = pd.make_scene(6, 3)
    off3, b3, x3, mc3, sm3 = pd.pack([s3], [pd.draw_samples(6, 3, 30)])
    g = pd.oracle_ransac(orc, off3, b3, x3, mc3, sm3, min_num_inliers=0)
    assert g[0][0] == 0 and (g[3] == 255).all()
