"""CPU tests of the plane RANSAC restatement: estimate_plane_SVD against numpy's SVD (the object Eigen::JacobiSVD
computes), both RANSAC loops on synthetic plane clouds, and the reference's quirks."""

import numpy as np
import pytest

import plane_data


def _svd_fit(P):
    """planar_mapping_module.cc:735-771 with numpy's SVD in place of Eigen::JacobiSVD."""
    c = P.mean(0)
    U = np.linalg.svd((P - c).T, full_matrices=True)[0]
    n = U[:, 2] / np.linalg.norm(U[:, 2])
    d = -n @ c
    return np.append(n, d), abs(np.linalg.norm(P @ n + d) / len(P))


@pytest.mark.parametrize("seed", range(5))
def test_plane_fit_equals_svd_restatement(orc, seed):
    pts, _, truth, on_plane = plane_data.make_plane_cloud(seed, n=200, outlier_frac=0.0)
    for cnt in (3, 18, 200):
        idx = np.random.default_rng(seed).choice(200, cnt, replace=False).astype(np.int32)
        eq, res = orc.plane_fit(pts, idx)
        eq_s, res_s = _svd_fit(pts[idx])
        if eq[:3] @ eq_s[:3] < 0:
            eq_s = -eq_s
        assert np.abs(eq - eq_s).max() < 1e-9 and abs(res - res_s) < 1e-12
        assert abs(np.linalg.norm(eq[:3]) - 1) < 1e-15
    if truth[:3] @ eq[:3] < 0:
        truth = -truth
    assert np.abs(eq - truth).max() < 5e-3


@pytest.mark.parametrize("seed", range(4))
def test_plane_ransac_estimate_and_update(orc, seed):
    pts, valid, truth, on_plane = plane_data.make_plane_cloud(seed + 10, n=300)
    smp = plane_data.draw_plane_samples(seed, valid, 50, 18)
    st, eq, err, inl = orc.plane_ransac(pts, valid, smp, plane_data.CFG_ESTIMATE)
    assert st == 1 and err < 0.002
    assert np.all(inl[valid == 0] == 0)
    kept = inl.astype(bool)
    assert kept.sum() >= 18 and (kept & ~on_plane).sum() <= 0.05 * kept.sum()
    dist = np.abs(pts @ eq[:3] + eq[3]) / np.linalg.norm(eq[:3])
    assert np.all(dist[kept] < 0.02)
    # update mode: 80 % samples, no ratio gate, starts from the plane's stored error
    smp_u = plane_data.draw_plane_samples(seed + 1, valid, 20, int(np.ceil(0.8 * len(pts))))
    st2, eq2, err2, inl2 = orc.plane_ransac(pts, valid, smp_u, plane_data.CFG_UPDATE, eq, 0.01)
    assert st2 in (0, 1)        # may fail when no refit beats the stored error; never crashes
    if st2 == 1:
        assert inl2.sum() >= 18


def test_plane_ransac_failure_paths(orc):
    pts, valid, _, _ = plane_data.make_plane_cloud(3, n=60)
    smp = plane_data.draw_plane_samples(0, valid, 10, 18)
    # fewer landmarks than POINTS_PER_RANSAC: estimate -> false, update -> invalid (:428 / :602)
    assert orc.plane_ransac(pts[:10], None, smp % 10, plane_data.CFG_ESTIMATE)[0] == 0
    assert orc.plane_ransac(pts[:10], None, smp % 10, plane_data.CFG_UPDATE)[0] == 2
    # a scattered cloud never reaches the inlier ratio: not found, but the Plane object was still mutated (:466-467)
    rng = np.random.default_rng(1)
    cloud = rng.uniform(-1, 1, (80, 3))
    st, eq, err, inl = orc.plane_ransac(cloud, None, plane_data.draw_plane_samples(2, np.ones(80), 15, 18), plane_data.CFG_ESTIMATE)
    assert st == 0 and inl.sum() == 0 and abs(np.linalg.norm(eq[:3]) - 1) < 1e-12 and err > 0.002


@pytest.mark.parametrize("seed", range(6))
def test_plane_ransac_oracle_matches_python_restatement(orc, seed):
    """The C++ oracle's loop bookkeeping (best_error also fed by sample residuals, the Plane taking every sample fit, the
    final filter with the LAST equation) against a second implementation written from the reference text."""
    n = [300, 150, 500, 90, 260, 40][seed]
    pts, valid, _, _ = plane_data.make_plane_cloud(seed + 40, n=n, outlier_frac=[0.25, 0.1, 0.35, 0.2, 0.5, 0.1][seed])
    for cfg, size, e0 in ((plane_data.CFG_ESTIMATE, 18, 0.0), (plane_data.CFG_UPDATE, int(np.ceil(0.8 * n)), 0.01)):
        smp = plane_data.draw_plane_samples(seed, valid, 30, size)
        st, eq, err, inl = orc.plane_ransac(pts, valid, smp, cfg, (0, 0, 1, 0), e0)
        ps, peq, perr, pinl = plane_data.plane_ransac_python(pts, valid, smp, cfg, (0, 0, 1, 0), e0)
        assert st == ps
        assert np.array_equal(inl, pinl)
        if eq[:3] @ peq[:3] < 0:
            peq = -peq
        assert np.abs(eq - peq).max() < 1e-8 and abs(err - perr) < 1e-10
