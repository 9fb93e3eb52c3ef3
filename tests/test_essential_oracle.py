"""CPU tests of the solve::essential_solver restatement: the Jacobi-based eight-point solve against numpy's SVD (the
object Eigen::JacobiSVD computes in the reference), the epipolar geometry it must satisfy, and RANSAC behaviour."""

import numpy as np
import pytest

import ess_data


def _svd_compute_E21(b1, b2):
    """essential_solver.cc:123-160 with numpy's SVD in place of Eigen::JacobiSVD."""
    A = np.stack([np.concatenate([b2[i, 0] * b1[i], b2[i, 1] * b1[i], b2[i, 2] * b1[i]]) for i in range(len(b1))])
    v = np.linalg.svd(A, full_matrices=True)[2][8]
    U, lam, Vt = np.linalg.svd(v.reshape(3, 3))
    lam[2] = 0.0
    return U @ np.diag(lam) @ Vt


@pytest.mark.parametrize("seed", range(5))
def test_compute_E21_equals_svd_restatement(orc, seed):
    b1, b2, matches, E_true = ess_data.make_two_view(seed, n=60, outlier_frac=0.0, noise=0.0)
    for n in (8, 9, 25, 60):
        m = matches[:n]
        E = orc.essential_compute_E21(b1[m[:, 0]], b2[m[:, 1]])
        Es = _svd_compute_E21(b1[m[:, 0]], b2[m[:, 1]])
        if np.sum(E * Es) < 0:
            Es = -Es
        # A^T A squares the condition number of a minimal sample: agreement with the SVD of A is eps * cond(A)^2, far
        # below the 1-degree inlier threshold (0.01745) the hypotheses are scored with
        assert np.abs(E - Es).max() < (1e-5 if n == 8 else 1e-8)
        s = np.linalg.svd(E, compute_uv=False)
        assert s[2] < 1e-12 * s[0]                               # rank 2
        res = np.abs(np.einsum("ij,jk,ik->i", b2[m[:, 1]], E, b1[m[:, 0]]))
        assert res.max() < 1e-7                                  # noise-free data satisfy b2^T E b1 = 0
        Et = E_true / np.linalg.norm(E_true) * np.linalg.norm(E)
        assert min(np.abs(E - Et).max(), np.abs(E + Et).max()) < 1e-5


@pytest.mark.parametrize("seed", range(4))
def test_ransac_finds_the_inliers(orc, seed):
    b1, b2, matches, E_true = ess_data.make_two_view(seed + 10, n=400, outlier_frac=0.3)
    samples = ess_data.draw_samples(seed, len(matches), 50)      # robust.cc:232: find_via_ransac(50, false)
    valid, inl, E, score, scores = orc.essential_ransac(b1, b2, matches, samples, False)
    assert valid == 1 and score > 0 and score == float(scores.max())
    assert int(np.argmax(scores)) == int(np.nonzero(scores == scores.max())[0][0])
    # ground truth inliers by the same threshold on the true E
    r = np.abs(np.einsum("ij,jk,ik->i", b2[matches[:, 1]], E_true, b1[matches[:, 0]]))
    r /= np.linalg.norm(b1[matches[:, 0]] @ E_true.T, axis=1)
    truth = r < 0.0174524
    assert (inl.astype(bool) & truth).sum() > 0.5 * truth.sum()   # a minimal noisy sample, best of 50
    assert (inl.astype(bool) & ~truth).sum() < 0.15 * inl.sum()
    # recompute with all inliers keeps (most of) them and returns the refined score
    v2, inl2, E2, score2, _ = orc.essential_ransac(b1, b2, matches, samples, True)
    assert v2 == 1 and inl2.sum() >= 0.9 * inl.sum()


def test_ransac_degenerate_inputs(orc):
    b1, b2, matches, _ = ess_data.make_two_view(3, n=40)
    samples = np.zeros((3, 8), np.int32)
    valid, inl, E, score, _ = orc.essential_ransac(b1, b2, matches[:7], samples, False)   # < 8 matches (:45-49)
    assert valid == 0 and inl.sum() == 0 and score == 0.0
    # all-outlier matches: the solution is (almost surely) invalid or tiny, and never crashes
    rng = np.random.default_rng(0)
    bad = np.stack([rng.integers(0, 40, 40), rng.integers(0, 40, 40)], 1).astype(np.int32)
    valid, inl, _, _, _ = orc.essential_ransac(b1, b2, bad, ess_data.draw_samples(1, 40, 50), False)
    assert inl.sum() < 25
