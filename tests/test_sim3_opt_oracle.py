"""The Sim3 optimiser's oracle (oracle/transform_opt.cc + sim3optmath.h), pinned from independent directions because g2o
itself is not available: the Sim3 exponential against scipy's matrix exponential on both sides of every branch threshold,
the group operations against 4 x 4 similarity matrices, the numeric Jacobian against a numpy central difference, the
optimum against scipy.optimize.least_squares on the same robust cost, and the reference's control flow."""
from __future__ import annotations

from pathlib import Path

import numpy as np
import pytest
from scipy.linalg import expm
from scipy.optimize import least_squares
from scipy.spatial.transform import Rotation

import sim3_opt_data as sd

ROOT = Path(__file__).resolve().parents[1]


def generator(u):
    """4 x 4 sim(3) generator of update (omega, upsilon, sigma): [[Omega + sigma I, upsilon], [0, 0]]."""
    w, v, sg = u[:3], u[3:6], u[6]
    G = np.zeros((4, 4))
    G[:3, :3] = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]]) + sg * np.eye(3)
    G[:3, 3] = v
    return G


def test_math_header_copies_identical():
    a = (ROOT / "oracle" / "sim3optmath.h").read_bytes()
    b = (ROOT / "structure-plp-slam_b200" / "csrc" / "sim3optmath.h").read_bytes()
    assert a == b


# theta and sigma on both sides of g2o's eps = 1e-5 (and exactly zero)
THETAS = [0.0, 1e-8, 9.9e-6, 1.01e-5, 1e-3, 0.4, 2.5]
SIGMAS = [0.0, -1e-8, 9.9e-6, -1.01e-5, 1e-3, 0.3, -0.6]


@pytest.mark.parametrize("theta", THETAS)
@pytest.mark.parametrize("sigma", SIGMAS)
def test_exp_equals_matrix_exponential(orc, theta, sigma):
    rng = np.random.default_rng(int(theta * 1e6) + int(abs(sigma) * 1e7) + 3)
    axis = rng.normal(size=3)
    u = np.concatenate([axis / np.linalg.norm(axis) * theta, rng.normal(size=3), [sigma]])
    S = sd.oracle_exp(orc, u)
    want = expm(generator(u))
    got = sd.to_matrix(S)
    assert np.abs(got[:3, :3] - want[:3, :3]).max() < 1e-9
    # g2o's |sigma| < 1e-5 branches take C = 1 (and their A, B) at sigma = 0: a first-order truncation, so there the
    # translation is off by O(|sigma| |upsilon|); everywhere else it is the exponential's
    slack = abs(sigma) * np.linalg.norm(u[3:6]) if abs(sigma) < 1e-5 else 0.0
    assert np.abs(got[:3, 3] - want[:3, 3]).max() < 1e-9 + slack
    assert S[7] == np.exp(sigma) or abs(S[7] - np.exp(sigma)) < 1e-15


def random_sim3(orc, rng):
    return sd.oracle_exp(orc, np.concatenate([rng.normal(size=3) * 0.8, rng.normal(size=3), [rng.normal() * 0.4]]))


def test_group_operations_equal_similarity_matrices(orc):
    rng = np.random.default_rng(5)
    for _ in range(50):
        a, b = random_sim3(orc, rng), random_sim3(orc, rng)
        Ta, Tb = sd.to_matrix(a), sd.to_matrix(b)
        assert np.allclose(sd.to_matrix(sd.oracle_mul(orc, a, b)), Ta @ Tb, rtol=0, atol=1e-12)
        assert np.allclose(sd.to_matrix(sd.oracle_inverse(orc, a)), np.linalg.inv(Ta), rtol=0, atol=1e-12)
        x = rng.normal(size=3) * 5
        assert np.allclose(sd.oracle_map(orc, a, x), (Ta @ np.append(x, 1.0))[:3], rtol=0, atol=1e-12)
        R = sd.oracle_rotation(orc, a)
        # Sim3(R, t, s) round trip: a unit quaternion with w >= 0 and the same rotation
        b2 = sd.sim3(orc, R, a[4:7], a[7])
        assert b2[0] >= 0 and abs(np.linalg.norm(b2[:4]) - 1) < 1e-15
        assert np.allclose(sd.to_matrix(b2), Ta, rtol=0, atol=1e-13)


def _numpy_error(backward, T12, rot_kw, trans_kw, pos_w, obs):
    pc = rot_kw @ pos_w + trans_kw
    T = np.linalg.inv(T12) if backward else T12
    p = (T @ np.append(pc, 1.0))[:3]
    return obs - np.array([sd.FX * p[0] / p[2] + sd.CX, sd.FY * p[1] / p[2] + sd.CY])


@pytest.mark.parametrize("backward", [False, True])
@pytest.mark.parametrize("fix_scale", [False, True])
def test_numeric_jacobian_equals_numpy_central_difference(orc, backward, fix_scale):
    sc = sd.make_scene(11, 30)
    S = sd.sim3(orc, sc["R0"], sc["t0"], sc["s0"])
    T = sd.to_matrix(S)
    pose = sc["pose_1w"] if backward else sc["pose_2w"]
    R_kw, t_kw = pose[:9].reshape(3, 3), pose[9:]
    for i in range(len(sc["pos_w_1"])):
        pos_w = sc["pos_w_1" if backward else "pos_w_2"][i]
        obs = sc["obs_2" if backward else "obs_1"][i].astype(np.float64)
        e, J = sd.oracle_edge(orc, backward, S, R_kw, t_kw, pos_w, obs, fix_scale)
        assert np.allclose(e, _numpy_error(backward, T, R_kw, t_kw, pos_w, obs), rtol=0, atol=1e-9)
        want = np.zeros((2, 7))
        h = 1e-6
        for d in range(7):
            if fix_scale and d == 6:
                continue
            u = np.zeros(7)
            u[d] = h
            ep = _numpy_error(backward, expm(generator(u)) @ T, R_kw, t_kw, pos_w, obs)
            em = _numpy_error(backward, expm(generator(-u)) @ T, R_kw, t_kw, pos_w, obs)
            want[:, d] = (ep - em) / (2 * h)
        assert np.abs(J - want).max() <= 1e-4 * np.abs(want).max()
        if fix_scale:
            assert (J[:, 6] == 0).all()


def _noise_free(seed, fix_scale):
    sc = sd.make_scene(seed, 400, 0.0, noise_px=0.0, fix_scale=fix_scale)
    return sc, sd.pack([sc])


@pytest.mark.parametrize("fix_scale", [False, True])
def test_noise_free_scene_recovers_truth(orc, fix_scale):
    for seed in (21, 22, 23):
        sc, d = _noise_free(seed, fix_scale)
        num, rot, trans, scale, inl = sd.oracle_optimize(orc, d, fix_scale=fix_scale)
        assert num[0] == 400 and inl.all()
        # the observations are float (undist_keypts_): rounding the exact projections by up to 3e-5 px moves the optimum
        # by ~1e-8 from the truth (up to 5e-8 in translation and scale over depths of 3 - 12 m), not by 1e-9
        assert np.abs(rot[0] - sc["R"]).max() < 1e-8
        assert np.abs(trans[0] - sc["t"]).max() < 1e-7
        assert abs(scale[0] - sc["s"]) < 1e-7
        if fix_scale:
            assert scale[0] == d["scale"][0]


def test_fix_scale_keeps_input_scale_bits(orc):
    for name, sc, _ in sd.scenes(40):
        d = sd.pack([sc])
        d["scale"] = np.array([1.0 + 2.0 ** -40])  # a stereo map's Sim3 scale need not be exactly 1
        num, rot, trans, scale, inl = sd.oracle_optimize(orc, d, fix_scale=True)
        assert scale[0] == d["scale"][0], name


def _huber(e2, delta):
    return np.where(e2 <= delta * delta, e2, 2 * np.sqrt(e2) * delta - delta * delta)


def _robust_residuals(x, sc, active, fix_scale, s_fixed):
    R = Rotation.from_rotvec(x[:3]).as_matrix()
    s = s_fixed if fix_scale else np.exp(x[6])
    T = np.eye(4)
    T[:3, :3] = s * R
    T[:3, 3] = x[3:6]
    Ti = np.linalg.inv(T)
    P1, P2 = sc["pose_1w"], sc["pose_2w"]
    pc2 = sc["pos_w_2"][active] @ P2[:9].reshape(3, 3).T + P2[9:]
    pc1 = sc["pos_w_1"][active] @ P1[:9].reshape(3, 3).T + P1[9:]
    out = []
    delta = float(np.sqrt(np.float32(sd.CHI_SQ)).astype(np.float32))
    for pc, M, obs, w in ((pc2, T, sc["obs_1"][active], sc["w_1"][active]),
                          (pc1, Ti, sc["obs_2"][active], sc["w_2"][active])):
        p = pc @ M[:3, :3].T + M[:3, 3]
        e = obs.astype(np.float64) - np.stack([sd.FX * p[:, 0] / p[:, 2] + sd.CX, sd.FY * p[:, 1] / p[:, 2] + sd.CY], 1)
        e2 = np.sum(e * e, 1) * w.astype(np.float64)
        f = np.sqrt(_huber(e2, delta) / np.maximum(e2, 1e-300))
        out.append((e * np.sqrt(w.astype(np.float64))[:, None] * f[:, None]).reshape(-1))
    return np.concatenate(out)


@pytest.mark.parametrize("fix_scale", [False, True])
def test_many_iterations_reach_the_robust_least_squares_minimum(orc, fix_scale):
    sc = sd.make_scene(31 + fix_scale, 200, 0.15, noise_px=1.2, fix_scale=fix_scale)
    d = sd.pack([sc])
    num, rot, trans, scale, inl, r1 = sd.oracle_optimize(orc, d, fix_scale=fix_scale, num_iter=200, round1=True)
    assert num[0] >= 100
    active = r1.astype(bool)  # round 2 optimises over the round-1 survivors
    x0 = np.concatenate([Rotation.from_matrix(sc["R0"]).as_rotvec(), sc["t0"], [np.log(sc["s0"])]])
    fun = lambda x: _robust_residuals(np.append(x, 0.0) if fix_scale else x, sc, active, fix_scale, d["scale"][0])
    res = least_squares(fun, x0[:6] if fix_scale else x0, xtol=1e-15, ftol=1e-15, gtol=1e-15, max_nfev=2000)
    R_want = Rotation.from_rotvec(res.x[:3]).as_matrix()
    s_want = d["scale"][0] if fix_scale else np.exp(res.x[6])
    assert np.abs(rot[0] - R_want).max() <= 1e-6
    assert np.abs(trans[0] - res.x[3:6]).max() <= 1e-6 * max(1.0, np.abs(res.x[3:6]).max())
    assert abs(scale[0] - s_want) <= 1e-6 * s_want


def test_control_flow(orc):
    scs = sd.scenes(50)
    d = sd.pack([sc for _, sc, _ in scs])
    num, rot, trans, scale, inl, r1 = sd.oracle_optimize(orc, d, round1=True)
    names = [n for n, _, _ in scs]
    for p, name in enumerate(names):
        lo, hi = d["off"][p], d["off"][p + 1]
        f, f1 = inl[lo:hi], r1[lo:hi]
        assert set(np.unique(f)) <= {0, 1} and set(np.unique(f1)) <= {0, 1}
        assert not (f & ~f1).any()             # round 2 only adds outliers
        if name in ("few_survivors", "tiny", "empty"):
            assert f1.sum() < 10 and num[p] == 0
            assert np.array_equal(f, f1)       # the round-1 flags are what the caller sees
            assert rot[p].reshape(-1).tobytes() == d["rot"][p].tobytes()
            assert trans[p].tobytes() == d["trans"][p].tobytes() and scale[p] == d["scale"][p]
        else:
            assert num[p] == f.sum() >= 10
            assert not np.array_equal(rot[p].reshape(-1), d["rot"][p])
    # the round-1 rule counts survivors, not matches: a problem that starts with >= 10 matches can still return 0
    few = names.index("few_survivors")
    assert d["off"][few + 1] - d["off"][few] >= 10
    # the outlier flags follow the planted outliers on clean geometry
    mono = scs[names.index("mono")][1]
    lo = d["off"][names.index("mono")]
    assert np.array_equal(inl[lo:lo + len(mono["outlier"])] == 0, mono["outlier"])
