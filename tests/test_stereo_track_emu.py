"""The stereo rows of the batched tracker's DEVICE code executed on the CPU through tests/cta_emu, equal to the oracle:
the shared motion_assumption (match_common.cuh) against the oracle's match_current_and_last_frames, the shared tail's
gather (track_common.cuh) with the current frames' x_right, and the local-map stage (local_map_kernels.cuh) with
x_right_in_tracking_ and the matcher's x_right gate.  Observations are compared with the arrays pose_optimizer.cc:126-151
builds: x_right >= 0 is a stereo edge (0 included), < 0 a 2-D edge."""
import ctypes as C
import shutil
import subprocess

import numpy as np
import pytest

import local_map_data as lmd
import oracle_api
import scene
import stereo_track_data as std
import synth

_P = C.c_void_p
MAX_LOCAL = 4096
BF = 40.0


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    so = tmp_path_factory.mktemp("emu") / "libstereo_track_emu.so"
    csrc = lmd.ROOT / "structure-plp-slam_b200" / "csrc"
    cmd = ["g++", "-O2", "-std=c++17", "-pthread", "-shared", "-fPIC", "-ffp-contract=off", "-fno-fast-math",
           f"-I{csrc}", f"-I{lmd.ROOT / 'tests' / 'cta_emu'}", str(lmd.ROOT / "tests" / "cta_emu" / "stereo_track_emu.cc"),
           "-o", str(so)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[:3000]
    return C.CDLL(str(so))


def _a(x, dt):
    return np.ascontiguousarray(x, dt)


def _p(a):
    return None if a is None else a.ctypes.data_as(_P)


def _stereo_cam(plp):
    return plp.capi.make_camera(synth.FX, synth.FY, synth.CX, synth.CY, synth.COLS, synth.ROWS, bf=BF, setup_type=1)


# ---- motion_assumption ------------------------------------------------------------------------------------------------
def _oracle_flags(orc, plp, cam, Tc, Tl):
    """The oracle's forward / backward flags, read from match_current_and_last_frames: landmark A (octave 3) is seen by
    a keypoint at octave 5 only in the forward range [3, 7], landmark B by one at octave 1 only in the backward range
    [0, 3]; the monocular range of both is [2, 4]."""
    X = np.array([[0.3, 0.2, 6.0], [-0.4, -0.1, 6.0]])
    R, t = Tc[:3, :3], Tc[:3, 3]
    pc = X @ R.T + t
    uv = np.stack([synth.FX * pc[:, 0] / pc[:, 2] + synth.CX, synth.FY * pc[:, 1] / pc[:, 2] + synth.CY], 1)
    desc = synth.rand_desc(np.random.default_rng(5), 2)
    curr = dict(x=_a(uv[:, 0], np.float32), y=_a(uv[:, 1], np.float32), octave=_a([5, 1], np.int32),
                angle=_a([10, 10], np.float32), desc=desc)
    last = dict(pos_w=X, octave=_a([3, 3], np.int32), angle=_a([10, 10], np.float32), desc=desc)
    grid = plp.capi.make_grid(synth.COLS, synth.ROWS)
    m, _ = orc.match_current_and_last_frames(grid, synth.scale_factors(), cam, curr, Tc, Tl, last, 10.0, False)
    return int(m[0] == 0), int(m[1] == 1)


def _emu_flags(emu, cam, Tc, Tl):
    f, b = C.c_int(-1), C.c_int(-1)
    emu.emu_motion_assumption(C.byref(cam), _p(_a(Tc, np.float64)), _p(_a(Tl, np.float64)), C.byref(f), C.byref(b))
    return f.value, b.value


def test_motion_assumption_equals_oracle(emu, orc, plp):
    """trans_lc.z exactly at +-true_baseline and one ulp above and below it, on an axis-aligned pose (the sums are
    exact) and on rotated poses; a monocular camera is neither forward nor backward."""
    cam = _stereo_cam(plp)
    b = cam.true_baseline
    zs = [b, np.nextafter(b, np.inf), np.nextafter(b, -np.inf), -b, np.nextafter(-b, np.inf), np.nextafter(-b, -np.inf),
          0.0, 3 * b, -3 * b]
    seen = set()
    for z in zs:
        Tc = np.eye(4)
        Tc[2, 3] = -z  # trans_wc = (0, 0, z), trans_lc = trans_wc with the last frame at the origin
        want = _oracle_flags(orc, plp, cam, Tc, np.eye(4))
        assert _emu_flags(emu, cam, Tc, np.eye(4)) == want, z
        assert want == (int(z > b), int(-z > b)), z
        seen.add(want)
    assert seen == {(0, 0), (1, 0), (0, 1)}
    rng = np.random.default_rng(3)
    for k in range(24):
        Tc = synth.make_pose(rng, 0.02, 0.05)
        Tl = synth.make_pose(rng, 0.02, 0.05)
        twc = -(Tc[:3, :3].T @ Tc[:3, 3])
        z = (1 if k % 2 else -1) * b
        Tl[2, 3] = z - Tl[2, :3] @ twc  # trans_lc.z within an ulp or two of +-true_baseline
        for step in range(-2, 3):
            T = Tl.copy()
            for _ in range(abs(step)):
                T[2, 3] = np.nextafter(T[2, 3], np.inf if step > 0 else -np.inf)
            assert _emu_flags(emu, cam, Tc, T) == _oracle_flags(orc, plp, cam, Tc, T), (k, step)
    mono = plp.capi.make_camera(synth.FX, synth.FY, synth.CX, synth.CY, synth.COLS, synth.ROWS)
    Tc = np.eye(4)
    Tc[2, 3] = -3 * b
    assert _emu_flags(emu, mono, Tc, np.eye(4)) == (0, 0) == _oracle_flags(orc, plp, mono, Tc, np.eye(4))


# ---- the shared tail's gather -----------------------------------------------------------------------------------------
def _pose_opt_obs(pos_w, x, y, octave, x_right, idx, rows):
    """pose_optimizer.cc:126-151: one observation per matched keypoint idx (landmark rows `rows`), in keypoint order."""
    o = np.zeros(len(idx), oracle_api.PT_OBS_DTYPE)
    o["pos_w"] = pos_w[rows]
    o["obs_x"], o["obs_y"] = x[idx], y[idx]
    o["x_right"] = -1.0 if x_right is None else x_right[idx]
    o["inv_sigma_sq"] = lmd.ISIG[octave[idx]]
    return o


def test_tail_gather_stereo_rows(emu):
    """Three frames: x_right -1, 0 and > 0 among the matched keypoints of each, one frame below the gate; and the same
    gather without x_right (a monocular tracker) writes -1 everywhere."""
    rng = np.random.default_rng(11)
    scenes = [synth.make_tracking_scene(40 + b, n_last=500, n_extra=100, stereo=True) for b in range(3)]
    B = len(scenes)
    n_kp = _a([len(s[0]["x"]) for s in scenes], np.int32)
    cap = int(n_kp.max())
    X, Y, XR = (np.zeros((B, cap), np.float32) for _ in range(3))
    O = np.zeros((B, cap), np.int32)
    matched = np.full((B, cap), -1, np.int32)
    for b, (curr, last, _, _) in enumerate(scenes):
        n = n_kp[b]
        X[b, :n], Y[b, :n], O[b, :n] = curr["x"], curr["y"], curr["octave"]
        xr = curr["x_right"].copy()
        xr[rng.choice(n, 40, replace=False)] = 0.0
        XR[b, :n] = xr
        sel = rng.choice(n, 300, replace=False)
        matched[b, sel] = rng.integers(0, len(last["octave"]), 300)
    count = _a([300, 300, 12], np.int32)
    pos_w = _a(np.concatenate([s[1]["pos_w"] for s in scenes]), np.float64)
    offs = _a(np.concatenate([[0], np.cumsum([len(s[1]["octave"]) for s in scenes])]), np.int32)
    pose_in = _a(np.tile(np.eye(4), (B, 1, 1)), np.float64)
    isig = _a(lmd.ISIG, np.float32)
    for xr_arg in (XR, None):
        obs = np.zeros((B, cap), oracle_api.PT_OBS_DTYPE)
        obs_kp = np.full((B, cap), -7, np.int32)
        n_obs = np.full(B, -7, np.int32)
        m = matched.copy()
        emu.emu_tail_gather_stereo(C.c_int(B), C.c_int(cap), _p(n_kp), _p(X), _p(Y), _p(O), _p(xr_arg), _p(isig),
                                   C.c_int(lmd.NUM_LEVELS), _p(count), _p(pos_w), _p(offs), _p(pose_in), _p(m),
                                   _p(obs), _p(obs_kp), _p(n_obs))
        assert n_obs[2] == 0
        for b in range(2):
            idx = np.nonzero(matched[b, :n_kp[b]] >= 0)[0]
            want = _pose_opt_obs(pos_w[offs[b]:offs[b + 1]], X[b], Y[b], O[b], None if xr_arg is None else XR[b], idx,
                                 matched[b, idx])
            assert n_obs[b] == len(idx) and np.array_equal(obs_kp[b, :len(idx)], idx), b
            assert obs[b, :len(idx)].tobytes() == want.tobytes(), b
            got = obs[b, :len(idx)]["x_right"]
            if xr_arg is None:
                assert (got == -1).all()
            else:
                assert (got == 0).any() and (got < 0).any() and (got > 0).any(), b


# ---- the local-map stage ----------------------------------------------------------------------------------------------
def _frame(orc, plp, seed):
    seq = scene.PlanarSequence(seed=seed, n_frames=4)
    cam, right = std.stereo_sequence(plp, seq, BF)
    p = oracle_api.orb_params()
    res = [orc.orb_extract(p, f) for f in seq.frames]
    t = 3
    xr, _, _ = orc.stereo_compute(res[t], orc.orb_extract(p, right[t]), lmd.SF, (1.0 / lmd.SF).astype(np.float32),
                                  cam.focal_x_baseline, cam.true_baseline)
    return seq, cam, res, t, np.asarray(xr, np.float32)


def _oracle_local(orc, plp, seq, cam, res, t, xr, pred, last, loc):
    grid = plp.capi.make_grid(seq.cols, seq.rows)
    curr = dict(lmd.curr_frame(res[t]), x_right=xr)
    motion = std.oracle_motion(orc, grid, cam, curr, last, pred, seq.poses[t - 1])
    return curr, motion, std.oracle_local_track(orc, grid, cam, curr, last, loc, motion, MAX_LOCAL)


def _emu_local(emu, plp, seq, cam, curr, motion, last, loc, stereo=True):
    grid = plp.capi.make_grid(seq.cols, seq.rows)
    n = len(curr["x"])
    cap = n
    pre, post, T, nv = motion[0], motion[1], motion[2], motion[3]
    rows = pre[pre >= 0] if nv >= 20 else pre[:0]
    m_obs_row = np.zeros(cap, np.int32)
    m_obs_row[:len(rows)] = rows
    nl = len(loc["max_valid_dist"])
    thr = _a(plp.capi.fuse_level_thresholds(float(lmd.LOG_SF), lmd.NUM_LEVELS), np.float32)
    qxr = np.full(MAX_LOCAL, 777.0, np.float32)
    best = np.full(MAX_LOCAL, -7, np.int32)
    matched, local = np.full(cap, -7, np.int32), np.full(cap, -7, np.int32)
    obs = np.zeros(cap, oracle_api.PT_OBS_DTYPE)
    obs_kp, n_obs = np.zeros(cap, np.int32), np.zeros(1, np.int32)
    arrs = [_a(curr["x"], np.float32), _a(curr["y"], np.float32), _a(curr["octave"], np.int32),
            _a(curr["desc"], np.uint8), _a(curr["x_right"], np.float32) if stereo else None, _a(lmd.ISIG, np.float32),
            _a(post, np.int32), _a(T, np.float64), _a([nv], np.int32), _a([len(rows)], np.int32), m_obs_row,
            _a(last["pos_w"], np.float64), _a([0, len(last["octave"])], np.int32), _a(loc["pos_w"], np.float64),
            _a(loc["normal"], np.float64), _a(loc["min_valid_dist"], np.float32), _a(loc["max_valid_dist"], np.float32),
            _a(loc["max_valid_dist_raw"], np.float32), _a(loc["desc"], np.uint8), _a([0, nl], np.int32),
            _a(loc["last_local_idx"], np.int32), _a(lmd.SF, np.float32), thr]
    emu.emu_local_stereo(C.byref(grid), C.byref(cam), C.c_int(1), C.c_int(cap), C.c_int(MAX_LOCAL),
                         _p(_a([n], np.int32)), *[_p(a) for a in arrs], C.c_int(lmd.NUM_LEVELS),
                         C.c_float(lmd.MARGIN), _p(qxr), _p(best), _p(matched), _p(local), _p(obs), _p(obs_kp),
                         _p(n_obs))
    return dict(qxr=qxr[:nl], best=best[:nl], matched=matched, local=local, obs=obs[:n_obs[0]], obs_kp=obs_kp[:n_obs[0]])


def _want_obs(curr, last, loc, motion, want):
    """The observations of pose-opt #2 before the outlier drop (pose_optimizer.cc:126-151)."""
    post = motion[1]
    n = len(post)
    loc_kp = np.full(n, -1, np.int32)
    for j in np.nonzero(want["best"] >= 0)[0]:
        loc_kp[want["best"][j]] = j
    idx = np.nonzero((post >= 0) | (loc_kp >= 0))[0]
    pos = np.where((post[idx] >= 0)[:, None], np.asarray(last["pos_w"])[np.maximum(post[idx], 0)],
                   np.asarray(loc["pos_w"]).reshape(-1, 3)[np.maximum(loc_kp[idx], 0)])
    o = np.zeros(len(idx), oracle_api.PT_OBS_DTYPE)
    o["pos_w"] = pos
    o["obs_x"], o["obs_y"] = curr["x"][idx], curr["y"][idx]
    o["x_right"] = curr["x_right"][idx]
    o["inv_sigma_sq"] = lmd.ISIG[curr["octave"][idx]]
    return idx, o


def _on_radius(qxr, r, above):
    """A positive x_right whose float |qxr - x_right| is exactly r, or None where no float is (above: the largest one
    whose distance exceeds r)."""
    q = np.float32(qxr)
    xr = np.float32(q - r)
    if above:
        while np.float32(abs(q - xr)) <= r:
            xr = np.nextafter(xr, np.float32(-np.inf))
        return xr
    for _ in range(64):
        d = np.float32(abs(q - xr))
        if d == r:
            return xr if xr > 0 else None
        xr = np.nextafter(xr, np.float32(-np.inf) if d < r else np.float32(np.inf))
    return None


def test_local_map_kernels_stereo_equal_oracle(emu, orc, plp):
    """One frame with x_right -1, 0 and > 0, a local-map candidate whose x_right is exactly the search radius away from
    the query's predicted x_right (kept), and one a float beyond it (rejected by the x_right gate alone): the qxr row,
    the matches and the gathered observations equal the oracle's."""
    seq, cam, res, t, xr = _frame(orc, plp, 53)
    rng = np.random.default_rng(12)
    pred = seq.predicted_pose(t, rng)
    last = seq.last_frame_landmarks(t - 1, res[t - 1]["kps"], res[t - 1]["desc"])
    loc = lmd.build_local_map(seq, res, t, rng, last_frame=last, drop_last=10)
    xr = xr.copy()
    zero = np.nonzero(xr < 0)[0][:30]
    xr[zero] = 0.0  # not stereo for the gate, stereo for the edge
    curr, motion, want = _oracle_local(orc, plp, seq, cam, res, t, xr, pred, last, loc)
    assert want["status"] == 0 and motion[3] >= 20
    # two keypoints matched from the local map only, moved onto / just past the radius of their query
    _, _, _, lvl, _ = lmd.can_observe(cam, motion[2], loc)
    radius = lambda j: np.float32(np.float32(lmd.MARGIN) * lmd.SF[lvl[j]])
    cand = [j for j in np.nonzero(want["best"] >= 0)[0] if motion[0][want["best"][j]] < 0]
    exact = [j for j in cand if _on_radius(want["qxr"][j], radius(j), False) is not None]
    edited = None
    for j1, j2 in zip(exact, [j for j in cand if j not in exact]):
        i1, i2 = want["best"][j1], want["best"][j2]
        trial = xr.copy()
        trial[i1] = _on_radius(want["qxr"][j1], radius(j1), False)
        trial[i2] = _on_radius(want["qxr"][j2], radius(j2), True)
        c2, m2, w2 = _oracle_local(orc, plp, seq, cam, res, t, trial, pred, last, loc)
        if np.array_equal(m2[0], motion[0]) and w2["best"][j1] == i1 and w2["best"][j2] != i2:
            edited = (c2, m2, w2)
            break
    assert edited is not None, "no local-map pair to put on the radius"
    curr, motion, want = edited
    got = _emu_local(emu, plp, seq, cam, curr, motion, last, loc)
    obs_rows = want["observable"] != 0
    assert obs_rows.sum() > 100
    assert np.array_equal(got["qxr"][obs_rows], want["qxr"][obs_rows])
    assert (got["qxr"][~obs_rows] == 777.0).all()  # the observe kernel writes the rows it queries only
    assert np.array_equal(got["best"], want["best"])
    assert np.array_equal(got["matched"], motion[1])
    idx, wobs = _want_obs(curr, last, loc, motion, want)
    assert np.array_equal(got["obs_kp"], idx) and got["obs"].tobytes() == wobs.tobytes()
    xo = wobs["x_right"]
    assert (xo == 0).any() and (xo < 0).any() and (xo > 0).any()
    # without x_right the stage is the monocular one: no qxr row written, the gate off, 2-D edges only
    mono = _emu_local(emu, plp, seq, cam, curr, motion, last, loc, stereo=False)
    assert (mono["qxr"] == 777.0).all() and (mono["obs"]["x_right"] == -1).all()
    assert not np.array_equal(mono["best"], got["best"])
