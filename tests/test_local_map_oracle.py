"""CPU tests of the local-map oracle (oracle/local_map_oracle.cc + local_map_data's chain): known answers for each
frame::can_observe gate and its boundary values, the exclusion of every landmark the motion track matched (the outliers
of its pose optimisation included), and the pass-through of frames whose motion track failed."""
import numpy as np
import pytest

import local_map_data as lmd
import oracle_api
import scene
import synth


@pytest.fixture(scope="module")
def cam(plp):
    return plp.capi.make_camera(synth.FX, synth.FY, synth.CX, synth.CY, synth.COLS, synth.ROWS)


def _pose(seed=0):
    T = np.eye(4)
    T[:3, :3] = synth.so3_exp(np.array([0.02, -0.01, 0.03]) * (seed + 1))
    T[:3, 3] = [0.1, -0.05, 0.2]
    return T


def _row(T, cam, u, v, z, normal_angle=0.0, min_d=0.0, max_d=np.inf, raw=None):
    """A landmark seen at pixel (u, v) at depth z from the pose T; its normal is the viewing ray turned by normal_angle."""
    R, t = T[:3, :3], T[:3, 3]
    pc = np.array([(u - cam.cx) / cam.fx * z, (v - cam.cy) / cam.fy * z, z])
    X = R.T @ (pc - t)
    c = lmd.cam_center(T)
    ray = (X - c) / np.linalg.norm(X - c)
    perp = np.cross(ray, [0.0, 0.0, 1.0] if abs(ray[2]) < 0.9 else [1.0, 0.0, 0.0])
    perp /= np.linalg.norm(perp)
    n = np.cos(normal_angle) * ray + np.sin(normal_angle) * perp
    fd = lmd.fdist(X, c)
    return dict(pos_w=X[None], normal=n[None], min_valid_dist=np.float32([min_d]), max_valid_dist=np.float32([max_d]),
                max_valid_dist_raw=np.float32([fd if raw is None else raw]), desc=np.zeros((1, 32), np.uint8),
                valid=np.ones(1, np.uint8)), fd, X, c


def test_can_observe_gates(cam):
    T = _pose()
    rows, skip = [], []
    ok, fd, _, _ = _row(T, cam, 300, 200, 4.0)
    rows.append(ok)                                                            # observable
    r, _, X, c = _row(T, cam, 300, 200, 4.0)
    r["pos_w"] = (2 * c - X)[None]                                             # behind the camera
    rows.append(r)
    rows.append(_row(T, cam, cam.max_x + 1.0, 200, 4.0)[0])                    # outside the bounds
    rows.append(_row(T, cam, 300, cam.max_y, 4.0)[0])                          # on the bound: strictly inside only
    rows.append(_row(T, cam, 300, 200, 4.0, min_d=fd * 2)[0])                  # too near
    rows.append(_row(T, cam, 300, 200, 4.0, max_d=fd / 2)[0])                  # too far
    rows.append(_row(T, cam, 300, 200, 4.0, normal_angle=np.pi)[0])            # normal turned away
    rows.append(_row(T, cam, 300, 200, 4.0)[0])                                # erased / excluded
    lms = lmd.concat(rows)
    skip = np.zeros(len(rows), np.uint8)
    skip[-1] = 1
    obs, rx, ry, lvl, gate = lmd.can_observe(cam, T, lms, skip)
    assert list(gate) == [0, 2, 2, 2, 3, 3, 4, 1]
    assert list(obs) == [1, 0, 0, 0, 0, 0, 0, 0]
    assert abs(rx[0] - 300) < 1e-3 and abs(ry[0] - 200) < 1e-3 and lvl[0] == 0 and (lvl[1:] == -1).all()


def test_can_observe_distance_bounds_are_float_and_inclusive(cam):
    T = _pose(1)
    _, fd, _, _ = _row(T, cam, 250, 180, 3.0)
    up, down = np.nextafter(fd, np.float32(np.inf)), np.nextafter(fd, np.float32(0))
    cases = [(fd, np.inf, 1), (up, np.inf, 0), (0.0, fd, 1), (0.0, down, 0), (fd, fd, 1)]
    lms = lmd.concat([_row(T, cam, 250, 180, 3.0, min_d=a, max_d=b)[0] for a, b, _ in cases])
    obs, *_ = lmd.can_observe(cam, T, lms)
    assert list(obs) == [w for *_, w in cases]


def test_can_observe_ray_cos_either_side_of_half(cam):
    """ray_cos = (pos - c) . normal / d in double, rejected iff < 0.5."""
    T = _pose(2)
    rows, want = [], []
    for k in range(-40, 41):
        r, _, X, c = _row(T, cam, 200, 150, 5.0, normal_angle=np.pi / 3 + k * 2e-16)
        d0, d1, d2 = (float(X[i]) - float(c[i]) for i in range(3))
        n = r["normal"][0]
        dist = np.sqrt(d0 * d0 + d1 * d1 + d2 * d2)
        ray_cos = (d0 * n[0] + d1 * n[1] + d2 * n[2]) / dist
        rows.append(r)
        want.append(int(not ray_cos < 0.5))
    obs, *_ = lmd.can_observe(cam, T, lmd.concat(rows))
    assert list(obs) == want
    assert 0 < sum(want) < len(want)  # both sides reached


def test_can_observe_levels_next_to_thresholds(cam):
    """predict_scale_level = ceil(logf(max_valid_dist_ / d) / log_scale_factor_), clamped, on floats; ratios on and next
    to every level threshold."""
    T = _pose(3)
    thr = lmd.level_thresholds()
    rows, want = [], []
    _, fd, _, _ = _row(T, cam, 320, 240, 4.0)
    for k in range(1, lmd.NUM_LEVELS):
        for raw in (np.nextafter(np.float32(thr[k] * fd), np.float32(0)), np.float32(thr[k] * fd),
                    np.nextafter(np.float32(thr[k] * fd), np.float32(np.inf)), np.float32(1e-3), np.float32(1e6)):
            rows.append(_row(T, cam, 320, 240, 4.0, raw=raw)[0])
            p = int(np.ceil(np.float32(lmd.logf(np.float32(raw) / fd) / lmd.LOG_SF)))
            want.append(min(max(p, 0), lmd.NUM_LEVELS - 1))
    obs, _, _, lvl, _ = lmd.can_observe(cam, T, lmd.concat(rows))
    assert obs.all() and list(lvl) == want
    assert set(want) == set(range(lmd.NUM_LEVELS))


@pytest.fixture(scope="module")
def two_frames(orc):
    seq = scene.PlanarSequence(seed=41, n_frames=3)
    res = [orc.orb_extract(oracle_api.orb_params(), f) for f in seq.frames]
    return seq, res


def test_motion_matches_are_excluded_outliers_included(orc, plp, cam, two_frames):
    """Landmarks the motion track matched are never queried again, including the outliers of pose-opt #1 (whose
    keypoints are free again): with those excluded the outliers' rows are not observable; without the exclusion they
    would be."""
    seq, res = two_frames
    grid = plp.capi.make_grid(seq.cols, seq.rows)
    t = 2
    last = seq.last_frame_landmarks(t - 1, res[t - 1]["kps"], res[t - 1]["desc"])
    rng = np.random.default_rng(2)
    bad = rng.choice(len(last["octave"]), 60, replace=False)
    last["pos_w"] = last["pos_w"].copy()
    last["pos_w"][bad, :2] += rng.normal(0, 0.02, (60, 2))   # a few pixels off: matched, then rejected by the optimiser
    curr = lmd.curr_frame(res[t])
    motion = lmd.oracle_motion(orc, grid, cam, curr, last, seq.predicted_pose(t, rng), seq.poses[t - 1])
    pre, post = motion[0], motion[1]
    outl = pre[(pre >= 0) & (post < 0)]
    assert motion[3] >= 20 and len(outl) >= 5
    loc = lmd.build_local_map(seq, res, t, rng, last_frame=last)
    lli = loc["last_local_idx"]
    got = lmd.oracle_local_track(orc, grid, cam, curr, last, loc, motion, 4096)
    assert not got["observable"][lli[pre[pre >= 0]]].any()
    assert got["num_tracked"] >= motion[3] and (got["local"] >= 0).sum() > 0
    # the same rows are observable once the exclusion is lifted (their positions are those the motion track used)
    obs, *_ = lmd.can_observe(cam, motion[2], loc)
    assert obs[lli[outl]].sum() >= len(outl) // 2
    # no keypoint holds a landmark twice, and every local match is an observable row
    assert not ((got["matched"] >= 0) & (got["local"] >= 0)).any()
    assert got["observable"][got["local"][got["local"] >= 0]].all()


def test_failed_motion_frames_pass_through(orc, plp, cam, two_frames):
    seq, res = two_frames
    grid = plp.capi.make_grid(seq.cols, seq.rows)
    t = 2
    last = seq.last_frame_landmarks(t - 1, res[t - 1]["kps"], res[t - 1]["desc"])
    T_pred = seq.poses[t].copy()
    T_pred[:3, 3] += [1.0, 0.5, 0.0]
    curr = lmd.curr_frame(res[t])
    motion = lmd.oracle_motion(orc, grid, cam, curr, last, T_pred, seq.poses[t - 1])
    assert motion[3] < 20
    loc = lmd.build_local_map(seq, res, t, np.random.default_rng(1), last_frame=last)
    got = lmd.oracle_local_track(orc, grid, cam, curr, last, loc, motion, 4096)
    assert got["status"] == 0 and got["num_tracked"] == 0 and got["lm_iters"] == 0 and got["n_inliers"] == 0
    assert (got["matched"] == -1).all() and (got["local"] == -1).all() and not got["observable"].any()
    assert np.array_equal(got["pose"], motion[2])  # the motion track's pose, whatever it is
