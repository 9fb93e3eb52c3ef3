"""The local-map DEVICE code (structure-plp-slam_b200/csrc/local_map_kernels.cuh, with the window matcher between observe
and gather) executed on the CPU through tests/cta_emu, equal to the oracle chain: a batch of frames with a tracked frame
whose local map spans many observe CTAs, a frame whose motion track failed, an empty local map, and both status cases.
The pose optimiser between gather and finish is the oracle's, run on the observations the emulated gather produced."""
import ctypes as C
import shutil
import subprocess

import numpy as np
import pytest

import local_map_data as lmd
import oracle_api
import scene

_P = C.c_void_p
MAX_LOCAL = 2500


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    so = tmp_path_factory.mktemp("emu") / "liblocal_map_emu.so"
    csrc = lmd.ROOT / "structure-plp-slam_b200" / "csrc"
    cmd = ["g++", "-O2", "-std=c++17", "-pthread", "-shared", "-fPIC", "-ffp-contract=off", "-fno-fast-math",
           f"-I{csrc}", f"-I{lmd.ROOT / 'tests' / 'cta_emu'}", str(lmd.ROOT / "tests" / "cta_emu" / "local_map_emu.cc"),
           "-o", str(so)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[:3000]
    return C.CDLL(str(so))


def _a(x, dt):
    return np.ascontiguousarray(x, dt)


def test_local_map_kernels_on_cpu_equal_oracle(emu, orc, plp):
    seq = scene.PlanarSequence(seed=51, n_frames=5)
    res = [orc.orb_extract(oracle_api.orb_params(), f) for f in seq.frames]
    grid, cam = plp.capi.make_grid(seq.cols, seq.rows), seq.camera(plp)
    rng = np.random.default_rng(8)
    # frames: tracked (a ~2 k map over 16 observe CTAs, led by 64 erased rows), motion failed, empty map, over capacity,
    # bad last_local_idx
    ts = [2, 2, 3, 4, 1]
    preds = [seq.predicted_pose(t, rng) for t in ts]
    preds[1] = preds[1].copy()
    preds[1][:3, 3] += [1.0, 0.5, 0.0]
    lasts = [seq.last_frame_landmarks(t - 1, res[t - 1]["kps"], res[t - 1]["desc"]) for t in ts]
    B = len(ts)
    curr = [lmd.curr_frame(res[t]) for t in ts]
    motion = [lmd.oracle_motion(orc, grid, cam, curr[b], lasts[b], preds[b], seq.poses[t - 1]) for b, t in enumerate(ts)]
    locs = []
    for b, t in enumerate(ts):
        if b == 2:
            loc = lmd.empty_rows()
            loc["last_local_idx"] = np.full(len(lasts[b]["octave"]), -1, np.int32)
        else:
            loc = lmd.build_local_map(seq, res, t, rng, n_earlier=2, last_frame=lasts[b], drop_last=10)
            good = lmd.take(loc, np.arange(200))
            good.pop("last_local_idx")
            loc = lmd.with_rows(loc, lmd.distractors(cam, motion[b][2], good, rng))
            loc = lmd.with_erased_run(loc)  # whole warps of invalid queries in front
        if b == 4:
            loc["last_local_idx"] = loc["last_local_idx"].copy()
            loc["last_local_idx"][3] = len(loc["max_valid_dist"])
        locs.append(loc)
    sizes = [len(l["max_valid_dist"]) for l in locs]
    assert sizes[0] > 10 * 128 and sizes[0] <= MAX_LOCAL and sizes[3] > MAX_LOCAL, sizes
    assert motion[1][3] < 20 and all(motion[b][3] >= 20 for b in (0, 2, 3, 4))
    wants = [lmd.oracle_local_track(orc, grid, cam, curr[b], lasts[b], locs[b], motion[b], MAX_LOCAL) for b in range(B)]
    assert [w["status"] for w in wants] == [0, 0, 0, 1, 2]

    cap = max(len(c["x"]) for c in curr)
    n_kp = _a([len(c["x"]) for c in curr], np.int32)
    X = np.zeros((B, cap), np.float32)
    Y = np.zeros((B, cap), np.float32)
    O = np.zeros((B, cap), np.int32)
    Dsc = np.zeros((B, cap, 32), np.uint8)
    mm = np.full((B, cap), -1, np.int32)
    obs_last = np.zeros((B, cap), np.int32)
    n_obs1 = np.zeros(B, np.int32)
    for b, c in enumerate(curr):
        n = len(c["x"])
        X[b, :n], Y[b, :n], O[b, :n], Dsc[b, :n] = c["x"], c["y"], c["octave"], c["desc"]
        mm[b, :n] = motion[b][1]
        pre = motion[b][0]
        rows = pre[pre >= 0] if motion[b][3] >= 20 else pre[:0]
        n_obs1[b] = len(rows)
        obs_last[b, :len(rows)] = rows
    last_off = _a(np.concatenate([[0], np.cumsum([len(l["octave"]) for l in lasts])]), np.int32)
    last_pos = _a(np.concatenate([l["pos_w"] for l in lasts]), np.float64)
    pose = _a(np.stack([np.asarray(m[2]).reshape(4, 4) for m in motion]), np.float64)
    nv = _a([m[3] for m in motion], np.int32)
    offs = _a(np.concatenate([[0], np.cumsum(sizes)]), np.int32)
    cat = lambda k, dt: _a(np.concatenate([np.asarray(l[k], dt).ravel() for l in locs]), dt)
    lli = _a(np.concatenate([l["last_local_idx"] for l in locs]), np.int32)
    thr = plp.capi.fuse_level_thresholds(float(lmd.LOG_SF), lmd.NUM_LEVELS)
    matched = np.full((B, cap), -7, np.int32)
    local = np.full((B, cap), -7, np.int32)
    observable = np.full(max(int(offs[-1]), 1), 7, np.uint8)
    status = np.full(B, -7, np.int32)
    obs = np.zeros((B, cap), oracle_api.PT_OBS_DTYPE)
    obs_kp = np.zeros((B, cap), np.int32)
    n_obs = np.zeros(B, np.int32)
    keep = [X, Y, O, Dsc, mm, obs_last, n_obs1, last_off, last_pos, pose, nv, offs, lli, thr]
    arrays = [cat("pos_w", np.float64), cat("normal", np.float64), cat("min_valid_dist", np.float32),
              cat("max_valid_dist", np.float32), cat("max_valid_dist_raw", np.float32), cat("desc", np.uint8),
              cat("valid", np.uint8)]
    sf = _a(lmd.SF, np.float32)
    isig = _a(lmd.ISIG, np.float32)
    p = lambda a: a.ctypes.data_as(_P)
    emu.emu_local_begin(C.byref(grid), C.byref(cam), C.c_int(B), C.c_int(cap), C.c_int(MAX_LOCAL), p(n_kp), p(X), p(Y),
                        p(O), p(Dsc), p(last_pos), p(last_off), p(mm), p(pose), p(nv), p(n_obs1), p(obs_last), p(isig),
                        *[p(a) for a in arrays], p(offs), p(lli), p(sf), p(_a(thr, np.float32)),
                        C.c_int(lmd.NUM_LEVELS), C.c_float(lmd.MARGIN), p(matched), p(local), p(observable), p(status),
                        p(obs), p(obs_kp), p(n_obs))
    del keep
    outlier = np.zeros((B, cap), np.uint8)
    for b in range(B):
        if n_obs[b] >= 5:
            _, pout, _, _, _ = orc.pose_optimize(cam, pose[b], obs[b, :n_obs[b]])
            outlier[b, :n_obs[b]] = pout
    num_tracked = np.full(B, -7, np.int32)
    emu.emu_local_finish(p(outlier), p(num_tracked))
    for b, w in enumerate(wants):
        n = int(n_kp[b])
        assert status[b] == w["status"], b
        assert np.array_equal(observable[offs[b]:offs[b + 1]], w["observable"]), b
        assert np.array_equal(matched[b, :n], w["matched"]), b
        assert np.array_equal(local[b, :n], w["local"]), b
        assert num_tracked[b] == w["num_tracked"], (b, num_tracked[b], w["num_tracked"])
    assert (local[0] >= 0).sum() > 20
