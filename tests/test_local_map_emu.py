"""The local-map DEVICE code (structure-plp-slam_b200/csrc/local_map_kernels.cuh, with the window matcher between observe
and gather) executed on the CPU through tests/cta_emu, equal to the oracle chain: a batch of frames with a tracked frame
whose local map spans many observe CTAs, a frame whose motion track failed, an empty local map, and both status cases.
The pose optimiser between gather and finish is the oracle's, run on the observations the emulated gather produced."""
import ctypes as C

import numpy as np
import pytest

import emu_build
import local_map_data as lmd
import oracle_api
import scene

_P = C.c_void_p
MAX_LOCAL = 2500


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return emu_build.emu("local_map_emu", tmp_path_factory)


def _a(x, dt):
    return np.ascontiguousarray(x, dt)


_REC_FIELDS = ("stage", "status", "matched", "pose", "num_valid", "n_obs", "obs_row", "pos_w", "offsets", "of_frame",
               "local_idx", "local_idx_offsets")


class _EmuRecord(C.Structure):  # tests/cta_emu/local_map_emu.cc
    _fields_ = [(f, _P) for f in _REC_FIELDS]


def _record(B, cap):
    """A record in which every frame failed its tracker."""
    return dict(matched=np.full((B, cap), -1, np.int32), pose=np.tile(np.eye(4), (B, 1, 1)), num_valid=np.zeros(B, np.int32),
                n_obs=np.zeros(B, np.int32), obs_row=np.zeros((B, cap), np.int32))


def _put(rec, b, motion):
    """Frame b of rec holds a tracker result in oracle_motion's form: its matches, pose, num_valid and the rows of its
    pose-opt observations (the matches before discard_outliers, none below 20)."""
    pre, post = motion[0], motion[1]
    rows = pre[pre >= 0] if motion[3] >= 20 else pre[:0]
    rec["matched"][b, :len(post)] = post
    rec["pose"][b] = np.asarray(motion[2]).reshape(4, 4)
    rec["num_valid"][b] = motion[3]
    rec["n_obs"][b] = len(rows)
    rec["obs_row"][b, :len(rows)] = rows


def _emu_local(emu, orc, plp, grid, cam, curr, locs, records, lli):
    """prep -> observe -> match -> gather (emulated) -> the oracle's pose optimiser -> finish (emulated), the frames
    starting from records (motion, keyframe, robust; None: no such record)."""
    B = len(curr)
    n_kp = _a([len(c["x"]) for c in curr], np.int32)
    cap = int(n_kp.max())
    X = np.zeros((B, cap), np.float32)
    Y = np.zeros((B, cap), np.float32)
    O = np.zeros((B, cap), np.int32)
    Dsc = np.zeros((B, cap, 32), np.uint8)
    for b, c in enumerate(curr):
        n = len(c["x"])
        X[b, :n], Y[b, :n], O[b, :n], Dsc[b, :n] = c["x"], c["y"], c["octave"], c["desc"]
    sizes = [len(l["max_valid_dist"]) for l in locs]
    offs = _a(np.concatenate([[0], np.cumsum(sizes)]), np.int32)
    cat = lambda k, dt: _a(np.concatenate([np.asarray(l[k], dt).ravel() for l in locs]), dt)
    thr = _a(plp.capi.fuse_level_thresholds(float(lmd.LOG_SF), lmd.NUM_LEVELS), np.float32)
    matched = np.full((B, cap), -7, np.int32)
    local = np.full((B, cap), -7, np.int32)
    observable = np.full(max(int(offs[-1]), 1), 7, np.uint8)
    status = np.full(B, -7, np.int32)
    obs = np.zeros((B, cap), oracle_api.PT_OBS_DTYPE)
    obs_kp = np.zeros((B, cap), np.int32)
    n_obs = np.zeros(B, np.int32)
    arrays = [cat("pos_w", np.float64), cat("normal", np.float64), cat("min_valid_dist", np.float32),
              cat("max_valid_dist", np.float32), cat("max_valid_dist_raw", np.float32), cat("desc", np.uint8),
              cat("valid", np.uint8)]
    sf = _a(lmd.SF, np.float32)
    isig = _a(lmd.ISIG, np.float32)
    p = lambda a: None if a is None else a.ctypes.data_as(_P)
    keep, recs = [], (_EmuRecord * 3)()
    for r, rec in zip(recs, records):
        for f in _REC_FIELDS:
            a = None if rec is None or rec.get(f) is None else _a(rec[f], np.float64 if f in ("pose", "pos_w") else np.int32)
            keep.append(a)
            setattr(r, f, p(a))
    emu.emu_local_begin(C.byref(grid), C.byref(cam), C.c_int(B), C.c_int(cap), C.c_int(MAX_LOCAL), p(n_kp), p(X), p(Y),
                        p(O), p(Dsc), recs, p(isig), *[p(a) for a in arrays], p(offs), p(lli), p(sf), p(thr),
                        C.c_int(lmd.NUM_LEVELS), C.c_float(lmd.MARGIN), p(matched), p(local), p(observable), p(status),
                        p(obs), p(obs_kp), p(n_obs))
    outlier = np.zeros((B, cap), np.uint8)
    for b in range(B):
        if n_obs[b] >= 5:
            T_in = records[0]["pose"][b]
            for rec in records[1:]:  # the pose the stage started from: the last stage that ran
                if rec is not None and rec["stage"][b]:
                    T_in = rec["pose"][b]
            _, pout, _, _, _ = orc.pose_optimize(cam, T_in, obs[b, :n_obs[b]])
            outlier[b, :n_obs[b]] = pout
    num_tracked = np.full(B, -7, np.int32)
    emu.emu_local_finish(p(outlier), p(num_tracked))
    return status, observable, matched, local, num_tracked, offs


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

    n_kp = _a([len(c["x"]) for c in curr], np.int32)
    cap = int(n_kp.max())
    mrec = _record(B, cap)
    for b in range(B):
        _put(mrec, b, motion[b])
    mrec.update(pos_w=_a(np.concatenate([l["pos_w"] for l in lasts]), np.float64),
                offsets=_a(np.concatenate([[0], np.cumsum([len(l["octave"]) for l in lasts])]), np.int32))
    lli = _a(np.concatenate([l["last_local_idx"] for l in locs]), np.int32)
    status, observable, matched, local, num_tracked, offs = _emu_local(emu, orc, plp, grid, cam, curr, locs,
                                                                       [mrec, None, None], lli)
    for b, w in enumerate(wants):
        n = len(curr[b]["x"])
        assert status[b] == w["status"], b
        assert np.array_equal(observable[offs[b]:offs[b + 1]], w["observable"]), b
        assert np.array_equal(matched[b, :n], w["matched"]), b
        assert np.array_equal(local[b, :n], w["local"]), b
        assert num_tracked[b] == w["num_tracked"], (b, num_tracked[b], w["num_tracked"])
    assert (local[0] >= 0).sum() > 20


def test_local_map_kernels_from_keyframe_and_robust_records(emu, orc, plp):
    """Frames that start from a keyframe or a robust record: the record's own matches, pose and observation rows, the
    keyframe rows through kf_of_frame, and local_idx in place of last_local_idx.  The reference is the motion chain with
    the keyframe rows as the last frame's.  A start record with a non-zero status reads no row table (kf_of_frame out of
    range) and leaves the frame inactive; a local_idx block of the wrong length is status 2."""
    seq = scene.PlanarSequence(seed=52, n_frames=4)
    res = [orc.orb_extract(oracle_api.orb_params(), f) for f in seq.frames]
    grid, cam = plp.capi.make_grid(seq.cols, seq.rows), seq.camera(plp)
    rng = np.random.default_rng(9)
    # frames: motion-started, keyframe-started, robust-started, keyframe status 2, keyframe-started with a short block
    ts = [2, 3, 2, 1, 3]
    B = len(ts)
    preds = [seq.predicted_pose(t, rng) for t in ts]
    lasts = [seq.last_frame_landmarks(t - 1, res[t - 1]["kps"], res[t - 1]["desc"]) for t in ts]
    curr = [lmd.curr_frame(res[t]) for t in ts]
    motion = [lmd.oracle_motion(orc, grid, cam, curr[b], lasts[b], preds[b], seq.poses[t - 1]) for b, t in enumerate(ts)]
    locs = []
    for b, t in enumerate(ts):
        locs.append(lmd.build_local_map(seq, res, t, rng, n_earlier=1, last_frame=lasts[b], drop_last=10))
    sizes = [len(l["max_valid_dist"]) for l in locs]
    assert all(s <= MAX_LOCAL for s in sizes) and all(motion[b][3] >= 20 for b in range(B)), (sizes, motion)

    n_kp = _a([len(c["x"]) for c in curr], np.int32)
    cap = int(n_kp.max())
    mrec, krec, rrec = _record(B, cap), _record(B, cap), _record(B, cap)
    for b, rec in ((0, mrec), (1, krec), (2, rrec), (3, mrec), (4, krec)):
        _put(rec, b, motion[b])
    krec["num_valid"][2], krec["n_obs"][2] = 3, 3  # frame 2's keyframe track failed
    krec["matched"][2, :3] = [0, 1, 2]
    mrec.update(pos_w=_a(np.concatenate([l["pos_w"] for l in lasts]), np.float64),
                offsets=_a(np.concatenate([[0], np.cumsum([len(l["octave"]) for l in lasts])]), np.int32))
    # the keyframe table holds frame 4's, 2's and 1's last-frame rows, in that order
    order = [4, 2, 1]
    kf_rows = dict(pos_w=_a(np.concatenate([lasts[f]["pos_w"] for f in order]), np.float64),
                   offsets=_a(np.concatenate([[0], np.cumsum([len(lasts[f]["octave"]) for f in order])]), np.int32),
                   of_frame=_a([0, 2, 1, 99, 0], np.int32))
    blocks = [[], locs[1]["last_local_idx"], locs[2]["last_local_idx"], [], locs[4]["last_local_idx"][:-1]]
    kf_rows.update(local_idx=_a(np.concatenate(blocks), np.int32),
                   local_idx_offsets=_a(np.concatenate([[0], np.cumsum([len(x) for x in blocks])]), np.int32))
    krec.update(kf_rows, stage=_a([0, 1, 1, 1, 1], np.int32), status=_a([0, 0, 0, 2, 0], np.int32))
    rrec.update(kf_rows, stage=_a([0, 0, 1, 0, 0], np.int32), status=krec["status"])
    krec["num_valid"][3] = 0
    lli = _a(np.concatenate([l["last_local_idx"] for l in locs]), np.int32)
    status, observable, matched, local, num_tracked, offs = _emu_local(emu, orc, plp, grid, cam, curr, locs,
                                                                       [mrec, krec, rrec], lli)
    for b in range(B):
        n = len(curr[b]["x"])
        if b in (3, 4):
            w = dict(status=2 if b == 4 else 0, observable=np.zeros(sizes[b], np.uint8), matched=np.full(n, -1, np.int32),
                     local=np.full(n, -1, np.int32), num_tracked=0)
        else:
            w = lmd.oracle_local_track(orc, grid, cam, curr[b], lasts[b], locs[b], motion[b], MAX_LOCAL)
            assert w["status"] == 0 and (w["local"] >= 0).sum() > 10, b
        assert status[b] == w["status"], b
        assert np.array_equal(observable[offs[b]:offs[b + 1]], w["observable"]), b
        assert np.array_equal(matched[b, :n], w["matched"]), b
        assert np.array_equal(local[b, :n], w["local"]), b
        assert num_tracked[b] == w["num_tracked"], (b, num_tracked[b], w["num_tracked"])
