"""GPU parity of the batched local-map update (plp_tracker_update_local_map_batch_dev, tracking.FrontEnd.update_local_map)
against the restatement of update_local_map (tests/local_map_update_data.py), and of the local-map stage that takes its
list: the chain motion -> keyframe -> robust -> update -> local map against the oracle chain with the oracle-built list,
and against the same stage given that list through set_local_maps, byte for byte."""
import ctypes as C

import numpy as np
import pytest

import keyframe_track_data as ktd
import local_map_data as lmd
import local_map_update_data as lmu
import oracle_api
import robust_track_data as rtd
import scene

pytestmark = pytest.mark.gpu
MAX_LKF = 128


def _vocab(orc, plp, ctx, res, seed):
    v = ktd.make_scene_vocab(np.concatenate([r["desc"] for r in res]), seed)
    ov = orc.bow_vocab_create(v["k"], v["L"], v["parent"], v["desc"], v["weight"], v["is_leaf"])
    gv = plp.BowVocabulary(ctx, k=v["k"], L=v["L"], parent=v["parent"], desc=v["desc"], weight=v["weight"],
                           is_leaf=v["is_leaf"])
    return ov, gv


def _bytes(d):
    out = {}
    for k, v in d.items():
        if k == "bow":
            out[k] = b"".join(x.tobytes() for t in v for x in t)
        elif isinstance(v, list):
            out[k] = b"".join(np.asarray(x).tobytes() for x in v)
        else:
            out[k] = np.asarray(v).tobytes()
    return out


def _snapshot(seq, res, ts, kfs, rng, undistort=None):
    """A snapshot along the sequence with the chain's rows mapped: last-frame row i of frame t is landmark (t - 1, i),
    keyframe-table row i of keyframe kf is landmark (kf["t"], i); a keyframe's erased rows are erased landmarks, and two
    keyframes are erased."""
    n_kf = max(max(ts), max(kf["t"] for kf in kfs) + 1)
    snap, lm_id = lmu.scene_snapshot(seq, res, n_kf, rng, undistort=undistort)
    for kf in kfs:
        snap["lm_erased"][lm_id[kf["t"]][np.asarray(kf["valid"]) == 0]] = 1
    snap["kf_erased"][[1, n_kf - 3]] = 1
    snap["last_row_lm"] = np.concatenate([lm_id[t - 1] for t in ts]).astype(np.int32)
    snap["kf_row_lm"] = np.concatenate([lm_id[kf["t"]] for kf in kfs]).astype(np.int32)
    return snap


def _tracked(r, b, snap, lasts_off, kf_off, kf_of_frame):
    """The landmarks frame b holds after its last tracking stage (the device results, which run_case checked)."""
    if r["rb_stage"][b]:
        m, rows, nv, st = r["rb"]["matched"][b], snap["kf_row_lm"][kf_off[kf_of_frame[b]]:], r["rb"]["num_valid"][b], \
            r["rb"]["status"][b]
    elif r["kf_stage"][b]:
        m, rows, nv, st = r["kf"]["matched"][b], snap["kf_row_lm"][kf_off[kf_of_frame[b]]:], r["kf"]["num_valid"][b], \
            r["kf"]["status"][b]
    else:
        m, rows, nv, st = r["mot"]["matched"][b], snap["last_row_lm"][lasts_off[b]:], r["mot"]["num_valid"][b], 0
    return np.array([rows[q] if q >= 0 else -1 for q in m], np.int32), nv >= 20 and st == 0


def _chain(ctx, orc, plp, fe, ov, gv, seq, res, ts, kfs, kf_of_frame, motion_valid, fail=(), seed=0, rb_seed=0,
           grid=None, cam=None, undistort=None):
    B = len(ts)
    grid, cam = grid or fe.grid, cam or fe.cam
    r = rtd.run_case(orc, plp, fe, ov, gv, seq, res, ts, kfs, kf_of_frame, motion_valid, fail=fail, seed=seed,
                     rb_seed=rb_seed, grid=grid, cam=cam, undistort=undistort)
    rng = np.random.default_rng(seed)  # run_case's predicted poses, for the oracle's motion track
    preds = [seq.predicted_pose(t, rng) for t in ts]
    for b in fail:
        preds[b] = preds[b].copy()
        preds[b][:3, 3] += np.asarray((1.0, 0.5, 0.0))
    rng = np.random.default_rng(seed + 100)
    snap = _snapshot(seq, res, ts, kfs, rng, undistort)
    fe.set_map(snap)
    lasts_off = fe._last_offsets
    kf_off = np.concatenate([[0], np.cumsum([len(kf["desc"]) for kf in kfs])])
    before = [_bytes(fe.download_tracking(B)), _bytes(fe.download_keyframe_tracking(B)), _bytes(fe.download_robust_tracking(B))]
    fe.update_local_map(B)
    u = fe.download_local_map_update(B)
    after = [_bytes(fe.download_tracking(B)), _bytes(fe.download_keyframe_tracking(B)), _bytes(fe.download_robust_tracking(B))]
    assert before == after  # the tracking outputs, byte for byte
    wants = []
    for b, t in enumerate(ts):
        tracked, active = _tracked(r, b, snap, lasts_off, kf_off, kf_of_frame)
        w = lmu.device_update(snap, tracked, fe.max_local, MAX_LKF, active)
        if active:
            assert lmu.update_local_map(snap, tracked) == lmu.oracle_update(snap, tracked), b
        last_rows = snap["last_row_lm"][lasts_off[b]:lasts_off[b + 1]]
        w["last_local_idx"] = lmu.mapping(w["local_lm"], last_rows)
        kfr = snap["kf_row_lm"][kf_off[kf_of_frame[b]]:kf_off[kf_of_frame[b] + 1]]
        w["local_idx"] = lmu.mapping(w["local_lm"], kfr) if r["kf_stage"][b] and r["kf"]["status"][b] == 0 else \
            np.zeros(0, np.int32)
        wants.append(w)
        what = f"frame {b}"
        assert u["status"][b] == w["status"] and u["nearest"][b] == w["nearest"], (what, u["status"][b], w)
        assert list(u["local_kf"][b]) == w["local_kf"] and list(u["local_lm"][b]) == w["local_lm"], what
        rows = lmu.local_rows(snap, w["local_lm"])
        for k, v in rows.items():
            assert np.asarray(u["rows"][b][k]).tobytes() == np.asarray(v, u["rows"][b][k].dtype).tobytes(), (what, k)
        assert np.array_equal(u["last_local_idx"][b], w["last_local_idx"]), what
        assert np.array_equal(u["local_idx"][b], w["local_idx"]), what
    # the local-map stage on the device list against the oracle chain on the oracle list
    fe.track_local_map(B, lmd.MARGIN, updated=True)
    lout = fe.download_local_tracking(B)
    curr = [lmd.curr_frame_u(res[t], undistort) for t in ts]
    lists, lwants = [], []
    for b, t in enumerate(ts):
        w = wants[b]
        loc = lmu.local_rows(snap, w["local_lm"])
        lasts = seq.last_frame_landmarks(t - 1, lmd._kps(res[t - 1], undistort), res[t - 1]["desc"])
        lists.append(dict(loc, last_local_idx=w["last_local_idx"]))
        if r["kf_stage"][b]:
            kf = kfs[kf_of_frame[b]]
            src = r["rb_wants"][b] if r["rb_stage"][b] else r["kf_wants"][b]
            out = r["rb"] if r["rb_stage"][b] else r["kf"]
            tr = (src["matched_pre"], src["matched"], out["pose"][b], int(out["num_valid"][b]))
            lwants.append(lmd.oracle_local_track(orc, grid, cam, curr[b], kf, dict(loc, last_local_idx=w["local_idx"]),
                                                 tr, fe.max_local))
        else:
            mo = lmd.oracle_motion(orc, grid, cam, curr[b], lasts, preds[b], seq.poses[t - 1])
            assert np.array_equal(mo[1], r["mot"]["matched"][b]), b
            lwants.append(lmd.oracle_local_track(orc, grid, cam, curr[b], lasts, lists[b],
                                                 (mo[0], mo[1], r["mot"]["pose"][b], int(r["mot"]["num_valid"][b])),
                                                 fe.max_local))
    got_it, want_it = lmd.compare(lout, lwants)
    scene.check_lm_iters(got_it, want_it, "local map on the device list")
    # the same stage given the oracle list through set_local_maps and set_keyframes' local_idx: byte for byte
    fe.set_keyframes(kfs, kf_of_frame, [w["local_idx"] if r["kf_stage"][b] else np.zeros(0, np.int32)
                                        for b, w in enumerate(wants)])
    fe.track_keyframe(B, gv, motion_valid)
    fe.track_robust(B, rb_seed)
    fe.set_local_maps(lists)
    fe.track_local_map(B, lmd.MARGIN)
    hout = fe.download_local_tracking(B)
    assert _bytes(hout) == _bytes(lout)
    return r, u, lout


def test_update_chain_mixed_batch(ctx, orc, plp):
    """Batch of 8 over 5 keyframes (robust_track's mixed case): motion successes, a BoW success, robust rescues, a
    robust failure and shared keyframes, then the update and the local map on its list."""
    from plpslam_b200.tracking import FrontEnd
    ts = [2, 3, 4, 5, 6, 7, 8, 2]
    seq = scene.PlanarSequence(seed=41, n_frames=9)
    res = [orc.orb_extract(oracle_api.orb_params(), f) for f in seq.frames]
    ov, gv = _vocab(orc, plp, ctx, res, 5)
    fe = FrontEnd(ctx, seq.rows, seq.cols, seq.camera(plp), max_batch=8)
    try:
        fe.reserve_local_map(4096)
        fe.reserve_keyframe_track(5, 1500)
        fe.reserve_robust_track()
        fe.reserve_local_map_update(MAX_LKF)
        rng = np.random.default_rng(8)
        cam = fe.cam
        kfs = [rtd.keyframe(orc, ov, seq, res, 0, rng, cam, empty_fv=True),
               rtd.keyframe(orc, ov, seq, res, 1, rng, cam),
               rtd.keyframe(orc, ov, seq, res, 4, rng, cam, erased_frac=0.99),
               rtd.keyframe(orc, ov, seq, res, 1, rng, cam, empty_fv=True),
               rtd.keyframe(orc, ov, seq, res, 4, rng, cam, empty_fv=True)]
        r, u, lout = _chain(ctx, orc, plp, fe, ov, gv, seq, res, ts, kfs, [0, 1, 0, 2, 3, 1, 4, 0],
                            [1, 1, 0, 0, 0, 1, 0, 0], fail=(1,), seed=9, rb_seed=1234)
        assert r["rb_stage"] == [0, 0, 1, 1, 1, 0, 1, 1]
        ok = [b for b in range(8) if u["status"][b] == 0 and len(u["local_lm"][b])]
        assert len(ok) >= 6 and all(lout["num_tracked"][b] > 0 for b in ok), (u["status"], ok)
    finally:
        fe.close()
        gv.close()
        orc.bow_vocab_destroy(ov)


def test_update_leaves_tracking_records_alone(ctx, orc, plp):
    """An update does not change what the keyframe and robust stages hand to a local-map call given another list:
    keyframe -> update -> robust -> local map on the host list, and robust -> update -> a new update reservation ->
    local map on the host list, equal byte for byte to the same chain without an update (robust_track's mixed batch)."""
    from plpslam_b200.tracking import FrontEnd
    ts = [2, 3, 4, 5, 6, 7, 8, 2]
    B = len(ts)
    seq = scene.PlanarSequence(seed=41, n_frames=9)
    res = [orc.orb_extract(oracle_api.orb_params(), f) for f in seq.frames]
    ov, gv = _vocab(orc, plp, ctx, res, 5)
    fe = FrontEnd(ctx, seq.rows, seq.cols, seq.camera(plp), max_batch=8)
    try:
        fe.reserve_local_map(4096)
        fe.reserve_keyframe_track(5, 1500)
        fe.reserve_robust_track()
        fe.reserve_local_map_update(MAX_LKF)
        rng = np.random.default_rng(8)
        cam = fe.cam
        kfs = [rtd.keyframe(orc, ov, seq, res, 0, rng, cam, empty_fv=True),
               rtd.keyframe(orc, ov, seq, res, 1, rng, cam),
               rtd.keyframe(orc, ov, seq, res, 4, rng, cam, erased_frac=0.99),
               rtd.keyframe(orc, ov, seq, res, 1, rng, cam, empty_fv=True),
               rtd.keyframe(orc, ov, seq, res, 4, rng, cam, empty_fv=True)]
        kf_of_frame, motion_valid = [0, 1, 0, 2, 3, 1, 4, 0], [1, 1, 0, 0, 0, 1, 0, 0]
        # the chain without an update, checked against the oracle; its host lists and local_idx stay set
        r = rtd.run_case(orc, plp, fe, ov, gv, seq, res, ts, kfs, kf_of_frame, motion_valid, fail=(1,), seed=9,
                         rb_seed=1234)
        lmd.compare(r["local"], r["local_wants"])
        want = _bytes(r["local"])
        fe.set_map(_snapshot(seq, res, ts, kfs, np.random.default_rng(5)))
        # keyframe -> update -> robust -> local map on the host list
        fe.step(B, 20.0)
        fe.track_keyframe(B, gv, motion_valid)
        fe.update_local_map(B)
        fe.track_robust(B, 1234)
        fe.track_local_map(B, lmd.MARGIN)
        assert _bytes(fe.download_local_tracking(B)) == want
        # robust -> update -> a new update reservation -> local map on the host list
        fe.step(B, 20.0)
        fe.track_keyframe(B, gv, motion_valid)
        fe.track_robust(B, 1234)
        fe.update_local_map(B)
        fe.reserve_local_map_update(MAX_LKF)
        fe.track_local_map(B, lmd.MARGIN)
        assert _bytes(fe.download_local_tracking(B)) == want
        with pytest.raises(plp.PlpError):
            fe.track_local_map(B, lmd.MARGIN, updated=True)  # the reservation ended the update's list
    finally:
        fe.close()
        gv.close()
        orc.bow_vocab_destroy(ov)


def test_update_chain_distorted_camera(ctx, orc, plp):
    """The same chain through plp_tracker_create_ex (EuRoC's radial-tangential model); every frame falls through to the
    robust stage."""
    import camera_data as cd
    import distorted_scene
    from plpslam_b200.tracking import FrontEnd
    model, cols, rows, K, D = cd.CONFIGS["euroc_mono"]
    ts = list(range(2, 6))
    seq = distorted_scene.DistortedPlanarSequence((model, D), seed=43, n_frames=6, rows=rows, cols=cols,
                                                  fx=K[0], fy=K[1], cx=K[2], cy=K[3])
    res = [orc.orb_extract(oracle_api.orb_params(1000, 1.2, 8, 20, 7), f) for f in seq.frames]
    ov, gv = _vocab(orc, plp, ctx, res, 6)
    fe = FrontEnd(ctx, rows, cols, seq.camera(plp), max_batch=4, distortion=plp.capi.make_distortion(model, *D))
    try:
        fe.reserve_local_map(4096)
        fe.reserve_keyframe_track(2, 1500)
        fe.reserve_robust_track()
        fe.reserve_local_map_update(MAX_LKF)
        b = seq.bounds()
        grid = plp.capi.make_grid(cols, rows, min_x=b[0], min_y=b[2], max_x=b[1], max_y=b[3])
        cam = seq.camera(plp)
        cam.min_x, cam.max_x, cam.min_y, cam.max_y = (float(v) for v in b)
        rng = np.random.default_rng(10)
        kfs = [rtd.keyframe(orc, ov, seq, res, t, rng, cam, undistort=seq.undistort, empty_fv=True) for t in (0, 1)]
        r, u, _ = _chain(ctx, orc, plp, fe, ov, gv, seq, res, ts, kfs, [0, 0, 1, 1], [0, 0, 0, 0], seed=11, rb_seed=7,
                         grid=grid, cam=cam, undistort=seq.undistort)
        assert r["rb_stage"] == [1, 1, 1, 1]
    finally:
        fe.close()
        gv.close()
        orc.bow_vocab_destroy(ov)


def test_update_rejections(ctx, orc, plp):
    """No reservation, no motion call, a batch above the last tracking call's, kf_row_lm missing after a keyframe call,
    and null arrays are refused before anything is launched; the list cannot be read before an update or after a new
    tracking call, and a local-map call after an update must take its list."""
    from plpslam_b200.tracking import FrontEnd, TrackLocal, TrackMap
    ts = list(range(2, 6))
    seq = scene.PlanarSequence(seed=44, n_frames=6)
    res = [orc.orb_extract(oracle_api.orb_params(), f) for f in seq.frames]
    ov, gv = _vocab(orc, plp, ctx, res, 7)
    fe = FrontEnd(ctx, seq.rows, seq.cols, seq.camera(plp), max_batch=4)
    try:
        rng = np.random.default_rng(12)
        lib, o = fe.lib, fe.d_n_inl.ptr
        assert lib.plp_tracker_reserve_local_map_update(fe._trk, C.c_int(128)) == 1  # before reserve_local_map
        fe.reserve_local_map(4096)
        assert lib.plp_tracker_reserve_local_map_update(fe._trk, C.c_int(63)) == 1
        assert lib.plp_tracker_reserve_local_map_update(fe._trk, C.c_int(1 << 18)) == 4  # vote table beyond shared memory
        kf0 = rtd.keyframe(orc, ov, seq, res, 0, rng, fe.cam, empty_fv=True)
        snap = _snapshot(seq, res, ts, [kf0], rng)
        fe.set_map(snap)

        def call(batch, m=None):
            return lib.plp_tracker_update_local_map_batch_dev(fe._trk, C.c_int(batch), C.byref(m or fe._map), o, o, o,
                                                              fe.d_matched.ptr, o)
        ctx.sync()
        n0 = ctx.launch_count()
        assert call(2) == 1 and ctx.launch_count() == n0  # no reservation
        fe.reserve_keyframe_track(2, 1500)
        fe.reserve_local_map_update(MAX_LKF)
        assert call(2) == 1 and ctx.launch_count() == n0  # no motion call
        preds = [seq.predicted_pose(t, rng) for t in ts]
        lasts = [seq.last_frame_landmarks(t - 1, res[t - 1]["kps"], res[t - 1]["desc"]) for t in ts]
        fe.upload_images(seq.frames[ts])
        fe.set_last_frames(lasts, np.stack(preds), np.stack([seq.poses[t - 1] for t in ts]))
        fe.step(3, 20.0)
        ctx.sync()
        n0 = ctx.launch_count()
        assert call(4) == 1 and ctx.launch_count() == n0  # above the motion call's batch
        bad = TrackMap(*[getattr(fe._map, f) for f, _ in TrackMap._fields_])
        bad.row_lm = None
        assert call(3, bad) == 1 and ctx.launch_count() == n0  # a null required array
        loc = TrackLocal()
        assert lib.plp_tracker_updated_local_map(fe._trk, C.byref(loc)) == 1  # no update yet
        fe.set_keyframes([kf0], [0, 0, 0, 0])
        fe.track_keyframe(2, gv, [0, 0])
        ctx.sync()
        n0 = ctx.launch_count()
        assert call(3) == 1 and ctx.launch_count() == n0  # above the keyframe call's batch
        nokf = TrackMap(*[getattr(fe._map, f) for f, _ in TrackMap._fields_])
        nokf.kf_row_lm = None
        assert call(2, nokf) == 1 and ctx.launch_count() == n0  # kf_row_lm missing after a keyframe call
        odd = TrackMap(*[getattr(fe._map, f) for f, _ in TrackMap._fields_])
        odd.desc = C.c_void_p(fe._map.desc + 1)
        assert call(2, odd) == 1 and ctx.launch_count() == n0  # a desc that is not 4-byte aligned
        fe.update_local_map(2)
        assert lib.plp_tracker_updated_local_map(fe._trk, C.byref(loc)) == 0
        fe.set_local_maps([dict(lmu.local_rows(snap, []), last_local_idx=np.full(len(l["octave"]), -1, np.int32))
                           for l in lasts[:3]])
        fe.track_local_map(2, lmd.MARGIN)  # another list after an update: plp_track_keyframe.local_idx as before
        fe.track_local_map(2, lmd.MARGIN, updated=True)
        lo = fe._local_out

        def local_call(batch, lst):
            return lib.plp_tracker_local_map_track_batch_dev(fe._trk, C.c_int(batch), C.byref(lst), C.c_float(lmd.MARGIN),
                                                             lo["matched"].ptr, lo["local"].ptr,
                                                             fe._upd_out["observable"].ptr, lo["pose"].ptr,
                                                             lo["num_tracked"].ptr, lo["n_inliers"].ptr,
                                                             lo["lm_iters"].ptr, lo["status"].ptr)
        fe.step(3, 20.0)  # a motion call ends the list
        assert lib.plp_tracker_updated_local_map(fe._trk, C.byref(TrackLocal())) == 1
        ctx.sync()
        n0 = ctx.launch_count()
        assert local_call(2, loc) == 1 and ctx.launch_count() == n0  # the ended list is refused
        fe.track_local_map(3, lmd.MARGIN)  # the host list is taken as before
        ctx.sync()
    finally:
        fe.close()
        gv.close()
        orc.bow_vocab_destroy(ov)


def test_update_bench_batch(ctx, orc, plp):
    """bench.py's 512-frame batch over a 128-keyframe map: every frame's update equals the restatement, and the
    local-map stage runs on the device list."""
    B = 512
    fe, snap, _ = lmu.bench_setup(plp, ctx, B)
    try:
        fe.step(B, 20.0)
        fe.update_local_map(B)
        u = fe.download_local_map_update(B)
        mot = fe.download_tracking(B)
        lo = fe._last_offsets
        n_ok = 0
        for b in range(B):
            rows = snap["last_row_lm"][lo[b]:lo[b + 1]]
            tracked = np.array([rows[q] if q >= 0 else -1 for q in mot["matched"][b]], np.int32)
            w = lmu.device_update(snap, tracked, fe.max_local, lmu.BENCH_MAX_LKF, mot["num_valid"][b] >= 20)
            assert u["status"][b] == w["status"] and u["nearest"][b] == w["nearest"], b
            assert list(u["local_kf"][b]) == w["local_kf"] and list(u["local_lm"][b]) == w["local_lm"], b
            assert np.array_equal(u["last_local_idx"][b], lmu.mapping(w["local_lm"], rows) if w["status"] == 0
                                  else np.full(len(rows), -1, np.int32)), b
            n_ok += w["status"] == 0 and len(w["local_lm"]) > 0
        assert n_ok >= B // 2, n_ok
        fe.track_local_map(B, lmd.MARGIN, updated=True)
        lout = fe.download_local_tracking(B)
        assert all(s == 0 for s in lout["status"])
    finally:
        fe.close()
