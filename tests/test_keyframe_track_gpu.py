"""GPU parity of the batched keyframe tracker (plp_tracker_keyframe_track_batch_dev, tracking.FrontEnd.track_keyframe)
against the oracle chain transform -> fold_bow -> bow_tree -> pose optimiser -> discard_outliers, and of the local-map
stage that follows it against optimize_current_frame_with_local_map from each frame's successful tracker."""
import ctypes as C

import numpy as np
import pytest

import keyframe_track_data as ktd
import local_map_data as lmd
import oracle_api
import scene

pytestmark = pytest.mark.gpu


def _vocab(orc, plp, ctx, res, seed):
    v = ktd.make_scene_vocab(np.concatenate([r["desc"] for r in res]), seed)
    ov = orc.bow_vocab_create(v["k"], v["L"], v["parent"], v["desc"], v["weight"], v["is_leaf"])
    gv = plp.BowVocabulary(ctx, k=v["k"], L=v["L"], parent=v["parent"], desc=v["desc"], weight=v["weight"],
                           is_leaf=v["is_leaf"])
    return ov, gv


def _check(mot, out, wants, stage, lout, lwants):
    got_it, want_it = ktd.compare(out, wants, stage)
    scene.check_lm_iters(got_it, want_it, "keyframe track")
    got_it, want_it = lmd.compare(lout, lwants)
    scene.check_lm_iters(got_it, want_it, "local map after the keyframe track")


def test_keyframe_track_mixed_batch_matches_oracle(ctx, orc, plp):
    """Batch of 7 over 3 keyframes (frames share them): motion track succeeded (0, 2, 4), failed (1, 5), motion model
    unusable (3); frame 6's keyframe has almost every landmark erased, so it finds fewer than 20 BoW matches."""
    from plpslam_b200.tracking import FrontEnd
    ts = list(range(2, 9))
    seq = scene.PlanarSequence(seed=41, n_frames=9)
    res = [orc.orb_extract(oracle_api.orb_params(), f) for f in seq.frames]
    ov, gv = _vocab(orc, plp, ctx, res, 5)
    fe = FrontEnd(ctx, seq.rows, seq.cols, seq.camera(plp), max_batch=8)
    try:
        fe.reserve_local_map(4096)
        fe.reserve_keyframe_track(4, 1500)
        rng = np.random.default_rng(8)
        kfs = [ktd.keyframe(orc, ov, seq, res, 0, rng), ktd.keyframe(orc, ov, seq, res, 1, rng),
               ktd.keyframe(orc, ov, seq, res, 4, rng, erased_frac=0.99)]
        kf_of_frame = [0, 0, 0, 1, 1, 1, 2]
        mot, out, wants, stage, lout, lwants = ktd.run_case(orc, plp, fe, ov, gv, seq, res, ts, kfs, kf_of_frame,
                                                            [1, 1, 1, 0, 1, 1, 0], fail=(1, 5), seed=9)
        assert stage == [0, 1, 0, 1, 0, 1, 1], stage
        _check(mot, out, wants, stage, lout, lwants)
        assert out["num_bow_matches"][6] < 20 and out["num_valid"][6] == 0 and out["lm_iters"][6] == 0
        assert np.array_equal(out["pose"][6], seq.poses[ts[6] - 1])
        for b in (1, 3, 5):
            assert out["num_valid"][b] >= 20 and lout["num_tracked"][b] > out["num_valid"][b], b
        assert lout["num_tracked"][6] == 0 and lout["status"][6] == 0
        # the BoW rows of the frames that ran the stage equal plp_bow_transform's
        kps = fe.download_keypoints(len(ts))
        for b in (1, 3, 5, 6):
            for g, w in zip(out["bow"][b], gv.transform(kps[b][1], 4)):
                assert np.array_equal(g, w)
    finally:
        fe.close()
        gv.close()
        orc.bow_vocab_destroy(ov)


def test_keyframe_track_distorted_camera(ctx, orc, plp):
    """The same chain through plp_tracker_create_ex (EuRoC's radial-tangential model): every frame runs the stage."""
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
        b = seq.bounds()
        grid = plp.capi.make_grid(cols, rows, min_x=b[0], min_y=b[2], max_x=b[1], max_y=b[3])
        cam = seq.camera(plp)
        cam.min_x, cam.max_x, cam.min_y, cam.max_y = (float(v) for v in b)
        rng = np.random.default_rng(10)
        kfs = [ktd.keyframe(orc, ov, seq, res, t, rng, undistort=seq.undistort) for t in (0, 1)]
        mot, out, wants, stage, lout, lwants = ktd.run_case(orc, plp, fe, ov, gv, seq, res, ts, kfs, [0, 0, 1, 1],
                                                            [0, 0, 0, 0], seed=11, grid=grid, cam=cam,
                                                            undistort=seq.undistort)
        assert stage == [1, 1, 1, 1]
        _check(mot, out, wants, stage, lout, lwants)
        assert all(out["num_valid"][b] >= 20 for b in range(len(ts)))
    finally:
        fe.close()
        gv.close()
        orc.bow_vocab_destroy(ov)


def test_keyframe_track_rejections(ctx, orc, plp):
    """kf_of_frame out of range (status 2) and a keyframe over the reserved rows (status 1) skip their frames only; a
    keyframe-tracked frame without local_idx gets local-map status 2; calls without a reservation, with too many
    keyframes or with a batch above the motion track's are refused before anything is launched."""
    from plpslam_b200.tracking import FrontEnd
    ts = list(range(2, 6))
    seq = scene.PlanarSequence(seed=44, n_frames=6)
    res = [orc.orb_extract(oracle_api.orb_params(), f) for f in seq.frames]
    ov, gv = _vocab(orc, plp, ctx, res, 7)
    fe = FrontEnd(ctx, seq.rows, seq.cols, seq.camera(plp), max_batch=4)
    try:
        rng = np.random.default_rng(12)
        preds = [seq.predicted_pose(t, rng) for t in ts]
        lasts = [seq.last_frame_landmarks(t - 1, res[t - 1]["kps"], res[t - 1]["desc"]) for t in ts]
        fe.upload_images(seq.frames[ts])
        fe.set_last_frames(lasts, np.stack(preds), np.stack([seq.poses[t - 1] for t in ts]))
        fe.step(3, 20.0)
        kf0 = ktd.keyframe(orc, ov, seq, res, 0, rng)
        big = len(kf0["desc"])  # the reservation; keyframe 1 is keyframe 0 with one row more
        kf1 = {k: (np.concatenate([v, v[:1]]) if k in ("desc", "angle", "valid", "pos_w") else v) for k, v in kf0.items()}
        kfs = [kf0, kf1]
        fe.set_keyframes(kfs, [0, 5, 1, 0])
        lib, o = fe.lib, fe.d_n_inl.ptr

        def call(batch):
            return lib.plp_tracker_keyframe_track_batch_dev(fe._trk, gv.handle, C.c_int(batch), C.byref(fe._kf), None,
                                                            o, fe.d_matched.ptr, o, fe.d_pose.ptr, o, o, o, o)
        ctx.sync()
        n0 = ctx.launch_count()
        assert call(3) == 1 and ctx.launch_count() == n0  # no reservation
        fe.reserve_keyframe_track(1, big)
        assert call(3) == 1 and ctx.launch_count() == n0  # two keyframes, one reserved
        fe.reserve_keyframe_track(2, big)
        assert call(4) == 1 and ctx.launch_count() == n0  # batch above the motion track's
        fe.reserve_local_map(4096)
        fe.track_keyframe(3, gv, [0, 0, 0])
        out = fe.download_keyframe_tracking(3)
        assert list(out["status"]) == [0, 2, 1] and list(out["stage"]) == [1, 1, 1]
        for b in (1, 2):
            assert out["num_valid"][b] == 0 and out["num_bow_matches"][b] == 0 and (out["matched"][b] == -1).all()
            assert out["lm_iters"][b] == 0 and np.array_equal(out["pose"][b], seq.poses[ts[b] - 1])
        assert out["num_valid"][0] >= 20
        # frame 0 tracked against its keyframe, but set_keyframes gave no local_idx: local-map status 2
        fe.set_local_maps([dict(lmd.empty_rows(), last_local_idx=np.full(len(l["octave"]), -1, np.int32))
                           for l in lasts[:3]])
        fe.track_local_map(3, lmd.MARGIN)
        lout = fe.download_local_tracking(3)
        assert list(lout["status"]) == [2, 0, 0] and (lout["num_tracked"] == 0).all()
        assert np.array_equal(lout["pose"][0], out["pose"][0])
    finally:
        fe.close()
        gv.close()
        orc.bow_vocab_destroy(ov)
