"""GPU parity of the batched robust tracker (plp_tracker_robust_track_batch_dev, tracking.FrontEnd.track_robust) against
the oracle chain brute_force_match (0.8, no orientation check) -> ordered pair list -> essential RANSAC with the
device's sample sets -> pose optimiser -> discard_outliers, and of the local-map stage that follows it against
optimize_current_frame_with_local_map from each frame's successful tracker."""
import ctypes as C

import numpy as np
import pytest

import keyframe_track_data as ktd
import local_map_data as lmd
import oracle_api
import robust_track_data as rtd
import scene

pytestmark = pytest.mark.gpu


def _vocab(orc, plp, ctx, res, seed):
    v = ktd.make_scene_vocab(np.concatenate([r["desc"] for r in res]), seed)
    ov = orc.bow_vocab_create(v["k"], v["L"], v["parent"], v["desc"], v["weight"], v["is_leaf"])
    gv = plp.BowVocabulary(ctx, k=v["k"], L=v["L"], parent=v["parent"], desc=v["desc"], weight=v["weight"],
                           is_leaf=v["is_leaf"])
    return ov, gv


def _check(r, seed):
    got_it, want_it = ktd.compare(r["kf"], r["kf_wants"], r["kf_stage"])
    scene.check_lm_iters(got_it, want_it, "keyframe track")
    got_it, want_it = rtd.compare(r["rb"], r["rb_wants"], r["rb_stage"], seed)
    scene.check_lm_iters(got_it, want_it, "robust track")
    got_it, want_it = lmd.compare(r["local"], r["local_wants"])
    scene.check_lm_iters(got_it, want_it, "local map after the robust track")


def test_robust_track_mixed_batch_matches_oracle(ctx, orc, plp):
    """Batch of 8 over 5 keyframes: motion track succeeded (0, 5); motion failed and the BoW track succeeded (1); the
    BoW track of frames 2, 4, 6 and 7 finds nothing (their keyframes' bow_feat_vec_ is empty) and the robust stage
    rescues them (2 and 7 share a keyframe); frame 3's keyframe has 99 % of its landmarks erased, so both stages fail."""
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
        rng = np.random.default_rng(8)
        cam = fe.cam
        kfs = [rtd.keyframe(orc, ov, seq, res, 0, rng, cam, empty_fv=True),
               rtd.keyframe(orc, ov, seq, res, 1, rng, cam),
               rtd.keyframe(orc, ov, seq, res, 4, rng, cam, erased_frac=0.99),
               rtd.keyframe(orc, ov, seq, res, 1, rng, cam, empty_fv=True),
               rtd.keyframe(orc, ov, seq, res, 4, rng, cam, empty_fv=True)]
        kf_of_frame = [0, 1, 0, 2, 3, 1, 4, 0]
        r = rtd.run_case(orc, plp, fe, ov, gv, seq, res, ts, kfs, kf_of_frame, [1, 1, 0, 0, 0, 1, 0, 0], fail=(1,),
                         seed=9, rb_seed=1234)
        assert r["kf_stage"] == [0, 1, 1, 1, 1, 0, 1, 1], r["kf_stage"]
        assert r["rb_stage"] == [0, 0, 1, 1, 1, 0, 1, 1], r["rb_stage"]
        _check(r, 1234)
        out, lout = r["rb"], r["local"]
        for b in (2, 4, 6, 7):
            assert out["num_bf_matches"][b] >= 100 and out["num_valid"][b] >= 20, (b, out["num_valid"][b])
            assert lout["num_tracked"][b] > 0 and lout["status"][b] == 0, b
        assert out["num_bf_matches"][3] < 20 and out["num_valid"][3] == 0 and out["lm_iters"][3] == 0
        assert np.array_equal(out["pose"][3], seq.poses[ts[3] - 1])
        assert lout["num_tracked"][3] == 0
        # the winner's inlier flags, E and score of every frame that ran the RANSAC equal plp_essential_ransac's
        for b in (2, 4, 6, 7):
            w = r["rb_wants"][b]
            valid, inl, E, score = ctx.essential_ransac(r["frm_bearings"][b], kfs[kf_of_frame[b]]["bearings"],
                                                        w["pairs"], out["samples"][b])
            assert valid == w["valid"] == 1 and np.array_equal(inl, w["inlier"]), b
            assert np.array_equal(E, w["E"]) and score == w["score"], b
    finally:
        fe.close()
        gv.close()
        orc.bow_vocab_destroy(ov)


def test_robust_track_distorted_camera(ctx, orc, plp):
    """The same chain through plp_tracker_create_ex (EuRoC's radial-tangential model): the frame bearings are the
    undistortion's; every frame falls through to the robust stage."""
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
        b = seq.bounds()
        grid = plp.capi.make_grid(cols, rows, min_x=b[0], min_y=b[2], max_x=b[1], max_y=b[3])
        cam = seq.camera(plp)
        cam.min_x, cam.max_x, cam.min_y, cam.max_y = (float(v) for v in b)
        rng = np.random.default_rng(10)
        kfs = [rtd.keyframe(orc, ov, seq, res, t, rng, cam, undistort=seq.undistort, empty_fv=True) for t in (0, 1)]
        r = rtd.run_case(orc, plp, fe, ov, gv, seq, res, ts, kfs, [0, 0, 1, 1], [0, 0, 0, 0], seed=11, rb_seed=7,
                         grid=grid, cam=cam, undistort=seq.undistort)
        assert r["rb_stage"] == [1, 1, 1, 1]
        # the frame bearings the device read are the undistortion's
        und = fe.download_undistorted(len(ts))
        for bb in range(len(ts)):
            assert np.array_equal(und[bb][1], r["frm_bearings"][bb]), bb
        _check(r, 7)
        assert all(r["rb"]["num_valid"][bb] >= 20 for bb in range(len(ts)))
    finally:
        fe.close()
        gv.close()
        orc.bow_vocab_destroy(ov)


def test_robust_track_rejections(ctx, orc, plp):
    """Calls without a reservation, without a keyframe call since the last motion call, or with a batch above the
    keyframe call's are refused before anything is launched; keyframe status 1 and 2 carry over and those frames fail
    like a track with no match."""
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
        fe.step(4, 20.0)
        cam = fe.cam
        kf0 = rtd.keyframe(orc, ov, seq, res, 0, rng, cam, empty_fv=True)
        big = len(kf0["desc"])  # the reservation; keyframe 1 is keyframe 0 with one row more
        kf1 = {k: (np.concatenate([v, v[:1]]) if k in ("desc", "angle", "valid", "pos_w", "bearings") else v)
               for k, v in kf0.items()}
        fe.reserve_keyframe_track(2, big)
        fe.set_keyframes([kf0, kf1], [0, 5, 1, 0])
        lib, o = fe.lib, fe.d_n_inl.ptr

        def call(batch):
            return lib.plp_tracker_robust_track_batch_dev(fe._trk, C.c_int(batch), fe._kf_bearings.ptr, C.c_uint64(0),
                                                          o, fe.d_matched.ptr, o, o, fe.d_pose.ptr, o, o, o, o)
        ctx.sync()
        n0 = ctx.launch_count()
        assert call(3) == 1 and ctx.launch_count() == n0  # no reservation
        fe.reserve_robust_track()
        assert call(3) == 1 and ctx.launch_count() == n0  # no keyframe call since the motion call
        fe.track_keyframe(3, gv, [0, 0, 0])
        ctx.sync()
        n0 = ctx.launch_count()
        assert call(4) == 1 and ctx.launch_count() == n0  # batch above the keyframe call's
        fe.step(4, 20.0)  # a motion call clears the keyframe record
        ctx.sync()
        n0 = ctx.launch_count()
        assert call(3) == 1 and ctx.launch_count() == n0
        fe.track_keyframe(3, gv, [0, 0, 0])
        fe.track_robust(3, 5)
        out = fe.download_robust_tracking(3)
        assert list(out["status"]) == [0, 2, 1] and list(out["stage"]) == [1, 1, 1]
        for b in (1, 2):
            assert out["num_valid"][b] == 0 and out["num_bf_matches"][b] == 0 and (out["matched"][b] == -1).all()
            assert out["num_robust_matches"][b] == 0 and (out["samples"][b] == -1).all()
            assert out["lm_iters"][b] == 0 and np.array_equal(out["pose"][b], seq.poses[ts[b] - 1])
        assert out["num_valid"][0] >= 20
    finally:
        fe.close()
        gv.close()
        orc.bow_vocab_destroy(ov)
