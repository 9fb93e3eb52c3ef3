"""GPU parity of the batched tracker on rectified stereo frames (setup_type 1, plp_tracker_bind_stereo) against the
oracle: stereo_x_right_ from match::stereo::compute, the motion stage with the forward / backward assumption and the
x_right gate, stereo edges in every pose optimisation, and the local-map stage's x_right_in_tracking_ gate."""
import ctypes as C

import numpy as np
import pytest

import local_map_data as lmd
import oracle_api
import scene
import stereo_track_data as std
import synth

pytestmark = pytest.mark.gpu

BF = 47.906                                        # example/euroc/EuRoC_stereo.yaml: focal_x_baseline
EUROC_K = (458.654, 457.296, 367.215, 248.375)     # fx, fy, cx, cy
ROWS, COLS = 480, 752


def _stereo_sequence(plp, seed, n_frames):
    fx, fy, cx, cy = EUROC_K
    seq = scene.PlanarSequence(seed=seed, n_frames=n_frames, rows=ROWS, cols=COLS, fx=fx, fy=fy, cx=cx, cy=cy)
    return (seq,) + std.stereo_sequence(plp, seq, BF)


def _oracle_x_right(orc, fe, res_l, res_r, cam):
    xr, _, _ = orc.stereo_compute(res_l, res_r, fe.orb.scale_factors, fe.orb.inv_scale_factors, cam.focal_x_baseline,
                                  cam.true_baseline)
    return np.asarray(xr, np.float32)


def test_stereo_sequence_motion_and_local_map_match_oracle(ctx, orc, plp):
    """A rendered stereo sequence at EuRoC's K and size: x_right equals the oracle's stereo::compute, then the motion
    stage (margin 10) and the local-map stage (margin 5) equal the oracle chain with the stereo camera."""
    from plpslam_b200.tracking import FrontEnd
    ts = list(range(2, 7))  # every frame has two earlier keyframes for its local map
    B = len(ts)
    seq, cam, right = _stereo_sequence(plp, 61, B + 2)
    p = oracle_api.orb_params()
    res = [orc.orb_extract(p, f) for f in seq.frames]
    res_r = [orc.orb_extract(p, f) for f in right]
    fe = FrontEnd(ctx, ROWS, COLS, cam, max_batch=B)
    try:
        fe.reserve_local_map(4096)
        grid = fe.grid
        rng = np.random.default_rng(6)
        preds = [seq.predicted_pose(t, rng) for t in ts]
        lasts = [seq.last_frame_landmarks(t - 1, res[t - 1]["kps"], res[t - 1]["desc"]) for t in ts]
        fe.upload_images(seq.frames[ts], right[ts])
        fe.set_last_frames(lasts, np.stack(preds), np.stack([seq.poses[t - 1] for t in ts]))
        fe.extract(B)
        fe.track(B, 10.0)
        kps = fe.download_keypoints(B)
        st = fe.download_stereo(B)
        mot = fe.download_tracking(B)
        xrs = []
        for b, t in enumerate(ts):
            assert np.array_equal(kps[b][0], res[t]["kps"]), b
            want = _oracle_x_right(orc, fe, res[t], res_r[t], cam)
            assert np.array_equal(st[b][0], want), f"x_right of frame {b}"
            assert (want >= 0).sum() > 300, b
            xrs.append(want)
        # the motion stage: the oracle chain with the stereo camera and each frame's x_right
        got_it, want_it = [], []
        for b, t in enumerate(ts):
            curr = dict(lmd.curr_frame(res[t]), x_right=xrs[b])
            _, m, T, nv, n_inl, iters = std.oracle_motion(orc, grid, cam, curr, lasts[b], preds[b], seq.poses[t - 1],
                                                          margin=10.0)
            assert np.array_equal(mot["matched"][b], m), f"motion matches of frame {b}"
            assert mot["num_valid"][b] == nv and mot["n_inliers"][b] == n_inl, b
            assert np.linalg.norm(mot["pose"][b] - T) / np.linalg.norm(T) <= 1e-4, b
            assert nv >= 20 and (xrs[b][m >= 0] >= 0).sum() > 50, b  # stereo edges took part
            got_it.append(int(mot["lm_iters"][b]))
            want_it.append(iters)
        scene.check_lm_iters(got_it, want_it, "stereo motion")
        # the local-map stage, chained on the device's motion outputs
        local_list, wants = [], []
        for b, t in enumerate(ts):
            curr = dict(lmd.curr_frame(res[t]), x_right=xrs[b])
            motion = std.oracle_motion(orc, grid, cam, curr, lasts[b], preds[b], seq.poses[t - 1], margin=10.0)
            assert np.array_equal(motion[1], mot["matched"][b]), b
            loc = lmd.build_local_map(seq, res, t, rng, last_frame=lasts[b], drop_last=20)
            good = lmd.take(loc, np.arange(min(200, len(loc["max_valid_dist"]))))
            good.pop("last_local_idx")
            loc = lmd.with_rows(loc, lmd.distractors(cam, mot["pose"][b], good, rng))
            local_list.append(loc)
            dev_motion = (motion[0], motion[1], mot["pose"][b], int(mot["num_valid"][b]))
            wants.append(std.oracle_local_track(orc, grid, cam, curr, lasts[b], loc, dev_motion, 4096, 5.0))
        fe.set_local_maps(local_list)
        fe.track_local_map(B, 5.0)
        out = fe.download_local_tracking(B)
        got_it, want_it = lmd.compare(out, wants)
        scene.check_lm_iters(got_it, want_it, "stereo local map")
        for b in range(B):
            assert (out["local"][b] >= 0).sum() > 50, b
    finally:
        fe.close()


def _motion_scene_batch(seed, kinds, cam):
    """One synthetic frame per entry of kinds ("fwd", "bwd", "none"): the predicted pose is the scene's, and the last
    frame's pose puts the current camera centre's z in the last frame's coordinates above +true_baseline, below
    -true_baseline, or between."""
    frames = []
    for b, kind in enumerate(kinds):
        curr, last, Tc, _ = synth.make_tracking_scene(seed + b, n_last=600, n_extra=150, stereo=True)
        curr.pop("claimed")  # the motion track starts from a frame without landmarks (frame_tracker.cc:61)
        twc = -Tc[:3, :3].T @ Tc[:3, 3]
        z = {"fwd": 3.0, "bwd": -3.0, "none": 0.3}[kind] * cam.true_baseline
        Tl = np.eye(4)
        Tl[2, 3] = z - twc[2]
        frames.append((curr, last, Tc, Tl))
    return frames


def test_motion_stage_forward_and_backward_assumption(ctx, orc, plp):
    """Keypoint batches uploaded straight to the motion stage: frames moving forward, backward and neither, each equal
    to the oracle chain, and each kind with matches that differ from the monocular chain on the same inputs."""
    from plpslam_b200.tracking import FrontEnd
    kinds = ["fwd", "bwd", "none", "fwd", "bwd", "none"]
    B = len(kinds)
    bf = 40.0
    cam = plp.capi.make_camera(synth.FX, synth.FY, synth.CX, synth.CY, synth.COLS, synth.ROWS, bf=bf, setup_type=1)
    mono = plp.capi.make_camera(synth.FX, synth.FY, synth.CX, synth.CY, synth.COLS, synth.ROWS)
    frames = _motion_scene_batch(700, kinds, cam)
    fe = FrontEnd(ctx, synth.ROWS, synth.COLS, cam, max_batch=B, max_last_points=1200)
    try:
        grid = fe.grid
        cap = fe.cap
        kp = np.zeros((B, cap), plp.KP_DTYPE)
        desc = np.zeros((B, cap, 32), np.uint8)
        xr = np.full((B, cap), -1.0, np.float32)
        n = np.zeros(B, np.int32)
        for b, (curr, _, _, _) in enumerate(frames):
            k = len(curr["x"])
            assert k <= cap
            n[b] = k
            kp["x"][b, :k], kp["y"][b, :k] = curr["x"], curr["y"]
            kp["octave"][b, :k], kp["angle"][b, :k] = curr["octave"], curr["angle"]
            desc[b, :k] = curr["desc"]
            xr[b, :k] = curr["x_right"]
        fe.d_kp.upload(kp)
        fe.d_desc.upload(desc)
        fe.d_n.upload(n)
        fe.d_x_right.upload(xr)
        fe.set_last_frames([f[1] for f in frames], np.stack([f[2] for f in frames]), np.stack([f[3] for f in frames]))
        fe.track(B, 10.0)
        mot = fe.download_tracking(B)
        differs = set()
        for b, (curr, last, Tc, Tl) in enumerate(frames):
            w = std.oracle_motion(orc, grid, cam, curr, last, Tc, Tl, margin=10.0)
            assert np.array_equal(mot["matched"][b], w[1]), f"frame {b} ({kinds[b]})"
            assert mot["num_valid"][b] == w[3] and mot["n_inliers"][b] == w[4], b
            assert np.linalg.norm(mot["pose"][b] - w[2]) / np.linalg.norm(w[2]) <= 1e-4, b
            mono_curr = {k: v for k, v in curr.items() if k != "x_right"}
            wm = lmd.oracle_motion(orc, grid, mono, mono_curr, last, Tc, Tl, margin=10.0)
            pre_s, _ = orc.match_current_and_last_frames(grid, lmd.SF, cam, curr, Tc, Tl, last, 10.0, True)
            pre_m, _ = orc.match_current_and_last_frames(grid, lmd.SF, mono, mono_curr, Tc, Tl, last, 10.0, True)
            if not np.array_equal(pre_s, pre_m) and not np.array_equal(w[1], wm[1]):
                differs.add(kinds[b])
        assert differs == {"fwd", "bwd", "none"}, differs
    finally:
        fe.close()


def test_stereo_refusals_write_nothing(ctx, plp):
    """RGB-D, stereo with distortion, bf <= 0, a stage call with no x_right bound and a binding on a monocular tracker
    are refused: no tracker is made, and the refused call writes nothing."""
    lib = plp.lib()
    fx, fy, cx, cy = EUROC_K
    grid = plp.capi.make_grid(COLS, ROWS)
    sf = np.ascontiguousarray(synth.scale_factors(), np.float32)
    isig = np.ascontiguousarray(synth.inv_level_sigma_sq(), np.float32)

    def create(cam, dist=None):
        h = C.c_void_p(12345)
        st = lib.plp_tracker_create_ex(ctx.handle, C.byref(cam), C.byref(grid), sf.ctypes.data_as(C.c_void_p),
                                       isig.ctypes.data_as(C.c_void_p), C.c_int(8), C.c_int(2), C.c_int(1000),
                                       C.c_int(100), None if dist is None else C.byref(dist), C.byref(h))
        return st, h

    rgbd = plp.capi.make_camera(fx, fy, cx, cy, COLS, ROWS, bf=BF, setup_type=2)
    no_bf = plp.capi.make_camera(fx, fy, cx, cy, COLS, ROWS, setup_type=1)
    stereo = plp.capi.make_camera(fx, fy, cx, cy, COLS, ROWS, bf=BF, setup_type=1)
    dist = plp.capi.make_distortion(0, -0.28, 0.07, 0.0002, 0.00002, 0.0)
    for cam, d in ((rgbd, None), (no_bf, None), (stereo, dist)):
        st, h = create(cam, d)
        assert st != 0 and h.value == 12345, (cam.setup_type, d is not None)
    from plpslam_b200.tracking import DeviceBuffer, FrontEnd, TrackLast
    # a stereo tracker with nothing bound: the motion call launches nothing
    st, h = create(stereo)
    assert st == 0 and h.value
    try:
        n = DeviceBuffer.from_array(ctx, np.zeros(2, np.int32))
        outs = [DeviceBuffer.from_array(ctx, np.full(2 * 1000 * 16, 7, np.int32)) for _ in range(5)]
        last = TrackLast(*[n.ptr] * 8)
        st = lib.plp_tracker_motion_track_batch_dev(h, C.c_int(2), n.ptr, n.ptr, n.ptr, C.byref(last), C.c_float(10.0),
                                                    *[o.ptr for o in outs])
        assert st != 0 and b"plp_tracker_bind_stereo" in lib.plp_last_error()
        ctx.sync()
        for o in outs:
            assert (o.download(np.int32, (2 * 1000 * 16,)) == 7).all()
            o.free()
        n.free()
    finally:
        lib.plp_tracker_destroy(h)
    # a binding on a monocular tracker
    fe = FrontEnd(ctx, ROWS, COLS, plp.capi.make_camera(fx, fy, cx, cy, COLS, ROWS), max_batch=2)
    try:
        buf = DeviceBuffer(ctx, 2 * fe.cap * 4)
        assert lib.plp_tracker_bind_stereo(fe._trk, buf.ptr) != 0
        buf.free()
        with pytest.raises(plp.PlpError):
            fe.upload_images(np.zeros((2, ROWS, COLS), np.uint8), np.zeros((2, ROWS, COLS), np.uint8))
    finally:
        fe.close()


def _bench_batch(seq, right, B):
    """B stereo frames cycling over the frames of a short sequence that have a predecessor."""
    n = len(seq.frames) - 1
    ts = [1 + b % n for b in range(B)]
    return ts, seq.frames[ts], right[ts]


def test_stereo_bench_batch_two_contexts(ctx, orc, plp):
    """A batch of 148 stereo frames through FrontEnd's stereo mode with a separate tracking context and a separate
    right-image context: every output equals a one-context run of the same batch."""
    from plpslam_b200.tracking import FrontEnd
    B = 148
    seq, cam, right = _stereo_sequence(plp, 62, 5)
    res = [orc.orb_extract(oracle_api.orb_params(), f) for f in seq.frames]
    rng = np.random.default_rng(8)
    ts, left_imgs, right_imgs = _bench_batch(seq, right, B)
    preds = [seq.predicted_pose(t, rng) for t in ts]
    lasts = [seq.last_frame_landmarks(t - 1, res[t - 1]["kps"], res[t - 1]["desc"]) for t in ts]
    local_list = [lmd.build_local_map(seq, res, t, np.random.default_rng(b), last_frame=lasts[b], drop_last=20)
                  for b, t in enumerate(ts)]

    def run(track_ctx, right_ctx):
        fe = FrontEnd(ctx, ROWS, COLS, cam, max_batch=B, track_ctx=track_ctx, right_ctx=right_ctx)
        try:
            fe.reserve_local_map(4096)
            fe.upload_images(left_imgs, right_imgs)
            fe.set_last_frames(lasts, np.stack(preds), np.stack([seq.poses[t - 1] for t in ts]))
            fe.set_local_maps(local_list)
            for cx in {ctx, track_ctx or ctx, right_ctx or ctx}:
                cx.sync()
            fe.extract(B)
            fe.track(B, 10.0)
            fe.track_local_map(B, 5.0)
            return fe.download_stereo(B), fe.download_tracking(B), fe.download_local_tracking(B)
        finally:
            fe.close()

    tctx, rctx = plp.Context(ctx.device), plp.Context(ctx.device)
    try:
        two = run(tctx, rctx)
    finally:
        tctx.close()
        rctx.close()
    one = run(None, None)
    for b in range(B):
        assert np.array_equal(two[0][b][0], one[0][b][0]) and np.array_equal(two[0][b][1], one[0][b][1]), b
    for k in ("pose", "num_valid", "n_inliers", "lm_iters", "status"):
        assert np.array_equal(two[1][k], one[1][k]), k
    for k in ("pose", "num_tracked", "n_inliers", "lm_iters", "status"):
        assert np.array_equal(two[2][k], one[2][k]), k
    for b in range(B):
        assert np.array_equal(two[1]["matched"][b], one[1]["matched"][b]), b
        for k in ("matched", "local", "observable"):
            assert np.array_equal(two[2][k][b], one[2][k][b]), (k, b)
    assert sum((one[1]["num_valid"] >= 20)) > B // 2


def test_keyframe_and_robust_stages_on_a_stereo_tracker(ctx, orc, plp):
    """The mixed batch of the robust-track tests on a stereo tracker: motion, keyframe and robust stages, each frame's
    matches, counts, outlier flags and pose equal to the oracle's pose optimisation with stereo edges."""
    import keyframe_track_data as ktd
    import robust_track_data as rtd
    from plpslam_b200.tracking import FrontEnd
    ts = [2, 3, 4, 5, 6, 7, 8, 2]
    B = len(ts)
    seq = scene.PlanarSequence(seed=41, n_frames=9)
    cam, right = std.stereo_sequence(plp, seq, 40.0)
    res = [orc.orb_extract(oracle_api.orb_params(), f) for f in seq.frames]
    v = ktd.make_scene_vocab(np.concatenate([r["desc"] for r in res]), 5)
    ov = orc.bow_vocab_create(v["k"], v["L"], v["parent"], v["desc"], v["weight"], v["is_leaf"])
    gv = plp.BowVocabulary(ctx, k=v["k"], L=v["L"], parent=v["parent"], desc=v["desc"], weight=v["weight"],
                           is_leaf=v["is_leaf"])
    fe = FrontEnd(ctx, seq.rows, seq.cols, cam, max_batch=B)
    try:
        fe.reserve_keyframe_track(5, 1500)
        fe.reserve_robust_track()
        rng = np.random.default_rng(8)
        kfs = [rtd.keyframe(orc, ov, seq, res, 0, rng, cam, empty_fv=True),
               rtd.keyframe(orc, ov, seq, res, 1, rng, cam),
               rtd.keyframe(orc, ov, seq, res, 4, rng, cam, erased_frac=0.99),
               rtd.keyframe(orc, ov, seq, res, 1, rng, cam, empty_fv=True),
               rtd.keyframe(orc, ov, seq, res, 4, rng, cam, empty_fv=True)]
        kf_of_frame = [0, 1, 0, 2, 3, 1, 4, 0]
        motion_valid = [1, 1, 0, 0, 0, 1, 0, 0]
        rng = np.random.default_rng(9)
        preds = [seq.predicted_pose(t, rng) for t in ts]
        preds[1] = preds[1].copy()
        preds[1][:3, 3] += np.array([1.0, 0.5, 0.0])  # a metre off: frame 1's motion track fails
        lasts = [seq.last_frame_landmarks(t - 1, res[t - 1]["kps"], res[t - 1]["desc"]) for t in ts]
        pose_last = [seq.poses[t - 1] for t in ts]
        fe.upload_images(seq.frames[ts], right[ts])
        fe.set_last_frames(lasts, np.stack(preds), np.stack(pose_last))
        fe.step(B, 20.0)
        mot = fe.download_tracking(B)
        xr = fe.download_stereo(B)
        curr = [dict(lmd.curr_frame(res[t]), x_right=xr[b][0]) for b, t in enumerate(ts)]
        for b in range(B):
            w = std.oracle_motion(orc, fe.grid, cam, curr[b], lasts[b], preds[b], pose_last[b])
            assert np.array_equal(mot["matched"][b], w[1]) and mot["num_valid"][b] == w[3], f"motion {b}"
        # the keyframe stage
        kf_stage = [int(motion_valid[b] == 0 or mot["num_valid"][b] < 20) for b in range(B)]
        assert kf_stage == [0, 1, 1, 1, 1, 0, 1, 1], kf_stage
        kf_wants = [std.oracle_keyframe_track(orc, ov, cam, curr[b], kfs[kf_of_frame[b]], pose_last[b])
                    if kf_stage[b] else None for b in range(B)]
        fe.set_keyframes(kfs, kf_of_frame)
        fe.track_keyframe(B, gv, motion_valid)
        kout = fe.download_keyframe_tracking(B)
        got_it, want_it = ktd.compare(kout, kf_wants, kf_stage)
        scene.check_lm_iters(got_it, want_it, "keyframe track")
        assert kout["num_valid"][1] >= 20 and (xr[1][0][kout["matched"][1] >= 0] >= 0).sum() > 50
        # the robust stage
        rb_stage = [int(kf_stage[b] and kf_wants[b]["num_valid"] < 20) for b in range(B)]
        assert rb_stage == [0, 0, 1, 1, 1, 0, 1, 1], rb_stage
        fe.track_robust(B, 1234)
        out = fe.download_robust_tracking(B)
        rb_wants = [std.oracle_robust_track(orc, cam, curr[b], kfs[kf_of_frame[b]],
                                            rtd.bearings(cam, curr[b]["x"], curr[b]["y"]), out["samples"][b],
                                            pose_last[b]) if rb_stage[b] else None for b in range(B)]
        got_it, want_it = rtd.compare(out, rb_wants, rb_stage, 1234)
        scene.check_lm_iters(got_it, want_it, "robust track")
        for b in (2, 4, 6, 7):
            assert out["num_valid"][b] >= 20 and (xr[b][0][out["matched"][b] >= 0] >= 0).sum() > 20, b
    finally:
        fe.close()
        gv.close()
        orc.bow_vocab_destroy(ov)
