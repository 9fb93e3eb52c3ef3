"""GPU parity of the batched local-map stage (plp_tracker_local_map_track_batch_dev, tracking.FrontEnd.track_local_map)
against the oracle chain extract -> motion_based_track -> search_local_landmarks -> pose_optimize -> outlier drop.

The oracle's local stage starts from the device's motion pose (the motion outputs themselves are compared with the
oracle's first): the distractor rows sit on the gates' boundaries at that pose, and a pose that differs in its last
bits could flip them."""
import ctypes as C
import importlib.util
import time

import numpy as np
import pytest

import local_map_data as lmd
import oracle_api
import scene

pytestmark = pytest.mark.gpu


def _motion_inputs(seq, res, ts, rng, fail=()):
    preds = [seq.predicted_pose(t, rng) for t in ts]
    for b in fail:  # a predicted pose a metre off: nothing projects near its match, the motion track fails
        preds[b] = preds[b].copy()
        preds[b][:3, 3] += np.array([1.0, 0.5, 0.0])
    lasts = [seq.last_frame_landmarks(t - 1, res[t - 1]["kps"], res[t - 1]["desc"]) for t in ts]
    return preds, lasts


def _chain(ctx, orc, plp, fe, seq, res, ts, preds, lasts, max_local, rng, empty=(), grid=None, cam=None,
           undistort=None, edit=None):
    fe.upload_images(seq.frames[ts])
    fe.set_last_frames(lasts, np.stack(preds), np.stack([seq.poses[t - 1] for t in ts]))
    B = len(ts)
    fe.step(B, 20.0)
    mot = fe.download_tracking(B)
    local_list, wants = lmd.chain_case(orc, seq, res, ts, preds, lasts, mot, grid or fe.grid, cam or fe.cam, rng,
                                       max_local, empty=empty, undistort=undistort)
    if edit is not None:
        local_list, wants = edit(local_list, wants, mot)
    fe.set_local_maps(local_list)
    fe.track_local_map(B, lmd.MARGIN)
    return mot, fe.download_local_tracking(B), wants


def test_local_map_chain_matches_oracle(ctx, orc, plp):
    """Batch of 7: one frame whose motion track fails, one with an empty local list, the rest with ~3 k landmarks
    from the last and two earlier keyframes plus a distractor row for every gate."""
    from plpslam_b200.tracking import FrontEnd
    ts = list(range(1, 8))
    seq = scene.PlanarSequence(seed=21, n_frames=len(ts) + 1)
    res = [orc.orb_extract(oracle_api.orb_params(), f) for f in seq.frames]
    fe = FrontEnd(ctx, seq.rows, seq.cols, seq.camera(plp), max_batch=8)
    try:
        fe.reserve_local_map(4096)
        rng = np.random.default_rng(4)
        preds, lasts = _motion_inputs(seq, res, ts, rng, fail=(2,))
        mot, out, wants = _chain(ctx, orc, plp, fe, seq, res, ts, preds, lasts, 4096, rng, empty=(4,))
        assert mot["num_valid"][2] < 20 and all(mot["num_valid"][b] >= 20 for b in range(7) if b != 2)
        got_it, want_it = lmd.compare(out, wants)
        scene.check_lm_iters(got_it, want_it, "local map")
        # the failed frame passes through with the motion pose; the tracked frames gain landmarks from the local map
        assert out["lm_iters"][2] == 0 and out["num_tracked"][2] == 0 and np.array_equal(out["pose"][2], mot["pose"][2])
        assert not out["observable"][2].any() and (out["local"][2] == -1).all() and (out["matched"][2] == -1).all()
        assert len(out["observable"][4]) == 0 and out["num_tracked"][4] >= 20
        for b in (0, 1, 3, 5, 6):
            assert (out["local"][b] >= 0).sum() > 50 and out["num_tracked"][b] > mot["num_valid"][b], b
    finally:
        fe.close()


def test_local_map_leaves_motion_outputs_alone(ctx, orc, plp):
    from plpslam_b200.tracking import FrontEnd
    ts = list(range(1, 5))
    seq = scene.PlanarSequence(seed=22, n_frames=len(ts) + 1)
    res = [orc.orb_extract(oracle_api.orb_params(), f) for f in seq.frames]
    fe = FrontEnd(ctx, seq.rows, seq.cols, seq.camera(plp), max_batch=4)
    try:
        fe.reserve_local_map(4096)
        rng = np.random.default_rng(5)
        preds, lasts = _motion_inputs(seq, res, ts, rng)
        mot, out, wants = _chain(ctx, orc, plp, fe, seq, res, ts, preds, lasts, 4096, rng)
        after = fe.download_tracking(len(ts))
        for k in ("pose", "num_valid", "n_inliers", "lm_iters", "status"):
            assert after[k].tobytes() == mot[k].tobytes(), k
        for b in range(len(ts)):
            assert after["matched"][b].tobytes() == mot["matched"][b].tobytes()
        lmd.compare(out, wants)
    finally:
        fe.close()


def test_local_map_distorted_camera(ctx, orc, plp):
    """The same chain through plp_tracker_create_ex (EuRoC's radial-tangential model): the stage reads the tracker's
    undistorted keypoints."""
    import camera_data as cd
    import distorted_scene
    from plpslam_b200.tracking import FrontEnd
    model, cols, rows, K, D = cd.CONFIGS["euroc_mono"]
    ts = list(range(1, 5))
    seq = distorted_scene.DistortedPlanarSequence((model, D), seed=23, n_frames=len(ts) + 1, rows=rows, cols=cols,
                                                  fx=K[0], fy=K[1], cx=K[2], cy=K[3])
    res = [orc.orb_extract(oracle_api.orb_params(1000, 1.2, 8, 20, 7), f) for f in seq.frames]
    dist = plp.capi.make_distortion(model, *D)
    fe = FrontEnd(ctx, rows, cols, seq.camera(plp), max_batch=4, distortion=dist)
    try:
        fe.reserve_local_map(4096)
        b = seq.bounds()
        grid = plp.capi.make_grid(cols, rows, min_x=b[0], min_y=b[2], max_x=b[1], max_y=b[3])
        cam = seq.camera(plp)
        cam.min_x, cam.max_x, cam.min_y, cam.max_y = (float(v) for v in b)
        rng = np.random.default_rng(6)
        preds, lasts = _motion_inputs(seq, res, ts, rng)
        mot, out, wants = _chain(ctx, orc, plp, fe, seq, res, ts, preds, lasts, 4096, rng, grid=grid, cam=cam,
                                 undistort=seq.undistort)
        got_it, want_it = lmd.compare(out, wants)
        scene.check_lm_iters(got_it, want_it, "distorted local map")
        assert all(out["num_tracked"][b] >= 20 for b in range(len(ts)))
    finally:
        fe.close()


def test_local_map_rejections(ctx, orc, plp):
    """A local list over the reserved capacity (status 1) and an out-of-range last_local_idx (status 2) skip their
    frames only; a call without a reservation is refused before anything is launched."""
    from plpslam_b200.tracking import FrontEnd
    ts = list(range(1, 5))
    seq = scene.PlanarSequence(seed=24, n_frames=len(ts) + 1)
    res = [orc.orb_extract(oracle_api.orb_params(), f) for f in seq.frames]
    fe = FrontEnd(ctx, seq.rows, seq.cols, seq.camera(plp), max_batch=4)
    try:
        rng = np.random.default_rng(7)
        preds, lasts = _motion_inputs(seq, res, ts, rng)
        fe.upload_images(seq.frames[ts])
        fe.set_last_frames(lasts, np.stack(preds), np.stack([seq.poses[t - 1] for t in ts]))
        fe.step(len(ts), 20.0)
        fe.set_local_maps([dict(lmd.empty_rows(), last_local_idx=np.full(len(l["octave"]), -1, np.int32)) for l in lasts])
        ctx.sync()
        n0 = ctx.launch_count()
        d = fe.d_n_inl.ptr
        st = fe.lib.plp_tracker_local_map_track_batch_dev(fe._trk, C.c_int(len(ts)), C.byref(fe._local), C.c_float(5.0),
                                                         fe.d_matched.ptr, fe.d_matched.ptr, fe.d_status.ptr,
                                                         fe.d_pose.ptr, d, d, d, d)
        assert st == 1 and ctx.launch_count() == n0  # PLP_ERR_INVALID, nothing launched
        max_local = 2500

        def edit(local_list, wants, mot):  # frame 1: a last_local_idx entry one past its local list
            lli = local_list[1]["last_local_idx"].copy()
            lli[0] = len(local_list[1]["max_valid_dist"])
            local_list[1]["last_local_idx"] = lli
            wants[1] = lmd.oracle_local_track(orc, fe.grid, fe.cam, lmd.curr_frame(res[ts[1]]), lasts[1], local_list[1],
                                              (None, None, mot["pose"][1], int(mot["num_valid"][1])), max_local)
            assert wants[1]["status"] == 2
            return local_list, wants
        fe.reserve_local_map(max_local)
        mot, out, wants = _chain(ctx, orc, plp, fe, seq, res, ts, preds, lasts, max_local, rng, edit=edit)
        sizes = [len(o) for o in out["observable"]]
        over = [b for b in (0, 2, 3) if sizes[b] > max_local]
        assert over and sizes[0] <= max_local, sizes
        assert [int(s) for s in out["status"]] == [1 if b in over else (2 if b == 1 else 0) for b in range(4)]
        for b in over + [1]:
            assert not out["observable"][b].any() and out["num_tracked"][b] == 0 and out["lm_iters"][b] == 0
            assert np.array_equal(out["pose"][b], mot["pose"][b])
        lmd.compare(out, wants)
    finally:
        fe.close()


def test_local_map_bench_batch_two_contexts(ctx, orc, plp):
    """bench.py's batch of 512 on an extraction and a tracking context: step() + track_local_map() enqueue without
    waiting for the device, and a seeded sample of frames equals the oracle."""
    spec = importlib.util.spec_from_file_location("bench_local_map", lmd.ROOT / "tools" / "bench_local_map.py")
    bench_local_map = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench_local_map)
    tctx = plp.Context(ctx.device, high_priority=True)
    fe, aux = bench_local_map.setup(plp, ctx, 512, 1234, tctx)
    try:
        for cx in (ctx, tctx):
            cx.sync()
        t0 = time.perf_counter()
        fe.step(512)
        fe.track_local_map(512)
        t_enq = time.perf_counter() - t0
        for cx in (ctx, tctx):
            cx.sync()
        t_all = time.perf_counter() - t0
        assert t_enq < 0.5 * t_all, (t_enq, t_all)
        bench_local_map.check_sample(orc, plp, fe, aux, np.random.default_rng(11).choice(512, 6, replace=False))
    finally:
        fe.close()


def test_window_matcher_ratio_path_with_whole_warps_of_invalid_queries(ctx, orc, plp):
    """plp_match_frame_and_landmarks (the ratio path the local-map stage launches) when the first 8 warps' queries are
    all invalid: their choice scratch is never scanned, and a leftover value there must not become a match.  The same
    call first runs on all-valid queries so that the pooled scratch holds real choices."""
    import synth
    curr, _, _, _ = synth.make_tracking_scene(321, n_last=900)
    grid = plp.capi.make_grid(synth.COLS, synth.ROWS)
    sf = synth.scale_factors()
    q = synth.make_landmark_queries(5, curr, m=2000)
    q["valid"] = np.ones(2000, np.uint8)
    g, _ = ctx.match_frame_and_landmarks(grid, sf, curr, q, 5.0, 0.8)
    assert (g[:64] >= 0).sum() > 10
    q["valid"][:64] = 0
    g, gn = ctx.match_frame_and_landmarks(grid, sf, curr, q, 5.0, 0.8)
    o, on = orc.match_frame_and_landmarks(grid, sf, curr, q, 5.0, 0.8)
    assert np.array_equal(g, o) and gn == on and (g[:64] == -1).all()
