"""GPU parity of keypoint undistortion (camera::{perspective,fisheye}::undistort_keypoints, convert_keypoints_to_bearings,
compute_image_bounds) and of the batched front end for distorted cameras.  Every comparison is with the oracle, which
tests/test_camera_oracle.py pins to cv2; the coordinates and bearings must be bit-identical."""
import ctypes as C

import numpy as np
import pytest

import camera_data as cd
import distorted_scene
import oracle_api
import scene
import synth

pytestmark = pytest.mark.gpu
KP_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"),
                     ("octave", "<i4"), ("class_id", "<i4")])


def _dist(plp, model, D):
    return plp.capi.make_distortion(model, *(list(D)[:4] if model == cd.FISHEYE else list(D)))


def _kps(x, y, rng):
    k = np.zeros(len(x), KP_DTYPE)
    k["x"], k["y"] = x, y
    k["size"] = rng.uniform(1, 40, len(x))
    k["angle"] = rng.uniform(0, 360, len(x))
    k["response"] = rng.uniform(0, 1, len(x))
    k["octave"] = rng.integers(0, 8, len(x))
    k["class_id"] = 7
    return k


def _check(orc, model, K, D, kin, kout, bear, what):
    wx, wy = cd.undistort_keypoints(orc, model, K, D, kin["x"], kin["y"])
    assert np.array_equal(kout["x"].view(np.uint32), wx.view(np.uint32)), f"{what}: x"
    assert np.array_equal(kout["y"].view(np.uint32), wy.view(np.uint32)), f"{what}: y"
    assert np.array_equal(kout["angle"], kin["angle"]) and np.array_equal(kout["size"], kin["size"])
    assert np.array_equal(kout["octave"], kin["octave"])
    assert (kout["response"] == 0).all() and (kout["class_id"] == -1).all()
    if bear is not None:
        assert np.array_equal(bear.view(np.uint64), cd.bearings(orc, K, wx, wy).view(np.uint64)), f"{what}: bearings"


@pytest.mark.parametrize("name", list(cd.ALL))
def test_undistort_host_equals_oracle(ctx, orc, plp, name):
    model, cols, rows, K, D = cd.ALL[name]
    x, y = cd.test_points(cols, rows, seed=11)
    xs, ys = cd.orb_level_coordinates(cols, rows, synth.scale_factors())
    rng = np.random.default_rng(12)
    x = np.concatenate([x, xs, rng.choice(xs, len(ys))]).astype(np.float32)
    y = np.concatenate([y, rng.choice(ys, len(xs)), ys]).astype(np.float32)
    kin = _kps(x, y, rng)
    cam = plp.capi.make_camera(*K, cols, rows)
    kout, bear = ctx.undistort_keypoints(cam, _dist(plp, model, D), kin)
    _check(orc, model, K, D, kin, kout, bear, name)
    # empty input: PLP_OK, nothing written
    e, eb = ctx.undistort_keypoints(cam, _dist(plp, model, D), kin[:0])
    assert len(e) == 0 and len(eb) == 0


@pytest.mark.parametrize("name", list(cd.ALL))
def test_image_bounds_equal_oracle(plp, orc, name):
    model, cols, rows, K, D = cd.ALL[name]
    got = plp.capi.image_bounds(plp.capi.make_camera(*K, cols, rows), _dist(plp, model, D), cols, rows)
    assert np.array_equal(got.view(np.uint32), cd.image_bounds(orc, model, K, D, cols, rows).view(np.uint32))


@pytest.mark.parametrize("name,batch", [("euroc_mono", 3), ("tum_mono_2", 3), ("tumvi_fisheye", 3), ("tum_mono_1", 256)])
def test_undistort_batch_dev_after_orb_extract(ctx, orc, plp, name, batch):
    """plp_undistort_keypoints_batch_dev chained on the device after plp_orb_extract_batch_dev; frame 1 is blank (no
    keypoints)."""
    from plpslam_b200.tracking import DeviceBuffer, FrontEnd
    model, cols, rows, K, D = cd.ALL[name]
    seq = scene.PlanarSequence(seed=21, n_frames=3, rows=rows, cols=cols, fx=K[0], fy=K[1], cx=K[2], cy=K[3])
    imgs = np.stack([seq.frames[b % 3] for b in range(batch)])
    imgs[1] = 0
    fe = FrontEnd(ctx, rows, cols, plp.capi.make_camera(*K, cols, rows), max_batch=batch)
    try:
        fe.upload_images(imgs)
        fe.extract(batch)
        out = DeviceBuffer(ctx, batch * fe.cap * 28)
        bear = DeviceBuffer(ctx, batch * fe.cap * 24)
        ctx.undistort_keypoints_dev(fe.cam, _dist(plp, model, D), batch, fe.cap, fe.d_kp.ptr, fe.d_n.ptr, out.ptr, bear.ptr)
        kps = fe.download_keypoints(batch)
        n = fe.d_n.download(np.int32, (batch,))
        assert n[1] == 0 and (n[np.arange(batch) != 1] > 500).all()
        ko = out.download(plp.capi.KP_DTYPE, (batch, fe.cap))
        bo = bear.download(np.float64, (batch, fe.cap, 3))
        for b in range(batch) if batch <= 8 else [0, 1, 2, 100, batch - 1]:
            _check(orc, model, K, D, kps[b][0], ko[b, :n[b]], bo[b, :n[b]], f"{name} frame {b}")
        out.free()
        bear.free()
    finally:
        fe.close()


@pytest.mark.parametrize("name", ["euroc_mono", "tum_mono_1", "tumvi_fisheye"])
def test_front_end_with_distortion(ctx, orc, plp, name):
    """tracking.FrontEnd with a distortion on an extraction and a high-priority tracking context, two steps over two
    input sets: matches, counts and poses equal the oracle chain (undistort -> grid from the undistorted bounds ->
    match -> pose-opt), and download_undistorted equals the oracle's undistortion."""
    from plpslam_b200.tracking import FrontEnd
    model, cols, rows, K, D = cd.CONFIGS[name]
    dist = (model, D)
    B = 4
    seq = distorted_scene.DistortedPlanarSequence(dist, seed=13, n_frames=2 * B + 1, rows=rows, cols=cols, fx=K[0],
                                                  fy=K[1], cx=K[2], cy=K[3])
    p = oracle_api.orb_params(1000, 1.2, 8, 20, 7)
    res = [orc.orb_extract(p, f) for f in seq.frames]
    tctx = plp.Context(ctx.device, high_priority=True)
    fe = FrontEnd(ctx, rows, cols, seq.camera(plp), max_batch=8, track_ctx=tctx, distortion=_dist(plp, model, D))
    try:
        rng = np.random.default_rng(5)
        for step in range(2):
            ts = list(range(1 + step * B, 1 + (step + 1) * B))
            preds = [seq.predicted_pose(t, rng) for t in ts]
            lasts = [seq.last_frame_landmarks(t - 1, res[t - 1]["kps"], res[t - 1]["desc"]) for t in ts]
            fe.upload_images(seq.frames[ts])
            fe.set_last_frames(lasts, np.stack(preds), np.stack([seq.poses[t - 1] for t in ts]))
            fe.step(B, 20.0)
            kps = fe.download_keypoints(B)
            und = fe.download_undistorted(B)
            out = fe.download_tracking(B)
            assert not out["status"].any()
            want_iters = []
            for b, t in enumerate(ts):
                assert np.array_equal(kps[b][0], res[t]["kps"]) and np.array_equal(kps[b][1], res[t]["desc"])
                _check(orc, model, K, D, res[t]["kps"], und[b][0], und[b][1], f"{name} step {step} frame {b}")
                m, T, nv, n_inl, iters = distorted_scene.oracle_track(orc, plp, seq, res, t, preds[b])
                what = f"{name} step {step} frame {b}"
                assert np.array_equal(out["matched"][b], m), what
                assert out["num_valid"][b] == nv and out["n_inliers"][b] == n_inl, what
                assert nv >= 20, what
                want_iters.append(iters)
                rel = np.linalg.norm(out["pose"][b] - T) / np.linalg.norm(T)
                assert rel < 1e-8, (what, rel)
            scene.check_lm_iters(out["lm_iters"], want_iters, f"{name} step {step}")
    finally:
        fe.close()
        tctx.close()


def test_zero_distortion_tracker_is_the_plain_tracker(ctx, orc, plp):
    """plp_tracker_create_ex with a zero perspective distortion: bit-identical outputs and the same launch count as
    plp_tracker_create."""
    from plpslam_b200.tracking import FrontEnd
    B = 4
    seq = scene.PlanarSequence(seed=31, n_frames=B + 1)
    p = oracle_api.orb_params(1000, 1.2, 8, 20, 7)
    res = [orc.orb_extract(p, f) for f in seq.frames[:B]]
    rng = np.random.default_rng(9)
    preds = np.stack([seq.predicted_pose(t, rng) for t in range(1, B + 1)])
    lasts = [seq.last_frame_landmarks(t - 1, res[t - 1]["kps"], res[t - 1]["desc"]) for t in range(1, B + 1)]
    outs, counts = [], []
    for dist in (None, plp.capi.make_distortion(0, 0.0, 0.0, 0.0, 0.0, 0.0)):
        fe = FrontEnd(ctx, seq.rows, seq.cols, seq.camera(plp), max_batch=8)
        try:
            if dist is not None:  # same camera and grid, tracker made through the _ex entry point
                h = C.c_void_p()
                sf = np.ascontiguousarray(fe.orb.scale_factors, np.float32)
                isig = np.ascontiguousarray(fe.orb.inv_level_sigma_sq, np.float32)
                ctx._check(fe.lib.plp_tracker_create_ex(ctx.handle, C.byref(fe.cam), C.byref(fe.grid), sf.ctypes.data_as(C.c_void_p),
                                                        isig.ctypes.data_as(C.c_void_p), C.c_int(8), C.c_int(8),
                                                        C.c_int(fe.cap), C.c_int(fe.max_last), C.byref(dist), C.byref(h)))
                fe.lib.plp_tracker_destroy(fe._trk)
                fe._trk = h
                assert fe.lib.plp_tracker_undistorted(h, C.byref(C.c_void_p()), C.byref(C.c_void_p())) != 0
            fe.upload_images(seq.frames[1:B + 1])
            fe.set_last_frames(lasts, preds, np.stack(seq.poses[0:B]))
            ctx.sync()
            c0 = ctx.launch_count()
            fe.step(B, 20.0)
            ctx.sync()
            counts.append(ctx.launch_count() - c0)
            outs.append(fe.download_tracking(B))
        finally:
            fe.close()
    assert counts[0] == counts[1]
    for k in ("pose", "num_valid", "n_inliers", "lm_iters"):
        assert np.array_equal(outs[0][k], outs[1][k]), k
    for b in range(B):
        assert np.array_equal(outs[0]["matched"][b], outs[1]["matched"][b])
    assert (outs[0]["num_valid"] >= 20).all()
