"""smoke(): a rectified stereo pair tracked on two frames (ORB left + right -> stereo::compute -> motion track with
stereo edges), against the oracle."""
import numpy as np


def run(pkg, ctx, orc):
    import local_map_data as lmd
    import oracle_api
    import scene
    import stereo_track_data as std
    from plpslam_b200.tracking import FrontEnd

    ts = [1, 2]
    fx, fy, cx, cy = 458.654, 457.296, 367.215, 248.375  # EuRoC
    seq = scene.PlanarSequence(seed=33, n_frames=3, rows=480, cols=752, fx=fx, fy=fy, cx=cx, cy=cy)
    cam, right = std.stereo_sequence(pkg, seq, 47.906)
    p = oracle_api.orb_params()
    res = [orc.orb_extract(p, f) for f in seq.frames]
    fe = FrontEnd(ctx, seq.rows, seq.cols, cam, max_batch=2)
    try:
        rng = np.random.default_rng(3)
        preds = [seq.predicted_pose(t, rng) for t in ts]
        lasts = [seq.last_frame_landmarks(t - 1, res[t - 1]["kps"], res[t - 1]["desc"]) for t in ts]
        fe.upload_images(seq.frames[ts], right[ts])
        fe.set_last_frames(lasts, np.stack(preds), np.stack([seq.poses[t - 1] for t in ts]))
        fe.step(2, 10.0)
        xr = fe.download_stereo(2)
        mot = fe.download_tracking(2)
        for b, t in enumerate(ts):
            want, _, _ = orc.stereo_compute(res[t], orc.orb_extract(p, right[t]), fe.orb.scale_factors,
                                            fe.orb.inv_scale_factors, cam.focal_x_baseline, cam.true_baseline)
            assert np.array_equal(xr[b][0], want), "stereo x_right disagrees with the oracle"
            curr = dict(lmd.curr_frame(res[t]), x_right=xr[b][0])
            _, m, T, nv, _, _ = std.oracle_motion(orc, fe.grid, cam, curr, lasts[b], preds[b], seq.poses[t - 1],
                                                  margin=10.0)
            assert np.array_equal(mot["matched"][b], m) and mot["num_valid"][b] == nv >= 20, b
            assert np.linalg.norm(mot["pose"][b] - T) / np.linalg.norm(T) <= 1e-4, b
        print(f"smoke stereo track ok: num_valid {list(mot['num_valid'])}, "
              f"{[int((x[0] >= 0).sum()) for x in xr]} stereo keypoints, bit-exact")
    finally:
        fe.close()
