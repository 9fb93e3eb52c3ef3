"""GPU parity of the device-resident batched front-end (extract -> motion_based_track) against the oracle chain
orb_extract -> match_current_and_last_frames (+ widened retry) -> pose_optimize -> discard_outliers."""
import numpy as np
import pytest

import oracle_api
import scene
import synth
from scene import oracle_track as _oracle_track

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("margin,pred_sigma", [(20.0, (0.003, 0.01)), (3.0, (0.02, 0.06))])
def test_front_end_matches_oracle_chain(ctx, orc, plp, margin, pred_sigma):
    from plpslam_b200.tracking import FrontEnd
    B = 5
    seq = scene.PlanarSequence(seed=7, n_frames=B + 1)
    p = oracle_api.orb_params()
    res = [orc.orb_extract(p, f) for f in seq.frames]
    cam = plp.capi.make_camera(synth.FX, synth.FY, synth.CX, synth.CY, seq.cols, seq.rows)
    fe = FrontEnd(ctx, seq.rows, seq.cols, cam, max_batch=8)
    rng = np.random.default_rng(3)
    preds = [seq.predicted_pose(t, rng, *pred_sigma) for t in range(1, B + 1)]
    lasts = [seq.last_frame_landmarks(t - 1, res[t - 1]["kps"], res[t - 1]["desc"]) for t in range(1, B + 1)]
    fe.upload_images(seq.frames[1:B + 1])
    fe.set_last_frames(lasts, np.stack(preds), np.stack(seq.poses[0:B]))
    fe.step(B, margin)
    kps = fe.download_keypoints(B)
    out = fe.download_tracking(B)
    assert not out["status"].any()
    retried = 0
    want_iters = []
    for b in range(B):
        t = b + 1
        # extraction identical to the oracle's
        assert np.array_equal(kps[b][0], res[t]["kps"]) and np.array_equal(kps[b][1], res[t]["desc"])
        m, T, nv, n_inl, iters = _oracle_track(orc, plp, seq, res, t, preds[b], margin)
        assert np.array_equal(out["matched"][b], m), f"frame {b}"
        assert out["num_valid"][b] == nv and out["n_inliers"][b] == n_inl
        want_iters.append(iters)
        rel = np.linalg.norm(out["pose"][b] - T) / np.linalg.norm(T)
        assert rel < 1e-4, rel
        if margin >= 20.0:
            assert nv >= 20  # the easy case really tracks; the hard case exercises the retry / failure branches
    scene.check_lm_iters(out["lm_iters"], want_iters, "front end")
    fe.close()
