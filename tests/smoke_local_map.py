"""smoke(): the local-map stage of tracking on two frames (extract -> motion track -> local map), against the oracle."""
import numpy as np


def run(pkg, ctx, orc):
    import local_map_data as lmd
    import oracle_api
    import scene
    from plpslam_b200.tracking import FrontEnd

    ts = [1, 2]
    seq = scene.PlanarSequence(seed=31, n_frames=3)
    res = [orc.orb_extract(oracle_api.orb_params(), f) for f in seq.frames]
    fe = FrontEnd(ctx, seq.rows, seq.cols, seq.camera(pkg), max_batch=2)
    try:
        fe.reserve_local_map(4096)
        rng = np.random.default_rng(3)
        preds = [seq.predicted_pose(t, rng) for t in ts]
        lasts = [seq.last_frame_landmarks(t - 1, res[t - 1]["kps"], res[t - 1]["desc"]) for t in ts]
        fe.upload_images(seq.frames[ts])
        fe.set_last_frames(lasts, np.stack(preds), np.stack([seq.poses[t - 1] for t in ts]))
        fe.step(2)
        mot = fe.download_tracking(2)
        local_list, wants = lmd.chain_case(orc, seq, res, ts, preds, lasts, mot, fe.grid, fe.cam, rng, 4096)
        fe.set_local_maps(local_list)
        fe.track_local_map(2)
        out = fe.download_local_tracking(2)
        lmd.compare(out, wants)
        assert all(out["num_tracked"] >= 20), out["num_tracked"]
        print(f"smoke local map ok: num_tracked {list(out['num_tracked'])} (motion {list(mot['num_valid'])}), "
              f"{[int((x >= 0).sum()) for x in out['local']]} local matches, bit-exact")
    finally:
        fe.close()
