"""smoke(): the local-map update on three motion-tracked frames (extract -> motion track -> update -> local map on the
device list) against the restatement of update_local_map and the oracle's local-map chain on the same list."""
import numpy as np


def run(pkg, ctx, orc):
    import local_map_data as lmd
    import local_map_update_data as lmu
    import oracle_api
    import scene
    from plpslam_b200.tracking import FrontEnd

    ts = [2, 3, 4]
    seq = scene.PlanarSequence(seed=41, n_frames=5)
    res = [orc.orb_extract(oracle_api.orb_params(), f) for f in seq.frames]
    fe = FrontEnd(ctx, seq.rows, seq.cols, seq.camera(pkg), max_batch=3)
    try:
        fe.reserve_local_map(4096)
        fe.reserve_local_map_update(64)
        rng = np.random.default_rng(4)
        preds = [seq.predicted_pose(t, rng) for t in ts]
        lasts = [seq.last_frame_landmarks(t - 1, res[t - 1]["kps"], res[t - 1]["desc"]) for t in ts]
        fe.set_last_frames(lasts, np.stack(preds), np.stack([seq.poses[t - 1] for t in ts]))
        snap, lm_id = lmu.scene_snapshot(seq, res, max(ts), rng)
        snap["last_row_lm"] = np.concatenate([lm_id[t - 1] for t in ts]).astype(np.int32)
        fe.set_map(snap)
        fe.upload_images(seq.frames[ts])
        fe.step(3, 20.0)
        fe.update_local_map(3)
        fe.track_local_map(3, lmd.MARGIN, updated=True)
        mot, u, lout = fe.download_tracking(3), fe.download_local_map_update(3), fe.download_local_tracking(3)
        wants = []
        for b, t in enumerate(ts):
            curr = lmd.curr_frame(res[t])
            mo = lmd.oracle_motion(orc, fe.grid, fe.cam, curr, lasts[b], preds[b], seq.poses[t - 1])
            assert np.array_equal(mo[1], mot["matched"][b]), b
            rows = snap["last_row_lm"][fe._last_offsets[b]:fe._last_offsets[b + 1]]
            tracked = np.array([rows[q] if q >= 0 else -1 for q in mo[1]], np.int32)
            w = lmu.device_update(snap, tracked, fe.max_local, 64, mo[3] >= 20)
            assert u["status"][b] == w["status"] == 0 and u["nearest"][b] == w["nearest"], b
            assert list(u["local_kf"][b]) == w["local_kf"] and list(u["local_lm"][b]) == w["local_lm"], b
            loc = dict(lmu.local_rows(snap, w["local_lm"]), last_local_idx=lmu.mapping(w["local_lm"], rows))
            assert np.array_equal(u["last_local_idx"][b], loc["last_local_idx"]), b
            wants.append(lmd.oracle_local_track(orc, fe.grid, fe.cam, curr, lasts[b], loc,
                                                (mo[0], mo[1], mot["pose"][b], int(mot["num_valid"][b])), fe.max_local))
        lmd.compare(lout, wants)
        print(f"smoke local-map update ok: nearest {list(u['nearest'])}, local keyframes "
              f"{[len(x) for x in u['local_kf']]}, local landmarks {[len(x) for x in u['local_lm']]}, "
              f"num_tracked {list(lout['num_tracked'])}, bit-exact")
    finally:
        fe.close()
