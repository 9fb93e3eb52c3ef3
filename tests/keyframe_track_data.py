"""Scenes and the oracle chain of the batched keyframe tracker (plp_tracker_keyframe_track_batch_dev):
oracle transform -> capi.fold_bow -> oracle bow_tree (frame vs reference keyframe) -> oracle pose optimiser ->
discard_outliers, and the local-map stage that follows it.  No reference files: the vocabulary is synthetic."""
from __future__ import annotations

import numpy as np

import local_map_data as lmd
import oracle_api
import synth

NUM_MATCHES_THR = 20
LOWE = 0.7


def make_scene_vocab(desc_pool, seed, k=10, L=6, inner=2, zero_weight_frac=0.1):
    """A vocabulary of the shipped shape (k = 10, L = 6: transform with levelsup 4 reports level-2 nodes) whose
    level-1 and level-2 centres are descriptors of the scene, so that the descriptors of one landmark seen from two
    frames usually descend into the same level-2 node.  Below level 2 every inner node has `inner` children (bit-flipped
    copies of their parent), which keeps the tree small.  Record layout of bow_data.make_vocab."""
    rng = np.random.default_rng(seed)
    pool = np.asarray(desc_pool, np.uint8).reshape(-1, 32)
    parent, desc, weight, leaf = [], [], [], []
    frontier, next_id = [(0, None, 0)], 1
    while frontier:
        new = []
        for pid, pdesc, plevel in frontier:
            lvl = plevel + 1
            nc = k if lvl <= 2 else inner
            for _ in range(nc):
                d = pool[rng.integers(len(pool))] if lvl <= 2 else synth.flip_bits(rng, pdesc[None, :], 40)[0]
                is_leaf = lvl == L
                parent.append(pid)
                desc.append(d)
                leaf.append(1 if is_leaf else 0)
                weight.append(0.0 if (not is_leaf or rng.random() < zero_weight_frac) else float(rng.uniform(0.1, 9.7)))
                if not is_leaf:
                    new.append((next_id, d, lvl))
                next_id += 1
        frontier = new
    return dict(k=k, L=L, parent=np.array(parent, np.int32), desc=np.array(desc, np.uint8).reshape(-1, 32),
                weight=np.array(weight, np.float32), is_leaf=np.array(leaf, np.uint8))


def keyframe(orc, ov, seq, res, t_ref, rng, erased_frac=0.1, undistort=None):
    """Reference keyframe from frame t_ref: its keypoints' descriptors and angles, the plane points as landmarks (a
    fraction erased), and its bow_feat_vec_ from the oracle's transform folded like DBoW2."""
    kps = lmd._kps(res[t_ref], undistort)
    desc = np.ascontiguousarray(res[t_ref]["desc"], np.uint8)
    pos_w = seq.backproject(seq.poses[t_ref], kps["x"].astype(np.float64), kps["y"].astype(np.float64))
    valid = (rng.random(len(desc)) >= erased_frac).astype(np.uint8)
    _, _, fv = fold_bow(*orc.bow_transform(ov, desc, 4))
    return dict(t=t_ref, desc=desc, angle=kps["angle"].astype(np.float32), valid=valid, pos_w=pos_w, fv=fv)


def fold_bow(word_id, node_id, weight):
    from plpslam_b200.capi import fold_bow as fold
    return fold(word_id, node_id, weight)


def oracle_keyframe_track(orc, ov, cam, curr, kf, pose_last):
    """bow_match_based_track of one frame (frame_tracker.cc:126-189).  -> dict(matched_pre, matched, bow, num_bow,
    pose, num_valid, n_inliers, lm_iters)."""
    bow = orc.bow_transform(ov, curr["desc"], 4)
    _, _, fv = fold_bow(*bow)
    frm = dict(desc=curr["desc"], angle=np.asarray(curr["angle"], np.float32), valid=None, fv=fv)
    _, m12, num = orc.bow_tree_match(kf, frm, LOWE, True)
    n = len(curr["x"])
    out = dict(matched_pre=np.full(n, -1, np.int32), matched=np.full(n, -1, np.int32), bow=bow, num_bow=num,
               pose=np.asarray(pose_last, np.float64).reshape(4, 4), num_valid=0, n_inliers=0, lm_iters=0)
    if num < NUM_MATCHES_THR:
        return out
    idx = np.nonzero(m12 >= 0)[0]
    pts = np.zeros(len(idx), oracle_api.PT_OBS_DTYPE)
    pts["pos_w"] = kf["pos_w"][m12[idx]]
    pts["obs_x"], pts["obs_y"] = curr["x"][idx], curr["y"][idx]
    pts["x_right"] = -1.0
    pts["inv_sigma_sq"] = lmd.ISIG[curr["octave"][idx]]
    T, pout, _, n_inl, iters = orc.pose_optimize(cam, pose_last, pts)
    post = m12.astype(np.int32)
    post[idx[pout != 0]] = -1
    out.update(matched_pre=m12.astype(np.int32), matched=post, pose=T, num_valid=int((post >= 0).sum()),
               n_inliers=int(n_inl), lm_iters=int(iters))
    return out


def compare(out, wants, motion_stage, pose_tol=1e-4):
    """Device results of download_keyframe_tracking against the oracle's, frame by frame; -> LM iteration lists of the
    frames that ran the stage."""
    got_it, want_it = [], []
    for b, w in enumerate(wants):
        what = f"frame {b}"
        assert out["stage"][b] == motion_stage[b], what
        assert out["status"][b] == 0, what
        if not motion_stage[b]:
            assert out["num_bow_matches"][b] == 0 and out["num_valid"][b] == 0 and (out["matched"][b] == -1).all(), what
            continue
        assert out["num_bow_matches"][b] == w["num_bow"], (what, out["num_bow_matches"][b], w["num_bow"])
        for g, o in zip(out["bow"][b], w["bow"]):
            assert np.array_equal(g, o), what
        assert np.array_equal(out["matched"][b], w["matched"]), what
        assert out["num_valid"][b] == w["num_valid"] and out["n_inliers"][b] == w["n_inliers"], \
            (what, out["num_valid"][b], w["num_valid"], out["n_inliers"][b], w["n_inliers"])
        rel = np.linalg.norm(out["pose"][b] - w["pose"]) / np.linalg.norm(w["pose"])
        assert rel <= pose_tol, (what, rel)
        got_it.append(int(out["lm_iters"][b]))
        want_it.append(w["lm_iters"])
    return got_it, want_it


def run_case(orc, plp, fe, ov, gv, seq, res, ts, kfs, kf_of_frame, motion_valid, fail=(), seed=0, grid=None, cam=None,
             undistort=None, local=True):
    """One batch: motion track (frames in `fail` get a predicted pose a metre off), keyframe track, then (local=True)
    the local-map stage.  Returns (motion outputs, keyframe outputs, keyframe wants, stage, local outputs, local
    wants)."""
    rng = np.random.default_rng(seed)
    grid, cam = grid or fe.grid, cam or fe.cam
    preds = [seq.predicted_pose(t, rng) for t in ts]
    for b in fail:
        preds[b] = preds[b].copy()
        preds[b][:3, 3] += np.array([1.0, 0.5, 0.0])
    lasts = [seq.last_frame_landmarks(t - 1, lmd._kps(res[t - 1], undistort), res[t - 1]["desc"]) for t in ts]
    B = len(ts)
    fe.upload_images(seq.frames[ts])
    fe.set_last_frames(lasts, np.stack(preds), np.stack([seq.poses[t - 1] for t in ts]))
    fe.step(B, 20.0)
    mot = fe.download_tracking(B)
    curr = [lmd.curr_frame_u(res[t], undistort) for t in ts]
    motions = [lmd.oracle_motion(orc, grid, cam, curr[b], lasts[b], preds[b], seq.poses[t - 1]) for b, t in enumerate(ts)]
    for b in range(B):
        assert np.array_equal(motions[b][1], mot["matched"][b]) and motions[b][3] == mot["num_valid"][b], f"motion {b}"
    mv = np.ones(B, np.uint8) if motion_valid is None else np.asarray(motion_valid, np.uint8)
    stage = [int(mv[b] == 0 or mot["num_valid"][b] < NUM_MATCHES_THR) for b in range(B)]
    wants = [oracle_keyframe_track(orc, ov, cam, curr[b], kfs[kf_of_frame[b]], seq.poses[t - 1]) if stage[b] else None
             for b, t in enumerate(ts)]
    # the local maps: for a keyframe-tracked frame they hold its keyframe's landmarks (local_idx), else the last frame's
    local_list, local_idx = [], []
    for b, t in enumerate(ts):
        if stage[b]:
            kf = kfs[kf_of_frame[b]]
            kfl = dict(pos_w=kf["pos_w"], octave=np.zeros(len(kf["desc"]), np.int32))
            loc = lmd.build_local_map(seq, res, kf["t"] + 1, rng, last_frame=kfl, drop_last=20, undistort=undistort)
            local_idx.append(loc["last_local_idx"])
            loc["last_local_idx"] = np.full(len(lasts[b]["octave"]), -1, np.int32)
        else:
            loc = lmd.build_local_map(seq, res, t, rng, last_frame=lasts[b], drop_last=20, undistort=undistort)
            local_idx.append(np.zeros(0, np.int32))
        local_list.append(loc)
    fe.set_keyframes(kfs, kf_of_frame, local_idx)
    before = fe.download_tracking(B)
    fe.track_keyframe(B, gv, motion_valid)
    out = fe.download_keyframe_tracking(B)
    after = fe.download_tracking(B)
    for key in ("pose", "num_valid", "n_inliers", "lm_iters", "status"):
        assert after[key].tobytes() == before[key].tobytes(), key
    assert all(after["matched"][b].tobytes() == before["matched"][b].tobytes() for b in range(B))
    lout = lwants = None
    if local:
        fe.set_local_maps(local_list)
        fe.track_local_map(B, lmd.MARGIN)
        lout = fe.download_local_tracking(B)
        lwants = []
        for b in range(B):
            if stage[b]:
                kf = kfs[kf_of_frame[b]]
                loc = dict(local_list[b], last_local_idx=local_idx[b])
                tr = (wants[b]["matched_pre"], wants[b]["matched"], out["pose"][b], int(out["num_valid"][b]))
                lwants.append(lmd.oracle_local_track(orc, grid, cam, curr[b], kf, loc, tr, fe.max_local))
            else:
                dev_motion = (motions[b][0], motions[b][1], mot["pose"][b], int(mot["num_valid"][b]))
                lwants.append(lmd.oracle_local_track(orc, grid, cam, curr[b], lasts[b], local_list[b], dev_motion,
                                                     fe.max_local))
    return mot, out, wants, stage, lout, lwants
