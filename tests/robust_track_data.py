"""The sample draw and the oracle chain of the batched robust tracker (plp_tracker_robust_track_batch_dev):
oracle brute_force_match (Lowe 0.8, no orientation check) -> the ordered pair list -> oracle essential RANSAC with the
device's sample sets -> oracle pose optimiser -> discard_outliers, and the local-map stage that follows it.  Plus a
Python restatement of csrc/ransac_sample.h."""
from __future__ import annotations

import numpy as np

import keyframe_track_data as ktd
import local_map_data as lmd
import oracle_api

NUM_MATCHES_THR = 20
LOWE = 0.8
NUM_ITER = 50
_M64 = (1 << 64) - 1
_G = 0x9E3779B97F4A7C15


# ------------------------------------------------------------------ csrc/ransac_sample.h restated
def _mix(z):
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    return z ^ (z >> 31)


class _Stream:
    def __init__(self, seed, b, it):
        self.s = _mix((_mix((seed + _G * (b + 1)) & _M64) + _G * (it + 1)) & _M64)
        self.draws = 0

    def next(self):
        self.s = (self.s + _G) & _M64
        self.draws += 1
        return _mix(self.s)

    def uniform(self, n):
        reject_below = (1 << 64) % n
        while True:
            r = self.next()
            if r >= reject_below:
                return r % n


def draw_sample(seed, b, it, n, trace=None):
    """create_random_array(8, 0, n - 1) of hypothesis `it` of frame `b` (n >= 8).  trace (a list) receives the size of
    the de-duplicated set after every round."""
    st = _Stream(seed, b, it)
    v = []
    while len(v) != 8:
        while len(v) < 9:
            v.append(st.uniform(n))
        v = sorted(set(v))[:8]
        if trace is not None:
            trace.append(len(v))
    for i in range(7, 0, -1):
        j = st.uniform(i + 1)
        v[i], v[j] = v[j], v[i]
    return np.array(v, np.int32)


def draw_samples(seed, b, n):
    """The 50 x 8 sample sets of frame b, or -1 where fewer than 8 matches leave nothing to draw."""
    if n < 8:
        return np.full((NUM_ITER, 8), -1, np.int32)
    return np.stack([draw_sample(seed, b, it, n) for it in range(NUM_ITER)])


# ------------------------------------------------------------------ the oracle chain
def bearings(cam, x, y):
    """convert_keypoints_to_bearings (perspective.cc:165-175) with the camera's double parameters"""
    xn = (np.asarray(x, np.float32).astype(np.float64) - cam.cx) / cam.fx
    yn = (np.asarray(y, np.float32).astype(np.float64) - cam.cy) / cam.fy
    l2 = np.sqrt(xn * xn + yn * yn + 1.0)
    return np.stack([xn / l2, yn / l2, 1.0 / l2], 1)


def keyframe(orc, ov, seq, res, t_ref, rng, cam, erased_frac=0.1, undistort=None, empty_fv=False):
    """ktd.keyframe plus keyfrm->bearings_; empty_fv: an empty bow_feat_vec_, so that its BoW track finds nothing."""
    kf = ktd.keyframe(orc, ov, seq, res, t_ref, rng, erased_frac=erased_frac, undistort=undistort)
    kps = lmd._kps(res[t_ref], undistort)
    kf["bearings"] = bearings(cam, kps["x"], kps["y"])
    if empty_fv:
        kf["fv"] = (np.zeros(0, np.uint32), np.zeros(1, np.int32), np.zeros(0, np.uint32))
    return kf


def match_list(orc, curr, kf):
    """robust::brute_force_match (frame = side 1) -> (matched per frame keypoint, pairs in frame keypoint order)"""
    m, _ = orc.brute_force_match(curr["desc"], np.asarray(curr["angle"], np.float32), kf["desc"], kf["angle"],
                                 kf["valid"], LOWE, False)
    idx = np.nonzero(m >= 0)[0]
    return m.astype(np.int32), np.stack([idx, m[idx]], 1).astype(np.int32)


def oracle_robust_track(orc, cam, curr, kf, frm_bearings, samples, pose_last):
    """robust_match_based_track of one frame (frame_tracker.cc:192-245) with the given sample sets.  -> dict(pairs,
    inlier, valid, E, score, matched_pre, matched, num_bf, num_robust, pose, num_valid, n_inliers, lm_iters)."""
    n = len(curr["x"])
    _, pairs = match_list(orc, curr, kf)
    out = dict(pairs=pairs, inlier=np.zeros(len(pairs), np.uint8), valid=0, E=None, score=0.0,
               matched_pre=np.full(n, -1, np.int32), matched=np.full(n, -1, np.int32), num_bf=len(pairs), num_robust=0,
               pose=np.asarray(pose_last, np.float64).reshape(4, 4), num_valid=0, n_inliers=0, lm_iters=0)
    if len(pairs) < 8:
        return out
    valid, inl, E, score, _ = orc.essential_ransac(frm_bearings, kf["bearings"], pairs, samples)
    out.update(inlier=inl, valid=valid, E=E, score=score)
    if not valid:
        return out
    pre = np.full(n, -1, np.int32)
    keep = pairs[inl != 0]
    pre[keep[:, 0]] = keep[:, 1]
    out.update(matched_pre=pre, num_robust=len(keep))
    if len(keep) < NUM_MATCHES_THR:
        return out
    idx = np.nonzero(pre >= 0)[0]
    pts = np.zeros(len(idx), oracle_api.PT_OBS_DTYPE)
    pts["pos_w"] = kf["pos_w"][pre[idx]]
    pts["obs_x"], pts["obs_y"] = curr["x"][idx], curr["y"][idx]
    pts["x_right"] = -1.0
    pts["inv_sigma_sq"] = lmd.ISIG[curr["octave"][idx]]
    T, pout, _, n_inl, iters = orc.pose_optimize(cam, pose_last, pts)
    post = pre.copy()
    post[idx[pout != 0]] = -1
    out.update(matched=post, pose=T, num_valid=int((post >= 0).sum()), n_inliers=int(n_inl), lm_iters=int(iters))
    return out


def compare(out, wants, stage, seed, pose_tol=1e-4, frames=None):
    """Device results of download_robust_tracking against the oracle's, frame by frame (only `frames`, if given); -> LM
    iteration lists of the frames that ran the stage."""
    got_it, want_it = [], []
    for b, w in enumerate(wants):
        if frames is not None and b not in frames:
            continue
        what = f"frame {b}"
        assert out["stage"][b] == stage[b], what
        if not stage[b]:
            assert out["num_bf_matches"][b] == 0 and out["num_robust_matches"][b] == 0, what
            assert out["num_valid"][b] == 0 and (out["matched"][b] == -1).all() and (out["samples"][b] == -1).all(), what
            continue
        assert out["num_bf_matches"][b] == w["num_bf"], (what, out["num_bf_matches"][b], w["num_bf"])
        assert np.array_equal(out["samples"][b], draw_samples(seed, b, w["num_bf"])), what
        assert out["num_robust_matches"][b] == w["num_robust"], (what, out["num_robust_matches"][b], w["num_robust"])
        assert np.array_equal(out["matched"][b], w["matched"]), what
        assert out["num_valid"][b] == w["num_valid"] and out["n_inliers"][b] == w["n_inliers"], \
            (what, out["num_valid"][b], w["num_valid"], out["n_inliers"][b], w["n_inliers"])
        rel = np.linalg.norm(out["pose"][b] - w["pose"]) / np.linalg.norm(w["pose"])
        assert rel <= pose_tol, (what, rel)
        got_it.append(int(out["lm_iters"][b]))
        want_it.append(w["lm_iters"])
    return got_it, want_it


def upload_keypoints(fe, res_list):
    """The frames' keypoints and descriptors written straight into the front end's extraction outputs (in place of
    extract()), e.g. an extraction with more keypoints than the device extractor's budget allows."""
    from plpslam_b200.capi import KP_DTYPE
    B = len(res_list)
    kp = np.zeros((B, fe.cap), KP_DTYPE)
    desc = np.zeros((B, fe.cap, 32), np.uint8)
    n = np.array([len(r["kps"]) for r in res_list], np.int32)
    assert n.max() <= fe.cap, (n.max(), fe.cap)
    for b, r in enumerate(res_list):
        kp[b, :n[b]] = r["kps"]
        desc[b, :n[b]] = r["desc"]
    fe.d_kp.upload(kp)
    fe.d_desc.upload(desc)
    fe.d_n.upload(n)


def run_case(orc, plp, fe, ov, gv, seq, res, ts, kfs, kf_of_frame, motion_valid, fail=(), seed=0, rb_seed=0,
             grid=None, cam=None, undistort=None, over=(), kps_given=False, fail_shift=(1.0, 0.5, 0.0)):
    """One batch: motion track (frames in `fail` get a predicted pose shifted by fail_shift), keyframe track, robust
    track, then the local-map stage.  kps_given: the frames' keypoints are res[t], uploaded (upload_keypoints), and the ORB
    extractor does not run.  over: frames with more keypoints than the window matcher holds; their motion and local-map
    results are not compared here (local_wants None) but left to the caller.  Returns dict(mot, kf, kf_wants, kf_stage,
    rb, rb_wants, rb_stage, local, local_wants, frm_bearings)."""
    rng = np.random.default_rng(seed)
    grid, cam = grid or fe.grid, cam or fe.cam
    preds = [seq.predicted_pose(t, rng) for t in ts]
    for b in fail:
        preds[b] = preds[b].copy()
        preds[b][:3, 3] += np.asarray(fail_shift)
    lasts = [seq.last_frame_landmarks(t - 1, lmd._kps(res[t - 1], undistort), res[t - 1]["desc"]) for t in ts]
    B = len(ts)
    fe.set_last_frames(lasts, np.stack(preds), np.stack([seq.poses[t - 1] for t in ts]))
    if kps_given:
        upload_keypoints(fe, [res[t] for t in ts])
        fe.track(B, 20.0)
    else:
        fe.upload_images(seq.frames[ts])
        fe.step(B, 20.0)
    mot = fe.download_tracking(B)
    curr = [lmd.curr_frame_u(res[t], undistort) for t in ts]
    motions = [lmd.oracle_motion(orc, grid, cam, curr[b], lasts[b], preds[b], seq.poses[t - 1])
               if b not in over else None for b, t in enumerate(ts)]
    for b in range(B):
        if b in over:
            continue
        assert np.array_equal(motions[b][1], mot["matched"][b]) and motions[b][3] == mot["num_valid"][b], f"motion {b}"
    mv = np.ones(B, np.uint8) if motion_valid is None else np.asarray(motion_valid, np.uint8)
    kf_stage = [int(mv[b] == 0 or mot["num_valid"][b] < NUM_MATCHES_THR) for b in range(B)]
    kf_wants = [ktd.oracle_keyframe_track(orc, ov, cam, curr[b], kfs[kf_of_frame[b]], seq.poses[t - 1])
                if kf_stage[b] else None for b, t in enumerate(ts)]
    rb_stage = [int(kf_stage[b] and kf_wants[b]["num_valid"] < NUM_MATCHES_THR) for b in range(B)]
    # the local maps: for a keyframe-tracked frame they hold its keyframe's landmarks (local_idx), else the last frame's
    local_list, local_idx = [], []
    for b, t in enumerate(ts):
        if kf_stage[b]:
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
    fe.track_keyframe(B, gv, motion_valid)
    kout = fe.download_keyframe_tracking(B)
    ktd.compare(kout, kf_wants, kf_stage)
    before = (fe.download_tracking(B), fe.download_keyframe_tracking(B))
    fe.track_robust(B, rb_seed)
    out = fe.download_robust_tracking(B)
    after = (fe.download_tracking(B), fe.download_keyframe_tracking(B))
    for g, w in zip(after, before):  # the motion and keyframe outputs, byte for byte
        for key, v in w.items():
            if key == "bow":
                assert all(x.tobytes() == y.tobytes() for gb, wb in zip(g[key], v) for x, y in zip(gb, wb)), key
            elif isinstance(v, list):
                assert all(x.tobytes() == y.tobytes() for x, y in zip(g[key], v)), key
            else:
                assert g[key].tobytes() == v.tobytes(), key
    frm_bearings = [bearings(cam, c["x"], c["y"]) for c in curr]
    wants = [oracle_robust_track(orc, cam, curr[b], kfs[kf_of_frame[b]], frm_bearings[b], out["samples"][b],
                                 seq.poses[t - 1]) if rb_stage[b] else None for b, t in enumerate(ts)]
    fe.set_local_maps(local_list)
    fe.track_local_map(B, lmd.MARGIN)
    lout = fe.download_local_tracking(B)
    lwants = []
    for b in range(B):
        if b in over:
            lwants.append(None)
        elif kf_stage[b]:
            kf = kfs[kf_of_frame[b]]
            loc = dict(local_list[b], last_local_idx=local_idx[b])
            if rb_stage[b]:
                tr = (wants[b]["matched_pre"], wants[b]["matched"], out["pose"][b], int(out["num_valid"][b]))
            else:
                tr = (kf_wants[b]["matched_pre"], kf_wants[b]["matched"], kout["pose"][b], int(kout["num_valid"][b]))
            lwants.append(lmd.oracle_local_track(orc, grid, cam, curr[b], kf, loc, tr, fe.max_local))
        else:
            dev_motion = (motions[b][0], motions[b][1], mot["pose"][b], int(mot["num_valid"][b]))
            lwants.append(lmd.oracle_local_track(orc, grid, cam, curr[b], lasts[b], local_list[b], dev_motion,
                                                 fe.max_local))
    return dict(mot=mot, kf=kout, kf_wants=kf_wants, kf_stage=kf_stage, rb=out, rb_wants=wants, rb_stage=rb_stage,
                local=lout, local_wants=lwants, frm_bearings=frm_bearings)
