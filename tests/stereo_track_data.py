"""Rectified stereo inputs and the oracle chain of the batched tracker's stereo path (plp_tracker_bind_stereo): the right
images of a PlanarSequence, the stereo camera, and the motion, keyframe, robust and local-map chains of
local_map_data / keyframe_track_data / robust_track_data with the frame's stereo_x_right_: the matchers' x_right gates
and the pose optimiser's stereo edges (pose_optimizer.cc:126-151: x_right >= 0 is a stereo edge, 0 included)."""
from __future__ import annotations

import numpy as np

import keyframe_track_data as ktd
import local_map_data as lmd
import oracle_api
import robust_track_data as rtd

NUM_MATCHES_THR = 20


# ---- inputs ---------------------------------------------------------------------------------------------------------
def stereo_camera(plp, seq, bf):
    """The stereo plp_camera (setup_type 1) of the sequence's K and size with focal_x_baseline bf."""
    K = seq.K
    return plp.capi.make_camera(K[0, 0], K[1, 1], K[0, 2], K[1, 2], seq.cols, seq.rows, bf=bf, setup_type=1)


def right_frames(seq, true_baseline):
    """The right images of a rectified rig: each frame rendered from the camera shifted by true_baseline along its own
    x axis, as PlanarSequence renders the left ones."""
    import cv2
    shift = np.eye(4)
    shift[0, 3] = -true_baseline
    return np.stack([cv2.warpPerspective(seq.tex, seq._tex_to_frame(shift @ T), (seq.cols, seq.rows),
                                         flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_REFLECT_101)
                     for T in seq.poses])


def stereo_sequence(plp, seq, bf):
    """(stereo camera, right images) of a PlanarSequence."""
    cam = stereo_camera(plp, seq, bf)
    return cam, right_frames(seq, cam.true_baseline)


# ---- the pose optimisation with stereo edges --------------------------------------------------------------------------
def pose_obs(curr, idx, pos_w):
    """pose_optimizer.cc:126-151: the observations of keypoints idx (in keypoint order) of landmarks at pos_w."""
    o = np.zeros(len(idx), oracle_api.PT_OBS_DTYPE)
    o["pos_w"] = pos_w
    o["obs_x"], o["obs_y"] = curr["x"][idx], curr["y"][idx]
    o["x_right"] = np.asarray(curr["x_right"], np.float32)[idx]
    o["inv_sigma_sq"] = lmd.ISIG[curr["octave"][idx]]
    return o


def optimise(orc, cam, curr, pre, rows_pos_w, T_in):
    """pose_optimize over the matches pre (keypoint -> row of rows_pos_w) with stereo edges, then discard_outliers
    (frame_tracker.cc:253-283).  -> (matched, pose, num_valid, n_inliers, lm_iters)."""
    idx = np.nonzero(pre >= 0)[0]
    T, pout, _, n_inl, iters = orc.pose_optimize(cam, T_in, pose_obs(curr, idx, np.asarray(rows_pos_w)[pre[idx]]))
    post = np.asarray(pre, np.int32).copy()
    post[idx[pout != 0]] = -1
    return post, T, int((post >= 0).sum()), int(n_inl), int(iters)


# ---- the stages -------------------------------------------------------------------------------------------------------
def oracle_motion(orc, grid, cam, curr, last, T_pred, T_last, margin=20.0):
    """motion_based_track of a stereo frame (curr["x_right"]): the matches of lmd.oracle_motion, whose matcher already
    takes the camera's motion assumption and the frame's x_right, optimised with stereo edges.
    -> (matched_pre, matched, pose, num_valid, n_inliers, iters), as lmd.oracle_motion."""
    pre = lmd.oracle_motion(orc, grid, cam, curr, last, T_pred, T_last, margin)[0]
    if (pre >= 0).sum() < NUM_MATCHES_THR:  # below the threshold after the retry: no pose optimisation
        return pre, pre.copy(), np.asarray(T_pred), 0, 0, 0
    return (pre,) + optimise(orc, cam, curr, pre, last["pos_w"], T_pred)


def oracle_keyframe_track(orc, ov, cam, curr, kf, pose_last):
    """bow_match_based_track of a stereo frame: ktd.oracle_keyframe_track's BoW matches optimised with stereo edges."""
    w = ktd.oracle_keyframe_track(orc, ov, cam, curr, kf, pose_last)
    if w["num_bow"] >= NUM_MATCHES_THR:
        post, T, nv, n_inl, iters = optimise(orc, cam, curr, w["matched_pre"], kf["pos_w"], pose_last)
        w.update(matched=post, pose=T, num_valid=nv, n_inliers=n_inl, lm_iters=iters)
    return w


def oracle_robust_track(orc, cam, curr, kf, frm_bearings, samples, pose_last):
    """robust_match_based_track of a stereo frame: rtd.oracle_robust_track's inlier matches optimised with stereo
    edges."""
    w = rtd.oracle_robust_track(orc, cam, curr, kf, frm_bearings, samples, pose_last)
    if w["num_robust"] >= NUM_MATCHES_THR:
        post, T, nv, n_inl, iters = optimise(orc, cam, curr, w["matched_pre"], kf["pos_w"], pose_last)
        w.update(matched=post, pose=T, num_valid=nv, n_inliers=n_inl, lm_iters=iters)
    return w


def predicted_x_right(cam, T, pos_w):
    """x_right_in_tracking_ (tracking_module.cc:953) of each row: camera::reproject_to_image's u - bf / z, summed in
    the reference's order and rounded to float."""
    T = np.asarray(T, np.float64).reshape(16)
    out = np.zeros(len(pos_w), np.float32)
    for i, X in enumerate(np.asarray(pos_w, np.float64).reshape(-1, 3)):
        X = [float(v) for v in X]
        pc0 = T[0] * X[0] + T[1] * X[1] + T[2] * X[2] + T[3]
        pc2 = T[8] * X[0] + T[9] * X[1] + T[10] * X[2] + T[11]
        if pc2 > 0.0:
            z_inv = 1.0 / pc2
            u = cam.fx * pc0 * z_inv + cam.cx
            out[i] = np.float32(u - cam.focal_x_baseline * z_inv)
    return out


def oracle_local_track(orc, grid, cam, curr, last, local, motion, max_local, margin=lmd.MARGIN):
    """optimize_current_frame_with_local_map of a stereo frame, as lmd.oracle_local_track: the queries carry
    x_right_in_tracking_, the matcher gates the keypoints with 0 < x_right on it, and the pose optimisation has stereo
    edges.  -> lmd.oracle_local_track's dict plus best (the matcher's keypoint per local row, None for a skipped frame)
    and qxr (the queries' predicted x_right, 0 on the rows that are not observable)."""
    m_pre, m_post, T_motion, nv = motion[0], motion[1], motion[2], motion[3]
    n, nl = len(curr["x"]), len(local["max_valid_dist"])
    lli = np.asarray(local["last_local_idx"], np.int64)
    status = 1 if nl > max_local else (2 if ((lli < -1) | (lli >= nl)).any() else 0)
    out = dict(matched=np.full(n, -1, np.int32), local=np.full(n, -1, np.int32), observable=np.zeros(nl, np.uint8),
               pose=np.asarray(T_motion, np.float64).reshape(4, 4), num_tracked=0, n_inliers=0, lm_iters=0,
               status=status, best=None, qxr=None)
    if nv < lmd.NUM_TRACKED_THR or status:
        return out
    skip = np.asarray(local["valid"], np.uint8) == 0
    for r in m_pre[m_pre >= 0]:
        if lli[r] >= 0:
            skip[lli[r]] = True
    obs, rx, ry, lvl, _ = lmd.can_observe(cam, T_motion, local, skip)
    qxr = np.where(obs != 0, predicted_x_right(cam, T_motion, local["pos_w"]), 0).astype(np.float32)
    q = dict(reproj_x=rx, reproj_y=ry, scale_level=np.maximum(lvl, 0), desc=local["desc"], valid=obs, x_right=qxr)
    frm = dict(x=curr["x"], y=curr["y"], octave=curr["octave"], desc=curr["desc"], x_right=curr["x_right"],
               claimed=(m_post >= 0).astype(np.uint8))
    best, _ = orc.match_frame_and_landmarks(grid, lmd.SF, frm, q, margin, 0.8)
    matched, loc = m_post.copy(), np.full(n, -1, np.int32)
    for j in np.nonzero(best >= 0)[0]:
        loc[best[j]] = j
    idx = np.nonzero((matched >= 0) | (loc >= 0))[0]
    from_last = matched[idx] >= 0
    pos = np.zeros((len(idx), 3))
    pos[from_last] = np.asarray(last["pos_w"])[matched[idx[from_last]]]
    pos[~from_last] = np.asarray(local["pos_w"]).reshape(-1, 3)[loc[idx[~from_last]]]
    T, pout, _, n_inl, iters = orc.pose_optimize(cam, T_motion, pose_obs(curr, idx, pos))
    if len(idx) >= 5:  # tracking_module.cc:762-784
        matched[idx[pout != 0]] = -1
        loc[idx[pout != 0]] = -1
    out.update(matched=matched, local=loc, observable=obs, pose=T, num_tracked=int(((matched >= 0) | (loc >= 0)).sum()),
               n_inliers=int(n_inl), lm_iters=int(iters), best=best, qxr=qxr)
    return out
