"""Scenes and the oracle chain of the local-map stage of tracking (tracking_module::optimize_current_frame_with_local_map,
monocular points): local maps derived from earlier keyframes of scene.PlanarSequence, distractor rows for every
can_observe gate, and the oracle chain motion_based_track -> search_local_landmarks -> pose_optimize -> outlier drop.

The can_observe restatement (oracle/local_map_oracle.cc), the matcher and the pose optimiser are the oracle library's."""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

import oracle_api
import synth

ROOT = Path(__file__).resolve().parent.parent
_P = C.c_void_p
NUM_LEVELS = 8
MARGIN = 5.0        # tracking_module.cc:976-981 (20 right after a relocalisation)
NUM_TRACKED_THR = 20


def logf(x) -> np.float32:
    libm = C.CDLL("libm.so.6")
    libm.logf.restype = C.c_float
    libm.logf.argtypes = [C.c_float]
    return np.float32(libm.logf(float(np.float32(x))))


LOG_SF = logf(1.2)  # frame::log_scale_factor_ = std::log(scale_factor_) on floats
SF = synth.scale_factors()
ISIG = synth.inv_level_sigma_sq()


def cam_center(T):
    """frame.cc:750 cam_center_ = -R^T t, summed in the oracle's order."""
    T = np.asarray(T, np.float64).reshape(16)
    return np.array([-(T[0 + r] * T[3] + T[4 + r] * T[7] + T[8 + r] * T[11]) for r in range(3)])


def fdist(p, c) -> np.float32:
    """The camera-to-landmark distance as can_observe compares it: a double norm summed left to right, then float."""
    d0, d1, d2 = (float(p[i]) - float(c[i]) for i in range(3))
    return np.float32(np.sqrt(d0 * d0 + d1 * d1 + d2 * d2))


def can_observe(cam, T, lms, skip=None):
    """-> (observable, reproj_x, reproj_y, level, gate) per row; gate 0 observable, 1 skipped, 2 reprojection,
    3 distance, 4 viewing angle."""
    m = len(lms["max_valid_dist"])
    ocam = oracle_api.as_camera(cam)
    T = np.ascontiguousarray(np.asarray(T, np.float64).reshape(16))
    arrs = [np.ascontiguousarray(lms["pos_w"], np.float64).reshape(-1, 3), np.ascontiguousarray(lms["normal"], np.float64).reshape(-1, 3),
            np.ascontiguousarray(lms["min_valid_dist"], np.float32), np.ascontiguousarray(lms["max_valid_dist"], np.float32),
            np.ascontiguousarray(lms["max_valid_dist_raw"], np.float32)]
    sk = np.ascontiguousarray(np.zeros(m, np.uint8) if skip is None else skip, np.uint8)
    obs = np.zeros(max(m, 1), np.uint8)
    rx, ry = np.zeros(max(m, 1), np.float32), np.zeros(max(m, 1), np.float32)
    lvl, gate = np.zeros(max(m, 1), np.int32), np.zeros(max(m, 1), np.int32)
    oracle_api.lib().lmo_can_observe(C.byref(ocam), T.ctypes.data_as(_P), C.c_int(m),
                                     *[a.ctypes.data_as(_P) for a in arrs], sk.ctypes.data_as(_P), C.c_float(LOG_SF),
                                     C.c_int(NUM_LEVELS), obs.ctypes.data_as(_P), rx.ctypes.data_as(_P),
                                     ry.ctypes.data_as(_P), lvl.ctypes.data_as(_P), gate.ctypes.data_as(_P))
    return obs[:m], rx[:m], ry[:m], lvl[:m], gate[:m]


# ---- landmarks ---------------------------------------------------------------------------------------------------
def landmark_rows(seq, t_ref, kps, desc, observers):
    """Landmarks created at keyframe t_ref from its keypoints: position on the plane, obs_mean_normal from the centres
    of the observing keyframes, and the valid distances of landmark::update_normal_and_depth (landmark.cc:283-293)."""
    pos = seq.backproject(seq.poses[t_ref], kps["x"].astype(np.float64), kps["y"].astype(np.float64))
    normal = np.zeros_like(pos)
    for k in observers:
        v = pos - cam_center(seq.poses[k])
        normal += v / np.linalg.norm(v, axis=1, keepdims=True)
    normal /= np.linalg.norm(normal, axis=1, keepdims=True)
    dist = np.linalg.norm(pos - cam_center(seq.poses[t_ref]), axis=1)
    oct_ = kps["octave"].astype(np.int64)
    max_raw = (dist * SF[oct_].astype(np.float64)).astype(np.float32)      # max_valid_dist_ = dist * scale_factor
    min_raw = (max_raw / SF[NUM_LEVELS - 1]).astype(np.float32)             # max_valid_dist_ / scale_factors[L-1]
    return dict(pos_w=pos, normal=normal,
                min_valid_dist=(0.7 * min_raw.astype(np.float64)).astype(np.float32),   # get_min_valid_distance()
                max_valid_dist=(1.3 * max_raw.astype(np.float64)).astype(np.float32),   # get_max_valid_distance()
                max_valid_dist_raw=max_raw, desc=np.ascontiguousarray(desc, np.uint8),
                valid=np.ones(len(pos), np.uint8))


def concat(rows_list):
    keys = ["pos_w", "normal", "min_valid_dist", "max_valid_dist", "max_valid_dist_raw", "desc", "valid"]
    out = {}
    for k in keys:
        parts = [r[k] for r in rows_list if len(r["max_valid_dist"])]
        if parts:
            out[k] = np.concatenate(parts)
        else:
            proto = rows_list[0][k] if rows_list else np.zeros(0)
            out[k] = np.zeros((0,) + np.asarray(proto).shape[1:], np.asarray(proto).dtype)
    return out


def empty_rows():
    return dict(pos_w=np.zeros((0, 3)), normal=np.zeros((0, 3)), min_valid_dist=np.zeros(0, np.float32),
                max_valid_dist=np.zeros(0, np.float32), max_valid_dist_raw=np.zeros(0, np.float32),
                desc=np.zeros((0, 32), np.uint8), valid=np.zeros(0, np.uint8))


def take(rows, idx):
    return {k: np.asarray(v)[idx] for k, v in rows.items()}


def level_thresholds():
    """The predict_scale_level table of the device (smallest ratio per level), from the oracle's own logf."""
    thr = np.zeros(NUM_LEVELS, np.float32)
    for k in range(1, NUM_LEVELS):
        lo, hi = np.float32(1e-3), np.float32(1e3)
        pred = lambda r: int(np.ceil(np.float32(logf(r) / LOG_SF)))
        lo_i, hi_i = int(lo.view(np.int32)), int(hi.view(np.int32))
        while hi_i - lo_i > 1:
            mid = (lo_i + hi_i) // 2
            if pred(np.int32(mid).view(np.float32)) >= k:
                hi_i = mid
            else:
                lo_i = mid
        thr[k] = np.int32(hi_i).view(np.float32)
    return thr


def distractors(cam, T, good, rng):
    """Rows built from the observable landmarks `good` (at least 12) at the pose T, one group per gate: behind the
    camera, outside the bounds, too near, too far, normal turned away, erased, distances on the float bounds, ray_cos
    on either side of 0.5, and ratios next to every level threshold."""
    c = cam_center(T)
    R = np.asarray(T, np.float64).reshape(4, 4)[:3, :3]
    rows = []
    n = len(good["max_valid_dist"])
    pick = lambda k: take(good, rng.choice(n, k, replace=n < k))
    # behind the camera: mirror through the centre
    r = pick(3)
    r["pos_w"] = 2 * c - r["pos_w"]
    rows.append(r)
    # outside the image: push sideways along the camera's x axis
    r = pick(3)
    r["pos_w"] = r["pos_w"] + 10.0 * R[0]
    rows.append(r)
    # distances on and next to the float bounds
    r = pick(6)
    fd = np.array([fdist(p, c) for p in r["pos_w"]], np.float32)
    r["min_valid_dist"] = np.array([np.nextafter(fd[0], np.float32(np.inf)), fd[1], fd[2] * 2, 0, 0, 0], np.float32)
    r["max_valid_dist"] = np.array([fd[0] * 2, fd[1] * 2, fd[2] * 3, fd[3], np.nextafter(fd[4], np.float32(0)),
                                    fd[5] / 2], np.float32)
    rows.append(r)
    # normal turned away, and ray_cos next to 0.5
    r = pick(8)
    for i, p in enumerate(r["pos_w"]):
        u = (p - c) / np.linalg.norm(p - c)
        v = np.cross(u, R[2] if abs(u @ R[2]) < 0.9 else R[0])
        v /= np.linalg.norm(v)
        ang = [np.pi, 0.6 * np.pi, np.pi / 3 - 1e-9, np.pi / 3 + 1e-9, np.pi / 3 - 1e-15, np.pi / 3 + 1e-15,
               np.pi / 3, np.pi / 3 - 2e-16][i]
        r["normal"][i] = np.cos(ang) * u + np.sin(ang) * v
    rows.append(r)
    # erased
    r = pick(3)
    r["valid"] = np.zeros(3, np.uint8)
    rows.append(r)
    # ratios on, just below and just above every level threshold
    thr = level_thresholds()
    for k in range(1, NUM_LEVELS):
        r = pick(3)
        for i, p in enumerate(r["pos_w"]):
            fdi = fdist(p, c)
            raw = np.float32(thr[k] * fdi)
            raw = [np.nextafter(raw, np.float32(0)), raw, np.nextafter(raw, np.float32(np.inf))][i]
            r["max_valid_dist_raw"][i] = raw
            r["min_valid_dist"][i] = 0.0
            r["max_valid_dist"][i] = np.float32(np.inf)
        rows.append(r)
    return concat(rows)


# ---- the oracle chain ----------------------------------------------------------------------------------------------
def oracle_motion(orc, grid, cam, curr, last, T_pred, T_last, margin=20.0):
    """motion_based_track as scene.oracle_track, also returning the matches BEFORE discard_outliers.
    -> (matched_pre, matched, pose, num_valid, n_inliers, iters)."""
    m, nm = orc.match_current_and_last_frames(grid, SF, cam, curr, T_pred, T_last, last, margin, True)
    if nm < 20:
        m, nm = orc.match_current_and_last_frames(grid, SF, cam, curr, T_pred, T_last, last, 2 * margin, True)
    n = len(curr["x"])
    if nm < 20:
        return np.full(n, -1, np.int32), np.full(n, -1, np.int32), np.asarray(T_pred), 0, 0, 0
    idx = np.nonzero(m >= 0)[0]
    pts = np.zeros(len(idx), oracle_api.PT_OBS_DTYPE)
    pts["pos_w"] = last["pos_w"][m[idx]]
    pts["obs_x"], pts["obs_y"] = curr["x"][idx], curr["y"][idx]
    pts["x_right"] = -1.0
    pts["inv_sigma_sq"] = ISIG[curr["octave"][idx]]
    T, pout, _, n_inl, iters = orc.pose_optimize(cam, T_pred, pts)
    post = m.copy()
    post[idx[pout != 0]] = -1
    return m, post, T, int((post >= 0).sum()), n_inl, iters


def oracle_local_track(orc, grid, cam, curr, last, local, motion, max_local, margin=MARGIN):
    """optimize_current_frame_with_local_map after `motion` (oracle_motion's tuple; its pose may be the device's).
    local: rows of this frame + last_local_idx.  -> dict(matched, local, observable, pose, num_tracked, n_inliers,
    lm_iters, status)."""
    m_pre, m_post, T_motion, nv = motion[0], motion[1], motion[2], motion[3]
    n, nl = len(curr["x"]), len(local["max_valid_dist"])
    lli = np.asarray(local["last_local_idx"], np.int64)
    status = 1 if nl > max_local else (2 if ((lli < -1) | (lli >= nl)).any() else 0)
    out = dict(matched=np.full(n, -1, np.int32), local=np.full(n, -1, np.int32), observable=np.zeros(nl, np.uint8),
               pose=np.asarray(T_motion, np.float64).reshape(4, 4), num_tracked=0, n_inliers=0, lm_iters=0,
               status=status)
    if nv < NUM_TRACKED_THR or status:
        return out
    # search_local_landmarks: the motion track's landmarks, inliers and outliers alike, and the erased ones are skipped
    skip = np.asarray(local["valid"], np.uint8) == 0
    for r in m_pre[m_pre >= 0]:
        if lli[r] >= 0:
            skip[lli[r]] = True
    obs, rx, ry, lvl, _ = can_observe(cam, T_motion, local, skip)
    q = dict(reproj_x=rx, reproj_y=ry, scale_level=np.maximum(lvl, 0), desc=local["desc"], valid=obs)
    frm = dict(x=curr["x"], y=curr["y"], octave=curr["octave"], desc=curr["desc"], claimed=(m_post >= 0).astype(np.uint8))
    best, _ = orc.match_frame_and_landmarks(grid, SF, frm, q, margin, 0.8)
    matched, loc = m_post.copy(), np.full(n, -1, np.int32)
    for j in np.nonzero(best >= 0)[0]:
        loc[best[j]] = j
    idx = np.nonzero((matched >= 0) | (loc >= 0))[0]
    pts = np.zeros(len(idx), oracle_api.PT_OBS_DTYPE)
    from_last = matched[idx] >= 0
    pts["pos_w"][from_last] = np.asarray(last["pos_w"])[matched[idx[from_last]]]
    pts["pos_w"][~from_last] = np.asarray(local["pos_w"]).reshape(-1, 3)[loc[idx[~from_last]]]
    pts["obs_x"], pts["obs_y"] = curr["x"][idx], curr["y"][idx]
    pts["x_right"] = -1.0
    pts["inv_sigma_sq"] = ISIG[curr["octave"][idx]]
    T, pout, _, n_inl, iters = orc.pose_optimize(cam, T_motion, pts)
    if len(idx) >= 5:  # tracking_module.cc:762-784
        matched[idx[pout != 0]] = -1
        loc[idx[pout != 0]] = -1
    out.update(matched=matched, local=loc, observable=obs, pose=T, num_tracked=int(((matched >= 0) | (loc >= 0)).sum()),
               n_inliers=int(n_inl), lm_iters=int(iters))
    return out


def curr_frame(res_t):
    k = res_t["kps"]
    return dict(x=k["x"], y=k["y"], octave=k["octave"], angle=k["angle"], desc=res_t["desc"])


def _kps(res_k, undistort):
    k = res_k["kps"]
    if undistort is None:
        return k
    k = k.copy()
    k["x"], k["y"] = undistort(k["x"], k["y"])
    return k


def build_local_map(seq, res, t, rng, n_earlier=2, last_frame=None, drop_last=0, undistort=None):
    """Frame t's local map: the last frame's landmarks (rows of `last_frame`, the plp_track_last input, with
    last_local_idx pointing at them) and the landmarks of the n_earlier keyframes before it, in a shuffled
    local_landmarks_ order.  drop_last: that many last-frame landmarks are left out (last_local_idx -1).  undistort:
    the keypoint undistortion of a distorted camera (None: none)."""
    lf = last_frame
    nlast = len(lf["octave"])
    last_rows = landmark_rows(seq, t - 1, _kps(res[t - 1], undistort), res[t - 1]["desc"], [k for k in (t - 2, t - 1) if k >= 0])
    last_rows["pos_w"] = np.asarray(lf["pos_w"], np.float64)  # the same landmarks as the motion track's input
    keep = np.ones(nlast, bool)
    if drop_last:
        keep[rng.choice(nlast, drop_last, replace=False)] = False
    parts, src = [take(last_rows, np.nonzero(keep)[0])], [np.nonzero(keep)[0]]
    for k in range(t - 2, t - 2 - n_earlier, -1):
        if k < 0:
            break
        rows = landmark_rows(seq, k, _kps(res[k], undistort), res[k]["desc"], [j for j in (k - 1, k) if j >= 0])
        parts.append(rows)
        src.append(np.full(len(rows["max_valid_dist"]), -1))
    rows = concat(parts)
    origin = np.concatenate(src)  # last-frame row or -1
    perm = rng.permutation(len(origin))
    rows = take(rows, perm)
    origin = origin[perm]
    lli = np.full(nlast, -1, np.int32)
    lli[origin[origin >= 0]] = np.nonzero(origin >= 0)[0]
    rows["last_local_idx"] = lli
    return rows


def with_rows(local, extra):
    """local + extra rows appended (last_local_idx unchanged)."""
    out = concat([{k: local[k] for k in extra}, extra])
    out["last_local_idx"] = local["last_local_idx"]
    return out


def with_erased_run(local, n=64):
    """n erased copies of the first rows put in front of the local list (last_local_idx shifted): the matcher then
    starts with n / 8 warps whose queries are all invalid."""
    k = min(n, len(local["max_valid_dist"]))
    run = {key: np.asarray(local[key])[:k].copy() for key in local if key != "last_local_idx"}
    run["valid"] = np.zeros(k, np.uint8)
    out = concat([run, {key: local[key] for key in run}])
    lli = np.asarray(local["last_local_idx"]).copy()
    lli[lli >= 0] += k
    out["last_local_idx"] = lli
    return out


def curr_frame_u(res_t, undistort=None):
    """curr_frame with the keypoints undistorted (the tracker's undist_keypts_)."""
    k = _kps(res_t, undistort)
    return dict(x=k["x"], y=k["y"], octave=k["octave"], angle=k["angle"], desc=res_t["desc"])


def chain_case(orc, seq, res, ts, preds, lasts, motion_out, grid, cam, rng, max_local, empty=(), undistort=None,
               margin=MARGIN):
    """Local maps for the frames ts (with distractors at the device's motion pose; frames listed in `empty` get none)
    and the oracle's answer for each, given the device's motion outputs.  -> (local_list, wants)."""
    local_list, wants = [], []
    for b, t in enumerate(ts):
        curr = curr_frame_u(res[t], undistort)
        motion = oracle_motion(orc, grid, cam, curr, lasts[b], preds[b], seq.poses[t - 1])
        assert np.array_equal(motion[1], motion_out["matched"][b]), f"motion track of frame {b}"
        if b in empty:
            loc = empty_rows()
            loc["last_local_idx"] = np.full(len(lasts[b]["octave"]), -1, np.int32)
        else:
            loc = build_local_map(seq, res, t, rng, last_frame=lasts[b], drop_last=20, undistort=undistort)
            good = take(loc, np.arange(min(200, len(loc["max_valid_dist"]))))
            good.pop("last_local_idx")
            loc = with_rows(loc, distractors(cam, motion_out["pose"][b], good, rng))
            loc = with_erased_run(loc)
        local_list.append(loc)
        dev_motion = (motion[0], motion[1], motion_out["pose"][b], int(motion_out["num_valid"][b]))
        wants.append(oracle_local_track(orc, grid, cam, curr, lasts[b], loc, dev_motion, max_local, margin))
    return local_list, wants


def compare(out, wants, frames=None, pose_tol=1e-4):
    """Device results of download_local_tracking against the oracle's, frame by frame; -> the LM iteration lists."""
    got_it, want_it = [], []
    for b, w in enumerate(wants):
        if frames is not None and b not in frames:
            continue
        what = f"frame {b}"
        assert out["status"][b] == w["status"], what
        assert np.array_equal(out["observable"][b], w["observable"]), what
        assert np.array_equal(out["matched"][b], w["matched"]), what
        assert np.array_equal(out["local"][b], w["local"]), what
        assert out["num_tracked"][b] == w["num_tracked"] and out["n_inliers"][b] == w["n_inliers"], \
            (what, out["num_tracked"][b], w["num_tracked"], out["n_inliers"][b], w["n_inliers"])
        rel = np.linalg.norm(out["pose"][b] - w["pose"]) / np.linalg.norm(w["pose"])
        assert rel <= pose_tol, (what, rel)
        got_it.append(int(out["lm_iters"][b]))
        want_it.append(w["lm_iters"])
    return got_it, want_it
