"""Synthetic monocular sequence with exact geometry (SURVEY.md section 8(d), config 2): a textured plane viewed by a
camera on a smooth SE3 path (<= ~10 px inter-frame flow).  Every keypoint back-projects to a known 3-D point on
the plane, which gives the "last frame landmarks" the tracking stage consumes."""
from __future__ import annotations

import numpy as np

import synth

Z0 = 4.0  # plane depth [m]
# LM iteration counts are compared loosely.  An optimize() call ends when a step leaves the robust chi2 sum exactly
# unchanged (rho == 0, g2o's "terminate").  After convergence that test compares sums whose last bits depend on the
# summation order, which differs between the kernel's warp reductions and the oracle's sequential sums: one side stops,
# the other keeps taking rejected or negligible steps until the trial's 10 iterations run out.  The pose agrees (1e-8
# relative) but a frame's count can differ by up to 9 per trial, either way.  What is checked: a frame runs iterations
# iff the oracle's does, and a batch's total is within LM_ITERS_TOTAL_TOL of the oracle's (plus LM_ITERS_SLACK, for
# batches of a few frames).
LM_ITERS_TOTAL_TOL, LM_ITERS_SLACK = 0.1, 20


def check_lm_iters(got, want, what=""):
    got, want = np.asarray(got, np.int64), np.asarray(want, np.int64)
    assert np.array_equal(got == 0, want == 0), f"{what}: frames without LM iterations differ: {got} vs {want}"
    assert abs(int(got.sum()) - int(want.sum())) <= LM_ITERS_TOTAL_TOL * want.sum() + LM_ITERS_SLACK, \
        f"{what}: {got.sum()} LM iterations vs the oracle's {want.sum()}"


class PlanarSequence:
    def __init__(self, seed=1234, n_frames=9, rows=synth.ROWS, cols=synth.COLS, fx=synth.FX, fy=synth.FY,
                 cx=synth.CX, cy=synth.CY, tex_scale=1.6, plp=False):
        import cv2
        self.rows, self.cols = rows, cols
        self.K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1.0]])
        th, tw = int(rows * tex_scale), int(cols * tex_scale)
        if plp:  # point- and line-rich texture (~1000 ORB + ~200 keylines per frame)
            self.tex = synth.make_plp_texture(seed, th, tw)
        else:
            self.tex = synth.make_texture(seed, th, tw, n_rect=int(400 * tex_scale ** 2), n_blob=int(2000 * tex_scale ** 2))
        s = fx / Z0  # texture pixels per metre: ~1 texture px per image px at depth Z0
        self.A = np.array([[s, 0, tw / 2.0], [0, s, th / 2.0], [0, 0, 1.0]])
        rng = np.random.default_rng(seed + 1)
        # smooth path: constant small velocity + slow sinusoids; <= ~10 px flow per frame
        v = rng.normal(0, 1, 3)
        v = 0.012 * v / np.linalg.norm(v)
        w = rng.normal(0, 1, 3)
        w = 0.0025 * w / np.linalg.norm(w)
        self.poses = []
        for t in range(n_frames):
            T = np.eye(4)
            T[:3, :3] = synth.so3_exp(w * t + 0.002 * np.sin(0.3 * t) * np.array([1.0, 0.5, 0.2]))
            T[:3, 3] = v * t * np.array([1.0, 1.0, 0.3]) + np.array([0.0, 0.0, 0.0])
            self.poses.append(T)
        self.frames = []
        for T in self.poses:
            G = self._tex_to_frame(T)
            self.frames.append(cv2.warpPerspective(self.tex, G, (cols, rows), flags=cv2.INTER_LINEAR,
                                                   borderMode=cv2.BORDER_REFLECT_101))
        self.frames = np.stack(self.frames)

    def camera(self, plp):
        """The plp_camera of K at this sequence's size."""
        K = self.K
        return plp.capi.make_camera(K[0, 0], K[1, 1], K[0, 2], K[1, 2], self.cols, self.rows)

    def _KM(self, T):
        R, t = T[:3, :3], T[:3, 3]
        M = np.stack([R[:, 0], R[:, 1], R[:, 2] * Z0 + t], 1)
        return self.K @ M

    def _tex_to_frame(self, T):
        return self._KM(T) @ np.linalg.inv(self.A)

    def backproject(self, T, x, y):
        """World points on the plane seen at pixel (x, y) of the frame with pose T (cw)."""
        Hinv = np.linalg.inv(self._KM(T))
        u = np.stack([x, y, np.ones_like(x)], 0).astype(np.float64)
        p = Hinv @ u
        return np.stack([p[0] / p[2], p[1] / p[2], np.full(p.shape[1], Z0)], 1)

    def last_frame_landmarks(self, t_last, kps, desc):
        """The arrays of plp_track_last for the frame at index t_last, given its extracted keypoints."""
        pos_w = self.backproject(self.poses[t_last], kps["x"].astype(np.float64), kps["y"].astype(np.float64))
        return dict(pos_w=pos_w, octave=kps["octave"].astype(np.int32), angle=kps["angle"].astype(np.float32),
                    desc=desc.copy(), valid=np.ones(len(kps), np.uint8))

    def predicted_pose(self, t, rng, rot_sigma=0.003, trans_sigma=0.01):
        """Motion-model prediction = ground truth composed with a small error."""
        xi = np.concatenate([rng.normal(0, rot_sigma, 3), rng.normal(0, trans_sigma, 3)])
        dT = np.eye(4)
        dT[:3, :3] = synth.so3_exp(xi[:3])
        dT[:3, 3] = xi[3:]
        return dT @ self.poses[t]


def oracle_track(orc, plp, seq, res, t, T_pred, margin=20.0):
    """The oracle chain of frame_tracker::motion_based_track for frame t of `seq`: match_current_and_last_frames
    (retried with 2 x margin below 20 matches) -> pose_optimize -> discard_outliers.  res[t - 1] / res[t] are oracle
    ORB extractions; plp is the package (only its ctypes structures are used).  The camera is the sequence's own (K).
    Returns (matched, pose, num_valid, n_inliers, LM iterations)."""
    import oracle_api
    grid = plp.capi.make_grid(seq.cols, seq.rows)
    cam = seq.camera(plp)
    sf, isig = synth.scale_factors(), synth.inv_level_sigma_sq()
    last = seq.last_frame_landmarks(t - 1, res[t - 1]["kps"], res[t - 1]["desc"])
    k = res[t]["kps"]
    curr = dict(x=k["x"], y=k["y"], octave=k["octave"], angle=k["angle"], desc=res[t]["desc"])
    # module/frame_tracker.cc:63-77
    m, nm = orc.match_current_and_last_frames(grid, sf, cam, curr, T_pred, seq.poses[t - 1], last, margin, True)
    if nm < 20:
        m, nm = orc.match_current_and_last_frames(grid, sf, cam, curr, T_pred, seq.poses[t - 1], last, 2 * margin, True)
    if nm < 20:  # no pose optimisation: the tracker reports 0 LM iterations
        return np.full(len(k), -1, np.int32), T_pred, 0, 0, 0
    idx = np.nonzero(m >= 0)[0]
    pts = np.zeros(len(idx), oracle_api.PT_OBS_DTYPE)
    pts["pos_w"] = last["pos_w"][m[idx]]
    pts["obs_x"], pts["obs_y"] = k["x"][idx], k["y"][idx]
    pts["x_right"] = -1.0
    pts["inv_sigma_sq"] = isig[k["octave"][idx]]
    T, pout, _, n_inl, iters = orc.pose_optimize(cam, T_pred, pts)
    m = m.copy()
    m[idx[pout != 0]] = -1  # discard_outliers (frame_tracker.cc:253-283)
    return m, T, int((m >= 0).sum()), n_inl, iters
