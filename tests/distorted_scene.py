"""scene.PlanarSequence seen through a distorted camera, and the oracle's tracking chain for it.

Every frame is rendered through the distortion model: each distorted pixel samples the plane texture at its undistorted
position, which the oracle computes.  Landmarks are back-projected from undistorted keypoints, and oracle_track
undistorts the current keypoints and builds the grid from the undistorted image bounds, as data::frame does
(frame.cc:68-86)."""
from __future__ import annotations

import numpy as np

import camera_data
import scene
import synth


class DistortedPlanarSequence(scene.PlanarSequence):
    def __init__(self, dist, seed=1234, n_frames=9, rows=synth.ROWS, cols=synth.COLS, fx=synth.FX, fy=synth.FY,
                 cx=synth.CX, cy=synth.CY, tex_scale=1.6, plp=False):
        """dist = (model, coefficients) of camera_data (0 perspective, 1 fisheye), the coefficients as a config gives
        them."""
        import cv2
        import oracle_api
        super().__init__(seed=seed, n_frames=n_frames, rows=rows, cols=cols, fx=fx, fy=fy, cx=cx, cy=cy,
                         tex_scale=tex_scale, plp=plp)
        self.dist = dist
        self.orc = oracle_api.Oracle()
        v, u = np.mgrid[0:rows, 0:cols].astype(np.float32)
        ux, uy = self.undistort(u.ravel(), v.ravel())
        und = np.stack([ux.astype(np.float64), uy.astype(np.float64), np.ones(ux.size)], 0)
        frames = []
        for T in self.poses:
            t = np.linalg.inv(self._tex_to_frame(T)) @ und
            mx = (t[0] / t[2]).reshape(rows, cols).astype(np.float32)
            my = (t[1] / t[2]).reshape(rows, cols).astype(np.float32)
            frames.append(cv2.remap(self.tex, mx, my, cv2.INTER_LINEAR, borderMode=cv2.BORDER_REFLECT_101))
        self.frames = np.stack(frames)

    def kvec(self):
        return (self.K[0, 0], self.K[1, 1], self.K[0, 2], self.K[1, 2])

    def undistort(self, x, y):
        """The oracle's undistort_keypoints of this sequence's camera."""
        return camera_data.undistort_keypoints(self.orc, self.dist[0], self.kvec(), self.dist[1], x, y)

    def bounds(self):
        return camera_data.image_bounds(self.orc, self.dist[0], self.kvec(), self.dist[1], self.cols, self.rows)

    def last_frame_landmarks(self, t_last, kps, desc):
        """As scene.PlanarSequence, with the landmarks back-projected from the undistorted keypoints."""
        k = kps.copy()
        k["x"], k["y"] = self.undistort(kps["x"], kps["y"])
        return super().last_frame_landmarks(t_last, k, desc)


def oracle_track(orc, plp, seq: DistortedPlanarSequence, res, t, T_pred, margin=20.0):
    """scene.oracle_track for a distorted sequence: the current keypoints are undistorted with the oracle, the camera
    bounds and the grid come from the oracle's image bounds, the pose optimiser observes undistorted coordinates.
    Returns (matched, pose, num_valid, n_inliers, LM iterations)."""
    import oracle_api
    b = seq.bounds()
    grid = plp.capi.make_grid(seq.cols, seq.rows, min_x=b[0], min_y=b[2], max_x=b[1], max_y=b[3])
    cam = seq.camera(plp)
    cam.min_x, cam.max_x, cam.min_y, cam.max_y = (float(v) for v in b)
    sf, isig = synth.scale_factors(), synth.inv_level_sigma_sq()
    last = seq.last_frame_landmarks(t - 1, res[t - 1]["kps"], res[t - 1]["desc"])
    k = res[t]["kps"].copy()
    k["x"], k["y"] = seq.undistort(k["x"], k["y"])
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
