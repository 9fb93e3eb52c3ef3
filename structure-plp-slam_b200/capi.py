"""ctypes binding of libplpslam_b200.so -- mirrors the reference operator classes by name.

Only marshals numpy arrays into the PODs of include/plpslam_b200.h.  No compute happens here.
"""
from __future__ import annotations

import ctypes as C
import re
from pathlib import Path

import numpy as np

_HERE = Path(__file__).resolve().parent
_LIB = None


class PlpError(RuntimeError):
    pass


def lib_path() -> Path:
    return _HERE / "libplpslam_b200.so"


def declared_symbols() -> list[str]:
    """Every PLP_API function declared in include/plpslam_b200.h."""
    hdr = (_HERE.parent / "include" / "plpslam_b200.h").read_text()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    return sorted(set(re.findall(r"PLP_API[^;{]*?\b(plp_[a-z0-9_]+)\s*\(", hdr)))


def lib() -> C.CDLL:
    """Load the CUDA library; fails loudly when it has not been built (no CPU fallback)."""
    global _LIB
    if _LIB is None:
        p = lib_path()
        if not p.exists():
            raise PlpError(
                f"{p} is missing: build it with `python structure-plp-slam_b200/build.py` "
                "(or __graft_entry__.build()); there is no CPU fallback"
            )
        _LIB = C.CDLL(str(p))
        _LIB.plp_last_error.restype = C.c_char_p
        _LIB.plp_ctx_stream.restype = C.c_void_p
        _LIB.plp_ctx_launch_count.restype = C.c_uint64
    return _LIB


# ----------------------------------------------------------------------------- PODs
class Grid(C.Structure):
    _fields_ = [("min_x", C.c_float), ("min_y", C.c_float), ("inv_cell_width", C.c_double),
                ("inv_cell_height", C.c_double), ("num_cols", C.c_int32), ("num_rows", C.c_int32)]


class Camera(C.Structure):
    _fields_ = [("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double),
                ("focal_x_baseline", C.c_double), ("true_baseline", C.c_double),
                ("min_x", C.c_float), ("max_x", C.c_float), ("min_y", C.c_float), ("max_y", C.c_float),
                ("setup_type", C.c_int32)]


_P = C.c_void_p


class Distortion(C.Structure):
    _fields_ = [("model", C.c_int32), ("k", C.c_double * 5)]


PERSPECTIVE, FISHEYE = 0, 1


class FramePoints(C.Structure):
    _fields_ = [("n", C.c_int32), ("x", _P), ("y", _P), ("octave", _P), ("angle", _P), ("x_right", _P),
                ("desc", _P), ("claimed", _P)]


class FrameLines(C.Structure):
    _fields_ = [("n", C.c_int32), ("sx", _P), ("sy", _P), ("ex", _P), ("ey", _P), ("octave", _P),
                ("ratio_level", _P), ("x_right_sp", _P), ("x_right_ep", _P), ("desc", _P), ("claimed", _P)]


class LandmarkQueries(C.Structure):
    _fields_ = [("m", C.c_int32), ("reproj_x", _P), ("reproj_y", _P), ("x_right", _P), ("scale_level", _P),
                ("desc", _P), ("valid", _P)]


class LastFramePoints(C.Structure):
    _fields_ = [("n", C.c_int32), ("pos_w", _P), ("octave", _P), ("angle", _P), ("desc", _P), ("valid", _P)]


class LineQueries(C.Structure):
    _fields_ = [("m", C.c_int32), ("sp_x", _P), ("sp_y", _P), ("ep_x", _P), ("ep_y", _P), ("scale_level", _P),
                ("desc", _P), ("valid", _P)]


class LastFrameLines(C.Structure):
    _fields_ = [("n", C.c_int32), ("pos_w", _P), ("octave", _P), ("desc", _P), ("valid", _P)]


class KeyframePoints(C.Structure):
    _fields_ = [("n", C.c_int32), ("desc", _P), ("angle", _P), ("octave", _P), ("bearings", _P), ("has_landmark", _P),
                ("x_right", _P)]


class BowFeatureVector(C.Structure):
    _fields_ = [("num_nodes", C.c_int32), ("node_ids", _P), ("offsets", _P), ("indices", _P)]


class FuseLandmarks(C.Structure):
    _fields_ = [("m", C.c_int32), ("pos_w", _P), ("obs_mean_normal", _P), ("min_valid_dist", _P),
                ("max_valid_dist", _P), ("max_valid_dist_raw", _P), ("desc", _P), ("valid", _P)]


class FuseTargetPoints(C.Structure):
    _fields_ = [("pts", FramePoints), ("rot_cw", C.c_double * 9), ("trans_cw", C.c_double * 3),
                ("cam_center", C.c_double * 3), ("skip", _P)]


class FuseTargetLines(C.Structure):
    _fields_ = [("lines", FrameLines), ("rot_cw", C.c_double * 9), ("trans_cw", C.c_double * 3),
                ("cam_center", C.c_double * 3), ("skip", _P)]


FUSE_DETECT, FUSE_REPLACE = 0, 1


def fuse_level_thresholds(log_scale_factor: float, num_levels: int) -> np.ndarray:
    """Host-side table behind the device predict_scale_level (no GPU needed)."""
    out = np.zeros(max(num_levels, 1), np.float32)
    st = lib().plp_fuse_level_thresholds(C.c_float(log_scale_factor), C.c_int(num_levels), out.ctypes.data_as(_P))
    if st != 0:
        raise PlpError(f"plp status {st}: {lib().plp_last_error().decode()}")
    return out


class BowSide(C.Structure):
    _fields_ = [("n", C.c_int32), ("desc", _P), ("angle", _P), ("valid", _P), ("fv", BowFeatureVector)]


class BowPair(C.Structure):
    _fields_ = [("side1", C.POINTER(BowSide)), ("side2", C.POINTER(BowSide)), ("matched_2_of_1_out", _P),
                ("matched_1_of_2_out", _P), ("num_matches", C.c_uint32)]


class PlaneRansacCfg(C.Structure):
    _fields_ = [("mode", C.c_int32), ("points_per_ransac", C.c_int32), ("planar_distance_thresh", C.c_double),
                ("final_error_thresh", C.c_double), ("inliers_ratio_thr", C.c_double), ("initial_best_error", C.c_double)]


class OrbParams(C.Structure):
    _fields_ = [("max_num_keypts", C.c_uint32), ("scale_factor", C.c_float), ("num_levels", C.c_uint32),
                ("ini_fast_thr", C.c_uint32), ("min_fast_thr", C.c_uint32)]


class ImageView(C.Structure):
    _fields_ = [("data", _P), ("rows", C.c_int32), ("cols", C.c_int32), ("step", C.c_size_t)]


PT_OBS_DTYPE = np.dtype([("pos_w", "<f8", 3), ("obs_x", "<f4"), ("obs_y", "<f4"), ("x_right", "<f4"),
                         ("inv_sigma_sq", "<f4")])
LINE_OBS_DTYPE = np.dtype([("plucker", "<f8", 6), ("sp_x", "<f4"), ("sp_y", "<f4"), ("ep_x", "<f4"), ("ep_y", "<f4"),
                           ("inv_sigma_sq", "<f4"), ("pad", "<f4")])


class PoseOptCfg(C.Structure):
    _fields_ = [("num_trials", C.c_int32), ("num_each_iter", C.c_int32)]


# binary layout of plp_keypoint / cv::KeyPoint
KP_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"),
                     ("octave", "<i4"), ("class_id", "<i4")])


# ----------------------------------------------------------------------------- helpers
class _Keep:
    """Keeps converted numpy arrays alive for the duration of a call."""

    def __init__(self):
        self.refs = []

    def arr(self, a, dtype, allow_none=True):
        if a is None:
            if not allow_none:
                raise PlpError("required array is None")
            return None
        a = np.ascontiguousarray(a, dtype=dtype)
        self.refs.append(a)
        return a.ctypes.data_as(_P)


def make_grid(cols: int, rows: int, num_cols: int = 64, num_rows: int = 48, min_x=0.0, min_y=0.0,
              max_x=None, max_y=None) -> Grid:
    """camera::perspective ctor (camera/perspective.cc:53-56) for an undistorted camera."""
    max_x = float(cols) if max_x is None else max_x
    max_y = float(rows) if max_y is None else max_y
    fmin_x, fmax_x = np.float32(min_x), np.float32(max_x)
    fmin_y, fmax_y = np.float32(min_y), np.float32(max_y)
    return Grid(float(fmin_x), float(fmin_y), float(num_cols) / float(np.float32(fmax_x - fmin_x)),
                float(num_rows) / float(np.float32(fmax_y - fmin_y)), num_cols, num_rows)


def make_camera(fx, fy, cx, cy, cols, rows, bf=-1.0, setup_type=0) -> Camera:
    return Camera(fx, fy, cx, cy, bf, (bf / fx) if bf > 0 else -1.0, 0.0, float(cols), 0.0, float(rows), setup_type)


def make_distortion(model, *k) -> Distortion:
    """plp_distortion of a config: model 0 perspective (k1, k2, p1, p2, k3) or 1 fisheye (k1, k2, k3, k4); the
    coefficients as the YAML gives them (the library rounds them to float like the reference)."""
    if model not in (PERSPECTIVE, FISHEYE) or len(k) > (5 if model == PERSPECTIVE else 4):
        raise PlpError(f"distortion model {model} with {len(k)} coefficients")
    return Distortion(model, (C.c_double * 5)(*([float(v) for v in k] + [0.0] * (5 - len(k)))))


def image_bounds(cam: Camera, dist: Distortion, cols: int, rows: int) -> np.ndarray:
    """camera::*::compute_image_bounds through plp_camera_image_bounds -> float32 (min_x, max_x, min_y, max_y)."""
    out = np.zeros(4, np.float32)
    st = lib().plp_camera_image_bounds(C.byref(cam), C.byref(dist), C.c_int(cols), C.c_int(rows), out.ctypes.data_as(_P))
    if st != 0:
        raise PlpError(f"plp status {st}: {lib().plp_last_error().decode()}")
    return out


def make_distorted_camera(fx, fy, cx, cy, cols, rows, dist: Distortion, num_cols: int = 64, num_rows: int = 48):
    """(plp_camera, plp_grid) of a distorted camera: img_bounds_ and the grid from the undistorted image corners, as the
    camera::perspective / camera::fisheye constructors compute them."""
    cam = make_camera(fx, fy, cx, cy, cols, rows)
    b = image_bounds(cam, dist, cols, rows)
    cam.min_x, cam.max_x, cam.min_y, cam.max_y = (float(v) for v in b)
    grid = make_grid(cols, rows, num_cols, num_rows, min_x=b[0], min_y=b[2], max_x=b[1], max_y=b[3])
    return cam, grid


class Context:
    """One plp_ctx (device + stream).  Methods are named after the reference methods they replace."""

    def __init__(self, device: int = 0, high_priority: bool = False):
        self._lib = lib()
        self.device = int(device)
        h = C.c_void_p()
        self._h = None
        self._check(self._lib.plp_ctx_create_ex(C.c_int(device), C.c_int(1 if high_priority else 0), C.byref(h)))
        self._h = h

    def close(self):
        if self._h is not None:
            self._lib.plp_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, status: int):
        if status != 0:
            raise PlpError(f"plp status {status}: {self._lib.plp_last_error().decode()}")

    @property
    def handle(self):
        return self._h

    def wait(self, other: "Context"):
        """This context's stream waits for everything enqueued so far on `other`."""
        self._check(self._lib.plp_ctx_wait_ctx(self._h, other._h))

    def sync(self):
        self._check(self._lib.plp_ctx_sync(self._h))

    def launch_count(self) -> int:
        return int(self._lib.plp_ctx_launch_count(self._h))

    # ------------------------------------------------------------------ camera::{perspective,fisheye}
    def undistort_keypoints(self, cam, dist, kps):
        """undistort_keypoints + convert_keypoints_to_bearings of a host KP_DTYPE array -> (undistorted kps, bearings)."""
        kp = np.ascontiguousarray(kps, KP_DTYPE)
        out = np.zeros(len(kp), KP_DTYPE)
        bear = np.zeros((len(kp), 3), np.float64)
        self._check(self._lib.plp_undistort_keypoints(self._h, C.byref(cam), C.byref(dist), kp.ctypes.data_as(_P),
                                                      C.c_int(len(kp)), out.ctypes.data_as(_P), bear.ctypes.data_as(_P)))
        return out, bear

    def undistort_keypoints_dev(self, cam, dist, batch, cap, d_kp, d_n_kp, d_undist_out, d_bearings_out=None):
        """Device-resident form on the arrays OrbExtractor / plp_orb_extract_batch_dev write (device pointers)."""
        self._check(self._lib.plp_undistort_keypoints_batch_dev(self._h, C.byref(cam), C.byref(dist), C.c_int(batch),
                                                                C.c_int(cap), d_kp, d_n_kp, d_undist_out, d_bearings_out))

    # ------------------------------------------------------------------ match/base.h
    def hamming_matrix(self, a, b):
        k = _Keep()
        a = np.ascontiguousarray(a, np.uint8).reshape(-1, 32)
        b = np.ascontiguousarray(b, np.uint8).reshape(-1, 32)
        out = np.zeros((a.shape[0], b.shape[0]), np.uint16)
        self._check(self._lib.plp_hamming_matrix(self._h, k.arr(a, np.uint8), C.c_int(a.shape[0]),
                                                 k.arr(b, np.uint8), C.c_int(b.shape[0]), out.ctypes.data_as(_P)))
        return out

    def hamming_nn(self, query, train):
        k = _Keep()
        q = np.ascontiguousarray(query, np.uint8).reshape(-1, 32)
        t = np.ascontiguousarray(train, np.uint8).reshape(-1, 32)
        idx = np.zeros(q.shape[0], np.int32)
        dist = np.zeros(q.shape[0], np.uint16)
        self._check(self._lib.plp_hamming_nn(self._h, k.arr(q, np.uint8), C.c_int(q.shape[0]), k.arr(t, np.uint8),
                                             C.c_int(t.shape[0]), idx.ctypes.data_as(_P), dist.ctypes.data_as(_P)))
        return idx, dist

    # ------------------------------------------------------------------ match::projection
    @staticmethod
    def _frame_points(k, x, y, octave, desc, angle=None, x_right=None, claimed=None):
        n = len(x)
        return FramePoints(n, k.arr(x, np.float32), k.arr(y, np.float32), k.arr(octave, np.int32),
                           k.arr(angle, np.float32), k.arr(x_right, np.float32), k.arr(desc, np.uint8),
                           k.arr(claimed, np.uint8))

    def match_frame_and_landmarks(self, grid, scale_factors, frm, queries, margin, lowe_ratio=0.6):
        """projection::match_frame_and_landmarks. frm/queries are dicts of arrays."""
        k = _Keep()
        fp = self._frame_points(k, frm["x"], frm["y"], frm["octave"], frm["desc"], frm.get("angle"),
                                frm.get("x_right"), frm.get("claimed"))
        m = len(queries["reproj_x"])
        q = LandmarkQueries(m, k.arr(queries["reproj_x"], np.float32), k.arr(queries["reproj_y"], np.float32),
                            k.arr(queries.get("x_right"), np.float32), k.arr(queries["scale_level"], np.int32),
                            k.arr(queries["desc"], np.uint8), k.arr(queries.get("valid"), np.uint8))
        sf = np.ascontiguousarray(scale_factors, np.float32)
        best = np.full(m, -2, np.int32)
        num = C.c_uint32(0)
        self._check(self._lib.plp_match_frame_and_landmarks(
            self._h, C.byref(fp), C.byref(grid), sf.ctypes.data_as(_P), C.c_int(len(sf)), C.byref(q),
            C.c_float(margin), C.c_float(lowe_ratio), best.ctypes.data_as(_P), C.byref(num)))
        return best, int(num.value)

    def match_current_and_last_frames(self, grid, scale_factors, cam, curr, pose_cw_curr, pose_cw_last, last,
                                      margin, check_orientation=True):
        k = _Keep()
        fp = self._frame_points(k, curr["x"], curr["y"], curr["octave"], curr["desc"], curr.get("angle"),
                                curr.get("x_right"), curr.get("claimed"))
        n_last = len(last["octave"])
        lp = LastFramePoints(n_last, k.arr(last["pos_w"], np.float64), k.arr(last["octave"], np.int32),
                             k.arr(last.get("angle"), np.float32), k.arr(last["desc"], np.uint8),
                             k.arr(last.get("valid"), np.uint8))
        sf = np.ascontiguousarray(scale_factors, np.float32)
        Tc = np.ascontiguousarray(pose_cw_curr, np.float64).reshape(4, 4)
        Tl = np.ascontiguousarray(pose_cw_last, np.float64).reshape(4, 4)
        matched = np.full(fp.n, -2, np.int32)
        num = C.c_uint32(0)
        self._check(self._lib.plp_match_current_and_last_frames(
            self._h, C.byref(fp), C.byref(grid), sf.ctypes.data_as(_P), C.c_int(len(sf)), C.byref(cam),
            Tc.ctypes.data_as(_P), Tl.ctypes.data_as(_P), C.byref(lp), C.c_float(margin),
            C.c_int(1 if check_orientation else 0), matched.ctypes.data_as(_P), C.byref(num)))
        return matched, int(num.value)

    def match_frame_and_keyframe(self, grid, scale_factors, frm, q, margin, hamm_dist_thr, check_orientation=True):
        """projection::match_frame_and_keyframe; q = flattened queries (reproj_x/y, scale_level, desc, angle, valid)."""
        k = _Keep()
        fp = self._frame_points(k, frm["x"], frm["y"], frm["octave"], frm["desc"], frm.get("angle"), None,
                                frm.get("claimed"))
        m = len(q["scale_level"])
        lq = LandmarkQueries(m, k.arr(q["reproj_x"], np.float32), k.arr(q["reproj_y"], np.float32), None,
                             k.arr(q["scale_level"], np.int32), k.arr(q["desc"], np.uint8), k.arr(q.get("valid"), np.uint8))
        sf = np.ascontiguousarray(scale_factors, np.float32)
        matched = np.full(fp.n, -2, np.int32)
        num = C.c_uint32(0)
        self._check(self._lib.plp_match_frame_and_keyframe(
            self._h, C.byref(fp), C.byref(grid), sf.ctypes.data_as(_P), C.c_int(len(sf)), C.byref(lq),
            k.arr(q.get("angle"), np.float32), C.c_float(margin), C.c_uint(hamm_dist_thr),
            C.c_int(1 if check_orientation else 0), matched.ctypes.data_as(_P), C.byref(num)))
        return matched, int(num.value)

    def match_frame_and_keyframe_line(self, scale_factors_lsd, frm, q, margin, hamm_dist_thr):
        """projection::match_frame_and_keyframe_line; q = flattened queries (sp/ep, scale_level, desc, valid)."""
        k = _Keep()
        fl = self._frame_lines(k, frm)
        m = len(q["scale_level"])
        lq = LineQueries(m, k.arr(q["sp_x"], np.float32), k.arr(q["sp_y"], np.float32), k.arr(q["ep_x"], np.float32),
                         k.arr(q["ep_y"], np.float32), k.arr(q["scale_level"], np.int32), k.arr(q["desc"], np.uint8),
                         k.arr(q.get("valid"), np.uint8))
        sf = np.ascontiguousarray(scale_factors_lsd, np.float32)
        matched = np.full(fl.n, -2, np.int32)
        num = C.c_uint32(0)
        self._check(self._lib.plp_match_frame_and_keyframe_line(
            self._h, C.byref(fl), sf.ctypes.data_as(_P), C.c_int(len(sf)), C.byref(lq), C.c_float(margin),
            C.c_uint(hamm_dist_thr), matched.ctypes.data_as(_P), C.byref(num)))
        return matched, int(num.value)

    # ------------------------------------------------------------------ match::fuse
    @staticmethod
    def _fuse_landmarks(k, lms, width):
        m = len(lms["min_valid_dist"])
        pos = np.ascontiguousarray(lms["pos_w"], np.float64).reshape(m, width)
        return FuseLandmarks(m, k.arr(pos, np.float64), k.arr(lms.get("obs_mean_normal"), np.float64),
                             k.arr(lms["min_valid_dist"], np.float32), k.arr(lms["max_valid_dist"], np.float32),
                             k.arr(lms["max_valid_dist_raw"], np.float32), k.arr(lms["desc"], np.uint8),
                             k.arr(lms.get("valid"), np.uint8))

    @staticmethod
    def _fuse_pose(t, tgt):
        R = np.ascontiguousarray(tgt["rot_cw"], np.float64).reshape(9)
        tr = np.ascontiguousarray(tgt["trans_cw"], np.float64).reshape(3)
        cc = np.ascontiguousarray(tgt["cam_center"], np.float64).reshape(3)
        t.rot_cw = (C.c_double * 9)(*R)
        t.trans_cw = (C.c_double * 3)(*tr)
        t.cam_center = (C.c_double * 3)(*cc)

    def fuse_search_points(self, grid, cam, scale_factors, inv_level_sigma_sq, log_scale_factor, targets, lms, margin,
                           mode=FUSE_REPLACE):
        """match::fuse::replace_duplication / detect_duplication search for a (target keyframe x landmark) batch.
        targets: list of dict(x, y, octave, desc[, x_right], rot_cw, trans_cw, cam_center[, skip]);
        lms: dict(pos_w, obs_mean_normal, min_valid_dist, max_valid_dist, max_valid_dist_raw, desc[, valid]).
        Returns (best_idx[num_targets, m], best_dist[num_targets, m])."""
        k = _Keep()
        L = self._fuse_landmarks(k, lms, 3)
        arr = (FuseTargetPoints * max(len(targets), 1))()
        for i, tgt in enumerate(targets):
            arr[i].pts = self._frame_points(k, tgt["x"], tgt["y"], tgt["octave"], tgt["desc"], None, tgt.get("x_right"))
            self._fuse_pose(arr[i], tgt)
            arr[i].skip = k.arr(tgt.get("skip"), np.uint8)
        sf = np.ascontiguousarray(scale_factors, np.float32)
        isg = np.ascontiguousarray(inv_level_sigma_sq, np.float32)
        best = np.full((len(targets), L.m), -2, np.int32)
        dist = np.full((len(targets), L.m), 0xFFFE, np.uint16)
        self._check(self._lib.plp_fuse_search_points(
            self._h, arr, C.c_int(len(targets)), C.byref(grid), C.byref(cam), sf.ctypes.data_as(_P),
            isg.ctypes.data_as(_P), C.c_int(len(sf)), C.c_float(log_scale_factor), C.byref(L), C.c_float(margin),
            C.c_int(mode), best.ctypes.data_as(_P), dist.ctypes.data_as(_P)))
        return best, dist

    def fuse_search_lines(self, cam, scale_factors_lsd, inv_level_sigma_sq_lsd, log_scale_factor_lsd, targets, lms,
                          margin):
        """match::fuse::replace_duplication_line search; targets: list of dict(sx, sy, ex, ey, octave, desc, rot_cw,
        trans_cw, cam_center[, skip]); lms: dict(pos_w (m x 6), min/max_valid_dist, max_valid_dist_raw, desc[, valid])."""
        k = _Keep()
        L = self._fuse_landmarks(k, lms, 6)
        arr = (FuseTargetLines * max(len(targets), 1))()
        for i, tgt in enumerate(targets):
            arr[i].lines = self._frame_lines(k, tgt)
            self._fuse_pose(arr[i], tgt)
            arr[i].skip = k.arr(tgt.get("skip"), np.uint8)
        sf = np.ascontiguousarray(scale_factors_lsd, np.float32)
        isg = np.ascontiguousarray(inv_level_sigma_sq_lsd, np.float32)
        best = np.full((len(targets), L.m), -2, np.int32)
        dist = np.full((len(targets), L.m), 0xFFFE, np.uint16)
        self._check(self._lib.plp_fuse_search_lines(
            self._h, arr, C.c_int(len(targets)), C.byref(cam), sf.ctypes.data_as(_P), isg.ctypes.data_as(_P),
            C.c_int(len(sf)), C.c_float(log_scale_factor_lsd), C.byref(L), C.c_float(margin), best.ctypes.data_as(_P),
            dist.ctypes.data_as(_P)))
        return best, dist

    # ------------------------------------------------------------------ match::bow_tree
    def match_bow_tree(self, pairs, lowe_ratio, check_orientation=True):
        """match::bow_tree::match_frame_and_keyframe / match_keyframes for a batch of (side1, side2) pairs.
        A side is a dict(desc, angle[, valid], fv=(node_ids, offsets, indices)); dict objects may be shared between pairs.
        Returns a list of (matched_2_of_1, matched_1_of_2, num_matches)."""
        k = _Keep()
        sides = {}

        def side(f):
            if id(f) not in sides:
                fv = f["fv"]
                s = BowSide(len(f["desc"]), k.arr(f["desc"], np.uint8), k.arr(f.get("angle"), np.float32),
                            k.arr(f.get("valid"), np.uint8),
                            BowFeatureVector(len(fv[0]), k.arr(fv[0], np.uint32), k.arr(fv[1], np.int32),
                                             k.arr(fv[2], np.uint32)))
                sides[id(f)] = s
            return sides[id(f)]
        arr = (BowPair * max(len(pairs), 1))()
        outs = []
        for i, (a, b) in enumerate(pairs):
            sa, sb = side(a), side(b)
            m21 = np.full(max(sa.n, 1), -2, np.int32)
            m12 = np.full(max(sb.n, 1), -2, np.int32)
            arr[i].side1 = C.pointer(sa)
            arr[i].side2 = C.pointer(sb)
            arr[i].matched_2_of_1_out = m21.ctypes.data_as(_P)
            arr[i].matched_1_of_2_out = m12.ctypes.data_as(_P)
            outs.append((m21, m12, sa.n, sb.n))
        self._check(self._lib.plp_match_bow_tree(self._h, arr, C.c_int(len(pairs)), C.c_float(lowe_ratio),
                                                 C.c_int(1 if check_orientation else 0)))
        return [(m21[:n1].copy(), m12[:n2].copy(), int(arr[i].num_matches)) for i, (m21, m12, n1, n2) in enumerate(outs)]

    # ------------------------------------------------------------------ solve::essential_solver
    def essential_ransac(self, bearings_1, bearings_2, matches_12, samples, recompute=False):
        """solve::essential_solver::find_via_ransac with caller-drawn sample sets (num_iter x 8 match indices).
        Returns (solution_is_valid, is_inlier, E_21, best_score)."""
        b1 = np.ascontiguousarray(bearings_1, np.float64).reshape(-1, 3)
        b2 = np.ascontiguousarray(bearings_2, np.float64).reshape(-1, 3)
        m = np.ascontiguousarray(matches_12, np.int32).reshape(-1, 2)
        sm = np.ascontiguousarray(samples, np.int32).reshape(-1, 8)
        inl = np.zeros(max(len(m), 1), np.uint8)
        E = np.zeros(9, np.float64)
        score, valid = C.c_double(0.0), C.c_int32(0)
        self._check(self._lib.plp_essential_ransac(
            self._h, b1.ctypes.data_as(_P), C.c_int(len(b1)), b2.ctypes.data_as(_P), C.c_int(len(b2)),
            m.ctypes.data_as(_P), C.c_int(len(m)), sm.ctypes.data_as(_P), C.c_int(len(sm)), C.c_int(1 if recompute else 0),
            inl.ctypes.data_as(_P), E.ctypes.data_as(_P), C.byref(score), C.byref(valid)))
        return int(valid.value), inl[:len(m)].copy(), E.reshape(3, 3), float(score.value)

    # ------------------------------------------------------------------ solve::pnp_solver
    def pnp_ransac(self, corr_offsets, bearings, pos_w, max_cos_error, samples, min_num_inliers=10, recompute=True):
        """solve::pnp_solver::find_via_ransac of P problems in one call (plp_pnp_ransac).  corr_offsets: P + 1; bearings,
        pos_w: N x 3; max_cos_error: N float; samples: P x num_iter x 4 problem-local indices.  Returns (valid (P),
        num_inliers (P), pose_cw (P x 4 x 4, NaN where not written), is_inlier (N, 255 where not written))."""
        off = np.ascontiguousarray(corr_offsets, np.int32)
        P = len(off) - 1
        N = int(off[-1]) if P >= 0 and len(off) else 0
        k = _Keep()
        sm = np.ascontiguousarray(samples, np.int32)
        num_iter = int(sm.shape[1]) if sm.ndim == 3 else 0
        valid = np.zeros(max(P, 1), np.int32)
        num = np.zeros(max(P, 1), np.int32)
        pose = np.full((max(P, 1), 16), np.nan)
        flags = np.full(max(N, 1), 255, np.uint8)
        self._check(self._lib.plp_pnp_ransac(
            self._h, C.c_int(P), k.arr(off, np.int32), k.arr(np.reshape(bearings, -1), np.float64),
            k.arr(np.reshape(pos_w, -1), np.float64), k.arr(max_cos_error, np.float32), k.arr(sm.reshape(-1), np.int32),
            C.c_int(num_iter), C.c_int(min_num_inliers), C.c_int(1 if recompute else 0), valid.ctypes.data_as(_P),
            num.ctypes.data_as(_P), pose.ctypes.data_as(_P), flags.ctypes.data_as(_P)))
        return valid[:P].copy(), num[:P].copy(), pose[:P].reshape(P, 4, 4).copy(), flags[:N].copy()

    # ------------------------------------------------------------------ solve::sim3_solver
    def sim3_ransac(self, corr_offsets, cams, pts_1, pts_2, chi_sq_1, chi_sq_2, samples, fix_scale=False,
                    min_num_inliers=20):
        """solve::sim3_solver::find_via_ransac of P problems in one call (plp_sim3_ransac).  corr_offsets: P + 1; cams: P
        Camera structs (fx, fy, cx, cy read); pts_1, pts_2: N x 3 camera-frame points; chi_sq_1, chi_sq_2: N float;
        samples: P x num_iter x 3 problem-local indices.  Returns (valid (P), num_inliers (P), rot_12 (P x 3 x 3),
        trans_12 (P x 3), scale_12 (P, float32))."""
        off = np.ascontiguousarray(corr_offsets, np.int32)
        P = len(off) - 1
        if len(cams) != P:
            raise PlpError(f"sim3_ransac: {len(cams)} cameras for {P} problems")
        k = _Keep()
        cam_arr = (Camera * max(P, 1))(*cams)
        sm = np.ascontiguousarray(samples, np.int32)
        num_iter = int(sm.shape[1]) if sm.ndim == 3 else 0
        valid = np.zeros(max(P, 1), np.int32)
        num = np.zeros(max(P, 1), np.int32)
        rot = np.zeros((max(P, 1), 9))
        trans = np.zeros((max(P, 1), 3))
        scale = np.zeros(max(P, 1), np.float32)
        self._check(self._lib.plp_sim3_ransac(
            self._h, C.c_int(P), k.arr(off, np.int32), cam_arr, k.arr(np.reshape(pts_1, -1), np.float64),
            k.arr(np.reshape(pts_2, -1), np.float64), k.arr(chi_sq_1, np.float32), k.arr(chi_sq_2, np.float32),
            k.arr(sm.reshape(-1), np.int32), C.c_int(num_iter), C.c_int(1 if fix_scale else 0), C.c_int(min_num_inliers),
            valid.ctypes.data_as(_P), num.ctypes.data_as(_P), rot.ctypes.data_as(_P), trans.ctypes.data_as(_P),
            scale.ctypes.data_as(_P)))
        return valid[:P].copy(), num[:P].copy(), rot[:P].reshape(P, 3, 3).copy(), trans[:P].copy(), scale[:P].copy()

    # ------------------------------------------------------------------ optimize::transform_optimizer
    def sim3_optimize(self, match_offsets, cams, rot_1w, trans_1w, rot_2w, trans_2w, rot_12, trans_12, scale_12, pos_w_1,
                      pos_w_2, obs_1, obs_2, inv_sigma_sq_1, inv_sigma_sq_2, chi_sq=10.0, num_iter=10, fix_scale=False):
        """transform_optimizer::optimize of P problems in one call (plp_sim3_optimize).  match_offsets: P + 1; cams: P
        Camera structs (fx, fy, cx, cy read); rot_1w, rot_2w, rot_12: P x 3 x 3; trans_1w, trans_2w, trans_12: P x 3;
        scale_12: P (double); pos_w_1, pos_w_2: N x 3; obs_1, obs_2: N x 2 float; inv_sigma_sq_1, _2: N float.  Returns
        (num_inliers (P), rot_12 (P x 3 x 3), trans_12 (P x 3), scale_12 (P), inlier (N, uint8))."""
        off = np.ascontiguousarray(match_offsets, np.int32)
        P = len(off) - 1
        if len(cams) != P:
            raise PlpError(f"sim3_optimize: {len(cams)} cameras for {P} problems")
        N = int(off[-1]) if P >= 0 and len(off) else 0
        k = _Keep()
        cam_arr = (Camera * max(P, 1))(*cams)
        num = np.zeros(max(P, 1), np.int32)
        rot = np.zeros((max(P, 1), 9))
        trans = np.zeros((max(P, 1), 3))
        scale = np.zeros(max(P, 1))
        inl = np.zeros(max(N, 1), np.uint8)
        d = lambda a: k.arr(np.reshape(a, -1), np.float64)
        f = lambda a: k.arr(np.reshape(a, -1), np.float32)
        self._check(self._lib.plp_sim3_optimize(
            self._h, C.c_int(P), k.arr(off, np.int32), cam_arr, d(rot_1w), d(trans_1w), d(rot_2w), d(trans_2w), d(rot_12),
            d(trans_12), d(scale_12), d(pos_w_1), d(pos_w_2), f(obs_1), f(obs_2), f(inv_sigma_sq_1), f(inv_sigma_sq_2),
            C.c_float(chi_sq), C.c_int(num_iter), C.c_int(1 if fix_scale else 0), num.ctypes.data_as(_P),
            rot.ctypes.data_as(_P), trans.ctypes.data_as(_P), scale.ctypes.data_as(_P), inl.ctypes.data_as(_P)))
        return num[:P].copy(), rot[:P].reshape(P, 3, 3).copy(), trans[:P].copy(), scale[:P].copy(), inl[:N].copy()

    # ------------------------------------------------------------------ Planar_Mapping_module
    def plane_ransac(self, pos_w, valid, samples, cfg, eq0=(0, 0, 0, 0), err0=0.0):
        """estimate_plane_sequential_RANSAC (cfg['mode'] = 0) / update_plane_via_RANSAC (1) with caller-drawn index samples
        (num_iter x sample_size).  Returns (status, eq, plane_error, inlier flags)."""
        P = np.ascontiguousarray(pos_w, np.float64).reshape(-1, 3)
        sm = np.ascontiguousarray(samples, np.int32)
        sm = sm.reshape(len(sm), -1) if sm.size else sm.reshape(0, 1)
        v = None if valid is None else np.ascontiguousarray(valid, np.uint8)
        c = PlaneRansacCfg(cfg["mode"], cfg["points_per_ransac"], cfg["planar_distance_thresh"], cfg["final_error_thresh"],
                           cfg["inliers_ratio_thr"], cfg.get("initial_best_error", 0.0))
        eq = np.array(eq0, np.float64)
        err = C.c_double(err0)
        inl = np.zeros(max(len(P), 1), np.uint8)
        st = C.c_int32(0)
        self._check(self._lib.plp_plane_ransac(
            self._h, P.ctypes.data_as(_P), None if v is None else v.ctypes.data_as(_P), C.c_int(len(P)),
            sm.ctypes.data_as(_P), C.c_int(sm.shape[0]), C.c_int(sm.shape[1]), C.byref(c), eq.ctypes.data_as(_P),
            C.byref(err), inl.ctypes.data_as(_P), C.byref(st)))
        return int(st.value), eq, float(err.value), inl[:len(P)].copy()

    def landmark_compute_descriptor_batch(self, descs, offsets):
        """landmark::compute_descriptor for a batch: index of the median-distance observation per landmark."""
        d = np.ascontiguousarray(descs, np.uint8).reshape(-1, 32)
        o = np.ascontiguousarray(offsets, np.int32)
        out = np.full(max(len(o) - 1, 1), -2, np.int32)
        self._check(self._lib.plp_landmark_compute_descriptor_batch(self._h, d.ctypes.data_as(_P), o.ctypes.data_as(_P),
                                                                   C.c_int(len(o) - 1), out.ctypes.data_as(_P)))
        return out[:len(o) - 1].copy()

    def match_for_triangulation(self, kf1, kf2, fv1, fv2, E_12, epipole, scale_factors_1, check_orientation=True):
        """robust::match_for_triangulation; kf = dict(desc, angle, octave, bearings, has_landmark[, x_right]);
        fv = (node_ids, offsets, indices)."""
        k = _Keep()

        def kp(f):
            return KeyframePoints(len(f["desc"]), k.arr(f["desc"], np.uint8), k.arr(f.get("angle"), np.float32),
                                  k.arr(f.get("octave"), np.int32), k.arr(f["bearings"], np.float64),
                                  k.arr(f["has_landmark"], np.uint8), k.arr(f.get("x_right"), np.float32))

        def bv(f):
            return BowFeatureVector(len(f[0]), k.arr(f[0], np.uint32), k.arr(f[1], np.int32), k.arr(f[2], np.uint32))
        a, b, va, vb = kp(kf1), kp(kf2), bv(fv1), bv(fv2)
        sf = np.ascontiguousarray(scale_factors_1, np.float32)
        E = np.ascontiguousarray(E_12, np.float64).reshape(9)
        ep = np.ascontiguousarray(epipole, np.float64).reshape(3)
        matched = np.full(max(a.n, 1), -2, np.int32)
        num = C.c_uint32(0)
        self._check(self._lib.plp_match_for_triangulation(
            self._h, C.byref(a), C.byref(b), C.byref(va), C.byref(vb), E.ctypes.data_as(_P), ep.ctypes.data_as(_P),
            sf.ctypes.data_as(_P), C.c_int(len(sf)), C.c_int(1 if check_orientation else 0), matched.ctypes.data_as(_P),
            C.byref(num)))
        return matched[:a.n].copy(), int(num.value)

    @staticmethod
    def _frame_lines(k, f):
        n = len(f["sx"])
        return FrameLines(n, k.arr(f["sx"], np.float32), k.arr(f["sy"], np.float32), k.arr(f["ex"], np.float32),
                          k.arr(f["ey"], np.float32), k.arr(f["octave"], np.int32),
                          k.arr(f.get("ratio_level"), np.int32), k.arr(f.get("x_right_sp"), np.float32),
                          k.arr(f.get("x_right_ep"), np.float32), k.arr(f["desc"], np.uint8),
                          k.arr(f.get("claimed"), np.uint8))

    def match_frame_and_landmarks_line(self, scale_factors_lsd, frm, queries, margin, lowe_ratio=0.6):
        k = _Keep()
        fl = self._frame_lines(k, frm)
        m = len(queries["sp_x"])
        q = LineQueries(m, k.arr(queries["sp_x"], np.float32), k.arr(queries["sp_y"], np.float32),
                        k.arr(queries["ep_x"], np.float32), k.arr(queries["ep_y"], np.float32),
                        k.arr(queries["scale_level"], np.int32), k.arr(queries["desc"], np.uint8),
                        k.arr(queries.get("valid"), np.uint8))
        sf = np.ascontiguousarray(scale_factors_lsd, np.float32)
        best = np.full(m, -2, np.int32)
        num = C.c_uint32(0)
        self._check(self._lib.plp_match_frame_and_landmarks_line(
            self._h, C.byref(fl), sf.ctypes.data_as(_P), C.c_int(len(sf)), C.byref(q), C.c_float(margin),
            C.c_float(lowe_ratio), best.ctypes.data_as(_P), C.byref(num)))
        return best, int(num.value)

    def match_current_and_last_frames_line(self, scale_factors_lsd, cam, curr, pose_cw_curr, pose_cw_last, last,
                                           margin):
        k = _Keep()
        fl = self._frame_lines(k, curr)
        n_last = len(last["octave"])
        ll = LastFrameLines(n_last, k.arr(last["pos_w"], np.float64), k.arr(last["octave"], np.int32),
                            k.arr(last["desc"], np.uint8), k.arr(last.get("valid"), np.uint8))
        sf = np.ascontiguousarray(scale_factors_lsd, np.float32)
        Tc = np.ascontiguousarray(pose_cw_curr, np.float64).reshape(4, 4)
        Tl = np.ascontiguousarray(pose_cw_last, np.float64).reshape(4, 4)
        matched = np.full(fl.n, -2, np.int32)
        num = C.c_uint32(0)
        self._check(self._lib.plp_match_current_and_last_frames_line(
            self._h, C.byref(fl), sf.ctypes.data_as(_P), C.c_int(len(sf)), C.byref(cam), Tc.ctypes.data_as(_P),
            Tl.ctypes.data_as(_P), C.byref(ll), C.c_float(margin), matched.ctypes.data_as(_P), C.byref(num)))
        return matched, int(num.value)

    # ------------------------------------------------------------------ optimize::pose_optimizer
    def pose_optimize(self, cam, T_cw, pts, lines=None, num_trials=4, num_each_iter=10):
        """pose_optimizer::optimize / pose_optimizer_extended_line::optimize for one frame."""
        r = self.pose_optimize_batch(cam, [T_cw], [pts], None if lines is None else [lines], num_trials, num_each_iter)
        return r[0][0], r[1][0], (None if lines is None else r[2][0]), int(r[3][0])

    def pose_optimize_batch(self, cam, T_cws, pts_list, lines_list=None, num_trials=4, num_each_iter=10):
        B = len(pts_list)
        T_in = np.ascontiguousarray(np.stack([np.asarray(t, np.float64).reshape(4, 4) for t in T_cws]))
        pts = np.ascontiguousarray(np.concatenate([np.asarray(p, PT_OBS_DTYPE) for p in pts_list]) if B else
                                   np.zeros(0, PT_OBS_DTYPE))
        po = np.zeros(B + 1, np.int32)
        po[1:] = np.cumsum([len(p) for p in pts_list])
        has_lines = lines_list is not None and sum(len(l) for l in lines_list) > 0
        if has_lines:
            lines = np.ascontiguousarray(np.concatenate([np.asarray(l, LINE_OBS_DTYPE) for l in lines_list]))
            lo = np.zeros(B + 1, np.int32)
            lo[1:] = np.cumsum([len(l) for l in lines_list])
        T_out = np.zeros((B, 4, 4), np.float64)
        pout = np.zeros(max(len(pts), 1), np.uint8)
        lout = np.zeros(max(len(lines) if has_lines else 0, 1), np.uint8)
        ninl = np.zeros(B, np.int32)
        cfg = PoseOptCfg(num_trials, num_each_iter)
        self._check(self._lib.plp_pose_optimize_batch(
            self._h, C.byref(cam), C.c_int(B), T_in.ctypes.data_as(_P), pts.ctypes.data_as(_P), po.ctypes.data_as(_P),
            lines.ctypes.data_as(_P) if has_lines else None, lo.ctypes.data_as(_P) if has_lines else None,
            C.byref(cfg), T_out.ctypes.data_as(_P), pout.ctypes.data_as(_P), lout.ctypes.data_as(_P),
            ninl.ctypes.data_as(_P)))
        p_split = [pout[po[b]:po[b + 1]].copy() for b in range(B)]
        l_split = [lout[lo[b]:lo[b + 1]].copy() for b in range(B)] if has_lines else None
        return T_out, p_split, l_split, ninl

    # ------------------------------------------------------------------ match::robust
    def brute_force_match(self, frm_desc, frm_angle, kf_desc, kf_angle, kf_valid=None, lowe_ratio=0.8,
                          check_orientation=False):
        k = _Keep()
        fd = np.ascontiguousarray(frm_desc, np.uint8).reshape(-1, 32)
        kd = np.ascontiguousarray(kf_desc, np.uint8).reshape(-1, 32)
        matched = np.full(fd.shape[0], -2, np.int32)
        num = C.c_uint32(0)
        self._check(self._lib.plp_match_brute_force(
            self._h, k.arr(fd, np.uint8), k.arr(frm_angle, np.float32), C.c_int(fd.shape[0]), k.arr(kd, np.uint8),
            k.arr(kf_angle, np.float32), k.arr(kf_valid, np.uint8), C.c_int(kd.shape[0]), C.c_float(lowe_ratio),
            C.c_int(1 if check_orientation else 0), matched.ctypes.data_as(_P), C.byref(num)))
        return matched, int(num.value)


class BowVocabulary:
    """data::bow_vocabulary (DBoW2 tree) resident on the device; transform() = the per-row part of frame::compute_bow."""

    def __init__(self, ctx: Context, path=None, k=None, L=None, parent=None, desc=None, weight=None, is_leaf=None):
        self._ctx = ctx
        self._lib = ctx._lib
        self._h = None
        h = C.c_void_p()
        if path is not None:
            ctx._check(self._lib.plp_bow_vocab_load(ctx.handle, str(path).encode(), C.byref(h)))
        else:
            kk = _Keep()
            parent = np.ascontiguousarray(parent, np.int32)
            ctx._check(self._lib.plp_bow_vocab_create(
                ctx.handle, C.c_int(k), C.c_int(L), C.c_int(len(parent) + 1), kk.arr(parent, np.int32),
                kk.arr(np.ascontiguousarray(desc, np.uint8).reshape(-1, 32), np.uint8), kk.arr(weight, np.float32),
                kk.arr(is_leaf, np.uint8), C.byref(h)))
        self._h = h

    def close(self):
        if self._h is not None:
            self._lib.plp_bow_vocab_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def handle(self):
        return self._h

    def info(self):
        v = [C.c_int32() for _ in range(4)]
        self._ctx._check(self._lib.plp_bow_vocab_info(self._h, *[C.byref(x) for x in v]))
        return dict(k=v[0].value, L=v[1].value, num_nodes=v[2].value, num_words=v[3].value)

    def transform(self, desc, levelsup=4):
        """-> (word_id, node_id, weight) per descriptor row."""
        d = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32)
        n = d.shape[0]
        word = np.full(max(n, 1), -2, np.int32)
        node = np.full(max(n, 1), -2, np.int32)
        w = np.full(max(n, 1), -1, np.float32)
        self._ctx._check(self._lib.plp_bow_transform(self._h, d.ctypes.data_as(_P), C.c_int(n), C.c_int(levelsup),
                                                     word.ctypes.data_as(_P), node.ctypes.data_as(_P),
                                                     w.ctypes.data_as(_P)))
        return word[:n].copy(), node[:n].copy(), w[:n].copy()


class StereoRectifierParams(C.Structure):
    _fields_ = [("model", C.c_int32), ("K_left", C.c_double * 9), ("D_left", C.c_double * 5), ("R_left", C.c_double * 9),
                ("K_right", C.c_double * 9), ("D_right", C.c_double * 5), ("R_right", C.c_double * 9),
                ("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double)]


class StereoRectifier:
    """util::stereo_rectifier backed by plp_stereo_rectifier: model 0 perspective (D = k1, k2, p1, p2, k3) or 1 fisheye
    (D = k1..k4); K and R row-major 3x3 as the StereoRectifier.* config keys list them; (fx, fy, cx, cy) the rectified
    camera."""

    def __init__(self, ctx: Context, rows: int, cols: int, model, K_l, D_l, R_l, K_r, D_r, R_r, fx, fy, cx, cy):
        self._ctx = ctx
        self._lib = ctx._lib
        self.rows, self.cols = int(rows), int(cols)

        def arr(a, n):
            v = np.asarray(a, np.float64).ravel()
            if len(v) > n or (n == 9 and len(v) != 9):
                raise PlpError(f"expected {n} values, got {len(v)}")
            return (C.c_double * n)(*(list(v) + [0.0] * (n - len(v))))

        self.params = StereoRectifierParams(int(model), arr(K_l, 9), arr(D_l, 5), arr(R_l, 9), arr(K_r, 9), arr(D_r, 5),
                                            arr(R_r, 9), fx, fy, cx, cy)
        h = C.c_void_p()
        self._h = None
        ctx._check(self._lib.plp_stereo_rectifier_create(ctx.handle, C.byref(self.params), C.c_int(rows), C.c_int(cols),
                                                         C.byref(h)))
        self._h = h

    def close(self):
        if self._h is not None:
            self._lib.plp_stereo_rectifier_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def handle(self):
        return self._h

    def rectify(self, left, right):
        """stereo_rectifier::rectify of two host images -> (left_rect, right_rect)."""
        left = np.ascontiguousarray(left, np.uint8)
        right = np.ascontiguousarray(right, np.uint8)
        if left.shape != (self.rows, self.cols) or right.shape != left.shape:
            raise PlpError(f"images must be {self.rows} x {self.cols}")
        out_l = np.zeros_like(left)
        out_r = np.zeros_like(right)
        self._ctx._check(self._lib.plp_stereo_rectify(self._ctx.handle, self._h, left.ctypes.data_as(_P),
                                                      right.ctypes.data_as(_P), C.c_size_t(left.strides[0]),
                                                      out_l.ctypes.data_as(_P), out_r.ctypes.data_as(_P),
                                                      C.c_size_t(out_l.strides[0])))
        return out_l, out_r

    def rectify_dev(self, side, d_in, batch, in_step, d_out, out_step, ctx: Context = None):
        """Device-resident batch of one side (device pointers), enqueued on ctx's stream (default: the creating one)."""
        ctx = ctx or self._ctx
        ctx._check(self._lib.plp_stereo_rectify_batch_dev(ctx.handle, self._h, C.c_int(side), d_in, C.c_int(batch),
                                                          C.c_size_t(in_step), d_out, C.c_size_t(out_step)))

    def maps(self, side):
        """The float maps (map_x, map_y) of one side, rows x cols each."""
        mx = np.zeros((self.rows, self.cols), np.float32)
        my = np.zeros_like(mx)
        self._ctx._check(self._lib.plp_stereo_rectifier_maps(self._h, C.c_int(side), mx.ctypes.data_as(_P),
                                                             my.ctypes.data_as(_P)))
        return mx, my


def fold_bow(word_id, node_id, weight):
    """The adapter's fold of transform() rows into DBoW2's two maps (TemplatedVocabulary::transform(features, v, fv,
    levelsup) with TF_IDF weighting and L1 scoring): rows with weight > 0 only; bow_vec[word] += weight in row order,
    then L1-normalised over ascending word ids; bow_feat_vec[node].push_back(row).  Returns (words, values, fv) with
    fv = (node_ids, offsets, indices) flattened in map order."""
    word_id, node_id = np.asarray(word_id), np.asarray(node_id)
    weight = np.asarray(weight, np.float32)
    keep = np.nonzero(weight > 0)[0]
    vec, feat = {}, {}
    for i in keep:
        vec[int(word_id[i])] = vec.get(int(word_id[i]), 0.0) + float(weight[i])
        feat.setdefault(int(node_id[i]), []).append(int(i))
    words = np.array(sorted(vec), np.int64)
    vals = np.array([vec[int(w)] for w in words], np.float64)
    norm = 0.0
    for v in vals:
        norm += abs(v)
    if norm > 0.0:
        vals = vals / norm
    nodes = sorted(feat)
    offsets = np.zeros(len(nodes) + 1, np.int32)
    for i, nd in enumerate(nodes):
        offsets[i + 1] = offsets[i] + len(feat[nd])
    indices = np.array([i for nd in nodes for i in feat[nd]], np.uint32)
    return words, vals, (np.array(nodes, np.uint32), offsets, indices)


def _csr(lists, dtype):
    """Ragged lists -> (offsets int32[n + 1], flat dtype[max(total, 1)])."""
    lists = [np.asarray(v, dtype).ravel() for v in lists]
    offsets = np.zeros(len(lists) + 1, np.int32)
    for i, v in enumerate(lists):
        offsets[i + 1] = offsets[i] + len(v)
    flat = np.zeros(max(int(offsets[-1]), 1), dtype)
    if offsets[-1]:
        flat[:offsets[-1]] = np.concatenate(lists)
    return offsets, flat


class BowDatabase:
    """data::bow_database backed by plp_bow_db: keyframes are keyframe-table indices, vectors are (words, values) pairs
    (bow_vec_: ascending word ids, double values, as fold_bow returns them).  Candidate lists come back ascending."""

    def __init__(self, ctx: Context, vocab: BowVocabulary, max_keyframes: int, max_words_per_keyframe: int):
        self._ctx = ctx
        self._lib = ctx._lib
        self.max_keyframes = int(max_keyframes)
        self._h = None
        h = C.c_void_p()
        ctx._check(self._lib.plp_bow_db_create(ctx.handle, vocab.handle, C.c_int(max_keyframes),
                                               C.c_int(max_words_per_keyframe), C.byref(h)))
        self._h = h

    def close(self):
        if self._h is not None:
            self._lib.plp_bow_db_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def handle(self):
        return self._h

    def add(self, kf_index, vectors):
        """add_keyframe of keyframe kf_index[i] with bow_vec_ vectors[i] = (words, values)."""
        kf = np.ascontiguousarray(kf_index, np.int32).ravel()
        off, words = _csr([v[0] for v in vectors], np.int32)
        _, vals = _csr([v[1] for v in vectors], np.float64)
        self._ctx._check(self._lib.plp_bow_db_add_keyframes(self._h, C.c_int(len(kf)), kf.ctypes.data_as(_P),
                                                            off.ctypes.data_as(_P), words.ctypes.data_as(_P),
                                                            vals.ctypes.data_as(_P)))

    def erase(self, kf_index):
        kf = np.ascontiguousarray(kf_index, np.int32).ravel()
        self._ctx._check(self._lib.plp_bow_db_erase_keyframes(self._h, C.c_int(len(kf)), kf.ctypes.data_as(_P)))

    def score_pairs(self, kf_a, kf_b) -> np.ndarray:
        a = np.ascontiguousarray(kf_a, np.int32).ravel()
        b = np.ascontiguousarray(kf_b, np.int32).ravel()
        out = np.zeros(max(len(a), 1), np.float32)
        self._ctx._check(self._lib.plp_bow_db_score_pairs(self._h, C.c_int(len(a)), a.ctypes.data_as(_P),
                                                          b.ctypes.data_as(_P), out.ctypes.data_as(_P)))
        return out[:len(a)].copy()

    @staticmethod
    def _graph(cov):
        """cov[k] = keyframe k's get_top_n_covisibilities(10), for every keyframe index below len(cov)."""
        off, flat = _csr(cov, np.int32)
        return len(cov), off, flat

    def _results(self, n, max_candidates, cand, num, status):
        lists = [cand[q, :num[q]].copy() for q in range(n)]
        return lists, status[:n].copy()

    def relocalization_candidates(self, vectors, cov, max_candidates=256):
        """acquire_relocalization_candidates of each query vector -> (candidate lists, status per query)."""
        n = len(vectors)
        off, words = _csr([v[0] for v in vectors], np.int32)
        _, vals = _csr([v[1] for v in vectors], np.float64)
        nk, coff, ckf = self._graph(cov)
        cand = np.zeros((max(n, 1), max(max_candidates, 1)), np.int32)
        num = np.zeros(max(n, 1), np.int32)
        status = np.full(max(n, 1), -1, np.int32)
        self._ctx._check(self._lib.plp_bow_db_relocalization_candidates(
            self._h, C.c_int(n), off.ctypes.data_as(_P), words.ctypes.data_as(_P), vals.ctypes.data_as(_P),
            C.c_int(nk), coff.ctypes.data_as(_P), ckf.ctypes.data_as(_P), C.c_int(max_candidates),
            cand.ctypes.data_as(_P), num.ctypes.data_as(_P), status.ctypes.data_as(_P)))
        return self._results(n, max_candidates, cand, num, status)

    def loop_candidates(self, query_kf, min_score, connected, cov, max_candidates=256):
        """acquire_loop_candidates(query_kf[q], min_score[q]) with connected[q] = its get_connected_keyframes()."""
        qk = np.ascontiguousarray(query_kf, np.int32).ravel()
        n = len(qk)
        ms = np.ascontiguousarray(np.broadcast_to(np.asarray(min_score, np.float32), (n,)))
        conn_off, conn = _csr(connected, np.int32)
        nk, coff, ckf = self._graph(cov)
        cand = np.zeros((max(n, 1), max(max_candidates, 1)), np.int32)
        num = np.zeros(max(n, 1), np.int32)
        status = np.full(max(n, 1), -1, np.int32)
        self._ctx._check(self._lib.plp_bow_db_loop_candidates(
            self._h, C.c_int(n), qk.ctypes.data_as(_P), ms.ctypes.data_as(_P), conn_off.ctypes.data_as(_P),
            conn.ctypes.data_as(_P), C.c_int(nk), coff.ctypes.data_as(_P), ckf.ctypes.data_as(_P),
            C.c_int(max_candidates), cand.ctypes.data_as(_P), num.ctypes.data_as(_P), status.ctypes.data_as(_P)))
        return self._results(n, max_candidates, cand, num, status)


class OrbExtractor:
    """feature::orb_extractor (feature/orb_extractor.h:46-98) backed by plp_orb."""

    def __init__(self, ctx: Context, rows: int, cols: int, max_num_keypts=1000, scale_factor=1.2, num_levels=8,
                 ini_fast_thr=20, min_fast_thr=7, max_batch=1):
        self._ctx = ctx
        self._lib = ctx._lib
        self.rows, self.cols, self.max_batch = rows, cols, max_batch
        self.params = OrbParams(max_num_keypts, scale_factor, num_levels, ini_fast_thr, min_fast_thr)
        h = C.c_void_p()
        self._h = None
        ctx._check(self._lib.plp_orb_create(ctx.handle, C.byref(self.params), C.c_int(rows), C.c_int(cols),
                                            C.c_int(max_batch), C.byref(h)))
        self._h = h
        self.capacity = int(self._lib.plp_orb_capacity(self._h))
        L = num_levels
        self.scale_factors, self.inv_scale_factors = np.zeros(L, np.float32), np.zeros(L, np.float32)
        self.level_sigma_sq, self.inv_level_sigma_sq = np.zeros(L, np.float32), np.zeros(L, np.float32)
        self.num_keypts_per_level = np.zeros(L, np.uint32)
        ctx._check(self._lib.plp_orb_get_tables(self._h, self.scale_factors.ctypes.data_as(_P),
                                                self.inv_scale_factors.ctypes.data_as(_P),
                                                self.level_sigma_sq.ctypes.data_as(_P),
                                                self.inv_level_sigma_sq.ctypes.data_as(_P),
                                                self.num_keypts_per_level.ctypes.data_as(_P)))

    def close(self):
        if self._h is not None:
            self._lib.plp_orb_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def handle(self):
        return self._h

    def extract(self, img, mask=None):
        """orb_extractor::extract -> (keypoints[KP_DTYPE], descriptors[n,32])."""
        if img is None or img.size == 0:
            n = C.c_int(-1)
            self._ctx._check(self._lib.plp_orb_extract(self._h, None, 0, 0, C.c_size_t(0), None, C.c_size_t(0), None,
                                                       None, C.byref(n)))
            return np.zeros(0, KP_DTYPE), np.zeros((0, 32), np.uint8)
        img = np.ascontiguousarray(img, np.uint8)
        kps = np.zeros(self.capacity, KP_DTYPE)
        desc = np.zeros((self.capacity, 32), np.uint8)
        n = C.c_int(0)
        mk = None if mask is None else np.ascontiguousarray(mask, np.uint8)
        self._ctx._check(self._lib.plp_orb_extract(
            self._h, img.ctypes.data_as(_P), C.c_int(img.shape[0]), C.c_int(img.shape[1]), C.c_size_t(img.strides[0]),
            None if mk is None else mk.ctypes.data_as(_P), C.c_size_t(0 if mk is None else mk.strides[0]),
            kps.ctypes.data_as(_P), desc.ctypes.data_as(_P), C.byref(n)))
        return kps[:n.value].copy(), desc[:n.value].copy()

    def extract_batch(self, imgs):
        imgs = np.ascontiguousarray(imgs, np.uint8)
        B = imgs.shape[0]
        kps = np.zeros((B, self.capacity), KP_DTYPE)
        desc = np.zeros((B, self.capacity, 32), np.uint8)
        n = np.zeros(B, np.int32)
        self._ctx._check(self._lib.plp_orb_extract_batch(self._h, imgs.ctypes.data_as(_P), C.c_int(B),
                                                         C.c_size_t(imgs.strides[1]), kps.ctypes.data_as(_P),
                                                         desc.ctypes.data_as(_P), n.ctypes.data_as(_P)))
        return [(kps[b, :n[b]].copy(), desc[b, :n[b]].copy()) for b in range(B)]

    def stereo_compute(self, right: "OrbExtractor", kp_left, desc_left, kp_right, desc_right, focal_x_baseline,
                       true_baseline):
        """match::stereo::compute with this extractor as the left one -> (stereo_x_right, depths, best_right_idx)."""
        kl = np.ascontiguousarray(kp_left, KP_DTYPE)
        kr = np.ascontiguousarray(kp_right, KP_DTYPE)
        dl = np.ascontiguousarray(desc_left, np.uint8)
        dr = np.ascontiguousarray(desc_right, np.uint8)
        xr = np.zeros(max(len(kl), 1), np.float32)
        dp = np.zeros(max(len(kl), 1), np.float32)
        br = np.zeros(max(len(kl), 1), np.int32)
        self._ctx._check(self._lib.plp_stereo_compute(
            self._ctx.handle, self._h, right._h, kl.ctypes.data_as(_P), dl.ctypes.data_as(_P), C.c_int(len(kl)),
            kr.ctypes.data_as(_P), dr.ctypes.data_as(_P), C.c_int(len(kr)), C.c_float(focal_x_baseline),
            C.c_float(true_baseline), xr.ctypes.data_as(_P), dp.ctypes.data_as(_P), br.ctypes.data_as(_P)))
        return xr[:len(kl)].copy(), dp[:len(kl)].copy(), br[:len(kl)].copy()

    def pyramid_level(self, b: int, level: int) -> np.ndarray:
        """orb_extractor::image_pyramid_[level] of frame b of the last extraction (downloaded)."""
        v = ImageView()
        self._ctx._check(self._lib.plp_orb_get_pyramid(self._h, C.c_int(b), C.c_int(level), C.byref(v)))
        buf = np.zeros((v.rows, v.step), np.uint8)
        self._ctx._check(self._lib.plp_dev_download(self._ctx.handle, buf.ctypes.data_as(_P), C.c_void_p(v.data),
                                                    C.c_size_t(v.rows * v.step)))
        return buf[:, :v.cols].copy()

    def debug_candidates(self, b: int, level: int) -> np.ndarray:
        cap = 70000
        out = np.zeros(cap, KP_DTYPE)
        n = C.c_int(0)
        self._ctx._check(self._lib.plp_orb_debug_candidates(self._h, C.c_int(b), C.c_int(level),
                                                            out.ctypes.data_as(_P), C.c_int(cap), C.byref(n)))
        return out[:min(n.value, cap)].copy()

    def debug_blurred(self, b: int, level: int) -> np.ndarray:
        """The blurred level the descriptors of frame b of the last extraction sample (downloaded)."""
        v = ImageView()
        self._ctx._check(self._lib.plp_orb_get_pyramid(self._h, C.c_int(b), C.c_int(level), C.byref(v)))
        out = np.zeros((v.rows, v.cols), np.uint8)
        self._ctx._check(self._lib.plp_orb_debug_blurred(self._h, C.c_int(b), C.c_int(level), out.ctypes.data_as(_P)))
        return out


# binary layout of plp_keyline / cv::line_descriptor::KeyLine (descriptor_custom.hpp:105-199)
KEYLINE_DTYPE = np.dtype([("angle", "<f4"), ("class_id", "<i4"), ("octave", "<i4"), ("pt_x", "<f4"), ("pt_y", "<f4"),
                          ("response", "<f4"), ("size", "<f4"), ("start_x", "<f4"), ("start_y", "<f4"),
                          ("end_x", "<f4"), ("end_y", "<f4"), ("s_oct_x", "<f4"), ("s_oct_y", "<f4"),
                          ("e_oct_x", "<f4"), ("e_oct_y", "<f4"), ("line_length", "<f4"), ("num_pixels", "<i4")])


class LineFeatureTracker:
    """feature::LineFeatureTracker (feature/line_extractor.h:62-108) backed by plp_line."""

    def __init__(self, ctx: Context, rows: int, cols: int, max_batch=1):
        self._ctx = ctx
        self._lib = ctx._lib
        self.rows, self.cols, self.max_batch = rows, cols, max_batch
        h = C.c_void_p()
        self._h = None
        ctx._check(self._lib.plp_line_create(ctx.handle, C.c_int(rows), C.c_int(cols), C.c_int(max_batch), C.byref(h)))
        self._h = h
        self.capacity = int(self._lib.plp_line_capacity(self._h))

    def close(self):
        if self._h is not None:
            self._lib.plp_line_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def handle(self):
        return self._h

    def extract_LSD_LBD(self, img):
        """LineFeatureTracker::extract_LSD_LBD -> (keylines[KEYLINE_DTYPE], lbd[n,32], line functions[n,3])."""
        img = np.asarray(img, np.uint8)
        if img.ndim != 2 or img.strides[1] != 1:
            img = np.ascontiguousarray(img)
        kl = np.zeros(self.capacity, KEYLINE_DTYPE)
        lbd = np.zeros((self.capacity, 32), np.uint8)
        fn = np.zeros((self.capacity, 3), np.float64)
        n = C.c_int(0)
        self._ctx._check(self._lib.plp_line_extract(
            self._h, img.ctypes.data_as(_P), C.c_int(img.shape[0]), C.c_int(img.shape[1]), C.c_size_t(img.strides[0]),
            kl.ctypes.data_as(_P), lbd.ctypes.data_as(_P), fn.ctypes.data_as(_P), C.byref(n)))
        return kl[:n.value].copy(), lbd[:n.value].copy(), fn[:n.value].copy()

    def extract_batch(self, imgs):
        imgs = np.ascontiguousarray(imgs, np.uint8)
        B = imgs.shape[0]
        kl = np.zeros((B, self.capacity), KEYLINE_DTYPE)
        lbd = np.zeros((B, self.capacity, 32), np.uint8)
        fn = np.zeros((B, self.capacity, 3), np.float64)
        n = np.zeros(B, np.int32)
        self._ctx._check(self._lib.plp_line_extract_batch(
            self._h, imgs.ctypes.data_as(_P), C.c_int(B), C.c_size_t(imgs.strides[1]), kl.ctypes.data_as(_P),
            lbd.ctypes.data_as(_P), fn.ctypes.data_as(_P), n.ctypes.data_as(_P)))
        return [(kl[b, :n[b]].copy(), lbd[b, :n[b]].copy(), fn[b, :n[b]].copy()) for b in range(B)]

    def force_global_image(self, on: bool):
        self._ctx._check(self._lib.plp_line_debug_force_global_image(self._h, C.c_int(1 if on else 0)))

    def grow_variant(self, variant: int):
        """0 automatic, 1 one warp per frame, 2 speculative multi-warp region growing (same result, bit for bit)."""
        self._ctx._check(self._lib.plp_line_debug_grow_variant(self._h, C.c_int(variant)))

    def ooo_fallbacks(self) -> int:
        """Host calls that were re-run with the round protocol because the out-of-order region growing gave up (expected 0)."""
        return int(self._lib.plp_line_debug_ooo_fallbacks(self._h))

    def grow_stats(self, b: int = 0, ooo: bool = False):
        """{rounds, seeds run, seeds redone after a conflict, cycle counters} of frame b in the last multi-warp run; with ooo:
        the counters of the out-of-order variant."""
        out = (C.c_ulonglong * 8)()
        self._ctx._check(self._lib.plp_line_debug_grow_stats(self._h, C.c_int(b), out))
        if ooo:
            return dict(tickets=int(out[0]), void=int(out[1]), deferred=int(out[2]), parked=int(out[3]), held=int(out[4]),
                        executed_at_head=int(out[5]), conflicts=int(out[6]), aborted=int(out[7]))
        return dict(rounds=int(out[0]), seeds_run=int(out[1]), seeds_redone=int(out[2]), cyc_scan=int(out[3]),
                    cyc_own=int(out[4]), cyc_wait=int(out[5]), cyc_commit=int(out[6]))

    def debug_segments(self, b: int) -> np.ndarray:
        cap = 20000
        out = np.zeros((cap, 4), np.float32)
        n = C.c_int(0)
        self._ctx._check(self._lib.plp_line_debug_segments(self._h, C.c_int(b), out.ctypes.data_as(_P), C.c_int(cap),
                                                           C.byref(n)))
        return out[:n.value].copy()

    def debug_scaled(self, b: int) -> np.ndarray:
        out = np.zeros((int(round(self.rows * 0.5)), int(round(self.cols * 0.5))), np.uint8)
        self._ctx._check(self._lib.plp_line_debug_scaled(self._h, C.c_int(b), out.ctypes.data_as(_P)))
        return out

    def debug_lbd_float(self, b: int, n: int) -> np.ndarray:
        out = np.zeros((max(n, 1), 72), np.float32)
        self._ctx._check(self._lib.plp_line_debug_lbd_float(self._h, C.c_int(b), out.ctypes.data_as(_P), C.c_int(n)))
        return out[:n].copy()
