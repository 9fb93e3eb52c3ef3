"""Camera models of the reference's monocular example configs, synthetic strongly distorted ones, the ctypes wrappers of
the oracle's camera functions (oracle/camera.h), and cv2 restatements of camera::{perspective,fisheye}::
undistort_keypoints / compute_image_bounds (the cv2 side of the oracle pins)."""
from __future__ import annotations

import ctypes as C

import numpy as np

_P = C.c_void_p

PERSPECTIVE, FISHEYE = 0, 1

# name: (model, cols, rows, (fx, fy, cx, cy), coefficients as the YAML gives them)
CONFIGS = {
    # example/euroc/EuRoC_mono.yaml
    "euroc_mono": (PERSPECTIVE, 752, 480, (458.654, 457.296, 367.215, 248.375),
                   (-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05, 0.0)),
    # example/tum_rgbd/TUM_RGBD_mono_1.yaml
    "tum_mono_1": (PERSPECTIVE, 640, 480, (517.306408, 516.469215, 318.643040, 255.313989),
                   (0.262383, -0.953104, -0.005358, 0.002628, 1.163314)),
    # example/tum_rgbd/TUM_RGBD_mono_2.yaml
    "tum_mono_2": (PERSPECTIVE, 640, 480, (520.908620, 521.007327, 325.141442, 249.701764),
                   (0.231222, -0.784899, -0.003257, -0.000105, 0.917205)),
    # example/tum_vi/TUM_VI_mono.yaml
    "tumvi_fisheye": (FISHEYE, 512, 512, (190.97847715128717, 190.9733070521226, 254.93170605935475, 256.8974428996504),
                      (0.0034823894022493434, 0.0007150348452162257, -0.0020532361418706202, 0.00020293673591811182)),
}

# synthetic strong distortions that reach the edge branches
SYNTHETIC = {
    # 1 + k1 r^2 < 0 towards the corners: OpenCV gives up on those points (icdist < 0)
    "strong_barrel": (PERSPECTIVE, 640, 480, (300.0, 300.0, 320.0, 240.0), (-0.6, 0.05, 0.001, -0.002, 0.0)),
    # Newton on theta that fails to converge or changes sign -> (-1e6, -1e6)
    "fisheye_unstable": (FISHEYE, 640, 480, (260.0, 260.0, 320.0, 240.0), (-0.4, 0.3, -0.2, 0.05)),
    # theta_d > pi/2 at the corners: the clamp and the wide-FOV branch of compute_image_bounds
    "fisheye_wide": (FISHEYE, 640, 480, (110.0, 110.0, 318.5, 241.25), (0.02, -0.01, 0.004, -0.001)),
}

ALL = {**CONFIGS, **SYNTHETIC}


def coeffs5(D):
    D = np.zeros(5) if D is None else np.asarray(D, np.float64).ravel()
    return np.concatenate([D, np.zeros(5 - len(D))])


# ---- oracle/camera.h (K = config fx, fy, cx, cy; D = config coefficients); orc is an oracle_api.Oracle
def _kd(K, D):
    return np.ascontiguousarray(K, np.float64).reshape(4), np.ascontiguousarray(coeffs5(D))


def _xy(x, y):
    return np.ascontiguousarray(np.stack([np.asarray(x, np.float32), np.asarray(y, np.float32)], 1))


def undistort_keypoints(orc, model, K, D, x, y):
    """The oracle's undistort_keypoints of the points (x, y) -> (x_undist, y_undist) as float32."""
    xy = _xy(x, y)
    out = np.zeros_like(xy)
    Kd, Dd = _kd(K, D)
    orc.lib.orc_undistort_keypoints(C.c_int(model), Kd.ctypes.data_as(_P), Dd.ctypes.data_as(_P), xy.ctypes.data_as(_P),
                                    C.c_int(len(xy)), out.ctypes.data_as(_P))
    return out[:, 0].copy(), out[:, 1].copy()


def bearings(orc, K, x, y):
    """The oracle's convert_keypoints_to_bearings of undistorted points -> n x 3."""
    xy = _xy(x, y)
    out = np.zeros((len(xy), 3), np.float64)
    Kd = np.ascontiguousarray(K, np.float64)
    orc.lib.orc_bearings(Kd.ctypes.data_as(_P), xy.ctypes.data_as(_P), C.c_int(len(xy)), out.ctypes.data_as(_P))
    return out


def image_bounds(orc, model, K, D, cols, rows):
    """The oracle's compute_image_bounds -> float32 (min_x, max_x, min_y, max_y)."""
    out = np.zeros(4, np.float32)
    Kd, Dd = _kd(K, D)
    orc.lib.orc_image_bounds(C.c_int(model), Kd.ctypes.data_as(_P), Dd.ctypes.data_as(_P), C.c_int(cols), C.c_int(rows),
                             out.ctypes.data_as(_P))
    return out


def cv2_undistort(model, K, D, x, y):
    """The reference's undistort_keypoints through cv2: float32 K / D, P = K, the reference's criteria."""
    import cv2
    fx, fy, cx, cy = K
    Km = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32)
    pts = np.stack([np.asarray(x, np.float32), np.asarray(y, np.float32)], 1).reshape(-1, 1, 2)
    if model == FISHEYE:
        out = cv2.fisheye.undistortPoints(pts, Km, np.asarray(D[:4], np.float32).reshape(4, 1), R=None, P=Km)
    else:
        out = cv2.undistortPointsIter(pts, Km, np.asarray(D[:5], np.float32).reshape(5, 1), None, Km,
                                      (cv2.TERM_CRITERIA_EPS | cv2.TERM_CRITERIA_MAX_ITER, 20, 1e-6))
    out = out.reshape(-1, 2).astype(np.float32)
    return out[:, 0].copy(), out[:, 1].copy()


def cv2_image_bounds(model, K, D, cols, rows):
    """compute_image_bounds (perspective.cc:100-127, fisheye.cc:101-169) with cv2 doing the undistortion."""
    fx, fy, cx, cy = K
    D = coeffs5(D)
    f32 = np.float32
    if not np.any(D[:4 if model == FISHEYE else 5]):
        return np.array([0.0, cols, 0.0, rows], f32)
    if model == FISHEYE:
        pwx, pwy = (0.0 - cx) / fx, (0.0 - cy) / fy
        if np.sqrt(pwx * pwx + pwy * pwy) > np.pi / 2:
            ux, uy = cv2_undistort(model, K, D, [f32(cx), cols, 0.0, f32(cx)], [0.0, f32(cy), f32(cy), rows])
            t = np.tan(float(f32(5.0)) * np.pi / 180.0)
            dx, dy = f32(fx / t), f32(fy / t)
            mnx, mxx = f32(-float(dx) + cx), f32(float(dx) + cx)
            mny, mxy = f32(-float(dy) + cy), f32(float(dy) + cy)
            a, b, c, d = float(ux[2]), float(ux[1]), float(uy[0]), float(uy[3])
            return np.array([mnx if (a < mnx or a > cx) else a, mxx if (b > mxx or b < cx) else b,
                             mny if (c < mny or c > cy) else c, mxy if (d > mxy or d < cy) else d], f32)
    ux, uy = cv2_undistort(model, K, D, [0.0, cols, 0.0, cols], [0.0, 0.0, rows, rows])
    return np.array([min(ux[0], ux[2]), max(ux[1], ux[3]), min(uy[0], uy[1]), max(uy[2], uy[3])], f32)


def bearings_np(K, x, y):
    """convert_keypoints_to_bearings in numpy (the config's double fx_, cx_)."""
    fx, fy, cx, cy = K
    xn = (np.asarray(x, np.float32).astype(np.float64) - cx) / fx
    yn = (np.asarray(y, np.float32).astype(np.float64) - cy) / fy
    l2 = np.sqrt(xn * xn + yn * yn + 1.0)
    return np.stack([xn / l2, yn / l2, 1.0 / l2], 1)


def test_points(cols, rows, seed=0, n=20000):
    """Random points in and around the image, the corners, the principal-point neighbourhood and points outside."""
    rng = np.random.default_rng(seed)
    xs = [rng.uniform(0, cols, n), [0, cols, 0, cols, cols / 2, cols - 1, 0.5],
          rng.uniform(-0.5 * cols, 1.5 * cols, n // 10)]
    ys = [rng.uniform(0, rows, n), [0, 0, rows, rows, rows / 2, rows - 1, 0.5],
          rng.uniform(-0.5 * rows, 1.5 * rows, n // 10)]
    return (np.concatenate(xs).astype(np.float32), np.concatenate(ys).astype(np.float32))


def orb_level_coordinates(cols, rows, scale_factors):
    """Every coordinate value the ORB extractor can emit at this size: level-grid positions times the level's float
    scale factor (the keypoints of level l are scaled by scale_factors_[l] in float)."""
    xs, ys = [], []
    for sf in np.asarray(scale_factors, np.float32):
        xs.append(np.arange(int(np.ceil(cols / float(sf))) + 1, dtype=np.float32) * sf)
        ys.append(np.arange(int(np.ceil(rows / float(sf))) + 1, dtype=np.float32) * sf)
    return np.unique(np.concatenate(xs)), np.unique(np.concatenate(ys))
