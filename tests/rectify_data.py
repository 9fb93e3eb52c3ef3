"""Stereo rectification test data: the StereoRectifier configs the reference ships plus synthetic ones, the CPU oracle of
rectification (oracle/rectify_oracle.cc, part of the oracle library) and its cv2 counterparts."""
from __future__ import annotations

import ctypes as C

import numpy as np

import oracle_api

_P = C.c_void_p

PERSPECTIVE, FISHEYE = 0, 1


def _rot(rx, ry, rz):
    """A rotation matrix from small Euler angles (radians), row-major 3x3."""
    cx, sx, cy, sy, cz, sz = np.cos(rx), np.sin(rx), np.cos(ry), np.sin(ry), np.cos(rz), np.sin(rz)
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def _k(fx, fy, cx, cy):
    return np.array([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]])


# name: dict(model, cols, rows, K_l, D_l, R_l, K_r, D_r, R_r, rect = (fx, fy, cx, cy), bf)
CASES = {
    # example/euroc/EuRoC_stereo.yaml
    "euroc": dict(
        model=PERSPECTIVE, cols=752, rows=480,
        K_l=np.array([458.654, 0.0, 367.215, 0.0, 457.296, 248.375, 0.0, 0.0, 1.0]).reshape(3, 3),
        D_l=np.array([-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05, 0.0]),
        R_l=np.array([0.999966347530033, -0.001422739138722922, 0.008079580483432283, 0.001365741834644127,
                      0.9999741760894847, 0.007055629199258132, -0.008089410156878961, -0.007044357138835809,
                      0.9999424675829176]).reshape(3, 3),
        K_r=np.array([457.587, 0.0, 379.999, 0.0, 456.134, 255.238, 0.0, 0.0, 1]).reshape(3, 3),
        D_r=np.array([-0.28368365, 0.07451284, -0.00010473, -3.555907e-05, 0.0]),
        R_r=np.array([0.9999633526194376, -0.003625811871560086, 0.007755443660172947, 0.003680398547259526,
                      0.9999684752771629, -0.007035845251224894, -0.007729688520722713, 0.007064130529506649,
                      0.999945173484644]).reshape(3, 3),
        rect=(435.2046959714599, 435.2046959714599, 367.4517211914062, 252.2008514404297), bf=47.90639384423901),
    # example/tum_vi/TUM_VI_stereo.yaml
    "tumvi": dict(
        model=FISHEYE, cols=512, rows=512,
        K_l=np.array([190.97847715128717, 0.0, 254.93170605935475, 0.0, 190.9733070521226, 256.8974428996504, 0.0, 0.0,
                      1.0]).reshape(3, 3),
        D_l=np.array([0.0034823894022493434, 0.0007150348452162257, -0.0020532361418706202, 0.00020293673591811182]),
        R_l=np.array([0.9997641946925044, 0.01925271884177015, 0.010044293307535757, -0.01901185247371587,
                      0.9995418997803748, -0.02354867403818772, -0.010493068014919314, 0.02335216051329943,
                      0.99967223234568]).reshape(3, 3),
        K_r=np.array([190.44236969414825, 0.0, 252.59949716835982, 0.0, 190.4344384721956, 254.91723064636983, 0.0, 0.0,
                      1.0]).reshape(3, 3),
        D_r=np.array([0.0034003170790442797, 0.001766278153469831, -0.00266312569781606, 0.0003299517423931039]),
        R_r=np.array([0.9997411981023351, 0.01955199401713946, 0.011629976219300583, -0.019819377433695273,
                      0.9995311538731381, 0.02333805294307984, -0.011168218078479885, -0.023562511898925578,
                      0.9996599816627474]).reshape(3, 3),
        rect=(61.75453410721205, 61.75453410721205, 240.22941720459062, 255.73235402091632), bf=6.242596912726197),
    # strong barrel: 1 + k1 r^2 turns negative towards the corners
    "strong_barrel": dict(
        model=PERSPECTIVE, cols=640, rows=480,
        K_l=_k(300.0, 301.5, 320.25, 239.75), D_l=np.array([-0.6, 0.05, 0.001, -0.002, 0.0]), R_l=_rot(0.01, -0.02, 0.005),
        K_r=_k(298.0, 299.0, 318.5, 241.0), D_r=np.array([-0.55, 0.04, -0.001, 0.002, 0.01]), R_r=_rot(-0.01, 0.015, 0.0),
        rect=(280.0, 280.0, 321.5, 240.5), bf=30.0),
    # an odd size whose tiles are partial, tangential distortion and a large rotation
    "odd_tangential": dict(
        model=PERSPECTIVE, cols=131, rows=97,
        K_l=_k(120.0, 118.0, 65.3, 48.1), D_l=np.array([0.05, -0.02, 0.01, -0.008, 0.003]), R_l=_rot(0.2, -0.1, 0.2),
        K_r=_k(121.0, 119.5, 64.7, 47.6), D_r=np.array([-0.03, 0.01, -0.006, 0.009, 0.0]), R_r=_rot(-0.15, 0.12, -0.2),
        rect=(110.0, 110.0, 65.0, 48.0), bf=12.0),
    # a wide fisheye with a short rectified focal length: large angles towards the corners
    "fisheye_wide": dict(
        model=FISHEYE, cols=640, rows=480,
        K_l=_k(110.0, 110.5, 318.5, 241.25), D_l=np.array([0.02, -0.01, 0.004, -0.001]), R_l=_rot(0.03, 0.02, -0.01),
        K_r=_k(111.0, 110.0, 320.5, 239.75), D_r=np.array([0.015, -0.008, 0.003, -0.0005]), R_r=_rot(-0.02, 0.01, 0.02),
        rect=(70.0, 70.0, 320.0, 240.0), bf=8.0),
}

REFERENCE_CASES = ("euroc", "tumvi")


def d5(D):
    D = np.asarray(D, np.float64).ravel()
    return np.concatenate([D, np.zeros(5 - len(D))])


def side_params(case, side):
    c = CASES[case]
    s = "l" if side == 0 else "r"
    return c[f"K_{s}"], c[f"D_{s}"], c[f"R_{s}"]


def rectifier_args(case):
    """The positional arguments of capi.StereoRectifier after (ctx, rows, cols)."""
    c = CASES[case]
    return (c["model"], c["K_l"], c["D_l"], c["R_l"], c["K_r"], c["D_r"], c["R_r"], *c["rect"])


def k_rect32(rect):
    """camera::perspective::cv_cam_matrix_: the rectified camera matrix as cv::Mat_<float>."""
    fx, fy, cx, cy = rect
    return np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32)


# ---- the oracle
def oracle_maps_raw(model, K, D, R, rect, rows, cols):
    """-> (status, map_x, map_y)."""
    mx = np.zeros((rows, cols), np.float32) if rows > 0 and cols > 0 else np.zeros(1, np.float32)
    my = np.zeros_like(mx)
    Kd, Dd, Rd = (np.ascontiguousarray(a, np.float64).ravel() for a in (K, d5(D), R))
    Kr = np.ascontiguousarray(rect, np.float64)
    st = oracle_api.lib().orc_rect_maps(C.c_int(model), Kd.ctypes.data_as(_P), Dd.ctypes.data_as(_P),
                                        Rd.ctypes.data_as(_P), Kr.ctypes.data_as(_P), C.c_int(rows), C.c_int(cols),
                                        mx.ctypes.data_as(_P), my.ctypes.data_as(_P))
    return st, mx, my


def oracle_maps(case, side):
    c = CASES[case]
    K, D, R = side_params(case, side)
    st, mx, my = oracle_maps_raw(c["model"], K, D, R, c["rect"], c["rows"], c["cols"])
    assert st == 0
    return mx, my


def oracle_remap(src, map_x, map_y, out=None):
    """cv::remap(INTER_LINEAR, BORDER_CONSTANT 0) of a 2-D uint8 view (any row stride) -> out (a new dense image unless
    given; only its first map-width bytes per row are written)."""
    assert src.dtype == np.uint8 and src.strides[1] == 1
    map_x = np.ascontiguousarray(map_x, np.float32)
    map_y = np.ascontiguousarray(map_y, np.float32)
    orows, ocols = map_x.shape
    if out is None:
        out = np.zeros((orows, ocols), np.uint8)
    assert out.strides[1] == 1
    oracle_api.lib().orc_remap_linear_u8(src.ctypes.data_as(_P), C.c_int(src.shape[0]), C.c_int(src.shape[1]),
                                         C.c_size_t(src.strides[0]), map_x.ctypes.data_as(_P), map_y.ctypes.data_as(_P),
                                         C.c_int(orows), C.c_int(ocols), out.ctypes.data_as(_P),
                                         C.c_size_t(out.strides[0]))
    return out


# ---- cv2 (the reference's calls)
def cv2_maps(case, side):
    import cv2
    c = CASES[case]
    K, D, R = side_params(case, side)
    P = k_rect32(c["rect"])
    size = (c["cols"], c["rows"])
    if c["model"] == FISHEYE:
        return cv2.fisheye.initUndistortRectifyMap(K, np.asarray(D, np.float64)[:4], R, P, size, cv2.CV_32FC1)
    return cv2.initUndistortRectifyMap(K, np.asarray(D, np.float64), R, P, size, cv2.CV_32FC1)


def texture(seed, rows, cols):
    """A seeded texture with structure at several scales (random blocks plus noise)."""
    rng = np.random.default_rng(seed)
    coarse = rng.integers(0, 256, (rows // 8 + 2, cols // 8 + 2)).astype(np.float64)
    img = np.kron(coarse, np.ones((8, 8)))[:rows, :cols]
    img = 0.7 * img + 0.3 * rng.integers(0, 256, (rows, cols))
    return np.clip(img, 0, 255).astype(np.uint8)


def random_maps(seed, rows, cols, src_rows, src_cols):
    """Random float maps over [-3, size + 3] with extreme and exactly representable coordinates mixed in."""
    rng = np.random.default_rng(seed)
    mx = rng.uniform(-3, src_cols + 3, (rows, cols)).astype(np.float32)
    my = rng.uniform(-3, src_rows + 3, (rows, cols)).astype(np.float32)
    special = np.array([0.0, -0.5, -1.0, 1.0, 0.5, src_cols - 1, src_rows - 1, src_cols - 1.0 + 1 / 64, -1e6, 1e6,
                        -40000.0, 40000.0, 32767.5, -32768.5, 1e9, -1e9, 2.5, 1.0 / 64, 3.0 / 64, -1.0 / 64, 1e-7],
                       np.float32)
    n = rows * cols // 4
    idx = rng.integers(0, rows * cols, n)
    mx.ravel()[idx] = special[rng.integers(0, len(special), n)]
    idx = rng.integers(0, rows * cols, n)
    my.ravel()[idx] = special[rng.integers(0, len(special), n)]
    # whole-pixel maps: every integer position of the source, the last row and column included, plus (-1, 0)
    k = min(rows * cols, src_rows * src_cols)
    ys, xs = np.divmod(np.arange(k), src_cols)
    mx.ravel()[:k], my.ravel()[:k] = xs.astype(np.float32), ys.astype(np.float32)
    mx.ravel()[0], my.ravel()[0] = -1.0, 0.0
    return mx, my
