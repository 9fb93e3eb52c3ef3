"""Scenes and restatements for solve::sim3_solver (Sim3 RANSAC, solve/sim3_solver.cc):

- `make_scene`: two keyframes that share landmarks under a known Sim3 (X_2 = s R X_1 + t), noise scaled by each
  keypoint's octave, a chosen outlier fraction, optional points behind either camera, s = 1 for `fix_scale` (stereo);
- `draw_samples` (distinct triples, as util::create_random_array(3, 0, n - 1)) and `pack` (plp_sim3_ransac's layout);
- `oracle_ransac` / `oracle_compute`: ctypes calls of oracle/sim3.cc in liboracle.so;
- `numpy_*`: an independent numpy restatement (Horn's rotation from np.linalg.eigh, the reference's scale, translation
  and inlier rule)."""
from __future__ import annotations

import ctypes as C

import numpy as np

_P = C.c_void_p
FX, FY = 500.0, 510.0
CX, CY = 320.0, 240.0
COLS, ROWS = 640, 480
CAM = np.array([FX, FY, CX, CY])
NUM_LEVELS, SCALE_FACTOR = 8, 1.2
# keyframe::level_sigma_sq_ (orb_params: scale_factor^(2 level), float) and the constructor's chi_sq_2D * sigma_sq
LEVEL_SIGMA_SQ = np.array([np.float32(SCALE_FACTOR ** k) ** 2 for k in range(NUM_LEVELS)], np.float32)
CHI_SQ_2D = np.float32(9.21034)


def chi_sq(octaves):
    return (CHI_SQ_2D * LEVEL_SIGMA_SQ[octaves]).astype(np.float32)


# ----------------------------------------------------------------------------- scenes
def rotation(w):
    th = np.linalg.norm(w)
    if th == 0:
        return np.eye(3)
    k = w / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


def octaves(rng, n):
    """ORB level budgets: features per level proportional to scale_factor^-level."""
    w = np.array([SCALE_FACTOR ** -k for k in range(NUM_LEVELS)])
    return rng.choice(NUM_LEVELS, size=n, p=w / w.sum()).astype(np.int32)


def _pixel_noise(rng, X, octv, noise_px):
    """Moves each point across the image plane by a pixel noise of noise_px x scale_factor^octave at its own depth."""
    sf = SCALE_FACTOR ** octv.astype(np.float64)
    z = X[:, 2]
    out = X.copy()
    out[:, 0] += rng.normal(size=len(X)) * noise_px * sf * z / FX
    out[:, 1] += rng.normal(size=len(X)) * noise_px * sf * z / FY
    return out


def make_scene(seed, n, outlier_frac=0.0, noise_px=0.5, fix_scale=False, scale=None, behind_1=0, behind_2=0):
    """Returns dict(pts_1, pts_2, chi_sq_1, chi_sq_2, R, t, s, outlier): the keyframe-1 / keyframe-2 camera-frame points of
    n matched landmarks, X_2 = s R X_1 + t for inliers.  behind_1 / behind_2 points get a negative depth in keyframe 1 / 2."""
    rng = np.random.default_rng(seed)
    w = rng.normal(size=3)
    R = rotation(w * rng.uniform(0.05, 0.4) / np.linalg.norm(w))
    s = 1.0 if fix_scale else (float(rng.uniform(0.6, 1.7)) if scale is None else float(scale))
    t = rng.normal(size=3) * 0.3
    u, v, z = rng.uniform(20, COLS - 20, n), rng.uniform(20, ROWS - 20, n), rng.uniform(3.0, 12.0, n)
    X1 = np.stack([(u - CX) / FX * z, (v - CY) / FY * z, z], 1)
    X2 = s * X1 @ R.T + t
    o1, o2 = octaves(rng, n), octaves(rng, n)
    if noise_px > 0:
        X1, X2 = _pixel_noise(rng, X1, o1, noise_px), _pixel_noise(rng, X2, o2, noise_px)
    out = rng.random(n) < outlier_frac
    k = int(out.sum())
    zo = rng.uniform(3.0, 12.0, k) * s
    X2[out] = np.stack([(rng.uniform(0, COLS, k) - CX) / FX * zo, (rng.uniform(0, ROWS, k) - CY) / FY * zo, zo], 1)
    if behind_1:
        X1[:behind_1, 2] *= -1
    if behind_2:
        X2[n - behind_2:, 2] *= -1
    return dict(pts_1=X1, pts_2=X2, chi_sq_1=chi_sq(o1), chi_sq_2=chi_sq(o2), R=R, t=t, s=s, outlier=out)


def concat(*scenes):
    return {k: np.concatenate([sc[k] for sc in scenes]) for k in ("pts_1", "pts_2", "chi_sq_1", "chi_sq_2", "outlier")}


def random_array(rng, size, lo, hi):
    """util::create_random_array(size, lo, hi): `size` distinct values in [lo, hi], in random order."""
    return rng.permutation(np.arange(lo, hi + 1))[:size].astype(np.int32)


def draw_samples(seed, n, num_iter):
    rng = np.random.default_rng(seed)
    if n < 3 or num_iter == 0:
        return np.zeros((num_iter, 3), np.int32)
    return np.stack([random_array(rng, 3, 0, n - 1) for _ in range(num_iter)])


def pack(scenes, samples):
    """Concatenates per-problem scenes / samples into plp_sim3_ransac's flat layout: (off, pts_1, pts_2, chi_sq_1,
    chi_sq_2, samples)."""
    off = np.zeros(len(scenes) + 1, np.int32)
    for i, sc in enumerate(scenes):
        off[i + 1] = off[i] + len(sc["pts_1"])
    cat = lambda k, shape, dt: (np.concatenate([sc[k] for sc in scenes]).astype(dt) if off[-1] else np.zeros(shape, dt))
    return (off, cat("pts_1", (0, 3), np.float64), cat("pts_2", (0, 3), np.float64), cat("chi_sq_1", (0,), np.float32),
            cat("chi_sq_2", (0,), np.float32),
            np.ascontiguousarray(np.stack(samples), np.int32) if len(samples) else np.zeros((0, 0, 3), np.int32))


def problems(seed, P, sizes, num_iter=200, outlier_frac=0.5, fix_scale=False):
    """P problems of the given sizes (cycled), each with its own scene and samples."""
    scenes, samples = [], []
    for i in range(P):
        n = sizes[i % len(sizes)]
        scenes.append(make_scene(seed * 1000 + i, n, outlier_frac, fix_scale=fix_scale))
        samples.append(draw_samples(seed * 1000 + i, n, num_iter))
    return pack(scenes, samples)


# ----------------------------------------------------------------------------- oracle (oracle/sim3.cc)
def _ptr(a):
    return None if a is None else a.ctypes.data_as(_P)


_I = C.c_int
_SIGNATURES = {  # oracle/sim3.cc's entries: (restype, argtypes)
    "orc_sim3_ransac": (None, [_I, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _P, _P]),
    "orc_sim3_compute": (None, [_P, _P, _I, _P, _P, _P, _P, _P, _P]),
}


def _lib(orc):
    """liboracle.so with the signatures of the Sim3 entries declared (once per library handle)."""
    L = orc.lib
    if not getattr(L, "_sim3_bound", False):
        for name, (res, args) in _SIGNATURES.items():
            f = getattr(L, name)
            f.restype, f.argtypes = res, args
        L._sim3_bound = True
    return L


def oracle_ransac(orc, off, pts_1, pts_2, chi_sq_1, chi_sq_2, samples, fix_scale=False, min_num_inliers=20,
                  cams=None, with_hyp=False):
    """orc_sim3_ransac.  cams: P x 4 (fx, fy, cx, cy), CAM for every problem by default.  Returns (valid, num_inliers,
    rot_12 (P x 3 x 3), trans_12 (P x 3), scale_12 (P)[, hypothesis counts (P x num_iter)])."""
    P = len(off) - 1
    N = int(off[-1])
    num_iter = samples.shape[1] if samples.ndim == 3 else 0
    cams = np.ascontiguousarray(np.tile(CAM, (P, 1)) if cams is None else cams, np.float64).reshape(-1)
    sm = np.ascontiguousarray(samples, np.int32).reshape(-1) if samples.size else np.zeros(1, np.int32)
    x1 = np.ascontiguousarray(pts_1, np.float64).reshape(-1) if N else np.zeros(3)
    x2 = np.ascontiguousarray(pts_2, np.float64).reshape(-1) if N else np.zeros(3)
    c1 = np.ascontiguousarray(chi_sq_1, np.float32) if N else np.zeros(1, np.float32)
    c2 = np.ascontiguousarray(chi_sq_2, np.float32) if N else np.zeros(1, np.float32)
    valid, num = np.full(max(P, 1), 7, np.int32), np.full(max(P, 1), 7, np.int32)
    rot, trans, scale = np.full((max(P, 1), 9), np.nan), np.full((max(P, 1), 3), np.nan), np.full(max(P, 1), np.nan, np.float32)
    hyp = np.zeros(max(P * num_iter, 1), np.int32)
    _lib(orc).orc_sim3_ransac(P, _ptr(np.ascontiguousarray(off, np.int32)), _ptr(cams if P else np.zeros(4)), _ptr(x1),
                              _ptr(x2), _ptr(c1), _ptr(c2), _ptr(sm), num_iter, 1 if fix_scale else 0, min_num_inliers,
                              _ptr(valid), _ptr(num), _ptr(rot), _ptr(trans), _ptr(scale), _ptr(hyp))
    res = (valid[:P], num[:P], rot[:P].reshape(P, 3, 3), trans[:P], scale[:P])
    return res + (hyp[:P * num_iter].reshape(P, num_iter),) if with_hyp else res


def oracle_compute(orc, p1, p2, fix_scale=False):
    """orc_sim3_compute on three points: (rot_12, trans_12, scale_12, rot_21, trans_21, scale_21)."""
    p1 = np.ascontiguousarray(p1, np.float64)
    p2 = np.ascontiguousarray(p2, np.float64)
    R12, t12, R21, t21 = np.zeros(9), np.zeros(3), np.zeros(9), np.zeros(3)
    s12, s21 = C.c_float(0), C.c_float(0)
    _lib(orc).orc_sim3_compute(_ptr(p1), _ptr(p2), 1 if fix_scale else 0, _ptr(R12), _ptr(t12), C.byref(s12), _ptr(R21),
                               _ptr(t21), C.byref(s21))
    return R12.reshape(3, 3), t12, np.float32(s12.value), R21.reshape(3, 3), t21, np.float32(s21.value)


def assert_same(got, want):
    """Bit-equal outputs (NaN never appears in written outputs; equal_nan guards the helpers' fill values)."""
    for g, w in zip(got, want):
        assert g.dtype == w.dtype and g.shape == w.shape
        assert np.array_equal(g, w, equal_nan=True), (g, w)


# ----------------------------------------------------------------------------- numpy restatement
def numpy_compute(p1, p2, fix_scale=False):
    """compute_Sim3 (:193-288) with numpy: Horn's quaternion from np.linalg.eigh, the reference's float scales.
    Returns (rot_12, trans_12, scale_12, rot_21, trans_21, scale_21, eigengap)."""
    c1, c2 = p1.mean(0), p2.mean(0)
    A1, A2 = (p1 - c1).T, (p2 - c2).T
    M = A1 @ A2.T
    (Sxx, Sxy, Sxz), (Syx, Syy, Syz), (Szx, Szy, Szz) = M
    N = np.array([[Sxx + Syy + Szz, Syz - Szy, Szx - Sxz, Sxy - Syx],
                  [Syz - Szy, Sxx - Syy - Szz, Sxy + Syx, Szx + Sxz],
                  [Szx - Sxz, Sxy + Syx, -Sxx + Syy - Szz, Syz + Szy],
                  [Sxy - Syx, Szx + Sxz, Syz + Szy, -Sxx - Syy + Szz]])
    lam, V = np.linalg.eigh(N)
    w, x, y, z = V[:, -1] / np.linalg.norm(V[:, -1])
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                  [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                  [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
    s21 = np.float32(1.0) if fix_scale else np.float32(np.sum(A2 * (R @ A1)) / np.sum(A1 * A1))
    t21 = c2 - float(s21) * R @ c1
    s12 = np.float32(1.0 / float(s21))
    t12 = -float(s12) * R.T @ t21
    gap = (lam[-1] - lam[-2]) / max(abs(lam[-1]), 1e-300)
    return R.T, t12, s12, R, t21, s21, gap


def numpy_reproject(R, t, s, X):
    """reproject_to_image(s R, t, X) of many points; NaN behind the camera (sim3math.h's deviation 1)."""
    pc = X @ (float(s) * R).T + t
    with np.errstate(divide="ignore", invalid="ignore"):
        uv = np.stack([FX * pc[:, 0] / pc[:, 2] + CX, FY * pc[:, 1] / pc[:, 2] + CY], 1)
    uv[pc[:, 2] <= 0] = np.nan
    return uv


def numpy_errors(model, pts_1, pts_2):
    """count_inliers' squared errors (error_in_1, error_in_2) of one hypothesis."""
    R12, t12, s12, R21, t21, s21 = model[:6]
    r1 = numpy_reproject(np.eye(3), np.zeros(3), 1.0, pts_1)
    r2 = numpy_reproject(np.eye(3), np.zeros(3), 1.0, pts_2)
    e2 = np.sum((numpy_reproject(R21, t21, s21, pts_1) - r2) ** 2, 1)
    e1 = np.sum((numpy_reproject(R12, t12, s12, pts_2) - r1) ** 2, 1)
    return e1, e2


def numpy_inliers(model, sc, rtol=0.0):
    """Inlier flags of one hypothesis: (sure, possible) -- `possible` also takes errors within rtol of a threshold."""
    e1, e2 = numpy_errors(model, sc["pts_1"], sc["pts_2"])
    c1, c2 = sc["chi_sq_1"].astype(np.float64), sc["chi_sq_2"].astype(np.float64)
    with np.errstate(invalid="ignore"):
        sure = (e1 < c1 * (1 - rtol)) & (e2 < c2 * (1 - rtol))
        possible = (e1 < c1 * (1 + rtol)) & (e2 < c2 * (1 + rtol))
    return sure, possible
