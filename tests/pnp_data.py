"""Scenes and restatements for solve::pnp_solver (EPnP RANSAC, solve/pnp_solver.cc):

- `make_scene`: landmarks in front of a ground-truth pose, bearings from pixel projections with noise scaled by octave,
  octaves drawn from the ORB level budgets, a chosen outlier fraction;
- degenerate inputs: planar scenes, a bearing with z == 0, bearings with negative z, duplicate sample indices;
- `numpy_*`: an independent numpy restatement of the solver (numpy's svd, lstsq and inv in place of pnpmath.h's Jacobi
  code and cofactor inverse);
- `oracle_ransac` / `oracle_compute_pose` ...: ctypes calls of oracle/pnp.cc in liboracle.so."""
from __future__ import annotations

import ctypes as C

import numpy as np

_P = C.c_void_p
FX = FY = 500.0
CX, CY = 320.0, 240.0
COLS, ROWS = 640, 480
NUM_LEVELS, SCALE_FACTOR = 8, 1.2
SCALE_FACTORS = np.array([SCALE_FACTOR ** k for k in range(NUM_LEVELS)], np.float32)


# ----------------------------------------------------------------------------- util::cos (util/trigonometric.h)
def util_cos(v):
    """util::cos(float): the reference's polynomial cosine, in float32."""
    f = np.float32
    pi = f(3.14159265358979)
    pi_2, two_pi = f(pi / f(2)), f(f(2) * pi)
    inv_two_pi, three_pi_2 = f(f(1) / two_pi), f(f(3) * pi_2)

    def _cos(x):
        x2 = f(x * x)
        return f(f(0.99940307) + f(x2 * f(f(-0.49558072) + f(f(0.03679168) * x2))))

    v = f(v)
    v = f(v - f(f(np.floor(f(v * inv_two_pi))) * two_pi))
    v = v if f(0) < v else f(-v)
    if v < pi_2:
        return _cos(v)
    if v < pi:
        return f(-_cos(f(pi - v)))
    if v < three_pi_2:
        return f(-_cos(f(v - pi)))
    return _cos(f(two_pi - v))


def max_cos_errors(octaves):
    """pnp_solver's constructor (:47-52): util::cos(scale_factors[octave] * 1 degree) as float."""
    rad = 1.0 * np.pi / 180.0
    return np.array([util_cos(np.float32(float(SCALE_FACTORS[o]) * rad)) for o in octaves], np.float32)


# ----------------------------------------------------------------------------- scenes
def random_pose(rng):
    w = rng.normal(size=3)
    w *= rng.uniform(0.05, 0.6) / np.linalg.norm(w)
    th = np.linalg.norm(w)
    k = w / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    R = np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx
    return R, rng.normal(size=3) * 0.5


def octaves(rng, n):
    """ORB level budgets: features per level proportional to scale_factor^-level (orb_extractor's allocation)."""
    w = SCALE_FACTORS.astype(np.float64) ** -1
    return rng.choice(NUM_LEVELS, size=n, p=w / w.sum()).astype(np.int32)


def make_scene(seed, n, outlier_frac=0.0, noise_px=0.5, planar=False):
    """Returns dict(bearings, pos_w, octave, max_cos, R, t, outlier).  Bearings are unit vectors; an outlier's bearing
    points at a random pixel."""
    rng = np.random.default_rng(seed)
    R, t = random_pose(rng)
    u = rng.uniform(20, COLS - 20, n)
    v = rng.uniform(20, ROWS - 20, n)
    if planar:  # points on a tilted world plane seen by the camera
        nrm = rng.normal(size=3)
        nrm /= np.linalg.norm(nrm)
        rays_c = np.stack([(u - CX) / FX, (v - CY) / FY, np.ones(n)], 1)
        # plane n . X_w = d in camera coordinates: (R n) . X_c = d + (R n) . t
        nc = R @ nrm
        d = 4.0 + nc @ t
        if abs(nc[2]) < 0.3:
            nc = np.array([0.2, -0.1, 1.0])
            nc /= np.linalg.norm(nc)
        depth = (4.0 * nc[2] + 0.0) / (rays_c @ nc)
        Xc = rays_c * np.abs(depth)[:, None]
        del d
    else:
        z = rng.uniform(2.0, 10.0, n)
        Xc = np.stack([(u - CX) / FX * z, (v - CY) / FY * z, z], 1)
    Xw = (Xc - t) @ R           # R^T (Xc - t)
    octv = octaves(rng, n)
    sf = SCALE_FACTORS[octv].astype(np.float64)
    pu = FX * Xc[:, 0] / Xc[:, 2] + CX + rng.normal(size=n) * noise_px * sf
    pv = FY * Xc[:, 1] / Xc[:, 2] + CY + rng.normal(size=n) * noise_px * sf
    out = rng.random(n) < outlier_frac
    pu[out] = rng.uniform(0, COLS, out.sum())
    pv[out] = rng.uniform(0, ROWS, out.sum())
    b = np.stack([(pu - CX) / FX, (pv - CY) / FY, np.ones(n)], 1)
    b /= np.linalg.norm(b, axis=1, keepdims=True)
    return dict(bearings=b, pos_w=Xw, octave=octv, max_cos=max_cos_errors(octv), R=R, t=t, outlier=out)


def tie_scene(orc, seed, m=20):
    """Two noise-free groups of m points under two different poses, concatenated, and one minimal sample of each group
    (problem-local indices) whose EPnP solve recovers its group's pose exactly: two hypotheses with m inliers each and
    disjoint inlier sets."""
    a, b = make_scene(seed, m, 0.0, noise_px=0.0), make_scene(seed + 1000, m, 0.0, noise_px=0.0)
    s = {k: np.concatenate([a[k], b[k]]) for k in ("bearings", "pos_w", "octave", "max_cos", "outlier")}
    rng = np.random.default_rng(seed)
    picks = []
    for base, g in ((0, a), (m, b)):
        while True:
            smp = random_array(rng, 4, 0, m - 1) + base
            R, t, err, _ = oracle_compute_pose(orc, s["bearings"][smp], s["pos_w"][smp])
            if err < 1e-9 and np.abs(R - g["R"]).max() < 1e-6:
                picks.append(smp.astype(np.int32))
                break
    return s, picks[0], picks[1]


def random_array(rng, size, lo, hi):
    """util::create_random_array(size, lo, hi) (util/random_array.cc:46-89): `size` distinct values in [lo, hi], in
    random order."""
    return rng.permutation(np.arange(lo, hi + 1))[:size].astype(np.int32)


def draw_samples(seed, n, num_iter):
    rng = np.random.default_rng(seed)
    if n < 4:
        return np.zeros((num_iter, 4), np.int32)
    return np.stack([random_array(rng, 4, 0, n - 1) for _ in range(num_iter)]) if num_iter else np.zeros((0, 4), np.int32)


def pack(scenes, samples):
    """Concatenates per-problem scenes / samples into plp_pnp_ransac's flat layout."""
    off = np.zeros(len(scenes) + 1, np.int32)
    for i, s in enumerate(scenes):
        off[i + 1] = off[i] + len(s["bearings"])
    cat = lambda k, shape, dt: (np.concatenate([s[k] for s in scenes]).astype(dt) if off[-1] else np.zeros(shape, dt))
    return (off, cat("bearings", (0, 3), np.float64), cat("pos_w", (0, 3), np.float64), cat("max_cos", (0,), np.float32),
            np.ascontiguousarray(np.stack(samples), np.int32) if len(samples) else np.zeros((0, 0, 4), np.int32))


# ----------------------------------------------------------------------------- oracle (oracle/pnp.cc)
def _ptr(a):
    return None if a is None else a.ctypes.data_as(_P)


_I = C.c_int
_SIGNATURES = {  # oracle/pnp.cc's entries: (restype, argtypes)
    "orc_pnp_ransac": (None, [_I, _P, _P, _P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _P]),
    "orc_pnp_compute_pose": (C.c_double, [_P, _P, _I, _P, _P, _P]),
    "orc_pnp_min_norm_solve": (None, [_I, _P, _P, _P]),
    "orc_pnp_estimate_R_and_t": (None, [_P, _P, _I, _P, _P]),
    "orc_pnp_qr_solve": (None, [_P, _P, _P]),
}


def _lib(orc):
    """liboracle.so with the signatures of the EPnP entries declared (once per library handle)."""
    L = orc.lib
    if not getattr(L, "_pnp_bound", False):
        for name, (res, args) in _SIGNATURES.items():
            f = getattr(L, name)
            f.restype, f.argtypes = res, args
        L._pnp_bound = True
    return L


def oracle_ransac(orc, off, bearings, pos_w, max_cos, samples, min_num_inliers=10, recompute=True, with_hyp=False):
    """orc_pnp_ransac.  Returns (valid, num_inliers, pose (P x 4 x 4, NaN where not written), flags (N, 255 where not
    written)[, hypothesis counts])."""
    P = len(off) - 1
    N = int(off[-1])
    num_iter = samples.shape[1] if samples.ndim == 3 else 0
    sm = np.ascontiguousarray(samples, np.int32).reshape(-1) if samples.size else np.zeros(1, np.int32)
    b = np.ascontiguousarray(bearings, np.float64).reshape(-1)
    x = np.ascontiguousarray(pos_w, np.float64).reshape(-1)
    mc = np.ascontiguousarray(max_cos, np.float32)
    valid = np.zeros(P, np.int32)
    num = np.zeros(P, np.int32)
    pose = np.full((max(P, 1), 16), np.nan)
    flags = np.full(max(N, 1), 255, np.uint8)
    hyp = np.zeros(max(P * num_iter, 1), np.int32)
    _lib(orc).orc_pnp_ransac(C.c_int(P), _ptr(np.ascontiguousarray(off, np.int32)), _ptr(b if N else np.zeros(3)),
                           _ptr(x if N else np.zeros(3)), _ptr(mc if N else np.zeros(1, np.float32)), _ptr(sm),
                           C.c_int(num_iter), C.c_int(min_num_inliers), C.c_int(1 if recompute else 0), _ptr(valid),
                           _ptr(num), _ptr(pose), _ptr(flags), _ptr(hyp))
    res = (valid, num, pose[:P].reshape(P, 4, 4), flags[:N])
    return res + (hyp[:P * num_iter].reshape(P, num_iter),) if with_hyp else res


def oracle_compute_pose(orc, bearings, pos_w):
    b = np.ascontiguousarray(bearings, np.float64)
    x = np.ascontiguousarray(pos_w, np.float64)
    R, t, used = np.zeros(9), np.zeros(3), C.c_int(0)
    err = _lib(orc).orc_pnp_compute_pose(_ptr(b), _ptr(x), C.c_int(len(b)), _ptr(R), _ptr(t), C.byref(used))
    return R.reshape(3, 3), t, float(err), int(used.value)


def oracle_min_norm_solve(orc, L, rho):
    L = np.ascontiguousarray(L, np.float64)
    rho = np.ascontiguousarray(rho, np.float64)
    x = np.zeros(L.shape[1])
    _lib(orc).orc_pnp_min_norm_solve(C.c_int(L.shape[1]), _ptr(L), _ptr(rho), _ptr(x))
    return x


def oracle_estimate_R_and_t(orc, pcs, pws):
    pcs = np.ascontiguousarray(pcs, np.float64)
    pws = np.ascontiguousarray(pws, np.float64)
    R, t = np.zeros(9), np.zeros(3)
    _lib(orc).orc_pnp_estimate_R_and_t(_ptr(pcs), _ptr(pws), C.c_int(len(pcs)), _ptr(R), _ptr(t))
    return R.reshape(3, 3), t


def oracle_qr_solve(orc, A, b):
    A = np.ascontiguousarray(A, np.float64)
    b = np.ascontiguousarray(b, np.float64)
    X = np.zeros(4)
    _lib(orc).orc_pnp_qr_solve(_ptr(A), _ptr(b), _ptr(X))
    return X


# ----------------------------------------------------------------------------- numpy restatement
def numpy_min_norm_solve(L, rho):
    k = L.shape[1]
    return np.linalg.lstsq(L, rho, rcond=k * np.finfo(np.float64).eps)[0]


def numpy_estimate_R_and_t(pcs, pws):
    pc0, pw0 = pcs.mean(0), pws.mean(0)
    Abt = (pcs - pc0).T @ (pws - pw0)
    U, _, Vt = np.linalg.svd(Abt)
    V = Vt.T
    R = U @ V.T
    if np.linalg.det(R) < 0:   # change 1 (:501-514)
        V[:, 2] = -V[:, 2]
        R = U @ V.T
    return R, pc0 - R @ pw0


def numpy_compute_pose(bearings, pos_w):
    """compute_pose (:230-290) with numpy's linear algebra."""
    keep = bearings[:, 2] != 0
    b, pws = bearings[keep], pos_w[keep]
    n = len(b)
    us = b[:, :2] / b[:, 2:3]
    signs = np.where(b[:, 2] > 0, 1, -1)
    c0 = pws.mean(0)
    PW0 = pws - c0
    U, D, _ = np.linalg.svd(PW0.T @ PW0)
    # pnpmath.h's sign convention for the control-point directions: largest-magnitude component positive
    U = U * np.where(U[np.argmax(np.abs(U), 0), np.arange(3)] < 0, -1.0, 1.0)
    cws = np.vstack([c0] + [c0 + np.sqrt(D[i] / n) * U[:, i] for i in range(3)])
    CC = (cws[1:] - c0).T
    alphas = np.zeros((n, 4))
    alphas[:, 1:] = (np.linalg.inv(CC) @ (pws - c0).T).T
    alphas[:, 0] = 1.0 - alphas[:, 1:].sum(1)
    M = np.zeros((2 * n, 12))
    for k in range(4):
        M[0::2, 3 * k] = alphas[:, k]
        M[0::2, 3 * k + 2] = -alphas[:, k] * us[:, 0]
        M[1::2, 3 * k + 1] = alphas[:, k]
        M[1::2, 3 * k + 2] = -alphas[:, k] * us[:, 1]
    Um, _, _ = np.linalg.svd(M.T @ M)
    Ut = Um.T
    pairs = [(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)]
    dv = [[Ut[11 - i].reshape(4, 3)[a] - Ut[11 - i].reshape(4, 3)[c] for a, c in pairs] for i in range(4)]
    L = np.zeros((6, 10))
    terms = [(0, 0, 1), (0, 1, 2), (1, 1, 1), (0, 2, 2), (1, 2, 2), (2, 2, 1), (0, 3, 2), (1, 3, 2), (2, 3, 2), (3, 3, 1)]
    for r in range(6):
        for c, (i, j, f) in enumerate(terms):
            L[r, c] = f * dv[i][r] @ dv[j][r]
    rho = np.array([np.sum((cws[a] - cws[c]) ** 2) for a, c in pairs])

    def gauss_newton(betas):
        for _ in range(5):
            B = betas
            A = np.stack([2 * L[:, 0] * B[0] + L[:, 1] * B[1] + L[:, 3] * B[2] + L[:, 6] * B[3],
                          L[:, 1] * B[0] + 2 * L[:, 2] * B[1] + L[:, 4] * B[2] + L[:, 7] * B[3],
                          L[:, 3] * B[0] + L[:, 4] * B[1] + 2 * L[:, 5] * B[2] + L[:, 8] * B[3],
                          L[:, 6] * B[0] + L[:, 7] * B[1] + L[:, 8] * B[2] + 2 * L[:, 9] * B[3]], 1)
            q = np.array([B[0] * B[0], B[0] * B[1], B[1] * B[1], B[0] * B[2], B[1] * B[2], B[2] * B[2], B[0] * B[3],
                          B[1] * B[3], B[2] * B[3], B[3] * B[3]])
            betas = betas + np.linalg.lstsq(A, rho - L @ q, rcond=None)[0]
        return betas

    def sq(x):
        return np.sqrt(x)

    cand = []
    b4 = numpy_min_norm_solve(L[:, [0, 1, 3, 6]], rho)
    s = -1.0 if b4[0] < 0 else 1.0
    bb = sq(s * b4[0])
    cand.append(np.array([bb, s * b4[1] / bb, s * b4[2] / bb, s * b4[3] / bb]))
    b3 = numpy_min_norm_solve(L[:, :3], rho)
    if b3[0] < 0:
        be = [sq(-b3[0]), sq(-b3[2]) if b3[2] < 0 else 0.0]
    else:
        be = [sq(b3[0]), sq(b3[2]) if b3[2] > 0 else 0.0]
    if b3[1] < 0:
        be[0] = -be[0]
    cand.append(np.array(be + [0.0, 0.0]))
    b5 = numpy_min_norm_solve(L[:, :5], rho)
    if b5[0] < 0:
        be = [sq(-b5[0]), sq(-b5[2]) if b5[2] < 0 else 0.0]
    else:
        be = [sq(b5[0]), sq(b5[2]) if b5[2] > 0 else 0.0]
    if b5[1] < 0:
        be[0] = -be[0]
    cand.append(np.array(be + [b5[3] / be[0], 0.0]))
    best = None
    for betas in cand:
        betas = gauss_newton(betas)
        ccs = sum(betas[i] * Ut[11 - i].reshape(4, 3) for i in range(4))
        pcs = alphas @ ccs
        if (pcs[0, 2] < 0 and signs[0] > 0) or (pcs[0, 2] > 0 and signs[0] < 0):
            pcs = -pcs
        R, t = numpy_estimate_R_and_t(pcs, pws)
        pc = pws @ R.T + t
        err = np.mean(np.hypot(us[:, 0] - pc[:, 0] / pc[:, 2], us[:, 1] - pc[:, 1] / pc[:, 2]))
        if best is None or err < best[2]:
            best = (R, t, err)
    return best


def numpy_check_inliers(R, t, bearings, pos_w, max_cos):
    pc = pos_w @ R.T + t
    cos = np.sum(pc * bearings, 1) / np.linalg.norm(pc, axis=1)
    return (max_cos.astype(np.float64) < cos).astype(np.uint8)


def numpy_ransac(bearings, pos_w, max_cos, samples, min_num_inliers=10, recompute=True):
    """find_via_ransac (:70-153) of one problem with the numpy solver: (valid, num_inliers, R, t, flags, winner, counts)."""
    n = len(bearings)
    best, best_n, flags, Rb, tb, counts = -1, 0, np.zeros(n, np.uint8), None, None, []
    for it, s in enumerate(samples):
        R, t, _ = numpy_compute_pose(bearings[s], pos_w[s])
        f = numpy_check_inliers(R, t, bearings, pos_w, max_cos)
        counts.append(int(f.sum()))
        if best_n < f.sum():
            best, best_n, flags, Rb, tb = it, int(f.sum()), f, R, t
    valid = best_n > min_num_inliers
    if valid and recompute:
        m = flags.astype(bool)
        Rb, tb, _ = numpy_compute_pose(bearings[m], pos_w[m])
    return valid, best_n, Rb, tb, flags, best, counts


def rot_angle_deg(Ra, Rb):
    c = (np.trace(Ra.T @ Rb) - 1) / 2
    return float(np.degrees(np.arccos(np.clip(c, -1, 1))))
