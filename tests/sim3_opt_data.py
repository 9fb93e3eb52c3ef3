"""Scenes and oracle calls for optimize::transform_optimizer (the Sim3 optimiser, optimize/transform_optimizer.cc):

- `make_scene`: two keyframe poses and a ground-truth Sim3_12 with scale drift; landmarks X_2 in world coordinates and
  their partners X_1 = R_1w^T (S_12 (R_2w X_2 + t_2w) - t_1w), observed at random octaves (scale factor 1.2, 8 levels) with
  noise scaled by the octave, a chosen outlier fraction, and an initial Sim3 perturbed from the truth;
- `pack`: plp_sim3_optimize's flat layout of several scenes;
- `oracle_optimize` and the `oracle_*` Sim3 helpers: ctypes calls of oracle/transform_opt.cc in liboracle.so;
- `assert_close`: the comparison the emulator and GPU tests make against the oracle."""
from __future__ import annotations

import ctypes as C

import numpy as np

_P = C.c_void_p
FX, FY = 500.0, 510.0
CX, CY = 320.0, 240.0
COLS, ROWS = 640, 480
CAM = np.array([FX, FY, CX, CY])
NUM_LEVELS, SCALE_FACTOR = 8, 1.2
# keyframe::inv_level_sigma_sq_ (orb_params: 1 / scale_factor^(2 level), float)
INV_LEVEL_SIGMA_SQ = np.array([1.0 / np.float32(SCALE_FACTOR ** k) ** 2 for k in range(NUM_LEVELS)], np.float32)
CHI_SQ = np.float32(10.0)  # loop_detector.cc:397
NUM_ITER = 10              # transform_optimizer's default


def rotation(w):
    th = np.linalg.norm(w)
    if th == 0:
        return np.eye(3)
    k = w / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


def random_rotation(rng, max_angle):
    w = rng.normal(size=3)
    return rotation(w / np.linalg.norm(w) * rng.uniform(0.0, max_angle))


def project(X):
    return np.stack([FX * X[:, 0] / X[:, 2] + CX, FY * X[:, 1] / X[:, 2] + CY], 1)


def octaves(rng, n):
    w = np.array([SCALE_FACTOR ** -k for k in range(NUM_LEVELS)])
    return rng.choice(NUM_LEVELS, size=n, p=w / w.sum()).astype(np.int32)


def make_scene(seed, n, outlier_frac=0.0, noise_px=0.7, fix_scale=False, init_rot=0.03, init_trans=0.05,
               init_log_scale=0.03):
    """dict(pos_w_1, pos_w_2, obs_1, obs_2, w_1, w_2, pose_1w, pose_2w (12 each), R, t, s (truth), R0, t0, s0 (initial),
    outlier).  s = 1 with fix_scale (stereo / RGB-D)."""
    rng = np.random.default_rng(seed)
    R1w, R2w = random_rotation(rng, 1.0), random_rotation(rng, 1.0)
    t1w, t2w = rng.normal(size=3), rng.normal(size=3)
    R = random_rotation(rng, 0.3)
    s = 1.0 if fix_scale else float(np.exp(rng.uniform(-0.4, 0.4)))
    t = rng.normal(size=3) * 0.3
    # keyframe-2 camera points whose Sim3 images lie in front of keyframe 1, inside its image
    X2c = np.zeros((0, 3))
    while len(X2c) < n:
        m = 4 * n + 16
        z = rng.uniform(3.0, 12.0, m)
        c = np.stack([(rng.uniform(0, COLS, m) - CX) / FX * z, (rng.uniform(0, ROWS, m) - CY) / FY * z, z], 1)
        X1c = s * c @ R.T + t
        with np.errstate(divide="ignore", invalid="ignore"):
            uv = project(X1c)
        ok = (X1c[:, 2] > 0.5) & (uv[:, 0] > 0) & (uv[:, 0] < COLS) & (uv[:, 1] > 0) & (uv[:, 1] < ROWS)
        X2c = np.concatenate([X2c, c[ok]])
    X2c = X2c[:n]
    X1c = s * X2c @ R.T + t
    pos_w_2 = (X2c - t2w) @ R2w        # R_2w^T (X_2c - t_2w)
    pos_w_1 = (X1c - t1w) @ R1w
    o1, o2 = octaves(rng, n), octaves(rng, n)
    sf1, sf2 = SCALE_FACTOR ** o1.astype(np.float64), SCALE_FACTOR ** o2.astype(np.float64)
    obs_1 = project(X1c) + rng.normal(size=(n, 2)) * noise_px * sf1[:, None]
    obs_2 = project(X2c) + rng.normal(size=(n, 2)) * noise_px * sf2[:, None]
    out = rng.random(n) < outlier_frac
    k = int(out.sum())
    obs_1[out] = np.stack([rng.uniform(0, COLS, k), rng.uniform(0, ROWS, k)], 1)
    R0 = rotation(rng.normal(size=3) * init_rot) @ R
    t0 = t + rng.normal(size=3) * init_trans
    s0 = s if fix_scale else s * float(np.exp(rng.normal() * init_log_scale))
    return dict(pos_w_1=pos_w_1, pos_w_2=pos_w_2, obs_1=obs_1.astype(np.float32), obs_2=obs_2.astype(np.float32),
                w_1=INV_LEVEL_SIGMA_SQ[o1], w_2=INV_LEVEL_SIGMA_SQ[o2],
                pose_1w=np.concatenate([R1w.reshape(-1), t1w]), pose_2w=np.concatenate([R2w.reshape(-1), t2w]),
                R=R, t=t, s=s, R0=R0, t0=t0, s0=s0, outlier=out)


# the named cases every parity test runs: monocular, stereo (fix_scale), 40 % outliers, the < 10 return, no matches, and
# 1000+ matches -- (name, seed offset, make_scene arguments, fix_scale)
SCENES = [("mono", 1, dict(n=300, outlier_frac=0.1), False),
          ("stereo", 2, dict(n=250, outlier_frac=0.1, fix_scale=True), True),
          ("outliers40", 3, dict(n=400, outlier_frac=0.4, init_rot=0.08, init_trans=0.2, init_log_scale=0.1), False),
          ("few_survivors", 4, dict(n=24, outlier_frac=0.75), False),
          ("tiny", 5, dict(n=6), False),
          ("empty", 6, dict(n=0), False),
          ("large", 7, dict(n=1500, outlier_frac=0.2), False)]


def scene(k, seed=0):
    """The k-th named case (cyclic): (name, scene, fix_scale)."""
    name, off, kw, fix = SCENES[k % len(SCENES)]
    return name, make_scene(seed + off, **kw), fix


def scenes(seed=0):
    """Every named case once: [(name, scene, fix_scale)]."""
    return [scene(k, seed) for k in range(len(SCENES))]


def pack(scs, sim3_in=None):
    """plp_sim3_optimize's layout of several scenes: dict of arrays.  sim3_in: per-scene (R, t, s) overriding the
    scene's initial Sim3."""
    P = len(scs)
    off = np.zeros(P + 1, np.int32)
    for i, sc in enumerate(scs):
        off[i + 1] = off[i] + len(sc["pos_w_1"])
    cat = lambda k, shape, dt: (np.ascontiguousarray(np.concatenate([sc[k] for sc in scs]), dt) if off[-1]
                                else np.zeros(shape, dt))
    init = sim3_in or [(sc["R0"], sc["t0"], sc["s0"]) for sc in scs]
    return dict(off=off, cams=np.tile(CAM, (P, 1)),
                pose_1w=np.array([sc["pose_1w"] for sc in scs]).reshape(P, 12),
                pose_2w=np.array([sc["pose_2w"] for sc in scs]).reshape(P, 12),
                rot=np.array([np.asarray(r, np.float64).reshape(9) for r, _, _ in init]).reshape(P, 9),
                trans=np.array([np.asarray(t_, np.float64) for _, t_, _ in init]).reshape(P, 3),
                scale=np.array([s_ for _, _, s_ in init], np.float64).reshape(P),
                pos_w_1=cat("pos_w_1", (0, 3), np.float64), pos_w_2=cat("pos_w_2", (0, 3), np.float64),
                obs_1=cat("obs_1", (0, 2), np.float32), obs_2=cat("obs_2", (0, 2), np.float32),
                w_1=cat("w_1", (0,), np.float32), w_2=cat("w_2", (0,), np.float32))


# ----------------------------------------------------------------------------- oracle (oracle/transform_opt.cc)
def _ptr(a):
    return None if a is None else a.ctypes.data_as(_P)


_I, _D, _F = C.c_int, C.c_double, C.c_float
_SIGNATURES = {
    "orc_sim3_optimize": (None, [_I] + [_P] * 13 + [_F, _I, _I] + [_P] * 6),
    "orc_sim3o_exp": (None, [_P, _P]),
    "orc_sim3o_from_Rts": (None, [_P, _P, _D, _P]),
    "orc_sim3o_rotation": (None, [_P, _P]),
    "orc_sim3o_mul": (None, [_P, _P, _P]),
    "orc_sim3o_inverse": (None, [_P, _P]),
    "orc_sim3o_map": (None, [_P, _P, _P]),
    "orc_sim3o_edge": (None, [_I, _P, _P, _P, _P, _P, _P, _I, _P, _P]),
}


def _lib(orc):
    L = orc.lib
    if not getattr(L, "_sim3opt_bound", False):
        for name, (res, args) in _SIGNATURES.items():
            f = getattr(L, name)
            f.restype, f.argtypes = res, args
        L._sim3opt_bound = True
    return L


def _c(a, dt):
    a = np.ascontiguousarray(a, dt).reshape(-1)
    return a if a.size else np.zeros(1, dt)


def call(fn, d, chi_sq=CHI_SQ, num_iter=NUM_ITER, fix_scale=False, round1=False):
    """Calls an entry with plp_sim3_optimize's argument order (oracle or emulator) on a `pack` dict.  Returns
    (num_inliers (P), rot_12 (P x 3 x 3), trans_12 (P x 3), scale_12 (P), inlier (N)[, round-1 inlier (N)])."""
    P, N = len(d["off"]) - 1, int(d["off"][-1])
    keep = [_c(d["off"], np.int32), _c(d["cams"], np.float64), _c(d["pose_1w"], np.float64), _c(d["pose_2w"], np.float64),
            _c(d["rot"], np.float64), _c(d["trans"], np.float64), _c(d["scale"], np.float64),
            _c(d["pos_w_1"], np.float64), _c(d["pos_w_2"], np.float64), _c(d["obs_1"], np.float32),
            _c(d["obs_2"], np.float32), _c(d["w_1"], np.float32), _c(d["w_2"], np.float32)]
    num = np.full(max(P, 1), -7, np.int32)
    rot, trans, scale = np.full((max(P, 1), 9), np.nan), np.full((max(P, 1), 3), np.nan), np.full(max(P, 1), np.nan)
    inl, r1 = np.full(max(N, 1), 7, np.uint8), np.full(max(N, 1), 7, np.uint8)
    extra = [_ptr(r1) if round1 else None] if fn.__name__ == "orc_sim3_optimize" else []
    fn(C.c_int(P), *[_ptr(a) for a in keep], C.c_float(chi_sq), C.c_int(num_iter), C.c_int(1 if fix_scale else 0),
       _ptr(num), _ptr(rot), _ptr(trans), _ptr(scale), _ptr(inl), *extra)
    res = (num[:P], rot[:P].reshape(P, 3, 3), trans[:P], scale[:P], inl[:N])
    return res + (r1[:N],) if round1 else res


def oracle_optimize(orc, d, **kw):
    return call(_lib(orc).orc_sim3_optimize, d, **kw)


def sim3(orc, R, t, s):
    """g2o::Sim3(R, t, s) as the oracle's 8 doubles (q w x y z, t, s)."""
    out = np.zeros(8)
    _lib(orc).orc_sim3o_from_Rts(_ptr(np.ascontiguousarray(R, np.float64)), _ptr(np.ascontiguousarray(t, np.float64)),
                                 float(s), _ptr(out))
    return out


def _unary(orc, name, *args):
    out = np.zeros(8)
    getattr(_lib(orc), name)(*[_ptr(np.ascontiguousarray(a, np.float64)) for a in args], _ptr(out))
    return out


def oracle_exp(orc, u):
    return _unary(orc, "orc_sim3o_exp", u)


def oracle_mul(orc, a, b):
    return _unary(orc, "orc_sim3o_mul", a, b)


def oracle_inverse(orc, a):
    return _unary(orc, "orc_sim3o_inverse", a)


def oracle_map(orc, a, x):
    out = np.zeros(3)
    _lib(orc).orc_sim3o_map(_ptr(np.ascontiguousarray(a, np.float64)), _ptr(np.ascontiguousarray(x, np.float64)), _ptr(out))
    return out


def oracle_rotation(orc, a):
    out = np.zeros(9)
    _lib(orc).orc_sim3o_rotation(_ptr(np.ascontiguousarray(a, np.float64)), _ptr(out))
    return out.reshape(3, 3)


def oracle_edge(orc, backward, S, rot_kw, trans_kw, pos_w, obs, fix_scale=False):
    """One edge's error (2) and numeric Jacobian (2 x 7) at the oracle Sim3 S."""
    e, J = np.zeros(2), np.zeros(14)
    args = [np.ascontiguousarray(a, np.float64) for a in (CAM, S, rot_kw, trans_kw, pos_w, obs)]
    _lib(orc).orc_sim3o_edge(1 if backward else 0, *[_ptr(a) for a in args], 1 if fix_scale else 0, _ptr(e), _ptr(J))
    return e, J.reshape(2, 7)


def to_matrix(S):
    """4 x 4 similarity matrix [s R, t; 0, 1] of an oracle Sim3 (rotation from the unit quaternion)."""
    w, x, y, z = S[:4]
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                  [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                  [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
    T = np.eye(4)
    T[:3, :3] = S[7] * R
    T[:3, 3] = S[4:7]
    return T


# ----------------------------------------------------------------------------- comparisons
def max_rel_error(got, want):
    """Largest Sim3 difference of got vs want, relative to each output's magnitude (at least 1)."""
    err = 0.0
    for g, w in zip(got[1:4], want[1:4]):
        for gp, wp in zip(g, w):
            err = max(err, float(np.abs(gp - wp).max() / max(1.0, float(np.abs(wp).max())))) if np.size(wp) else err
    return err


def assert_close(got, want, rtol=1e-8):
    """Counts and inlier flags equal; the Sim3 within rtol relative (max_rel_error)."""
    assert np.array_equal(got[0], want[0]), (got[0], want[0])
    assert np.array_equal(got[4], want[4])
    for g, w in zip(got[1:4], want[1:4]):
        assert np.isfinite(g).all() and g.shape == w.shape
    err = max_rel_error(got, want)
    assert err <= rtol, err
    return err
