"""Local-BA problems: seeded generator (SURVEY.md section 8(d) config 4), ctypes marshalling for the oracle and
for the C ABI (both use the same field order), result containers."""
from __future__ import annotations

import ctypes as C

import numpy as np

import synth

_P = C.c_void_p


class BAProblemStruct(C.Structure):
    _fields_ = [("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double),
                ("focal_x_baseline", C.c_double), ("setup_type", C.c_int32),
                ("n_kf", C.c_int32), ("kf_pose_cw", _P), ("kf_fixed", _P),
                ("n_pts", C.c_int32), ("pt_pos_w", _P),
                ("n_pt_edges", C.c_int32), ("pt_edge_kf", _P), ("pt_edge_lm", _P), ("pt_edge_obs", _P),
                ("pt_edge_inv_sigma_sq", _P),
                ("n_lines", C.c_int32), ("line_plucker", _P),
                ("n_line_edges", C.c_int32), ("line_edge_kf", _P), ("line_edge_lm", _P), ("line_edge_obs", _P),
                ("line_edge_inv_sigma_sq", _P),
                ("n_plane_edges", C.c_int32), ("plane_edge_lm", _P), ("plane_edge_fn", _P)]


class BAResultStruct(C.Structure):
    _fields_ = [("kf_pose_cw", _P), ("pt_pos_w", _P), ("line_plucker", _P), ("pt_edge_outlier", _P),
                ("line_edge_outlier", _P), ("iters_first", C.c_int32), ("iters_second", C.c_int32),
                ("lm_tries", C.c_int32), ("final_chi2", C.c_double)]


class BAProblem:
    """Numpy-side container; .struct() gives the POD view (arrays are kept alive by the object)."""

    def __init__(self, **kw):
        self.stereo = kw.get("stereo", False)
        self.kf_pose_cw = np.ascontiguousarray(kw["kf_pose_cw"], np.float64)
        self.kf_fixed = np.ascontiguousarray(kw["kf_fixed"], np.uint8)
        self.pt_pos_w = np.ascontiguousarray(kw["pt_pos_w"], np.float64)
        self.pt_edge_kf = np.ascontiguousarray(kw["pt_edge_kf"], np.int32)
        self.pt_edge_lm = np.ascontiguousarray(kw["pt_edge_lm"], np.int32)
        self.pt_edge_obs = np.ascontiguousarray(kw["pt_edge_obs"], np.float32)
        self.pt_edge_inv_sigma_sq = np.ascontiguousarray(kw["pt_edge_inv_sigma_sq"], np.float32)
        z = lambda dt, *s: np.zeros(s, dt)
        self.line_plucker = np.ascontiguousarray(kw.get("line_plucker", z(np.float64, 0, 6)), np.float64)
        self.line_edge_kf = np.ascontiguousarray(kw.get("line_edge_kf", z(np.int32, 0)), np.int32)
        self.line_edge_lm = np.ascontiguousarray(kw.get("line_edge_lm", z(np.int32, 0)), np.int32)
        self.line_edge_obs = np.ascontiguousarray(kw.get("line_edge_obs", z(np.float32, 0, 4)), np.float32)
        self.line_edge_inv_sigma_sq = np.ascontiguousarray(kw.get("line_edge_inv_sigma_sq", z(np.float32, 0)), np.float32)
        self.plane_edge_lm = np.ascontiguousarray(kw.get("plane_edge_lm", z(np.int32, 0)), np.int32)
        self.plane_edge_fn = np.ascontiguousarray(kw.get("plane_edge_fn", z(np.float64, 0, 4)), np.float64)
        self.gt = kw.get("gt")

    def shard(self, world: int, rank: int, shard_boundaries, shard_edges):
        """This rank's block of landmarks (all keyframes replicated) for landmark-sharded multi-GPU BA."""
        n_pts, n_lines = len(self.pt_pos_w), len(self.line_plucker)
        pb = shard_boundaries(np.bincount(self.pt_edge_lm, minlength=n_pts), world)
        lb = shard_boundaries(np.bincount(self.line_edge_lm, minlength=n_lines) if n_lines else np.zeros(0, int), world)
        p0, p1, l0, l1 = pb[rank], pb[rank + 1], lb[rank], lb[rank + 1]
        pe, pe_lm = shard_edges(self.pt_edge_lm, p0, p1)
        le, le_lm = shard_edges(self.line_edge_lm, l0, l1)
        pl = np.nonzero((self.plane_edge_lm >= p0) & (self.plane_edge_lm < p1))[0]
        sub = BAProblem(stereo=self.stereo, kf_pose_cw=self.kf_pose_cw, kf_fixed=self.kf_fixed,
                        pt_pos_w=self.pt_pos_w[p0:p1], pt_edge_kf=self.pt_edge_kf[pe], pt_edge_lm=pe_lm,
                        pt_edge_obs=self.pt_edge_obs[pe], pt_edge_inv_sigma_sq=self.pt_edge_inv_sigma_sq[pe],
                        line_plucker=self.line_plucker[l0:l1], line_edge_kf=self.line_edge_kf[le], line_edge_lm=le_lm,
                        line_edge_obs=self.line_edge_obs[le], line_edge_inv_sigma_sq=self.line_edge_inv_sigma_sq[le],
                        plane_edge_lm=(self.plane_edge_lm[pl] - p0).astype(np.int32), plane_edge_fn=self.plane_edge_fn[pl])
        sub.block = dict(pts=(p0, p1), lines=(l0, l1), pt_edges=pe, line_edges=le)
        return sub

    @staticmethod
    def _p(a):
        return a.ctypes.data_as(_P) if a.size else None

    def struct(self) -> BAProblemStruct:
        p = self._p
        return BAProblemStruct(synth.FX, synth.FY, synth.CX, synth.CY, synth.BF if self.stereo else -1.0,
                               1 if self.stereo else 0,
                               len(self.kf_fixed), p(self.kf_pose_cw), p(self.kf_fixed),
                               len(self.pt_pos_w), p(self.pt_pos_w),
                               len(self.pt_edge_kf), p(self.pt_edge_kf), p(self.pt_edge_lm), p(self.pt_edge_obs),
                               p(self.pt_edge_inv_sigma_sq),
                               len(self.line_plucker), p(self.line_plucker),
                               len(self.line_edge_kf), p(self.line_edge_kf), p(self.line_edge_lm), p(self.line_edge_obs),
                               p(self.line_edge_inv_sigma_sq),
                               len(self.plane_edge_lm), p(self.plane_edge_lm), p(self.plane_edge_fn))


class BAResult:
    def __init__(self, prob: BAProblem):
        self.kf_pose_cw = np.zeros_like(prob.kf_pose_cw)
        self.pt_pos_w = np.zeros_like(prob.pt_pos_w)
        self.line_plucker = np.zeros((max(len(prob.line_plucker), 1), 6), np.float64)
        self.pt_edge_outlier = np.zeros(max(len(prob.pt_edge_kf), 1), np.uint8)
        self.line_edge_outlier = np.zeros(max(len(prob.line_edge_kf), 1), np.uint8)
        self._n_lines, self._n_pe, self._n_le = len(prob.line_plucker), len(prob.pt_edge_kf), len(prob.line_edge_kf)
        self.st = BAResultStruct(self.kf_pose_cw.ctypes.data_as(_P), self.pt_pos_w.ctypes.data_as(_P),
                                 self.line_plucker.ctypes.data_as(_P), self.pt_edge_outlier.ctypes.data_as(_P),
                                 self.line_edge_outlier.ctypes.data_as(_P), 0, 0, 0, 0.0)

    def finish(self):
        self.line_plucker = self.line_plucker[:self._n_lines]
        self.pt_edge_outlier = self.pt_edge_outlier[:self._n_pe]
        self.line_edge_outlier = self.line_edge_outlier[:self._n_le]
        self.iters_first, self.iters_second = self.st.iters_first, self.st.iters_second
        self.lm_tries, self.final_chi2 = self.st.lm_tries, self.st.final_chi2
        return self


def oracle_local_ba(orc, prob: BAProblem, num_first=5, num_second=10, force_stop=None) -> BAResult:
    res = BAResult(prob)
    st = prob.struct()
    fs = None if force_stop is None else np.ascontiguousarray(force_stop, np.uint8).ctypes.data_as(_P)
    orc.lib.orc_local_ba(C.byref(st), C.c_int(num_first), C.c_int(num_second), fs, C.byref(res.st))
    return res.finish()


def oracle_global_ba(orc, prob: BAProblem, num_iter=20, use_huber_kernel=True) -> BAResult:
    res = BAResult(prob)
    st = prob.struct()
    orc.lib.orc_global_ba(C.byref(st), C.c_int(num_iter), C.c_int(1 if use_huber_kernel else 0), None, C.byref(res.st))
    return res.finish()


def make_ba_problem(seed, n_local=20, n_fixed=10, n_points=4000, n_lines=800, n_plane_pts=200, stereo=False,
                    outlier_frac=0.05, pose_sigma=(0.01, 0.03), point_sigma=0.05, fast=False):
    """Config 4: local keyframes on a 4 m arc looking at a landmark cloud, fixed keyframes further along the arc,
    k ~ U{3..9} observations per landmark, octave-scaled pixel noise, 5 % outlier observations, perturbed poses
    and points; 3 planes own `n_plane_pts` of the points."""
    rng = np.random.default_rng(seed)
    n_kf = n_local + n_fixed
    sf, isig = synth.scale_factors(), synth.inv_level_sigma_sq()
    # cameras on an arc of radius 6 m around the cloud centre (0, 0, 6), looking at it
    ang = np.linspace(-0.33, 0.33, n_kf)
    order = rng.permutation(n_kf)  # which arc position is local / fixed
    poses_gt = []
    for a in ang:
        c = np.array([6.0 * np.sin(a), 0.15 * np.cos(3 * a), 6.0 - 6.0 * np.cos(a)])  # camera centre
        zc = np.array([0.0, 0.0, 6.0]) - c
        zc /= np.linalg.norm(zc)
        xc = np.cross([0.0, 1.0, 0.0], zc)
        xc /= np.linalg.norm(xc)
        yc = np.cross(zc, xc)
        R = np.stack([xc, yc, zc])  # world -> camera
        T = np.eye(4)
        T[:3, :3] = R
        T[:3, 3] = -R @ c
        poses_gt.append(T)
    poses_gt = np.stack(poses_gt)[order]
    fixed = np.zeros(n_kf, np.uint8)
    fixed[n_local:] = 1
    # planes: z = 7.5, x = 3, y = 1.5  (n, d) with n.X + d = 0
    planes = np.array([[0, 0, 1.0, -7.5], [1.0, 0, 0, -3.0], [0, 1.0, 0, -1.5]])
    X = np.stack([rng.uniform(-3, 3, n_points), rng.uniform(-2, 2, n_points), rng.uniform(4, 8, n_points)], 1)
    plane_of = np.full(n_points, -1)
    if n_plane_pts:
        own = rng.choice(n_points, n_plane_pts, replace=False)
        plane_of[own] = rng.integers(0, 3, n_plane_pts)
        for pi in range(3):
            sel = plane_of == pi
            ax = int(np.argmax(np.abs(planes[pi, :3])))
            X[sel, ax] = -planes[pi, 3]

    def observe(Xw_list_fn, n_lm):
        if fast:  # vectorised draw for the scaled-up problems (another random stream than the loop below)
            k = np.minimum(rng.integers(3, 10, n_lm), n_kf)
            pick = np.argsort(rng.random((n_lm, n_kf)), axis=1)[:, :9]
            pick = np.where(np.arange(pick.shape[1])[None, :] < k[:, None], pick, n_kf + 1)
            pick.sort(axis=1)
            sel = pick < n_kf
            return pick[sel].astype(np.int32), np.repeat(np.arange(n_lm), sel.sum(1)).astype(np.int32)
        kfs, lms = [], []
        for l in range(n_lm):
            k = int(rng.integers(3, 10))
            ks = rng.choice(n_kf, min(k, n_kf), replace=False)
            ks = ks[np.argsort(ks)]
            for kk in ks:
                kfs.append(kk)
                lms.append(l)
        return np.array(kfs, np.int32), np.array(lms, np.int32)

    ekf, elm = observe(None, n_points)
    Xc = np.einsum("eij,ej->ei", poses_gt[ekf, :3, :3], X[elm]) + poses_gt[ekf, :3, 3]
    keep = Xc[:, 2] > 0.5
    ekf, elm, Xc = ekf[keep], elm[keep], Xc[keep]
    octv = rng.choice(8, len(ekf), p=np.array([217, 181, 151, 126, 105, 87, 73, 60]) / 1000.0)
    u = synth.FX * Xc[:, 0] / Xc[:, 2] + synth.CX + rng.normal(0, 1, len(ekf)) * sf[octv]
    v = synth.FY * Xc[:, 1] / Xc[:, 2] + synth.CY + rng.normal(0, 1, len(ekf)) * sf[octv]
    out = rng.random(len(ekf)) < outlier_frac
    u[out] += rng.normal(0, 30, out.sum())
    v[out] += rng.normal(0, 30, out.sum())
    xr = np.full(len(ekf), -1.0)
    if stereo:
        has = rng.random(len(ekf)) < 0.7
        xr[has] = (u - synth.BF / Xc[:, 2] + rng.normal(0, 1, len(ekf)) * sf[octv])[has]
    obs = np.stack([u, v, xr], 1).astype(np.float32)
    # lines
    if n_lines:
        P = np.stack([rng.uniform(-3, 3, n_lines), rng.uniform(-2, 2, n_lines), rng.uniform(4, 8, n_lines)], 1)
        d = rng.normal(0, 1, (n_lines, 3))
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        Q = P + d * rng.uniform(0.5, 2.0, (n_lines, 1))
        lkf, llm = observe(None, n_lines)
        Pc = np.einsum("eij,ej->ei", poses_gt[lkf, :3, :3], P[llm]) + poses_gt[lkf, :3, 3]
        Qc = np.einsum("eij,ej->ei", poses_gt[lkf, :3, :3], Q[llm]) + poses_gt[lkf, :3, 3]
        keep = (Pc[:, 2] > 0.5) & (Qc[:, 2] > 0.5)
        lkf, llm, Pc, Qc = lkf[keep], llm[keep], Pc[keep], Qc[keep]
        lobs = np.stack([synth.FX * Pc[:, 0] / Pc[:, 2] + synth.CX, synth.FY * Pc[:, 1] / Pc[:, 2] + synth.CY,
                         synth.FX * Qc[:, 0] / Qc[:, 2] + synth.CX, synth.FY * Qc[:, 1] / Qc[:, 2] + synth.CY], 1)
        lobs += rng.normal(0, 1, lobs.shape)
        lout = rng.random(len(lkf)) < outlier_frac
        lobs[lout, :2] += rng.normal(0, 30, (lout.sum(), 2))
        # perturbed 3-D lines (endpoints jittered) -> Pluecker
        Pn = P + rng.normal(0, point_sigma, P.shape)
        Qn = Q + rng.normal(0, point_sigma, Q.shape)
        plucker = synth.plucker_from_endpoints(Pn, Qn)
        line_endpoints = np.concatenate([Pn, Qn], 1)
        line_kw = dict(line_plucker=plucker, line_edge_kf=lkf, line_edge_lm=llm, line_edge_obs=lobs.astype(np.float32),
                       line_edge_inv_sigma_sq=np.ones(len(lkf), np.float32))
    else:
        line_kw, line_endpoints = {}, np.zeros((0, 6))
    # perturb the free poses and all points
    poses = poses_gt.copy()
    for k in range(n_kf):
        if fixed[k]:
            continue
        xi = np.concatenate([rng.normal(0, pose_sigma[0], 3), rng.normal(0, pose_sigma[1], 3)])
        dT = np.eye(4)
        dT[:3, :3] = synth.so3_exp(xi[:3])
        dT[:3, 3] = xi[3:]
        poses[k] = dT @ poses[k]
    Xn = X + rng.normal(0, point_sigma, X.shape)
    pl_lm = np.nonzero(plane_of >= 0)[0].astype(np.int32)
    return BAProblem(stereo=stereo, kf_pose_cw=poses, kf_fixed=fixed, pt_pos_w=Xn, pt_edge_kf=ekf, pt_edge_lm=elm,
                     pt_edge_obs=obs, pt_edge_inv_sigma_sq=isig[octv], plane_edge_lm=pl_lm,
                     plane_edge_fn=planes[plane_of[pl_lm]] if len(pl_lm) else np.zeros((0, 4)),
                     gt=dict(poses=poses_gt, points=X, line_endpoints=line_endpoints), **line_kw)


def make_ba_shape_problem(seed, n_free, n_fixed, points, lines=(), stereo_frac=0.0, global_ba=False, empty_free=(),
                          outlier_free=(), outlier_frac=0.02, pose_sigma=(0.01, 0.03), point_sigma=0.05):
    """A problem whose OBSERVATION STRUCTURE is prescribed (make_ba_problem draws k ~ U{3..9} observers uniformly, so it never
    makes a long track, a landmark without a free observer or a keyframe without edges).  Same camera arc, cloud, noise model
    and field layout as make_ba_problem.

    points / lines: groups of landmarks, in landmark order, each a dict
        n      landmarks in the group
        k      observations per landmark: an int, "all" (every keyframe of the pool) or (lo, hi) for U{lo..hi}
        who    pool the observers are drawn from: "any" keyframe, "free", "fixed", or "one_free" (exactly one free observer,
               the other k - 1 fixed)
        plane  (points) True: every point of the group lies on one of the 3 planes and gets a plane edge
    global_ba: keyframe 0 is the only fixed one (n_fixed is ignored), as optimize::global_bundle_adjuster sets it up;
        otherwise keyframes [0, n_free) are free and [n_free, n_free + n_fixed) fixed.
    empty_free: keyframe indices left out of every pool (free keyframes without a single edge).
    outlier_free: keyframe indices whose every observation (both end points of a line) is displaced by 100..200 px.
    stereo_frac: fraction of the point edges that carry a right-image coordinate (0: monocular problem).

    The cloud (z in 4..8 m) is in front of every camera of the arc by more than 3 m, so no edge is ever dropped; the degrees
    that came out are checked against the request and returned as prob.shape = dict(pt_deg, pt_free_deg, ln_deg,
    ln_free_deg, kf_deg)."""
    rng = np.random.default_rng(seed)
    n_kf = n_free + 1 if global_ba else n_free + n_fixed
    sf, isig = synth.scale_factors(), synth.inv_level_sigma_sq()
    fixed = np.zeros(n_kf, np.uint8)
    if global_ba:
        fixed[0] = 1
    else:
        fixed[n_free:] = 1
    ang = np.linspace(-0.33, 0.33, n_kf)[rng.permutation(n_kf)]
    poses_gt = np.zeros((n_kf, 4, 4))
    for i, a in enumerate(ang):
        c = np.array([6.0 * np.sin(a), 0.15 * np.cos(3 * a), 6.0 - 6.0 * np.cos(a)])
        zc = np.array([0.0, 0.0, 6.0]) - c
        zc /= np.linalg.norm(zc)
        xc = np.cross([0.0, 1.0, 0.0], zc)
        xc /= np.linalg.norm(xc)
        R = np.stack([xc, np.cross(zc, xc), zc])
        poses_gt[i, :3, :3], poses_gt[i, :3, 3], poses_gt[i, 3, 3] = R, -R @ c, 1.0
    usable = np.ones(n_kf, bool)
    usable[list(empty_free)] = False
    pools = dict(any=np.nonzero(usable)[0], free=np.nonzero(usable & (fixed == 0))[0], fixed=np.nonzero(usable & (fixed == 1))[0])

    def observe(groups):
        kfs, lms, want, l = [], [], [], 0
        for g in groups:
            who = g.get("who", "any")
            for _ in range(g["n"]):
                pool = pools["fixed" if who == "one_free" else who]
                k = g["k"]
                if k == "all":
                    k = len(pool) + (who == "one_free")
                elif isinstance(k, tuple):  # like make_ba_problem: a small window caps the draw
                    k = min(int(rng.integers(k[0], k[1] + 1)), len(pool))
                if who == "one_free":
                    ks = np.concatenate([rng.choice(pools["free"], 1), rng.choice(pool, k - 1, replace=False)])
                else:
                    ks = rng.choice(pool, k, replace=False)
                kfs.append(rng.permutation(ks))  # the C ABI groups edges by landmark only: free and fixed observers mix
                lms.append(np.full(k, l))
                want.append(k)
                l += 1
        cat = lambda x: np.concatenate(x).astype(np.int32) if x else np.zeros(0, np.int32)
        return cat(kfs), cat(lms), np.array(want, int)

    def in_camera(ekf, Xw):
        Xc = np.einsum("eij,ej->ei", poses_gt[ekf, :3, :3], Xw) + poses_gt[ekf, :3, 3]
        assert (Xc[:, 2] > 0.5).all(), "a landmark is behind (or too close to) a camera of the arc"
        return Xc

    def project(Xc):
        return np.stack([synth.FX * Xc[:, 0] / Xc[:, 2] + synth.CX, synth.FY * Xc[:, 1] / Xc[:, 2] + synth.CY], 1)

    def displaced(n):  # gross outliers: 100..200 px in a random direction
        th, r = rng.uniform(0, 2 * np.pi, n), rng.uniform(100, 200, n)
        return np.stack([r * np.cos(th), r * np.sin(th)], 1)

    bad_kf = np.zeros(n_kf, bool)
    bad_kf[list(outlier_free)] = True
    # ---- points
    n_points = sum(g["n"] for g in points)
    planes = np.array([[0, 0, 1.0, -7.5], [1.0, 0, 0, -3.0], [0, 1.0, 0, -1.5]])
    X = np.stack([rng.uniform(-3, 3, n_points), rng.uniform(-2, 2, n_points), rng.uniform(4, 8, n_points)], 1)
    plane_of = np.full(n_points, -1)
    l = 0
    for g in points:
        if g.get("plane"):
            plane_of[l:l + g["n"]] = rng.integers(0, 3, g["n"])
        l += g["n"]
    for pi in range(3):
        X[plane_of == pi, int(np.argmax(np.abs(planes[pi, :3])))] = -planes[pi, 3]
    ekf, elm, pt_want = observe(points)
    Xc = in_camera(ekf, X[elm])
    octv = rng.choice(8, len(ekf), p=np.array([217, 181, 151, 126, 105, 87, 73, 60]) / 1000.0)
    uv = project(Xc) + rng.normal(0, 1, (len(ekf), 2)) * sf[octv][:, None]
    out = rng.random(len(ekf)) < outlier_frac
    uv[out] += rng.normal(0, 30, (out.sum(), 2))
    uv[bad_kf[ekf]] += displaced(int(bad_kf[ekf].sum()))
    xr = np.full(len(ekf), -1.0)
    if stereo_frac > 0:
        has = rng.random(len(ekf)) < stereo_frac
        xr[has] = (uv[:, 0] - synth.BF / Xc[:, 2] + rng.normal(0, 1, len(ekf)) * sf[octv])[has]
    obs = np.concatenate([uv, xr[:, None]], 1).astype(np.float32)
    # ---- lines
    n_lines = sum(g["n"] for g in lines)
    line_kw, line_endpoints, lkf, llm, ln_want = {}, np.zeros((0, 6)), np.zeros(0, np.int32), np.zeros(0, np.int32), np.zeros(0, int)
    if n_lines:
        P = np.stack([rng.uniform(-3, 3, n_lines), rng.uniform(-2, 2, n_lines), rng.uniform(4.5, 7.5, n_lines)], 1)
        d = rng.normal(0, 1, (n_lines, 3))
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        Q = P + d * rng.uniform(0.5, 2.0, (n_lines, 1))
        lkf, llm, ln_want = observe(lines)
        lobs = np.concatenate([project(in_camera(lkf, P[llm])), project(in_camera(lkf, Q[llm]))], 1)
        lobs += rng.normal(0, 1, lobs.shape)
        lout = rng.random(len(lkf)) < outlier_frac
        lobs[lout, :2] += rng.normal(0, 30, (lout.sum(), 2))
        lobs[bad_kf[lkf]] += np.concatenate([displaced(int(bad_kf[lkf].sum())), displaced(int(bad_kf[lkf].sum()))], 1)
        Pn, Qn = P + rng.normal(0, point_sigma, P.shape), Q + rng.normal(0, point_sigma, Q.shape)
        line_endpoints = np.concatenate([Pn, Qn], 1)
        line_kw = dict(line_plucker=synth.plucker_from_endpoints(Pn, Qn), line_edge_kf=lkf, line_edge_lm=llm,
                       line_edge_obs=lobs.astype(np.float32), line_edge_inv_sigma_sq=np.ones(len(lkf), np.float32))
    # ---- perturbed free poses and landmarks
    poses = poses_gt.copy()
    for k in np.nonzero(fixed == 0)[0]:
        xi = np.concatenate([rng.normal(0, pose_sigma[0], 3), rng.normal(0, pose_sigma[1], 3)])
        dT = np.eye(4)
        dT[:3, :3], dT[:3, 3] = synth.so3_exp(xi[:3]), xi[3:]
        poses[k] = dT @ poses[k]
    pl_lm = np.nonzero(plane_of >= 0)[0].astype(np.int32)
    prob = BAProblem(stereo=stereo_frac > 0, kf_pose_cw=poses, kf_fixed=fixed, pt_pos_w=X + rng.normal(0, point_sigma, X.shape),
                     pt_edge_kf=ekf, pt_edge_lm=elm, pt_edge_obs=obs, pt_edge_inv_sigma_sq=isig[octv], plane_edge_lm=pl_lm,
                     plane_edge_fn=planes[plane_of[pl_lm]] if len(pl_lm) else np.zeros((0, 4)),
                     gt=dict(poses=poses_gt, points=X, line_endpoints=line_endpoints), **line_kw)
    # ---- the shape that came out is the shape that was asked for
    free_e, free_l = (fixed[prob.pt_edge_kf] == 0).astype(float), (fixed[prob.line_edge_kf] == 0).astype(float)
    prob.shape = dict(pt_deg=np.bincount(prob.pt_edge_lm, minlength=n_points),
                      pt_free_deg=np.bincount(prob.pt_edge_lm, weights=free_e, minlength=n_points).astype(int),
                      ln_deg=np.bincount(prob.line_edge_lm, minlength=n_lines),
                      ln_free_deg=np.bincount(prob.line_edge_lm, weights=free_l, minlength=n_lines).astype(int),
                      kf_deg=np.bincount(np.concatenate([prob.pt_edge_kf, prob.line_edge_kf]), minlength=n_kf))
    assert np.array_equal(prob.shape["pt_deg"], pt_want) and np.array_equal(prob.shape["ln_deg"], ln_want)
    assert (prob.shape["kf_deg"][list(empty_free)] == 0).all()
    return prob
