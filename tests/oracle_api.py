"""ctypes wrapper of oracle/liboracle.so -- TEST INFRASTRUCTURE ONLY (never imported by the product)."""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
ORACLE_DIR = ROOT / "oracle"
_P = C.c_void_p


class OGrid(C.Structure):
    _fields_ = [("min_x", C.c_float), ("min_y", C.c_float), ("inv_cell_width", C.c_double),
                ("inv_cell_height", C.c_double), ("num_cols", C.c_int32), ("num_rows", C.c_int32)]


class OCamera(C.Structure):
    _fields_ = [("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double),
                ("focal_x_baseline", C.c_double), ("true_baseline", C.c_double),
                ("min_x", C.c_float), ("max_x", C.c_float), ("min_y", C.c_float), ("max_y", C.c_float),
                ("setup_type", C.c_int32)]


_LIB = None


def lib():
    """liboracle.so, loaded once per process.  oracle/Makefile tracks every header the library includes, so running make
    first only rebuilds what changed (and writes nothing when it is up to date)."""
    global _LIB
    if _LIB is None:
        res = subprocess.run(["make", "-C", str(ORACLE_DIR), "-j8"], capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("oracle build failed:\n" + res.stdout + res.stderr)
        _LIB = C.CDLL(str(ORACLE_DIR / "liboracle.so"))
    return _LIB


def _a(x, dt):
    if x is None:
        return None, None
    x = np.ascontiguousarray(x, dt)
    return x, x.ctypes.data_as(_P)


def as_grid(g) -> OGrid:
    return OGrid(g.min_x, g.min_y, g.inv_cell_width, g.inv_cell_height, g.num_cols, g.num_rows)


def as_camera(c) -> OCamera:
    return OCamera(c.fx, c.fy, c.cx, c.cy, c.focal_x_baseline, c.true_baseline, c.min_x, c.max_x, c.min_y, c.max_y,
                   c.setup_type)


class Oracle:
    def __init__(self):
        self.lib = lib()
        L = self.lib
        for f in ("orc_hamming_32", "orc_hamming_64", "orc_match_frame_and_landmarks",
                  "orc_match_current_and_last_frames", "orc_match_frame_and_landmarks_line",
                  "orc_match_current_and_last_frames_line", "orc_brute_force_match"):
            getattr(L, f).restype = C.c_uint

    # ---- match/base.h
    def hamming_32(self, a, b):
        a, pa = _a(a, np.uint8)
        b, pb = _a(b, np.uint8)
        return int(self.lib.orc_hamming_32(pa, pb))

    def hamming_64(self, a, b):
        a, pa = _a(a, np.uint8)
        b, pb = _a(b, np.uint8)
        return int(self.lib.orc_hamming_64(pa, pb))

    def hamming_matrix(self, a, b):
        a, pa = _a(np.asarray(a).reshape(-1, 32), np.uint8)
        b, pb = _a(np.asarray(b).reshape(-1, 32), np.uint8)
        out = np.zeros((a.shape[0], b.shape[0]), np.uint16)
        self.lib.orc_hamming_matrix(pa, C.c_int(a.shape[0]), pb, C.c_int(b.shape[0]), out.ctypes.data_as(_P))
        return out

    def hamming_nn(self, q, t):
        q, pq = _a(np.asarray(q).reshape(-1, 32), np.uint8)
        t, pt = _a(np.asarray(t).reshape(-1, 32), np.uint8)
        idx = np.zeros(q.shape[0], np.int32)
        dist = np.zeros(q.shape[0], np.uint16)
        self.lib.orc_hamming_nn(pq, C.c_int(q.shape[0]), pt, C.c_int(t.shape[0]), idx.ctypes.data_as(_P),
                                dist.ctypes.data_as(_P))
        return idx, dist

    # ---- angle checker
    def angle_checker(self, deltas, matches, hist_len=30, num_bins=3, valid=False):
        d, pd = _a(deltas, np.float32)
        m, pm = _a(matches, np.int32)
        out = np.zeros(len(d), np.int32)
        fn = self.lib.orc_angle_checker_valid if valid else self.lib.orc_angle_checker_invalid
        n = fn(pd, pm, C.c_int(len(d)), C.c_int(hist_len), C.c_int(num_bins), out.ctypes.data_as(_P))
        return out[:n].copy()

    # ---- grid
    def get_cell_indices(self, grid, x, y):
        cx, cy = C.c_int(), C.c_int()
        ok = self.lib.orc_get_cell_indices(C.byref(as_grid(grid)), C.c_float(x), C.c_float(y), C.byref(cx), C.byref(cy))
        return bool(ok), cx.value, cy.value

    def get_keypoints_in_cell(self, grid, x, y, octave, ref_x, ref_y, margin, min_level, max_level):
        x, px = _a(x, np.float32)
        y, py = _a(y, np.float32)
        o, po = _a(octave, np.int32)
        out = np.zeros(len(x), np.int32)
        n = self.lib.orc_get_keypoints_in_cell(C.byref(as_grid(grid)), px, py, po, C.c_int(len(x)), C.c_float(ref_x),
                                               C.c_float(ref_y), C.c_float(margin), C.c_int(min_level),
                                               C.c_int(max_level), out.ctypes.data_as(_P))
        return out[:n].copy()

    # ---- projection matchers
    def match_frame_and_landmarks(self, grid, scale_factors, frm, q, margin, lowe_ratio=0.6):
        keep = []

        def A(v, dt):
            arr, p = _a(v, dt)
            keep.append(arr)
            return p
        n, m = len(frm["x"]), len(q["reproj_x"])
        best = np.full(m, -2, np.int32)
        sf, psf = _a(scale_factors, np.float32)
        num = self.lib.orc_match_frame_and_landmarks(
            C.byref(as_grid(grid)), C.c_int(n), A(frm["x"], np.float32), A(frm["y"], np.float32),
            A(frm["octave"], np.int32), A(frm.get("x_right"), np.float32), A(frm["desc"], np.uint8),
            A(frm.get("claimed"), np.uint8), psf, C.c_int(len(sf)), C.c_int(m), A(q["reproj_x"], np.float32),
            A(q["reproj_y"], np.float32), A(q.get("x_right", np.zeros(m)), np.float32), A(q["scale_level"], np.int32),
            A(q["desc"], np.uint8), A(q.get("valid"), np.uint8), C.c_float(margin), C.c_float(lowe_ratio),
            best.ctypes.data_as(_P))
        return best, int(num)

    def match_current_and_last_frames(self, grid, scale_factors, cam, curr, Tc, Tl, last, margin,
                                      check_orientation=True):
        keep = []

        def A(v, dt):
            arr, p = _a(v, dt)
            keep.append(arr)
            return p
        n, m = len(curr["x"]), len(last["octave"])
        matched = np.full(n, -2, np.int32)
        sf, psf = _a(scale_factors, np.float32)
        num = self.lib.orc_match_current_and_last_frames(
            C.byref(as_grid(grid)), C.c_int(n), A(curr["x"], np.float32), A(curr["y"], np.float32),
            A(curr["octave"], np.int32), A(curr.get("angle"), np.float32), A(curr.get("x_right"), np.float32),
            A(curr["desc"], np.uint8), A(curr.get("claimed"), np.uint8), psf, C.c_int(len(sf)),
            C.byref(as_camera(cam)), A(np.asarray(Tc).reshape(16), np.float64), A(np.asarray(Tl).reshape(16), np.float64),
            C.c_int(m), A(last["pos_w"], np.float64), A(last["octave"], np.int32), A(last.get("angle"), np.float32),
            A(last["desc"], np.uint8), A(last.get("valid"), np.uint8), C.c_float(margin),
            C.c_int(1 if check_orientation else 0), matched.ctypes.data_as(_P))
        return matched, int(num)

    def match_frame_and_keyframe(self, grid, scale_factors, cam, frm, Tc, kf, margin, hamm_dist_thr,
                                 check_orientation=True):
        """kf: pos_w, min_valid_dist, max_valid_dist, angle, desc, valid.  Returns (matched, num, queries)."""
        keep = []

        def A(v, dt):
            arr, p = _a(v, dt)
            keep.append(arr)
            return p
        n, m = len(frm["x"]), len(kf["pos_w"])
        matched = np.full(n, -2, np.int32)
        sf, psf = _a(scale_factors, np.float32)
        qx, qy = np.zeros(m, np.float32), np.zeros(m, np.float32)
        ql, qv = np.zeros(m, np.int32), np.zeros(m, np.uint8)
        lsf = np.float32(np.log(np.float32(sf[1] / sf[0]))) if len(sf) > 1 else np.float32(1.0)
        self.lib.orc_match_frame_and_keyframe.restype = C.c_uint
        num = self.lib.orc_match_frame_and_keyframe(
            C.byref(as_grid(grid)), C.c_int(n), A(frm["x"], np.float32), A(frm["y"], np.float32),
            A(frm["octave"], np.int32), A(frm.get("angle"), np.float32), A(frm["desc"], np.uint8),
            A(frm.get("claimed"), np.uint8), psf, C.c_int(len(sf)), C.c_float(lsf), C.byref(as_camera(cam)),
            A(np.asarray(Tc).reshape(16), np.float64), C.c_int(m), A(kf["pos_w"], np.float64),
            A(kf["min_valid_dist"], np.float32), A(kf["max_valid_dist"], np.float32), A(kf.get("angle"), np.float32),
            A(kf["desc"], np.uint8), A(kf.get("valid"), np.uint8), C.c_float(margin), C.c_uint(hamm_dist_thr),
            C.c_int(1 if check_orientation else 0), matched.ctypes.data_as(_P), qx.ctypes.data_as(_P),
            qy.ctypes.data_as(_P), ql.ctypes.data_as(_P), qv.ctypes.data_as(_P))
        q = dict(reproj_x=qx, reproj_y=qy, scale_level=ql, valid=qv, desc=kf["desc"], angle=kf.get("angle"))
        return matched, int(num), q

    def match_frame_and_keyframe_line(self, scale_factors_lsd, log_scale_factor_lsd, cam, frm, Tc, kf, margin,
                                      hamm_dist_thr):
        keep = []

        def A(v, dt):
            arr, p = _a(v, dt)
            keep.append(arr)
            return p
        n, m = len(frm["sx"]), len(kf["pos_w"])
        matched = np.full(n, -2, np.int32)
        sf, psf = _a(scale_factors_lsd, np.float32)
        q4 = [np.zeros(m, np.float32) for _ in range(4)]
        ql, qv = np.zeros(m, np.int32), np.zeros(m, np.uint8)
        self.lib.orc_match_frame_and_keyframe_line.restype = C.c_uint
        num = self.lib.orc_match_frame_and_keyframe_line(
            C.c_int(n), A(frm["sx"], np.float32), A(frm["sy"], np.float32), A(frm["ex"], np.float32),
            A(frm["ey"], np.float32), A(frm["octave"], np.int32), A(frm["desc"], np.uint8), A(frm.get("claimed"), np.uint8),
            psf, C.c_int(len(sf)), C.c_float(log_scale_factor_lsd), C.byref(as_camera(cam)),
            A(np.asarray(Tc).reshape(16), np.float64), C.c_int(m), A(kf["pos_w"], np.float64),
            A(kf["min_valid_dist"], np.float32), A(kf["max_valid_dist"], np.float32), A(kf["desc"], np.uint8),
            A(kf.get("valid"), np.uint8), C.c_float(margin), C.c_uint(hamm_dist_thr), matched.ctypes.data_as(_P),
            q4[0].ctypes.data_as(_P), q4[1].ctypes.data_as(_P), q4[2].ctypes.data_as(_P), q4[3].ctypes.data_as(_P),
            ql.ctypes.data_as(_P), qv.ctypes.data_as(_P))
        q = dict(sp_x=q4[0], sp_y=q4[1], ep_x=q4[2], ep_y=q4[3], scale_level=ql, valid=qv, desc=kf["desc"])
        return matched, int(num), q

    def fuse_search_points(self, grid, cam, scale_factors, inv_level_sigma_sq, log_scale_factor, tgt, lms, margin, mode=1):
        """match::fuse::{detect,replace}_duplication search against ONE target keyframe -> (best_idx, best_dist, level)."""
        keep = []

        def A(v, dt):
            arr, ptr = _a(v, dt)
            keep.append(arr)
            return ptr
        g, c = as_grid(grid), as_camera(cam)
        n, m = len(tgt["x"]), len(lms["min_valid_dist"])
        sf = np.ascontiguousarray(scale_factors, np.float32)
        isg = np.ascontiguousarray(inv_level_sigma_sq, np.float32)
        best = np.full(m, -2, np.int32)
        dist = np.full(m, 0xFFFE, np.uint16)
        lvl = np.full(m, -2, np.int32)
        self.lib.orc_fuse_search_points(
            C.byref(g), C.byref(c), C.c_int(n), A(tgt["x"], np.float32), A(tgt["y"], np.float32),
            A(tgt["octave"], np.int32), A(tgt.get("x_right"), np.float32), A(tgt["desc"], np.uint8),
            A(np.asarray(tgt["rot_cw"], np.float64).reshape(9), np.float64),
            A(np.asarray(tgt["trans_cw"], np.float64).reshape(3), np.float64),
            A(np.asarray(tgt["cam_center"], np.float64).reshape(3), np.float64), sf.ctypes.data_as(C.c_void_p),
            isg.ctypes.data_as(C.c_void_p), C.c_int(len(sf)), C.c_float(log_scale_factor), C.c_int(m),
            A(np.asarray(lms["pos_w"], np.float64).reshape(m, 3), np.float64), A(lms["obs_mean_normal"], np.float64),
            A(lms["min_valid_dist"], np.float32), A(lms["max_valid_dist"], np.float32),
            A(lms["max_valid_dist_raw"], np.float32), A(lms["desc"], np.uint8), A(lms.get("valid"), np.uint8),
            A(tgt.get("skip"), np.uint8), C.c_float(margin), C.c_int(mode), best.ctypes.data_as(C.c_void_p),
            dist.ctypes.data_as(C.c_void_p), lvl.ctypes.data_as(C.c_void_p))
        return best, dist, lvl

    def fuse_search_lines(self, cam, scale_factors_lsd, inv_level_sigma_sq_lsd, log_scale_factor_lsd, tgt, lms, margin):
        """match::fuse::replace_duplication_line search against ONE target keyframe -> (best_idx, best_dist, level)."""
        keep = []

        def A(v, dt):
            arr, ptr = _a(v, dt)
            keep.append(arr)
            return ptr
        c = as_camera(cam)
        n, m = len(tgt["sx"]), len(lms["min_valid_dist"])
        sf = np.ascontiguousarray(scale_factors_lsd, np.float32)
        isg = np.ascontiguousarray(inv_level_sigma_sq_lsd, np.float32)
        best = np.full(m, -2, np.int32)
        dist = np.full(m, 0xFFFE, np.uint16)
        lvl = np.full(m, -2, np.int32)
        self.lib.orc_fuse_search_lines(
            C.byref(c), C.c_int(n), A(tgt["sx"], np.float32), A(tgt["sy"], np.float32), A(tgt["ex"], np.float32),
            A(tgt["ey"], np.float32), A(tgt["octave"], np.int32), A(tgt["desc"], np.uint8),
            A(np.asarray(tgt["rot_cw"], np.float64).reshape(9), np.float64),
            A(np.asarray(tgt["trans_cw"], np.float64).reshape(3), np.float64),
            A(np.asarray(tgt["cam_center"], np.float64).reshape(3), np.float64), sf.ctypes.data_as(C.c_void_p),
            isg.ctypes.data_as(C.c_void_p), C.c_int(len(sf)), C.c_float(log_scale_factor_lsd), C.c_int(m),
            A(np.asarray(lms["pos_w"], np.float64).reshape(m, 6), np.float64), A(lms["min_valid_dist"], np.float32),
            A(lms["max_valid_dist"], np.float32), A(lms["max_valid_dist_raw"], np.float32), A(lms["desc"], np.uint8),
            A(lms.get("valid"), np.uint8), A(tgt.get("skip"), np.uint8), C.c_float(margin),
            best.ctypes.data_as(C.c_void_p), dist.ctypes.data_as(C.c_void_p), lvl.ctypes.data_as(C.c_void_p))
        return best, dist, lvl

    def predict_scale_level(self, max_valid_dist, cam_to_lm_dist, log_scale_factor, num_levels):
        self.lib.orc_predict_scale_level.restype = C.c_uint
        return int(self.lib.orc_predict_scale_level(C.c_float(max_valid_dist), C.c_float(cam_to_lm_dist),
                                                    C.c_float(log_scale_factor), C.c_uint(num_levels)))

    # ---- DBoW2 vocabulary + match::bow_tree
    def bow_vocab_create(self, k, L, parent, desc, weight, is_leaf):
        self.lib.orc_bow_vocab_create.restype = C.c_void_p
        parent = np.ascontiguousarray(parent, np.int32)
        h = self.lib.orc_bow_vocab_create(C.c_int(k), C.c_int(L), C.c_int(len(parent) + 1), _a(parent, np.int32)[1],
                                          _a(np.ascontiguousarray(desc, np.uint8).reshape(-1, 32), np.uint8)[1],
                                          _a(np.ascontiguousarray(weight, np.float32), np.float32)[1],
                                          _a(np.ascontiguousarray(is_leaf, np.uint8), np.uint8)[1])
        if not h:
            raise RuntimeError("orc_bow_vocab_create failed")
        return C.c_void_p(h)

    def bow_vocab_load(self, path):
        self.lib.orc_bow_vocab_load.restype = C.c_void_p
        h = self.lib.orc_bow_vocab_load(str(path).encode())
        if not h:
            raise RuntimeError(f"orc_bow_vocab_load({path}) failed")
        return C.c_void_p(h)

    def bow_vocab_destroy(self, v):
        self.lib.orc_bow_vocab_destroy(v)

    def bow_vocab_info(self, v):
        o = [C.c_int32() for _ in range(4)]
        self.lib.orc_bow_vocab_info(v, *[C.byref(x) for x in o])
        return dict(k=o[0].value, L=o[1].value, num_nodes=o[2].value, num_words=o[3].value)

    def bow_transform(self, v, desc, levelsup=4):
        d = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32)
        n = d.shape[0]
        word, node, w = np.full(n, -2, np.int32), np.full(n, -2, np.int32), np.full(n, -1, np.float32)
        self.lib.orc_bow_transform(v, d.ctypes.data_as(_P), C.c_int(n), C.c_int(levelsup), word.ctypes.data_as(_P),
                                   node.ctypes.data_as(_P), w.ctypes.data_as(_P))
        return word, node, w

    def bow_tree_match(self, side1, side2, lowe_ratio, check_orientation=True):
        keep = []

        def A(v, dt):
            arr, ptr = _a(v, dt)
            keep.append(arr)
            return ptr
        n1, n2 = len(side1["desc"]), len(side2["desc"])
        m21, m12 = np.full(max(n1, 1), -2, np.int32), np.full(max(n2, 1), -2, np.int32)
        f1, f2 = side1["fv"], side2["fv"]
        self.lib.orc_bow_tree_match.restype = C.c_uint
        num = self.lib.orc_bow_tree_match(
            C.c_int(n1), A(side1["desc"], np.uint8), A(side1.get("angle"), np.float32), A(side1.get("valid"), np.uint8),
            C.c_int(n2), A(side2["desc"], np.uint8), A(side2.get("angle"), np.float32), A(side2.get("valid"), np.uint8),
            C.c_int(len(f1[0])), A(f1[0], np.uint32), A(f1[1], np.int32), A(f1[2], np.uint32),
            C.c_int(len(f2[0])), A(f2[0], np.uint32), A(f2[1], np.int32), A(f2[2], np.uint32),
            C.c_float(lowe_ratio), C.c_int(1 if check_orientation else 0), m21.ctypes.data_as(_P), m12.ctypes.data_as(_P))
        return m21[:n1].copy(), m12[:n2].copy(), int(num)

    # ---- solve::essential_solver
    def essential_compute_E21(self, b1, b2):
        b1 = np.ascontiguousarray(b1, np.float64).reshape(-1, 3)
        b2 = np.ascontiguousarray(b2, np.float64).reshape(-1, 3)
        E = np.zeros(9, np.float64)
        self.lib.orc_essential_compute_E21(b1.ctypes.data_as(_P), b2.ctypes.data_as(_P), C.c_int(len(b1)), E.ctypes.data_as(_P))
        return E.reshape(3, 3)

    def essential_ransac(self, b1, b2, matches, samples, recompute=False):
        """-> (valid, is_inlier, E_21, best_score, scores)"""
        b1 = np.ascontiguousarray(b1, np.float64).reshape(-1, 3)
        b2 = np.ascontiguousarray(b2, np.float64).reshape(-1, 3)
        m = np.ascontiguousarray(matches, np.int32).reshape(-1, 2)
        sm = np.ascontiguousarray(samples, np.int32).reshape(-1, 8)
        inl = np.zeros(max(len(m), 1), np.uint8)
        E, score, scores = np.zeros(9), C.c_double(0), np.zeros(max(len(sm), 1), np.float32)
        valid = self.lib.orc_essential_ransac(b1.ctypes.data_as(_P), b2.ctypes.data_as(_P), m.ctypes.data_as(_P),
                                              C.c_int(len(m)), sm.ctypes.data_as(_P), C.c_int(len(sm)),
                                              C.c_int(1 if recompute else 0), inl.ctypes.data_as(_P), E.ctypes.data_as(_P),
                                              C.byref(score), scores.ctypes.data_as(_P))
        return int(valid), inl[:len(m)].copy(), E.reshape(3, 3), float(score.value), scores[:len(sm)].copy()

    # ---- Planar_Mapping_module plane RANSAC
    def plane_fit(self, pos_w, idx):
        P = np.ascontiguousarray(pos_w, np.float64).reshape(-1, 3)
        ix = np.ascontiguousarray(idx, np.int32)
        eq = np.zeros(4, np.float64)
        self.lib.orc_plane_fit.restype = C.c_double
        r = self.lib.orc_plane_fit(P.ctypes.data_as(_P), ix.ctypes.data_as(_P), C.c_int(len(ix)), eq.ctypes.data_as(_P))
        return eq, float(r)

    def plane_ransac(self, pos_w, valid, samples, cfg, eq0=(0, 0, 0, 0), err0=0.0):
        """cfg = dict(mode, points_per_ransac, planar_distance_thresh, final_error_thresh, inliers_ratio_thr,
        initial_best_error) -> (status, eq, plane_error, inlier flags)."""
        class Cfg(C.Structure):
            _fields_ = [("mode", C.c_int32), ("points_per_ransac", C.c_int32), ("planar_distance_thresh", C.c_double),
                        ("final_error_thresh", C.c_double), ("inliers_ratio_thr", C.c_double),
                        ("initial_best_error", C.c_double)]
        P = np.ascontiguousarray(pos_w, np.float64).reshape(-1, 3)
        sm = np.ascontiguousarray(samples, np.int32)
        sm = sm.reshape(len(sm), -1) if sm.size else sm.reshape(0, 1)
        v = None if valid is None else np.ascontiguousarray(valid, np.uint8)
        c = Cfg(cfg["mode"], cfg["points_per_ransac"], cfg["planar_distance_thresh"], cfg["final_error_thresh"],
                cfg["inliers_ratio_thr"], cfg.get("initial_best_error", 0.0))
        eq = np.array(eq0, np.float64)
        err = C.c_double(err0)
        inl = np.zeros(max(len(P), 1), np.uint8)
        st = self.lib.orc_plane_ransac(P.ctypes.data_as(_P), None if v is None else v.ctypes.data_as(_P), C.c_int(len(P)),
                                       sm.ctypes.data_as(_P), C.c_int(sm.shape[0]), C.c_int(sm.shape[1]), C.byref(c),
                                       eq.ctypes.data_as(_P), C.byref(err), inl.ctypes.data_as(_P))
        return int(st), eq, float(err.value), inl[:len(P)].copy()

    def landmark_compute_descriptor_batch(self, descs, offsets):
        d, pd = _a(np.asarray(descs).reshape(-1, 32), np.uint8)
        o, po = _a(offsets, np.int32)
        out = np.full(max(len(o) - 1, 1), -2, np.int32)
        self.lib.orc_landmark_compute_descriptor_batch(pd, po, C.c_int(len(o) - 1), out.ctypes.data_as(_P))
        return out[:len(o) - 1].copy()

    def match_for_triangulation(self, kf1, kf2, fv1, fv2, E_12, epipole, scale_factors_1, check_orientation=True,
                                libm=0):
        keep = []

        def A(v, dt):
            arr, p = _a(v, dt)
            keep.append(arr)
            return p
        n1, n2 = len(kf1["desc"]), len(kf2["desc"])
        matched = np.full(max(n1, 1), -2, np.int32)
        self.lib.orc_match_for_triangulation.restype = C.c_uint
        num = self.lib.orc_match_for_triangulation(
            C.c_int(n1), A(kf1["desc"], np.uint8), A(kf1.get("angle"), np.float32), A(kf1["octave"], np.int32),
            A(kf1["bearings"], np.float64), A(kf1["has_landmark"], np.uint8), A(kf1.get("x_right"), np.float32),
            C.c_int(n2), A(kf2["desc"], np.uint8), A(kf2.get("angle"), np.float32), A(kf2["bearings"], np.float64),
            A(kf2["has_landmark"], np.uint8), A(kf2.get("x_right"), np.float32),
            C.c_int(len(fv1[0])), A(fv1[0], np.uint32), A(fv1[1], np.int32), A(fv1[2], np.uint32),
            C.c_int(len(fv2[0])), A(fv2[0], np.uint32), A(fv2[1], np.int32), A(fv2[2], np.uint32),
            A(np.asarray(E_12).reshape(9), np.float64), A(np.asarray(epipole).reshape(3), np.float64),
            A(scale_factors_1, np.float32), C.c_int(1 if check_orientation else 0), C.c_int(libm),
            matched.ctypes.data_as(_P))
        return matched[:n1].copy(), int(num)

    def match_frame_and_landmarks_line(self, scale_factors, frm, q, margin, lowe_ratio=0.6):
        keep = []

        def A(v, dt):
            arr, p = _a(v, dt)
            keep.append(arr)
            return p
        n, m = len(frm["sx"]), len(q["sp_x"])
        best = np.full(m, -2, np.int32)
        sf, psf = _a(scale_factors, np.float32)
        rl = frm.get("ratio_level")
        if rl is None:
            rl = frm["octave"]
        num = self.lib.orc_match_frame_and_landmarks_line(
            C.c_int(n), A(frm["sx"], np.float32), A(frm["sy"], np.float32), A(frm["ex"], np.float32),
            A(frm["ey"], np.float32), A(frm["octave"], np.int32), A(rl, np.int32), A(frm["desc"], np.uint8),
            A(frm.get("claimed"), np.uint8), psf, C.c_int(len(sf)), C.c_int(m), A(q["sp_x"], np.float32),
            A(q["sp_y"], np.float32), A(q["ep_x"], np.float32), A(q["ep_y"], np.float32),
            A(q["scale_level"], np.int32), A(q["desc"], np.uint8), A(q.get("valid"), np.uint8), C.c_float(margin),
            C.c_float(lowe_ratio), best.ctypes.data_as(_P))
        return best, int(num)

    def match_current_and_last_frames_line(self, scale_factors, cam, curr, Tc, Tl, last, margin):
        keep = []

        def A(v, dt):
            arr, p = _a(v, dt)
            keep.append(arr)
            return p
        n, m = len(curr["sx"]), len(last["octave"])
        matched = np.full(n, -2, np.int32)
        sf, psf = _a(scale_factors, np.float32)
        num = self.lib.orc_match_current_and_last_frames_line(
            C.c_int(n), A(curr["sx"], np.float32), A(curr["sy"], np.float32), A(curr["ex"], np.float32),
            A(curr["ey"], np.float32), A(curr["octave"], np.int32), A(curr.get("x_right_sp"), np.float32),
            A(curr.get("x_right_ep"), np.float32), A(curr["desc"], np.uint8), A(curr.get("claimed"), np.uint8), psf,
            C.c_int(len(sf)), C.byref(as_camera(cam)), A(np.asarray(Tc).reshape(16), np.float64),
            A(np.asarray(Tl).reshape(16), np.float64), C.c_int(m), A(last["pos_w"], np.float64),
            A(last["octave"], np.int32), A(last["desc"], np.uint8), A(last.get("valid"), np.uint8), C.c_float(margin),
            matched.ctypes.data_as(_P))
        return matched, int(num)

    def brute_force_match(self, frm_desc, frm_angle, kf_desc, kf_angle, kf_valid=None, lowe_ratio=0.8,
                          check_orientation=False):
        fd, pfd = _a(np.asarray(frm_desc).reshape(-1, 32), np.uint8)
        kd, pkd = _a(np.asarray(kf_desc).reshape(-1, 32), np.uint8)
        fa, pfa = _a(frm_angle, np.float32)
        ka, pka = _a(kf_angle, np.float32)
        kv, pkv = _a(kf_valid, np.uint8)
        matched = np.full(fd.shape[0], -2, np.int32)
        num = self.lib.orc_brute_force_match(pfd, pfa, C.c_int(fd.shape[0]), pkd, pka, pkv, C.c_int(kd.shape[0]),
                                             C.c_float(lowe_ratio), C.c_int(1 if check_orientation else 0),
                                             matched.ctypes.data_as(_P))
        return matched, int(num)


# ======================================================================== ORB (oracle/orb.cc)
class OKeyPoint(C.Structure):
    _fields_ = [("x", C.c_float), ("y", C.c_float), ("size", C.c_float), ("angle", C.c_float),
                ("response", C.c_float), ("octave", C.c_int32), ("class_id", C.c_int32)]


KP_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"),
                     ("octave", "<i4"), ("class_id", "<i4")])


class OOrbParams(C.Structure):
    _fields_ = [("max_num_keypts", C.c_uint32), ("scale_factor", C.c_float), ("num_levels", C.c_uint32),
                ("ini_fast_thr", C.c_uint32), ("min_fast_thr", C.c_uint32)]


def orb_params(max_kp=1000, sf=1.2, levels=8, ini=20, mn=7):
    return OOrbParams(max_kp, sf, levels, ini, mn)


def _orb_init(self):
    L = self.lib
    L.orc_fast_atan2.restype = C.c_float
    L.orc_fast_atan2.argtypes = [C.c_float, C.c_float]
    L.orc_util_cos.restype = C.c_float
    L.orc_util_cos.argtypes = [C.c_float]
    L.orc_util_sin.restype = C.c_float
    L.orc_util_sin.argtypes = [C.c_float]
    L.orc_orb_ic_angle.restype = C.c_float


def _resize_linear(self, src, dw, dh):
    src = np.ascontiguousarray(src, np.uint8)
    dst = np.zeros((dh, dw), np.uint8)
    self.lib.orc_resize_linear(src.ctypes.data_as(_P), C.c_int(src.shape[1]), C.c_int(src.shape[0]),
                               C.c_int(src.strides[0]), dst.ctypes.data_as(_P), C.c_int(dw), C.c_int(dh), C.c_int(dw))
    return dst


def _fast(self, img, thr, nonmax=True):
    """cv::FAST on an ROI given as a (possibly strided) uint8 2-D view."""
    assert img.dtype == np.uint8 and img.strides[1] == 1
    cap = img.shape[0] * img.shape[1]
    out = np.zeros(max(cap, 1), KP_DTYPE)
    n = self.lib.orc_fast9_16(C.c_void_p(img.ctypes.data), C.c_int(img.shape[1]), C.c_int(img.shape[0]),
                              C.c_int(img.strides[0]), C.c_int(thr), C.c_int(1 if nonmax else 0),
                              out.ctypes.data_as(_P), C.c_int(cap))
    return out[:n].copy()


def _blur7(self, img):
    img = np.ascontiguousarray(img, np.uint8)
    dst = np.zeros_like(img)
    self.lib.orc_gaussian_blur_7x7(img.ctypes.data_as(_P), C.c_int(img.shape[1]), C.c_int(img.shape[0]),
                                   C.c_int(img.shape[1]), dst.ctypes.data_as(_P), C.c_int(img.shape[1]))
    return dst


def _blur5(self, img):
    img = np.ascontiguousarray(img, np.uint8)
    dst = np.zeros_like(img)
    self.lib.orc_gaussian_blur_5x5(img.ctypes.data_as(_P), C.c_int(img.shape[1]), C.c_int(img.shape[0]),
                                   C.c_int(img.shape[1]), dst.ctypes.data_as(_P), C.c_int(img.shape[1]))
    return dst


def _orb_tables(self, p):
    L = p.num_levels
    sf, isf, ls, ils = (np.zeros(L, np.float32) for _ in range(4))
    nk = np.zeros(L, np.uint32)
    um = np.zeros(16, np.int32)
    self.lib.orc_orb_tables(C.byref(p), sf.ctypes.data_as(_P), isf.ctypes.data_as(_P), ls.ctypes.data_as(_P),
                            ils.ctypes.data_as(_P), nk.ctypes.data_as(_P), um.ctypes.data_as(_P))
    return dict(scale_factors=sf, inv_scale_factors=isf, level_sigma_sq=ls, inv_level_sigma_sq=ils,
                num_keypts_per_level=nk, u_max=um)


def _orb_level_sizes(self, p, rows, cols):
    w = np.zeros(p.num_levels, np.int32)
    h = np.zeros(p.num_levels, np.int32)
    self.lib.orc_orb_level_sizes(C.byref(p), C.c_int(rows), C.c_int(cols), w.ctypes.data_as(_P), h.ctypes.data_as(_P))
    return w, h


def _orb_distribute(self, p, cands, min_x, max_x, min_y, max_y, num_keypts):
    cands = np.ascontiguousarray(cands, KP_DTYPE)
    out = np.zeros(max(len(cands), 1), KP_DTYPE)
    n = self.lib.orc_orb_distribute(C.byref(p), cands.ctypes.data_as(_P), C.c_int(len(cands)), C.c_int(min_x),
                                    C.c_int(max_x), C.c_int(min_y), C.c_int(max_y), C.c_uint(num_keypts),
                                    out.ctypes.data_as(_P))
    return out[:n].copy()


def _orb_ic_angle(self, p, img, x, y):
    img = np.ascontiguousarray(img, np.uint8)
    return float(self.lib.orc_orb_ic_angle(C.byref(p), img.ctypes.data_as(_P), C.c_int(img.shape[1]),
                                           C.c_int(img.shape[0]), C.c_float(x), C.c_float(y)))


def _orb_describe(self, p, blurred, kp):
    blurred = np.ascontiguousarray(blurred, np.uint8)
    k = np.ascontiguousarray(kp, KP_DTYPE).reshape(1)
    d = np.zeros(32, np.uint8)
    self.lib.orc_orb_describe(C.byref(p), blurred.ctypes.data_as(_P), C.c_int(blurred.shape[1]),
                              C.c_int(blurred.shape[0]), k.ctypes.data_as(_P), d.ctypes.data_as(_P))
    return d


def _orb_extract(self, p, img, mask=None, debug=False):
    img = np.ascontiguousarray(img, np.uint8)
    rows, cols = img.shape
    cap = int(p.max_num_keypts) * 2 + 64
    kps = np.zeros(cap, KP_DTYPE)
    desc = np.zeros((cap, 32), np.uint8)
    w, h = self.orb_level_sizes(p, rows, cols)
    pyr = np.zeros(int((w.astype(np.int64) * h).sum()), np.uint8)
    cands_cap = 400000
    cands = np.zeros(cands_cap if debug else 1, KP_DTYPE)
    cpl = np.zeros(p.num_levels, np.int32)
    kpl = np.zeros(p.num_levels, np.int32)
    mk = None if mask is None else np.ascontiguousarray(mask, np.uint8)
    n = self.lib.orc_orb_extract(C.byref(p), img.ctypes.data_as(_P), C.c_int(rows), C.c_int(cols), C.c_int(cols),
                                 None if mk is None else mk.ctypes.data_as(_P),
                                 C.c_int(0 if mk is None else mk.shape[1]), kps.ctypes.data_as(_P),
                                 desc.ctypes.data_as(_P), C.c_int(cap), pyr.ctypes.data_as(_P),
                                 cands.ctypes.data_as(_P) if debug else None, C.c_int(cands_cap if debug else 0),
                                 cpl.ctypes.data_as(_P), kpl.ctypes.data_as(_P))
    assert n >= 0
    res = dict(kps=kps[:n].copy(), desc=desc[:n].copy(), kps_per_level=kpl, cands_per_level=cpl)
    levels, off = [], 0
    for l in range(p.num_levels):
        levels.append(pyr[off:off + int(w[l]) * int(h[l])].reshape(int(h[l]), int(w[l])))
        off += int(w[l]) * int(h[l])
    res["pyramid"] = levels
    if debug:
        res["cands"] = cands[:int(cpl.sum())].copy()
    return res


Oracle.resize_linear = _resize_linear
Oracle.fast = _fast
Oracle.blur7 = _blur7
Oracle.blur5 = _blur5
Oracle.orb_tables = _orb_tables
Oracle.orb_level_sizes = _orb_level_sizes
Oracle.orb_distribute = _orb_distribute
Oracle.orb_ic_angle = _orb_ic_angle
Oracle.orb_describe = _orb_describe
Oracle.orb_extract = _orb_extract
_old_init = Oracle.__init__


def _new_init(self):
    _old_init(self)
    _orb_init(self)


Oracle.__init__ = _new_init


# ======================================================================== pose optimiser (oracle/pose_opt.cc)
class OPoseCam(C.Structure):
    _fields_ = [("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double),
                ("focal_x_baseline", C.c_double), ("setup_type", C.c_int32)]


PT_OBS_DTYPE = np.dtype([("pos_w", "<f8", 3), ("obs_x", "<f4"), ("obs_y", "<f4"), ("x_right", "<f4"),
                         ("inv_sigma_sq", "<f4")])
LINE_OBS_DTYPE = np.dtype([("plucker", "<f8", 6), ("sp_x", "<f4"), ("sp_y", "<f4"), ("ep_x", "<f4"), ("ep_y", "<f4"),
                           ("inv_sigma_sq", "<f4"), ("pad", "<f4")])


def _pose_optimize(self, cam, T_cw, pts, lines=None, num_trials=4, num_each_iter=10):
    pc = OPoseCam(cam.fx, cam.fy, cam.cx, cam.cy, cam.focal_x_baseline, cam.setup_type)
    T_in = np.ascontiguousarray(np.asarray(T_cw, np.float64).reshape(16))
    pts = np.ascontiguousarray(pts, PT_OBS_DTYPE)
    nl = 0 if lines is None else len(lines)
    ln = np.ascontiguousarray(lines if nl else np.zeros(1, LINE_OBS_DTYPE), LINE_OBS_DTYPE)
    T_out = np.zeros(16, np.float64)
    pout = np.zeros(max(len(pts), 1), np.uint8)
    lout = np.zeros(max(nl, 1), np.uint8)
    iters = C.c_int(0)
    n = self.lib.orc_pose_optimize(C.byref(pc), T_in.ctypes.data_as(_P), pts.ctypes.data_as(_P), C.c_int(len(pts)),
                                   ln.ctypes.data_as(_P), C.c_int(nl), C.c_int(num_trials), C.c_int(num_each_iter),
                                   T_out.ctypes.data_as(_P), pout.ctypes.data_as(_P), lout.ctypes.data_as(_P),
                                   C.byref(iters))
    return T_out.reshape(4, 4), pout[:len(pts)].copy(), (lout[:nl].copy() if lines is not None else None), int(n), iters.value


Oracle.pose_optimize = _pose_optimize


# ======================================================================== line front end (oracle/lines.cc)
class OLsdCfg(C.Structure):
    _fields_ = [("seed_order", C.c_int32), ("libm_float", C.c_int32), ("sum_order", C.c_int32)]


KEYLINE_DTYPE = np.dtype([("angle", "<f4"), ("class_id", "<i4"), ("octave", "<i4"), ("pt_x", "<f4"), ("pt_y", "<f4"),
                          ("response", "<f4"), ("size", "<f4"), ("start_x", "<f4"), ("start_y", "<f4"),
                          ("end_x", "<f4"), ("end_y", "<f4"), ("s_oct_x", "<f4"), ("s_oct_y", "<f4"),
                          ("e_oct_x", "<f4"), ("e_oct_y", "<f4"), ("line_length", "<f4"), ("num_pixels", "<i4")])

LSD_DET = (0, 0, 1)   # the determinism rules the CUDA path implements (see oracle/lines.cc)
LSD_CV = (0, 1, 0)    # libm + sequential sums, as lsd.cpp is written


def _lsd_scaled(self, img):
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape
    out = np.zeros((int(round(h * 0.5)), int(round(w * 0.5))), np.uint8)
    self.lib.orc_lsd_scaled_image(img.ctypes.data_as(_P), C.c_int(w), C.c_int(h), C.c_int(w), out.ctypes.data_as(_P))
    return out


def _lsd_detect(self, img, mode=LSD_DET):
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape
    cap = 30000
    out = np.zeros((cap, 4), np.float32)
    cfg = OLsdCfg(*mode)
    n = self.lib.orc_lsd_detect(img.ctypes.data_as(_P), C.c_int(w), C.c_int(h), C.c_int(w), C.byref(cfg),
                                out.ctypes.data_as(_P), C.c_int(cap))
    assert n >= 0
    return out[:n].copy()


def _lsd_keylines(self, img, min_length, mode=LSD_DET):
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape
    cap = 30000
    out = np.zeros(cap, KEYLINE_DTYPE)
    cfg = OLsdCfg(*mode)
    n = self.lib.orc_lsd_keylines(img.ctypes.data_as(_P), C.c_int(w), C.c_int(h), C.c_int(w), C.byref(cfg),
                                  C.c_double(min_length), out.ctypes.data_as(_P), C.c_int(cap))
    assert n >= 0
    return out[:n].copy()


def _lbd_gradients(self, img):
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape
    dx, dy = np.zeros((h, w), np.int16), np.zeros((h, w), np.int16)
    self.lib.orc_lbd_gradients(img.ctypes.data_as(_P), C.c_int(w), C.c_int(h), C.c_int(w), dx.ctypes.data_as(_P),
                               dy.ctypes.data_as(_P))
    return dx, dy


def _lbd_compute(self, img, keylines, libm=0):
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape
    kl = np.ascontiguousarray(keylines, KEYLINE_DTYPE)
    n = len(kl)
    desc = np.zeros((max(n, 1), 32), np.uint8)
    fl = np.zeros((max(n, 1), 72), np.float32)
    self.lib.orc_lbd_compute(img.ctypes.data_as(_P), C.c_int(w), C.c_int(h), C.c_int(w), kl.ctypes.data_as(_P),
                             C.c_int(n), C.c_int(libm), desc.ctypes.data_as(_P), fl.ctypes.data_as(_P))
    return desc[:n].copy(), fl[:n].copy()


def _line_extract(self, img, mode=LSD_DET):
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape
    cap = 8192
    kl = np.zeros(cap, KEYLINE_DTYPE)
    lbd = np.zeros((cap, 32), np.uint8)
    fn = np.zeros((cap, 3), np.float64)
    cfg = OLsdCfg(*mode)
    n = self.lib.orc_line_extract(img.ctypes.data_as(_P), C.c_int(w), C.c_int(h), C.c_int(w), C.byref(cfg),
                                  kl.ctypes.data_as(_P), lbd.ctypes.data_as(_P), fn.ctypes.data_as(_P), C.c_int(cap))
    assert n >= 0
    return kl[:n].copy(), lbd[:n].copy(), fn[:n].copy()


Oracle.lsd_scaled = _lsd_scaled
Oracle.lsd_detect = _lsd_detect
Oracle.lsd_keylines = _lsd_keylines
Oracle.lbd_gradients = _lbd_gradients
Oracle.lbd_compute = _lbd_compute
Oracle.line_extract = _line_extract


# ======================================================================== stereo matcher (oracle/stereo.cc)
def _stereo_compute(self, res_left, res_right, scale_factors, inv_scale_factors, focal_x_baseline, true_baseline):
    """res_* = outputs of Oracle.orb_extract (pyramid, kps, desc) of the left / right image."""
    pl = np.ascontiguousarray(np.concatenate([l.ravel() for l in res_left["pyramid"]]))
    pr = np.ascontiguousarray(np.concatenate([l.ravel() for l in res_right["pyramid"]]))
    w = np.array([l.shape[1] for l in res_left["pyramid"]], np.int32)
    h = np.array([l.shape[0] for l in res_left["pyramid"]], np.int32)
    kl, kr = np.ascontiguousarray(res_left["kps"]), np.ascontiguousarray(res_right["kps"])
    dl, dr = np.ascontiguousarray(res_left["desc"]), np.ascontiguousarray(res_right["desc"])
    sf = np.ascontiguousarray(scale_factors, np.float32)
    isf = np.ascontiguousarray(inv_scale_factors, np.float32)
    n = len(kl)
    xr, dp, br = np.zeros(max(n, 1), np.float32), np.zeros(max(n, 1), np.float32), np.zeros(max(n, 1), np.int32)
    self.lib.orc_stereo_compute(pl.ctypes.data_as(_P), pr.ctypes.data_as(_P), w.ctypes.data_as(_P), h.ctypes.data_as(_P),
                                C.c_int(len(w)), kl.ctypes.data_as(_P), dl.ctypes.data_as(_P), C.c_int(n),
                                kr.ctypes.data_as(_P), dr.ctypes.data_as(_P), C.c_int(len(kr)), sf.ctypes.data_as(_P),
                                isf.ctypes.data_as(_P), C.c_float(focal_x_baseline), C.c_float(true_baseline),
                                xr.ctypes.data_as(_P), dp.ctypes.data_as(_P), br.ctypes.data_as(_P))
    return xr[:n].copy(), dp[:n].copy(), br[:n].copy()


Oracle.stereo_compute = _stereo_compute


# ======================================================================== native thread pool (oracle/frontend_mt.cc)
def _host_cpus(self):
    return int(self.lib.orc_host_cpus())


def _frontend_track_batch(self, p, grid, cam, imgs, lasts, pose_pred, pose_last, margin=20.0, threads=1, pin=True):
    """extract -> match_current_and_last_frames (+ widened retry) -> pose_optimizer -> discard_outliers for a batch of
    independent frames on `threads` native threads.  lasts[b]: dict(pos_w, octave, angle, desc, valid|None)."""
    imgs = np.ascontiguousarray(imgs, np.uint8)
    B, rows, cols = imgs.shape
    offs = np.zeros(B + 1, np.int32)
    offs[1:] = np.cumsum([len(l["octave"]) for l in lasts])
    cat = lambda k, dt: np.ascontiguousarray(np.concatenate([np.asarray(l[k], dt) for l in lasts]))
    pos, octv, ang, desc = cat("pos_w", np.float64), cat("octave", np.int32), cat("angle", np.float32), cat("desc", np.uint8)
    valid = np.ascontiguousarray(np.concatenate([np.asarray(l["valid"] if l.get("valid") is not None else
                                                            np.ones(len(l["octave"]), np.uint8), np.uint8) for l in lasts]))
    pp = np.ascontiguousarray(np.asarray(pose_pred, np.float64).reshape(B, 16))
    pl = np.ascontiguousarray(np.asarray(pose_last, np.float64).reshape(B, 16))
    pose = np.zeros((B, 16), np.float64)
    n_inl, n_valid, n_kp = np.zeros(B, np.int32), np.zeros(B, np.int32), np.zeros(B, np.int32)
    sec = C.c_double(0)
    g, c = as_grid(grid), as_camera(cam)
    P = lambda a: a.ctypes.data_as(_P)
    self.lib.orc_frontend_track_batch(C.byref(p), C.byref(g), C.byref(c), P(imgs), C.c_int(B), C.c_int(rows), C.c_int(cols),
                                      P(pos), P(octv), P(ang), P(desc), P(valid), P(offs), P(pp), P(pl), C.c_float(margin),
                                      C.c_int(threads), C.c_int(1 if pin else 0), P(pose), P(n_inl), P(n_valid), P(n_kp),
                                      C.byref(sec))
    return dict(pose=pose.reshape(B, 4, 4), n_inliers=n_inl, num_valid=n_valid, n_kp=n_kp, seconds=sec.value)


def _line_extract_batch_mt(self, imgs, threads=1, pin=True, mode=LSD_DET):
    imgs = np.ascontiguousarray(imgs, np.uint8)
    B, rows, cols = imgs.shape
    n = np.zeros(B, np.int32)
    sec = C.c_double(0)
    cfg = OLsdCfg(*mode)
    self.lib.orc_line_extract_batch_mt(imgs.ctypes.data_as(_P), C.c_int(B), C.c_int(rows), C.c_int(cols), C.byref(cfg),
                                       C.c_int(threads), C.c_int(1 if pin else 0), n.ctypes.data_as(_P), C.byref(sec))
    return n, sec.value


def _stereo_frontend_batch_mt(self, p, left, right, focal_x_baseline, true_baseline, threads=1, pin=True, mode=LSD_DET):
    """ORB left + right, match::stereo::compute, LSD + LBD left + right (data/frame.cc:456-480) per stereo frame."""
    left, right = np.ascontiguousarray(left, np.uint8), np.ascontiguousarray(right, np.uint8)
    B, rows, cols = left.shape
    n_kp, n_st, n_ln = np.zeros((B, 2), np.int32), np.zeros(B, np.int32), np.zeros((B, 2), np.int32)
    sec = C.c_double(0)
    cfg = OLsdCfg(*mode)
    self.lib.orc_stereo_frontend_batch_mt(C.byref(p), C.byref(cfg), left.ctypes.data_as(_P), right.ctypes.data_as(_P),
                                          C.c_int(B), C.c_int(rows), C.c_int(cols), C.c_float(focal_x_baseline),
                                          C.c_float(true_baseline), C.c_int(threads), C.c_int(1 if pin else 0),
                                          n_kp.ctypes.data_as(_P), n_st.ctypes.data_as(_P), n_ln.ctypes.data_as(_P),
                                          C.byref(sec))
    return dict(n_kp=n_kp, n_stereo=n_st, n_lines=n_ln, seconds=sec.value)


Oracle.host_cpus = _host_cpus
Oracle.frontend_track_batch = _frontend_track_batch
Oracle.line_extract_batch_mt = _line_extract_batch_mt
Oracle.stereo_frontend_batch_mt = _stereo_frontend_batch_mt
