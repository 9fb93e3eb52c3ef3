"""The plane RANSAC DEVICE code (structure-plp-slam_b200/csrc/plane_kernels.cuh) executed on the CPU: tests/cta_emu compiles
the same kernel text for the host (one host thread per CUDA thread, a pthread barrier for __syncthreads, blocks one
after the other) and this test compares it with the oracle bit for bit.  It checks the kernels' logic -- indexing, phase
structure, replay bookkeeping -- in a container without a GPU; the GPU parity run is tests/test_plane_gpu.py."""
import ctypes as C

import numpy as np
import pytest

import emu_build
import plane_data

_P = C.c_void_p


class Cfg(C.Structure):
    _fields_ = [("mode", C.c_int32), ("points_per_ransac", C.c_int32), ("planar_distance_thresh", C.c_double),
                ("final_error_thresh", C.c_double), ("inliers_ratio_thr", C.c_double), ("initial_best_error", C.c_double)]


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return emu_build.emu("plane_emu", tmp_path_factory, opt="-O1")


def _run(emu, pts, valid, smp, cfg, eq0=(0, 0, 0, 0), err0=0.0):
    P = np.ascontiguousarray(pts, np.float64).reshape(-1, 3)
    sm = np.ascontiguousarray(smp, np.int32)
    v = None if valid is None else np.ascontiguousarray(valid, np.uint8)
    c = Cfg(cfg["mode"], cfg["points_per_ransac"], cfg["planar_distance_thresh"], cfg["final_error_thresh"],
            cfg["inliers_ratio_thr"], cfg.get("initial_best_error", 0.0))
    eq = np.array(eq0, np.float64)
    err = C.c_double(err0)
    inl = np.zeros(max(len(P), 1), np.uint8)
    st = emu.emu_plane_ransac(P.ctypes.data_as(_P), None if v is None else v.ctypes.data_as(_P), C.c_int(len(P)),
                              sm.ctypes.data_as(_P), C.c_int(sm.shape[0]), C.c_int(sm.shape[1]), C.byref(c),
                              eq.ctypes.data_as(_P), C.byref(err), inl.ctypes.data_as(_P))
    return int(st), eq, float(err.value), inl[:len(P)].copy()


@pytest.mark.parametrize("seed", range(4))
def test_plane_kernels_on_cpu_match_oracle(emu, orc, seed):
    n = [300, 120, 60, 18][seed]
    pts, valid, _, _ = plane_data.make_plane_cloud(seed + 10, n=n)
    smp = plane_data.draw_plane_samples(seed, valid, 12, 18)
    want = orc.plane_ransac(pts, valid, smp, plane_data.CFG_ESTIMATE)
    got = _run(emu, pts, valid, smp, plane_data.CFG_ESTIMATE)
    assert got[0] == want[0] and np.array_equal(got[1], want[1]) and got[2] == want[2] and np.array_equal(got[3], want[3])
    # update mode from a stored plane
    eq0, err0 = orc.plane_fit(pts, np.nonzero(valid)[0][:18].astype(np.int32))
    smp_u = plane_data.draw_plane_samples(seed + 1, valid, 6, int(np.ceil(0.8 * n)))
    want = orc.plane_ransac(pts, valid, smp_u, plane_data.CFG_UPDATE, eq0, err0)
    got = _run(emu, pts, valid, smp_u, plane_data.CFG_UPDATE, eq0, err0)
    assert got[0] == want[0] and np.array_equal(got[1], want[1]) and got[2] == want[2] and np.array_equal(got[3], want[3])


def test_plane_kernels_on_cpu_failure_paths(emu, orc):
    cloud = np.random.default_rng(1).uniform(-1, 1, (80, 3))
    smp = plane_data.draw_plane_samples(2, np.ones(80), 8, 18)
    want = orc.plane_ransac(cloud, None, smp, plane_data.CFG_ESTIMATE)
    got = _run(emu, cloud, None, smp, plane_data.CFG_ESTIMATE)
    assert got[0] == want[0] == 0 and np.array_equal(got[1], want[1]) and got[2] == want[2] and got[3].sum() == 0


# ---------------------------------------------------------------------------------------------------------------------
# the essential-matrix RANSAC kernels are GPU-verified (tests/test_essential_gpu.py): running them through the emulator as
# well validates the emulator itself
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ess_emu(tmp_path_factory):
    return emu_build.emu("essential_emu", tmp_path_factory, opt="-O1")


@pytest.mark.parametrize("seed", range(3))
def test_essential_kernels_on_cpu_match_oracle(ess_emu, orc, seed):
    import ess_data
    n = [200, 60, 33][seed]
    b1, b2, matches, _ = ess_data.make_two_view(seed + 10, n=n)
    smp = ess_data.draw_samples(seed, len(matches), 12)
    for recompute in (False, True):
        want = orc.essential_ransac(b1, b2, matches, smp, recompute)
        B1, B2 = np.ascontiguousarray(b1, np.float64), np.ascontiguousarray(b2, np.float64)
        m, sm = np.ascontiguousarray(matches, np.int32), np.ascontiguousarray(smp, np.int32)
        inl, E, score = np.zeros(len(m), np.uint8), np.zeros(9), C.c_double(0)
        valid = ess_emu.emu_essential_ransac(B1.ctypes.data_as(_P), B2.ctypes.data_as(_P), m.ctypes.data_as(_P),
                                             C.c_int(len(m)), sm.ctypes.data_as(_P), C.c_int(len(sm)),
                                             C.c_int(1 if recompute else 0), inl.ctypes.data_as(_P), E.ctypes.data_as(_P),
                                             C.byref(score))
        assert valid == want[0] and np.array_equal(inl, want[1]) and np.array_equal(E.reshape(3, 3), want[2])
        assert score.value == want[3]


# ---------------------------------------------------------------------------------------------------------------------
# DBoW2 transform and match::bow_tree kernels (GPU-verified, tests/test_bow_gpu.py): warp shuffles / ballots / match on the
# emulator's per-warp exchange
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def bow_emu(tmp_path_factory):
    lib = emu_build.emu("bow_emu", tmp_path_factory, opt="-O1")
    lib.emu_bow_match.restype = C.c_uint
    return lib


def _csr_vocab(vocab):
    """The device layout plp_bow_vocab_create builds (csrc/bow.cu): node 0 = root, children grouped by parent."""
    parent = vocab["parent"]
    N = len(parent) + 1
    cnt = np.bincount(parent, minlength=N)
    child_begin = np.zeros(N + 1, np.uint32)
    child_begin[1:] = np.cumsum(cnt)
    fill = child_begin[:-1].astype(np.int64).copy()
    children = np.zeros(max(N - 1, 1), np.uint32)
    for i, p in enumerate(parent):
        children[fill[p]] = i + 1
        fill[p] += 1
    desc = np.zeros((N, 32), np.uint8)
    desc[1:] = vocab["desc"]
    weight = np.zeros(N, np.float32)
    weight[1:] = vocab["weight"]
    word = np.full(N, -1, np.int32)
    word[1:][vocab["is_leaf"] > 0] = np.arange(int(vocab["is_leaf"].sum()))
    return child_begin, children, desc, weight, word, int(cnt.max())


@pytest.mark.parametrize("k,L,levelsup", [(10, 3, 1), (4, 4, 4), (20, 2, 1)])
def test_bow_transform_kernel_on_cpu_matches_oracle(bow_emu, orc, k, L, levelsup):
    import bow_data
    import synth
    vocab = bow_data.make_vocab(k * 100 + L, k=k, L=L)
    child_begin, children, ndesc, weight, word, maxc = _csr_vocab(vocab)
    rng = np.random.default_rng(L)
    n = 70
    desc = synth.rand_desc(rng, n)
    ov = orc.bow_vocab_create(k, L, vocab["parent"], vocab["desc"], vocab["weight"], vocab["is_leaf"])
    want = orc.bow_transform(ov, desc, levelsup)
    orc.bow_vocab_destroy(ov)
    G = 4 if maxc <= 4 else 8 if maxc <= 8 else 16 if maxc <= 16 else 32
    w_out, n_out, f_out = np.full(n, -2, np.int32), np.full(n, -2, np.int32), np.full(n, -1, np.float32)
    bow_emu.emu_bow_transform(C.c_int(G), ndesc.ctypes.data_as(_P), child_begin.ctypes.data_as(_P),
                              children.ctypes.data_as(_P), weight.ctypes.data_as(_P), word.ctypes.data_as(_P),
                              desc.ctypes.data_as(_P), C.c_int(n), C.c_int(L - levelsup), w_out.ctypes.data_as(_P),
                              n_out.ctypes.data_as(_P), f_out.ctypes.data_as(_P))
    assert np.array_equal(w_out, want[0]) and np.array_equal(n_out, want[1]) and np.array_equal(f_out, want[2])


@pytest.mark.parametrize("seed", range(2))
def test_bow_match_kernel_on_cpu_matches_oracle(bow_emu, orc, seed):
    import bow_data
    s1, s2, _ = bow_data.make_bow_sides(seed, n1=160, n2=180, num_nodes=14)
    for ratio, check, use_valid2 in [(0.75, True, True), (0.9, False, False)]:
        b = dict(s2)
        if not use_valid2:
            b.pop("valid")
        want = orc.bow_tree_match(s1, b, ratio, check)
        f1, f2 = s1["fv"], b["fv"]
        nb1, ne1, nb2, ne2 = [], [], [], []
        i = j = 0
        while i < len(f1[0]) and j < len(f2[0]):      # the host's merge-join (csrc/bow.cu)
            if f1[0][i] == f2[0][j]:
                nb1.append(f1[1][i]); ne1.append(f1[1][i + 1]); nb2.append(f2[1][j]); ne2.append(f2[1][j + 1])
                i += 1
                j += 1
            elif f1[0][i] < f2[0][j]:
                i += 1
            else:
                j += 1
        A = lambda v, dt: np.ascontiguousarray(v, dt)  # noqa: E731
        d1, d2 = A(s1["desc"], np.uint8), A(b["desc"], np.uint8)
        a1, a2 = A(s1["angle"], np.float32), A(b["angle"], np.float32)
        v1 = A(s1["valid"], np.uint8)
        v2 = A(b["valid"], np.uint8) if "valid" in b else None
        i1, i2 = A(f1[2], np.uint32), A(f2[2], np.uint32)
        nb1, ne1, nb2, ne2 = (A(x, np.int32) for x in (nb1, ne1, nb2, ne2))
        m21, m12 = np.full(len(d1), -2, np.int32), np.full(len(d2), -2, np.int32)
        num = bow_emu.emu_bow_match(C.c_int(len(d1)), d1.ctypes.data_as(_P), a1.ctypes.data_as(_P), v1.ctypes.data_as(_P),
                                    C.c_int(len(d2)), d2.ctypes.data_as(_P), a2.ctypes.data_as(_P),
                                    None if v2 is None else v2.ctypes.data_as(_P), i1.ctypes.data_as(_P),
                                    i2.ctypes.data_as(_P), C.c_int(len(nb1)), nb1.ctypes.data_as(_P), ne1.ctypes.data_as(_P),
                                    nb2.ctypes.data_as(_P), ne2.ctypes.data_as(_P), C.c_float(ratio),
                                    C.c_int(1 if check else 0), m21.ctypes.data_as(_P), m12.ctypes.data_as(_P))
        assert np.array_equal(m21, want[0]) and np.array_equal(m12, want[1]) and num == want[2]
        assert want[2] > 20


# ---------------------------------------------------------------------------------------------------------------------
# match::fuse search kernel (GPU-verified, tests/test_fuse_gpu.py): dynamic shared memory, counting sort with atomics
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def fuse_emu(tmp_path_factory):
    return emu_build.emu("fuse_emu", tmp_path_factory, opt="-O1")


@pytest.mark.parametrize("seed,mode,stereo", [(0, 1, False), (1, 0, False), (2, 1, True)])
def test_fuse_points_kernel_on_cpu_matches_oracle(fuse_emu, orc, plp, seed, mode, stereo):
    import fuse_data
    import synth
    lms, targets = fuse_data.make_point_fuse_scene(seed + 60, m=90, num_targets=2, n_extra=40, stereo=stereo)
    grid = plp.capi.make_grid(synth.COLS, synth.ROWS)
    cam = plp.capi.make_camera(synth.FX, synth.FY, synth.CX, synth.CY, synth.COLS, synth.ROWS,
                               bf=synth.BF if stereo else -1.0, setup_type=1 if stereo else 0)
    sf, isg = synth.scale_factors(), fuse_data.inv_level_sigma_sq()
    thr = plp.capi.fuse_level_thresholds(fuse_data.LOG_SF, len(sf))       # the product's host-side table
    thr[0] = np.inf
    keep = []

    def A(v, dt):
        a = np.ascontiguousarray(v, dt)
        keep.append(a)
        return a
    K = len(targets)
    n_arr = A([len(t["x"]) for t in targets], np.int32)
    ptrs = {k: (C.c_void_p * K)() for k in ("x", "y", "xr", "oct", "desc", "skip")}
    pose = np.zeros((K, 15), np.float64)
    for i, t in enumerate(targets):
        ptrs["x"][i] = A(t["x"], np.float32).ctypes.data
        ptrs["y"][i] = A(t["y"], np.float32).ctypes.data
        ptrs["xr"][i] = A(t["x_right"], np.float32).ctypes.data if "x_right" in t else None
        ptrs["oct"][i] = A(t["octave"], np.int32).ctypes.data
        ptrs["desc"][i] = A(t["desc"], np.uint8).ctypes.data
        ptrs["skip"][i] = A(t["skip"], np.uint8).ctypes.data
        pose[i, :9] = np.asarray(t["rot_cw"]).reshape(9)
        pose[i, 9:12] = t["trans_cw"]
        pose[i, 12:] = t["cam_center"]
    m = len(lms["desc"])
    best = np.full((K, m), -2, np.int32)
    dist = np.full((K, m), 0xFFFE, np.uint16)
    fuse_emu.emu_fuse_points(
        C.c_int(K), n_arr.ctypes.data_as(_P), ptrs["x"], ptrs["y"], ptrs["xr"], ptrs["oct"], ptrs["desc"], ptrs["skip"],
        pose.ctypes.data_as(_P), C.byref(grid), C.byref(cam), sf.ctypes.data_as(_P), isg.ctypes.data_as(_P),
        thr.ctypes.data_as(_P), C.c_int(len(sf)), C.c_float(3.0), C.c_int(mode), C.c_int(m),
        A(lms["pos_w"], np.float64).ctypes.data_as(_P), A(lms["obs_mean_normal"], np.float64).ctypes.data_as(_P),
        A(lms["min_valid_dist"], np.float32).ctypes.data_as(_P), A(lms["max_valid_dist"], np.float32).ctypes.data_as(_P),
        A(lms["max_valid_dist_raw"], np.float32).ctypes.data_as(_P), A(lms["desc"], np.uint8).ctypes.data_as(_P),
        A(lms["valid"], np.uint8).ctypes.data_as(_P), C.c_int(48), best.ctypes.data_as(_P), dist.ctypes.data_as(_P))
    total = 0
    for i, t in enumerate(targets):
        o_idx, o_dist, _ = orc.fuse_search_points(grid, cam, sf, isg, fuse_data.LOG_SF, t, lms, 3.0, mode)
        assert np.array_equal(best[i], o_idx) and np.array_equal(dist[i], o_dist)
        total += (o_idx >= 0).sum()
    assert total > 10


# ---------------------------------------------------------------------------------------------------------------------
# window matcher (csrc/point_match_kernels.cuh): 1024 threads, shared-memory counting sort, 4-lane query groups, deferred
# acceptance -- checked against the oracle before any GPU time is spent on it
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pmatch_emu(tmp_path_factory):
    return emu_build.emu("pmatch_emu", tmp_path_factory, opt="-O1")


class _Grid(C.Structure):
    _fields_ = [("min_x", C.c_float), ("min_y", C.c_float), ("inv_cell_width", C.c_double),
                ("inv_cell_height", C.c_double), ("num_cols", C.c_int32), ("num_rows", C.c_int32)]


def _emu_point_match(emu, grid, frm, q, ratio_test, lowe_ratio, check_orientation, hamm_thr_p1=0):
    keep = []

    def A(v, dt):
        if v is None:
            return None
        a = np.ascontiguousarray(v, dt)
        keep.append(a)
        return a.ctypes.data_as(_P)
    n, m = len(frm["x"]), len(q["qx"])
    cap = max(64, (n + 63) // 64 * 64)
    choice = np.zeros(max(m, 1), np.int32)
    best = np.full(max(m, 1), -7, np.int32)
    matched = np.full(max(n, 1), -7, np.int32)
    num = np.zeros(1, np.uint32)
    g = _Grid(grid.min_x, grid.min_y, grid.inv_cell_width, grid.inv_cell_height, grid.num_cols, grid.num_rows)
    emu.emu_point_match(C.byref(g), C.c_int(n), A(frm["x"], np.float32), A(frm["y"], np.float32), A(frm["octave"], np.int32),
                        A(frm.get("angle"), np.float32), A(frm.get("x_right"), np.float32), A(frm["desc"], np.uint8),
                        A(frm.get("claimed"), np.uint8), C.c_int(m), A(q["qx"], np.float32), A(q["qy"], np.float32),
                        A(q.get("qxr"), np.float32), A(q["qradius"], np.float32), A(q["qmin"], np.int32),
                        A(q["qmax"], np.int32), A(q.get("qangle"), np.float32), A(q["qdesc"], np.uint8),
                        A(q.get("qvalid"), np.uint8), C.c_uint(hamm_thr_p1), C.c_int(ratio_test), C.c_float(lowe_ratio),
                        C.c_int(check_orientation), C.c_int(cap), choice.ctypes.data_as(_P), best.ctypes.data_as(_P),
                        matched.ctypes.data_as(_P), num.ctypes.data_as(_P))
    return best[:m], matched[:n], int(num[0])


@pytest.mark.parametrize("seed", range(3))
def test_point_match_kernel_on_cpu_ratio_path(pmatch_emu, orc, plp, seed):
    import synth
    grid = plp.capi.make_grid(synth.COLS, synth.ROWS)
    sf = synth.scale_factors()
    curr, last, Tc, Tl = synth.make_tracking_scene(seed, n_last=400, stereo=(seed == 2))
    q = synth.make_landmark_queries(seed + 50, curr, m=700)
    want, wn = orc.match_frame_and_landmarks(grid, sf, curr, q, 5.0 if seed else 12.0, 0.8)
    margin = np.float32(5.0 if seed else 12.0)
    lvl = np.asarray(q["scale_level"], np.int32)
    qq = dict(qx=q["reproj_x"], qy=q["reproj_y"], qxr=q.get("x_right", np.zeros(len(lvl), np.float32)),
              qradius=(margin * sf[lvl].astype(np.float32)).astype(np.float32), qmin=lvl - 1, qmax=lvl, qdesc=q["desc"],
              qvalid=q.get("valid"))
    best, _, num = _emu_point_match(pmatch_emu, grid, curr, qq, 1, 0.8, 0)
    assert np.array_equal(best, want) and num == wn


@pytest.mark.parametrize("seed", range(3))
def test_point_match_kernel_on_cpu_deferred_acceptance_path(pmatch_emu, orc, plp, seed):
    """match_current_and_last_frames: reprojection pre-pass restated in numpy (project_points_kernel, monocular level range),
    then the no-ratio path with the orientation histogram."""
    import synth
    grid = plp.capi.make_grid(synth.COLS, synth.ROWS)
    cam = plp.capi.make_camera(synth.FX, synth.FY, synth.CX, synth.CY, synth.COLS, synth.ROWS)
    sf = synth.scale_factors()
    curr, last, Tc, Tl = synth.make_tracking_scene(seed + 7, n_last=600, dup_frac=0.3)
    margin = 20.0 if seed < 2 else 40.0
    want, wn = orc.match_current_and_last_frames(grid, sf, cam, curr, Tc, Tl, last, margin, True)
    P = np.asarray(Tc, np.float64).reshape(4, 4)
    X = np.asarray(last["pos_w"], np.float64)
    pc = [((P[r, 0] * X[:, 0] + P[r, 1] * X[:, 1]) + P[r, 2] * X[:, 2]) + P[r, 3] for r in range(3)]
    front = pc[2] > 0.0
    zi = 1.0 / np.where(front, pc[2], 1.0)
    u = cam.fx * pc[0] * zi + cam.cx
    v = cam.fy * pc[1] * zi + cam.cy
    in_img = front & (np.float64(cam.min_x) < u) & (u < np.float64(cam.max_x)) & (np.float64(cam.min_y) < v) & (v < np.float64(cam.max_y))
    lvl = np.asarray(last["octave"], np.int32)
    valid = (np.asarray(last.get("valid", np.ones(len(lvl))), np.uint8) != 0) & in_img
    qq = dict(qx=np.where(front, u, 0.0).astype(np.float32), qy=np.where(front, v, 0.0).astype(np.float32),
              qxr=np.where(front, u - cam.focal_x_baseline * zi, 0.0).astype(np.float32),
              qradius=(np.float32(margin) * sf[lvl].astype(np.float32)).astype(np.float32), qmin=lvl - 1, qmax=lvl + 1,
              qangle=last["angle"], qdesc=last["desc"], qvalid=valid.astype(np.uint8))
    _, matched, num = _emu_point_match(pmatch_emu, grid, curr, qq, 0, 0.0, 1)
    assert np.array_equal(matched, want) and num == wn


# ---------------------------------------------------------------------------------------------------------------------
# motion-only BA (csrc/pose_opt_kernels.cuh): one warp per frame, redundant 6x6 solve in every lane
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def poseopt_emu(tmp_path_factory):
    return emu_build.emu("poseopt_emu", tmp_path_factory, opt="-O1")


def _emu_pose_opt(emu, cam, scenes, with_lines):
    import oracle_api
    B = len(scenes)
    T_in = np.ascontiguousarray(np.stack([s[1] for s in scenes]), np.float64)
    pts = np.ascontiguousarray(np.concatenate([np.asarray(s[2], oracle_api.PT_OBS_DTYPE) for s in scenes]))
    pt_off = np.zeros(B + 1, np.int32)
    pt_off[1:] = np.cumsum([len(s[2]) for s in scenes])
    if with_lines:
        lines = np.ascontiguousarray(np.concatenate([np.asarray(s[3], oracle_api.LINE_OBS_DTYPE) for s in scenes]))
        ln_off = np.zeros(B + 1, np.int32)
        ln_off[1:] = np.cumsum([len(s[3]) for s in scenes])
    else:
        lines, ln_off = None, None
    T_out = np.zeros((B, 4, 4))
    pout = np.zeros(max(len(pts), 1), np.uint8)
    lout = np.zeros(max(len(lines) if lines is not None else 0, 1), np.uint8)
    ninl, its = np.zeros(B, np.int32), np.zeros(B, np.int32)
    emu.emu_pose_optimize_batch(C.byref(cam), C.c_int(B), T_in.ctypes.data_as(_P), pts.ctypes.data_as(_P),
                                pt_off.ctypes.data_as(_P), None if lines is None else lines.ctypes.data_as(_P),
                                None if lines is None else ln_off.ctypes.data_as(_P), C.c_int(4), C.c_int(10),
                                T_out.ctypes.data_as(_P), pout.ctypes.data_as(_P),
                                None if lines is None else lout.ctypes.data_as(_P), ninl.ctypes.data_as(_P),
                                its.ctypes.data_as(_P))
    return T_out, [pout[pt_off[b]:pt_off[b + 1]] for b in range(B)], \
        ([lout[ln_off[b]:ln_off[b + 1]] for b in range(B)] if lines is not None else None), ninl, its


@pytest.mark.parametrize("with_lines", [False, True])
def test_pose_opt_kernel_on_cpu_matches_oracle(poseopt_emu, orc, plp, with_lines):
    import synth
    scenes = [synth.make_pose_opt_scene(s, n_pts=[1000, 317, 40][s % 3], n_lines=[200, 37][s % 2], stereo=False)
              for s in range(5)]
    scenes.append(synth.make_pose_opt_scene(100, outlier_frac=0.45, pose_sigma=(0.15, 0.4)))   # rejected steps
    scenes.append(synth.make_pose_opt_scene(3, n_pts=4, n_lines=0))                              # < 5 observations
    cam = plp.capi.make_camera(synth.FX, synth.FY, synth.CX, synth.CY, synth.COLS, synth.ROWS)
    T, pf, lf, ninl, its = _emu_pose_opt(poseopt_emu, cam, scenes, with_lines)
    for b, (T_gt, T_init, pts, lines) in enumerate(scenes):
        ln = lines if (with_lines and len(lines)) else None
        To, po, lo, no, it_o = orc.pose_optimize(cam, T_init, pts, ln)
        assert np.linalg.norm(T[b] - To) / np.linalg.norm(To) < 1e-8, b
        # the LM iteration count is not compared: it may differ by a few near convergence: accept / terminate decisions at rounding level
        # (rho == 0, chi differences ~1e-13) depend on the summation order, the optimum does not
        assert np.array_equal(pf[b], po) and ninl[b] == no, b
        if ln is not None:
            assert np.array_equal(lf[b], lo), b


def test_pose_opt_kernel_on_cpu_stereo(poseopt_emu, orc, plp):
    import synth
    scenes = [synth.make_pose_opt_scene(20 + s, stereo=True, n_pts=300, n_lines=50) for s in range(3)]
    cam = plp.capi.make_camera(synth.FX, synth.FY, synth.CX, synth.CY, synth.COLS, synth.ROWS, bf=synth.BF, setup_type=1)
    T, pf, lf, ninl, its = _emu_pose_opt(poseopt_emu, cam, scenes, True)
    for b, (T_gt, T_init, pts, lines) in enumerate(scenes):
        To, po, lo, no, it_o = orc.pose_optimize(cam, T_init, pts, lines)
        assert np.linalg.norm(T[b] - To) / np.linalg.norm(To) < 1e-8
        assert np.array_equal(pf[b], po) and np.array_equal(lf[b], lo) and ninl[b] == no


def test_point_match_kernel_on_cpu_worklist_overflow(pmatch_emu, orc, plp):
    """Far more queries than keypoints: every keypoint is contested by ~10 queries, the bumped-query work list (cap / 2
    entries) overflows and the kernel finishes with full-scan rounds -- same sequential result."""
    import synth
    grid = plp.capi.make_grid(synth.COLS, synth.ROWS)
    cam = plp.capi.make_camera(synth.FX, synth.FY, synth.CX, synth.CY, synth.COLS, synth.ROWS)
    sf = synth.scale_factors()
    rng = np.random.default_rng(5)
    n, m = 48, 500
    curr = dict(x=rng.uniform(200, 440, n).astype(np.float32), y=rng.uniform(150, 330, n).astype(np.float32),
                octave=rng.integers(0, 3, n).astype(np.int32), angle=rng.uniform(0, 360, n).astype(np.float32),
                desc=synth.rand_desc(rng, n))
    src = rng.integers(0, n, m)
    lvl = np.clip(curr["octave"][src] + rng.integers(-1, 2, m), 0, 7).astype(np.int32)
    qq = dict(qx=(curr["x"][src] + rng.normal(0, 3, m)).astype(np.float32), qy=(curr["y"][src] + rng.normal(0, 3, m)).astype(np.float32),
              qxr=np.zeros(m, np.float32), qradius=(np.float32(20.0) * sf[lvl].astype(np.float32)).astype(np.float32),
              qmin=lvl - 1, qmax=lvl + 1, qangle=rng.uniform(0, 360, m).astype(np.float32),
              qdesc=synth.flip_bits(rng, curr["desc"][src], rng.integers(0, 40, m)), qvalid=np.ones(m, np.uint8))
    # sequential reference of the no-ratio path: best unclaimed candidate per query in index order (projection.cc:294-335)
    claimed = np.zeros(n, bool)
    want = np.full(n, -1, np.int32)
    order = np.lexsort((np.arange(n), np.floor(curr["y"] * grid.inv_cell_height).astype(int), np.floor(curr["x"] * grid.inv_cell_width).astype(int)))
    for q in range(m):
        best, best_i = 256, -1
        for i in order:
            if claimed[i] or not (qq["qmin"][q] <= curr["octave"][i] <= qq["qmax"][q]):
                continue
            if not (abs(curr["x"][i] - qq["qx"][q]) < qq["qradius"][q] and abs(curr["y"][i] - qq["qy"][q]) < qq["qradius"][q]):
                continue
            d = int(np.unpackbits(curr["desc"][i] ^ qq["qdesc"][q]).sum())
            if d < best:
                best, best_i = d, i
        if best_i >= 0 and best <= 100:
            claimed[best_i] = True
            want[best_i] = q
    _, matched, num = _emu_point_match(pmatch_emu, grid, curr, qq, 0, 0.0, 0)
    assert np.array_equal(matched, want) and num == int((want >= 0).sum()) and num >= 40


# ---------------------------------------------------------------------------------------------------------------------
# LSD region growing (csrc/lsd_grow_kernels.cuh): the one-warp kernel, the multi-warp round protocol and the out-of-order
# variant (tickets, reorder buffer, in-order commit, claim bitmap) on the host.  The warps of the multi-warp variants are
# real concurrent host threads here, so their locks and the commit order are exercised; all three must reproduce the
# oracle's segments bit for bit, in detection order.
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lsdgrow_emu(tmp_path_factory):
    return emu_build.emu("lsdgrow_emu", tmp_path_factory, opt="-O1")


def _lsd_grow_inputs(orc, img):
    """The half-resolution image and the seed list (y << 16 | x, gradient order) the region growing kernels start from."""
    import math
    import oracle_api
    scaled = np.ascontiguousarray(orc.lsd_scaled(img))
    sh, sw = scaled.shape
    ang, g2 = np.zeros((sh, sw), np.float32), np.zeros((sh, sw), np.int32)
    bins, order = np.zeros((sh, sw), np.int32), np.zeros(sh * sw, np.int32)
    cfg = oracle_api.OLsdCfg(*oracle_api.LSD_DET)
    P = C.c_void_p
    n = orc.lib.orc_lsd_ll_angle(scaled.ctypes.data_as(P), C.c_int(sw), C.c_int(sh), C.byref(cfg), ang.ctypes.data_as(P),
                                 g2.ctypes.data_as(P), bins.ctypes.data_as(P), order.ctypes.data_as(P))
    order = order[:n]
    rho = 2.0 / math.sin(math.pi * 22.5 / 180)   # lsd.cpp: quant / sin(prec)
    k = int(math.floor(4 * rho * rho)) + 2
    while k > 0 and not (math.sqrt(k / 4.0) <= rho):
        k -= 1
    o = order[g2.ravel()[order] > k]             # pixels whose level-line angle is defined
    return scaled, ((o // sw).astype(np.uint32) << 16 | (o % sw).astype(np.uint32)).astype(np.uint32)


@pytest.mark.parametrize("variant,warps", [(1, 1), (2, 4), (3, 4), (3, 6)])
def test_lsd_region_growing_variants_equal_oracle(lsdgrow_emu, variant, warps):
    import oracle_api
    import synth
    orc = oracle_api.Oracle()
    img = synth.make_line_image(3, 96, 160)
    scaled, oxy = _lsd_grow_inputs(orc, img)
    ref = orc.lsd_detect(img)
    cap = 4000
    segs, nseg, status, stat = np.zeros((cap, 4), np.float32), C.c_int(0), C.c_int(0), (C.c_ulonglong * 8)()
    P = C.c_void_p
    r = lsdgrow_emu.emu_lsd_grow(C.c_int(variant), C.c_int(warps), scaled.ctypes.data_as(P), C.c_int(scaled.shape[1]),
                                 C.c_int(scaled.shape[0]), oxy.ctypes.data_as(P), C.c_int(len(oxy)), segs.ctypes.data_as(P),
                                 C.c_int(cap), C.byref(nseg), C.byref(status), stat)
    assert r == 0 and status.value == 0
    assert nseg.value == len(ref) and len(ref) > 50
    assert np.array_equal(segs[:nseg.value], ref), "segments differ from the sequential detector"
    if variant == 3:
        assert stat[0] >= len(ref)  # tickets


# ---------------------------------------------------------------------------------------------------------------------
# Bundle adjustment (csrc/ba_lm_kernels.cuh): the decide / linearize / reduce / solve / update / classify kernels run whole
# local-BA solves on the host (tests/cta_emu/ba_emu.cc restates the LM try loop of ba_host.cu around them) and must follow the
# oracle try for try.  This is how the read-after-write race on BaState::phase in the solve / decide kernels was found.
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ba_emu(tmp_path_factory):
    return emu_build.emu("ba_emu", tmp_path_factory, opt="-O1")


def _emu_ba_solve(emu, prob, first=5, second=10, mode=0, ctas=3):
    import synth
    P = C.c_void_p
    p = lambda a: np.ascontiguousarray(a).ctypes.data_as(P)
    n_kf, n_pts, n_l = len(prob.kf_fixed), len(prob.pt_pos_w), len(prob.line_plucker)
    kf, pts, ln = np.zeros((n_kf, 4, 4)), np.zeros((max(n_pts, 1), 3)), np.zeros((max(n_l, 1), 6))
    po, lo = np.zeros(max(len(prob.pt_edge_kf), 1), np.uint8), np.zeros(max(len(prob.line_edge_kf), 1), np.uint8)
    it = np.zeros(3, np.int32)
    r = emu.emu_ba_solve(
        C.c_double(synth.FX), C.c_double(synth.FY), C.c_double(synth.CX), C.c_double(synth.CY),
        C.c_double(synth.BF if prob.stereo else -1.0), C.c_int(1 if prob.stereo else 0), C.c_int(n_kf), p(prob.kf_pose_cw),
        p(prob.kf_fixed), C.c_int(n_pts), p(prob.pt_pos_w), C.c_int(len(prob.pt_edge_kf)), p(prob.pt_edge_kf), p(prob.pt_edge_lm),
        p(prob.pt_edge_obs), p(prob.pt_edge_inv_sigma_sq), C.c_int(n_l), p(prob.line_plucker), C.c_int(len(prob.line_edge_kf)),
        p(prob.line_edge_kf), p(prob.line_edge_lm), p(prob.line_edge_obs), p(prob.line_edge_inv_sigma_sq),
        C.c_int(len(prob.plane_edge_lm)), p(prob.plane_edge_lm), p(prob.plane_edge_fn), C.c_int(first), C.c_int(second), C.c_int(mode),
        C.c_int(ctas), kf.ctypes.data_as(P), pts.ctypes.data_as(P), ln.ctypes.data_as(P), po.ctypes.data_as(P), lo.ctypes.data_as(P),
        it.ctypes.data_as(P))
    assert r == 0
    return kf, pts[:n_pts], ln[:n_l], po[:len(prob.pt_edge_kf)], lo[:len(prob.line_edge_kf)], tuple(int(v) for v in it)


def _ba_long_tracks(seed, n_free, n_fixed, lines=True, **kw):
    """<= 8 free keyframes and enough fixed ones for points with 33 and 65 edges: the second and third round of the point loop
    of ba_linearize_kernel (lane = edge, 32 edges per round) and of the edge strides of ba_update_kernel, lines with 40
    edges, landmarks with only fixed observers (no pool entry), 2-observation landmarks, plane edges on long tracks."""
    import ba_data
    n_kf = n_free + n_fixed
    prob = ba_data.make_ba_shape_problem(
        seed, n_free, n_fixed,
        points=[dict(n=2, k=33), dict(n=2, k=65), dict(n=1, k="all"), dict(n=2, k=64, plane=True), dict(n=2, k=32),
                dict(n=2, k=4, who="fixed"), dict(n=2, k=2), dict(n=2, k=34, who="one_free"), dict(n=24, k=(3, 9))],
        lines=[dict(n=2, k=40), dict(n=1, k=3, who="fixed"), dict(n=5, k=(3, 9))] if lines else (), **kw)
    sh = prob.shape
    assert list(sh["pt_deg"][:15]) == [33, 33, 65, 65, n_kf - len(kw.get("empty_free", ())), 64, 64, 32, 32, 4, 4, 2, 2, 34, 34]
    assert list(sh["pt_free_deg"][9:11]) == [0, 0] and list(sh["pt_free_deg"][13:15]) == [1, 1]
    assert not lines or (list(sh["ln_deg"][:3]) == [40, 40, 3] and sh["ln_free_deg"][2] == 0)
    return prob


_BA_EMU_CASES = {
    "pt33_pt65_ln40_6free_64fixed": lambda: _ba_long_tracks(5, 6, 64),
    "pt33_pt65_points_only": lambda: _ba_long_tracks(7, 6, 64, lines=False),
    "pt33_pt65_stereo_mixed_8free_62fixed_one_empty": lambda: _ba_long_tracks(6, 8, 62, stereo_frac=0.6, empty_free=(7,)),
}


def _emu_solve_equals_oracle(ba_emu, prob, ctas, first=5, second=10):
    import ba_data
    import oracle_api
    orc = oracle_api.Oracle()
    o = ba_data.oracle_local_ba(orc, prob, num_first=first, num_second=second)
    kf, pts, ln, po, lo, it = _emu_ba_solve(ba_emu, prob, first=first, second=second, ctas=ctas)
    assert it == (o.iters_first, o.iters_second, o.lm_tries)                       # same LM path, try for try
    assert np.linalg.norm(kf - o.kf_pose_cw) / np.linalg.norm(o.kf_pose_cw) < 1e-6
    assert np.abs(pts - o.pt_pos_w).max() < 1e-5
    assert np.abs(ln - o.line_plucker[:len(ln)]).max() < 1e-3                      # numeric line Jacobians (delta = 1e-9)
    assert np.array_equal(po, o.pt_edge_outlier[:len(po)]) and np.array_equal(lo, o.line_edge_outlier[:len(lo)])


def test_local_ba_kernels_equal_oracle(ba_emu):
    import ba_data
    prob = ba_data.make_ba_problem(3, n_local=4, n_fixed=2, n_points=60, n_lines=12, n_plane_pts=6)
    _emu_solve_equals_oracle(ba_emu, prob, ctas=3)


@pytest.mark.parametrize("case,ctas", [("pt33_pt65_ln40_6free_64fixed", 3), ("pt33_pt65_stereo_mixed_8free_62fixed_one_empty", 2)])
def test_local_ba_kernels_equal_oracle_on_long_tracks(ba_emu, case, ctas):
    """The same comparison on the shapes make_ba_problem cannot draw (see _ba_long_tracks): every point loop of the
    linearisation and of the back-substitution takes more than one round of 32 edges.  optimize(3), the outlier round,
    optimize(5): every kernel and both phases at half the emulation time of the full 5 + 10 iterations."""
    _emu_solve_equals_oracle(ba_emu, _BA_EMU_CASES[case](), ctas, first=3, second=5)


@pytest.mark.parametrize("case,ctas,tol", [("pt33_pt65_ln40_6free_64fixed", 3, 1e-5), ("pt33_pt65_points_only", 1, 1e-13)])
def test_local_ba_first_try_matches_full_normal_equations(ba_emu, case, ctas, tol):
    """The reduced camera system S, g, chi2 and lambda of the first real try, as ba_linearize_kernel / ba_reduce_kernel leave
    them, against the Schur complement of tests/ba_numpy.py's full normal equations in long double (lines: numeric
    Jacobians with delta = 1e-9 on both sides, hence 1e-5), and the step of ba_solve_kernel by its backward error."""
    import ba_system_ref as ref
    prob = _BA_EMU_CASES[case]()
    n_free = int((prob.kf_fixed == 0).sum())
    n_pairs = n_free * (n_free + 1) // 2
    packed, dp, lam = np.zeros(n_pairs * 36 + 12 * n_free + 1), np.zeros(6 * n_free), C.c_double(0.0)
    ba_emu.emu_ba_capture_try(packed.ctypes.data_as(_P), dp.ctypes.data_as(_P), C.byref(lam))
    _emu_ba_solve(ba_emu, prob, first=1, second=0, mode=1, ctas=ctas)
    nS = n_pairs * 36
    got = dict(S=packed[:nS].reshape(n_pairs, 6, 6), g=packed[nS:nS + 6 * n_free], bp=packed[nS + 6 * n_free:nS + 12 * n_free],
               chi2=float(packed[-1]), dp=dp, lam=lam.value)
    ref.check_system(got, prob, n_free, tol)
    assert np.abs(dp).max() > 1e-4
    assert ref.backward_error(ref.dense_from_blocks(got["S"], n_free), got["g"], dp, lam.value) < 5e-17
