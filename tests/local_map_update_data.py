"""The local-map update of tracking (tracking_module::update_local_map, tracking_module.cc:837-906, and
module::local_map_updater, local_map_updater.cc), restated in Python, and the map snapshots (plp_track_map) it reads.

The restatement walks the voted keyframes in ascending table index: the reference walks them in the iteration order of
an unordered_map keyed by pointer, which the device replaces by that canonical order (DESIGN.md §3.17).  The C++
restatement in oracle/local_map_update_oracle.cc must give the same lists; the tests check both against each other and
against the device code."""
from __future__ import annotations

import ctypes as C

import numpy as np

import local_map_data as lmd
import oracle_api

ROOT = lmd.ROOT
MAX_NUM_LOCAL_KEYFRMS = 60   # tracking_module.cc:873
WEIGHT_THR = 15              # graph_node::weight_thr_ (graph_node.h)
TOP_N_COV = 10               # local_map_updater.cc:179
_P = C.c_void_p


# ---- the Python restatement ------------------------------------------------------------------------------------------
def _span(offsets, items, i):
    return [int(x) for x in items[offsets[i]:offsets[i + 1]]]


def update_local_map(snap, tracked_lm):
    """update_local_map for one frame whose keypoints hold the landmarks tracked_lm (-1: none).  -> None when no keyframe
    voted (acquire_local_map fails and the previous local map stays), else dict(local_kf, nearest (-1: none), local_lm,
    num_voted)."""
    lm_erased, kf_erased = np.asarray(snap["lm_erased"]), np.asarray(snap["kf_erased"])
    weights = {}
    for lm in tracked_lm:  # the clean-up (:840-852), then count_keyframe_weights (:89-108)
        lm = int(lm)
        if lm < 0 or lm_erased[lm]:
            continue
        for kf in _span(snap["obs_offsets"], snap["obs_kf"], lm):
            weights[kf] = weights.get(kf, 0) + 1
    if not weights:
        return None
    first, nearest, max_weight = [], -1, 0
    for kf in sorted(weights):  # find_first_local_keyframes (:110-141) in the canonical order
        if kf_erased[kf]:
            continue
        first.append(kf)
        if max_weight < weights[kf]:
            max_weight, nearest = weights[kf], kf
    taken, second = set(first), []

    def add(kf):  # add_second_local_keyframe (:150-168)
        if kf < 0 or kf_erased[kf] or kf in taken:
            return False
        taken.add(kf)
        second.append(kf)
        return True

    for kf in first:  # find_second_local_keyframes (:169-201)
        if MAX_NUM_LOCAL_KEYFRMS < len(first) + len(second):
            break
        for nb in _span(snap["cov_offsets"], snap["cov_kf"], kf):
            if add(nb):
                break
        for ch in _span(snap["child_offsets"], snap["child_kf"], kf):
            if add(ch):
                break
        add(int(snap["parent"][kf]))
    local_kf = first + second
    seen, local_lm = set(), []
    for kf in local_kf:  # find_local_landmarks (:206-238)
        for lm in _span(snap["row_offsets"], snap["row_lm"], kf):
            if lm < 0 or lm_erased[lm] or lm in seen:
                continue
            seen.add(lm)
            local_lm.append(lm)
    return dict(local_kf=local_kf, nearest=nearest, local_lm=local_lm, num_voted=len(weights))


def device_update(snap, tracked_lm, max_local, max_local_kf, active=True):
    """What plp_tracker_update_local_map_batch_dev gives one frame: dict(status, nearest, local_kf, local_lm); status 1 /
    2 / 3 (and an inactive frame) with empty lists and nearest -1."""
    empty = dict(nearest=-1, local_kf=[], local_lm=[])
    if not active:
        return dict(status=0, **empty)
    r = update_local_map(snap, tracked_lm)
    if r is None:
        return dict(status=3, **empty)
    if r["num_voted"] > max_local_kf:
        return dict(status=2, **empty)
    if len(r["local_lm"]) > max_local:
        return dict(status=1, **empty)
    return dict(status=0, nearest=r["nearest"], local_kf=r["local_kf"], local_lm=r["local_lm"])


def mapping(local_lm, row_lm):
    """The local index of each row's landmark, or -1 (last_local_idx / local_idx)."""
    pos = {lm: j for j, lm in enumerate(local_lm)}
    return np.array([pos.get(int(lm), -1) for lm in row_lm], np.int32)


def local_rows(snap, local_lm):
    """The plp_track_local rows of a local list (local_map_data's field names)."""
    idx = np.asarray(local_lm, np.int64)
    return dict(pos_w=np.asarray(snap["pos_w"]).reshape(-1, 3)[idx], normal=np.asarray(snap["normal"]).reshape(-1, 3)[idx],
                min_valid_dist=np.asarray(snap["min_valid_dist"])[idx], max_valid_dist=np.asarray(snap["max_valid_dist"])[idx],
                max_valid_dist_raw=np.asarray(snap["max_valid_dist_raw"])[idx],
                desc=np.asarray(snap["desc"]).reshape(-1, 32)[idx], valid=np.ones(len(idx), np.uint8))


# ---- the C++ restatement ---------------------------------------------------------------------------------------------
def _i32(a):
    return np.ascontiguousarray(a, np.int32)


def oracle_update(snap, tracked_lm):
    """oracle/local_map_update_oracle.cc on one frame; the same result as update_local_map (None: no keyframe voted)."""
    K, L = len(snap["kf_erased"]), len(snap["lm_erased"])
    arrs = [_i32(tracked_lm), np.ascontiguousarray(snap["lm_erased"], np.uint8), _i32(snap["obs_offsets"]),
            _i32(snap["obs_kf"]), np.ascontiguousarray(snap["kf_erased"], np.uint8), _i32(snap["row_offsets"]),
            _i32(snap["row_lm"]), _i32(snap["cov_offsets"]), _i32(snap["cov_kf"]), _i32(snap["child_offsets"]),
            _i32(snap["child_kf"]), _i32(snap["parent"])]
    out_kf = np.zeros(max(K, 1), np.int32)
    out_lm = np.zeros(max(L, 1), np.int32)
    n = np.zeros(4, np.int32)  # num_local_kf, num_local_lm, nearest, num_voted
    ok = oracle_api.lib().lmuo_update_local_map(C.c_int(len(tracked_lm)), C.c_int(K), C.c_int(L),
                                                *[a.ctypes.data_as(_P) for a in arrs], out_kf.ctypes.data_as(_P),
                                                out_lm.ctypes.data_as(_P), n.ctypes.data_as(_P))
    if not ok:
        return None
    return dict(local_kf=[int(x) for x in out_kf[:n[0]]], nearest=int(n[2]), local_lm=[int(x) for x in out_lm[:n[1]]],
                num_voted=int(n[3]))


# ---- map snapshots ---------------------------------------------------------------------------------------------------
def csr(lists, dtype=np.int32):
    off = np.zeros(len(lists) + 1, np.int32)
    off[1:] = np.cumsum([len(x) for x in lists])
    flat = np.concatenate([np.asarray(x, dtype) for x in lists]) if lists and off[-1] else np.zeros(0, dtype)
    return off, np.ascontiguousarray(flat, dtype)


def graph(rows_of_kf, n_lm):
    """Observations, covisibilities and a spanning tree from the keyframes' rows (landmark per row, -1: none), keyframes in
    keyframe::id_ order.  Covisibility: graph_node::update_connections (graph_node.cc:120-216): the keyframes sharing
    landmarks, those with weight above 15 (the strongest when none is), ordered by descending (weight, keyframe) -- the
    pointer order of the reference's sort taken as id order -- and the first 10 of them.  Spanning parent: the strongest
    connection among the earlier keyframes (the first keyframe has none); children in id order (a std::set of pointers)."""
    K = len(rows_of_kf)
    obs = [[] for _ in range(n_lm)]
    for k, rows in enumerate(rows_of_kf):
        for lm in dict.fromkeys(int(x) for x in rows if x >= 0):
            obs[lm].append(k)
    cov, parent = [], np.full(K, -1, np.int32)
    for k, rows in enumerate(rows_of_kf):
        w = {}
        for lm in set(int(x) for x in rows if x >= 0):
            for j in obs[lm]:
                if j != k:
                    w[j] = w.get(j, 0) + 1
        pairs = [(wt, j) for j, wt in w.items() if WEIGHT_THR < wt]
        if not pairs and w:
            pairs = [max((wt, j) for j, wt in w.items())]
        pairs.sort(reverse=True)
        cov.append([j for _, j in pairs[:TOP_N_COV]])
        earlier = [(wt, j) for j, wt in w.items() if j < k]
        if earlier:
            parent[k] = max(earlier)[1]
    children = [[j for j in range(K) if parent[j] == k] for k in range(K)]
    obs_off, obs_kf = csr(obs)
    cov_off, cov_kf = csr(cov)
    ch_off, ch_kf = csr(children)
    row_off, row_lm = csr(rows_of_kf)
    return dict(obs_offsets=obs_off, obs_kf=obs_kf, cov_offsets=cov_off, cov_kf=cov_kf, child_offsets=ch_off,
                child_kf=ch_kf, parent=parent, row_offsets=row_off, row_lm=row_lm, kf_erased=np.zeros(K, np.uint8))


def random_geometry(n_lm, rng):
    """Landmark fields for snapshots whose geometry the update does not read."""
    return dict(pos_w=rng.normal(size=(n_lm, 3)), normal=rng.normal(size=(n_lm, 3)),
                min_valid_dist=rng.random(n_lm).astype(np.float32), max_valid_dist=(1 + rng.random(n_lm)).astype(np.float32),
                max_valid_dist_raw=rng.random(n_lm).astype(np.float32),
                desc=rng.integers(0, 256, (n_lm, 32), dtype=np.uint8), lm_erased=np.zeros(n_lm, np.uint8))


def band_map(n_kf, rows_per_kf, rng, reach=3, share=0.5, null_frac=0.05):
    """A keyframe trajectory: keyframe k's rows hold its own new landmarks and, with probability `share`, landmarks of the
    `reach` keyframes before it (so covisibility is a band along the trajectory).  -> (rows_of_kf, n_lm)."""
    rows_of_kf, own = [], []
    n_lm = 0
    for k in range(n_kf):
        mine = list(range(n_lm, n_lm + rows_per_kf))
        n_lm += rows_per_kf
        rows = []
        for i in range(rows_per_kf):
            r = rng.random()
            if r < null_frac:
                rows.append(-1)
            elif r < null_frac + share and k > 0:
                j = int(rng.integers(max(0, k - reach), k))
                rows.append(int(rng.choice(own[j])))
            else:
                rows.append(mine[i])
        own.append(mine)
        rows_of_kf.append(rows)
    return rows_of_kf, n_lm


def synthetic_snapshot(n_kf, rows_per_kf, rng, **kw):
    rows, n_lm = band_map(n_kf, rows_per_kf, rng, **kw)
    snap = graph(rows, n_lm)
    snap.update(random_geometry(n_lm, rng))
    return snap


def scene_snapshot(seq, res, n_kf, rng, share=0.4, undistort=None):
    """A snapshot along a scene.PlanarSequence: keyframe k is frame k (k < n_kf); landmark (k, i) is created from frame k's
    keypoint i (local_map_data.landmark_rows), and keyframe k's rows hold its own landmarks or, with probability
    `share`, the same-index landmark of one of the two keyframes before it.  -> (snapshot, lm_id) with lm_id[k][i] the
    index of landmark (k, i)."""
    base, parts, lm_id = 0, [], []
    for k in range(n_kf):
        kps = lmd._kps(res[k], undistort)
        parts.append(lmd.landmark_rows(seq, k, kps, res[k]["desc"], [j for j in (k - 1, k) if j >= 0]))
        lm_id.append(np.arange(base, base + len(kps["x"]), dtype=np.int32))
        base += len(kps["x"])
    rows_of_kf = []
    for k in range(n_kf):
        rows = lm_id[k].copy()
        for i in range(len(rows)):
            if k > 0 and rng.random() < share:
                j = int(rng.integers(max(0, k - 2), k))
                if i < len(lm_id[j]):
                    rows[i] = lm_id[j][i]
        rows_of_kf.append(rows)
    snap = graph(rows_of_kf, base)
    geo = lmd.concat(parts)
    snap.update(pos_w=geo["pos_w"], normal=geo["normal"], min_valid_dist=geo["min_valid_dist"],
                max_valid_dist=geo["max_valid_dist"], max_valid_dist_raw=geo["max_valid_dist_raw"], desc=geo["desc"],
                lm_erased=np.zeros(base, np.uint8))
    return snap, lm_id


# ---- bench.py's headline batch with a map snapshot ---------------------------------------------------------------------
BENCH_KEYFRAMES = 128
BENCH_MAX_LKF = 128
BENCH_MAX_LOCAL = 8192


def bench_snapshot(lasts, rng, n_kf=BENCH_KEYFRAMES, rows_per_kf=600):
    """A band-shaped snapshot of n_kf keyframes (synthetic geometry) whose landmarks the frames' last rows hold: frame
    b's rows take the landmarks of four consecutive keyframes starting at a frame-dependent keyframe."""
    snap = synthetic_snapshot(n_kf, rows_per_kf, rng, reach=3, share=0.5)
    ro, rl = snap["row_offsets"], snap["row_lm"]
    last_lm = []
    for b, last in enumerate(lasts):
        k0 = (7 * b) % (n_kf - 4)
        pool = np.array([int(x) for x in rl[ro[k0]:ro[k0 + 4]] if x >= 0], np.int32)
        last_lm.append(pool[rng.integers(0, len(pool), len(last["octave"]))])
    snap["last_row_lm"] = np.concatenate(last_lm).astype(np.int32)
    return snap


def bench_setup(pkg, ctx, batch=512, seed=1234, track_ctx=None):
    """bench.setup_front_end plus the local-map and update reservations and a map snapshot (bench_snapshot).
    -> (fe, snap, aux)."""
    import sys
    sys.path.insert(0, str(ROOT))
    import bench
    fe, frames, aux = bench.setup_front_end(pkg, ctx, batch, seed, track_ctx)
    fe.reserve_local_map(BENCH_MAX_LOCAL)
    fe.reserve_local_map_update(BENCH_MAX_LKF)
    snap = bench_snapshot(aux["lasts"], np.random.default_rng(seed + 7))
    fe.set_map(snap)
    for cx in {id(ctx): ctx, id(fe.track_ctx): fe.track_ctx}.values():
        cx.sync()
    return fe, snap, aux


def oracle_update_batch(snap, n_kp, matched, num_valid, last_offsets, max_local):
    """oracle/local_map_update_oracle.cc's lmuo_update_batch: the native host walk of a motion-tracked batch (matched:
    batch x cap last-frame rows).  -> (offsets, local landmarks per row of the concatenated lists, last_local_idx)."""
    B, cap = matched.shape
    K, L = len(snap["kf_erased"]), len(snap["lm_erased"])
    offs = np.zeros(B + 1, np.int32)
    out_lm = np.zeros(B * max_local, np.int32)
    lli = np.zeros(max(int(last_offsets[B]), 1), np.int32)
    arrs = [_i32(n_kp), _i32(matched), _i32(num_valid), _i32(last_offsets), _i32(snap["last_row_lm"]),
            np.ascontiguousarray(snap["lm_erased"], np.uint8), _i32(snap["obs_offsets"]), _i32(snap["obs_kf"]),
            np.ascontiguousarray(snap["kf_erased"], np.uint8), _i32(snap["row_offsets"]), _i32(snap["row_lm"]),
            _i32(snap["cov_offsets"]), _i32(snap["cov_kf"]), _i32(snap["child_offsets"]), _i32(snap["child_kf"]),
            _i32(snap["parent"]), offs, out_lm, lli]
    oracle_api.lib().lmuo_update_batch(C.c_int(B), C.c_int(cap), C.c_int(K), C.c_int(L), C.c_int(max_local),
                                       *[a.ctypes.data_as(_P) for a in arrs])
    lm = np.concatenate([out_lm[b * max_local:b * max_local + offs[b + 1] - offs[b]] for b in range(B)])
    return offs, lm, lli[:int(last_offsets[B])]
