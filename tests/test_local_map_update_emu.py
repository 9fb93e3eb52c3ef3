"""The local-map update's DEVICE code (structure-plp-slam_b200/csrc/local_map_update_kernels.cuh) executed on the CPU
through tests/cta_emu, equal to the Python restatement of update_local_map (tests/local_map_update_data.py), which in
turn equals the C++ restatement (oracle/local_map_update_oracle.cc) list for list.  Batches mix motion-, keyframe- and
robust-started frames, inactive frames and frames with every status, over band-shaped maps with erased landmarks and
keyframes, shared landmarks, weight ties, first levels above 60 and lists ending at 61-63."""
import ctypes as C

import numpy as np
import pytest

import emu_build
import local_map_update_data as lmu

_P = C.c_void_p
CAP = 96
_REC_FIELDS = ("stage", "status", "matched", "pose", "num_valid", "n_obs", "obs_row", "pos_w", "offsets", "of_frame",
               "local_idx", "local_idx_offsets")
_MAP_FIELDS = ("pos_w", "normal", "min_valid_dist", "max_valid_dist", "max_valid_dist_raw", "desc", "lm_erased",
               "obs_offsets", "obs_kf", "kf_erased", "row_offsets", "row_lm", "cov_offsets", "cov_kf", "child_offsets",
               "child_kf", "parent", "last_row_lm", "kf_row_lm")
_MAP_DT = dict(pos_w=np.float64, normal=np.float64, min_valid_dist=np.float32, max_valid_dist=np.float32,
               max_valid_dist_raw=np.float32, desc=np.uint8, lm_erased=np.uint8, kf_erased=np.uint8)


class _EmuRecord(C.Structure):  # tests/cta_emu/lmupdate_emu.cc
    _fields_ = [(f, _P) for f in _REC_FIELDS]


class _Map(C.Structure):  # plp_track_map
    _fields_ = [(f, _P) for f in _MAP_FIELDS]


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return emu_build.emu("lmupdate_emu", tmp_path_factory)


def _a(x, dt):
    return np.ascontiguousarray(x, dt)


def _frame_rows(tracked, extra, rng):
    """A row block holding the tracked landmarks (shuffled) and `extra` rows; -> (row_lm, matched per keypoint)."""
    held = sorted(set(int(l) for l in tracked if l >= 0))
    rows = np.array(held + list(extra), np.int32)
    perm = rng.permutation(len(rows))
    rows = rows[perm]
    pos = {}
    for r, lm in enumerate(rows):
        pos.setdefault(int(lm), r)
    matched = np.array([pos[int(l)] if l >= 0 else -1 for l in tracked], np.int32)
    return rows, matched


def run_batch(emu, snap, frames, max_local, max_lkf, rng):
    """frames[b] = dict(kind 'motion' | 'kf' | 'rb', tracked (landmark per keypoint, -1: none), optional num_valid,
    kf_status).  Runs the emulated update and returns (outputs, expected)."""
    B = len(frames)
    last_rows, kf_rows = [], []
    rec = {s: dict(stage=np.zeros(B, np.int32), status=np.zeros(B, np.int32), matched=np.full((B, CAP), -1, np.int32),
                   num_valid=np.zeros(B, np.int32)) for s in ("motion", "kf", "rb")}
    n_kp = np.zeros(B, np.int32)
    L = len(snap["lm_erased"])
    for b, f in enumerate(frames):
        tr = np.asarray(f["tracked"], np.int32)
        n_kp[b] = len(tr)
        extra = list(rng.integers(0, L, 5)) + [-1, -1]
        nv = f.get("num_valid", int((tr >= 0).sum()))
        rows, m = _frame_rows(tr, extra, rng)
        if f["kind"] == "motion":
            last_rows.append(rows)
            kf_rows.append(np.array(list(rng.integers(0, L, 4)), np.int32))
            rec["motion"]["matched"][b, :len(m)] = m
            rec["motion"]["num_valid"][b] = nv
        else:
            last_rows.append(np.array(list(rng.integers(0, L, 6)) + [-1], np.int32))
            kf_rows.append(rows)
            rec["kf"]["stage"][b] = 1
            rec["kf"]["status"][b] = f.get("kf_status", 0)
            if f["kind"] == "kf":
                rec["kf"]["matched"][b, :len(m)] = m
                rec["kf"]["num_valid"][b] = nv
            else:
                rec["rb"]["stage"][b] = 1
                rec["rb"]["status"][b] = f.get("kf_status", 0)
                rec["rb"]["matched"][b, :len(m)] = m
                rec["rb"]["num_valid"][b] = nv
    last_off, last_lm = lmu.csr(last_rows)
    # keyframe table: frame b's keyframe is table entry B - 1 - b (kf_of_frame is a real indirection)
    order = list(range(B - 1, -1, -1))
    kf_off, kf_lm = lmu.csr([kf_rows[b] for b in order])
    kf_of_frame = _a([order.index(b) for b in range(B)], np.int32)
    keep = []
    recs = []
    for s, offs, of in (("motion", last_off, None), ("kf", kf_off, kf_of_frame), ("rb", kf_off, kf_of_frame)):
        r = rec[s]
        arrs = dict(stage=r["stage"] if s != "motion" else None, status=r["status"] if s != "motion" else None,
                    matched=r["matched"], num_valid=r["num_valid"], offsets=offs, of_frame=of)
        keep.append(arrs)
        recs.append(_EmuRecord(**{k: (v.ctypes.data_as(_P) if v is not None else None) for k, v in arrs.items()}))
    recs = (_EmuRecord * 3)(*recs)
    snap = dict(snap, last_row_lm=last_lm, kf_row_lm=kf_lm)
    marr = {k: _a(snap[k], _MAP_DT.get(k, np.int32)) for k in _MAP_FIELDS}
    cmap = _Map(**{k: v.ctypes.data_as(_P) for k, v in marr.items()})
    max_kf_rows = int(np.diff(kf_off).max())
    out = dict(nearest=np.zeros(B, np.int32), local_kf=np.zeros((B, max_lkf), np.int32), num_local_kf=np.zeros(B, np.int32),
               local_lm=np.full(B * max_local, -5, np.int32), status=np.zeros(B, np.int32),
               pos_w=np.zeros((B * max_local, 3)), normal=np.zeros((B * max_local, 3)),
               min_d=np.zeros(B * max_local, np.float32), max_d=np.zeros(B * max_local, np.float32),
               max_raw=np.zeros(B * max_local, np.float32), desc=np.zeros((B * max_local, 32), np.uint8),
               valid=np.zeros(B * max_local, np.uint8), offsets=np.zeros(B + 1, np.int32),
               last_local_idx=np.full(int(last_off[-1]), -9, np.int32),
               local_idx=np.full(B * max_kf_rows, -9, np.int32), local_idx_offsets=np.zeros(B + 1, np.int32))
    order_out = ["nearest", "local_kf", "num_local_kf", "local_lm", "status", "pos_w", "normal", "min_d", "max_d",
                 "max_raw", "desc", "valid", "offsets", "last_local_idx", "local_idx", "local_idx_offsets"]
    emu.emu_lmu_run(C.c_int(B), C.c_int(CAP), C.c_int(max_local), C.c_int(max_lkf), n_kp.ctypes.data_as(_P), recs,
                    last_off.ctypes.data_as(_P), kf_of_frame.ctypes.data_as(_P), kf_off.ctypes.data_as(_P),
                    C.byref(cmap), *[out[k].ctypes.data_as(_P) for k in order_out])
    # what the device must give
    wants = []
    for b, f in enumerate(frames):
        tr = np.asarray(f["tracked"], np.int32)
        nv = f.get("num_valid", int((tr >= 0).sum()))
        active = nv >= 20 and f.get("kf_status", 0) == 0
        w = lmu.device_update(snap, tr, max_local, max_lkf, active)
        if active:  # the Python and C++ restatements agree list for list
            p, c = lmu.update_local_map(snap, tr), lmu.oracle_update(snap, tr)
            assert p == c, b
        w["last_local_idx"] = lmu.mapping(w["local_lm"], last_rows[b]) if w["status"] == 0 else \
            np.full(len(last_rows[b]), -1, np.int32)
        kf_block = f["kind"] != "motion" and f.get("kf_status", 0) == 0
        w["local_idx"] = (lmu.mapping(w["local_lm"], kf_rows[b]) if w["status"] == 0 else
                          np.full(len(kf_rows[b]), -1, np.int32)) if kf_block else np.zeros(0, np.int32)
        wants.append(w)
    return out, wants, dict(last_off=last_off, snap=snap)


def check(out, wants, ctx):
    snap, last_off = ctx["snap"], ctx["last_off"]
    offs, lio = out["offsets"], out["local_idx_offsets"]
    assert offs[0] == 0 and lio[0] == 0
    for b, w in enumerate(wants):
        what = f"frame {b}"
        assert out["status"][b] == w["status"], (what, out["status"][b], w["status"])
        assert out["nearest"][b] == w["nearest"], (what, out["nearest"][b], w["nearest"])
        assert list(out["local_kf"][b, :out["num_local_kf"][b]]) == w["local_kf"], what
        lm = out["local_lm"][offs[b]:offs[b + 1]]
        assert list(lm) == w["local_lm"], what
        rows = lmu.local_rows(snap, w["local_lm"])
        sl = slice(offs[b], offs[b + 1])
        assert np.array_equal(out["pos_w"][sl], rows["pos_w"]) and np.array_equal(out["normal"][sl], rows["normal"]), what
        assert np.array_equal(out["min_d"][sl], rows["min_valid_dist"]) and np.array_equal(out["max_d"][sl], rows["max_valid_dist"])
        assert np.array_equal(out["max_raw"][sl], rows["max_valid_dist_raw"]) and np.array_equal(out["desc"][sl], rows["desc"])
        assert (out["valid"][sl] == 1).all(), what
        assert np.array_equal(out["last_local_idx"][last_off[b]:last_off[b + 1]], w["last_local_idx"]), what
        assert np.array_equal(out["local_idx"][lio[b]:lio[b + 1]], w["local_idx"]), what


def _tracked_from(snap, kfs, per_kf, rng, n_none=4):
    """Tracked landmarks drawn from the rows of keyframes kfs (per_kf each), plus keypoints without a landmark."""
    ro, rl = snap["row_offsets"], snap["row_lm"]
    out = []
    for k in kfs:
        cand = [int(x) for x in rl[ro[k]:ro[k + 1]] if x >= 0]
        out += list(rng.choice(cand, min(per_kf, len(cand)), replace=False))
    out += [-1] * n_none
    return np.array(rng.permutation(out), np.int32)


def test_mixed_batch(emu):
    """Motion-, keyframe- and robust-started frames; erased landmarks among the tracked ones and in local keyframes;
    erased keyframes; inactive frames (num_valid < 20, keyframe status != 0); a weight tie; status 1 and 3."""
    rng = np.random.default_rng(1)
    snap = lmu.synthetic_snapshot(40, 60, rng, reach=4, share=0.5)
    K, L = len(snap["kf_erased"]), len(snap["lm_erased"])
    snap["lm_erased"][rng.choice(L, L // 12, replace=False)] = 1
    snap["kf_erased"][[7, 13, 22]] = 1
    single = [l for l in range(L) if snap["obs_offsets"][l + 1] - snap["obs_offsets"][l] == 1 and not snap["lm_erased"][l]]
    by_kf = {}
    for l in single:
        by_kf.setdefault(int(snap["obs_kf"][snap["obs_offsets"][l]]), []).append(l)
    a, b2 = [k for k in sorted(by_kf) if len(by_kf[k]) >= 12 and not snap["kf_erased"][k]][:2]
    tie = np.array(by_kf[a][:12] + by_kf[b2][:12] + [-1] * 3, np.int32)
    unobserved = np.full(30, -1, np.int32)
    frames = [
        dict(kind="motion", tracked=_tracked_from(snap, [10, 11, 12], 10, rng)),
        dict(kind="kf", tracked=_tracked_from(snap, [20, 21, 23], 10, rng)),
        dict(kind="rb", tracked=_tracked_from(snap, [5, 6, 7, 8], 8, rng)),
        dict(kind="motion", tracked=_tracked_from(snap, [30], 10, rng)),               # below 20: inactive
        dict(kind="kf", tracked=_tracked_from(snap, [2, 3], 15, rng), kf_status=1),    # keyframe status: inactive
        dict(kind="motion", tracked=tie),                                              # tie for the nearest keyframe
        dict(kind="rb", tracked=unobserved, num_valid=25),                             # status 3: no vote
        dict(kind="motion", tracked=_tracked_from(snap, list(range(0, 40, 3)), 3, rng)),
    ]
    # frame 6 holds landmarks no keyframe observes: a fresh landmark index past the table
    snap["obs_offsets"] = np.concatenate([snap["obs_offsets"], [snap["obs_offsets"][-1]] * 30]).astype(np.int32)
    for k in ("pos_w", "normal"):
        snap[k] = np.concatenate([snap[k], np.zeros((30, 3))])
    for k in ("min_valid_dist", "max_valid_dist", "max_valid_dist_raw"):
        snap[k] = np.concatenate([snap[k], np.zeros(30, np.float32)])
    snap["desc"] = np.concatenate([snap["desc"], np.zeros((30, 32), np.uint8)])
    snap["lm_erased"] = np.concatenate([snap["lm_erased"], np.zeros(30, np.uint8)])
    frames[6]["tracked"] = np.arange(L, L + 30, dtype=np.int32)
    out, wants, ctx = run_batch(emu, snap, frames, 2000, 64, rng)
    assert [w["status"] for w in wants] == [0, 0, 0, 0, 0, 0, 3, 0]
    assert wants[5]["nearest"] == a  # equal weights: the lower index
    assert wants[3]["local_kf"] == [] and wants[4]["local_kf"] == []
    assert 7 not in lmu.update_local_map(snap, frames[2]["tracked"])["local_kf"]  # voted, erased
    check(out, wants, ctx)
    # the same batch with a smaller list: the frames whose list exceeds it get status 1
    big = max(len(w["local_lm"]) for w in wants)
    out, wants, ctx = run_batch(emu, snap, frames, big - 1, 64, rng)
    assert 1 in [w["status"] for w in wants]
    check(out, wants, ctx)


def _level_sizes(snap, tracked):
    r = lmu.update_local_map(snap, tracked)
    voted_alive = sorted(k for k in set(int(snap["obs_kf"][o]) for l in tracked if l >= 0 and not snap["lm_erased"][l]
                                        for o in range(snap["obs_offsets"][l], snap["obs_offsets"][l + 1]))
                         if not snap["kf_erased"][k])
    return len(voted_alive), len(r["local_kf"])


def test_first_level_caps(emu):
    """First levels from a handful of keyframes up past 60: the second level stops when the list exceeds 60 at the top
    of its loop (lists of 61-63), a first level above 60 gets none, and the first level is never capped; covisibility
    lists whose first entries are already taken; erased keyframes among covisibilities, children and parents; status 2
    once the voted keyframes exceed the reservation."""
    rng = np.random.default_rng(2)
    snap = lmu.synthetic_snapshot(110, 80, rng, reach=3, share=0.7, null_frac=0.1)
    K = len(snap["kf_erased"])
    snap["kf_erased"][rng.choice(K, 8, replace=False)] = 1
    frames, sizes = [], []
    for n_first in (3, 20, 50, 56, 57, 58, 59, 60, 61, 64, 75):
        start = int(rng.integers(0, K - n_first))
        kfs = list(range(start, start + n_first))
        tr = _tracked_from(snap, kfs, 1, rng)
        frames.append(dict(kind=["motion", "kf", "rb"][len(frames) % 3], tracked=tr, num_valid=max(20, len(tr))))
        sizes.append(_level_sizes(snap, tr))
    # a frame whose first level is {k, cov(k)[0]} (landmarks only they observe): k's covisibility list starts taken
    L = len(snap["lm_erased"])
    only = {}
    for l in range(L):
        if snap["obs_offsets"][l + 1] - snap["obs_offsets"][l] == 1:
            only.setdefault(int(snap["obs_kf"][snap["obs_offsets"][l]]), []).append(l)
    k = next(k for k in range(K) if not snap["kf_erased"][k] and len(only.get(k, [])) >= 2 and
             snap["cov_offsets"][k + 1] - snap["cov_offsets"][k] >= 2 and
             len(only.get(int(snap["cov_kf"][snap["cov_offsets"][k]]), [])) >= 1 and
             not snap["kf_erased"][snap["cov_kf"][snap["cov_offsets"][k]]])
    c0 = int(snap["cov_kf"][snap["cov_offsets"][k]])
    frames.append(dict(kind="motion", tracked=np.array(only[k][:2] + only[c0][:1] + [-1] * 3, np.int32), num_valid=25))
    sizes.append(_level_sizes(snap, frames[-1]["tracked"]))
    out, wants, ctx = run_batch(emu, snap, frames, 3000, 128, rng)
    check(out, wants, ctx)
    ends = [n for f, n in sizes if f <= 60]
    assert any(61 <= n <= 63 for n in ends), sizes
    assert any(f > 60 and n == f for f, n in sizes), sizes
    # a covisibility list whose first entry is already in the list, and a later one taken
    seen = False
    for i, f in enumerate(frames):
        r = lmu.update_local_map(snap, f["tracked"])
        first = set(r["local_kf"][:sizes[i][0]])
        for k in list(first):
            cov = list(snap["cov_kf"][snap["cov_offsets"][k]:snap["cov_offsets"][k + 1]])
            if len(cov) > 1 and cov[0] in first and any(c in r["local_kf"] and c not in first for c in cov[1:]):
                seen = True
    assert seen
    # the same frames against a reservation of 64 keyframes: those voting for more get status 2
    out, wants, ctx = run_batch(emu, snap, frames, 3000, 64, rng)
    assert 2 in [w["status"] for w in wants]
    check(out, wants, ctx)


def test_restatements_agree_on_scene_snapshot():
    """The Python and C++ restatements on a snapshot built along scene.PlanarSequence-like keyframes (no GPU): many
    random tracked sets, erased landmarks and keyframes."""
    rng = np.random.default_rng(3)
    snap = lmu.synthetic_snapshot(30, 80, rng, reach=5, share=0.6)
    snap["lm_erased"][rng.choice(len(snap["lm_erased"]), 50, replace=False)] = 1
    snap["kf_erased"][[4, 9]] = 1
    for _ in range(40):
        kfs = rng.choice(30, int(rng.integers(1, 12)), replace=False)
        tr = _tracked_from(snap, kfs, int(rng.integers(1, 10)), rng)
        assert lmu.update_local_map(snap, tr) == lmu.oracle_update(snap, tr)


def test_status_2_boundary(emu):
    """A frame voting for exactly max_local_keyframes keyframes builds its list; one voting for one more gets status 2.
    Each tracked landmark has a single observer, so the voted keyframes are counted exactly."""
    rng = np.random.default_rng(4)
    snap = lmu.synthetic_snapshot(80, 40, rng, reach=3, share=0.4)
    only = {}
    for l in range(len(snap["lm_erased"])):
        if snap["obs_offsets"][l + 1] - snap["obs_offsets"][l] == 1:
            only.setdefault(int(snap["obs_kf"][snap["obs_offsets"][l]]), []).append(l)
    kfs = sorted(only)
    assert len(kfs) >= 66
    frames = []
    for n in (63, 64, 65):
        tracked = np.array([only[k][0] for k in kfs[:n]], np.int32)
        frames.append(dict(kind=["motion", "kf", "rb"][len(frames)], tracked=tracked))
    out, wants, ctx = run_batch(emu, snap, frames, 4000, 64, rng)
    assert [lmu.update_local_map(snap, f["tracked"])["num_voted"] for f in frames] == [63, 64, 65]
    assert [w["status"] for w in wants] == [0, 0, 2]
    check(out, wants, ctx)


def test_batch_host_walk_equals_restatement():
    """The native batch walk the benchmark times as the host path gives each frame the restatement's list and
    last_local_idx (empty for a frame below 20 matches or without a vote)."""
    rng = np.random.default_rng(5)
    snap = lmu.synthetic_snapshot(30, 50, rng, reach=3, share=0.5)
    L, B, cap = len(snap["lm_erased"]), 6, 40
    rows = [rng.integers(-1, L, 30).astype(np.int32) for _ in range(B)]
    lo, last_lm = lmu.csr(rows)
    snap["last_row_lm"] = last_lm
    matched = np.full((B, cap), -1, np.int32)
    n_kp = np.full(B, cap, np.int32)
    for b in range(B):
        matched[b, :30] = rng.permutation(30)
    num_valid = np.array([30, 30, 5, 30, 30, 30], np.int32)
    offs, lm, lli = lmu.oracle_update_batch(snap, n_kp, matched, num_valid, lo, 2000)
    for b in range(B):
        tracked = np.array([rows[b][q] if q >= 0 else -1 for q in matched[b]], np.int32)
        r = lmu.update_local_map(snap, tracked) if num_valid[b] >= 20 else None
        want = r["local_lm"] if r else []
        assert list(lm[offs[b]:offs[b + 1]]) == want, b
        assert np.array_equal(lli[lo[b]:lo[b + 1]], lmu.mapping(want, rows[b])), b
