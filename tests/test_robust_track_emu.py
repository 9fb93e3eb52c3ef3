"""The robust-tracker DEVICE code (structure-plp-slam_b200/csrc/robust_track_kernels.cuh, then the keyframe tracker's
gather and finish kernels) executed on the CPU through tests/cta_emu, against numpy and oracle restatements: the prep
flags, the sample draw of csrc/ransac_sample.h, the match list, the batched hypotheses and the select against the
oracle's essential RANSAC and plp_essential_ransac's device code on the same samples, then the gather and
discard_outliers.  The brute-force matches are given (the matcher is the existing brute_match_kernel)."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest

import emu_build
import ess_data
import oracle_api
import robust_track_data as rtd
import synth

_P = C.c_void_p
ISIG = synth.inv_level_sigma_sq()
CAM = SimpleNamespace(fx=500.0, fy=505.0, cx=320.5, cy=240.25)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return emu_build.emu("robust_emu", tmp_path_factory, extra=("-Wno-subobject-linkage",))


@pytest.fixture(scope="module")
def ess_emu(tmp_path_factory):
    return emu_build.emu("essential_emu", tmp_path_factory, extra=("-Wno-subobject-linkage",))


def _a(x, dt):
    return np.ascontiguousarray(x, dt)


def _ptr(a):
    return None if a is None else a.ctypes.data_as(_P)


def _c_sample(emu, seed, b, it, n):
    out = np.zeros(8, np.int32)
    emu.emu_rs_sample8(C.c_uint64(seed), C.c_uint32(b), C.c_uint32(it), C.c_uint32(n), _ptr(out))
    return out


# ------------------------------------------------------------------ prep
def test_robust_prep_flags(emu):
    """Every combination of keyframe stage, keyframe num_valid and keyframe status: the stage runs iff the keyframe
    stage ran and failed; the status carries over; only a frame with stage 1 and status 0 gets a non-empty job."""
    combos = [(s, nv, st) for s in (0, 1) for nv in (0, 19, 20, 300) for st in (0, 1, 2)]
    B, cap = len(combos), 64
    kf_stage, kf_nv, kf_status = (_a([c[i] for c in combos], np.int32) for i in range(3))
    n_kp = _a(np.arange(B) + 10, np.int32)
    rows = _a([0, 30, 75], np.int32)
    kof = _a(np.arange(B) % 2, np.int32)
    stage, status, n_frm, n_kf = (np.full(B, -3, np.int32) for _ in range(4))
    emu.emu_rt_prep(C.c_int(B), C.c_int(cap), _ptr(kf_stage), _ptr(kf_status), _ptr(kf_nv), _ptr(n_kp), _ptr(kof),
                    _ptr(rows), _ptr(stage), _ptr(status), _ptr(n_frm), _ptr(n_kf))
    for b, (s, nv, st) in enumerate(combos):
        want_stage = int(s == 1 and nv < 20)
        assert (stage[b], status[b]) == (want_stage, st), (b, s, nv, st)
        active = want_stage and st == 0
        assert n_frm[b] == (n_kp[b] if active else 0), b
        assert n_kf[b] == ((rows[kof[b] + 1] - rows[kof[b]]) if active else 0), b


# ------------------------------------------------------------------ samples
def test_robust_samples_equal_restatement(emu):
    """ransac_sample.h against the Python restatement: deterministic per (seed, b, iteration), 8 distinct indices in
    range, n = 8 (the only set is all of them), n = 9, and the top-up round when duplicates leave fewer than 8."""
    rng = np.random.default_rng(3)
    for seed in (0, 1, 2**63 + 5, 2**64 - 1):
        for n in (8, 9, 10, 17, 100, 4096, 2**31 + 11):
            for b in (0, 1, 511):
                for it in (0, 1, 49):
                    got = _c_sample(emu, seed, b, it, n)
                    assert np.array_equal(got, rtd.draw_sample(seed, b, it, n)), (seed, n, b, it)
                    assert len(set(got.tolist())) == 8 and got.min() >= 0 and got.max() < n
                    if n == 8:
                        assert sorted(got.tolist()) == list(range(8))
    # determinism, and different streams for different keys
    a = _c_sample(emu, 5, 3, 7, 1000)
    assert np.array_equal(a, _c_sample(emu, 5, 3, 7, 1000))
    others = [_c_sample(emu, 6, 3, 7, 1000), _c_sample(emu, 5, 4, 7, 1000), _c_sample(emu, 5, 3, 8, 1000)]
    assert all(not np.array_equal(a, o) for o in others)
    # the shuffle: the sets are not sorted in general
    assert any(not np.array_equal(np.sort(s), s) for s in (rtd.draw_sample(0, 0, it, 1000) for it in range(10)))
    # a draw whose first round leaves fewer than 8 distinct values tops up (n = 9: duplicates are frequent)
    topped = []
    for it in range(200):
        trace = []
        want = rtd.draw_sample(int(rng.integers(2**63)), 0, it, 9, trace)
        if trace[0] < 8:
            topped.append(it)
        assert len(trace) >= 1 and trace[-1] == 8
        del want
    assert topped
    for it in topped[:20]:
        seed = 77
        assert np.array_equal(_c_sample(emu, seed, 2, it, 9), rtd.draw_sample(seed, 2, it, 9))


# ------------------------------------------------------------------ the whole chain
def _frame_from_view(rng, seed, n_take, outlier_frac=0.3):
    """A frame (shot 1) and its keyframe (shot 2) from ess_data.make_two_view: pixel keypoints of shot 1, the
    brute-force matches (frame keypoint -> keyframe row) of n_take of its matches."""
    b1, b2, matches, _ = ess_data.make_two_view(seed, n=max(n_take, 60), outlier_frac=outlier_frac)
    n = len(b1)
    x = (CAM.fx * b1[:, 0] / b1[:, 2] + CAM.cx).astype(np.float32)
    y = (CAM.fy * b1[:, 1] / b1[:, 2] + CAM.cy).astype(np.float32)
    bf = np.full(n, -1, np.int32)
    take = matches[rng.permutation(len(matches))[:n_take]]
    bf[take[:, 0]] = take[:, 1]
    return dict(x=x, y=y, octave=rng.integers(0, 8, n).astype(np.int32), bf=bf), \
        dict(bearings=b2, pos_w=rng.normal(0, 3, (len(b2), 3)))


def test_robust_track_kernels_on_cpu_equal_restatement(emu, ess_emu, orc):
    rng = np.random.default_rng(71)
    f0, k0 = _frame_from_view(rng, 1, 300)            # 0: many matches, valid, >= 20 robust matches
    f1, k1 = _frame_from_view(rng, 2, 5)              # 1: fewer than 8 matches: no RANSAC
    f2, k2 = _frame_from_view(rng, 3, 15, 0.0)        # 2: valid, but fewer than 20 robust matches
    f3, _ = _frame_from_view(rng, 4, 200)             # 3: keyframe stage did not run
    f4, _ = _frame_from_view(rng, 5, 200)             # 4: keyframe stage succeeded
    f5, _ = _frame_from_view(rng, 6, 200)             # 5: keyframe status 2 carried over
    f6 = dict(f0, bf=np.where(rng.random(len(f0["bf"])) < 0.6, f0["bf"], -1).astype(np.int32))  # 6: shares keyframe 0
    frames = [f0, f1, f2, f3, f4, f5, f6]
    kfs = [k0, k1, k2]
    kf_of_frame = [0, 1, 2, 0, 1, 7, 0]
    kf_stage = [1, 1, 1, 0, 1, 1, 1]
    kf_nv = [0, 3, 19, 0, 25, 0, 0]
    kf_status = [0, 0, 0, 0, 0, 2, 0]
    B, cap, seed = len(frames), 416, 2024
    n_kp = _a([len(f["x"]) for f in frames], np.int32)

    def pad(key, dt, fill=0):
        out = np.full((B, cap), fill, dt)
        for b, f in enumerate(frames):
            out[b, :len(f[key])] = f[key]
        return out
    X, Y, O, BF = pad("x", np.float32), pad("y", np.float32), pad("octave", np.int32), pad("bf", np.int32, -9)
    rows = _a(np.concatenate([[0], np.cumsum([len(k["bearings"]) for k in kfs])]), np.int32)
    kb = _a(np.concatenate([k["bearings"] for k in kfs]), np.float64)
    kpos = _a(np.concatenate([k["pos_w"] for k in kfs]), np.float64)
    pose_last = _a(np.tile(np.eye(4), (B, 1, 1)), np.float64)
    K = _a([CAM.fx, CAM.fy, CAM.cx, CAM.cy], np.float64)
    bear = np.full((B, cap, 3), -7.0)
    stage, status, num_bf, valid, num_robust, n_obs = (np.full(B, -3, np.int32) for _ in range(6))
    matched = np.full((B, cap), -5, np.int32)
    pairs = np.zeros((B, cap, 2), np.int32)
    samples = np.full((B, 50, 8), -3, np.int32)
    E = np.zeros((B, 50, 9))
    score = np.full((B, 50), -1.0, np.float32)
    inlier = np.zeros((B, cap), np.uint8)
    best_score = np.full(B, -1.0)
    obs = np.zeros((B, cap), oracle_api.PT_OBS_DTYPE)
    obs_kp, obs_row = np.zeros((B, cap), np.int32), np.zeros((B, cap), np.int32)
    isig = _a(ISIG, np.float32)
    args = [_a(a, np.int32) for a in (kf_stage, kf_status, kf_nv, kf_of_frame)]
    emu.emu_rt_begin(C.c_int(B), C.c_int(cap), C.c_uint64(seed), _ptr(n_kp), _ptr(X), _ptr(Y), _ptr(O),
                     _ptr(pose_last), _ptr(isig), C.c_int(len(isig)), _ptr(K), *[_ptr(a) for a in args], _ptr(rows),
                     _ptr(kpos), _ptr(kb), _ptr(bear), C.c_int(1), _ptr(BF), _ptr(stage), _ptr(status), _ptr(matched),
                     _ptr(num_bf), _ptr(pairs), _ptr(samples), _ptr(E), _ptr(score), _ptr(inlier), _ptr(best_score),
                     _ptr(valid), _ptr(num_robust), _ptr(obs), _ptr(obs_kp), _ptr(obs_row), _ptr(n_obs))
    matched_sel = matched.copy()
    outlier = (rng.random((B, cap)) < 0.2).astype(np.uint8)  # the pose optimiser is not emulated
    num_valid = np.full(B, -3, np.int32)
    emu.emu_rt_finish(_ptr(outlier), _ptr(num_valid))

    assert list(stage) == [1, 1, 1, 0, 0, 1, 1] and list(status) == kf_status
    for b, f in enumerate(frames):
        n = len(f["x"])
        active = stage[b] and status[b] == 0
        if not active:
            assert num_bf[b] == 0 and num_robust[b] == 0 and n_obs[b] == 0 and num_valid[b] == 0, b
            assert (samples[b] == -1).all() and (matched[b, :n] == -1).all(), b
            continue
        # the frame's bearings (convert_keypoints_to_bearings of its keypoints)
        fb = rtd.bearings(CAM, f["x"], f["y"])
        assert np.array_equal(bear[b, :n], fb), b
        # the match list in frame keypoint order, and the samples
        idx = np.nonzero(f["bf"] >= 0)[0]
        M = len(idx)
        assert num_bf[b] == M and np.array_equal(pairs[b, :M], np.stack([idx, f["bf"][idx]], 1)), b
        assert np.array_equal(samples[b], rtd.draw_samples(seed, b, M)), b
        kb_b = kfs[kf_of_frame[b]]["bearings"]
        if M < 8:
            assert valid[b] == 0 and num_robust[b] == 0 and (matched_sel[b, :n] == -1).all(), b
        else:
            # the hypotheses, the select and the flags against the oracle and plp_essential_ransac's device code
            ov, oinl, oE, oscore, oscores = orc.essential_ransac(fb, kb_b, pairs[b, :M], samples[b])
            assert np.array_equal(score[b], oscores), b
            assert valid[b] == ov and best_score[b] == oscore and np.array_equal(inlier[b, :M], oinl), b
            # the first maximum: the reference replaces its best only on a strictly larger score
            best = int(np.argmax(oscores)) if oscore > 0 else -1
            if best >= 0:
                assert np.array_equal(E[b, best], oE.ravel()), b
            dinl, dE, dscore = np.zeros(M, np.uint8), np.zeros(9), C.c_double(0)
            dv = ess_emu.emu_essential_ransac(_ptr(_a(fb, np.float64)), _ptr(_a(kb_b, np.float64)),
                                              _ptr(_a(pairs[b, :M], np.int32)), C.c_int(M), _ptr(_a(samples[b], np.int32)),
                                              C.c_int(50), C.c_int(0), _ptr(dinl), _ptr(dE), C.byref(dscore))
            assert dv == valid[b] and np.array_equal(dinl, inlier[b, :M]) and dscore.value == best_score[b], b
            if best >= 0:
                assert np.array_equal(dE, E[b, best]), b
            robust = np.full(n, -1, np.int32)
            if ov:
                keep = pairs[b, :M][oinl != 0]
                robust[keep[:, 0]] = keep[:, 1]
            assert num_robust[b] == (robust >= 0).sum() and np.array_equal(matched_sel[b, :n], robust), b
        # gather and discard_outliers
        post = matched_sel[b, :n].copy()
        if num_robust[b] < 20:
            assert n_obs[b] == 0 and (matched[b, :n] == -1).all() and num_valid[b] == 0, b
            continue
        sel = np.nonzero(post >= 0)[0]
        no = len(sel)
        assert n_obs[b] == no and np.array_equal(obs_kp[b, :no], sel) and np.array_equal(obs_row[b, :no], post[sel]), b
        o = obs[b, :no]
        kpw = kfs[kf_of_frame[b]]["pos_w"]
        assert np.array_equal(o["pos_w"], kpw[post[sel]]), b
        assert np.array_equal(o["obs_x"], f["x"][sel]) and np.array_equal(o["obs_y"], f["y"][sel]), b
        assert np.array_equal(o["inv_sigma_sq"], ISIG[f["octave"][sel]]) and (o["x_right"] == -1.0).all(), b
        post[sel[outlier[b, :no] != 0]] = -1
        assert np.array_equal(matched[b, :n], post) and num_valid[b] == (post >= 0).sum(), b
    # the cases the batch is meant to cover
    assert valid[0] == 1 and num_robust[0] >= 20 and num_valid[0] > 0
    assert num_bf[1] < 8 and valid[1] == 0
    assert valid[2] == 1 and 8 <= num_robust[2] < 20
    assert valid[6] == 1 and num_robust[6] >= 20


def _run_chain(emu, frames, kfs, kf_of_frame, kf_stage, kf_nv, kf_status, cap, seed):
    """emu_rt_begin + emu_rt_finish (no outliers) over the frames; -> the outputs as a dict of arrays."""
    B = len(frames)
    n_kp = _a([len(f["x"]) for f in frames], np.int32)

    def pad(key, dt, fill=0):
        out = np.full((B, cap), fill, dt)
        for b, f in enumerate(frames):
            out[b, :len(f[key])] = f[key]
        return out
    X, Y, O, BF = pad("x", np.float32), pad("y", np.float32), pad("octave", np.int32), pad("bf", np.int32, -9)
    rows = _a(np.concatenate([[0], np.cumsum([len(k["bearings"]) for k in kfs])]), np.int32)
    kb = _a(np.concatenate([k["bearings"] for k in kfs]), np.float64)
    kpos = _a(np.concatenate([k["pos_w"] for k in kfs]), np.float64)
    pose_last = _a(np.tile(np.eye(4), (B, 1, 1)), np.float64)
    K = _a([CAM.fx, CAM.fy, CAM.cx, CAM.cy], np.float64)
    o = dict(bear=np.full((B, cap, 3), -7.0), matched=np.full((B, cap), -5, np.int32),
             pairs=np.zeros((B, cap, 2), np.int32), samples=np.full((B, 50, 8), -3, np.int32), E=np.zeros((B, 50, 9)),
             score=np.full((B, 50), -1.0, np.float32), inlier=np.zeros((B, cap), np.uint8), best_score=np.full(B, -1.0),
             obs=np.zeros((B, cap), oracle_api.PT_OBS_DTYPE), obs_kp=np.zeros((B, cap), np.int32),
             obs_row=np.zeros((B, cap), np.int32))
    for k in ("stage", "status", "num_bf", "valid", "num_robust", "n_obs", "num_valid"):
        o[k] = np.full(B, -3, np.int32)
    isig = _a(ISIG, np.float32)
    args = [_a(a, np.int32) for a in (kf_stage, kf_status, kf_nv, kf_of_frame)]
    emu.emu_rt_begin(C.c_int(B), C.c_int(cap), C.c_uint64(seed), _ptr(n_kp), _ptr(X), _ptr(Y), _ptr(O),
                     _ptr(pose_last), _ptr(isig), C.c_int(len(isig)), _ptr(K), *[_ptr(a) for a in args], _ptr(rows),
                     _ptr(kpos), _ptr(kb), _ptr(o["bear"]), C.c_int(1), _ptr(BF), _ptr(o["stage"]), _ptr(o["status"]),
                     _ptr(o["matched"]), _ptr(o["num_bf"]), _ptr(o["pairs"]), _ptr(o["samples"]), _ptr(o["E"]),
                     _ptr(o["score"]), _ptr(o["inlier"]), _ptr(o["best_score"]), _ptr(o["valid"]),
                     _ptr(o["num_robust"]), _ptr(o["obs"]), _ptr(o["obs_kp"]), _ptr(o["obs_row"]), _ptr(o["n_obs"]))
    emu.emu_rt_finish(_ptr(np.zeros((B, cap), np.uint8)), _ptr(o["num_valid"]))
    return o


def test_robust_frame_over_matcher_capacity(emu):
    """A frame with more keypoints than the brute-force matcher holds (4096; the matcher's guard leaves every match -1)
    lists nothing and reports num_bf = -1, draws no sample, gathers nothing and fails.  A frame with exactly 4096
    keypoints, an over-capacity frame whose keyframe track succeeded (the stage does not run: num_bf 0) and a normal
    frame are unaffected: they equal the same frames run without the over-capacity frame."""
    rng = np.random.default_rng(72)
    f1, k1 = _frame_from_view(rng, 12, 4096)          # 0: exactly the matcher's capacity
    f2, k0 = _frame_from_view(rng, 13, 4150)          # 1: over it, keyframe stage succeeded
    f3, _ = _frame_from_view(rng, 14, 120)            # 2: normal
    f0, _ = _frame_from_view(rng, 11, 4200)           # 3: over it, runs the stage
    over = dict(f0, bf=np.full(len(f0["bf"]), -1, np.int32))  # what the matcher's guard leaves
    frames = [f1, f2, f3, over]
    assert [len(f["x"]) for f in frames] == [4096, 4150, 120, 4200]
    kfs, kf_of_frame = [k0, k1], [1, 0, 1, 0]
    kf_stage, kf_nv, kf_status = [1, 1, 1, 1], [0, 25, 3, 0], [0, 0, 0, 0]
    cap, seed = 4224, 99
    got = _run_chain(emu, frames, kfs, kf_of_frame, kf_stage, kf_nv, kf_status, cap, seed)
    ref = _run_chain(emu, frames[:3], kfs, kf_of_frame[:3], kf_stage[:3], kf_nv[:3], kf_status[:3], cap, seed)
    assert list(got["stage"]) == [1, 0, 1, 1] and list(got["status"]) == [0, 0, 0, 0]
    # the over-capacity frame: the marker, no list, no samples, no RANSAC, no observations
    assert got["num_bf"][3] == -1
    assert (got["samples"][3] == -1).all() and got["valid"][3] == 0 and got["num_robust"][3] == 0
    assert got["n_obs"][3] == 0 and got["num_valid"][3] == 0 and (got["matched"][3, :4200] == -1).all()
    # the other frames equal the batch without it
    for b in range(3):
        n = len(frames[b]["x"])
        for k in ("stage", "num_bf", "valid", "num_robust", "n_obs", "num_valid", "best_score"):
            assert got[k][b] == ref[k][b], (b, k)
        M = max(int(got["num_bf"][b]), 0)
        for k in ("samples", "E", "score"):
            assert np.array_equal(got[k][b], ref[k][b]), (b, k)
        assert np.array_equal(got["pairs"][b, :M], ref["pairs"][b, :M]), b
        assert np.array_equal(got["matched"][b, :n], ref["matched"][b, :n]), b
    assert got["num_bf"][0] == 4096 and got["num_robust"][0] >= 20 and got["num_valid"][0] >= 20
    assert got["num_bf"][1] == 0 and got["num_bf"][2] == 120
