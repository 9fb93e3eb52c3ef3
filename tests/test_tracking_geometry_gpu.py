"""The batched tracker's motion -> keyframe -> robust -> local-map chain against the oracle chain at the geometries,
keypoint budgets and batch the library ships with or is timed at: the KITTI mono sizes at 2000 keypoints, TUM-VI's
fisheye and TUM mono 1's radial-tangential camera, keypoint capacities on both sides of the brute-force matcher's 4096,
frames over the window matcher's (3072) and the brute-force matcher's per-frame capacity, and bench.py's 512-frame
batch.  The comparisons are those of test_robust_track_gpu.py: exact match indices, counts and stage flags, poses
within 1e-4 relative."""
import importlib.util
from pathlib import Path

import numpy as np
import pytest

import camera_data as cd
import keyframe_track_data as ktd
import local_map_data as lmd
import oracle_api
import robust_track_data as rtd
import scene
from test_geometry_gpu import STEREO

pytestmark = pytest.mark.gpu

WINDOW_CAP, BRUTE_CAP = 3072, 4096  # the window matcher's and the brute-force matcher's per-frame keypoints
OVER = 0xFFFFFFFF                   # a matcher's count for a frame over its capacity
ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture
def own():
    """own(x) returns x and closes / frees it when the test ends, also after a failed assertion."""
    objs = []
    yield lambda x: objs.append(x) or x
    for x in reversed(objs):
        x.close()


class _OracleVocab:
    def __init__(self, orc, h):
        self.orc, self.h = orc, h

    def close(self):
        self.orc.bow_vocab_destroy(self.h)


def _vocab(orc, plp, ctx, own, res, seed):
    v = ktd.make_scene_vocab(np.concatenate([r["desc"] for r in res]), seed)
    ov = orc.bow_vocab_create(v["k"], v["L"], v["parent"], v["desc"], v["weight"], v["is_leaf"])
    own(_OracleVocab(orc, ov))
    gv = own(plp.BowVocabulary(ctx, k=v["k"], L=v["L"], parent=v["parent"], desc=v["desc"], weight=v["weight"],
                               is_leaf=v["is_leaf"]))
    return ov, gv


def _check(r, seed, rb_frames=None, local_frames=None):
    got_it, want_it = ktd.compare(r["kf"], r["kf_wants"], r["kf_stage"])
    scene.check_lm_iters(got_it, want_it, "keyframe track")
    got_it, want_it = rtd.compare(r["rb"], r["rb_wants"], r["rb_stage"], seed, frames=rb_frames)
    scene.check_lm_iters(got_it, want_it, "robust track")
    got_it, want_it = lmd.compare(r["local"], r["local_wants"], frames=local_frames)
    scene.check_lm_iters(got_it, want_it, "local map")


def _mixed_batch(ctx, orc, plp, own, seq, budget, dist=None, undistort=None, bounds=None, vocab_seed=5,
                 fail_shift=(1.0, 0.5, 0.0)):
    """Batch of 8 over 5 keyframes (test_robust_track_gpu's mixed batch): motion track succeeded (0, 5); motion failed
    and the BoW track succeeded (1); the keyframes of frames 2, 4, 6 and 7 have an empty bow_feat_vec_ and the robust
    stage rescues them (2 and 7 share a keyframe); frame 3's keyframe keeps ~10 landmarks, so both stages fail.  Then
    the local-map stage from each frame's record.  -> (front end, run_case result)."""
    from plpslam_b200.tracking import FrontEnd
    p = oracle_api.orb_params(budget, 1.2, 8, 20, 7)
    ts = [2, 3, 4, 5, 6, 7, 8, 2]
    res = [orc.orb_extract(p, f) for f in seq.frames]
    ov, gv = _vocab(orc, plp, ctx, own, res, vocab_seed)
    fe = own(FrontEnd(ctx, seq.rows, seq.cols, seq.camera(plp), max_batch=8, max_num_keypts=budget, ini_fast_thr=20,
                      min_fast_thr=7, distortion=dist))
    grid = cam = None
    if bounds is not None:
        grid = plp.capi.make_grid(seq.cols, seq.rows, min_x=bounds[0], min_y=bounds[2], max_x=bounds[1],
                                  max_y=bounds[3])
        cam = seq.camera(plp)
        cam.min_x, cam.max_x, cam.min_y, cam.max_y = (float(v) for v in bounds)
    fe.reserve_local_map(16384)
    fe.reserve_keyframe_track(5, max(len(r["kps"]) for r in res))
    fe.reserve_robust_track()
    rng = np.random.default_rng(8)
    kcam = cam or fe.cam
    erased = 1.0 - 10.0 / budget

    def kf(t, **kw):
        return rtd.keyframe(orc, ov, seq, res, t, rng, kcam, undistort=undistort, **kw)
    kfs = [kf(0, empty_fv=True), kf(1), kf(4, erased_frac=erased), kf(1, empty_fv=True), kf(4, empty_fv=True)]
    kf_of_frame = [0, 1, 0, 2, 3, 1, 4, 0]
    r = rtd.run_case(orc, plp, fe, ov, gv, seq, res, ts, kfs, kf_of_frame, [1, 1, 0, 0, 0, 1, 0, 0], fail=(1,), seed=9,
                     rb_seed=1234, grid=grid, cam=cam, undistort=undistort, fail_shift=fail_shift)
    # every branch occurs
    assert r["kf_stage"] == [0, 1, 1, 1, 1, 0, 1, 1], r["kf_stage"]
    assert r["rb_stage"] == [0, 0, 1, 1, 1, 0, 1, 1], r["rb_stage"]
    mot, kout, out, lout = r["mot"], r["kf"], r["rb"], r["local"]
    assert all(mot["num_valid"][b] >= 20 for b in (0, 5)), mot["num_valid"]
    assert kout["num_valid"][1] >= 20, kout["num_valid"][1]
    for b in (2, 4, 6, 7):
        assert out["num_bf_matches"][b] >= 100 and out["num_valid"][b] >= 20, (b, out["num_bf_matches"][b])
    assert out["num_bf_matches"][3] < 20 and out["num_valid"][3] == 0 and out["lm_iters"][3] == 0
    assert np.array_equal(out["pose"][3], seq.poses[ts[3] - 1])
    for b in (0, 1, 2, 4, 5, 6, 7):
        assert lout["num_tracked"][b] > 0 and lout["status"][b] == 0, b
    assert lout["num_tracked"][3] == 0
    _check(r, 1234)
    return fe, r


# ----------------------------------------------------------------------------------- a. the shipped configurations
@pytest.mark.parametrize("name", ["kitti00", "kitti03", "kitti04"])
def test_chain_kitti_2000_keypoints(ctx, orc, plp, own, name):
    """KITTI mono (2000 keypoints, FAST 20 / 7), principal point at the image centre: the frames carry well over 1000
    keypoints, the tracker's keypoint capacity is above the brute-force matcher's, and the robust stage runs."""
    (rows, cols), fx, _, _ = STEREO[name]
    seq = scene.PlanarSequence(seed=41, n_frames=9, rows=rows, cols=cols, fx=fx, fy=fx, cx=cols / 2.0, cy=rows / 2.0)
    fe, r = _mixed_batch(ctx, orc, plp, own, seq, 2000)
    assert fe.cap > BRUTE_CAP, fe.cap
    n = np.array([len(m) for m in r["mot"]["matched"]])
    assert (n > 1500).all() and (n <= WINDOW_CAP).all(), n


@pytest.mark.parametrize("name", ["tumvi_fisheye", "tum_mono_1"])
def test_chain_distorted_1000_keypoints(ctx, orc, plp, own, name):
    """TUM-VI's fisheye and TUM mono 1's radial-tangential camera through plp_tracker_create_ex: the frame bearings
    and every stage's observations are the undistortion's.  Frame 1's predicted pose is 3 m off: the fisheye's wide
    view still finds 20 matches a metre off."""
    import distorted_scene
    model, cols, rows, K, D = cd.CONFIGS[name]
    seq = distorted_scene.DistortedPlanarSequence((model, D), seed=43, n_frames=9, rows=rows, cols=cols, fx=K[0],
                                                  fy=K[1], cx=K[2], cy=K[3])
    fe, r = _mixed_batch(ctx, orc, plp, own, seq, 1000, dist=plp.capi.make_distortion(model, *D),
                         undistort=seq.undistort, bounds=seq.bounds(), vocab_seed=6, fail_shift=(3.0, 1.5, 0.0))
    und = fe.download_undistorted(8)
    for b in range(8):
        assert np.array_equal(und[b][1], r["frm_bearings"][b]), b


# ----------------------------------------------------------------------------------- b. the capacity boundary
@pytest.mark.parametrize("budget,above", [(1000, False), (1010, True)])
def test_chain_capacity_boundary(ctx, orc, plp, own, budget, above):
    """Two keypoint budgets whose tracker capacity (the extractor's slot capacity) lies on either side of the
    brute-force matcher's 4096: both reserve the robust stage and equal the oracle chain."""
    seq = scene.PlanarSequence(seed=41, n_frames=9)
    fe, _ = _mixed_batch(ctx, orc, plp, own, seq, budget)
    assert (fe.cap > BRUTE_CAP) == above, fe.cap


# ----------------------------------------------------------------------------------- c. over the matchers' capacities
def test_chain_frames_over_matcher_capacity(ctx, orc, plp, own):
    """KITTI 00 size, keypoints from the oracle extractor uploaded in place of the device extractor's (whose quadtree
    caps a level's budget well below 3072 keypoints per frame): frame 2 has 3073..4096 keypoints, over the window
    matcher's capacity but within the brute-force matcher's; frame 3 has more than 4096.  Frames 0 (motion track) and
    1 (motion fails, BoW track) are normal.
    - Frame 2: motion count 0xffffffff, nothing gathered, the motion track fails; the keyframe and robust stages equal
      the oracle chain; the local-map stage, started from the robust record, reports 0xffffffff and matches no local
      row.
    - Frame 3: motion count 0xffffffff; the robust stage reports num_bf_matches -1 and fails with pose_last; the
      local-map stage treats it as a frame whose start record failed.
    - Frames 0 and 1 equal the oracle chain."""
    from plpslam_b200.tracking import FrontEnd
    (rows, cols), fx, _, _ = STEREO["kitti00"]
    seq = scene.PlanarSequence(seed=21, n_frames=8, rows=rows, cols=cols, fx=fx, fy=fx, cx=cols / 2.0, cy=rows / 2.0)
    budgets = {4: 3500, 6: 5000}  # frames 2 and 3 of the batch; the others 2000
    res = [orc.orb_extract(oracle_api.orb_params(budgets.get(t, 2000), 1.2, 8, 20, 7), f)
           for t, f in enumerate(seq.frames)]
    ts = [2, 3, 4, 6]
    n = [len(res[t]["kps"]) for t in ts]
    assert all(k <= WINDOW_CAP for k in n[:2]) and WINDOW_CAP < n[2] <= BRUTE_CAP and n[3] > BRUTE_CAP, n
    ov, gv = _vocab(orc, plp, ctx, own, res, 5)
    fe = own(FrontEnd(ctx, rows, cols, seq.camera(plp), max_batch=4, max_num_keypts=1200, ini_fast_thr=20,
                      min_fast_thr=7))
    assert fe.cap >= n[3], (fe.cap, n)
    fe.reserve_local_map(16384)
    rng = np.random.default_rng(8)
    kfs = [rtd.keyframe(orc, ov, seq, res, 1, rng, fe.cam),
           rtd.keyframe(orc, ov, seq, res, 1, rng, fe.cam, empty_fv=True),
           rtd.keyframe(orc, ov, seq, res, 5, rng, fe.cam, empty_fv=True)]
    fe.reserve_keyframe_track(3, max(len(k["desc"]) for k in kfs))
    fe.reserve_robust_track()
    r = rtd.run_case(orc, plp, fe, ov, gv, seq, res, ts, kfs, [0, 0, 1, 2], None, fail=(1,), seed=9, rb_seed=77,
                     over=(2, 3), kps_given=True)
    mot, out, lout = r["mot"], r["rb"], r["local"]
    counts = fe.download_match_counts(4)
    assert r["kf_stage"] == [0, 1, 1, 1] and r["rb_stage"] == [0, 0, 1, 1], (r["kf_stage"], r["rb_stage"])
    # the motion track: the window matcher's guard on frames 2 and 3 only
    assert list(counts["motion"][2:]) == [OVER, OVER], counts["motion"]
    assert counts["motion"][0] >= 20 and counts["motion"][1] < OVER, counts["motion"]
    rng_pred = np.random.default_rng(9)
    preds = [seq.predicted_pose(t, rng_pred) for t in ts]
    for b in (2, 3):
        assert (mot["matched"][b] == -1).all() and mot["num_valid"][b] == 0 and mot["lm_iters"][b] == 0, b
        assert np.array_equal(mot["pose"][b], preds[b]), b
    # keyframe stage for all, robust stage for frames 0..2 against the oracle; frame 2 is rescued
    _check(r, 77, rb_frames=(0, 1, 2), local_frames=(0, 1))
    assert out["num_bf_matches"][2] >= 100 and out["num_valid"][2] >= 20, \
        (out["num_bf_matches"][2], out["num_valid"][2])
    # frame 3: over the brute-force matcher's capacity
    assert out["num_bf_matches"][3] == -1 and out["num_robust_matches"][3] == 0 and out["status"][3] == 0
    assert out["num_valid"][3] == 0 and out["lm_iters"][3] == 0 and (out["matched"][3] == -1).all()
    assert (out["samples"][3] == -1).all()
    assert np.array_equal(out["pose"][3], seq.poses[ts[3] - 1])
    # the local-map stage: frame 2 runs with the window matcher's guard, frame 3 does not run
    assert counts["local"][2] == OVER, counts["local"]
    assert lout["status"][2] == 0 and (lout["local"][2] == -1).all()
    assert lout["status"][3] == 0 and lout["num_tracked"][3] == 0 and lout["lm_iters"][3] == 0
    assert (lout["matched"][3] == -1).all() and (lout["local"][3] == -1).all() and not lout["observable"][3].any()
    assert np.array_equal(lout["pose"][3], out["pose"][3])


# ----------------------------------------------------------------------------------- d. the benchmark's batch
def test_chain_bench_batch(ctx, orc, plp, own):
    """bench.setup_front_end at B = 512 (32 frames from each of 16 sequences), 128 keyframes: frames 4g + 1 .. 4g + 4
    share frame 4g, whose bow_feat_vec_ is empty.  Even frames keep their motion model and succeed there; odd frames
    fall through to the keyframe and robust stages.  Every frame equals the oracle chain; the hypothesis grid is
    (50, 512)."""
    spec = importlib.util.spec_from_file_location("plp_bench", ROOT / "bench.py")
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    B, seed = 512, 1234
    fe, _, aux = bench.setup_front_end(plp, ctx, B, seed)
    own(fe)
    seqs, t_idx = aux["seqs"], aux["t_idx"]
    kf_t = [4 * ((t - 1) // 4) for (_, t) in t_idx]
    fe.upload_images(np.stack([seqs[s].frames[k] for (s, _), k in zip(t_idx, kf_t)]))
    fe.extract(B)
    prev = fe.download_keypoints(B)
    rng = np.random.default_rng(seed)
    pool = np.concatenate([prev[b][1] for b in rng.choice(B, 16, replace=False)])
    v = ktd.make_scene_vocab(pool, seed)
    gv = own(plp.BowVocabulary(ctx, k=v["k"], L=v["L"], parent=v["parent"], desc=v["desc"], weight=v["weight"],
                               is_leaf=v["is_leaf"]))
    empty_fv = (np.zeros(0, np.uint32), np.zeros(1, np.int32), np.zeros(0, np.uint32))
    keys, kfs, kf_of_frame = {}, [], []
    for b, (s, t) in enumerate(t_idx):
        key = (s, kf_t[b])
        if key not in keys:
            k, d = prev[b]
            pos_w = seqs[s].backproject(seqs[s].poses[key[1]], k["x"].astype(np.float64), k["y"].astype(np.float64))
            keys[key] = len(kfs)
            kfs.append(dict(t=key[1], desc=d, angle=k["angle"].astype(np.float32), valid=np.ones(len(d), np.uint8),
                            pos_w=pos_w, fv=empty_fv, bearings=rtd.bearings(fe.cam, k["x"], k["y"])))
        kf_of_frame.append(keys[key])
    assert len(kfs) == 128
    fe.reserve_keyframe_track(len(kfs), max(len(k["desc"]) for k in kfs))
    fe.reserve_robust_track()
    fe.set_keyframes(kfs, kf_of_frame)
    mv = (np.arange(B) % 2 == 0).astype(np.uint8)
    fe.upload_images(np.stack([seqs[s].frames[t] for (s, t) in t_idx]))
    fe.step(B)
    fe.track_keyframe(B, gv, mv)
    fe.track_robust(B, seed)
    kps = fe.download_keypoints(B)
    mot = fe.download_tracking(B)
    kout = fe.download_keyframe_tracking(B)
    out = fe.download_robust_tracking(B)
    stage = [int(mv[b] == 0 or mot["num_valid"][b] < 20) for b in range(B)]
    assert list(kout["stage"]) == stage and list(out["stage"]) == stage  # an empty bow_feat_vec_: no BoW match
    assert sum(stage) >= B // 2 and (out["num_valid"][np.array(stage, bool)] >= 20).mean() > 0.5
    grid, cam = fe.grid, fe.cam
    wants = []
    for b, (s, t) in enumerate(t_idx):
        k = kps[b][0]
        curr = dict(x=k["x"], y=k["y"], octave=k["octave"], angle=k["angle"], desc=kps[b][1])
        if not stage[b]:  # the motion track against the oracle
            _, m, T, nv, _, _ = lmd.oracle_motion(orc, grid, cam, curr, aux["lasts"][b], aux["preds"][b],
                                                  seqs[s].poses[t - 1])
            assert np.array_equal(mot["matched"][b], m) and mot["num_valid"][b] == nv >= 20, b
            assert np.linalg.norm(mot["pose"][b] - T) <= 1e-4 * np.linalg.norm(T), b
            wants.append(None)
            continue
        assert kout["num_bow_matches"][b] == 0 and kout["num_valid"][b] == 0, b
        # every (frame, keyframe) input is distinct: one brute-force oracle match and one RANSAC per frame
        wants.append(rtd.oracle_robust_track(orc, cam, curr, kfs[kf_of_frame[b]], rtd.bearings(cam, k["x"], k["y"]),
                                             out["samples"][b], seqs[s].poses[t - 1]))
    got_it, want_it = rtd.compare(out, wants, stage, seed)
    scene.check_lm_iters(got_it, want_it, "robust track, 512 frames")
