"""smoke(): the robust tracker on three frames (extract -> motion track -> keyframe track -> robust track -> local map):
one motion success, one robust rescue (its keyframe's BoW vector is empty), one robust failure (99 % of its
keyframe's landmarks erased), against the oracle, with a synthetic vocabulary."""
import numpy as np


def run(pkg, ctx, orc):
    import keyframe_track_data as ktd
    import local_map_data as lmd
    import oracle_api
    import robust_track_data as rtd
    import scene
    from plpslam_b200.tracking import FrontEnd

    ts = [2, 4, 3]
    seq = scene.PlanarSequence(seed=41, n_frames=5)
    res = [orc.orb_extract(oracle_api.orb_params(), f) for f in seq.frames]
    v = ktd.make_scene_vocab(np.concatenate([r["desc"] for r in res]), 3)
    ov = orc.bow_vocab_create(v["k"], v["L"], v["parent"], v["desc"], v["weight"], v["is_leaf"])
    gv = pkg.BowVocabulary(ctx, k=v["k"], L=v["L"], parent=v["parent"], desc=v["desc"], weight=v["weight"],
                           is_leaf=v["is_leaf"])
    fe = FrontEnd(ctx, seq.rows, seq.cols, seq.camera(pkg), max_batch=3)
    try:
        fe.reserve_local_map(4096)
        fe.reserve_keyframe_track(2, 1500)
        fe.reserve_robust_track()
        rng = np.random.default_rng(4)
        kfs = [rtd.keyframe(orc, ov, seq, res, 0, rng, fe.cam, empty_fv=True),
               rtd.keyframe(orc, ov, seq, res, 1, rng, fe.cam, erased_frac=0.99)]
        r = rtd.run_case(orc, pkg, fe, ov, gv, seq, res, ts, kfs, [0, 0, 1], [1, 0, 0], seed=5, rb_seed=11)
        assert r["rb_stage"] == [0, 1, 1], r["rb_stage"]
        ktd.compare(r["kf"], r["kf_wants"], r["kf_stage"])
        rtd.compare(r["rb"], r["rb_wants"], r["rb_stage"], 11)
        lmd.compare(r["local"], r["local_wants"])
        out = r["rb"]
        assert out["num_valid"][1] >= 20 and out["num_valid"][2] == 0, out["num_valid"]
        print(f"smoke robust track ok: stage {r['rb_stage']}, brute-force matches {list(out['num_bf_matches'])}, "
              f"robust matches {list(out['num_robust_matches'])}, num_valid {list(out['num_valid'])}, "
              f"local map num_tracked {list(r['local']['num_tracked'])}, bit-exact")
    finally:
        fe.close()
        gv.close()
        orc.bow_vocab_destroy(ov)
