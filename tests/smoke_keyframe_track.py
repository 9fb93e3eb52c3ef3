"""smoke(): the keyframe tracker on three frames (extract -> motion track -> keyframe track -> local map), one frame per
stage outcome, against the oracle, with a synthetic vocabulary."""
import numpy as np


def run(pkg, ctx, orc):
    import keyframe_track_data as ktd
    import local_map_data as lmd
    import oracle_api
    import scene
    from plpslam_b200.tracking import FrontEnd

    ts = [2, 3, 4]
    seq = scene.PlanarSequence(seed=32, n_frames=5)
    res = [orc.orb_extract(oracle_api.orb_params(), f) for f in seq.frames]
    v = ktd.make_scene_vocab(np.concatenate([r["desc"] for r in res]), 3)
    ov = orc.bow_vocab_create(v["k"], v["L"], v["parent"], v["desc"], v["weight"], v["is_leaf"])
    gv = pkg.BowVocabulary(ctx, k=v["k"], L=v["L"], parent=v["parent"], desc=v["desc"], weight=v["weight"],
                           is_leaf=v["is_leaf"])
    fe = FrontEnd(ctx, seq.rows, seq.cols, seq.camera(pkg), max_batch=3)
    try:
        fe.reserve_local_map(4096)
        fe.reserve_keyframe_track(1, 1500)
        kfs = [ktd.keyframe(orc, ov, seq, res, 1, np.random.default_rng(4))]
        # frame 0: motion track stands; 1: motion track fails; 2: motion model unusable
        mot, out, wants, stage, lout, lwants = ktd.run_case(orc, pkg, fe, ov, gv, seq, res, ts, kfs, [0, 0, 0],
                                                            [1, 1, 0], fail=(1,), seed=5)
        assert stage == [0, 1, 1], stage
        ktd.compare(out, wants, stage)
        lmd.compare(lout, lwants)
        assert all(out["num_valid"][b] >= 20 for b in (1, 2)), out["num_valid"]
        print(f"smoke keyframe track ok: stage {stage}, BoW matches {list(out['num_bow_matches'])}, "
              f"num_valid {list(out['num_valid'])}, local map num_tracked {list(lout['num_tracked'])}, bit-exact")
    finally:
        fe.close()
        gv.close()
        orc.bow_vocab_destroy(ov)
