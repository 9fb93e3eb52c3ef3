"""The keyframe BoW database on the GPU (plp_bow_db) against the Python restatement of data::bow_database
(tests/bow_db_data.py) and its C++ restatement (tests/bow_db_oracle.cc): candidate lists equal, scores bit-equal, at 1,
10, 128 and 3000 keyframes, single-keyframe adds and erases on a populated database, and the refusals."""
from __future__ import annotations

import numpy as np
import pytest

import bow_data
import bow_db_data as bdd

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def vocab(plp, ctx):
    v = bow_data.make_vocab(5, k=10, L=4)
    voc = plp.capi.BowVocabulary(ctx, k=v["k"], L=v["L"], parent=v["parent"], desc=v["desc"], weight=v["weight"],
                                 is_leaf=v["is_leaf"])
    yield voc
    voc.close()


def load(plp, ctx, vocab, db, K, W):
    dev = plp.capi.BowDatabase(ctx, vocab, K, W)
    ks = sorted(db.vec)
    dev.add(ks, [db.vec[k] for k in ks])
    gone = [k for k in ks if k not in set(db.members()) and len(db.vec[k][0])]
    if gone:
        dev.erase(gone)
    return dev


@pytest.fixture(scope="module")
def orc(tmp_path_factory):
    return bdd.build_oracle(tmp_path_factory.mktemp("bow_db_oracle"))


def check(dev, db, K, queries, loops, cov, orc=None):
    got, status = dev.relocalization_candidates(queries, cov)
    want = [db.relocalization_candidates(q, cov) for q in queries]
    assert [list(g) for g in got] == want
    assert list(status) == [0] * len(queries)
    got_l, status = dev.loop_candidates([q[0] for q in loops], [q[1] for q in loops], [q[2] for q in loops], cov)
    want_l = [db.loop_candidates(*q, cov) for q in loops]
    assert [list(g) for g in got_l] == want_l
    if orc is not None:
        nat = bdd.native_copy(orc, db)
        assert nat.relocalization_candidates_batch(queries, cov) == want
        assert nat.loop_candidates_batch(loops, cov) == want_l
        nat.close()
    a = np.array([q[0] for q in loops] * 2, np.int32)
    b = np.array([(q[2][0] if q[2] else q[0]) for q in loops] + list(range(len(loops))), np.int32) % K
    s = dev.score_pairs(a, b)
    assert s.tobytes() == np.array([bdd.l1_score(db.vec[x], db.vec[y]) for x, y in zip(a, b)], np.float32).tobytes()


def test_crafted(plp, ctx, vocab):
    db, vecs, cov, queries, loops = bdd.crafted()
    dev = load(plp, ctx, vocab, db, 10, 32)
    check(dev, db, 10, queries, loops, cov)
    dev.close()


def test_one_keyframe(plp, ctx, vocab):
    rng = np.random.default_rng(1)
    db = bdd.Database()
    v = bdd.random_vector(rng, np.arange(200), 40)
    db.add(0, v)
    dev = load(plp, ctx, vocab, db, 1, 64)
    check(dev, db, 1, [v, bdd.random_vector(rng, np.arange(200), 30)], [(0, np.float32(0.0), [])], [[]])
    dev.close()


@pytest.mark.parametrize("K,pool", [(128, 300), (3000, 2000)])
def test_scene(plp, ctx, vocab, orc, K, pool):
    nw = vocab.info()["num_words"]
    db, vecs, erased, cov, pool_ids, rng = bdd.scene(K, K, pool=min(pool, nw), words_per_kf=(20, 120))
    pool_ids = pool_ids % nw
    # the scene's word ids are drawn below 5000: keep them inside this vocabulary
    db2 = bdd.Database()
    for k in range(K):
        w, val = vecs[k]
        w2, idx = np.unique(w % nw, return_index=True)
        db2.add(k, bdd.normalise(w2, val[idx]))
    for k in erased:
        db2.erase(k)
    dev = load(plp, ctx, vocab, db2, K, 128)
    queries = [db2.vec[int(k)] for k in rng.integers(0, K, 20)] + \
              [bdd.random_vector(rng, np.unique(pool_ids), 80) for _ in range(20)]
    loops = []
    for _ in range(20):
        qk = int(rng.integers(0, K))
        conn = [int(x) for x in rng.choice(K, size=int(rng.integers(1, 20)), replace=False)]
        loops.append((qk, bdd.l1_score(db2.vec[qk], db2.vec[conn[0]]), conn))
    check(dev, db2, K, queries, loops, cov, orc)
    # one keyframe at a time, as the mapping thread adds and erases them: the index stays equal to the reference's
    for k in (K // 3, K - 1):
        if k in set(db2.members()):
            db2.erase(k)
            dev.erase([k])
    check(dev, db2, K, queries[:10], loops[:10], cov)
    rng2 = np.random.default_rng(K + 1)
    k = next(k for k in range(K) if k not in set(db2.members()))
    v = bdd.random_vector(rng2, np.unique(pool_ids), 100)
    db2.add(k, v)
    dev.add([k], [v])  # re-adding an erased index replaces its stored vector
    check(dev, db2, K, queries[:10] + [v], loops[:10] + [(k, np.float32(0.0), [])], cov)
    dev.close()


def test_refusals(plp, ctx, vocab):
    nw = vocab.info()["num_words"]
    dev = plp.capi.BowDatabase(ctx, vocab, 4, 3)
    with pytest.raises(plp.capi.PlpError, match="status 1"):
        dev.add([0], [(np.array([nw]), np.array([1.0]))])              # word outside the vocabulary
    with pytest.raises(plp.capi.PlpError, match="status 1"):
        dev.add([0], [(np.array([1, 2, 3, 4]), np.full(4, 0.25))])     # longer than max_words_per_keyframe
    with pytest.raises(plp.capi.PlpError, match="status 1"):
        dev.add([0], [(np.array([2, 1]), np.full(2, 0.5))])            # not ascending
    with pytest.raises(plp.capi.PlpError, match="status 1"):
        dev.erase([0])                                                 # not a member: nothing was stored
    dev.add([0], [(np.array([1, 2]), np.full(2, 0.5))])
    with pytest.raises(plp.capi.PlpError, match="status 1"):
        dev.add([0], [(np.array([1]), np.array([1.0]))])               # already a member
    with pytest.raises(plp.capi.PlpError, match="status 1"):
        dev.score_pairs([0], [1])                                      # no stored vector
    got, status = dev.relocalization_candidates([(np.array([1, 2]), np.full(2, 0.5))], [[], [], [], []])
    assert [list(g) for g in got] == [[0]] and list(status) == [0]
    got, status = dev.relocalization_candidates([(np.array([1, 2]), np.full(2, 0.5))], [[], [], [], []],
                                                max_candidates=0)
    assert list(status) == [1]
    dev.close()
    with pytest.raises(plp.capi.PlpError, match="status 4"):
        plp.capi.BowDatabase(ctx, vocab, 1 << 30, 1 << 10)
