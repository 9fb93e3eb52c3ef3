"""The C++ restatement of data::bow_database (oracle/bow_db_oracle.cc, the reference's containers) against the independent
Python restatement (tests/bow_db_data.py): candidate list for list and score for score, on the boundary scene, seeded
synthetic databases and vectors over the shipped vocabulary's golden subtree."""
from __future__ import annotations

import numpy as np
import pytest

import bow_db_data as bdd


@pytest.fixture(scope="module")
def lib():
    return bdd.oracle()


def _same(lib, db, queries, loops, cov):
    nat = bdd.native_copy(lib, db)
    assert nat.relocalization_candidates_batch(queries, cov) == [db.relocalization_candidates(q, cov) for q in queries]
    assert nat.loop_candidates_batch(loops, cov) == [db.loop_candidates(*q, cov) for q in loops]
    for a in sorted(db.vec):
        for b in sorted(db.vec)[:8]:
            assert nat.score(db.vec[a], db.vec[b]).tobytes() == bdd.l1_score(db.vec[a], db.vec[b]).tobytes()
    nat.close()


def test_crafted(lib):
    db, vecs, cov, queries, loops = bdd.crafted()
    _same(lib, db, queries, loops + [(0, np.float32(0.75), [5, 6, 2, 4])], cov)


@pytest.mark.parametrize("seed", [3, 4, 5, 6])
def test_random_scenes(lib, seed):
    K = 80
    db, vecs, erased, cov, pool, rng = bdd.scene(seed, K)
    queries = [bdd.random_vector(rng, pool, int(rng.integers(3, 40))) for _ in range(8)] + [vecs[1]]
    loops = []
    for _ in range(8):
        qk = int(rng.integers(0, K))
        conn = [int(x) for x in rng.choice(K, size=int(rng.integers(0, 15)), replace=False)]
        loops.append((qk, bdd.l1_score(vecs[qk], vecs[conn[0]]) if conn else np.float32(0.0), conn))
    _same(lib, db, queries, loops, cov)


def test_subtree_vectors(lib):
    rng = np.random.default_rng(17)
    K = 40
    db = bdd.Database()
    for k in range(K):
        db.add(k, bdd.subtree_vector(rng, int(rng.integers(20, 300))))
    db.erase(3)
    cov = bdd.random_graph(rng, K)
    queries = [bdd.subtree_vector(rng, 200) for _ in range(6)]
    loops = [(k, np.float32(0.01 * k), [(k + 1) % K, (k + 7) % K]) for k in range(0, K, 5)]
    _same(lib, db, queries, loops, cov)


def test_overflow_reported(lib):
    db, vecs, cov, queries, loops = bdd.crafted()
    nat = bdd.native_copy(lib, db)
    want = db.relocalization_candidates(queries[0], cov)
    assert len(want) >= 1
    assert nat.relocalization_candidates_batch(queries[:1], cov, max_candidates=len(want))[0] == want
    assert nat.relocalization_candidates_batch(queries[:1], cov, max_candidates=len(want) - 1)[0] is None
    nat.close()
