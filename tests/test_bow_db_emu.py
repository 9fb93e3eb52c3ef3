"""The keyframe BoW database's device code (csrc/bow_db_kernels.cuh) run on the CPU through tests/cta_emu: index build,
common-word counts, scores and the candidate selection, each equal to the Python restatement (tests/bow_db_data.py)."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import bow_db_data as bdd
import emu_build

_P = C.c_void_p
NUM_WORDS = 5000


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return emu_build.emu("bowdb_emu", tmp_path_factory)


def _ptr(a):
    return a.ctypes.data_as(_P)


def _csr(vecs, dtype, part):
    off = np.zeros(len(vecs) + 1, np.int32)
    for i, v in enumerate(vecs):
        off[i + 1] = off[i] + len(v[0])
    flat = np.zeros(max(int(off[-1]), 1), dtype)
    if off[-1]:
        flat[:off[-1]] = np.concatenate([np.asarray(v[part], dtype) for v in vecs])
    return off, flat


def build(emu, db, K, W):
    """Loads the restatement's database into the emulated one; returns the device index (offsets, lists)."""
    vecs = [db.vec.get(k, (np.zeros(0, np.int64), np.zeros(0))) for k in range(K)]
    off, words = _csr(vecs, np.int32, 0)
    _, vals = _csr(vecs, np.float64, 1)
    has = np.array([k in db.vec for k in range(K)], np.uint8)
    members = set(db.members())
    member = np.array([k in members for k in range(K)], np.uint8)
    num_words = max(NUM_WORDS, int(words.max()) + 1)
    inv_off = np.zeros(num_words + 1, np.int32)
    inv_kf = np.zeros(K * W, np.int32)
    emu.emu_bdb_build(C.c_int(K), C.c_int(W), C.c_int(num_words), _ptr(off), _ptr(words), _ptr(vals), _ptr(has),
                      _ptr(member), _ptr(inv_off), _ptr(inv_kf))
    return inv_off, inv_kf


def graph(cov, K):
    off = np.zeros(K + 1, np.int32)
    for k in range(K):
        off[k + 1] = off[k] + (len(cov[k]) if k < len(cov) else 0)
    flat = np.array([c for k in range(min(K, len(cov))) for c in cov[k]] or [0], np.int32)
    return off, flat


def reloc(emu, K, vecs, cov, max_candidates=64):
    n = len(vecs)
    off, words = _csr(vecs, np.int32, 0)
    _, vals = _csr(vecs, np.float64, 1)
    goff, gkf = graph(cov, K)
    cand = np.full((n, max_candidates), -7, np.int32)
    num = np.full(n, -7, np.int32)
    status = np.full(n, -7, np.int32)
    emu.emu_bdb_query(C.c_int(n), _ptr(off), _ptr(words), _ptr(vals), None, None, None, None, C.c_int(K), _ptr(goff), _ptr(gkf), C.c_int(max_candidates),
                      _ptr(cand), _ptr(num), _ptr(status))
    return [list(cand[q, :num[q]]) for q in range(n)], list(status)


def loop(emu, K, queries, cov, max_candidates=64):
    n = len(queries)
    qk = np.array([q[0] for q in queries], np.int32)
    ms = np.array([q[1] for q in queries], np.float32)
    coff = np.zeros(n + 1, np.int32)
    for i, q in enumerate(queries):
        coff[i + 1] = coff[i] + len(q[2])
    ckf = np.array([c for q in queries for c in q[2]] or [0], np.int32)
    goff, gkf = graph(cov, K)
    cand = np.full((n, max_candidates), -7, np.int32)
    num = np.full(n, -7, np.int32)
    status = np.full(n, -7, np.int32)
    emu.emu_bdb_query(C.c_int(n), None, None, None, _ptr(qk), _ptr(ms), _ptr(coff), _ptr(ckf), C.c_int(K),
                      _ptr(goff), _ptr(gkf), C.c_int(max_candidates), _ptr(cand), _ptr(num), _ptr(status))
    return [list(cand[q, :num[q]]) for q in range(n)], list(status)


def test_index_lists_members_ascending(emu):
    db, vecs, erased, cov, pool, rng = bdd.scene(1, 40)
    K, W = 40, 32
    inv_off, inv_kf = build(emu, db, K, W)
    for w in range(NUM_WORDS):
        got = list(inv_kf[inv_off[w]:inv_off[w + 1]])
        assert got == sorted(db.inv.get(w, [])), w


def test_crafted_boundaries(emu):
    db, vecs, cov, queries, loops = bdd.crafted()
    K = 10
    build(emu, db, K, 32)
    got, status = reloc(emu, K, queries, cov)
    want = [db.relocalization_candidates(q, cov) for q in queries]
    assert got == want and status == [0] * len(queries)
    # the boundaries the scene is built for
    assert 1 not in want[0]          # total exactly 0.75 x best: excluded
    assert 3 not in want[0]          # common words exactly min_common: excluded
    assert 7 not in want[0]          # erased
    assert want[2] == [] and want[3] == [] and want[4] == []  # empty vector, no shared word, unknown word
    got, status = loop(emu, K, loops, cov)
    want = [db.loop_candidates(*q, cov) for q in loops]
    assert got == want and status == [0] * len(loops)
    assert want[2] == []             # every sharer rejected
    pairs = [(k, q) for k in (0, 1, 2, 4, 6) for q in (0, 5)]
    out = np.zeros(len(pairs), np.float32)
    emu.emu_bdb_pairs(C.c_int(len(pairs)), _ptr(np.array([p[0] for p in pairs], np.int32)),
                      _ptr(np.array([p[1] for p in pairs], np.int32)), _ptr(out))
    assert [float(x) for x in out] == [float(bdd.l1_score(db.vec[a], db.vec[b])) for a, b in pairs]


def test_min_score_equal_to_a_score_is_included(emu):
    db, vecs, cov, _, _ = bdd.crafted()
    build(emu, db, 10, 32)
    # B (index 1) scores exactly 0.75 against A: with min_score 0.75 it is a pair (its total is its score)
    got, _ = loop(emu, 10, [(0, np.float32(0.75), [5, 6, 2, 4])], [[] for _ in range(10)])
    assert got == [db.loop_candidates(0, np.float32(0.75), [5, 6, 2, 4], [[] for _ in range(10)])]
    assert 1 in got[0]


@pytest.mark.parametrize("seed", [3, 4, 5])
def test_random_scenes(emu, seed):
    K = 60
    db, vecs, erased, cov, pool, rng = bdd.scene(seed, K)
    build(emu, db, K, 32)
    queries = [bdd.random_vector(rng, pool, int(rng.integers(3, 40))) for _ in range(5)] + [vecs[2]]
    got, status = reloc(emu, K, queries, cov)
    assert got == [db.relocalization_candidates(q, cov) for q in queries]
    assert status == [0] * len(queries)
    loops = []
    for _ in range(5):
        qk = int(rng.integers(0, K))
        conn = [int(x) for x in rng.choice(K, size=int(rng.integers(0, 12)), replace=False)]
        ms = bdd.l1_score(vecs[qk], vecs[conn[0]]) if conn else np.float32(0.0)
        loops.append((qk, ms, conn))
    got, status = loop(emu, K, loops, cov)
    assert got == [db.loop_candidates(*q, cov) for q in loops]


def test_subtree_vectors_and_overflow(emu):
    rng = np.random.default_rng(7)
    K = 24
    db = bdd.Database()
    vecs = [bdd.subtree_vector(rng, int(rng.integers(20, 200))) for _ in range(K)]
    for k, v in enumerate(vecs):
        db.add(k, v)
    cov = bdd.random_graph(rng, K)
    build(emu, db, K, 400)
    queries = [bdd.subtree_vector(rng, 150) for _ in range(4)]
    want = [db.relocalization_candidates(q, cov) for q in queries]
    got, status = reloc(emu, K, queries, cov)
    assert got == want and status == [0] * 4
    small = max(1, max(len(w) for w in want) - 1)
    got, status = reloc(emu, K, queries, cov, max_candidates=small)
    for q in range(4):
        if len(want[q]) > small:
            assert status[q] == 1 and got[q] == []
        else:
            assert status[q] == 0 and got[q] == want[q]
    assert 1 in status
