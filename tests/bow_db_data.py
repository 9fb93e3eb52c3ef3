"""Pure-Python restatement of data::bow_database (data/bow_database.cc:47-378) and DBoW2::L1Scoring::score, plus
seeded database scenes.  Keyframes are table indices; a vector is (ascending word ids, float64 values).  Float steps are
taken in numpy float32, as the reference takes them in float."""
from __future__ import annotations

from pathlib import Path

import numpy as np

F = np.float32
GOLDEN_SUBTREE = Path(__file__).resolve().parent / "golden" / "orb_vocab_subtree.npz"


def l1_score(a, b) -> np.float32:
    """L1Scoring::score(a, b): over the common words in ascending order s += |v - w| - |v| - |w| (double), then -s / 2,
    cast to float by bow_database / loop_detector."""
    wa, va = a
    wb, vb = b
    s, i, j = 0.0, 0, 0
    while i < len(wa) and j < len(wb):
        if wa[i] == wb[j]:
            vi, wi = float(va[i]), float(vb[j])
            s += abs(vi - wi) - abs(vi) - abs(wi)
            i += 1
            j += 1
        elif wa[i] < wb[j]:
            i += 1
        else:
            j += 1
    return F(-s / 2.0)


class Database:
    """keyfrms_in_node_ as word -> list of keyframes in insertion order; vectors outlive membership."""

    def __init__(self):
        self.vec = {}
        self.inv = {}

    def add(self, k, vec):  # add_keyframe (:47-56)
        self.vec[k] = (np.asarray(vec[0], np.int64), np.asarray(vec[1], np.float64))
        for w in self.vec[k][0]:
            self.inv.setdefault(int(w), []).append(k)

    def erase(self, k):  # erase_keyframe (:58-83)
        for w in self.vec[k][0]:
            lst = self.inv.get(int(w))
            if lst and k in lst:
                lst.remove(k)

    def members(self):
        return sorted({k for lst in self.inv.values() for k in lst})

    def _candidates(self, qvec, cov, reject, min_score):
        count, init = {}, set()
        for w in qvec[0]:  # set_candidates_sharing_words (:248-287)
            for k in self.inv.get(int(w), []):
                if k not in count:
                    count[k] = 0
                    if k not in reject:
                        init.add(k)
                count[k] += 1
        if not init:
            return []
        mx = max(count[k] for k in init)
        min_common = int(F(0.8) * F(mx))
        scores = {k: l1_score(qvec, self.vec[k]) for k in init if min_common < count[k]}  # compute_scores
        if not scores:
            return []
        pairs = [(scores[k], k) for k in init if min_common < count[k] and min_score <= scores[k]]
        if not pairs:
            return []
        best_total, totals = F(min_score), []
        for s, k in pairs:  # align_total_scores_and_keyframes (:333-378)
            total, best, bk = F(s), F(s), k
            for c in (cov[k] if k < len(cov) else [])[:10]:
                if c in init and min_common < count[c]:
                    total = F(total + scores[c])
                    if best < scores[c]:
                        best, bk = scores[c], c
            totals.append((total, bk))
            if best_total < total:
                best_total = total
        min_total = F(F(0.75) * best_total)
        return sorted({bk for total, bk in totals if min_total < total})

    def relocalization_candidates(self, qvec, cov):  # :170-236
        return self._candidates(qvec, cov, set(), F(0.0))

    def loop_candidates(self, qk, min_score, connected, cov):  # :97-168
        return self._candidates(self.vec[qk], cov, set(connected) | {qk}, F(min_score))


def normalise(words, vals):
    vals = np.asarray(vals, np.float64)
    norm = 0.0
    for v in vals:
        norm += abs(v)
    return np.asarray(words, np.int64), (vals / norm if norm > 0 else vals)


def random_vector(rng, pool, n):
    words = np.sort(rng.choice(pool, size=min(n, len(pool)), replace=False))
    return normalise(words, rng.uniform(0.05, 3.0, len(words)))


def subtree_words():
    """(word ids, idf weights) of the shipped vocabulary's golden subtree leaves."""
    d = np.load(GOLDEN_SUBTREE)
    leaf = d["is_leaf"] > 0
    return d["word_id"][leaf].astype(np.int64), d["weight"][leaf].astype(np.float32)


def subtree_vector(rng, n_rows):
    """A frame's bow_vec_ over the golden subtree: n_rows keypoints fall on random leaves, folded as capi.fold_bow does
    (weight > 0 rows, summed in row order, L1-normalised)."""
    words, weights = subtree_words()
    pick = rng.integers(0, len(words), n_rows)
    vec = {}
    for i in pick:
        if weights[i] > 0:
            vec[int(words[i])] = vec.get(int(words[i]), 0.0) + float(weights[i])
    ws = np.array(sorted(vec), np.int64)
    return normalise(ws, [vec[int(w)] for w in ws])


def random_graph(rng, K, max_cov=14):
    """Per keyframe index a covisibility list (distinct, not itself), longer than 10 for some."""
    cov = []
    for k in range(K):
        n = int(rng.integers(0, max_cov + 1))
        others = np.array([j for j in range(K) if j != k], np.int64)
        cov.append([int(x) for x in rng.choice(others, size=min(n, len(others)), replace=False)] if len(others) else [])
    return cov


def scene(seed, K, pool=60, words_per_kf=(5, 30), erase_frac=0.1):
    """A database of K keyframes over a pool of `pool` words (heavy sharing), a few erased, plus its graph."""
    rng = np.random.default_rng(seed)
    pool_ids = np.sort(rng.choice(5000, size=pool, replace=False))
    db = Database()
    vecs = []
    for k in range(K):
        v = random_vector(rng, pool_ids, int(rng.integers(*words_per_kf)))
        vecs.append(v)
        db.add(k, v)
    erased = [k for k in range(K) if rng.random() < erase_frac]
    for k in erased:
        db.erase(k)
    return db, vecs, erased, random_graph(rng, K), pool_ids, rng


def _vec(words, vals):
    return np.asarray(words, np.int64), np.asarray(vals, np.float64)


def crafted():
    """A small database whose scores are exact binary fractions (score = sum of min(v, w) over common words), built to
    hit every boundary of the selection.  Query words 0..15 at 1/16 each; min_common is int(0.8 * 16) = 12.
    Returns (db, vecs by index, cov, reloc queries, loop queries (query_kf, min_score, connected))."""
    q16 = np.arange(16)
    vecs = {
        0: _vec(q16, np.full(16, 1 / 16)),                                   # A: score 1
        1: _vec(list(q16) + [40], list(np.full(16, 3 / 64)) + [0.25]),      # B: score 0.75, total exactly 0.75 * best
        2: _vec(list(range(13)) + [41, 42, 43], np.full(16, 1 / 16)),        # D: 13 words, score 0.8125
        3: _vec(list(range(12)) + [44, 45, 46, 47], np.full(16, 1 / 16)),    # 12 words = min_common: never scored
        4: _vec(list(q16) + [48], list(np.full(16, 11 / 256)) + [0.3125]),  # E: score 0.6875 (< 0.75)
        5: _vec(q16, np.full(16, 1 / 16)),                                   # A2: ties A
        6: _vec(list(range(14)) + [49, 50], np.full(16, 1 / 16)),            # X: 14 words, score 0.875
        7: _vec(q16, np.full(16, 1 / 16)),                                   # erased copy of A
        8: _vec([], []),                                                     # an empty vector
        9: _vec([60, 61, 62], [0.5, 0.25, 0.25]),                            # shares nothing with the query
    }
    db = Database()
    for k in sorted(vecs):
        db.add(k, vecs[k])
    db.erase(7)
    # A's covisibilities: E (score below any min_score) and D; X's: A2 then A (a tie, the first wins) -> duplicates
    cov = [[4, 2], [], [], [0], [], [], [5, 0], [0], [], []]
    reloc = [vecs[0], _vec(list(q16) + [999], list(np.full(16, 1 / 17)) + [1 / 17]), _vec([], []), _vec([80, 81], [0.5, 0.5]),
             _vec([70], [1.0])]
    loops = [(0, F(0.75), []), (0, F(0.8125), [5]), (0, F(1.0), [1, 2, 3, 4, 5, 6]), (6, F(0.0), [0]),
             (9, F(0.0), []), (8, F(0.0), [])]
    return db, vecs, cov, reloc, loops


# ---------------------------------------------------------------------------------------------------- native oracle
def oracle():
    """The oracle library with the restypes of oracle/bow_db_oracle.cc's entries declared."""
    import ctypes

    import oracle_api

    lib = oracle_api.lib()
    lib.orc_bow_db_create.restype = ctypes.c_void_p
    lib.orc_bow_score.restype = ctypes.c_float
    for f in ("orc_bow_db_destroy", "orc_bow_db_add", "orc_bow_db_erase", "orc_bow_db_reloc", "orc_bow_db_loop"):
        getattr(lib, f).restype = None
    return lib


def _flat(vecs, part, dtype):
    off = np.zeros(len(vecs) + 1, np.int32)
    for i, v in enumerate(vecs):
        off[i + 1] = off[i] + len(v[0])
    flat = np.zeros(max(int(off[-1]), 1), dtype)
    if off[-1]:
        flat[:off[-1]] = np.concatenate([np.asarray(v[part], dtype) for v in vecs])
    return off, flat


def _graph_csr(cov):
    off = np.zeros(len(cov) + 1, np.int32)
    for k, c in enumerate(cov):
        off[k + 1] = off[k] + len(c)
    return off, np.array([c for lst in cov for c in lst] or [0], np.int32)


class NativeDatabase:
    """The C++ restatement (oracle/bow_db_oracle.cc) behind the same methods as Database."""

    def __init__(self, lib):
        import ctypes
        self._C = ctypes
        self.lib = lib
        self.h = ctypes.c_void_p(lib.orc_bow_db_create())

    def close(self):
        if self.h:
            self.lib.orc_bow_db_destroy(self.h)
            self.h = None

    def _p(self, a):
        return a.ctypes.data_as(self._C.c_void_p)

    def add(self, k, vec):
        w = np.ascontiguousarray(vec[0], np.int32)
        v = np.ascontiguousarray(vec[1], np.float64)
        self.lib.orc_bow_db_add(self.h, self._C.c_int32(k), self._C.c_int(len(w)), self._p(w), self._p(v))

    def erase(self, k):
        self.lib.orc_bow_db_erase(self.h, self._C.c_int32(k))

    def score(self, a, b):
        wa, va = np.ascontiguousarray(a[0], np.int32), np.ascontiguousarray(a[1], np.float64)
        wb, vb = np.ascontiguousarray(b[0], np.int32), np.ascontiguousarray(b[1], np.float64)
        return F(self.lib.orc_bow_score(len(wa), self._p(wa), self._p(va), len(wb), self._p(wb), self._p(vb)))

    def relocalization_candidates_batch(self, queries, cov, max_candidates=1 << 14):
        """Lists per query (None where the list exceeds max_candidates)."""
        C = self._C
        off, words = _flat(queries, 0, np.int32)
        _, vals = _flat(queries, 1, np.float64)
        goff, gkf = _graph_csr(cov)
        n = len(queries)
        cand = np.zeros((max(n, 1), max_candidates), np.int32)
        num = np.zeros(max(n, 1), np.int32)
        self.lib.orc_bow_db_reloc(self.h, C.c_int(n), self._p(off), self._p(words), self._p(vals), C.c_int(len(cov)),
                                  self._p(goff), self._p(gkf), C.c_int(max_candidates), self._p(cand), self._p(num))
        return [None if num[q] < 0 else list(cand[q, :num[q]]) for q in range(n)]

    def loop_candidates_batch(self, loops, cov, max_candidates=1 << 14):
        C = self._C
        n = len(loops)
        qk = np.array([q[0] for q in loops], np.int32)
        ms = np.array([q[1] for q in loops], np.float32)
        coff, ckf = _graph_csr([q[2] for q in loops])
        goff, gkf = _graph_csr(cov)
        cand = np.zeros((max(n, 1), max_candidates), np.int32)
        num = np.zeros(max(n, 1), np.int32)
        self.lib.orc_bow_db_loop(self.h, C.c_int(n), self._p(qk), self._p(ms), self._p(coff), self._p(ckf),
                                 C.c_int(len(cov)), self._p(goff), self._p(gkf), C.c_int(max_candidates),
                                 self._p(cand), self._p(num))
        return [None if num[q] < 0 else list(cand[q, :num[q]]) for q in range(n)]


def native_copy(lib, db):
    """A NativeDatabase holding the same vectors and members as the Python Database db (insertion order kept)."""
    nat = NativeDatabase(lib)
    members = set(db.members())
    for k in sorted(db.vec):
        nat.add(k, db.vec[k])
    for k in sorted(db.vec):
        if k not in members and len(db.vec[k][0]):
            nat.erase(k)
    return nat
