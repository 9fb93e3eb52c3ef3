"""Times plp_bow_db relocalisation queries: 512 queries per batch against K keyframes whose bow_vec_ hold ~1000 words
drawn from a scene vocabulary, for K in {128, 1000, 10000}.  The device time is the host entry's wall time (upload of
the queries and graph, the query kernel, download).  The host column is the C++ restatement (oracle/bow_db_oracle.cc,
-O3, the reference's containers) on one thread over the same 512 queries.  Also timed: adding all K keyframes in one
call, and, on the full database, erasing one keyframe and adding it back (the mapping thread's per-keyframe cost).
Prints the card's name and power limit from the same run.

    python tools/bench_bow_db.py [--reps 5]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tests"))

import bow_data  # noqa: E402
import bow_db_data as bdd  # noqa: E402
from conftest import load_package  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    plp = load_package()
    ctx = plp.Context(0)
    v = bow_data.make_vocab(9, k=10, L=5)
    voc = plp.capi.BowVocabulary(ctx, k=v["k"], L=v["L"], parent=v["parent"], desc=v["desc"], weight=v["weight"],
                                 is_leaf=v["is_leaf"])
    nw = voc.info()["num_words"]
    orc = bdd.oracle()
    rng = np.random.default_rng(0)
    scene_words = np.sort(rng.choice(nw, size=min(nw, 8000), replace=False))  # the words one scene uses
    print(f"card: {card()}; vocabulary words: {nw}; scene words: {len(scene_words)}")
    for K in (128, 1000, 10000):
        db = bdd.Database()
        vecs = [bdd.random_vector(rng, scene_words, 1000) for _ in range(K)]
        for k, vec in enumerate(vecs):
            db.add(k, vec)
        cov = bdd.random_graph(rng, K, max_cov=10) if K <= 1000 else \
            [[int(x) for x in rng.choice(K, 10, replace=False) if x != k] for k in range(K)]
        dev = plp.capi.BowDatabase(ctx, voc, K, 1000)
        t0 = time.perf_counter()
        dev.add(list(range(K)), vecs)
        t_add = time.perf_counter() - t0
        single = []
        for k in (K // 2, K // 3, K - 1):
            t0 = time.perf_counter()
            dev.erase([k])
            t1 = time.perf_counter()
            dev.add([k], [vecs[k]])
            single.append((t1 - t0, time.perf_counter() - t1))
        queries = [bdd.random_vector(rng, scene_words, 1000) for _ in range(512)]
        dev.relocalization_candidates(queries[:8], cov)  # warm-up
        times = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            got, status = dev.relocalization_candidates(queries, cov)
            times.append(time.perf_counter() - t0)
        nat = bdd.native_copy(orc, db)
        t0 = time.perf_counter()
        want = nat.relocalization_candidates_batch(queries, cov, max_candidates=256)
        t_host = time.perf_counter() - t0
        nat.close()
        assert [list(g) if s == 0 else None for g, s in zip(got, status)] == want
        print(json.dumps(dict(K=K, device_ms_per_512=round(1e3 * float(np.median(times)), 3),
                              device_ms_min=round(1e3 * min(times), 3), add_all_ms=round(1e3 * t_add, 3),
                              erase_one_ms=round(1e3 * float(np.median([e for e, _ in single])), 3),
                              add_one_ms=round(1e3 * float(np.median([a for _, a in single])), 3),
                              oracle_one_thread_ms_per_512=round(1e3 * t_host, 1),
                              mean_candidates=float(np.mean([len(g) for g in got])),
                              statuses=sorted(set(int(s) for s in status)))))
        dev.close()
    voc.close()
    ctx.close()


if __name__ == "__main__":
    main()
