"""smoke(): one relocalisation query against a three-keyframe BoW database on the GPU, equal to the restatement."""
from __future__ import annotations

import numpy as np

import bow_data
import bow_db_data as bdd


def run(pkg, ctx):
    v = bow_data.make_vocab(5, k=10, L=3)
    voc = pkg.capi.BowVocabulary(ctx, k=v["k"], L=v["L"], parent=v["parent"], desc=v["desc"], weight=v["weight"],
                                 is_leaf=v["is_leaf"])
    db, vecs, cov, queries, _ = bdd.crafted()
    dev = pkg.capi.BowDatabase(ctx, voc, 10, 32)
    ks = sorted(db.vec)
    dev.add(ks, [db.vec[k] for k in ks])
    dev.erase([7])
    got, status = dev.relocalization_candidates(queries[:1], cov)
    want = db.relocalization_candidates(queries[0], cov)
    assert list(got[0]) == want and int(status[0]) == 0, (got, want)
    dev.close()
    voc.close()
