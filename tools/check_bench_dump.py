#!/usr/bin/env python
"""Check what `bench.py --dump-outputs DIR` wrote against the CPU oracle.

    python tools/check_bench_dump.py DIR --seed 1234 --batch 512 --streams 2

Rebuilds the headline inputs of rank 0 the way bench.py does: sub-batch c of `streams` holds batch // streams problems
from build_inputs(batch // streams, seed + 37 c); their predicted poses come from default_rng(seed + 37 c) in problem
order; the last-frame landmarks back-project the keypoints extracted from frame t - 1 (the oracle's extraction here,
which the GPU parity tests prove equal to the GPU's).  Then it runs the oracle chain extract -> match_current_and_last_frames
(+ widened retry) -> pose_optimize -> discard_outliers and compares:
  every frame        n_keypoints, num_valid, n_inliers, status (exact), pose (<= 1e-4 relative), lm_iters (zero iff
                     the oracle's is; the total within scene.LM_ITERS_TOTAL_TOL, see there why not per frame)
  the sampled frames keypoints (every field), descriptors, matched landmark index (exact)
Exits 1 on any mismatch.  CPU only."""
from __future__ import annotations

import argparse
import importlib.util
import os
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests"))
POSE_REL_TOL = 1e-4


def _bench():
    spec = importlib.util.spec_from_file_location("plp_bench", ROOT / "bench.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def oracle_outputs(seed: int, batch: int, streams: int, threads: int | None = None):
    """Per-frame oracle results of the headline inputs, frames in bench.py's dump order (sub-batch after sub-batch)."""
    import oracle_api
    import scene
    bench = _bench()
    pkg = bench._load_pkg()
    orc = oracle_api.Oracle()
    p = oracle_api.orb_params()
    bs = batch // streams
    out = []
    with ThreadPoolExecutor(max_workers=threads or os.cpu_count() or 1) as ex:
        for c in range(streams):
            sub_seed = seed + 37 * c
            seqs, _, t_idx = bench.build_inputs(bs, sub_seed)
            rng = np.random.default_rng(sub_seed)
            preds = [seqs[s].predicted_pose(t, rng) for (s, t) in t_idx]
            keys = sorted({(s, u) for (s, t) in t_idx for u in (t - 1, t)})
            ext = dict(zip(keys, ex.map(lambda k: orc.orb_extract(p, seqs[k[0]].frames[k[1]]), keys)))
            for b, (s, t) in enumerate(t_idx):
                res = {t - 1: ext[(s, t - 1)], t: ext[(s, t)]}
                m, T, nv, n_inl, iters = scene.oracle_track(orc, pkg, seqs[s], res, t, preds[b])
                out.append(dict(kps=res[t]["kps"], desc=res[t]["desc"], matched=m, pose=T, num_valid=nv,
                                n_inliers=n_inl, lm_iters=iters))
    return out


def check(dump_dir: Path, seed: int, batch: int, streams: int, threads: int | None = None) -> list[str]:
    """Mismatches between the dump and the oracle (empty: none)."""
    import scene
    d = {f.stem: np.load(f) for f in Path(dump_dir).glob("*.npy")}
    ref = oracle_outputs(seed, batch, streams, threads)
    bad = []
    n_frames = len(ref)
    if len(d["n_keypoints"]) != n_frames:
        return [f"dump has {len(d['n_keypoints'])} frames, expected {n_frames}"]
    for f, r in enumerate(ref):
        for k in ("num_valid", "n_inliers"):
            if d[k][f] != r[k]:
                bad.append(f"frame {f}: {k} {d[k][f]:g} vs {r[k]}")
        if (d["lm_iters"][f] == 0) != (r["lm_iters"] == 0):
            bad.append(f"frame {f}: lm_iters {d['lm_iters'][f]:g} vs {r['lm_iters']}")
        if d["n_keypoints"][f] != len(r["kps"]):
            bad.append(f"frame {f}: n_keypoints {d['n_keypoints'][f]:g} vs {len(r['kps'])}")
        if d["status"][f] != 0:
            bad.append(f"frame {f}: status {d['status'][f]:g}")
        rel = np.linalg.norm(d["pose"][f] - r["pose"]) / np.linalg.norm(r["pose"])
        if not rel <= POSE_REL_TOL:
            bad.append(f"frame {f}: pose differs by {rel:.3g} relative")
    got_it, want_it = float(d["lm_iters"].sum()), float(sum(r["lm_iters"] for r in ref))
    if not abs(got_it - want_it) <= scene.LM_ITERS_TOTAL_TOL * want_it + scene.LM_ITERS_SLACK:
        bad.append(f"lm_iters: {got_it:g} in total vs the oracle's {want_it:g}")
    off = 0
    for f in d["sample_frames"].astype(np.int64):
        r = ref[f]
        n = len(r["kps"])
        sl = slice(off, off + n)
        off += n
        for k in r["kps"].dtype.names:
            if not np.array_equal(d[f"kp_{k}"][sl], r["kps"][k].astype(np.float64)):
                bad.append(f"frame {f}: keypoint field {k}")
        if not np.array_equal(d["descriptors"][sl], r["desc"].astype(np.float32)):
            bad.append(f"frame {f}: descriptors")
        if not np.array_equal(d["matched"][sl], r["matched"].astype(np.float64)):
            bad.append(f"frame {f}: matched landmark indices")
    if off != len(d["matched"]):
        bad.append(f"sampled keypoint rows: {len(d['matched'])} in the dump, {off} expected")
    return bad


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("dir", type=Path)
    ap.add_argument("--seed", type=int, default=1234)
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--streams", type=int, default=2)
    ap.add_argument("--threads", type=int, default=None, help="host threads for the oracle extraction (default: all)")
    a = ap.parse_args()
    bad = check(a.dir, a.seed, a.batch, a.streams, a.threads)
    for line in bad[:50]:
        print(line)
    print(f"{len(bad)} mismatches")
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
