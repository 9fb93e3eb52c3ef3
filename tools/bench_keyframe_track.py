"""Time the batched keyframe tracker (bow_match_based_track) next to bench.py's headline step.

    python tools/bench_keyframe_track.py [--batch 512] [--steps 20] [--warmup 3] [--seed 1234]

bench.py's headline problems (bench.setup_front_end: 512 planar-sequence frames, ORB 1000 keypoints, motion tracking
on a high-priority tracking context).  Each sequence's frames t = 1..32 are grouped by four: frames 4g + 1 .. 4g + 4
share frame 4g as their reference keyframe (one to four frames back), extracted on the GPU without timing: 128 keyframes
for 512 frames.  The vocabulary is
synthetic, of the shipped shape (k = 10, L = 6), built from the scene's descriptors.  The script
  1. checks a seeded sample of active frames against the oracle chain;
  2. times step() alone and step() + track_keyframe() with no frame active (every motion track usable and
     successful: the call every batch pays), with about 5 % active and with every frame active (motion model
     unusable), alternately, with a device synchronise around each timed step;
  3. times the stage's kernels (plp_ctx_kernel_timing) for the three shares;
  4. times the oracle's host chain (transform, fold, bow_tree, pose optimiser) per frame.
Prints one JSON line with the card's name, power limit and SM clock read in the same run; writes nothing."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

sys.dont_write_bytecode = True
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
import bench  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else f"nvidia-smi failed: {q.stderr.strip()}"


def main():
    import keyframe_track_data as ktd
    import oracle_api
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1234)
    ap.add_argument("--sample", type=int, default=4)
    args = ap.parse_args()
    pkg = bench._load_pkg()
    ctx = pkg.Context(0)
    tctx = pkg.Context(0, high_priority=True)
    B = args.batch
    fe, frames, aux = bench.setup_front_end(pkg, ctx, B, args.seed, tctx)
    seqs, t_idx = aux["seqs"], aux["t_idx"]

    def sync():
        ctx.sync()
        tctx.sync()

    # the keyframes: frame 4g of the sequence for frames 4g + 1 .. 4g + 4, extracted on the GPU (untimed)
    kf_t = [4 * ((t - 1) // 4) for (_, t) in t_idx]
    fe.upload_images(np.stack([seqs[s].frames[k] for (s, _), k in zip(t_idx, kf_t)]))
    fe.extract(B)
    prev = fe.download_keypoints(B)
    fe.upload_images(frames)
    sync()
    orc = oracle_api.Oracle()
    rng = np.random.default_rng(args.seed)
    pool = np.concatenate([prev[b][1] for b in rng.choice(B, min(B, 16), replace=False)])
    v = ktd.make_scene_vocab(pool, args.seed)
    ov = orc.bow_vocab_create(v["k"], v["L"], v["parent"], v["desc"], v["weight"], v["is_leaf"])
    gv = pkg.BowVocabulary(tctx, k=v["k"], L=v["L"], parent=v["parent"], desc=v["desc"], weight=v["weight"],
                           is_leaf=v["is_leaf"])
    keys, kfs, kf_of_frame = {}, [], []
    for b, (s, t) in enumerate(t_idx):
        key = (s, kf_t[b])
        if key not in keys:
            k, d = prev[b]
            pos_w = seqs[s].backproject(seqs[s].poses[key[1]], k["x"].astype(np.float64), k["y"].astype(np.float64))
            _, _, fv = ktd.fold_bow(*orc.bow_transform(ov, d, 4))
            keys[key] = len(kfs)
            kfs.append(dict(t=key[1], desc=d, angle=k["angle"].astype(np.float32), valid=np.ones(len(d), np.uint8),
                            pos_w=pos_w, fv=fv))
        kf_of_frame.append(keys[key])
    fe.reserve_keyframe_track(len(kfs), max(len(k["desc"]) for k in kfs))
    fe.set_keyframes(kfs, kf_of_frame)
    every = np.zeros(B, np.uint8)
    none = np.ones(B, np.uint8)
    some = np.ones(B, np.uint8)
    some[rng.choice(B, max(1, B // 20), replace=False)] = 0

    # 1. gate: a seeded sample of active frames against the oracle, fed the device's keypoints
    fe.step(B)
    fe.track_keyframe(B, gv, every)
    sync()
    kps = fe.download_keypoints(B)
    out = fe.download_keyframe_tracking(B)
    sample = rng.choice(B, min(args.sample, B), replace=False)
    host_ms = []
    for b in sample:
        s, t = t_idx[b]
        k = kps[b][0]
        curr = dict(x=k["x"], y=k["y"], octave=k["octave"], angle=k["angle"], desc=kps[b][1])
        t0 = time.perf_counter()
        w = ktd.oracle_keyframe_track(orc, ov, fe.cam, curr, kfs[kf_of_frame[b]], seqs[s].poses[t - 1])
        host_ms.append(1e3 * (time.perf_counter() - t0))
        assert out["num_bow_matches"][b] == w["num_bow"] and np.array_equal(out["matched"][b], w["matched"]), b
        assert np.linalg.norm(out["pose"][b] - w["pose"]) <= 1e-4 * np.linalg.norm(w["pose"]), b

    fe.step(B)
    fe.track_keyframe(B, gv, none)
    sync()
    out_none_active = int(fe.download_keyframe_tracking(B)["stage"].sum())  # every motion track succeeded: 0

    # 2. step() alone and with the stage on no frame / on ~5 % of the frames / on every frame, alternately
    def timed(mv):
        sync()
        t0 = time.perf_counter()
        fe.step(B)
        if mv is not None:
            fe.track_keyframe(B, gv, mv)
        sync()
        return 1e3 * (time.perf_counter() - t0)
    runs = {"step": None, "step_plus_none_active": none, "step_plus_5pct_active": some, "step_plus_all_active": every}
    for _ in range(args.warmup):
        for mv in runs.values():
            timed(mv)
    times = {k: [] for k in runs}
    for _ in range(args.steps):
        for k, mv in runs.items():
            times[k].append(timed(mv))

    # 3. the stage's kernels alone (the motion outputs stay as the last step() left them)
    lib = fe.lib
    kernels = {}
    for name, mv in (("none_active", none), ("5pct_active", some), ("all_active", every)):
        fe.track_keyframe(B, gv, mv)  # uploads motion_valid before the timed calls
        sync()
        tctx._check(lib.plp_ctx_kernel_timing(tctx.handle, 1))
        for _ in range(args.steps):
            fe.lib.plp_tracker_keyframe_track_batch_dev(
                fe._trk, gv.handle, C.c_int(B), C.byref(fe._kf), fe._kf_out["motion_valid"].ptr,
                *[fe._kf_out[k].ptr for k in ("stage", "matched", "num_bow", "pose", "num_valid", "n_inliers",
                                               "lm_iters", "status")])
        tctx.sync()
        buf = C.create_string_buffer(1 << 16)
        tctx._check(lib.plp_ctx_kernel_timing_report(tctx.handle, buf, C.c_size_t(len(buf))))
        tctx._check(lib.plp_ctx_kernel_timing(tctx.handle, 0))
        kt = json.loads(buf.value.decode())
        kernels[name] = {k: round(v["total_ms"] / args.steps, 4)
                         for k, v in sorted(kt.items(), key=lambda kv: -kv[1]["total_ms"])}
    fe.track_keyframe(B, gv, some)
    sync()
    out = fe.download_keyframe_tracking(B)
    med = {k: round(float(np.median(x)), 3) for k, x in times.items()}
    res = {"metric": "keyframe_track_ms_per_step", "batch": B, "steps": args.steps, "keyframes": len(kfs),
           "step_ms_median": med,
           "step_ms_range": {k: [round(min(x), 3), round(max(x), 3)] for k, x in times.items()},
           "stage_ms_median_difference": {k: round(med[k] - med["step"], 3) for k in runs if k != "step"},
           "stage_kernels_ms_per_call": kernels,
           "stage_kernels_ms_total": {k: round(sum(v.values()), 4) for k, v in kernels.items()},
           "active_frames": {"none_active": int(out_none_active), "5pct_active": int((some == 0).sum()), "all_active": B},
           "frames_per_keyframe_max": int(np.bincount(kf_of_frame).max()),
           "bow_matches_median": int(np.median(out["num_bow_matches"][some == 0])),
           "num_valid_median": int(np.median(out["num_valid"][some == 0])),
           "oracle_host_chain_ms_per_frame": round(float(np.median(host_ms)), 3),
           "oracle_sample": [int(b) for b in sample],
           "card": card()}
    print(json.dumps(res))
    fe.close()
    gv.close()
    orc.bow_vocab_destroy(ov)


if __name__ == "__main__":
    main()
