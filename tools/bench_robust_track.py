"""Time the batched robust tracker (robust_match_based_track) on bench.py's headline problems.

    python tools/bench_robust_track.py [--batch 512] [--steps 20] [--warmup 3] [--seed 1234] [--sample 4] [--host 16]

bench.py's headline problems (bench.setup_front_end: 512 planar-sequence frames, ORB 1000 keypoints, motion tracking
on a high-priority tracking context).  Each sequence's frames t = 1..32 are grouped by four: frames 4g + 1 .. 4g + 4
share frame 4g as their reference keyframe, extracted on the GPU without timing.  The keyframes carry an empty
bow_feat_vec_, so a frame handed to the keyframe track finds no BoW match and falls through to the robust stage.  The
script
  1. checks a seeded sample of active frames against the oracle chain (brute force -> essential RANSAC with the
     device's samples -> pose optimiser -> discard_outliers);
  2. times plp_tracker_robust_track_batch_dev alone with device events on the tracking stream, with no frame active
     (every motion track usable and successful: the cost of the chain when nothing falls through) and with every frame
     active (motion model unusable), alternately, each after its own step() + track_keyframe();
  3. times the stage's kernels with torch.profiler (a separate run);
  4. times the per-frame host path the stage replaces: plp_match_brute_force + plp_essential_ransac (samples drawn on
     the host) + plp_pose_optimize, one frame at a time.
Prints one JSON line with the card's name, power limit and SM clock read in the same run; writes nothing."""
from __future__ import annotations

import argparse
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
    import torch
    from torch.profiler import ProfilerActivity, profile

    import keyframe_track_data as ktd
    import local_map_data as lmd
    import oracle_api
    import robust_track_data as rtd
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1234)
    ap.add_argument("--sample", type=int, default=4)
    ap.add_argument("--host", type=int, default=16)
    args = ap.parse_args()
    pkg = bench._load_pkg()
    ctx = pkg.Context(0)
    tctx = pkg.Context(0, high_priority=True)
    stream = torch.cuda.ExternalStream(pkg.lib().plp_ctx_stream(tctx.handle), device="cuda:0")
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
    gv = pkg.BowVocabulary(tctx, k=v["k"], L=v["L"], parent=v["parent"], desc=v["desc"], weight=v["weight"],
                           is_leaf=v["is_leaf"])
    empty_fv = (np.zeros(0, np.uint32), np.zeros(1, np.int32), np.zeros(0, np.uint32))
    keys, kfs, kf_of_frame = {}, [], []
    for b, (s, t) in enumerate(t_idx):
        key = (s, kf_t[b])
        if key not in keys:
            k, d = prev[b]
            pos_w = seqs[s].backproject(seqs[s].poses[key[1]], k["x"].astype(np.float64), k["y"].astype(np.float64))
            keys[key] = len(kfs)
            kfs.append(dict(t=key[1], desc=d, angle=k["angle"].astype(np.float32), valid=np.ones(len(d), np.uint8),
                            pos_w=pos_w, fv=empty_fv, bearings=rtd.bearings(fe.cam, k["x"], k["y"])))
        kf_of_frame.append(keys[key])
    fe.reserve_keyframe_track(len(kfs), max(len(k["desc"]) for k in kfs))
    fe.reserve_robust_track()
    fe.set_keyframes(kfs, kf_of_frame)
    every = np.zeros(B, np.uint8)
    none = np.ones(B, np.uint8)
    shares = {"none_active": none, "all_active": every}

    def prepare(mv):
        fe.step(B)
        fe.track_keyframe(B, gv, mv)

    # 1. gate: a seeded sample of active frames against the oracle, fed the device's keypoints
    prepare(every)
    fe.track_robust(B, args.seed)
    sync()
    kps = fe.download_keypoints(B)
    out = fe.download_robust_tracking(B)
    assert (out["stage"] == 1).all()
    sample = rng.choice(B, min(args.sample, B), replace=False)
    for b in sample:
        s, t = t_idx[b]
        k = kps[b][0]
        curr = dict(x=k["x"], y=k["y"], octave=k["octave"], angle=k["angle"], desc=kps[b][1])
        w = rtd.oracle_robust_track(orc, fe.cam, curr, kfs[kf_of_frame[b]], rtd.bearings(fe.cam, k["x"], k["y"]),
                                    out["samples"][b], seqs[s].poses[t - 1])
        assert out["num_bf_matches"][b] == w["num_bf"] and out["num_robust_matches"][b] == w["num_robust"], b
        assert np.array_equal(out["matched"][b], w["matched"]), b
        assert np.linalg.norm(out["pose"][b] - w["pose"]) <= 1e-4 * np.linalg.norm(w["pose"]), b
    active_counts = {}
    for name, mv in shares.items():
        prepare(mv)
        fe.track_robust(B, args.seed)
        sync()
        active_counts[name] = int(fe.download_robust_tracking(B)["stage"].sum())
    tracked_all_active = int((out["num_valid"] >= 20).sum())

    # 2. the call alone, device events on the tracking stream, the two shares alternately
    def timed(mv):
        prepare(mv)
        sync()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        fe.track_robust(B, args.seed)
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1)
    for _ in range(args.warmup):
        for mv in shares.values():
            timed(mv)
    times = {k: [] for k in shares}
    for _ in range(args.steps):
        for k, mv in shares.items():
            times[k].append(timed(mv))

    # 3. the stage's kernels (torch.profiler, a run of its own)
    kernels = {}
    for name, mv in shares.items():
        prepare(mv)
        sync()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                fe.track_robust(B, args.seed)
            sync()
        per = {}
        for e in prof.key_averages():
            dt = getattr(e, "device_time_total", None)
            if dt is None:
                dt = e.cuda_time_total
            if dt > 0:
                per[e.key] = per.get(e.key, 0.0) + dt / 1e3 / args.steps
        kernels[name] = {k: round(v, 4) for k, v in sorted(per.items(), key=lambda kv: -kv[1])}

    # 4. the per-frame host path it replaces: one frame at a time, samples drawn on the host
    host_ms = []
    for b in rng.choice(B, min(args.host, B), replace=False):
        s, t = t_idx[b]
        k = kps[b][0]
        kf = kfs[kf_of_frame[b]]
        t0 = time.perf_counter()
        m, _ = ctx.brute_force_match(kps[b][1], k["angle"], kf["desc"], kf["angle"], kf["valid"], 0.8, False)
        idx = np.nonzero(m >= 0)[0]
        pairs = np.stack([idx, m[idx]], 1).astype(np.int32)
        smp = np.stack([rng.choice(len(pairs), 8, replace=False) for _ in range(50)]).astype(np.int32)
        valid, inl, _, _ = ctx.essential_ransac(rtd.bearings(fe.cam, k["x"], k["y"]), kf["bearings"], pairs, smp)
        keep = idx[inl != 0]
        pts = np.zeros(len(keep), oracle_api.PT_OBS_DTYPE)
        pts["pos_w"] = kf["pos_w"][m[keep]]
        pts["obs_x"], pts["obs_y"] = k["x"][keep], k["y"][keep]
        pts["x_right"] = -1.0
        pts["inv_sigma_sq"] = lmd.ISIG[k["octave"][keep]]
        if valid and len(keep) >= 20:
            ctx.pose_optimize(fe.cam, seqs[s].poses[t - 1], pts)
        host_ms.append(1e3 * (time.perf_counter() - t0))

    med = {k: round(float(np.median(x)), 3) for k, x in times.items()}
    host_med = float(np.median(host_ms))
    res = {"metric": "robust_track_ms_per_call", "batch": B, "steps": args.steps, "keyframes": len(kfs),
           "call_ms_median": med,
           "call_ms_range": {k: [round(min(x), 3), round(max(x), 3)] for k, x in times.items()},
           "stage_kernels_ms_per_call": kernels,
           "active_frames": active_counts,
           "tracked_frames_all_active": tracked_all_active,
           "bf_matches_median": int(np.median(out["num_bf_matches"])),
           "robust_matches_median": int(np.median(out["num_robust_matches"])),
           "host_path_ms_per_frame": round(host_med, 3),
           "host_path_ms_per_batch_estimate": round(host_med * B, 1),
           "oracle_sample": [int(b) for b in sample],
           "card": card()}
    print(json.dumps(res))
    fe.close()
    gv.close()


if __name__ == "__main__":
    main()
