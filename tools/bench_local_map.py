"""Time the batched local-map stage of tracking next to bench.py's headline step.

    python tools/bench_local_map.py [--batch 512] [--steps 20] [--warmup 3] [--seed 1234]

bench.py's headline problems (bench.build_inputs / setup_front_end: 512 planar-sequence frames, ORB 1000 keypoints,
motion-based tracking on a high-priority tracking context).  Every frame also gets a local map of about 3 k landmarks:
the last frame's landmarks and those of the two frames before it, extracted on the GPU without timing.  The script
  1. checks a seeded sample of frames against the oracle chain (motion track, then the local-map stage);
  2. times step() alone and step() + track_local_map() alternately, with a device synchronise around each timed step;
  3. times the new kernels (plp_ctx_kernel_timing) over further track_local_map() calls;
  4. reports the share of frames with num_tracked >= 20 and their pose error against ground truth.
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

MAX_LOCAL = 4096


def setup(pkg, ctx, batch, seed, track_ctx=None):
    """bench.setup_front_end plus local maps; the earlier frames are extracted on the GPU (untimed)."""
    import local_map_data as lmd
    fe, frames, aux = bench.setup_front_end(pkg, ctx, batch, seed, track_ctx)
    seqs, t_idx = aux["seqs"], aux["t_idx"]
    res = [dict() for _ in range(batch)]
    for back in (1, 2, 3):
        ks = [t - back for (s, t) in t_idx]
        fe.upload_images(np.stack([seqs[s].frames[max(k, 0)] for (s, _), k in zip(t_idx, ks)]))
        fe.extract(batch)
        kps = fe.download_keypoints(batch)
        for b, k in enumerate(ks):
            if k >= 0:
                res[b][k] = dict(kps=kps[b][0], desc=kps[b][1])
    fe.upload_images(frames)
    rng = np.random.default_rng(seed + 1)
    local_list = [lmd.build_local_map(seqs[s], res[b], t, rng, n_earlier=2, last_frame=aux["lasts"][b])
                  for b, (s, t) in enumerate(t_idx)]
    fe.reserve_local_map(MAX_LOCAL)
    fe.set_local_maps(local_list)
    for cx in {id(ctx): ctx, id(fe.track_ctx): fe.track_ctx}.values():
        cx.sync()
    aux.update(local_list=local_list)
    return fe, aux


def check_sample(orc, pkg, fe, aux, sample):
    """The frames `sample` of the most recent step() + track_local_map() against the oracle chain, fed the device's
    keypoints (extraction parity is tested on its own)."""
    import local_map_data as lmd
    batch = len(aux["t_idx"])
    kps = fe.download_keypoints(batch)
    mot = fe.download_tracking(batch)
    out = fe.download_local_tracking(batch)
    wants = {}
    for b in sample:
        s, t = aux["t_idx"][b]
        k = kps[b][0]
        curr = dict(x=k["x"], y=k["y"], octave=k["octave"], angle=k["angle"], desc=kps[b][1])
        last = aux["lasts"][b]
        motion = lmd.oracle_motion(orc, fe.grid, fe.cam, curr, last, aux["preds"][b], aux["seqs"][s].poses[t - 1])
        assert np.array_equal(motion[1], mot["matched"][b]), f"motion track of frame {b}"
        dev = (motion[0], motion[1], mot["pose"][b], int(mot["num_valid"][b]))
        wants[b] = lmd.oracle_local_track(orc, fe.grid, fe.cam, curr, last, aux["local_list"][b], dev, MAX_LOCAL)
    full = [wants.get(b) for b in range(batch)]
    got_it, want_it = [], []
    for b in sample:
        g, w = lmd.compare(out, full, frames={b})
        got_it += g
        want_it += w
    import scene
    scene.check_lm_iters(got_it, want_it, "local map sample")
    return out


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                        "--id=0"], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else f"nvidia-smi failed: {q.stderr.strip()}"


def pose_error(T, T_gt):
    dR = T[:3, :3] @ T_gt[:3, :3].T
    ang = np.degrees(np.arccos(np.clip((np.trace(dR) - 1) / 2, -1, 1)))
    c, c_gt = -T[:3, :3].T @ T[:3, 3], -T_gt[:3, :3].T @ T_gt[:3, 3]
    return ang, np.linalg.norm(c - c_gt)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1234)
    ap.add_argument("--sample", type=int, default=8)
    args = ap.parse_args()
    pkg = bench._load_pkg()
    import oracle_api
    ctx = pkg.Context(0)
    tctx = pkg.Context(0, high_priority=True)
    fe, aux = setup(pkg, ctx, args.batch, args.seed, tctx)
    B = args.batch

    def sync():
        ctx.sync()
        tctx.sync()

    # 1. gate: a seeded sample against the oracle
    fe.step(B)
    fe.track_local_map(B)
    sync()
    sample = np.random.default_rng(args.seed).choice(B, min(args.sample, B), replace=False)
    out = check_sample(oracle_api.Oracle(), pkg, fe, aux, sample)

    # 2. step() alone and step() + track_local_map(), alternately
    def timed(with_local):
        sync()
        t0 = time.perf_counter()
        fe.step(B)
        if with_local:
            fe.track_local_map(B)
        sync()
        return 1e3 * (time.perf_counter() - t0)
    for _ in range(args.warmup):
        timed(False)
        timed(True)
    alone, both = [], []
    for _ in range(args.steps):
        alone.append(timed(False))
        both.append(timed(True))

    # 3. the stage's kernels alone (the motion outputs stay as the last step() left them)
    lib = fe.lib
    tctx._check(lib.plp_ctx_kernel_timing(tctx.handle, 1))
    for _ in range(args.steps):
        fe.track_local_map(B)
    tctx.sync()
    buf = C.create_string_buffer(1 << 16)
    tctx._check(lib.plp_ctx_kernel_timing_report(tctx.handle, buf, C.c_size_t(len(buf))))
    tctx._check(lib.plp_ctx_kernel_timing(tctx.handle, 0))
    kt = json.loads(buf.value.decode())
    kernels = {k: round(v["total_ms"] / args.steps, 4) for k, v in sorted(kt.items(), key=lambda kv: -kv[1]["total_ms"])}

    # 4. tracking quality of the last step
    mot = fe.download_tracking(B)
    out = fe.download_local_tracking(B)
    ok = np.nonzero(out["num_tracked"] >= 20)[0]
    errs = np.array([pose_error(out["pose"][b], aux["gt"][b]) for b in ok]) if len(ok) else np.zeros((0, 2))
    errs_m = np.array([pose_error(mot["pose"][b], aux["gt"][b]) for b in ok]) if len(ok) else np.zeros((0, 2))
    rows = np.array([len(lm["max_valid_dist"]) for lm in aux["local_list"]])
    res = {"metric": "local_map_ms_per_step", "batch": B, "steps": args.steps,
           "step_ms_median": round(float(np.median(alone)), 3),
           "step_plus_local_ms_median": round(float(np.median(both)), 3),
           "local_ms_median_difference": round(float(np.median(both) - np.median(alone)), 3),
           "step_ms_range": [round(min(alone), 3), round(max(alone), 3)],
           "step_plus_local_ms_range": [round(min(both), 3), round(max(both), 3)],
           "local_kernels_ms_per_call": kernels,
           "local_kernels_ms_total": round(sum(kernels.values()), 4),
           "local_rows_per_frame": [int(rows.min()), int(np.median(rows)), int(rows.max())],
           "observable_per_frame_median": int(np.median([o.sum() for o in out["observable"]])),
           "local_matches_per_frame_median": int(np.median([(x >= 0).sum() for x in out["local"]])),
           "tracked_share": round(len(ok) / B, 4),
           "num_tracked_median": int(np.median(out["num_tracked"])),
           "rot_err_deg_median": round(float(np.median(errs[:, 0])), 5) if len(ok) else None,
           "center_err_m_median": round(float(np.median(errs[:, 1])), 6) if len(ok) else None,
           "motion_rot_err_deg_median": round(float(np.median(errs_m[:, 0])), 5) if len(ok) else None,
           "motion_center_err_m_median": round(float(np.median(errs_m[:, 1])), 6) if len(ok) else None,
           "oracle_sample": [int(b) for b in sample],
           "card": card()}
    print(json.dumps(res))
    fe.close()


if __name__ == "__main__":
    main()
