"""Time the batched tracker on rectified stereo frames next to the monocular chain on the same left images.

    python tools/bench_stereo_track.py [--batches 148 256] [--steps 10] [--warmup 3] [--seed 1234] [--sample 4]

The frames come from rendered stereo sequences at EuRoC's K and size (752 x 480, bf 47.906): a textured plane, the
right image rendered from the camera shifted by the true baseline.  Every frame gets its last frame's landmarks and a
local map of about 3 k landmarks (the last three frames', extracted on the GPU without timing).  One step is
  stereo:     ORB left + right -> match::stereo::compute -> motion track (margin 10) -> local-map track (margin 5)
  monocular:  ORB left -> motion track (margin 20) -> local-map track (margin 5)
each on one extraction and one tracking context, with a device synchronise around it; the two alternate.  The local
maps are uploaded lists, so the local-map update stage is not part of either step.  Before timing, a seeded sample of
frames of both chains is checked against the oracle (x_right, motion matches and pose, local-map matches and pose).
Prints one JSON line per batch with the card's name and power limit read in the same run; writes nothing."""
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

BF = 47.906
EUROC_K = (458.654, 457.296, 367.215, 248.375)
ROWS, COLS = 480, 752
MAX_LOCAL = 4096
N_SEQ, N_FRAMES = 6, 8


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "--id=0"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else f"nvidia-smi failed: {q.stderr.strip()}"


def make_inputs(pkg, batch, seed):
    """Frames (sequence, t >= 3) cycled over N_SEQ rendered stereo sequences, with predicted poses."""
    import scene
    import stereo_track_data as std
    fx, fy, cx, cy = EUROC_K
    seqs = [scene.PlanarSequence(seed=seed + 17 * s, n_frames=N_FRAMES, rows=ROWS, cols=COLS, fx=fx, fy=fy, cx=cx,
                                 cy=cy) for s in range(N_SEQ)]
    cam = std.stereo_camera(pkg, seqs[0], BF)
    rights = [std.right_frames(s, cam.true_baseline) for s in seqs]
    rng = np.random.default_rng(seed)
    t_idx = [(b % N_SEQ, 3 + (b // N_SEQ) % (N_FRAMES - 3)) for b in range(batch)]
    preds = [seqs[s].predicted_pose(t, rng) for s, t in t_idx]
    return dict(seqs=seqs, rights=rights, cam=cam, t_idx=t_idx, preds=preds)


def setup(pkg, ctx, tctx, inp, stereo, seed):
    """A FrontEnd with the last frames and local maps of every frame set; earlier frames extracted on the GPU."""
    import local_map_data as lmd
    from plpslam_b200.tracking import FrontEnd
    seqs, t_idx = inp["seqs"], inp["t_idx"]
    B = len(t_idx)
    cam = inp["cam"] if stereo else seqs[0].camera(pkg)
    fe = FrontEnd(ctx, ROWS, COLS, cam, max_batch=B, track_ctx=tctx)
    mono = fe if not stereo else FrontEnd(ctx, ROWS, COLS, seqs[0].camera(pkg), max_batch=B)
    res = [dict() for _ in range(B)]
    for back in (1, 2, 3):
        mono.upload_images(np.stack([seqs[s].frames[t - back] for s, t in t_idx]))
        mono.extract(B)
        kps = mono.download_keypoints(B)
        for b, (s, t) in enumerate(t_idx):
            res[b][t - back] = dict(kps=kps[b][0], desc=kps[b][1])
    if mono is not fe:
        mono.close()
    lasts = [seqs[s].last_frame_landmarks(t - 1, res[b][t - 1]["kps"], res[b][t - 1]["desc"])
             for b, (s, t) in enumerate(t_idx)]
    rng = np.random.default_rng(seed + 1)
    local_list = [lmd.build_local_map(seqs[s], res[b], t, rng, n_earlier=2, last_frame=lasts[b])
                  for b, (s, t) in enumerate(t_idx)]
    left = np.stack([seqs[s].frames[t] for s, t in t_idx])
    if stereo:
        fe.upload_images(left, np.stack([inp["rights"][s][t] for s, t in t_idx]))
    else:
        fe.upload_images(left)
    fe.set_last_frames(lasts, np.stack(inp["preds"]), np.stack([seqs[s].poses[t - 1] for s, t in t_idx]))
    fe.reserve_local_map(MAX_LOCAL)
    fe.set_local_maps(local_list)
    ctx.sync()
    tctx.sync()
    return fe, dict(lasts=lasts, local_list=local_list)


def check_sample(orc, fe, inp, aux, sample, stereo, margin):
    """The frames `sample` of the most recent step against the oracle chain, fed the device's left keypoints."""
    import local_map_data as lmd
    import oracle_api
    import scene
    import stereo_track_data as std
    B = len(inp["t_idx"])
    kps = fe.download_keypoints(B)
    mot = fe.download_tracking(B)
    out = fe.download_local_tracking(B)
    xr = fe.download_stereo(B) if stereo else None
    wants, got_it, want_it = [None] * B, [], []
    for b in sample:
        s, t = inp["t_idx"][b]
        k = kps[b][0]
        curr = dict(x=k["x"], y=k["y"], octave=k["octave"], angle=k["angle"], desc=kps[b][1])
        if stereo:
            p = oracle_api.orb_params()
            rl, rr = orc.orb_extract(p, inp["seqs"][s].frames[t]), orc.orb_extract(p, inp["rights"][s][t])
            want, _, _ = orc.stereo_compute(rl, rr, fe.orb.scale_factors, fe.orb.inv_scale_factors,
                                            fe.cam.focal_x_baseline, fe.cam.true_baseline)
            assert np.array_equal(rl["kps"], k) and np.array_equal(xr[b][0], want), f"x_right of frame {b}"
            curr["x_right"] = xr[b][0]
        last = aux["lasts"][b]
        chain = std if stereo else lmd
        motion = chain.oracle_motion(orc, fe.grid, fe.cam, curr, last, inp["preds"][b], inp["seqs"][s].poses[t - 1],
                                     margin)
        assert np.array_equal(motion[1], mot["matched"][b]), f"motion track of frame {b}"
        assert np.linalg.norm(mot["pose"][b] - motion[2]) / np.linalg.norm(motion[2]) <= 1e-4, b
        dev = (motion[0], motion[1], mot["pose"][b], int(mot["num_valid"][b]))
        wants[b] = chain.oracle_local_track(orc, fe.grid, fe.cam, curr, last, aux["local_list"][b], dev, MAX_LOCAL)
        g, w = lmd.compare(out, wants, frames={b})
        got_it += g
        want_it += w
    scene.check_lm_iters(got_it, want_it, "sample")


def run_batch(pkg, ctx, tctx, orc, B, args):
    inp = make_inputs(pkg, B, args.seed)
    chains = {}
    for stereo in (True, False):
        fe, aux = setup(pkg, ctx, tctx, inp, stereo, args.seed)
        chains[stereo] = (fe, aux, 10.0 if stereo else 20.0)

    def sync():
        ctx.sync()
        tctx.sync()

    def timed(stereo):
        fe, _, margin = chains[stereo]
        sync()
        t0 = time.perf_counter()
        fe.step(B, margin)
        fe.track_local_map(B, 5.0)
        sync()
        return 1e3 * (time.perf_counter() - t0)

    sample = np.random.default_rng(args.seed).choice(B, min(args.sample, B), replace=False)
    for stereo in (True, False):
        timed(stereo)
        fe, aux, margin = chains[stereo]
        check_sample(orc, fe, inp, aux, sample, stereo, margin)
    for _ in range(args.warmup):
        timed(True)
        timed(False)
    ms = {True: [], False: []}
    for _ in range(args.steps):
        for stereo in (True, False):
            ms[stereo].append(timed(stereo))
    fe_s = chains[True][0]
    xr = fe_s.download_stereo(B)
    stats = {}
    for stereo in (True, False):
        fe = chains[stereo][0]
        mot, out = fe.download_tracking(B), fe.download_local_tracking(B)
        stats[stereo] = dict(motion_ok_share=round(float((mot["num_valid"] >= 20).mean()), 4),
                             num_tracked_mean=round(float(out["num_tracked"].mean()), 1))
        fe.close()
    med_s, med_m = float(np.median(ms[True])), float(np.median(ms[False]))
    return {"metric": "stereo_track_ms_per_step", "batch": B, "steps": args.steps,
            "stereo_ms_median": round(med_s, 3), "stereo_ms_range": [round(min(ms[True]), 3), round(max(ms[True]), 3)],
            "mono_ms_median": round(med_m, 3), "mono_ms_range": [round(min(ms[False]), 3), round(max(ms[False]), 3)],
            "stereo_frames_per_s": round(1e3 * B / med_s, 1), "mono_frames_per_s": round(1e3 * B / med_m, 1),
            "stereo_keypoints_mean": round(float(np.mean([(x[0] >= 0).sum() for x in xr])), 1),
            "stereo": stats[True], "mono": stats[False],
            "oracle_sample": [int(b) for b in sample], "card": card()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[148, 256])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1234)
    ap.add_argument("--sample", type=int, default=4)
    args = ap.parse_args()
    pkg = bench._load_pkg()
    import oracle_api
    orc = oracle_api.Oracle()
    ctx = pkg.Context(0)
    tctx = pkg.Context(0, high_priority=True)
    for B in args.batches:
        print(json.dumps(run_batch(pkg, ctx, tctx, orc, B, args)), flush=True)
    tctx.close()
    ctx.close()


if __name__ == "__main__":
    main()
