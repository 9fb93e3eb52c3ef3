"""Time the batched front end for a distorted camera against the same front end without distortion.

    python tools/bench_distorted.py [--batch 256] [--steps 20] [--warmup 3] [--seed 1234]

The inputs are bench.py's headline inputs (rendered planar sequences, 640x480, ORB 1000 keypoints, last-frame landmarks
from a first GPU extraction).  One FrontEnd tracks them with the TUM RGB-D mono 1 K/D (example/tum_rgbd/
TUM_RGBD_mono_1.yaml), so every step runs the undistortion kernel before the window matcher; a second FrontEnd on the
same context tracks them without distortion.  Their steps alternate, CUDA events around each step.  Prints one JSON line;
writes nothing."""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import numpy as np

sys.dont_write_bytecode = True
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
import bench  # noqa: E402

# Camera.k1, k2, p1, p2, k3 of example/tum_rgbd/TUM_RGBD_mono_1.yaml
TUM_MONO_1_DIST = (0.262383, -0.953104, -0.005358, 0.002628, 1.163314)


def setup(pkg, ctx, batch, seed, distortion):
    """bench.setup_front_end with an optional distortion."""
    import synth
    from plpslam_b200.tracking import FrontEnd
    cam = pkg.capi.make_camera(synth.FX, synth.FY, synth.CX, synth.CY, bench.COLS, bench.ROWS)
    fe = FrontEnd(ctx, bench.ROWS, bench.COLS, cam, max_batch=batch, distortion=distortion)
    seqs, frames, t_idx = bench.build_inputs(batch, seed)
    fe.upload_images(np.stack([seqs[s].frames[t - 1] for (s, t) in t_idx]))
    fe.extract(batch)
    ctx.sync()
    kps = fe.download_keypoints(batch)
    rng = np.random.default_rng(seed)
    lasts = [seqs[s].last_frame_landmarks(t - 1, kps[b][0], kps[b][1]) for b, (s, t) in enumerate(t_idx)]
    preds = np.stack([seqs[s].predicted_pose(t, rng) for (s, t) in t_idx])
    fe.set_last_frames(lasts, preds, np.stack([seqs[s].poses[t - 1] for (s, t) in t_idx]))
    fe.upload_images(frames)
    return fe


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1234)
    args = ap.parse_args()
    import torch
    pkg = bench._load_pkg()
    ctx = pkg.Context(0)
    stream = torch.cuda.ExternalStream(pkg.lib().plp_ctx_stream(ctx.handle), device="cuda:0")
    fes = {"distorted": setup(pkg, ctx, args.batch, args.seed, pkg.capi.make_distortion(0, *TUM_MONO_1_DIST)),
           "plain": setup(pkg, ctx, args.batch, args.seed, None)}
    for _ in range(args.warmup):
        for fe in fes.values():
            fe.step(args.batch)
    ctx.sync()
    ms = {k: 0.0 for k in fes}
    for _ in range(args.steps):
        for k, fe in fes.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            fe.step(args.batch)
            e1.record(stream)
            e1.synchronize()
            ms[k] += e0.elapsed_time(e1)
    ok = {k: int((fe.download_tracking(args.batch)["num_valid"] >= 20).sum()) for k, fe in fes.items()}
    print(json.dumps({"frames_per_s": args.batch * args.steps / (ms["distorted"] * 1e-3),
                      "ms_per_step": ms["distorted"] / args.steps, "plain_ms_per_step": ms["plain"] / args.steps,
                      "frames_per_step": args.batch, "tracked_ok_frames": ok,
                      "undistort_alg_bytes_per_keypoint": 28 + 8 + 24, "gpu": torch.cuda.get_device_name(0)}))
    for fe in fes.values():
        fe.close()
    ctx.close()


if __name__ == "__main__":
    main()
