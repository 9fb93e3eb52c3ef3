"""Times plp_sim3_optimize: P (query keyframe, loop candidate) problems x n valid matches per problem, 20 % outliers, the
loop detector's chi_sq 10 and num_iter 10, for P in {1, 8, 64, 512} -- one candidate, one query's candidates, and batches
of many queries -- and n in {100, 300, 1000}.  The device time is one call's span between two CUDA events on the calling
stream (the call is synchronous, so transfers are included), the median of --reps after a warm-up call.  The host column
is the oracle (oracle/transform_opt.cc, the same sim3optmath.h compiled -O3) on one core, per problem, over the first
min(P, 8) problems; the largest relative Sim3 difference between the two on those problems is printed beside it.  Prints
the card's name and power limit from the same run.

    python tools/bench_sim3_opt.py [--reps 10]
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

import oracle_api  # noqa: E402
import sim3_opt_data as sd  # noqa: E402
from conftest import load_package  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def subset(d, k):
    """The first k problems of a pack dict."""
    n = int(d["off"][k])
    out = {key: v[:k] for key, v in d.items() if key in ("cams", "pose_1w", "pose_2w", "rot", "trans", "scale")}
    out["off"] = d["off"][:k + 1]
    for key in ("pos_w_1", "pos_w_2", "obs_1", "obs_2", "w_1", "w_2"):
        out[key] = d[key][:n]
    return out


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    pkg = load_package()
    ctx = pkg.Context(0)
    orc = oracle_api.Oracle()
    print(json.dumps({"card": card()}), flush=True)
    for P in (1, 8, 64, 512):
        cams = [pkg.capi.make_camera(sd.FX, sd.FY, sd.CX, sd.CY, sd.COLS, sd.ROWS)] * P
        for n in (100, 300, 1000):
            d = sd.pack([sd.make_scene(1000 * P + 7 * n + i, n, 0.2) for i in range(P)])
            p1, p2 = d["pose_1w"], d["pose_2w"]
            call = lambda: ctx.sim3_optimize(d["off"], cams, p1[:, :9], p1[:, 9:], p2[:, :9], p2[:, 9:], d["rot"],
                                             d["trans"], d["scale"], d["pos_w_1"], d["pos_w_2"], d["obs_1"], d["obs_2"],
                                             d["w_1"], d["w_2"])
            got = call()  # warm-up
            dev = []
            for _ in range(args.reps):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                got = call()
                b.record()
                b.synchronize()
                dev.append(a.elapsed_time(b))
            k = min(P, 8)
            dk = subset(d, k)
            t0 = time.perf_counter()
            want = sd.oracle_optimize(orc, dk)
            host_ms = 1e3 * (time.perf_counter() - t0) / k
            gk = (got[0][:k], got[1][:k], got[2][:k], got[3][:k], got[4][:int(d["off"][k])])
            print(json.dumps({"P": P, "n": n, "device_ms": round(float(np.median(dev)), 3),
                              "device_us_per_problem": round(1e3 * float(np.median(dev)) / P, 1),
                              "host_ms_per_problem": round(host_ms, 3), "mean_inliers": float(np.mean(got[0])),
                              "flags_equal": bool(np.array_equal(gk[4], want[4]) and np.array_equal(gk[0], want[0])),
                              "max_rel_err": sd.max_rel_error(gk, want)}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
