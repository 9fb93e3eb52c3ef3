"""Times plp_sim3_ransac: P (query keyframe, loop candidate) pairs x n correspondences, 200 hypotheses, 50 % outliers
(the loop detector's find_via_ransac(200)), for P in {1, 16, 256} -- one candidate, one query's candidates, a BoW
database batch's loop queries -- and n in {50, 300, 1000}.  The device time is the wall time of one call, transfers
included, as the median of --reps after a warm-up call.  The host column is the oracle (oracle/sim3.cc, the same
sim3math.h compiled -O3 for the CPU) on one thread over the same problems; the outputs of both are checked equal in the
same run.  Prints the card's name and power limit from the same run.

    python tools/bench_sim3.py [--reps 10]
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
import sim3_data as sd  # noqa: E402
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
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    pkg = load_package()
    ctx = pkg.Context(0)
    orc = oracle_api.Oracle()
    print(json.dumps({"card": card()}), flush=True)
    for P in (1, 16, 256):
        cams = [pkg.capi.make_camera(sd.FX, sd.FY, sd.CX, sd.CY, sd.COLS, sd.ROWS)] * P
        for n in (50, 300, 1000):
            off, x1, x2, c1, c2, sm = sd.problems(P, P, [n], num_iter=200, outlier_frac=0.5)
            got = ctx.sim3_ransac(off, cams, x1, x2, c1, c2, sm)  # warm-up
            dev = []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                got = ctx.sim3_ransac(off, cams, x1, x2, c1, c2, sm)
                dev.append(time.perf_counter() - t0)
            host = []
            for _ in range(max(1, args.reps // 3)):
                t0 = time.perf_counter()
                want = sd.oracle_ransac(orc, off, x1, x2, c1, c2, sm)
                host.append(time.perf_counter() - t0)
            equal = all(np.array_equal(g, w, equal_nan=True) for g, w in zip(got, want))
            print(json.dumps({"P": P, "n": n, "device_ms": round(1e3 * float(np.median(dev)), 3),
                              "host_ms": round(1e3 * float(np.median(host)), 3), "valid": int(got[0].sum()),
                              "equal": bool(equal)}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
