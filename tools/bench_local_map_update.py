"""Time the batched local-map update next to the host path it replaces.

    python tools/bench_local_map_update.py [--batch 512] [--steps 10] [--warmup 2] [--seed 1234]

bench.py's headline problems (bench.setup_front_end: 512 planar-sequence frames, ORB 1000 keypoints, motion-based
tracking on a high-priority tracking context) over a 128-keyframe map snapshot
(tests/local_map_update_data.bench_snapshot).  The script
  1. checks the device update of every frame against the restatement of update_local_map;
  2. times, alternately, step + update_local_map + track_local_map on the device list, and step + the host path
     (synchronise, download the matches, the native graph walk of tests/local_map_update_oracle.cc over the batch,
     gather and upload the lists and the row mappings) + track_local_map on the uploaded list, each part timed, with a
     device synchronise around each timed step;
  3. times the update's kernels (plp_ctx_kernel_timing) over further update_local_map() calls.
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
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                        "--id=0"], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else f"nvidia-smi failed: {q.stderr.strip()}"


def main():
    import local_map_update_data as lmu
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=1234)
    args = ap.parse_args()
    pkg = bench._load_pkg()
    ctx = pkg.Context(0)
    tctx = pkg.Context(0, high_priority=True)
    fe, snap, aux = lmu.bench_setup(pkg, ctx, args.batch, args.seed, tctx)
    B = args.batch
    lo = fe._last_offsets

    def sync():
        ctx.sync()
        tctx.sync()

    # 1. every frame's update against the restatement
    fe.step(B)
    fe.update_local_map(B)
    sync()
    mot, u = fe.download_tracking(B), fe.download_local_map_update(B)
    for b in range(B):
        rows = snap["last_row_lm"][lo[b]:lo[b + 1]]
        tracked = np.array([rows[q] if q >= 0 else -1 for q in mot["matched"][b]], np.int32)
        w = lmu.device_update(snap, tracked, fe.max_local, lmu.BENCH_MAX_LKF, mot["num_valid"][b] >= 20)
        assert u["status"][b] == w["status"] and list(u["local_lm"][b]) == w["local_lm"], b
    rows_per_frame = np.array([len(x) for x in u["local_lm"]])
    kf_per_frame = np.array([len(x) for x in u["local_kf"]])

    # 2. the device update against the host path, alternately
    def device_step():
        sync()
        t0 = time.perf_counter()
        fe.step(B)
        fe.update_local_map(B)
        fe.track_local_map(B, updated=True)
        sync()
        return 1e3 * (time.perf_counter() - t0)

    def host_step():
        """step, then the round trip the update replaces, each part timed: synchronise and download the matches, the
        native graph walk over the batch (one C++ call), gather the rows and upload the lists; then the local map."""
        sync()
        t0 = time.perf_counter()
        fe.step(B)
        sync()
        t1 = time.perf_counter()
        n_kp = fe.d_n.download(np.int32, (B,))
        matched = fe.d_matched.download(np.int32, (fe.max_batch, fe.cap))[:B]
        num_valid = fe.d_num_valid.download(np.int32, (B,))
        t2 = time.perf_counter()
        offs, lm, lli = lmu.oracle_update_batch(snap, n_kp, matched, num_valid, lo, fe.max_local)
        t3 = time.perf_counter()
        rows = lmu.local_rows(snap, lm)
        lists = [dict({k: v[offs[b]:offs[b + 1]] for k, v in rows.items()}, last_local_idx=lli[lo[b]:lo[b + 1]])
                 for b in range(B)]
        fe.set_local_maps(lists)
        sync()
        t4 = time.perf_counter()
        fe.track_local_map(B)
        sync()
        t5 = time.perf_counter()
        return dict(total=1e3 * (t5 - t0), step=1e3 * (t1 - t0), download=1e3 * (t2 - t1), walk=1e3 * (t3 - t2),
                    upload=1e3 * (t4 - t3), local=1e3 * (t5 - t4))

    for _ in range(args.warmup):
        device_step()
        host_step()
    dev, host = [], []
    for _ in range(args.steps):
        dev.append(device_step())
        host.append(host_step())
    host_total = [h["total"] for h in host]

    # 3. the update's kernels alone (the motion outputs stay as the last step() left them)
    fe.step(B)
    sync()
    lib = fe.lib
    tctx._check(lib.plp_ctx_kernel_timing(tctx.handle, 1))
    for _ in range(args.steps):
        fe.update_local_map(B)
    tctx.sync()
    buf = C.create_string_buffer(1 << 16)
    tctx._check(lib.plp_ctx_kernel_timing_report(tctx.handle, buf, C.c_size_t(len(buf))))
    tctx._check(lib.plp_ctx_kernel_timing(tctx.handle, 0))
    kt = json.loads(buf.value.decode())
    kernels = {k: round(v["total_ms"] / args.steps, 4) for k, v in sorted(kt.items(), key=lambda kv: -kv[1]["total_ms"])}
    res = {"metric": "local_map_update_ms_per_step", "batch": B, "steps": args.steps,
           "keyframes": int(len(snap["kf_erased"])), "landmarks": int(len(snap["lm_erased"])),
           "device_step_update_local_ms_median": round(float(np.median(dev)), 3),
           "host_step_download_walk_upload_local_ms_median": round(float(np.median(host_total)), 3),
           "host_parts_ms_median": {k: round(float(np.median([h[k] for h in host])), 3)
                                    for k in ("step", "download", "walk", "upload", "local")},
           "device_ms_range": [round(min(dev), 3), round(max(dev), 3)],
           "host_ms_range": [round(min(host_total), 3), round(max(host_total), 3)],
           "update_kernels_ms_per_call": kernels,
           "update_kernels_ms_total": round(sum(kernels.values()), 4),
           "local_rows_per_frame": [int(rows_per_frame.min()), int(np.median(rows_per_frame)), int(rows_per_frame.max())],
           "local_keyframes_per_frame": [int(kf_per_frame.min()), int(np.median(kf_per_frame)), int(kf_per_frame.max())],
           "status_counts": {int(s): int((u["status"] == s).sum()) for s in np.unique(u["status"])},
           "card": card()}
    print(json.dumps(res))
    fe.close()


if __name__ == "__main__":
    main()
