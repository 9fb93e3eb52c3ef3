"""Time stereo rectification inside the batched stereo front end.

    python tools/bench_rectify.py [--batch 148] [--steps 20] [--warmup 3] [--seed 1234]

bench.py's stereo layout (two contexts, 752x480, ORB 1000 keypoints, the right image on the second context) with the
EuRoC stereo rectifier (example/euroc/EuRoC_stereo.yaml).  The raw pairs are rendered from synth.make_stereo_pair's
rectified pairs through each camera's model (cv2.undistortPoints with R and P = K_rect gives a raw pixel's rectified
position).  Two chains alternate step by step in one process, CUDA events around each step:
  raw:        plp_stereo_rectify_batch_dev left / right -> ORB left / right on the rectified device buffers -> stereo
  rectified:  ORB left / right on the pre-rectified pairs -> stereo
and CUDA events around each rectify launch.  Then both sides' rectify launches alone, on their two streams, inside one
event span: the kernel's bytes over that span give its share of HBM bandwidth with the two sides overlapping as they do in
the chain.  Prints one JSON line with the card's name, power limit and SM clock read in
the same run; writes nothing."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import subprocess
import sys
from pathlib import Path

import numpy as np

sys.dont_write_bytecode = True
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
import bench  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def raw_pairs(batch, seed):
    import cv2
    import rectify_data as rd
    import synth
    c = rd.CASES["euroc"]
    H, W = c["rows"], c["cols"]
    maps = []
    for side in (0, 1):
        K, D, R = rd.side_params("euroc", side)
        yy, xx = np.mgrid[0:H, 0:W]
        pts = np.stack([xx.ravel(), yy.ravel()], 1).astype(np.float64).reshape(-1, 1, 2)
        u = cv2.undistortPoints(pts, K, D, R=R, P=rd.k_rect32(c["rect"]).astype(np.float64)).reshape(H, W, 2)
        maps.append((u[..., 0].astype(np.float32), u[..., 1].astype(np.float32)))
    n_base = min(batch, 6)
    pairs = [synth.make_stereo_pair(seed + 31 * i, H, W, bf=c["bf"], plp=True)[:2] for i in range(n_base)]
    rng = np.random.default_rng(seed)
    rect = np.empty((2, batch, H, W), np.uint8)
    raw = np.empty_like(rect)
    for b in range(batch):
        sh = (0, 0) if b < n_base else (int(rng.integers(-40, 41)), int(rng.integers(-60, 61)))
        for s in (0, 1):
            rect[s, b] = np.roll(pairs[b % n_base][s], sh, axis=(0, 1))
    for s in (0, 1):
        for b in range(batch):
            raw[s, b] = cv2.remap(rect[s, b], maps[s][0], maps[s][1], cv2.INTER_LINEAR)
    return rect, raw


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                        "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else f"nvidia-smi failed: {q.stderr.strip()}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=148)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1234)
    args = ap.parse_args()
    import torch
    import rectify_data as rd
    pkg = bench._load_pkg()
    from plpslam_b200.tracking import DeviceBuffer
    lib = pkg.lib()
    B = args.batch
    c = rd.CASES["euroc"]
    H, W, bf = c["rows"], c["cols"], c["bf"]
    baseline = bf / c["rect"][0]
    rect, raw = raw_pairs(B, args.seed)
    ctx, ctx_r = pkg.Context(0), pkg.Context(0)
    ctxs = (ctx, ctx_r)
    streams = [torch.cuda.ExternalStream(lib.plp_ctx_stream(cx.handle), device="cuda:0") for cx in ctxs]
    rectifier = pkg.StereoRectifier(ctx, H, W, *rd.rectifier_args("euroc"))
    ext = [pkg.OrbExtractor(cx, H, W, max_batch=B) for cx in ctxs]
    cap = ext[0].capacity
    step_out = (W + 15) // 16 * 16
    d_raw = [DeviceBuffer.from_array(ctxs[s], raw[s]) for s in (0, 1)]
    d_pre = [DeviceBuffer.from_array(ctxs[s], rect[s]) for s in (0, 1)]
    d_rect = [DeviceBuffer(ctxs[s], B * H * step_out) for s in (0, 1)]
    kp = [DeviceBuffer(ctx, B * cap * pkg.KP_DTYPE.itemsize) for _ in range(2)]
    ds = [DeviceBuffer(ctx, B * cap * 32) for _ in range(2)]
    nk = [DeviceBuffer(ctx, B * 4) for _ in range(2)]
    st = [DeviceBuffer(ctx, B * 4) for _ in range(2)]
    d_xr, d_dp = DeviceBuffer(ctx, B * cap * 4), DeviceBuffer(ctx, B * cap * 4)
    rect_ms = [[], []]

    def step(chain, timed=False):
        for s in (1, 0):
            cx = ctxs[s]
            if chain == "raw":
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
                ev[0].record(streams[s])
                rectifier.rectify_dev(s, d_raw[s].ptr, B, W, d_rect[s].ptr, step_out, ctx=cx)
                ev[1].record(streams[s])
                if timed:
                    rect_ms[s].append(ev)
                src, step_in = d_rect[s].ptr, step_out
            else:
                src, step_in = d_pre[s].ptr, W
            cx._check(lib.plp_orb_extract_batch_dev(ext[s].handle, src, C.c_int(B), C.c_size_t(step_in), kp[s].ptr,
                                                    ds[s].ptr, nk[s].ptr, st[s].ptr))
        ctx.wait(ctx_r)
        ctx._check(lib.plp_stereo_compute_batch_dev(ctx.handle, ext[0].handle, ext[1].handle, C.c_int(B), kp[0].ptr,
                                                    ds[0].ptr, nk[0].ptr, kp[1].ptr, ds[1].ptr, nk[1].ptr, C.c_float(bf),
                                                    C.c_float(baseline), d_xr.ptr, d_dp.ptr, None))
        ctx_r.wait(ctx)   # the next step's right ORB pass overwrites the right pyramid the stereo match reads

    chains = ("raw", "rectified")
    for _ in range(args.warmup):
        for ch in chains:
            step(ch)
    ctx.sync()
    ctx_r.sync()
    ms = {ch: 0.0 for ch in chains}
    matches = {}
    for _ in range(args.steps):
        for ch in chains:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(streams[0])
            step(ch, timed=True)
            e1.record(streams[0])
            e1.synchronize()
            ctx_r.sync()
            ms[ch] += e0.elapsed_time(e1)
            n_l = nk[0].download(np.int32, (B,))
            xr = d_xr.download(np.float32, (B, cap))
            matches[ch] = int(sum(int((xr[b, :n_l[b]] >= 0).sum()) for b in range(B)))
    r_ms = [float(np.mean([a.elapsed_time(b) for a, b in rect_ms[s]])) for s in (0, 1)]
    both = []
    for _ in range(args.steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(streams[0])
        ctx_r.wait(ctx)
        for s in (1, 0):
            rectifier.rectify_dev(s, d_raw[s].ptr, B, W, d_rect[s].ptr, step_out, ctx=ctxs[s])
        ctx.wait(ctx_r)
        e1.record(streams[0])
        e1.synchronize()
        both.append(e0.elapsed_time(e1))
    both_ms = float(np.mean(both))
    alg_bytes = 2 * (H * W + H * W)  # per stereo frame: each side gathers and writes W x H bytes
    map_bytes = 2 * H * ((W + 3) // 4 * 4) * 6  # both sides' fixed-point maps, read at least once per launch
    print(json.dumps({
        "raw_ms_per_step": ms["raw"] / args.steps, "rectified_ms_per_step": ms["rectified"] / args.steps,
        "raw_stereo_frames_per_s": B * args.steps / (ms["raw"] * 1e-3),
        "rectified_stereo_frames_per_s": B * args.steps / (ms["rectified"] * 1e-3),
        "rectify_launch_ms_in_chain": {"left": r_ms[0], "right": r_ms[1]}, "batch": B,
        "rectify_both_sides_ms_per_batch": both_ms,
        "rectify_alg_bytes_per_stereo_frame": alg_bytes, "rectify_map_bytes_per_batch": map_bytes,
        "rectify_kernel_share_of_hbm_peak": (alg_bytes * B + map_bytes) / (both_ms * 1e-3) / HBM_BYTES_PER_S,
        "stereo_matches_per_step": matches,
        "gpu_name_power_limit_sm_clock_max_sm_clock": gpu_info()}))
    for d in d_raw + d_pre + d_rect + kp + ds + nk + st + [d_xr, d_dp]:
        d.free()
    for e in ext:
        e.close()
    rectifier.close()
    ctx_r.close()
    ctx.close()


if __name__ == "__main__":
    main()
