"""Latency of LSD + LBD extraction for small batches: one warp per frame vs the speculative multi-warp region growing
(lines.cu lsd_grow_mw_kernel) and the out-of-order one (lsd_grow_ooo_kernel).  Run on the GPU box:
python tools/lsd_latency.py"""
import ctypes as C
import json
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests"))
import conftest  # noqa: E402
import synth  # noqa: E402

plp = conftest.load_package()
ctx = plp.Context(0)
lib = plp.lib()
H, W = 480, 640
frames = {"plp": np.stack([synth.make_plp_texture(100 + i, H, W) for i in range(8)]),
          "lines": np.stack([synth.make_line_image(20 + i, H, W) for i in range(8)]),
          "texture": np.stack([synth.make_texture(3 + i, H, W) for i in range(8)])}


def timed(trk, imgs, reps=5):
    trk.extract_batch(imgs)
    ctx.sync()
    t0 = time.perf_counter()
    for _ in range(reps):
        trk.extract_batch(imgs)
    ctx.sync()
    return 1e3 * (time.perf_counter() - t0) / reps


def kernel_ms(trk, imgs):
    ctx._check(lib.plp_ctx_kernel_timing(ctx.handle, 1))
    for _ in range(3):
        trk.extract_batch(imgs)
    buf = C.create_string_buffer(1 << 16)
    ctx._check(lib.plp_ctx_kernel_timing_report(ctx.handle, buf, C.c_size_t(len(buf))))
    ctx._check(lib.plp_ctx_kernel_timing(ctx.handle, 0))
    kt = json.loads(buf.value.decode())
    return {k.split("<")[0].replace("_kernel", ""): round(v["total_ms"] / v["count"], 3) for k, v in kt.items()}


for kind, fr in frames.items():
    for batch in (1,):
        imgs = np.concatenate([fr] * ((batch + 7) // 8))[:batch]
        trk = plp.LineFeatureTracker(ctx, H, W, max_batch=batch)
        out = {}
        for variant in (1, 2, 3):
            trk.grow_variant(variant)
            out[variant] = (timed(trk, imgs), kernel_ms(trk, imgs))
            if variant == 2:
                st = trk.grow_stats(0)
        st3 = trk.grow_stats(0, ooo=True)
        n = len(trk.extract_batch(imgs)[0][0])
        print(f"{kind:8s} batch={batch:3d} keylines[0]={n:4d}  one-warp: {out[1][0]:7.2f} ms/call (grow {out[1][1].get('lsd_grow')})"
              f"   multi-warp: {out[2][0]:7.2f} ms/call (grow {out[2][1].get('lsd_grow_mw')})  stats {st}\n"
              f"          out-of-order: {out[3][0]:7.2f} ms/call (grow {out[3][1].get('lsd_grow_ooo')})  stats {st3}")
        if batch == 1 and kind == "plp":
            print("    kernels (multi-warp run):", out[2][1])
        trk.close()
