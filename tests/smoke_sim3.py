"""smoke(): one batched Sim3 RANSAC call (a valid and a skipped problem) on the GPU, bit-equal to the oracle."""
from __future__ import annotations

import sim3_data as sd


def run(pkg, ctx, orc):
    scenes = [sd.make_scene(11, 120, 0.5), sd.make_scene(12, 2)]
    samples = [sd.draw_samples(11, 120, 200), sd.draw_samples(12, 2, 200)]
    off, x1, x2, c1, c2, sm = sd.pack(scenes, samples)
    cam = pkg.capi.make_camera(sd.FX, sd.FY, sd.CX, sd.CY, sd.COLS, sd.ROWS)
    got = ctx.sim3_ransac(off, [cam, cam], x1, x2, c1, c2, sm)
    want = sd.oracle_ransac(orc, off, x1, x2, c1, c2, sm)
    sd.assert_same(got, want)
    assert list(got[0]) == [1, 0], got[0]
