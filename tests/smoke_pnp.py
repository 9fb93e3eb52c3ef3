"""smoke(): one batched EPnP RANSAC call (a valid and a skipped candidate) on the GPU, bit-equal to the oracle."""
from __future__ import annotations

import numpy as np

import pnp_data as pd


def run(pkg, ctx, orc):
    scenes = [pd.make_scene(11, 120, 0.5), pd.make_scene(12, 3)]
    samples = [pd.draw_samples(11, 120, 30), pd.draw_samples(12, 3, 30)]
    off, b, x, mc, sm = pd.pack(scenes, samples)
    got = ctx.pnp_ransac(off, b, x, mc, sm)
    want = pd.oracle_ransac(orc, off, b, x, mc, sm)
    assert all(np.array_equal(g, w, equal_nan=True) for g, w in zip(got, want)), "EPnP RANSAC disagrees with the oracle"
    assert list(got[0]) == [1, 0], got[0]
