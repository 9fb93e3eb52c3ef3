"""smoke(): one batched Sim3 optimiser call (an optimised problem and one that returns after round 1) on the GPU,
checked against the oracle."""
from __future__ import annotations

import sim3_opt_data as sd


def run(pkg, ctx, orc):
    d = sd.pack([sd.make_scene(21, 150, 0.2), sd.make_scene(22, 15, 0.8)])
    cam = pkg.capi.make_camera(sd.FX, sd.FY, sd.CX, sd.CY, sd.COLS, sd.ROWS)
    p1, p2 = d["pose_1w"], d["pose_2w"]
    got = ctx.sim3_optimize(d["off"], [cam, cam], p1[:, :9], p1[:, 9:], p2[:, :9], p2[:, 9:], d["rot"], d["trans"],
                            d["scale"], d["pos_w_1"], d["pos_w_2"], d["obs_1"], d["obs_2"], d["w_1"], d["w_2"])
    want = sd.oracle_optimize(orc, d)
    sd.assert_close(got, want, rtol=1e-8)
    assert got[0][0] >= 100 and got[0][1] == 0, got[0]
