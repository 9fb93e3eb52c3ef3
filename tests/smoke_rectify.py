"""Smoke check of stereo rectification (called by __graft_entry__.smoke()): one small EuRoC-model pair rectified on the
GPU, byte for byte against the rectification oracle."""
import numpy as np


def run(pkg, ctx):
    import rectify_data as rd

    c = rd.CASES["euroc"]
    r = pkg.StereoRectifier(ctx, c["rows"], c["cols"], *rd.rectifier_args("euroc"))
    left, right = rd.texture(1, c["rows"], c["cols"]), rd.texture(2, c["rows"], c["cols"])
    gl, gr = r.rectify(left, right)
    assert np.array_equal(gl, rd.oracle_remap(left, *rd.oracle_maps("euroc", 0))), "left rectification differs"
    assert np.array_equal(gr, rd.oracle_remap(right, *rd.oracle_maps("euroc", 1))), "right rectification differs"
    r.close()
    print("smoke rectify ok: EuRoC stereo pair bit-exact")
