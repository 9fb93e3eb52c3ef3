"""GPU parity: solve::pnp_solver::find_via_ransac of many problems through plp_pnp_ransac vs the oracle.  Both sides
compile the same pnpmath.h text without FMA contraction, so poses, flags and counts must be bit-identical."""
import numpy as np
import pytest

import pnp_data as pd
from test_pnp_emu import assert_same, problems

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("P,sizes", [(1, [4096]), (10, [50, 300, 1000, 11]), (64, [30, 300, 1000, 4096])])
def test_pnp_ransac_equals_oracle(ctx, orc, P, sizes):
    off, b, x, mc, sm = problems(P, P, sizes)
    for recompute in (True, False):
        want = pd.oracle_ransac(orc, off, b, x, mc, sm, recompute=recompute)
        got = ctx.pnp_ransac(off, b, x, mc, sm, recompute=recompute)
        assert_same(got, want)
    assert want[0].sum() >= P // 2


def test_pnp_ransac_mixed_and_degenerate(ctx, orc):
    scenes = [pd.make_scene(1, 3), pd.make_scene(2, 8), pd.make_scene(3, 200, 0.5), pd.make_scene(4, 60, 1.0),
              pd.make_scene(5, 0), pd.make_scene(6, 40, planar=True), pd.make_scene(7, 50, 0.2),
              pd.make_scene(8, 500, 0.9)]
    scenes[6]["bearings"][[0, 5]] = [[0.6, 0.8, 0.0], [0.0, 1.0, 0.0]]
    scenes[6]["bearings"][10:20] *= -1
    samples = [pd.draw_samples(i, len(s["bearings"]), 30) for i, s in enumerate(scenes)]
    samples[6][:5] = [[0, 5, 3, 2]] * 5
    samples[2][3] = [7, 7, 7, 9]
    samples[6][7] = [10, 11, 12, 13]
    off, b, x, mc, sm = pd.pack(scenes, samples)
    for recompute in (True, False):
        for mni in (10, 0, 150):
            want = pd.oracle_ransac(orc, off, b, x, mc, sm, min_num_inliers=mni, recompute=recompute)
            assert_same(ctx.pnp_ransac(off, b, x, mc, sm, min_num_inliers=mni, recompute=recompute), want)
    want = pd.oracle_ransac(orc, off, b, x, mc, sm)
    assert want[0][0] == 0 and want[0][2] == 1 and want[0][3] == 0
    z = np.zeros((len(scenes), 0, 4), np.int32)
    assert_same(ctx.pnp_ransac(off, b, x, mc, z), pd.oracle_ransac(orc, off, b, x, mc, z))


def test_pnp_ransac_ties_and_small_problems(ctx, orc):
    """Equal counts with disjoint inlier sets (the first in sample order wins) and valid 4- and 10-point problems."""
    s, sa, sb = pd.tie_scene(orc, 7)
    mixed = np.array([sa[0], sa[1], sb[0], sb[1]], np.int32)
    off, b, x, mc, sm = pd.pack([s, s, s], [np.stack(o) for o in ((mixed, sa, sb), (mixed, sb, sa), (sb, sa, mixed))])
    for recompute in (True, False):
        assert_same(ctx.pnp_ransac(off, b, x, mc, sm, recompute=recompute),
                    pd.oracle_ransac(orc, off, b, x, mc, sm, recompute=recompute))
    off, b, x, mc, sm = problems(3, 8, [4, 10, 11, 5], outlier_frac=0.0)
    want = pd.oracle_ransac(orc, off, b, x, mc, sm, min_num_inliers=0)
    assert_same(ctx.pnp_ransac(off, b, x, mc, sm, min_num_inliers=0), want)
    assert want[0].all()


def test_pnp_ransac_refusals_write_nothing(ctx, plp):
    off, b, x, mc, sm = problems(3, 3, [40])
    bad_sm = sm.copy()
    bad_sm[1, 4, 2] = 40                      # outside [0, n_p)
    bad_off = off.copy()
    bad_off[2] = bad_off[1] - 1               # decreasing
    lib = plp.lib()
    import ctypes as C
    for o, s in ((off, bad_sm), (bad_off, sm), (off + 1, sm)):
        valid, num = np.full(3, 7, np.int32), np.full(3, 7, np.int32)
        pose, flags = np.full(48, 7.0), np.full(120, 7, np.uint8)
        o = np.ascontiguousarray(o, np.int32)
        st = lib.plp_pnp_ransac(ctx.handle, C.c_int(3), pd._ptr(o), pd._ptr(b), pd._ptr(x), pd._ptr(mc),
                                pd._ptr(np.ascontiguousarray(s)), C.c_int(30), C.c_int(10), C.c_int(1), pd._ptr(valid),
                                pd._ptr(num), pd._ptr(pose), pd._ptr(flags))
        assert st == 1
        assert (valid == 7).all() and (num == 7).all() and (pose == 7.0).all() and (flags == 7).all()
    with pytest.raises(plp.PlpError):
        ctx.pnp_ransac(off, b, x, mc, sm, min_num_inliers=-1)
    big = np.zeros((3, 65536, 4), np.int32)                     # num_iter beyond the grid: a capacity refusal
    valid = np.full(3, 7, np.int32)
    st = lib.plp_pnp_ransac(ctx.handle, C.c_int(3), pd._ptr(off), pd._ptr(b), pd._ptr(x), pd._ptr(mc), pd._ptr(big),
                            C.c_int(65536), C.c_int(10), C.c_int(1), pd._ptr(valid), pd._ptr(np.zeros(3, np.int32)),
                            pd._ptr(np.zeros(48)), pd._ptr(np.zeros(120, np.uint8)))
    assert st == 4 and (valid == 7).all()
    with pytest.raises(plp.PlpError):
        lib_st = lib.plp_pnp_ransac(ctx.handle, C.c_int(3), None, None, None, None, None, C.c_int(30), C.c_int(10),
                                    C.c_int(1), None, None, None, None)
        ctx._check(lib_st)
