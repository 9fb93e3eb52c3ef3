"""GPU parity: solve::sim3_solver::find_via_ransac of many problems through plp_sim3_ransac vs the oracle.  Both sides
compile the same sim3math.h text without FMA contraction, so validity, counts and the winning Sim3 must be bit-identical."""
import ctypes as C

import numpy as np
import pytest

import sim3_data as sd

pytestmark = pytest.mark.gpu


def cams(plp, P):
    return [plp.capi.make_camera(sd.FX, sd.FY, sd.CX, sd.CY, sd.COLS, sd.ROWS)] * P


@pytest.mark.parametrize("P,sizes", [(1, [4096]), (16, [20, 50, 300, 1000]), (256, [30, 120, 300, 4096, 50, 700])])
def test_sim3_ransac_equals_oracle(ctx, orc, plp, P, sizes):
    for fix_scale in (False, True):
        off, x1, x2, c1, c2, sm = sd.problems(P, P, sizes, fix_scale=fix_scale)
        want = sd.oracle_ransac(orc, off, x1, x2, c1, c2, sm, fix_scale=fix_scale)
        got = ctx.sim3_ransac(off, cams(plp, P), x1, x2, c1, c2, sm, fix_scale=fix_scale)
        sd.assert_same(got, want)
        assert want[0].sum() >= P // 2


def test_sim3_ransac_mixed_and_degenerate(ctx, orc, plp):
    scenes = [sd.make_scene(1, 2), sd.make_scene(2, 15), sd.make_scene(3, 200, 0.5), sd.make_scene(4, 60, 1.0),
              sd.make_scene(5, 0), sd.make_scene(6, 80, 0.3, behind_1=5, behind_2=4), sd.make_scene(7, 3),
              sd.make_scene(8, 500, 0.9)]
    samples = [sd.draw_samples(i, len(s["pts_1"]), 200) for i, s in enumerate(scenes)]
    samples[2][3] = [7, 7, 9]
    samples[2][4] = [1, 1, 1]
    samples[5][0] = [0, 1, 2]
    samples[5][1] = [79, 78, 77]
    off, x1, x2, c1, c2, sm = sd.pack(scenes, samples)
    P = len(scenes)
    for fix_scale in (False, True):
        for mni in (20, 0, 3, 150):
            want = sd.oracle_ransac(orc, off, x1, x2, c1, c2, sm, fix_scale=fix_scale, min_num_inliers=mni)
            sd.assert_same(ctx.sim3_ransac(off, cams(plp, P), x1, x2, c1, c2, sm, fix_scale=fix_scale,
                                           min_num_inliers=mni), want)
    want = sd.oracle_ransac(orc, off, x1, x2, c1, c2, sm)
    assert want[0][0] == 0 and want[0][2] == 1 and want[0][3] == 0 and want[0][5] == 1
    # per-problem cameras
    cs = [plp.capi.make_camera(400.0 + 10 * i, 420.0, 300.0 + i, 250.0, sd.COLS, sd.ROWS) for i in range(P)]
    cams4 = np.array([[c.fx, c.fy, c.cx, c.cy] for c in cs])
    sd.assert_same(ctx.sim3_ransac(off, cs, x1, x2, c1, c2, sm),
                   sd.oracle_ransac(orc, off, x1, x2, c1, c2, sm, cams=cams4))
    z = np.zeros((P, 0, 3), np.int32)
    for mni in (20, 0):
        sd.assert_same(ctx.sim3_ransac(off, cams(plp, P), x1, x2, c1, c2, z, min_num_inliers=mni),
                       sd.oracle_ransac(orc, off, x1, x2, c1, c2, z, min_num_inliers=mni))


def test_sim3_ransac_first_best_ties(ctx, orc, plp):
    tie = sd.concat(sd.make_scene(41, 20, noise_px=0.0, scale=2.0), sd.make_scene(42, 20, noise_px=0.0, scale=0.5))
    sa, sb = [0, 1, 2], [20, 21, 22]
    off, x1, x2, c1, c2, sm = sd.pack([tie, tie], [np.array([sa, sb] * 5, np.int32), np.array([sb, sa] * 5, np.int32)])
    want = sd.oracle_ransac(orc, off, x1, x2, c1, c2, sm)
    sd.assert_same(ctx.sim3_ransac(off, cams(plp, 2), x1, x2, c1, c2, sm), want)
    assert list(want[1]) == [20, 20] and want[4][0] != want[4][1]


def _raw(lib, ctx, off, cam_arr, x1, x2, c1, c2, sm, num_iter, outs, mni=20):
    p = sd._ptr
    return lib.plp_sim3_ransac(ctx.handle, C.c_int(len(off) - 1 if off is not None else 3), p(off), cam_arr, p(x1), p(x2),
                               p(c1), p(c2), p(sm), C.c_int(num_iter), C.c_int(0), C.c_int(mni), *[p(o) for o in outs])


def test_sim3_ransac_refusals_write_nothing(ctx, plp):
    off, x1, x2, c1, c2, sm = sd.problems(3, 3, [40], num_iter=30)
    cam_arr = (plp.capi.Camera * 3)(*cams(plp, 3))
    lib = plp.lib()
    bad_sm = sm.copy()
    bad_sm[1, 4, 2] = 40                      # outside [0, n_p)
    neg_sm = sm.copy()
    neg_sm[2, 0, 0] = -1
    bad_off = off.copy()
    bad_off[2] = bad_off[1] - 1               # decreasing

    def outs():
        return [np.full(3, 7, np.int32), np.full(3, 7, np.int32), np.full(27, 7.0), np.full(9, 7.0),
                np.full(3, 7, np.float32)]

    def untouched(o):
        return all((a == 7).all() for a in o)

    for o_, s_ in ((off, bad_sm), (off, neg_sm), (bad_off, sm), (off + 1, sm)):
        o = outs()
        st = _raw(lib, ctx, np.ascontiguousarray(o_, np.int32), cam_arr, x1, x2, c1, c2, np.ascontiguousarray(s_), 30, o)
        assert st == 1 and untouched(o)
    for args in ((None, cam_arr, x1), (off, None, x1), (off, cam_arr, None)):   # null pointers
        o = outs()
        st = _raw(lib, ctx, args[0], args[1], args[2], x2, c1, c2, sm, 30, o)
        assert st == 1 and untouched(o)
    o = outs()
    assert _raw(lib, ctx, off, cam_arr, x1, x2, c1, c2, sm, 30, o, mni=-1) == 1 and untouched(o)
    o = outs()
    assert _raw(lib, ctx, off, cam_arr, x1, x2, c1, c2, sm, -1, o) == 1 and untouched(o)
    with pytest.raises(plp.PlpError):
        ctx.sim3_ransac(off, cams(plp, 3), x1, x2, c1, c2, sm, min_num_inliers=-1)
    # a skipped problem's out-of-range samples are not read: n = 2 < 3
    o = outs()
    off2, y1, y2, d1, d2, _ = sd.pack([sd.make_scene(1, 2)] * 3, [np.zeros((30, 3), np.int32)] * 3)
    junk = np.full((3, 30, 3), 99, np.int32)
    assert _raw(lib, ctx, off2, cam_arr, y1, y2, d1, d2, junk, 30, o) == 0
    assert not o[0].any() and not o[1].any() and not o[2].any() and not o[3].any() and not o[4].any()
    # num_iter beyond the grid: a capacity refusal before anything is read or written
    big = np.zeros((3, 65536, 3), np.int32)
    o = outs()
    assert _raw(lib, ctx, off, cam_arr, x1, x2, c1, c2, big, 65536, o) == 4 and untouched(o)
