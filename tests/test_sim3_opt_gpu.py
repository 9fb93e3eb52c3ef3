"""GPU parity: optimize::transform_optimizer::optimize of many problems through plp_sim3_optimize vs the oracle.  Both
compile the same sim3optmath.h text without FMA contraction and reduce in the same order, but the device's sin / cos /
exp / pow are not glibc's, so the Sim3 is compared to a tolerance (1e-8 relative) while counts and inlier flags must be
equal; repeated and batched calls must be bit-identical."""
import ctypes as C

import numpy as np
import pytest

import sim3_opt_data as sd

pytestmark = pytest.mark.gpu


def cams(plp, P):
    return [plp.capi.make_camera(sd.FX, sd.FY, sd.CX, sd.CY, sd.COLS, sd.ROWS)] * P


def run(ctx, plp, d, **kw):
    P = len(d["off"]) - 1
    p1, p2 = d["pose_1w"].reshape(P, 12), d["pose_2w"].reshape(P, 12)
    return ctx.sim3_optimize(d["off"], cams(plp, P), p1[:, :9], p1[:, 9:], p2[:, :9], p2[:, 9:], d["rot"], d["trans"],
                             d["scale"], d["pos_w_1"], d["pos_w_2"], d["obs_1"], d["obs_2"], d["w_1"], d["w_2"], **kw)


def mixed(P, seed=0):
    """P problems cycling through the named scenes with fresh seeds (fix_scale problems keep s = 1)."""
    return [sd.scene(i, seed + 10 * i)[1] for i in range(P)]


@pytest.mark.parametrize("fix_scale", [False, True])
def test_sim3_optimize_equals_oracle_on_every_scene(ctx, orc, plp, fix_scale):
    d = sd.pack([sc for _, sc, _ in sd.scenes(0)])
    want = sd.oracle_optimize(orc, d, fix_scale=fix_scale)
    got = run(ctx, plp, d, fix_scale=fix_scale)
    err = sd.assert_close(got, want, rtol=1e-8)
    print(f"largest relative Sim3 difference to the oracle: {err:.3g}")


def test_sim3_optimize_batch_of_512_equals_oracle_and_is_batch_invariant(ctx, orc, plp):
    scs = mixed(512, 1000)
    d = sd.pack(scs)
    want = sd.oracle_optimize(orc, d)
    got = run(ctx, plp, d)
    err = sd.assert_close(got, want, rtol=1e-8)
    print(f"largest relative Sim3 difference to the oracle over 512 problems: {err:.3g}")
    again = run(ctx, plp, d)
    for a, b in zip(got, again):
        assert a.tobytes() == b.tobytes()
    for p in (0, 3, 6, 100, 511):   # a problem alone equals the same problem inside the batch
        alone = run(ctx, plp, sd.pack([scs[p]]))
        lo, hi = d["off"][p], d["off"][p + 1]
        assert alone[0][0] == got[0][p]
        assert alone[1][0].tobytes() == got[1][p].tobytes() and alone[2][0].tobytes() == got[2][p].tobytes()
        assert alone[3][0] == got[3][p] and alone[4].tobytes() == got[4][lo:hi].tobytes()


def test_sim3_optimize_iteration_counts_and_thresholds(ctx, orc, plp):
    d = sd.pack([sd.make_scene(7, 300, 0.3), sd.make_scene(8, 130, 0.1), sd.make_scene(9, 0),
                 sd.make_scene(10, 2000, 0.25)])
    for num_iter, chi_sq in ((0, 10.0), (1, 10.0), (25, 10.0), (10, 5.99), (1000, 10.0)):
        kw = dict(num_iter=num_iter, chi_sq=np.float32(chi_sq))
        sd.assert_close(run(ctx, plp, d, **kw), sd.oracle_optimize(orc, d, **kw), rtol=1e-8)


def _raw(lib, ctx, plp, d, outs, P=None, chi_sq=10.0, num_iter=10, null=None):
    P = len(d["off"]) - 1 if P is None else P
    cam_arr = (plp.capi.Camera * max(P, 1))(*cams(plp, max(P, 1)))
    p1, p2 = np.ascontiguousarray(d["pose_1w"][:, :9]), np.ascontiguousarray(d["pose_1w"][:, 9:])
    q1, q2 = np.ascontiguousarray(d["pose_2w"][:, :9]), np.ascontiguousarray(d["pose_2w"][:, 9:])
    args = [d["off"], cam_arr, p1, p2, q1, q2, d["rot"], d["trans"], d["scale"], d["pos_w_1"], d["pos_w_2"], d["obs_1"],
            d["obs_2"], d["w_1"], d["w_2"]]
    ptrs = [a if not isinstance(a, np.ndarray) else sd._ptr(a) for a in args]
    if null is not None:
        ptrs[null] = None
    return lib.plp_sim3_optimize(ctx.handle, C.c_int(P), *ptrs, C.c_float(chi_sq), C.c_int(num_iter), C.c_int(0),
                                 *[sd._ptr(o) for o in outs])


def test_sim3_optimize_refusals_write_nothing(ctx, plp):
    d = sd.pack([sd.make_scene(1, 40), sd.make_scene(2, 30), sd.make_scene(3, 20)])
    lib = plp.lib()

    def outs():
        return [np.full(3, 7, np.int32), np.full(27, 7.0), np.full(9, 7.0), np.full(3, 7.0), np.full(90, 7, np.uint8)]

    def untouched(o):
        return all((a == 7).all() for a in o)

    bad = dict(d)
    bad["off"] = d["off"].copy()
    bad["off"][2] = bad["off"][1] - 1                     # decreasing
    shifted = dict(d)
    shifted["off"] = d["off"] + 1                          # not from 0
    for dd in (bad, shifted):
        o = outs()
        assert _raw(lib, ctx, plp, dd, o) == 1 and untouched(o)
    for k in range(15):                                    # every input pointer null in turn
        o = outs()
        assert _raw(lib, ctx, plp, d, o, null=k) == 1 and untouched(o), k
    for k in range(5):                                     # every output pointer null in turn
        o = outs()
        o2 = [None if i == k else a for i, a in enumerate(o)]
        st = lib.plp_sim3_optimize(ctx.handle, C.c_int(3), *[sd._ptr(a) if isinstance(a, np.ndarray) else a for a in
                                   [d["off"], (plp.capi.Camera * 3)(*cams(plp, 3)), np.ascontiguousarray(d["pose_1w"][:, :9]),
                                    np.ascontiguousarray(d["pose_1w"][:, 9:]), np.ascontiguousarray(d["pose_2w"][:, :9]),
                                    np.ascontiguousarray(d["pose_2w"][:, 9:]), d["rot"], d["trans"], d["scale"],
                                    d["pos_w_1"], d["pos_w_2"], d["obs_1"], d["obs_2"], d["w_1"], d["w_2"]]],
                                   C.c_float(10.0), C.c_int(10), C.c_int(0), *[sd._ptr(a) for a in o2])
        assert st == 1 and all((a == 7).all() for i, a in enumerate(o) if i != k), k
    for chi in (0.0, -1.0, float("nan"), float("inf")):
        o = outs()
        assert _raw(lib, ctx, plp, d, o, chi_sq=chi) == 1 and untouched(o), chi
    o = outs()
    assert _raw(lib, ctx, plp, d, o, num_iter=-1) == 1 and untouched(o)
    o = outs()
    assert _raw(lib, ctx, plp, d, o, P=-1) == 1 and untouched(o)
    o = outs()
    assert _raw(lib, ctx, plp, d, o, num_iter=1001) == 4 and untouched(o)   # PLP_ERR_CAPACITY
    with pytest.raises(plp.PlpError):
        run(ctx, plp, d, num_iter=-1)
    # no problems: nothing to do
    o = outs()
    z = sd.pack([])
    assert lib.plp_sim3_optimize(ctx.handle, C.c_int(0), sd._ptr(z["off"]), *([None] * 14), C.c_float(10.0), C.c_int(10),
                                 C.c_int(0), *[sd._ptr(a) for a in o]) == 0 and untouched(o)
