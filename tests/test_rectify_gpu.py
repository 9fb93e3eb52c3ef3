"""GPU stereo rectification (plp_stereo_rectifier_*, plp_stereo_rectify, plp_stereo_rectify_batch_dev) against the oracle
(tests/rectify_oracle.cc, pinned to cv2 by test_rectify_oracle.py), and the device-resident chain raw pair -> rectify ->
ORB -> stereo against the oracle chain."""
import ctypes as C
import hashlib
from pathlib import Path

import numpy as np
import pytest

import oracle_api
import rectify_data as rd
import synth
from test_batch_dev_gpu import _OrbOut, _check_orb, _orb_ref

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).resolve().parent / "golden" / "cv2_rectify.npz"
PLP_ERR_INVALID = 1


def _rectifier(plp, ctx, case):
    c = rd.CASES[case]
    return plp.StereoRectifier(ctx, c["rows"], c["cols"], *rd.rectifier_args(case))


def _round16(n):
    return (n + 15) // 16 * 16


@pytest.mark.parametrize("case", list(rd.CASES))
def test_maps_equal_oracle_and_golden(ctx, plp, case):
    g = np.load(GOLDEN)
    r = _rectifier(plp, ctx, case)
    for side in (0, 1):
        mx, my = r.maps(side)
        ox, oy = rd.oracle_maps(case, side)
        assert np.array_equal(mx.view(np.uint32), ox.view(np.uint32)) and np.array_equal(my.view(np.uint32), oy.view(np.uint32))
        assert hashlib.sha256(mx.tobytes() + my.tobytes()).hexdigest() == str(g[f"{case}_{side}_sha256"])
    r.close()


@pytest.mark.parametrize("case", ["euroc", "tumvi", "odd_tangential"])
def test_host_rectify_equals_oracle(ctx, plp, case):
    c = rd.CASES[case]
    r = _rectifier(plp, ctx, case)
    left, right = rd.texture(60, c["rows"], c["cols"]), rd.texture(61, c["rows"], c["cols"])
    n0 = ctx.launch_count()
    gl, gr = r.rectify(left, right)
    assert ctx.launch_count() == n0 + 2
    assert np.array_equal(gl, rd.oracle_remap(left, *rd.oracle_maps(case, 0)))
    assert np.array_equal(gr, rd.oracle_remap(right, *rd.oracle_maps(case, 1)))
    # a row stride larger than cols on both sides
    lib = plp.lib()
    src = np.zeros((c["rows"], c["cols"] + 7), np.uint8)
    src[:, :c["cols"]] = left
    dst = np.full((2, c["rows"], c["cols"] + 3), 9, np.uint8)
    ctx._check(lib.plp_stereo_rectify(ctx.handle, r.handle, src.ctypes.data_as(C.c_void_p), src.ctypes.data_as(C.c_void_p),
                                      C.c_size_t(src.strides[0]), dst[0].ctypes.data_as(C.c_void_p),
                                      dst[1].ctypes.data_as(C.c_void_p), C.c_size_t(dst.strides[1])))
    assert np.array_equal(dst[0, :, :c["cols"]], gl) and np.array_equal(dst[1, :, :c["cols"]], rd.oracle_remap(
        left, *rd.oracle_maps(case, 1))) and (dst[:, :, c["cols"]:] == 9).all()
    r.close()


def _frames(seed, B, rows, cols):
    """B frames: a few textures, then shifted copies (like bench_stereo's batch), one unrelated noise frame."""
    base = [rd.texture(seed + i, rows, cols) for i in range(3)]
    rng = np.random.default_rng(seed)
    out = np.empty((B, rows, cols), np.uint8)
    for b in range(B):
        out[b] = np.roll(base[b % 3], (int(rng.integers(-40, 41)), int(rng.integers(-60, 61))), axis=(0, 1))
    out[B // 2] = rng.integers(0, 256, (rows, cols), dtype=np.uint8)
    return out


@pytest.mark.parametrize("case,batch,in_pad,out_extra", [
    ("euroc", 1, 0, 0), ("euroc", 3, 16, 64), ("euroc", 148, 0, 64), ("euroc", 148, 16, 0),
    ("tumvi", 1, 16, 0), ("tumvi", 3, 0, 64), ("tumvi", 148, 16, 64), ("odd_tangential", 3, 16, 0)])
def test_batch_dev_equals_oracle(ctx, plp, case, batch, in_pad, out_extra):
    """Left on one context, right on a second one, as bench_stereo runs them; pitched inputs and outputs; bytes past
    `cols` of every output row keep their value."""
    from plpslam_b200.tracking import DeviceBuffer
    c = rd.CASES[case]
    rows, cols = c["rows"], c["cols"]
    in_step, out_step = cols + in_pad, _round16(cols) + out_extra
    ctx_r = plp.Context(ctx.device)
    r = _rectifier(plp, ctx, case)
    sides = []
    for side, cx in ((0, ctx), (1, ctx_r)):
        frames = _frames(100 + 10 * side + batch, batch, rows, cols)
        host = np.random.default_rng(side).integers(0, 256, (batch, rows, in_step), dtype=np.uint8)
        host[:, :, :cols] = frames
        d_in = DeviceBuffer.from_array(cx, host)
        d_out = DeviceBuffer.from_array(cx, np.full((batch, rows, out_step), 0xA5, np.uint8))
        n0 = cx.launch_count()
        r.rectify_dev(side, d_in.ptr, batch, in_step, d_out.ptr, out_step, ctx=cx)
        assert cx.launch_count() == n0 + 1
        sides.append((frames, d_in, d_out, cx))
    for side, (frames, d_in, d_out, cx) in enumerate(sides):
        cx.sync()
        got = d_out.download(np.uint8, (batch, rows, out_step))
        mx, my = rd.oracle_maps(case, side)
        for b in range(batch):
            assert np.array_equal(got[b, :, :cols], rd.oracle_remap(frames[b], mx, my)), f"side {side} frame {b}"
        assert (got[:, :, cols:] == 0xA5).all()
        d_in.free()
        d_out.free()
    r.close()
    ctx_r.close()


def test_rejected_calls_launch_nothing(ctx, plp):
    from plpslam_b200.tracking import DeviceBuffer
    lib = plp.lib()
    c = rd.CASES["euroc"]
    rows, cols = c["rows"], c["cols"]
    r = _rectifier(plp, ctx, "euroc")
    d_in, d_out = DeviceBuffer(ctx, 2 * rows * 800), DeviceBuffer(ctx, 2 * rows * 800 + 64)
    n0 = ctx.launch_count()
    P = C.c_void_p
    ok = (ctx.handle, r.handle, 0, d_in.ptr, 2, cols, d_out.ptr, 768)

    def call(*a):
        h, rr, side, di, b, si, do, so = a
        return lib.plp_stereo_rectify_batch_dev(h, rr, C.c_int(side), di, C.c_int(b), C.c_size_t(si), do, C.c_size_t(so))

    bad = [(None,) + ok[1:], ok[:1] + (None,) + ok[2:], ok[:2] + (2,) + ok[3:], ok[:2] + (-1,) + ok[3:],
           ok[:3] + (None,) + ok[4:], ok[:4] + (-1,) + ok[5:], ok[:5] + (cols - 1,) + ok[6:], ok[:6] + (None, 768),
           ok[:6] + (P(d_out.ptr.value + 4), 768), ok[:6] + (d_out.ptr, 760), ok[:6] + (d_out.ptr, 752 + 4),
           ok[:6] + (d_out.ptr, 736)]
    for a in bad:
        assert call(*a) == PLP_ERR_INVALID, a
        assert lib.plp_last_error()
    img = np.zeros((rows, cols), np.uint8)
    p = img.ctypes.data_as(P)
    assert lib.plp_stereo_rectify(ctx.handle, r.handle, p, p, C.c_size_t(cols - 1), p, p, C.c_size_t(cols)) == PLP_ERR_INVALID
    assert lib.plp_stereo_rectify(ctx.handle, r.handle, p, None, C.c_size_t(cols), p, p, C.c_size_t(cols)) == PLP_ERR_INVALID
    assert lib.plp_stereo_rectify(ctx.handle, r.handle, p, p, C.c_size_t(cols), p, p, C.c_size_t(10)) == PLP_ERR_INVALID
    mx = np.zeros((rows, cols), np.float32)
    assert lib.plp_stereo_rectifier_maps(r.handle, C.c_int(2), mx.ctypes.data_as(P), mx.ctypes.data_as(P)) == PLP_ERR_INVALID
    assert ctx.launch_count() == n0
    assert call(*ok[:4] + (0,) + ok[5:]) == 0 and ctx.launch_count() == n0   # an empty batch: nothing to do
    # the constructor: model 2, a singular K_rect * R, sizes <= 0
    args = list(rd.rectifier_args("euroc"))
    for model, R_l, rc in ((2, args[3], (rows, cols)), (0, np.zeros((3, 3)), (rows, cols)), (0, args[3], (0, cols)),
                           (0, args[3], (rows, -3))):
        a = list(args)
        a[0], a[3] = model, R_l
        with pytest.raises(plp.PlpError, match="invalid argument"):
            plp.StereoRectifier(ctx, rc[0], rc[1], *a)
    assert ctx.launch_count() == n0
    d_in.free()
    d_out.free()
    r.close()


# ------------------------------------------------------------------------------------------------ raw pair -> stereo
def _unrectify_maps(case, side):
    """For every raw pixel, its position in the rectified image (cv2.undistortPoints / cv2.fisheye.undistortPoints with
    R and P = K_rect): remapping a rectified image through these maps renders the raw camera image."""
    import cv2
    c = rd.CASES[case]
    K, D, R = rd.side_params(case, side)
    P = rd.k_rect32(c["rect"]).astype(np.float64)
    yy, xx = np.mgrid[0:c["rows"], 0:c["cols"]]
    pts = np.stack([xx.ravel(), yy.ravel()], 1).astype(np.float64).reshape(-1, 1, 2)
    if c["model"] == rd.FISHEYE:
        u = cv2.fisheye.undistortPoints(pts, K, np.asarray(D, np.float64)[:4], R=R, P=P)
    else:
        u = cv2.undistortPoints(pts, K, np.asarray(D, np.float64), R=R, P=P)
    u = u.reshape(c["rows"], c["cols"], 2).astype(np.float32)
    return u[..., 0].copy(), u[..., 1].copy()


@pytest.mark.parametrize("case", list(rd.REFERENCE_CASES))
def test_chain_from_raw_pairs_equals_oracle(ctx, orc, plp, case):
    """Raw pairs rendered from rectified synthetic pairs -> plp_stereo_rectify_batch_dev (left and right on two
    contexts) -> plp_orb_extract_batch_dev on the rectified device buffers -> plp_stereo_compute_batch_dev, against
    oracle remap -> oracle ORB -> oracle stereo, bit for bit."""
    pytest.importorskip("cv2")
    from plpslam_b200.tracking import DeviceBuffer
    lib = plp.lib()
    c = rd.CASES[case]
    H, W, bf = c["rows"], c["cols"], c["bf"]
    baseline = bf / c["rect"][0]
    N = 3
    rect_pairs = [synth.make_stereo_pair(300 + 11 * i, H, W, bf=bf, plp=i % 2 == 0)[:2] for i in range(N)]
    raw = [np.stack([rd.oracle_remap(p[s], *_unrectify_maps(case, s)) for p in rect_pairs]) for s in (0, 1)]
    ctx_r = plp.Context(ctx.device)
    r = _rectifier(plp, ctx, case)
    step = _round16(W)
    el, er = plp.OrbExtractor(ctx, H, W, max_batch=N), plp.OrbExtractor(ctx_r, H, W, max_batch=N)
    cap = el.capacity
    d_raw = [DeviceBuffer.from_array(cx, raw[s]) for s, cx in ((0, ctx), (1, ctx_r))]
    d_rect = [DeviceBuffer(cx, N * H * step) for cx in (ctx, ctx_r)]
    out = [_OrbOut(plp, ctx, N, cap), _OrbOut(plp, ctx, N, cap)]
    d_xr, d_dp = DeviceBuffer(ctx, N * cap * 4), DeviceBuffer(ctx, N * cap * 4)
    r.rectify_dev(1, d_raw[1].ptr, N, W, d_rect[1].ptr, step, ctx=ctx_r)
    out[1].run(er, d_rect[1].ptr, N, step)
    r.rectify_dev(0, d_raw[0].ptr, N, W, d_rect[0].ptr, step, ctx=ctx)
    out[0].run(el, d_rect[0].ptr, N, step)
    ctx.wait(ctx_r)
    ctx._check(lib.plp_stereo_compute_batch_dev(ctx.handle, el.handle, er.handle, C.c_int(N), out[0].kp.ptr,
                                                out[0].desc.ptr, out[0].n.ptr, out[1].kp.ptr, out[1].desc.ptr, out[1].n.ptr,
                                                C.c_float(bf), C.c_float(baseline), d_xr.ptr, d_dp.ptr, None))
    xr = d_xr.download(np.float32, (N, cap))
    dp = d_dp.download(np.float32, (N, cap))
    # the oracle chain
    rect_o = [np.stack([rd.oracle_remap(raw[s][b], *rd.oracle_maps(case, s)) for b in range(N)]) for s in (0, 1)]
    n_l = _check_orb(orc, plp, out[0], rect_o[0], "left")
    _check_orb(orc, plp, out[1], rect_o[1], "right")
    tab = orc.orb_tables(oracle_api.orb_params())
    for b in range(N):
        ox, od, _ = orc.stereo_compute(_orb_ref(orc, rect_o[0][b]), _orb_ref(orc, rect_o[1][b]), tab["scale_factors"], tab["inv_scale_factors"], bf, baseline)
        k = n_l[b]
        assert np.array_equal(xr[b, :k], ox, equal_nan=True), f"frame {b}: stereo_x_right"
        assert np.array_equal(dp[b, :k], od, equal_nan=True), f"frame {b}: depths"
        assert int((ox >= 0).sum()) > 100, f"frame {b}: {int((ox >= 0).sum())} stereo matches"
    for d in d_raw + d_rect + [d_xr, d_dp]:
        d.free()
    for o in out:
        o.free()
    el.close()
    er.close()
    r.close()
    ctx_r.close()
