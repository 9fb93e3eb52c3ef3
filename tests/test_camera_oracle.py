"""The oracle's camera::{perspective,fisheye} undistortion, bearings and image bounds (oracle/camera.cc, cammath.h) pinned to
cv2: cv2.undistortPointsIter / cv2.fisheye.undistortPoints with float32 K and D, as the reference calls them.

Where OpenCV's fixed-point iteration converges, the oracle equals cv2 bit for bit.  The perspective loop restated in
cammath.h is the one the documented algorithm describes (20 iterations, stop on a reprojection error below 1e-6, give up
on icdist < 0).  For points where that iteration oscillates without converging -- far outside the image, or under the
synthetic strong barrel distortion -- cv2 4.13 returns other values (for the shipped EuRoC model it returns the exact
inverse of the distortion).  Those points are listed here, not compared; they never arise inside the image of a shipped
configuration, which the tests below check point by point."""

import numpy as np
import pytest

import camera_data as cd
import synth

cv2 = pytest.importorskip("cv2")


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _same(gx, gy, wx, wy):
    return (_bits(gx) == _bits(wx)) & (_bits(gy) == _bits(wy))


def _reprojects(model, K, D, x, y, ux, uy, tol=1e-3):
    """Points whose undistorted position maps back onto the input through the forward model (converged points)."""
    fx, fy, cx, cy = [float(np.float32(v)) for v in K]
    k = [float(np.float32(v)) for v in cd.coeffs5(D)]
    X, Y = (ux.astype(np.float64) - cx) / fx, (uy.astype(np.float64) - cy) / fy
    if model == cd.FISHEYE:
        r = np.hypot(X, Y)
        th = np.arctan(r)
        t2 = th * th
        thd = th * (1 + k[0] * t2 + k[1] * t2 ** 2 + k[2] * t2 ** 3 + k[3] * t2 ** 4)
        s = np.where(r > 0, thd / np.where(r > 0, r, 1), 1.0)
        xd, yd = X * s, Y * s
    else:
        r2 = X * X + Y * Y
        c = 1 + k[0] * r2 + k[1] * r2 ** 2 + k[4] * r2 ** 3
        xd = X * c + 2 * k[2] * X * Y + k[3] * (r2 + 2 * X * X)
        yd = Y * c + k[2] * (r2 + 2 * Y * Y) + 2 * k[3] * X * Y
    return (np.abs(xd * fx + cx - x) < tol) & (np.abs(yd * fy + cy - y) < tol)


@pytest.mark.parametrize("name", list(cd.CONFIGS))
def test_shipped_configs_equal_cv2_inside_the_image(orc, name):
    model, cols, rows, K, D = cd.CONFIGS[name]
    rng = np.random.default_rng(3)
    x = np.concatenate([rng.uniform(0, cols, 20000), [0, cols, 0, cols, K[2], np.float32(K[2])]]).astype(np.float32)
    y = np.concatenate([rng.uniform(0, rows, 20000), [0, 0, rows, rows, K[3], np.float32(K[3])]]).astype(np.float32)
    gx, gy = cd.undistort_keypoints(orc, model, K, D, x, y)
    wx, wy = cd.cv2_undistort(model, K, cd.coeffs5(D), x, y)
    same = _same(gx, gy, wx, wy)
    assert same.all(), f"{(~same).sum()} points differ, first at {x[~same][:3]}, {y[~same][:3]}"
    b = cd.bearings(orc, K, gx, gy)
    assert np.array_equal(b.view(np.uint64), cd.bearings_np(K, wx, wy).view(np.uint64))


@pytest.mark.parametrize("name", list(cd.CONFIGS))
def test_shipped_configs_equal_cv2_at_every_orb_coordinate(orc, name):
    """Every x and every y the extractor can emit at the config's size, paired with every row / column of the image."""
    model, cols, rows, K, D = cd.CONFIGS[name]
    xs, ys = cd.orb_level_coordinates(cols, rows, synth.scale_factors())
    xs, ys = xs[xs <= cols], ys[ys <= rows]
    rng = np.random.default_rng(4)
    x = np.concatenate([xs, rng.choice(xs, len(ys))]).astype(np.float32)
    y = np.concatenate([rng.choice(ys, len(xs)), ys]).astype(np.float32)
    gx, gy = cd.undistort_keypoints(orc, model, K, D, x, y)
    wx, wy = cd.cv2_undistort(model, K, cd.coeffs5(D), x, y)
    assert _same(gx, gy, wx, wy).all()


def test_shipped_configs_equal_cv2_on_real_orb_keypoints(orc):
    import scene
    for name in cd.CONFIGS:
        model, cols, rows, K, D = cd.CONFIGS[name]
        seq = scene.PlanarSequence(seed=5, n_frames=1, rows=rows, cols=cols, fx=K[0], fy=K[1], cx=K[2], cy=K[3])
        import oracle_api
        kps = orc.orb_extract(oracle_api.orb_params(1000, 1.2, 8, 20, 7), seq.frames[0])["kps"]
        assert len(kps) > 500
        gx, gy = cd.undistort_keypoints(orc, model, K, D, kps["x"], kps["y"])
        wx, wy = cd.cv2_undistort(model, K, cd.coeffs5(D), kps["x"], kps["y"])
        assert _same(gx, gy, wx, wy).all(), name


@pytest.mark.parametrize("name", list(cd.ALL))
def test_outside_and_strong_distortions_equal_cv2_where_the_iteration_converges(orc, name):
    model, cols, rows, K, D = cd.ALL[name]
    x, y = cd.test_points(cols, rows, seed=1)
    gx, gy = cd.undistort_keypoints(orc, model, K, D, x, y)
    wx, wy = cd.cv2_undistort(model, K, cd.coeffs5(D), x, y)
    conv = _reprojects(model, K, D, x, y, gx, gy)
    if model == cd.FISHEYE:
        conv |= gx == -1e6   # the failure value is compared too
    same = _same(gx, gy, wx, wy)
    assert same[conv].all(), f"{(~same[conv]).sum()} converged points differ"
    assert conv.sum() > 1000


def test_edge_branches_are_reached(orc):
    """The synthetic models reach fisheye failure (-1e6) where cv2 does, and theta_d > pi/2."""
    model, cols, rows, K, D = cd.SYNTHETIC["fisheye_unstable"]
    x, y = cd.test_points(cols, rows, seed=2)
    gx, _ = cd.undistort_keypoints(orc, model, K, D, x, y)
    wx, _ = cd.cv2_undistort(model, K, cd.coeffs5(D), x, y)
    assert (gx == -1e6).sum() > 100 and np.array_equal(gx == -1e6, wx == -1e6)
    model, cols, rows, K, D = cd.SYNTHETIC["fisheye_wide"]
    assert np.hypot(K[2] / K[0], K[3] / K[1]) > np.pi / 2


def test_zero_distortion(orc):
    """A perspective camera without distortion returns its input bit for bit wherever |x|, |y| >= 1 (every keypoint lies
    further inside than that), so the front end may skip the undistortion.  Near 0 the double round trip
    fx * ((u - cx) / fx) + cx can leave a residue of ~1e-14, which cv2 returns as well.  A fisheye camera with k = 0 is
    still the equidistant model: it is compared with cv2.  Both report the raw image bounds (the reference's
    zero-distortion shortcut)."""
    for name in cd.CONFIGS:
        model, cols, rows, K, _ = cd.CONFIGS[name]
        x, y = cd.test_points(cols, rows, seed=6)
        gx, gy = cd.undistort_keypoints(orc, model, K, np.zeros(5), x, y)
        wx, wy = cd.cv2_undistort(model, K, np.zeros(5), x, y)
        assert _same(gx, gy, wx, wy).all(), name
        if model == cd.PERSPECTIVE:
            away = (np.abs(x) >= 1) & (np.abs(y) >= 1)
            assert away.sum() > 20000 and _same(gx, gy, x, y)[away].all(), name
        assert np.array_equal(cd.image_bounds(orc, model, K, np.zeros(5), cols, rows), [0, cols, 0, rows])


@pytest.mark.parametrize("name", [n for n in cd.ALL if n != "strong_barrel"])  # its corners do not converge
def test_image_bounds_equal_cv2(orc, name):
    model, cols, rows, K, D = cd.ALL[name]
    got = cd.image_bounds(orc, model, K, D, cols, rows)
    want = cd.cv2_image_bounds(model, K, D, cols, rows)
    assert np.array_equal(_bits(got), _bits(want)), (got, want)
