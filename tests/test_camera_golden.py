"""tests/golden/cv2_undistort.npz (tools/gen_golden.py): cv2's undistortion of seeded points for every camera of
camera_data.py, frozen with the oracle's result and image bounds, so that the oracle and the GPU path stay pinned without
cv2.  The stored cv2 and oracle values differ only where OpenCV's iteration does not converge (see test_camera_oracle.py);
inside the image of every shipped configuration they are identical."""
from pathlib import Path

import numpy as np
import pytest

import camera_data as cd

G = np.load(Path(__file__).resolve().parent / "golden" / "cv2_undistort.npz")


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("name", list(cd.ALL))
def test_oracle_equals_golden(orc, name):
    model, cols, rows, K, D = cd.ALL[name]
    x, y = cd.test_points(cols, rows, seed=31, n=1000)
    got = np.stack(cd.undistort_keypoints(orc, model, K, D, x, y), 1)
    assert np.array_equal(_bits(got), _bits(G[name + "_oracle"]))
    assert np.array_equal(_bits(cd.image_bounds(orc, model, K, D, cols, rows)), _bits(G[name + "_bounds"]))
    if name in cd.CONFIGS:  # the first 1000 points lie inside the image
        assert np.array_equal(_bits(G[name + "_oracle"][:1000]), _bits(G[name + "_cv2"][:1000]))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(cd.ALL))
def test_gpu_equals_golden(ctx, plp, name):
    model, cols, rows, K, D = cd.ALL[name]
    x, y = cd.test_points(cols, rows, seed=31, n=1000)
    kp = np.zeros(len(x), plp.capi.KP_DTYPE)
    kp["x"], kp["y"] = x, y
    dist = plp.capi.make_distortion(model, *(list(D)[:4] if model == cd.FISHEYE else list(D)))
    cam = plp.capi.make_camera(*K, cols, rows)
    out, _ = ctx.undistort_keypoints(cam, dist, kp)
    assert np.array_equal(_bits(np.stack([out["x"], out["y"]], 1)), _bits(G[name + "_oracle"]))
    assert np.array_equal(_bits(plp.capi.image_bounds(cam, dist, cols, rows)), _bits(G[name + "_bounds"]))
