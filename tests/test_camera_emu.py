"""The keypoint-undistortion DEVICE code (structure-plp-slam_b200/csrc/camera_kernels.cuh) executed on the CPU through
tests/cta_emu (see test_cta_emu.py): batch x capacity slots, per-frame counts (one frame empty), untouched slots past a
frame's count, and the undistorted keypoints and bearings equal to the oracle bit for bit."""
import ctypes as C

import numpy as np
import pytest

import camera_data as cd
import emu_build

_P = C.c_void_p
KP_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"),
                     ("octave", "<i4"), ("class_id", "<i4")])


@pytest.fixture(scope="module")
def cam_emu(tmp_path_factory):
    return emu_build.emu("camera_emu", tmp_path_factory, opt="-O1")


@pytest.mark.parametrize("name", list(cd.ALL))
def test_undistort_kernel_on_cpu_equals_oracle(cam_emu, orc, name):
    model, cols, rows, K, D = cd.ALL[name]
    batch, cap = 3, 700
    n = np.array([700, 0, 313], np.int32)
    rng = np.random.default_rng(8)
    kp = np.zeros((batch, cap), KP_DTYPE)
    kp["x"] = rng.uniform(-20, cols + 20, (batch, cap))
    kp["y"] = rng.uniform(-20, rows + 20, (batch, cap))
    kp["angle"] = rng.uniform(0, 360, (batch, cap))
    kp["size"] = 31.0
    kp["octave"] = rng.integers(0, 8, (batch, cap))
    out = np.zeros((batch, cap), KP_DTYPE)
    out["x"] = 12345.0
    bear = np.full((batch, cap, 3), 7.0)
    Kd, Dd = np.ascontiguousarray(K, np.float64), np.ascontiguousarray(cd.coeffs5(D))
    cam_emu.emu_undistort_batch(C.c_int(model), Kd.ctypes.data_as(_P), Dd.ctypes.data_as(_P), C.c_int(batch), C.c_int(cap),
                                kp.ctypes.data_as(_P), n.ctypes.data_as(_P), out.ctypes.data_as(_P), bear.ctypes.data_as(_P))
    for b in range(batch):
        wx, wy = cd.undistort_keypoints(orc, model, K, D, kp["x"][b, :n[b]], kp["y"][b, :n[b]])
        o = out[b, :n[b]]
        assert np.array_equal(o["x"].view(np.uint32), wx.view(np.uint32)) and np.array_equal(o["y"].view(np.uint32),
                                                                                               wy.view(np.uint32))
        assert np.array_equal(o["angle"], kp["angle"][b, :n[b]]) and np.array_equal(o["octave"], kp["octave"][b, :n[b]])
        assert (o["class_id"] == -1).all() and (o["size"] == 31.0).all()
        assert np.array_equal(bear[b, :n[b]].view(np.uint64), cd.bearings(orc, K, wx, wy).view(np.uint64))
        assert (out["x"][b, n[b]:] == 12345.0).all() and (bear[b, n[b]:] == 7.0).all()
