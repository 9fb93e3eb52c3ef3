"""The rectification oracle (tests/rectify_oracle.cc: the maps from structure-plp-slam_b200/csrc/rectmath.h and an
independent fixed-point remap) pinned to cv2 bit for bit, and to tests/golden/cv2_rectify.npz without cv2."""
import hashlib
from pathlib import Path

import numpy as np
import pytest

import rectify_data as rd

GOLDEN = Path(__file__).resolve().parent / "golden" / "cv2_rectify.npz"
CASE_SIDES = [(c, s) for c in rd.CASES for s in (0, 1)]


@pytest.mark.parametrize("case,side", CASE_SIDES)
def test_maps_equal_cv2(case, side):
    pytest.importorskip("cv2")
    mx, my = rd.oracle_maps(case, side)
    cx, cy = rd.cv2_maps(case, side)
    assert np.array_equal(mx.view(np.uint32), cx.view(np.uint32))
    assert np.array_equal(my.view(np.uint32), cy.view(np.uint32))


@pytest.mark.parametrize("case", list(rd.CASES))
def test_remap_equals_cv2_on_rectifier_maps(case):
    cv2 = pytest.importorskip("cv2")
    c = rd.CASES[case]
    img = rd.texture(3, c["rows"], c["cols"])
    for side in (0, 1):
        mx, my = rd.cv2_maps(case, side)
        assert np.array_equal(rd.oracle_remap(img, mx, my), cv2.remap(img, mx, my, cv2.INTER_LINEAR))


@pytest.mark.parametrize("seed,src_shape,map_shape", [(1, (97, 131), (200, 300)), (2, (480, 752), (64, 900)),
                                                      (3, (5, 7), (40, 40))])
def test_remap_equals_cv2_on_random_and_extreme_maps(seed, src_shape, map_shape):
    """Random coordinates over [-3, size + 3], exact integers (the last row and column included), (-1, 0), values half a
    step from a tap, and coordinates far beyond +-32767."""
    cv2 = pytest.importorskip("cv2")
    img = rd.texture(seed + 10, *src_shape)
    mx, my = rd.random_maps(seed, *map_shape, *src_shape)
    assert np.array_equal(rd.oracle_remap(img, mx, my), cv2.remap(img, mx, my, cv2.INTER_LINEAR))


def test_remap_reads_row_stride_and_writes_only_map_width():
    img = rd.texture(4, 97, 131)
    padded = np.full((97, 131 + 9), 255, np.uint8)
    padded[:, :131] = img
    mx, my = rd.random_maps(4, 50, 70, 97, 131)
    out = np.full((50, 70 + 6), 7, np.uint8)
    rd.oracle_remap(padded[:, :131], mx, my, out[:, :70])
    assert np.array_equal(out[:, :70], rd.oracle_remap(img, mx, my)) and (out[:, 70:] == 7).all()


def test_oracle_equals_golden():
    """Without cv2: the oracle's maps at the stored pixels and their full-map digests, and the remapped images."""
    g = np.load(GOLDEN)
    for case, c in rd.CASES.items():
        idx = g[case + "_idx"]
        for side in (0, 1):
            mx, my = rd.oracle_maps(case, side)
            key = f"{case}_{side}"
            assert np.array_equal(mx.ravel()[idx].view(np.uint32), g[key + "_x"].view(np.uint32)), key
            assert np.array_equal(my.ravel()[idx].view(np.uint32), g[key + "_y"].view(np.uint32)), key
            assert hashlib.sha256(mx.tobytes() + my.tobytes()).hexdigest() == str(g[key + "_sha256"]), key
            if side == 0 and case in rd.REFERENCE_CASES:
                img = rd.texture(23, c["rows"], c["cols"])
                assert np.array_equal(rd.oracle_remap(img, mx, my), g[case + "_remap"]), case
    mx, my = rd.random_maps(1, 200, 300, 97, 131)
    assert np.array_equal(rd.oracle_remap(rd.texture(5, 97, 131), mx, my), g["random_remap"])


def test_invalid_parameters_rejected():
    c = rd.CASES["euroc"]
    K, D, R = rd.side_params("euroc", 0)
    assert rd.oracle_maps_raw(c["model"], K, D, R, c["rect"], 480, 752)[0] == 0
    assert rd.oracle_maps_raw(2, K, D, R, c["rect"], 480, 752)[0] == -1
    assert rd.oracle_maps_raw(c["model"], K, D, np.zeros((3, 3)), c["rect"], 480, 752)[0] == -1
    assert rd.oracle_maps_raw(c["model"], K, D, R, (0.0, 400.0, 300.0, 200.0), 480, 752)[0] == -1
    for rows, cols in ((0, 752), (480, 0), (-1, 5)):
        assert rd.oracle_maps_raw(c["model"], K, D, R, c["rect"], rows, cols)[0] == -1
