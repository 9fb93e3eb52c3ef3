"""The EPnP RANSAC's device code (csrc/pnp_kernels.cuh) run on the CPU through tests/cta_emu: poses, flags and counts
bit-equal to the oracle (oracle/pnp.cc), which compiles the same pnpmath.h text."""
from __future__ import annotations

import ctypes as C
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

import pnp_data as pd

ROOT = Path(__file__).resolve().parents[1]


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    so = tmp_path_factory.mktemp("emu") / "libpnp_emu.so"
    csrc = ROOT / "structure-plp-slam_b200" / "csrc"
    cmd = ["g++", "-O2", "-std=c++17", "-pthread", "-shared", "-fPIC", "-ffp-contract=off", "-fno-fast-math",
           f"-I{csrc}", f"-I{ROOT / 'tests' / 'cta_emu'}", str(ROOT / "tests" / "cta_emu" / "pnp_emu.cc"), "-o", str(so)]
    subprocess.run(cmd, check=True)
    return C.CDLL(str(so))


def emu_ransac(emu, off, b, x, mc, sm, min_num_inliers=10, recompute=True):
    P, N = len(off) - 1, int(off[-1])
    num_iter = sm.shape[1] if sm.ndim == 3 else 0
    valid, num = np.zeros(P, np.int32), np.zeros(P, np.int32)
    pose, flags = np.full((max(P, 1), 16), np.nan), np.full(max(N, 1), 255, np.uint8)
    p = pd._ptr
    keep = [np.ascontiguousarray(off, np.int32), np.ascontiguousarray(b, np.float64).reshape(-1),
            np.ascontiguousarray(x, np.float64).reshape(-1), np.ascontiguousarray(mc, np.float32),
            np.ascontiguousarray(sm, np.int32).reshape(-1) if sm.size else np.zeros(1, np.int32)]
    emu.emu_pnp_ransac(C.c_int(P), p(keep[0]), p(keep[1]), p(keep[2]), p(keep[3]), p(keep[4]), C.c_int(num_iter),
                       C.c_int(min_num_inliers), C.c_int(1 if recompute else 0), p(valid), p(num), p(pose), p(flags))
    return valid, num, pose[:P].reshape(P, 4, 4), flags[:N]


def assert_same(got, want):
    assert np.array_equal(got[0], want[0])
    assert np.array_equal(got[1], want[1])
    assert np.array_equal(got[2], want[2], equal_nan=True)   # bit-equal where written, untouched (NaN) elsewhere
    assert np.array_equal(got[3], want[3])


def problems(seed, P, sizes, num_iter=30, outlier_frac=0.5):
    scenes, samples = [], []
    for i in range(P):
        n = sizes[i % len(sizes)]
        scenes.append(pd.make_scene(seed * 100 + i, n, outlier_frac))
        samples.append(pd.draw_samples(seed * 100 + i, n, num_iter))
    return pd.pack(scenes, samples)


@pytest.mark.parametrize("P", [1, 7])
@pytest.mark.parametrize("n", [4, 10, 11, 300, 2000])
def test_emu_equals_oracle(emu, orc, P, n):
    off, b, x, mc, sm = problems(n + P, P, [n], outlier_frac=0.0 if n <= 11 else 0.5)
    # min_num_inliers 10 skips n = 4 and can never accept n = 10; 0 runs every size, small ones included
    for mni in ((10, 0) if n <= 11 else (10,)):
        for recompute in (True, False):
            want = pd.oracle_ransac(orc, off, b, x, mc, sm, min_num_inliers=mni, recompute=recompute)
            assert_same(emu_ransac(emu, off, b, x, mc, sm, min_num_inliers=mni, recompute=recompute), want)
        if n >= 300 or mni == 0:
            assert want[0].all()


def test_emu_edge_cases(emu, orc):
    # skipped (n < 4, n < min_num_inliers), invalid (outliers only) and valid problems in one call
    scenes = [pd.make_scene(1, 3), pd.make_scene(2, 8), pd.make_scene(3, 200, 0.5), pd.make_scene(4, 60, 1.0),
              pd.make_scene(5, 0), pd.make_scene(6, 40, planar=True), pd.make_scene(7, 50, 0.2)]
    scenes[6]["bearings"][[0, 5]] = [[0.6, 0.8, 0.0], [0.0, 1.0, 0.0]]            # z == 0: skipped by the solver
    scenes[6]["bearings"][10:20] *= -1                                            # negative z: the sign path
    samples = [pd.draw_samples(i, len(s["bearings"]), 30) for i, s in enumerate(scenes)]
    samples[6][:5] = [[0, 5, 3, 2]] * 5                                           # a sample with z == 0 bearings
    samples[2][3] = [7, 7, 7, 9]                                                  # duplicate indices
    samples[2][4] = [1, 1, 1, 1]
    samples[6][7] = [10, 11, 12, 13]                                              # all four with negative z
    off, b, x, mc, sm = pd.pack(scenes, samples)
    for recompute in (True, False):
        for mni in (10, 0, 150):
            want = pd.oracle_ransac(orc, off, b, x, mc, sm, min_num_inliers=mni, recompute=recompute)
            assert_same(emu_ransac(emu, off, b, x, mc, sm, min_num_inliers=mni, recompute=recompute), want)
    assert want[0][0] == 0 and want[1][0] == 0 and (want[3][:3] == 255).all()
    # num_iter = 0: every problem that runs is invalid with no inliers
    off, b, x, mc, _ = pd.pack(scenes[:3], samples[:3])
    z = np.zeros((3, 0, 4), np.int32)
    want = pd.oracle_ransac(orc, off, b, x, mc, z)
    assert_same(emu_ransac(emu, off, b, x, mc, z), want)
    assert not want[0].any() and not want[1].any()


def test_emu_first_best_wins_ties(emu, orc):
    s, sa, sb = pd.tie_scene(orc, 7)
    mixed = np.array([sa[0], sa[1], sb[0], sb[1]], np.int32)
    for order in ((sa, sb), (sb, sa), (mixed, sb, sa)):
        off, b, x, mc, sm = pd.pack([s], [np.stack(order)])
        for recompute in (True, False):
            want = pd.oracle_ransac(orc, off, b, x, mc, sm, recompute=recompute)
            assert_same(emu_ransac(emu, off, b, x, mc, sm, recompute=recompute), want)
