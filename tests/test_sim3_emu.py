"""The Sim3 RANSAC's device code (csrc/sim3_kernels.cuh) run on the CPU through tests/cta_emu: validity, counts and the
winning Sim3 bit-equal to the oracle (oracle/sim3.cc), which compiles the same sim3math.h text."""
from __future__ import annotations

import ctypes as C
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

import sim3_data as sd

ROOT = Path(__file__).resolve().parents[1]


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    so = tmp_path_factory.mktemp("emu") / "libsim3_emu.so"
    csrc = ROOT / "structure-plp-slam_b200" / "csrc"
    cmd = ["g++", "-O2", "-std=c++17", "-pthread", "-shared", "-fPIC", "-ffp-contract=off", "-fno-fast-math",
           f"-I{csrc}", f"-I{ROOT / 'tests' / 'cta_emu'}", str(ROOT / "tests" / "cta_emu" / "sim3_emu.cc"), "-o", str(so)]
    subprocess.run(cmd, check=True)
    return C.CDLL(str(so))


def emu_ransac(emu, off, x1, x2, c1, c2, sm, fix_scale=False, min_num_inliers=20):
    P, N = len(off) - 1, int(off[-1])
    num_iter = sm.shape[1] if sm.ndim == 3 else 0
    valid, num = np.full(max(P, 1), 7, np.int32), np.full(max(P, 1), 7, np.int32)
    rot, trans, scale = np.full((max(P, 1), 9), np.nan), np.full((max(P, 1), 3), np.nan), np.full(max(P, 1), np.nan, np.float32)
    p = sd._ptr
    keep = [np.ascontiguousarray(off, np.int32), np.ascontiguousarray(np.tile(sd.CAM, (max(P, 1), 1)), np.float64),
            np.ascontiguousarray(x1, np.float64).reshape(-1) if N else np.zeros(3),
            np.ascontiguousarray(x2, np.float64).reshape(-1) if N else np.zeros(3),
            np.ascontiguousarray(c1, np.float32) if N else np.zeros(1, np.float32),
            np.ascontiguousarray(c2, np.float32) if N else np.zeros(1, np.float32),
            np.ascontiguousarray(sm, np.int32).reshape(-1) if sm.size else np.zeros(1, np.int32)]
    emu.emu_sim3_ransac(C.c_int(P), *[p(a) for a in keep], C.c_int(num_iter), C.c_int(1 if fix_scale else 0),
                        C.c_int(min_num_inliers), p(valid), p(num), p(rot), p(trans), p(scale))
    return valid[:P], num[:P], rot[:P].reshape(P, 3, 3), trans[:P], scale[:P]


def check(emu, orc, off, x1, x2, c1, c2, sm, **kw):
    want = sd.oracle_ransac(orc, off, x1, x2, c1, c2, sm, **kw)
    sd.assert_same(emu_ransac(emu, off, x1, x2, c1, c2, sm, **kw), want)
    return want


@pytest.mark.parametrize("P", [1, 7])
@pytest.mark.parametrize("n", [3, 4, 20, 300, 2000])
def test_emu_equals_oracle(emu, orc, P, n):
    iters = (0, 1, 200) if n <= 300 else (1, 30)
    for num_iter in iters:
        for fix_scale in (False, True):
            off, x1, x2, c1, c2, sm = sd.problems(n + P, P, [n], num_iter=num_iter, outlier_frac=0.0 if n <= 4 else 0.5,
                                                  fix_scale=fix_scale)
            for mni in ((20, 3, 0) if n <= 20 else (20,)):
                want = check(emu, orc, off, x1, x2, c1, c2, sm, fix_scale=fix_scale, min_num_inliers=mni)
                if n >= 300 and num_iter == 200:
                    assert want[0].all()


def test_emu_edge_cases(emu, orc):
    # skipped (n = 2, n < min_num_inliers, n = 0), invalid (outliers only), valid, points behind either camera
    scenes = [sd.make_scene(1, 2), sd.make_scene(2, 15), sd.make_scene(3, 200, 0.5), sd.make_scene(4, 60, 1.0),
              sd.make_scene(5, 0), sd.make_scene(6, 80, 0.3, behind_1=5, behind_2=4),
              sd.make_scene(7, 50, 0.2, fix_scale=True)]
    samples = [sd.draw_samples(i, len(s["pts_1"]), 40) for i, s in enumerate(scenes)]
    samples[2][3] = [7, 7, 9]                     # duplicate indices
    samples[2][4] = [1, 1, 1]
    samples[5][0] = [0, 1, 2]                     # all three behind keyframe 1
    samples[5][1] = [79, 78, 77]                  # all three behind keyframe 2
    tie, sa, sb = sd.concat(sd.make_scene(41, 20, noise_px=0.0, scale=2.0),
                            sd.make_scene(42, 20, noise_px=0.0, scale=0.5)), [0, 1, 2], [20, 21, 22]
    scenes.append(tie)
    samples.append(np.array([sa, sb] * 20, np.int32))
    off, x1, x2, c1, c2, sm = sd.pack(scenes, samples)
    for fix_scale in (False, True):
        for mni in (20, 0, 3, 150):
            want = check(emu, orc, off, x1, x2, c1, c2, sm, fix_scale=fix_scale, min_num_inliers=mni)
    want = sd.oracle_ransac(orc, off, x1, x2, c1, c2, sm)
    assert list(want[0]) == [0, 0, 1, 0, 0, 1, 1, 1]
    # num_iter = 0: every problem that runs is invalid with no inliers (valid only when min_num_inliers is 0)
    z = np.zeros((len(scenes), 0, 3), np.int32)
    for mni in (20, 0):
        want = check(emu, orc, off, x1, x2, c1, c2, z, min_num_inliers=mni)
    assert list(want[0]) == [0, 1, 1, 1, 0, 1, 1, 1] and not want[1].any() and not want[4].any()
