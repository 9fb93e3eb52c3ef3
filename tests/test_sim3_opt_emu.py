"""The Sim3 optimiser's device code (csrc/sim3_opt_kernels.cuh) run on the CPU through tests/cta_emu over every scene of
sim3_opt_data, batched: counts and inlier flags equal to the oracle (oracle/transform_opt.cc), the Sim3 within 1e-8
relative.  Both compile sim3optmath.h and glibc's sin / cos / exp and reduce in the same fixed order, so here the results
are in fact bit-identical, and the test says so too."""
from __future__ import annotations

import numpy as np
import pytest

import emu_build
import sim3_opt_data as sd


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return emu_build.emu("sim3opt_emu", tmp_path_factory)


def check(emu, orc, d, **kw):
    want = sd.oracle_optimize(orc, d, **kw)
    got = sd.call(emu.emu_sim3_optimize, d, **kw)
    sd.assert_close(got, want, rtol=1e-8)
    for g, w in zip(got, want):
        assert g.tobytes() == w.tobytes()
    return want


@pytest.mark.parametrize("fix_scale", [False, True])
def test_emu_equals_oracle_on_every_scene_batched(emu, orc, fix_scale):
    scs = sd.scenes(0)
    # the stereo case keeps s = 1; the monocular scenes run with the scale fixed too, as a stereo map would
    d = sd.pack([sc for _, sc, _ in scs])
    want = check(emu, orc, d, fix_scale=fix_scale)
    names = [n for n, _, _ in scs]
    # with the scale fixed, only the stereo scene (true scale 1) keeps most of its matches
    for name in (("stereo",) if fix_scale else ("mono", "stereo", "outliers40", "large")):
        assert want[0][names.index(name)] >= 100, name
    for name in ("few_survivors", "tiny", "empty"):
        assert want[0][names.index(name)] == 0, name


def test_emu_iteration_counts_and_thresholds(emu, orc):
    scs = [sd.make_scene(7, 300, 0.3), sd.make_scene(8, 130, 0.1), sd.make_scene(9, 0)]
    d = sd.pack(scs)
    for num_iter, chi_sq in ((0, 10.0), (1, 10.0), (25, 10.0), (10, 5.99), (10, 100.0)):
        check(emu, orc, d, num_iter=num_iter, chi_sq=np.float32(chi_sq))
