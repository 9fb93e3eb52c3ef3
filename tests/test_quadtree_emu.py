"""The ORB quadtree DEVICE code (structure-plp-slam_b200/csrc/quadtree_kernels.cuh) executed on the CPU through tests/cta_emu
(see test_cta_emu.py): both kernel instances select the same keypoints, in the same order, as the oracle's
distribute_keypoints_via_tree -- on random candidates (duplicated coordinates, budgets 5 to 1000), on the real FAST
candidates of every pyramid level, and on a level larger than the shared-memory window (the global-scratch path)."""
import ctypes as C
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

import oracle_api
import synth

ROOT = Path(__file__).resolve().parent.parent
_P = C.c_void_p
LEVEL_KP = np.dtype([("x", "<i2"), ("y", "<i2"), ("response", "<i4")])
PATCH = 19


@pytest.fixture(scope="module")
def qt_emu(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    so = tmp_path_factory.mktemp("emu") / "libquadtree_emu.so"
    cmd = ["g++", "-O1", "-std=c++17", "-pthread", "-shared", "-fPIC", "-ffp-contract=off",
           f"-I{ROOT / 'structure-plp-slam_b200' / 'csrc'}", f"-I{ROOT / 'tests' / 'cta_emu'}",
           str(ROOT / "tests" / "cta_emu" / "quadtree_emu.cc"), "-o", str(so)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[:3000]
    return C.CDLL(str(so))


def _slot_cap(w, h, budget):  # orb.cu: initial nodes of the level, one sweep can quadruple them
    ratio = (w - 2 * PATCH) / (h - 2 * PATCH)
    g0 = int(round(ratio)) if ratio > 1 else int(round(1 / ratio))
    return 4 * max(budget, g0) + 8


def _run(qt_emu, instance, xs, ys, resp, w, h, budget, cell_size=1024):
    """Kernel on candidates relative to the patch border (x:11 | y:10 | score:11); level size w x h."""
    cand = (xs.astype(np.uint32) | (ys.astype(np.uint32) << 11) | (resp.astype(np.uint32) << 21)).astype(np.uint32)
    cap = _slot_cap(w, h, budget)
    out = np.zeros(cap, LEVEL_KP)
    status = C.c_int(-1)
    n = qt_emu.emu_quadtree(C.c_int(instance), cand.ctypes.data_as(_P), C.c_int(len(cand)), C.c_int(w), C.c_int(h),
                            C.c_int(budget), C.c_int(cell_size), out.ctypes.data_as(_P), C.c_int(cap), C.byref(status))
    return out[:n], status.value


def _check(qt_emu, orc, instances, xs, ys, resp, w, h, budget, cell_size=1024):
    p = oracle_api.orb_params()
    cands = np.zeros(len(xs), oracle_api.KP_DTYPE)
    cands["x"], cands["y"], cands["response"] = xs, ys, resp
    ref = orc.orb_distribute(p, cands, PATCH, w - PATCH, PATCH, h - PATCH, budget)
    for inst in instances:
        got, status = _run(qt_emu, inst, xs, ys, resp, w, h, budget, cell_size)
        assert status == 0, (inst, status)
        assert len(got) == len(ref), (inst, len(got), len(ref))
        assert np.array_equal(got["x"] - PATCH, ref["x"]) and np.array_equal(got["y"] - PATCH, ref["y"]), inst
        assert np.array_equal(got["response"], ref["response"]), inst


def _instances(w, h, budget):
    cap = _slot_cap(w, h, budget)
    return [i for i, nc in ((0, 1024), (1, 2048)) if cap <= nc] or [2]


@pytest.mark.parametrize("seed", range(25))
def test_random_candidates(qt_emu, orc, seed):
    # the cases of test_quadtree_model.py
    rng = np.random.default_rng(seed)
    w, h = [(602, 442), (714, 442), (141, 96), (300, 700), (495, 362)][seed % 5]
    n = int(rng.integers(1, 3000))
    budget = int(rng.choice([5, 60, 217, 1000]))
    xs = rng.integers(0, w, n).astype(np.float32)
    ys = rng.integers(0, h, n).astype(np.float32)
    if seed % 4 == 0:  # heavy duplication -> many equal-count leaves, exercises the tie-break
        xs = (xs // 16 * 16).astype(np.float32)
        ys = (ys // 16 * 16).astype(np.float32)
    resp = rng.integers(7, 255, n).astype(np.float32)
    W, H = w + 2 * PATCH, h + 2 * PATCH
    # cells of uneven fill, empty ones included, exercise the gather's search over the cell prefix
    _check(qt_emu, orc, _instances(W, H, budget), xs, ys, resp, W, H, budget, cell_size=int(rng.integers(1, 1025)))


def test_real_fast_candidates(qt_emu, orc):
    img = synth.make_texture(99)
    p = oracle_api.orb_params()
    r = orc.orb_extract(p, img, debug=True)
    w, h = orc.orb_level_sizes(p, *img.shape)
    t = orc.orb_tables(p)
    off = 0
    for l in range(8):
        c = r["cands"][off: off + r["cands_per_level"][l]]
        off += r["cands_per_level"][l]
        W, H, budget = int(w[l]), int(h[l]), int(t["num_keypts_per_level"][l])
        _check(qt_emu, orc, [0, 1], c["x"].copy(), c["y"].copy(), c["response"].copy(), W, H, budget, cell_size=700)


def test_level_beyond_shared_memory_window(qt_emu, orc):
    # more candidates than either instance's shared-memory window: the work arrays live in the global scratch block
    n = qt_emu.emu_quadtree_cand_cap(1) + 1500
    assert n > qt_emu.emu_quadtree_cand_cap(0)
    rng = np.random.default_rng(5)
    W, H, budget = 1280, 960, 217
    xs = rng.integers(0, W - 2 * PATCH, n).astype(np.float32)
    ys = rng.integers(0, H - 2 * PATCH, n).astype(np.float32)
    resp = rng.integers(7, 255, n).astype(np.float32)
    _check(qt_emu, orc, [0, 1], xs, ys, resp, W, H, budget)
