"""tools/check_bench_dump.py on a tiny dump written by bench.dump_outputs itself (from oracle results instead of a
GPU run): a faithful dump passes, and each kind of corruption is reported."""
import importlib.util
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
SEED, BATCH, STREAMS = 11, 4, 2


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


class _HostBuf:
    def __init__(self, a):
        self.a = a

    def download(self, dtype, shape):
        assert self.a.dtype == np.dtype(dtype)
        return self.a.reshape(shape).copy()


class _HostFrontEnd:
    """What bench.dump_outputs reads from a FrontEnd, backed by host arrays of per-frame results."""

    def __init__(self, frames, kp_dtype, cap=2064):
        B = len(frames)
        self.cap, self.max_batch = cap, B
        kp = np.zeros((B, cap), kp_dtype)
        desc = np.zeros((B, cap, 32), np.uint8)
        matched = np.full((B, cap), -1, np.int32)
        for b, r in enumerate(frames):
            n = len(r["kps"])
            kp[b, :n], desc[b, :n], matched[b, :n] = r["kps"], r["desc"], r["matched"]
        self.d_n = _HostBuf(np.array([len(r["kps"]) for r in frames], np.int32))
        self.d_kp, self.d_desc, self.d_matched = _HostBuf(kp), _HostBuf(desc), _HostBuf(matched)
        self._tracking = dict(pose=np.stack([r["pose"] for r in frames]),
                              **{k: np.array([r[k] for r in frames], np.int32) for k in ("num_valid", "n_inliers", "lm_iters")},
                              status=np.zeros(B, np.int32))

    def download_tracking(self, batch):
        return {k: v[:batch] for k, v in self._tracking.items()}


def _run(d):
    return subprocess.run([sys.executable, str(ROOT / "tools" / "check_bench_dump.py"), str(d), "--seed", str(SEED),
                           "--batch", str(BATCH), "--streams", str(STREAMS)], capture_output=True, text=True)


def test_check_bench_dump(tmp_path):
    tool = _load("check_bench_dump", ROOT / "tools" / "check_bench_dump.py")
    bench = _load("plp_bench", ROOT / "bench.py")
    frames = tool.oracle_outputs(SEED, BATCH, STREAMS)
    assert len(frames) == BATCH and min(r["num_valid"] for r in frames) >= 20 and min(r["lm_iters"] for r in frames) > 0
    bs = BATCH // STREAMS
    kp_dtype = bench._load_pkg().KP_DTYPE
    fes = [_HostFrontEnd(frames[c * bs:(c + 1) * bs], kp_dtype) for c in range(STREAMS)]
    good = tmp_path / "good"
    bench.dump_outputs(good, fes, bs, SEED)
    r = _run(good)
    assert r.returncode == 0 and "0 mismatches" in r.stdout, r.stdout + r.stderr

    def corrupted(name, edit, expect):
        d = tmp_path / name
        d.mkdir()
        for f in good.glob("*.npy"):
            a = np.load(f)
            np.save(d / f.name, edit(f.stem, a))
        r = _run(d)
        assert r.returncode == 1 and expect in r.stdout, r.stdout + r.stderr

    def bump(key, idx, delta):
        def edit(stem, a):
            if stem == key:
                a = a.copy()
                a[idx] += delta
            return a
        return edit

    corrupted("iters", bump("lm_iters", 1, -frames[1]["lm_iters"]), "frame 1: lm_iters")
    corrupted("iters_total", bump("lm_iters", slice(None), 12), "lm_iters: ")
    corrupted("desc", bump("descriptors", (5, 3), 1), "descriptors")
    corrupted("matched", bump("matched", 7, 1), "matched landmark indices")
    corrupted("pose", bump("pose", (2, 0, 3), 1e-2), "frame 2: pose")
    corrupted("kp", bump("kp_x", 0, 0.5), "keypoint field x")
