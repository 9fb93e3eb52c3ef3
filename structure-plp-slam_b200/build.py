"""Build libplpslam_b200.so in-tree with nvcc for sm_90a (H100) (no torch, no cmake).

Each .cu is compiled to an object with its own flags (parity-critical integer / fixed-point /
f32 files use -fmad=false so they round exactly like the oracle) and linked into one shared
library that only depends on libcudart (static) -- plus libnccl for the multi-GPU BA object.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

HERE = Path(__file__).resolve().parent
CSRC = HERE / "csrc"
OBJ = HERE / "build"
LIB = HERE / "libplpslam_b200.so"

NVCC = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC,-fvisibility=hidden", "--expt-relaxed-constexpr",
          "-Xptxas", "-v"]

# per-file extra flags
NO_FMA = ["-fmad=false"]
FILE_FLAGS = {
    "match.cu": NO_FMA,
    "orb.cu": NO_FMA,
    "lines.cu": NO_FMA,
    "stereo.cu": NO_FMA,
    "fuse.cu": NO_FMA,
    "bow.cu": NO_FMA,
    "essential.cu": NO_FMA,
    "plane.cu": NO_FMA,
    "camera.cu": NO_FMA,
    "local_map.cu": NO_FMA,
    "keyframe_track.cu": NO_FMA,
    "robust_track.cu": NO_FMA,
    "bow_db.cu": NO_FMA,
    "pnp.cu": NO_FMA,
    "sim3.cu": NO_FMA,
    "sim3_opt.cu": NO_FMA,
}


def _sources():
    return sorted(p for p in CSRC.glob("*.cu"))


def _stamp(src: Path, flags) -> str:
    h = hashlib.sha1()
    h.update(" ".join(flags).encode())
    h.update(src.read_bytes())
    for hdr in sorted(list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.inc")) + list(CSRC.glob("*.h")) + list((HERE.parent / "include").glob("*.h"))):
        h.update(hdr.read_bytes())
    return h.hexdigest()


def _compile(src: Path, verbose: bool) -> Path:
    flags = ARCH + COMMON + FILE_FLAGS.get(src.name, []) + os.environ.get("PLP_EXTRA_NVCC_FLAGS", "").split()
    obj = OBJ / (src.stem + ".o")
    stamp_file = OBJ / (src.stem + ".stamp")
    stamp = _stamp(src, flags)
    if obj.exists() and stamp_file.exists() and stamp_file.read_text() == stamp:
        return obj
    cmd = [NVCC] + flags + ["-c", str(src), "-o", str(obj)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    (OBJ / (src.stem + ".ptxas.log")).write_text(res.stderr)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError(f"nvcc failed on {src.name}")
    if verbose:
        sys.stderr.write(f"[build] {src.name} ok\n")
    stamp_file.write_text(stamp)
    return obj


def build(verbose: bool = False, force: bool = False) -> Path:
    OBJ.mkdir(exist_ok=True)
    if force:
        for f in OBJ.glob("*.stamp"):
            f.unlink()
    srcs = _sources()
    if not srcs:
        raise RuntimeError("no CUDA sources found")
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(lambda s: _compile(s, verbose), srcs))
    newest = max(o.stat().st_mtime for o in objs)
    if LIB.exists() and LIB.stat().st_mtime >= newest and not force:
        return LIB
    link = [NVCC] + ARCH + ["-shared", "-o", str(LIB)] + [str(o) for o in objs] + ["-cudart", "static"]
    if (CSRC / "ba_nccl.cu").exists():
        link += ["-lnccl"]
    res = subprocess.run(link, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError("link failed")
    if verbose:
        sys.stderr.write(f"[build] linked {LIB}\n")
    return LIB


if __name__ == "__main__":
    build(verbose=True, force="--force" in sys.argv)
