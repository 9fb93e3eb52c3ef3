"""Builds a CPU emulation of device code (tests/cta_emu/<name>.cc: a kernel header compiled by g++ against cta_emu.h).

Every emulator gets one flag set: -ffp-contract=off and -fno-fast-math keep g++ from contracting or reassociating the
kernel's floating-point expressions.  Only the optimisation level differs between emulators."""
from __future__ import annotations

import ctypes as C
import shutil
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
EMU_DIR = ROOT / "tests" / "cta_emu"
FLAGS = ["-std=c++17", "-pthread", "-shared", "-fPIC", "-ffp-contract=off", "-fno-fast-math",
         f"-I{ROOT / 'structure-plp-slam_b200' / 'csrc'}", f"-I{EMU_DIR}"]


def emu(name, tmp_path_factory, opt="-O2", extra=()):
    """Compiles tests/cta_emu/<name>.cc into a temporary directory and returns the loaded library; skips the test when
    g++ is absent."""
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    so = tmp_path_factory.mktemp("emu") / f"lib{name}.so"
    res = subprocess.run(["g++", opt, *FLAGS, *extra, str(EMU_DIR / f"{name}.cc"), "-o", str(so)],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[:3000]
    return C.CDLL(str(so))
