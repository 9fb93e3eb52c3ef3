"""The stereo rectification DEVICE code (structure-plp-slam_b200/csrc/rectify_kernels.cuh) executed on the CPU through
tests/cta_emu: the fixed-point map conversion, the tiles, the batch loop and the pitches, equal to the oracle byte for
byte, with the bytes past `cols` of every output row left as they were."""
import ctypes as C
import shutil

import numpy as np
import pytest

import rectify_data as rd

_P = C.c_void_p


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    return rd.build_emu(tmp_path_factory.mktemp("emu"))


def _run(emu, mx, my, frames, in_step, out_step):
    B, rows, cols = frames.shape
    src = np.random.default_rng(1).integers(0, 256, B * rows * in_step, dtype=np.uint8)
    src.reshape(B, rows, in_step)[:, :, :cols] = frames
    out = np.full(B * rows * out_step, 0xA5, np.uint8)
    emu.emu_rectify(np.ascontiguousarray(mx).ctypes.data_as(_P), np.ascontiguousarray(my).ctypes.data_as(_P),
                    C.c_int(rows), C.c_int(cols), C.c_int(B), src.ctypes.data_as(_P), C.c_size_t(in_step),
                    out.ctypes.data_as(_P), C.c_size_t(out_step))
    return out.reshape(B, rows, out_step)


@pytest.mark.parametrize("case,side,in_pad,out_pad", [("odd_tangential", 0, 0, 0), ("odd_tangential", 1, 16, 13),
                                                      ("euroc", 1, 16, 16), ("tumvi", 0, 0, 48)])
def test_rectify_kernel_on_cpu_equals_oracle(emu, case, side, in_pad, out_pad):
    """Batch 3: two rendered frames and one unrelated texture; an odd size whose tiles and last words are partial."""
    c = rd.CASES[case]
    rows, cols = c["rows"], c["cols"]
    mx, my = rd.oracle_maps(case, side)
    frames = np.stack([rd.texture(40 + side, rows, cols), rd.texture(41 + side, rows, cols),
                       np.random.default_rng(9).integers(0, 256, (rows, cols), dtype=np.uint8)])
    out = _run(emu, mx, my, frames, cols + in_pad, cols + out_pad)
    for b in range(3):
        assert np.array_equal(out[b, :, :cols], rd.oracle_remap(frames[b], mx, my)), f"frame {b}"
    assert (out[:, :, cols:] == 0xA5).all()


def test_rectify_kernel_on_cpu_random_maps(emu):
    """Random and extreme coordinates (beyond +-32767, the last row and column, (-1, 0)) through the kernel's fixed point."""
    mx, my = rd.random_maps(7, 97, 131, 97, 131)
    frames = np.stack([rd.texture(50, 97, 131), rd.texture(51, 97, 131)])
    out = _run(emu, mx, my, frames, 131 + 5, 136)
    for b in range(2):
        assert np.array_equal(out[b, :, :131], rd.oracle_remap(frames[b], mx, my)), f"frame {b}"
    assert (out[:, :, 131:] == 0xA5).all()


def test_rectify_kernel_on_cpu_batch_chunks(emu):
    """A batch larger than one CTA's chunk of frames: three chunks, the last one partial."""
    mx, my = rd.oracle_maps("odd_tangential", 1)
    frames = np.stack([rd.texture(60 + b, 97, 131) for b in range(37)])
    out = _run(emu, mx, my, frames, 131 + 3, 144)
    for b in range(37):
        assert np.array_equal(out[b, :, :131], rd.oracle_remap(frames[b], mx, my)), f"frame {b}"
    assert (out[:, :, 131:] == 0xA5).all()
