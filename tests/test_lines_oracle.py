"""CPU: pins the line front-end oracle (oracle/lines.cc).

* LSD: the restatement of cv::LineSegmentDetector is compared bit-for-bit with cv2 4.13
  `createLineSegmentDetector(1, 0.5, 0.6, 2.0, 22.5, 1.0, 0.6, 1024)` (the options of line_extractor.cc:113-122), in the
  "det" mode the CUDA path implements and in the "cv" mode (libm, sequential sums).
* the OpenCV primitives LBD uses (GaussianBlur 5x5 sigma 1, Sobel 3x3 -> CV_16S, LineIterator count) against cv2;
* LBD itself is vendored reference source (binary_descriptor_custom.cpp) restated line by line: structural checks.
* detmath (deterministic sin/cos/atan2) against libm.
"""
import functools
import math
from pathlib import Path

import numpy as np
import pytest

import oracle_api
import synth

cv2 = pytest.importorskip("cv2")
ROOT = Path(__file__).resolve().parent.parent


# camera geometries the reference ships (KITTI 00-02 1241 x 376, KITTI 03 1242 x 375, KITTI 04-12 1226 x 370, TUM-VI
# 512 x 512) and sizes that, with the rest, cover every residue mod 4 of rows and of cols: a dimension = 3 (mod 4) gives the
# half-resolution image a last row / column with a single source row / column
GEOMETRIES = [(375, 1242), (370, 1226), (376, 1241), (512, 512), (479, 639), (481, 641), (478, 637), (33, 47), (47, 33),
              (16, 16)] + [(64 + r, 96 + c) for r in range(4) for c in range(4)]


def _images():
    out = [("texture640", synth.make_texture(1)), ("texture752", synth.make_texture(2, h=480, w=752)),
           ("lines640", synth.make_line_image(1)), ("lines752", synth.make_line_image(2, 480, 752)),
           ("noise", np.random.default_rng(5).integers(0, 256, (480, 640), dtype=np.uint8)),
           ("flat", np.full((480, 640), 77, np.uint8))]
    # natural images: 180 x 240 centre crops of the reference's two test photographs (tools/gen_reference_fixtures.py),
    # not the whole 640 x 480 resized photographs -- less natural-image area per case, kept small to keep the fixture small
    crops = np.load(ROOT / "tests" / "golden" / "equirect_crops.npz")
    out += [(f, crops[f]) for f in sorted(crops.files)]
    return out


GEOMETRY_NAMES = [f"{'texture' if i % 2 == 0 else 'lines'}{h}x{w}" for i, (h, w) in enumerate(GEOMETRIES)]


@functools.lru_cache(maxsize=1)
def _geometry_images():
    """One seeded image per GEOMETRIES entry, textures and line images alternating."""
    return {n: synth.make_texture(40 + i, h, w) if i % 2 == 0 else synth.make_line_image(40 + i, h, w)
            for i, (n, (h, w)) in enumerate(zip(GEOMETRY_NAMES, GEOMETRIES))}


def _cv_lsd(img):
    lsd = cv2.createLineSegmentDetector(1, 0.5, 0.6, 2.0, 22.5, 1.0, 0.6, 1024)
    r = lsd.detect(img)[0]
    return np.zeros((0, 4), np.float32) if r is None else r.reshape(-1, 4)


def half_area(g):
    """resize(g, None, 0.5, 0.5, INTER_LINEAR_EXACT) as oracle/lines.cc states it: the mean of each 2x2 block's existing
    pixels -- 4 pixels (s + 2) >> 2, 2 pixels (last row or column of a dimension = 3 mod 4) s / 2 ties to even, 1 pixel
    (that corner) the pixel."""
    h, w = g.shape
    sh, sw = int(np.rint(h * 0.5)), int(np.rint(w * 0.5))
    gi = np.zeros((2 * sh, 2 * sw), np.int64)
    n = np.zeros_like(gi)
    hh, ww = min(h, 2 * sh), min(w, 2 * sw)
    gi[:hh, :ww] = g[:hh, :ww]
    n[:hh, :ww] = 1
    s = gi.reshape(sh, 2, sw, 2).sum((1, 3))
    c = n.reshape(sh, 2, sw, 2).sum((1, 3))
    return np.where(c == 4, (s + 2) >> 2, np.where(c == 2, (s + ((s >> 1) & 1)) >> 1, s)).astype(np.uint8)


def test_half_resize_border_rule_is_cv2s():
    """The border rule of half_area derived from cv2 itself: every value pair in a 2-pixel last column and last row, every
    value of the 1-pixel corner, impulses (each source pixel feeds only its own block, or nothing) and seeded images at
    every residue mod 4."""
    def cvr(img):
        return cv2.resize(img, None, fx=0.5, fy=0.5, interpolation=cv2.INTER_LINEAR_EXACT)
    a, b = np.meshgrid(np.arange(256), np.arange(256), indexing="ij")
    col = np.zeros((2 * 256 * 256, 7), np.uint8)            # 7 cols -> 4, last column from col 6 only
    col[0::2, 6], col[1::2, 6] = a.ravel(), b.ravel()
    assert np.array_equal(cvr(col)[:, 3].astype(np.int64), ((a + b) + (((a + b) >> 1) & 1)).ravel() >> 1)
    row = np.zeros((7, 2 * 256 * 256), np.uint8)
    row[6, 0::2], row[6, 1::2] = a.ravel(), b.ravel()
    assert np.array_equal(cvr(row)[3].astype(np.int64), ((a + b) + (((a + b) >> 1) & 1)).ravel() >> 1)
    corner = np.zeros((256, 7, 7), np.uint8)                # 7 x 7 -> 4 x 4, corner from pixel (6, 6) only
    corner[:, 6, 6] = np.arange(256)
    assert [int(cvr(c)[3, 3]) for c in corner] == list(range(256))
    for h, w in ((7, 7), (11, 15), (9, 13)):
        for y in range(h):
            for x in range(w):
                img = np.zeros((h, w), np.uint8)
                img[y, x] = 201
                r = cvr(img)
                # a dimension = 1 (mod 4) drops its last source row / column
                inside = y // 2 < r.shape[0] and x // 2 < r.shape[1]
                assert np.array_equal(np.argwhere(r), [[y // 2, x // 2]] if inside else np.zeros((0, 2)))
    rng = np.random.default_rng(0)
    for h in range(16, 24):
        for w in range(16, 24):
            g = rng.integers(0, 256, (h, w), dtype=np.uint8)
            assert np.array_equal(cvr(g), half_area(g)), (h, w)


def _cv_scaled(img):
    g = cv2.GaussianBlur(img, (11, 11), 1.2)
    return cv2.resize(g, None, fx=0.5, fy=0.5, interpolation=cv2.INTER_LINEAR_EXACT)


def _cv_lbd_gradients(img):
    g = cv2.GaussianBlur(img, (5, 5), 1)
    return cv2.Sobel(g, cv2.CV_16S, 1, 0, ksize=3), cv2.Sobel(g, cv2.CV_16S, 0, 1, ksize=3)


def test_scaled_image_matches_cv2(orc):
    for name, img in _images():
        assert np.array_equal(orc.lsd_scaled(img), _cv_scaled(img)), name


@pytest.mark.parametrize("mode", [oracle_api.LSD_DET, oracle_api.LSD_CV])
def test_lsd_segments_bit_exact_vs_cv2(orc, mode):
    total = 0
    for name, img in _images():
        ref = _cv_lsd(img)
        got = orc.lsd_detect(img, mode)
        assert got.shape == ref.shape, f"{name}: {len(got)} vs {len(ref)} segments"
        assert np.array_equal(got, ref), name
        total += len(ref)
    assert total > 2000


def test_lbd_gradients_match_cv2(orc):
    for name, img in _images()[:5]:
        dx, dy = _cv_lbd_gradients(img)
        ox, oy = orc.lbd_gradients(img)
        assert np.array_equal(ox, dx) and np.array_equal(oy, dy), name


# the same three comparisons at the camera geometries and at every residue mod 4, one case per size
@pytest.mark.parametrize("name", GEOMETRY_NAMES)
def test_scaled_image_matches_cv2_at_size(orc, name):
    img = _geometry_images()[name]
    assert np.array_equal(orc.lsd_scaled(img), _cv_scaled(img)), name


@pytest.mark.parametrize("mode", [oracle_api.LSD_DET, oracle_api.LSD_CV])
@pytest.mark.parametrize("name", GEOMETRY_NAMES)
def test_lsd_segments_bit_exact_vs_cv2_at_size(orc, mode, name):
    img = _geometry_images()[name]
    ref = _cv_lsd(img)
    got = orc.lsd_detect(img, mode)
    assert got.shape == ref.shape, f"{name}: {len(got)} vs {len(ref)} segments"
    assert np.array_equal(got, ref), name
    if min(img.shape) >= 64:
        assert len(ref) > 0


@pytest.mark.parametrize("name", GEOMETRY_NAMES)
def test_lbd_gradients_match_cv2_at_size(orc, name):
    img = _geometry_images()[name]
    dx, dy = _cv_lbd_gradients(img)
    ox, oy = orc.lbd_gradients(img)
    assert np.array_equal(ox, dx) and np.array_equal(oy, dy), name


def test_keyline_fields_and_line_iterator_count(orc):
    img = synth.make_line_image(3)
    kls = orc.lsd_keylines(img, 60.0)
    assert len(kls) > 50
    assert np.array_equal(kls["class_id"], np.arange(len(kls)))
    assert (kls["octave"] == 0).all() and (kls["line_length"] > 60).all()
    for k in kls[:40]:
        # cv::LineIterator count == number of pixels cv2.line sets (8-connected, thickness 1)
        canvas = np.zeros(img.shape, np.uint8)
        p0 = (int(np.rint(k["start_x"])), int(np.rint(k["start_y"])))
        p1 = (int(np.rint(k["end_x"])), int(np.rint(k["end_y"])))
        cv2.line(canvas, p0, p1, 255, 1, cv2.LINE_8)
        assert int(np.count_nonzero(canvas)) == int(k["num_pixels"])
        assert abs(k["angle"] - math.atan2(k["end_y"] - k["start_y"], k["end_x"] - k["start_x"])) < 1e-6
        assert k["response"] == np.float32(k["line_length"]) / np.float32(640)


def test_line_extract_structure(orc):
    img = synth.make_line_image(4)
    kl, lbd, fn = orc.line_extract(img)
    assert 60 < len(kl) < 1024 and lbd.shape == (len(kl), 32) and fn.shape == (len(kl), 3)
    assert (kl["line_length"] >= 60).all()
    # line function: both end points lie on it, normalised normal
    sp = np.stack([kl["start_x"], kl["start_y"], np.ones(len(kl))], 1).astype(np.float64)
    ep = np.stack([kl["end_x"], kl["end_y"], np.ones(len(kl))], 1).astype(np.float64)
    assert np.abs((sp * fn).sum(1)).max() < 1e-9 and np.abs((ep * fn).sum(1)).max() < 1e-9
    assert np.allclose(np.hypot(fn[:, 0], fn[:, 1]), 1.0, atol=1e-12)
    # float descriptor: unit norm, binary = 8 comparisons per band pair
    d8, df = orc.lbd_compute(img, kl)
    assert np.array_equal(d8, lbd)
    assert np.allclose((df.astype(np.float64) ** 2).sum(1), 1.0, atol=1e-5)
    comb = [(0, 1), (0, 2), (0, 3), (0, 4), (0, 5), (0, 6), (1, 2), (1, 3), (1, 4), (1, 5), (1, 6), (2, 3), (2, 4), (2, 5),
            (2, 6), (2, 7), (2, 8), (3, 4), (3, 5), (3, 6), (3, 7), (3, 8), (4, 5), (4, 6), (4, 7), (4, 8), (5, 6), (5, 7),
            (5, 8), (6, 7), (6, 8), (7, 8)]
    for c, (i, j) in enumerate(comb):
        bits = (df[:, 8 * i:8 * i + 8] > df[:, 8 * j:8 * j + 8]).astype(np.uint8)
        assert np.array_equal((bits << np.arange(8, dtype=np.uint8)).sum(1).astype(np.uint8), d8[:, c])
    # the descriptor of a line is (nearly) independent of libm vs detmath
    d8m, _ = orc.lbd_compute(img, kl, libm=1)
    assert (np.unpackbits(d8 ^ d8m, axis=1).sum(1) <= 2).all()
    # a flat image has no line and the extractor returns nothing
    kl0, lbd0, fn0 = orc.line_extract(np.full((480, 640), 9, np.uint8))
    assert len(kl0) == 0


def test_detmath_accurate(orc):
    import ctypes as C
    import subprocess
    import tempfile
    hdr = ROOT / "structure-plp-slam_b200" / "csrc" / "detmath.h"
    src = '#include "%s"\nextern "C" { double t_sin(double x){return det_sin(x);} double t_cos(double x){return det_cos(x);}' \
          ' double t_atan2(double y,double x){return det_atan2(y,x);} }\n' % hdr
    with tempfile.TemporaryDirectory() as d:
        (Path(d) / "t.cc").write_text(src)
        subprocess.run(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", str(Path(d) / "t.cc"), "-o",
                        str(Path(d) / "t.so")], check=True)
        lib = C.CDLL(str(Path(d) / "t.so"))
        for f in (lib.t_sin, lib.t_cos):
            f.restype, f.argtypes = C.c_double, [C.c_double]
        lib.t_atan2.restype, lib.t_atan2.argtypes = C.c_double, [C.c_double, C.c_double]
        rng = np.random.default_rng(0)
        for x in rng.uniform(-4 * math.pi, 4 * math.pi, 20000):
            assert abs(lib.t_sin(x) - math.sin(x)) < 2.3e-16 and abs(lib.t_cos(x) - math.cos(x)) < 2.3e-16
            xf = float(np.float32(x))
            assert np.float32(lib.t_cos(xf)) == np.float32(math.cos(xf))
        for y, x in rng.uniform(-700, 700, (20000, 2)):
            assert abs(lib.t_atan2(y, x) - math.atan2(y, x)) < 9e-16
        assert lib.t_atan2(0.0, -1.0) == math.pi and lib.t_atan2(1.0, 0.0) == math.pi / 2
