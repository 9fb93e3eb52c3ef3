"""GPU parity: LSD + LBD line extraction through the C ABI vs the oracle, stage by stage -- the half-resolution image,
the raw LSD segments (bit-exact floats, detection order), the KeyLines (every field), the LBD bytes and the 2-D line
functions.  Bar: bit-exact (the oracle's "det" mode is itself pinned bit-exactly against cv2 in test_lines_oracle.py)."""
import numpy as np
import pytest

import oracle_api
import synth

pytestmark = pytest.mark.gpu
VARIANTS = [1, 2, 3]

KL_FIELDS = ("angle", "class_id", "octave", "pt_x", "pt_y", "response", "size", "start_x", "start_y", "end_x", "end_y",
             "s_oct_x", "s_oct_y", "e_oct_x", "e_oct_y", "line_length", "num_pixels")


def _compare(trk, orc, img, b=0, got=None):
    kl, lbd, fn = trk.extract_LSD_LBD(img) if got is None else got
    assert np.array_equal(trk.debug_scaled(b), orc.lsd_scaled(img)), "half-resolution image"
    segs = trk.debug_segments(b)
    ref = orc.lsd_detect(img)
    assert segs.shape == ref.shape, f"{len(segs)} vs {len(ref)} segments"
    assert np.array_equal(segs, ref), "LSD segments"
    okl, olbd, ofn = orc.line_extract(img)
    assert len(kl) == len(okl)
    for f in KL_FIELDS:
        assert np.array_equal(kl[f], okl[f]), f
    if len(kl):
        _, ofl = orc.lbd_compute(img, okl)
        assert np.array_equal(trk.debug_lbd_float(b, len(kl)), ofl), "LBD float vectors"
    assert np.array_equal(lbd, olbd), "LBD bytes"
    assert np.array_equal(fn, ofn), "line functions"
    return len(segs), len(kl)


# region growing variants (lines.cu): 1 = one warp per frame, 2 = several warps per frame in speculative rounds with in-order commit,
# 3 = out of order with a reorder buffer and in-order commit
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("kind,seed,shape", [("lines", 1, (480, 640)), ("lines", 2, (480, 752)), ("texture", 1234, (480, 640)),
                                             ("texture", 7, (480, 752)), ("lines", 9, (376, 1240)), ("plp", 5, (480, 640))])
def test_line_extract_matches_oracle(ctx, orc, plp, kind, seed, shape, variant):
    img = (synth.make_line_image(seed, *shape) if kind == "lines" else synth.make_plp_texture(seed, *shape) if kind == "plp"
           else synth.make_texture(seed, *shape))
    trk = plp.LineFeatureTracker(ctx, shape[0], shape[1])
    trk.grow_variant(variant)
    nseg, nkl = _compare(trk, orc, img)
    assert nseg > 100
    if kind == "lines":
        assert nkl > 40
    if variant == 2:
        st = trk.grow_stats(0)
        assert st["rounds"] > 0 and st["seeds_run"] >= nseg
        print(f"[mw] {kind} {shape}: {st}, {nseg} segments")
    if variant == 3:
        st = trk.grow_stats(0, ooo=True)
        assert st["tickets"] >= nseg
        print(f"[ooo] {kind} {shape}: {st}, {nseg} segments")
    trk.close()


@pytest.mark.parametrize("variant", VARIANTS)
def test_edge_cases(ctx, orc, plp, variant):
    trk = plp.LineFeatureTracker(ctx, 480, 640)
    trk.grow_variant(variant)
    # flat image: no gradient above the threshold, no seed, no line (the reference returns empty outputs)
    kl, lbd, fn = trk.extract_LSD_LBD(np.full((480, 640), 128, np.uint8))
    assert len(kl) == 0 and lbd.shape == (0, 32) and fn.shape == (0, 3)
    assert len(trk.debug_segments(0)) == 0
    # pure noise: many seeds, hardly any accepted region
    rng = np.random.default_rng(3)
    _compare(trk, orc, rng.integers(0, 256, (480, 640), dtype=np.uint8))
    # two grey levels: every edge pixel falls into the same gradient bin (worst case of the seed ordering)
    img = np.full((480, 640), 40, np.uint8)
    img[100:380, 150:500] = 200
    img[200:300, 0:640] = 90
    nseg, nkl = _compare(trk, orc, img)
    assert nkl >= 4
    # a line touching the image border exercises checkLineExtremes and the reflect-101 borders
    img = np.full((480, 640), 30, np.uint8)
    img[:, 320:] = 220
    img[0:3, :] = 255
    _compare(trk, orc, img)
    trk.close()


def test_batch_equals_single(ctx, orc, plp):
    imgs = np.stack([synth.make_line_image(20 + i) for i in range(5)] + [synth.make_texture(3)])
    trk = plp.LineFeatureTracker(ctx, 480, 640, max_batch=6)
    # one warp per frame with both placements of the half-resolution image, then the multi-warp variant
    for variant, global_image in [(1, False), (1, True)] + [(v, False) for v in VARIANTS[1:]]:
        trk.grow_variant(variant)
        trk.force_global_image(global_image)
        res = trk.extract_batch(imgs)
        for b in range(len(imgs)):
            _compare(trk, orc, imgs[b], b=b, got=res[b])
    trk.force_global_image(False)
    trk.grow_variant(0)
    # strided input (step > cols) through the single-frame entry point
    wide = np.zeros((480, 700), np.uint8)
    wide[:, :640] = imgs[1]
    kl, lbd, fn = trk.extract_LSD_LBD(wide[:, :640])
    assert np.array_equal(kl, res[1][0]) and np.array_equal(lbd, res[1][1])
    trk.close()


def test_wrong_size_is_rejected(ctx, plp):
    trk = plp.LineFeatureTracker(ctx, 480, 640)
    with pytest.raises(plp.PlpError):
        trk.extract_LSD_LBD(np.zeros((100, 100), np.uint8))
    trk.close()
