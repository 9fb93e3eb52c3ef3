"""The FAST cell tiles arrive two ways: by TMA bulk tensor copies in runs of cells per CTA (fast_cells_tma_kernel, the
default) and by plain loads, one cell per CTA (fast_cells_kernel_v2, for caller buffers TMA cannot describe: a base or
pitch that is not a multiple of 16 bytes).  The plain-load arms reach that kernel the way a caller does: through the
device entry point from a buffer one byte past a 16-byte boundary, or through the host entry points (which stage the
frames at pitch `cols`) at a width that is not a multiple of 16.  Both paths must give the oracle's candidates, keypoints
and descriptors bit for bit, at the benchmark's batch and at the edges of the run logic: a run crossing a level boundary,
a partial last run, masked cells, the fallback threshold, and a frame whose candidates overflow the quadtree's clip."""
import numpy as np
import pytest

import oracle_api
import synth
from test_batch_dev_gpu import _OrbOut, _bench, _kernels_run, _pitched

pytestmark = pytest.mark.gpu
RUN = 4  # cells per CTA of fast_cells_tma_kernel (kFastRun in csrc/orb.cu)
MAX_ROWS, MAX_COLS = 1061, 2085
PLAIN_COLS = 632  # not a multiple of 16: the host entry points stage such frames at a pitch TMA cannot describe


@pytest.fixture
def own():
    objs = []
    yield lambda x: objs.append(x) or x
    for x in reversed(objs):
        (x.free if hasattr(x, "free") else x.close)()


def _run_plain(ctx, plp, run):
    """Run `run`, which must take the plain-load FAST and blur kernels and no TMA kernel."""
    names = _kernels_run(ctx, plp.lib(), run)
    assert {"fast_cells_kernel_v2", "blur_tiles_kernel"} <= names and not any("_tma_" in k for k in names), names


def _run_tma(ctx, plp, run):
    """Run `run`, which must take the TMA FAST kernel."""
    names = _kernels_run(ctx, plp.lib(), run)
    assert any(k.startswith("fast_cells_tma_kernel") for k in names), names


def _cells_per_level(orc, p, rows, cols):
    """The cell count of every level, as plp_orb_create lays the cells out (orb_extractor.cc:344-392)."""
    ws, hs = orc.orb_level_sizes(p, rows, cols)
    out = []
    for w, h in zip(ws, hs):
        w, h = int(w), int(h)
        if w <= 38 or h <= 38:
            out.append(0)
            continue
        mx, my = w - 19, h - 19
        ny = len([i for i in range((my - 19) // 64 + 1) if 19 + 64 * i < my - 6])
        nx = len([j for j in range((mx - 19) // 64 + 1) if 19 + 64 * j < mx - 6])
        out.append(nx * ny)
    return out


def _candidates(ext, b, levels):
    return [ext.debug_candidates(b, l) for l in range(levels)]


def _same_candidates(a, b, what):
    for l, (ca, cb) in enumerate(zip(a, b)):
        assert len(ca) == len(cb), f"{what}: candidate count level {l}"
        for f in ("x", "y", "response"):
            assert np.array_equal(ca[f], cb[f]), f"{what}: candidates level {l} field {f}"


def _check_oracle(orc, p, img, ext, b, got, mask=None):
    r = orc.orb_extract(p, img, mask=mask, debug=True)
    off = 0
    for l in range(p.num_levels):
        c = r["cands"][off: off + r["cands_per_level"][l]]
        off += r["cands_per_level"][l]
        g = ext.debug_candidates(b, l)
        assert len(g) == len(c), f"frame {b}: candidate count level {l}"
        for f in ("x", "y", "response"):
            assert np.array_equal(g[f], c[f]), f"frame {b}: candidates level {l} field {f}"
    kps, desc = got
    assert np.array_equal(kps, r["kps"]), f"frame {b}: keypoints"
    assert np.array_equal(desc, r["desc"]), f"frame {b}: descriptors"


def test_bench_batch_tma_equals_unaligned_plain_loads_and_oracle(ctx, orc, plp, own):
    """One 256-frame sub-batch of the benchmark's inputs.  At 640 x 480 the frame's 216 cells are 54 full runs, and
    level 0's 70 cells end in the middle of a run, so runs cross levels.  The plain-load arm reads the same frames from a
    caller buffer one byte past a 16-byte boundary; its status array must be all zero, as the host call's is (that call
    fails on a non-zero status)."""
    _, frames, _ = _bench().build_inputs(256, 1234)
    B, rows, cols = frames.shape
    p = oracle_api.orb_params()
    cells = _cells_per_level(orc, p, rows, cols)
    assert sum(cells) == 216 and cells[0] % RUN != 0
    tma = own(plp.OrbExtractor(ctx, rows, cols, max_batch=B))
    plain = own(plp.OrbExtractor(ctx, rows, cols, max_batch=B))
    got_t = {}
    _run_tma(ctx, plp, lambda: got_t.update(enumerate(tma.extract_batch(frames))))
    out = own(_OrbOut(plp, ctx, B, plain.capacity))
    d_img, ptr = _pitched(ctx, frames, cols, offset=1)
    own(d_img)
    _run_plain(ctx, plp, lambda: out.run(plain, ptr, B, cols))
    _, got_p, st = out.get(plp, B)
    assert not st.any(), st
    for b in range(B):
        _same_candidates(_candidates(tma, b, 8), _candidates(plain, b, 8), f"frame {b}")
        assert np.array_equal(got_t[b][0], got_p[b][0]), f"frame {b}: keypoints"
        assert np.array_equal(got_t[b][1], got_p[b][1]), f"frame {b}: descriptors"
    for b in (0, 70, 131, 255):
        _check_oracle(orc, p, frames[b], tma, b, got_t[b])


@pytest.mark.parametrize("rows,cols", [(480, 752), (512, 512)], ids=["euroc_752x480", "tumvi_512x512"])
def test_other_sizes_and_partial_last_run(ctx, orc, plp, own, rows, cols):
    """752 x 480 (EuRoC): 256 cells per frame, runs crossing the boundaries of levels 4 to 6.  512 x 512 (TUM-VI): 174
    cells, so the last CTA of a frame has a partial run.  A caller buffer and status array: status 0 (3 would be a tile
    copy that never arrived).  The plain-load arm reads a buffer one byte past a 16-byte boundary."""
    p = oracle_api.orb_params()
    cells = _cells_per_level(orc, p, rows, cols)
    assert (sum(cells) % RUN != 0) == (cols == 512)
    imgs = np.stack([synth.make_texture(60 + i, rows, cols) for i in range(3)] +
                    [synth.make_plp_texture(63, rows, cols), synth.make_line_image(64, rows, cols)])
    B = len(imgs)
    for offset, check in ((0, _run_tma), (1, _run_plain)):
        ext = own(plp.OrbExtractor(ctx, rows, cols, max_batch=B))
        out = own(_OrbOut(plp, ctx, B, ext.capacity))
        d_img, ptr = _pitched(ctx, imgs, cols, offset=offset)
        own(d_img)
        check(ctx, plp, lambda: out.run(ext, ptr, B, cols))
        n, got, st = out.get(plp, B)
        assert not st.any(), st
        for b in range(B):
            _check_oracle(orc, p, imgs[b], ext, b, got[b])


def test_mask_and_fallback_threshold(ctx, orc, plp, own):
    """A mask (cells whose corners are masked are skipped, keypoints under the mask dropped) and a low-contrast frame
    where about half of the cells find no corner at the initial threshold and fall back to the minimum one.  The
    plain-load arm takes the same frames and mask cropped to a width TMA cannot describe."""
    rows, cols = 480, 640
    p = oracle_api.orb_params()
    tex = synth.make_texture(71)
    weak = (100 + (tex.astype(np.int32) - 128) // 4).clip(0, 255).astype(np.uint8)
    mask = np.ones((rows, cols), np.uint8)
    mask[100:260, 200:420] = 0
    mask[400:, :90] = 0
    for w, check in ((cols, _run_tma), (PLAIN_COLS, _run_plain)):
        ext = own(plp.OrbExtractor(ctx, rows, w))
        for img, mk in ((tex, mask), (weak, None), (weak, mask)):
            img, mk = np.ascontiguousarray(img[:, :w]), None if mk is None else np.ascontiguousarray(mk[:, :w])
            got = []
            check(ctx, plp, lambda: got.extend(ext.extract(img, mk)))
            _check_oracle(orc, p, img, ext, 0, got, mask=mk)
    r = orc.orb_extract(p, weak, debug=True)
    assert 0 < (r["cands"]["response"] < 20).sum() < len(r["cands"])


def _skipped_cells(orc, p, rows, cols, mask):
    """Per cell, in the kernels' order (level-major, row-major), whether a masked corner skips it
    (orb_extractor.cc:395-401, the corners scaled to level 0 in f32 like the kernels)."""
    ws, hs = orc.orb_level_sizes(p, rows, cols)
    scale, out = np.float32(1), []
    for l, (w, h) in enumerate(zip(ws, hs)):
        if l > 0:
            scale = np.float32(scale * np.float32(p.scale_factor))
        w, h = int(w), int(h)
        if w <= 38 or h <= 38:
            continue
        mx, my = w - 19, h - 19
        masked = lambda y, x: mask[int(np.float32(y) * scale), int(np.float32(x) * scale)] == 0
        for i in range((my - 19) // 64 + 1):
            y0 = 19 + 64 * i
            if y0 >= my - 6:
                continue
            for j in range((mx - 19) // 64 + 1):
                x0 = 19 + 64 * j
                if x0 >= mx - 6:
                    continue
                x1, y1 = min(x0 + 70, mx), min(y0 + 70, my)
                out.append(masked(y0, x0) or masked(y1, x0) or masked(y0, x1) or masked(y1, x1))
    return np.array(out)


def test_masked_cells_inside_runs(ctx, orc, plp, own):
    """Cells skipped by the mask in the middle of a run: the TMA kernel writes the previous cell's output while it
    starts on the skipped one, whose (empty) counts must not overwrite what that output still reads.  The plain-load arm
    takes the same frames and mask cropped to a width TMA cannot describe."""
    rows, cols = 480, 640
    p = oracle_api.orb_params()
    rng = np.random.default_rng(97)
    mask = np.ones((rows, cols), np.uint8)
    for y, x in zip(rng.integers(0, rows - 12, 60), rng.integers(0, cols - 12, 60)):
        mask[y: y + 12, x: x + 12] = 0
    skip = _skipped_cells(orc, p, rows, cols, mask)
    assert len(skip) == 216
    inside = [c for c in range(1, len(skip)) if c % RUN != 0 and skip[c] and not skip[c - 1]]
    assert len(inside) >= 5, inside
    frames = [synth.make_texture(100 + i) for i in range(4)] + [synth.make_plp_texture(104)]
    tma, plain = own(plp.OrbExtractor(ctx, rows, cols)), own(plp.OrbExtractor(ctx, rows, PLAIN_COLS))
    mask_p = np.ascontiguousarray(mask[:, :PLAIN_COLS])
    for img in frames:
        got_t, got_p = [], []
        _run_tma(ctx, plp, lambda: got_t.extend(tma.extract(img, mask)))
        _check_oracle(orc, p, img, tma, 0, got_t, mask=mask)
        img_p = np.ascontiguousarray(img[:, :PLAIN_COLS])
        _run_plain(ctx, plp, lambda: got_p.extend(plain.extract(img_p, mask_p)))
        _check_oracle(orc, p, img_p, plain, 0, got_p, mask=mask_p)


def test_unaligned_caller_buffer_takes_plain_loads(ctx, orc, plp, own):
    """A caller buffer one byte past an aligned address cannot be described by TMA: the plain-load kernel serves every
    level, with the same candidates as the TMA path on an aligned copy of the frames."""
    imgs = np.stack([synth.make_texture(80 + i) for i in range(3)] + [synth.make_plp_texture(84)])
    B, rows, cols = imgs.shape
    ext_a = own(plp.OrbExtractor(ctx, rows, cols, max_batch=B))
    ext_u = own(plp.OrbExtractor(ctx, rows, cols, max_batch=B))
    out_a, out_u = own(_OrbOut(plp, ctx, B, ext_a.capacity)), own(_OrbOut(plp, ctx, B, ext_u.capacity))
    d_a, pa = _pitched(ctx, imgs, cols)
    d_u, pu = _pitched(ctx, imgs, cols, offset=1, seed=3)
    own(d_a)
    own(d_u)
    _run_tma(ctx, plp, lambda: out_a.run(ext_a, pa, B, cols))
    _run_plain(ctx, plp, lambda: out_u.run(ext_u, pu, B, cols))
    _, got_a, st_a = out_a.get(plp, B)
    _, got_u, st_u = out_u.get(plp, B)
    assert not st_a.any() and not st_u.any(), (st_a, st_u)
    p = oracle_api.orb_params()
    for b in range(B):
        _same_candidates(_candidates(ext_a, b, 8), _candidates(ext_u, b, 8), f"frame {b}")
        _check_oracle(orc, p, imgs[b], ext_u, b, got_u[b])


def test_noise_clip_status(ctx, orc, plp, own):
    """2085 x 1061 noise overflows the 65 535-candidate clip of level 0: status 1 on that frame only, on both paths (the
    plain-load arm reads a buffer one byte past a 16-byte boundary).  640 x 480 noise stays below it, and so does its
    632-pixel-wide crop, which takes the plain loads."""
    noise = np.random.default_rng(91).integers(0, 256, (MAX_ROWS, MAX_COLS), dtype=np.uint8)
    imgs = np.stack([synth.make_texture(92, MAX_ROWS, MAX_COLS), noise, synth.make_texture(93, MAX_ROWS, MAX_COLS)])
    cands = []
    for offset, check in ((0, _run_tma), (1, _run_plain)):
        ext = own(plp.OrbExtractor(ctx, MAX_ROWS, MAX_COLS, 2000, max_batch=3))
        out = own(_OrbOut(plp, ctx, 3, ext.capacity))
        d_img, ptr = _pitched(ctx, imgs, MAX_COLS + 11, offset=offset, seed=9)
        own(d_img)
        check(ctx, plp, lambda: out.run(ext, ptr, 3, MAX_COLS + 11))
        _, _, st = out.get(plp, 3)
        assert list(st) == [0, 1, 0], st
        cands.append([_candidates(ext, b, 8) for b in range(3)])
    for b in range(3):
        _same_candidates(cands[0][b], cands[1][b], f"2085 x 1061 frame {b}")
    small = np.random.default_rng(94).integers(0, 256, (480, 640), dtype=np.uint8)
    p = oracle_api.orb_params()
    for w, check in ((640, _run_tma), (PLAIN_COLS, _run_plain)):
        ext = own(plp.OrbExtractor(ctx, 480, w))
        img, got = np.ascontiguousarray(small[:, :w]), []
        check(ctx, plp, lambda: got.extend(ext.extract(img)))
        _check_oracle(orc, p, img, ext, 0, got)
