"""GPU parity at the camera geometries the reference ships and at the edges of the supported image sizes.

The other GPU tests run at 640 x 480 and 752 x 480 (a few at 1241 x 376, 600 x 600, 320 x 240).  The reference's example
configurations also use 1242 x 375 (KITTI 03), 1226 x 370 (KITTI 04-12) and 512 x 512 (TUM-VI), with their own feature
settings.  Image geometry is where the kernels keep their edge logic: 16-byte aligned TMA boxes (plain loads when level 0
is not aligned), 64 x 32 blur tiles in runs of 4 per CTA that can cross levels, reflect-101 fix-ups at tile borders, FAST
cells clipped at the right and bottom, the quadtree's initial nodes, the LSD 2x downscale.  Every comparison is against
the CPU oracle, bit-exact like the per-kernel tests."""
import ctypes as C

import numpy as np
import pytest

import oracle_api
import scene
import synth
from scene import oracle_track as _oracle_track
from test_batch_dev_gpu import _OrbOut, _kernels_run, _pitched
from test_lines_gpu import VARIANTS, _compare as _compare_lines

pytestmark = pytest.mark.gpu

# (rows, cols, Feature.max_num_keypoints, ini_fast_threshold, min_fast_threshold) of the reference's example configs
KITTI_00 = (376, 1241, 2000, 20, 7)
KITTI_03 = (375, 1242, 2000, 20, 7)
KITTI_04 = (370, 1226, 2000, 20, 7)
TUM_VI = (512, 512, 1000, 20, 7)
# Camera.fx and Camera.focal_x_baseline of the stereo configs (KITTI_stereo_*.yaml: ini_fast_threshold 12)
STEREO = {"kitti00": ((376, 1241), 718.856, 386.1448, 12), "kitti03": ((375, 1242), 721.5377, 387.5744, 12),
          "kitti04": ((370, 1226), 707.0912, 379.8145, 12), "tumvi": ((512, 512), 61.75453410721205, 6.242596912726197, 20)}
MAX_ROWS, MAX_COLS = 1061, 2085       # packed candidate coordinates: x < 2048, y < 1024 inside the 19-px border


@pytest.fixture
def own():
    """own(x) returns x and closes / frees it when the test ends, also after a failed assertion (a handle left to the
    garbage collector could outlive the session's context)."""
    objs = []
    yield lambda x: objs.append(x) or x
    for x in reversed(objs):
        (x.free if hasattr(x, "free") else x.close)()


def _params(mk, ini, mn, levels=8):
    return oracle_api.orb_params(mk, 1.2, levels, ini, mn)


def _orb_stages(ext, orc, p, img, got, b=0):
    """ext's frame b of its last extraction against the oracle, stage by stage: pyramid, blurred pyramid, FAST
    candidates, keypoints, descriptors.  got = (keypoints, descriptors) ext returned for that frame."""
    r = orc.orb_extract(p, img, debug=True)
    off = 0
    for l in range(p.num_levels):
        lvl = r["pyramid"][l]
        assert np.array_equal(ext.pyramid_level(b, l), lvl), f"pyramid level {l}"
        blurred = ext.debug_blurred(b, l)
        assert blurred.shape == lvl.shape
        bad = np.argwhere(blurred != orc.blur7(lvl))
        assert len(bad) == 0, f"blurred level {l} ({lvl.shape[1]} x {lvl.shape[0]}): {len(bad)} pixels differ, first {bad[:4]}"
        c = r["cands"][off: off + r["cands_per_level"][l]]
        off += r["cands_per_level"][l]
        g = ext.debug_candidates(b, l)
        assert len(g) == len(c), f"candidate count level {l}"
        for f in ("x", "y", "response"):
            assert np.array_equal(g[f], c[f]), f"candidates level {l} field {f}"
    kps, desc = got
    assert len(kps) == len(r["kps"])
    for f in ("x", "y", "size", "angle", "response", "octave", "class_id"):
        assert np.array_equal(kps[f], r["kps"][f]), f
    assert np.array_equal(desc, r["desc"])
    return r


def _blur_tiles(orc, p, rows, cols):
    w, h = orc.orb_level_sizes(p, rows, cols)
    return int(sum(((int(a) + 63) // 64) * ((int(b) + 31) // 32) for a, b in zip(w, h)))


def _budgets(max_kp, sf=1.2, levels=8):
    """orb_extractor.cc's per-level keypoint budget, as plp_orb_create computes it."""
    desired = max_kp * (1.0 - 1.0 / sf) / (1.0 - (1.0 / sf) ** levels)
    out, total = [], 0
    for _ in range(levels - 1):
        out.append(int(round(desired)))
        total += out[-1]
        desired *= 1.0 / sf
    return out + [max(max_kp - total, 0)]


# ----------------------------------------------------------------------------------------------------- ORB
@pytest.mark.parametrize("rows,cols,mk,ini,mn", [KITTI_03, KITTI_04, KITTI_00, TUM_VI, (479, 639, 1000, 20, 7),
                                                 (481, 641, 1000, 20, 7), (376, 1241, 2000, 12, 2), (375, 1242, 1500, 20, 7)],
                         ids=["kitti03", "kitti04", "kitti00", "tumvi", "479x639", "481x641", "kitti00_fast12_2",
                              "kitti03_1500"])
def test_orb_geometry_stages(ctx, orc, plp, own, rows, cols, mk, ini, mn):
    img = synth.make_texture(rows + cols, rows, cols)
    p = _params(mk, ini, mn)
    ext = own(plp.OrbExtractor(ctx, rows, cols, mk, 1.2, 8, ini, mn))
    r = _orb_stages(ext, orc, p, img, ext.extract(img))
    assert len(r["kps"]) > 0.8 * mk


def test_quadtree_instance_switch(ctx, orc, plp, own):
    """plp_orb_create picks the 1024-node quadtree instance while every level's 4 * max(budget, initial nodes) + 8 fits
    in 1024 nodes, the 2048-node one above.  One max_num_keypts on each side of the switch, at KITTI 03's size (initial
    nodes: round(1204 / 337) = 4, never the maximum here)."""
    lib = plp.lib()
    small = max(k for k in range(500, 3000) if 4 * max(_budgets(k)) + 8 <= 1024)
    rows, cols = KITTI_03[:2]
    img = synth.make_texture(71, rows, cols)
    for mk, inst in ((small, "quadtree_kernel<1024>"), (small + 1, "quadtree_kernel<2048>")):
        p = _params(mk, 20, 7)
        ext = own(plp.OrbExtractor(ctx, rows, cols, mk))
        got = {}
        names = _kernels_run(ctx, lib, lambda: got.update(r=ext.extract(img)))
        assert {n for n in names if n.startswith("quadtree_kernel")} == {inst}, (mk, names)
        _orb_stages(ext, orc, p, img, got["r"])


@pytest.mark.parametrize("rows,cols,pad,blur", [(375, 1242, 0, "plain"), (375, 1242, 6, "tma"), (370, 1226, 6, "tma"),
                                                (512, 512, 0, "tma"), (479, 639, 0, "plain"), (479, 639, 1, "tma")],
                         ids=["kitti03_step_eq_cols", "kitti03_step16", "kitti04_step16", "tumvi", "479x639",
                              "479x639_step16"])
def test_blurred_pyramid_batch_dev(ctx, orc, plp, own, rows, cols, pad, blur):
    """plp_orb_extract_batch_dev on a caller buffer: level 0 goes through TMA only when its pitch is a multiple of 16
    (step == cols at KITTI widths takes plain loads; step rounded up to 16 takes TMA).  A batch of 3 frames, so the runs
    of 4 tiles per CTA also cover frames after the first."""
    lib = plp.lib()
    step = cols + pad
    imgs = np.stack([synth.make_texture(300 + i, rows, cols) for i in range(2)] + [synth.make_line_image(302, rows, cols)])
    B = len(imgs)
    p = _params(1000, 20, 7)
    orb = own(plp.OrbExtractor(ctx, rows, cols, max_batch=B))
    out = own(_OrbOut(plp, ctx, B, orb.capacity))
    d_img, ptr = _pitched(ctx, imgs, step, seed=pad)
    own(d_img)
    names = _kernels_run(ctx, lib, lambda: out.run(orb, ptr, B, step))
    tma = any(k.startswith("blur_tiles_tma_kernel") for k in names)
    assert tma == (blur == "tma") and ("blur_tiles_kernel" in names) == (blur == "plain"), names
    n, got, st = out.get(plp, B)
    assert not st.any()
    for b in range(B):
        _orb_stages(orb, orc, p, imgs[b], got[b], b=b)


def test_blurred_pyramid_partial_last_run(ctx, orc, plp, own):
    """A blur tile list whose length is not a multiple of 4: the last CTA of each frame makes fewer tiles, and runs cross
    from one level into the next.  Both TMA (step rounded up to 16) and plain loads (step == cols)."""
    lib = plp.lib()
    rows, cols = 479, 641
    p = _params(1000, 20, 7)
    nt = _blur_tiles(orc, p, rows, cols)
    assert nt % 4 != 0, nt
    imgs = np.stack([synth.make_texture(400 + i, rows, cols) for i in range(2)])
    orb = own(plp.OrbExtractor(ctx, rows, cols, max_batch=2))
    out = own(_OrbOut(plp, ctx, 2, orb.capacity))
    for step, want in ((cols + 15, "tma"), (cols, "plain")):
        d_img, ptr = _pitched(ctx, imgs, step, seed=step)
        own(d_img)
        names = _kernels_run(ctx, lib, lambda: out.run(orb, ptr, 2, step))
        assert any(k.startswith("blur_tiles_tma_kernel") for k in names) == (want == "tma"), names
        n, got, st = out.get(plp, 2)
        assert not st.any()
        for b in range(2):
            _orb_stages(orb, orc, p, imgs[b], got[b], b=b)


@pytest.mark.parametrize("rows,cols", [(48, 64), (75, 100), (120, 160), (41, 40)])
def test_orb_small_images(ctx, orc, plp, own, rows, cols):
    """Upper levels with no FAST cell (w or h <= 38), levels narrower than one 64 x 32 blur tile and than the 96-byte
    TMA box; 41 x 40 yields no keypoint at all.  Host wrapper (TMA when cols % 16 == 0) and a 16-byte pitch."""
    lib = plp.lib()
    p = _params(1000, 20, 7)
    img = synth.make_texture(9, rows, cols)
    ext = own(plp.OrbExtractor(ctx, rows, cols))
    _orb_stages(ext, orc, p, img, ext.extract(img))
    step = (cols + 15) // 16 * 16
    orb = own(plp.OrbExtractor(ctx, rows, cols, max_batch=1))
    out = own(_OrbOut(plp, ctx, 1, orb.capacity))
    d_img, ptr = _pitched(ctx, img[None], step, seed=3)
    own(d_img)
    names = _kernels_run(ctx, lib, lambda: out.run(orb, ptr, 1, step))
    assert any(k.startswith("blur_tiles_tma_kernel") for k in names), names
    n, got, st = out.get(plp, 1)
    assert not st.any()
    r = _orb_stages(orb, orc, p, img, got[0])
    assert (len(r["kps"]) == 0) == ((rows, cols) == (41, 40))


def test_orb_size_limits(ctx, orc, plp, own):
    """2085 x 1061 is the largest image plp_orb_create accepts; one more row or column is rejected at create."""
    img = synth.make_texture(5, MAX_ROWS, MAX_COLS)
    p = _params(2000, 20, 7)
    ext = own(plp.OrbExtractor(ctx, MAX_ROWS, MAX_COLS, 2000))
    r = _orb_stages(ext, orc, p, img, ext.extract(img))
    assert len(r["kps"]) > 1600
    for rows, cols in ((MAX_ROWS + 1, MAX_COLS), (MAX_ROWS, MAX_COLS + 1)):
        with pytest.raises(plp.PlpError, match="2085 x 1061"):
            plp.OrbExtractor(ctx, rows, cols, 2000)


def test_orb_candidate_capacity_is_reported(ctx, orc, plp, own):
    """A level with more than 65 535 FAST candidates (a 2085 x 1061 noise frame has about 211 000 at level 0) is not
    extracted: the host call returns PLP_ERR_CAPACITY naming the frame, the handle stays usable, and in a device batch only
    that frame's status is set."""
    lib = plp.lib()
    p = _params(2000, 20, 7)
    noise = np.random.default_rng(17).integers(0, 256, (MAX_ROWS, MAX_COLS), dtype=np.uint8)
    tex = [synth.make_texture(6 + i, MAX_ROWS, MAX_COLS) for i in range(2)]
    ext = own(plp.OrbExtractor(ctx, MAX_ROWS, MAX_COLS, 2000, max_batch=3))
    with pytest.raises(plp.PlpError, match="frame 0"):
        ext.extract(noise)
    _orb_stages(ext, orc, p, tex[0], ext.extract(tex[0]))
    imgs = np.stack([tex[0], noise, tex[1]])
    out = own(_OrbOut(plp, ctx, 3, ext.capacity))
    d_img, ptr = _pitched(ctx, imgs, MAX_COLS + 11, seed=4)
    own(d_img)
    out.run(ext, ptr, 3, MAX_COLS + 11)
    n, got, st = out.get(plp, 3)
    assert st[0] == 0 and st[1] != 0 and st[2] == 0, st
    for b in (0, 2):
        _orb_stages(ext, orc, p, imgs[b], got[b], b=b)


# ----------------------------------------------------------------------------------------------------- lines
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("rows,cols", [(375, 1242), (370, 1226), (512, 512), (479, 639), (16, 16)])
def test_lines_geometry(ctx, orc, plp, own, rows, cols, variant):
    """LSD + LBD with every region-growing variant.  1242 x 375 and 479 x 639 have a half-resolution row (and column)
    with a single source row (column)."""
    img = synth.make_line_image(rows * 3 + cols, rows, cols)
    trk = own(plp.LineFeatureTracker(ctx, rows, cols))
    trk.grow_variant(variant)
    nseg, nkl = _compare_lines(trk, orc, img)
    if min(rows, cols) >= 370:
        assert nseg > 100 and nkl > 20


def test_lines_batch_dev_kitti03_odd_pitch(ctx, orc, plp, own):
    from plpslam_b200.tracking import DeviceBuffer
    lib = plp.lib()
    rows, cols, B = 375, 1242, 4
    step = cols + 7
    imgs = np.stack([synth.make_line_image(500 + i, rows, cols) for i in range(B - 1)] + [synth.make_texture(504, rows, cols)])
    trk = own(plp.LineFeatureTracker(ctx, rows, cols, max_batch=B))
    cap = trk.capacity
    d_img, ptr = _pitched(ctx, imgs, step, seed=7)
    own(d_img)
    d_kl = own(DeviceBuffer(ctx, B * cap * plp.KEYLINE_DTYPE.itemsize))
    d_lbd, d_fn = own(DeviceBuffer(ctx, B * cap * 32)), own(DeviceBuffer(ctx, B * cap * 24))
    d_n, d_st = own(DeviceBuffer(ctx, B * 4)), own(DeviceBuffer.from_array(ctx, np.full(B, -1, np.int32)))
    ctx._check(lib.plp_line_extract_batch_dev(trk.handle, ptr, C.c_int(B), C.c_size_t(step), d_kl.ptr, d_lbd.ptr, d_fn.ptr,
                                              d_n.ptr, d_st.ptr))
    assert not d_st.download(np.int32, (B,)).any()
    n = d_n.download(np.int32, (B,))
    kl = d_kl.download(plp.KEYLINE_DTYPE, (B, cap))
    lbd = d_lbd.download(np.uint8, (B, cap, 32))
    fn = d_fn.download(np.float64, (B, cap, 3))
    for b in range(B):
        _compare_lines(trk, orc, imgs[b], b=b, got=(kl[b, :n[b]], lbd[b, :n[b]], fn[b, :n[b]]))


# ----------------------------------------------------------------------------------------------------- stereo
def _stereo_inputs(orc, name, n):
    (rows, cols), fx, bf, ini = STEREO[name]
    p = _params(2000 if name.startswith("kitti") else 1000, ini, 7)
    pairs = [synth.make_stereo_pair(800 + 5 * i, rows, cols, bf=bf)[:2] for i in range(n)]
    res = [(orc.orb_extract(p, l), orc.orb_extract(p, r)) for l, r in pairs]
    tab = orc.orb_tables(p)
    refs = [orc.stereo_compute(a, c, tab["scale_factors"], tab["inv_scale_factors"], bf, bf / fx) for a, c in res]
    return p, pairs, res, refs, bf, bf / fx


def _check_stereo(got, ref, what):
    gx, gd, gb = got
    ox, od, ob = ref
    assert np.array_equal(gb, ob), f"{what}: Hamming-closest right keypoint"
    assert np.array_equal(gx, ox, equal_nan=True), f"{what}: stereo_x_right"
    assert np.array_equal(gd, od, equal_nan=True), f"{what}: depths"
    return int((ox >= 0).sum())


@pytest.mark.parametrize("name", list(STEREO))
def test_stereo_geometry(ctx, orc, plp, own, name):
    p, pairs, res, refs, bf, base = _stereo_inputs(orc, name, 1)
    (left, right), (rl, rr) = pairs[0], res[0]
    rows, cols = left.shape
    el = own(plp.OrbExtractor(ctx, rows, cols, p.max_num_keypts, 1.2, 8, p.ini_fast_thr, p.min_fast_thr))
    er = own(plp.OrbExtractor(ctx, rows, cols, p.max_num_keypts, 1.2, 8, p.ini_fast_thr, p.min_fast_thr))
    kl, dl = el.extract(left)
    kr, dr = er.extract(right)
    assert np.array_equal(kl, rl["kps"]) and np.array_equal(kr, rr["kps"])
    assert np.array_equal(dl, rl["desc"]) and np.array_equal(dr, rr["desc"])
    n_ok = _check_stereo(el.stereo_compute(er, kl, dl, kr, dr, bf, base), refs[0], name)
    assert n_ok > 50, n_ok


@pytest.mark.parametrize("name", list(STEREO))
def test_stereo_batch_dev_geometry(ctx, orc, plp, own, name):
    """The benchmark's stereo layout at each shipped stereo geometry: right ORB on a second context, left on the first,
    then plp_stereo_compute_batch_dev over 3 pairs."""
    from plpslam_b200.tracking import DeviceBuffer
    lib = plp.lib()
    N = 3
    p, pairs, res, refs, bf, base = _stereo_inputs(orc, name, N)
    left, right = np.stack([a for a, _ in pairs]), np.stack([c for _, c in pairs])
    rows, cols = left.shape[1:]
    step = cols + 16
    ctx_r = own(plp.Context(ctx.device))
    mk = (p.max_num_keypts, 1.2, 8, p.ini_fast_thr, p.min_fast_thr)
    el, er = own(plp.OrbExtractor(ctx, rows, cols, *mk, max_batch=N)), own(plp.OrbExtractor(ctx_r, rows, cols, *mk, max_batch=N))
    cap = el.capacity
    d_l, p_l = _pitched(ctx, left, step, seed=1)
    d_r, p_r = _pitched(ctx_r, right, step, seed=2)
    out_l, out_r = own(_OrbOut(plp, ctx, N, cap)), own(_OrbOut(plp, ctx, N, cap))
    d_xr, d_dp, d_br = (own(DeviceBuffer(ctx, N * cap * 4)) for _ in range(3))
    own(d_l), own(d_r)
    out_r.run(er, p_r, N, step)
    out_l.run(el, p_l, N, step)
    ctx.wait(ctx_r)
    ctx._check(lib.plp_stereo_compute_batch_dev(ctx.handle, el.handle, er.handle, C.c_int(N), out_l.kp.ptr, out_l.desc.ptr,
                                                out_l.n.ptr, out_r.kp.ptr, out_r.desc.ptr, out_r.n.ptr, C.c_float(bf),
                                                C.c_float(base), d_xr.ptr, d_dp.ptr, d_br.ptr))
    xr = d_xr.download(np.float32, (N, cap))
    dp = d_dp.download(np.float32, (N, cap))
    br = d_br.download(np.int32, (N, cap))
    nl, got_l, st_l = out_l.get(plp, N)
    nr, got_r, st_r = out_r.get(plp, N)
    assert not st_l.any() and not st_r.any()
    for b in range(N):
        for (k, d), r in ((got_l[b], res[b][0]), (got_r[b], res[b][1])):
            assert np.array_equal(k, r["kps"]) and np.array_equal(d, r["desc"]), f"{name} frame {b}: ORB"
        k = nl[b]
        _check_stereo((xr[b, :k], dp[b, :k], br[b, :k]), refs[b], f"{name} frame {b}")


# ----------------------------------------------------------------------------------------------------- front end
@pytest.mark.parametrize("rows,cols", [(376, 1241), (375, 1242)], ids=["kitti00", "kitti03"])
def test_front_end_geometry(ctx, orc, plp, own, rows, cols):
    """tracking.FrontEnd (extract -> motion_based_track) at KITTI sizes, principal point at the image centre: every frame
    equals the oracle chain."""
    from plpslam_b200.tracking import FrontEnd
    B = 4
    seq = scene.PlanarSequence(seed=13, n_frames=B + 1, rows=rows, cols=cols, cx=cols / 2.0, cy=rows / 2.0)
    p = _params(1000, 20, 7)
    res = [orc.orb_extract(p, f) for f in seq.frames]
    fe = own(FrontEnd(ctx, rows, cols, seq.camera(plp), max_batch=8))
    rng = np.random.default_rng(5)
    preds = [seq.predicted_pose(t, rng) for t in range(1, B + 1)]
    lasts = [seq.last_frame_landmarks(t - 1, res[t - 1]["kps"], res[t - 1]["desc"]) for t in range(1, B + 1)]
    fe.upload_images(seq.frames[1:B + 1])
    fe.set_last_frames(lasts, np.stack(preds), np.stack(seq.poses[0:B]))
    fe.step(B, 20.0)
    kps = fe.download_keypoints(B)
    out = fe.download_tracking(B)
    assert not out["status"].any()
    want_iters = []
    for b in range(B):
        t = b + 1
        assert np.array_equal(kps[b][0], res[t]["kps"]) and np.array_equal(kps[b][1], res[t]["desc"])
        m, T, nv, n_inl, iters = _oracle_track(orc, plp, seq, res, t, preds[b])
        assert np.array_equal(out["matched"][b], m), f"frame {b}"
        assert out["num_valid"][b] == nv and out["n_inliers"][b] == n_inl
        assert nv >= 20
        want_iters.append(iters)
        rel = np.linalg.norm(out["pose"][b] - T) / np.linalg.norm(T)
        assert rel < 1e-4, rel
    scene.check_lm_iters(out["lm_iters"], want_iters, "front end")
