"""GPU parity of the device-resident batched entry points (the `_dev` calls bench.py times) against the oracle, in the
configurations the benchmark runs them in: caller-owned device buffers (pitched, unaligned), batches of 100 to 1600
frames, extraction and tracking on separate streams with no host synchronisation between steps.

Every other GPU test reaches these kernels through the host-pointer wrappers, which always hand them a handle-owned,
aligned image buffer with step == cols, small batches and a single stream."""
import ctypes as C
import hashlib
import importlib.util
import json
from pathlib import Path

import numpy as np
import pytest

import bow_data
import oracle_api
import scene
import synth
from test_lines_gpu import _compare as _compare_lines
from scene import oracle_track as _oracle_track

pytestmark = pytest.mark.gpu
BF, BASELINE = 47.906, 0.11
ROOT = Path(__file__).resolve().parent.parent


def _bench():
    spec = importlib.util.spec_from_file_location("plp_bench", ROOT / "bench.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _pitched(ctx, imgs, step, offset=0, seed=0):
    """A caller-owned device buffer holding `imgs` (B x rows x cols) with row pitch `step`, starting `offset` bytes into
    the allocation.  The padding bytes are random: a kernel that reads them changes its answer."""
    from plpslam_b200.tracking import DeviceBuffer
    B, rows, cols = imgs.shape
    host = np.random.default_rng(seed).integers(0, 256, B * rows * step + offset, dtype=np.uint8)
    host[offset:].reshape(B, rows, step)[:, :, :cols] = imgs
    buf = DeviceBuffer.from_array(ctx, host)
    return buf, C.c_void_p(buf.ptr.value + offset)


def _kernels_run(ctx, lib, run):
    """Names of the kernels `run` launched on ctx (from the context's per-kernel timing report)."""
    ctx._check(lib.plp_ctx_kernel_timing(ctx.handle, 1))
    try:
        run()
        buf = C.create_string_buffer(1 << 16)
        ctx._check(lib.plp_ctx_kernel_timing_report(ctx.handle, buf, C.c_size_t(len(buf))))
    finally:
        ctx._check(lib.plp_ctx_kernel_timing(ctx.handle, 0))
    return set(json.loads(buf.value.decode()))


def _sm_count(device):
    cu = C.CDLL("libcuda.so.1")
    dev, n = C.c_int(), C.c_int()
    assert cu.cuInit(0) == 0 and cu.cuDeviceGet(C.byref(dev), device) == 0
    assert cu.cuDeviceGetAttribute(C.byref(n), 16, dev) == 0   # CU_DEVICE_ATTRIBUTE_MULTIPROCESSOR_COUNT
    return n.value


_ORB_REF = {}


def _orb_ref(orc, img):
    key = hashlib.sha1(np.ascontiguousarray(img).tobytes()).hexdigest()
    if key not in _ORB_REF:
        _ORB_REF[key] = orc.orb_extract(oracle_api.orb_params(), img)
    return _ORB_REF[key]


class _OrbOut:
    """Caller-owned outputs of plp_orb_extract_batch_dev; the status array starts non-zero so that the call must write it."""

    def __init__(self, plp, ctx, batch, cap):
        from plpslam_b200.tracking import DeviceBuffer
        self.cap = cap
        self.kp = DeviceBuffer(ctx, batch * cap * plp.KP_DTYPE.itemsize)
        self.desc = DeviceBuffer(ctx, batch * cap * 32)
        self.n = DeviceBuffer(ctx, batch * 4)
        self.st = DeviceBuffer.from_array(ctx, np.full(batch, -1, np.int32))

    def run(self, orb, ptr, batch, step):
        orb._ctx._check(orb._lib.plp_orb_extract_batch_dev(orb.handle, ptr, C.c_int(batch), C.c_size_t(step), self.kp.ptr,
                                                           self.desc.ptr, self.n.ptr, self.st.ptr))

    def get(self, plp, batch):
        n = self.n.download(np.int32, (batch,))
        kp = self.kp.download(plp.KP_DTYPE, (batch, self.cap))
        desc = self.desc.download(np.uint8, (batch, self.cap, 32))
        st = self.st.download(np.int32, (batch,))
        return n, [(kp[b, :n[b]], desc[b, :n[b]]) for b in range(batch)], st

    def free(self):
        for d in (self.kp, self.desc, self.n, self.st):
            d.free()


def _check_orb(orc, plp, out, imgs, what):
    n, got, st = out.get(plp, len(imgs))
    assert not st.any(), f"{what}: status {st}"
    for b, img in enumerate(imgs):
        ref = _orb_ref(orc, img)
        assert np.array_equal(got[b][0], ref["kps"]), f"{what}: keypoints of frame {b}"
        assert np.array_equal(got[b][1], ref["desc"]), f"{what}: descriptors of frame {b}"
    return n


# ----------------------------------------------------------------------------------------------------- ORB
def _orb_frames(seed):
    """8 frames of different content and keypoint counts, a flat one (no keypoint) among them."""
    seq = scene.PlanarSequence(seed=seed, n_frames=4)
    return np.stack(list(seq.frames) + [synth.make_texture(seed + 1), synth.make_plp_texture(seed + 2),
                                        np.full((480, 640), 77, np.uint8), synth.make_line_image(seed + 3)])


@pytest.mark.parametrize("pad,offset,blur", [(0, 0, "tma"), (16, 0, "tma"), (5, 0, "plain"), (0, 1, "plain")],
                         ids=["step_eq_cols", "pitched16", "pitched5", "base_plus_1"])
def test_orb_extract_batch_dev_layouts(ctx, orc, plp, pad, offset, blur):
    lib = plp.lib()
    imgs = _orb_frames(31)
    B, rows, cols = imgs.shape
    orb = plp.OrbExtractor(ctx, rows, cols, max_batch=B)
    out = _OrbOut(plp, ctx, B, orb.capacity)
    d_img, ptr = _pitched(ctx, imgs, cols + pad, offset, seed=pad + offset)
    names = _kernels_run(ctx, lib, lambda: out.run(orb, ptr, B, cols + pad))
    # 16-byte aligned base and pitch: the level-0 blur reads through a TMA descriptor; anything else: plain loads
    tma = any(k.startswith("blur_tiles_tma_kernel") for k in names)
    assert tma == (blur == "tma") and ("blur_tiles_kernel" in names) == (blur == "plain"), names
    n = _check_orb(orc, plp, out, imgs, f"pad {pad} offset {offset}")
    assert n[6] == 0 and len(np.unique(n)) > 4
    out.free()
    d_img.free()
    orb.close()


def test_orb_level0_descriptor_follows_pointer_step_and_batch(ctx, orc, plp):
    """One handle, caller buffers A and B: the cached level-0 TMA descriptor must be re-encoded whenever the buffer, its
    pitch or the batch changes (batch 3 -> 8 on the same buffer reads frames a 3-frame descriptor does not cover)."""
    lib = plp.lib()
    imgs_a, imgs_b = _orb_frames(41), _orb_frames(53)
    B, rows, cols = imgs_a.shape
    orb = plp.OrbExtractor(ctx, rows, cols, max_batch=B)
    out = _OrbOut(plp, ctx, B, orb.capacity)
    d_a, pa = _pitched(ctx, imgs_a, cols)
    d_b, pb = _pitched(ctx, imgs_b, cols)
    d_a2, pa2 = _pitched(ctx, imgs_a, cols + 32, seed=5)
    for tag, ptr, imgs, batch, step in [("A", pa, imgs_a, 8, cols), ("A", pa, imgs_a, 3, cols), ("B", pb, imgs_b, 8, cols),
                                        ("A", pa, imgs_a, 3, cols), ("A", pa, imgs_a, 8, cols),
                                        ("A pitched", pa2, imgs_a, 8, cols + 32), ("A", pa, imgs_a, 8, cols)]:
        names = _kernels_run(ctx, lib, lambda: out.run(orb, ptr, batch, step))
        assert any(k.startswith("blur_tiles_tma_kernel") for k in names), names
        _check_orb(orc, plp, out, imgs[:batch], f"{tag} batch {batch}")
    for d in (d_a, d_b, d_a2):
        d.free()
    out.free()
    orb.close()


# ----------------------------------------------------------------------------------------------------- stereo
@pytest.fixture(scope="module")
def stereo_case(orc):
    """12 rectified 752 x 480 pairs: rendered scenes of different content, then a flat right image (no right
    keypoint), left == right and two unrelated images.  Oracle ORB + stereo results per pair."""
    H, W = 480, 752
    pairs = [synth.make_stereo_pair(60 + 7 * i, H, W, plp=i % 2 == 0)[:2] for i in range(9)]
    tex = synth.make_texture(91, H, W)
    pairs += [(tex, np.full((H, W), 100, np.uint8)), (tex, tex.copy()), (tex, synth.make_texture(92, H, W))]
    left, right = np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs])
    tab = orc.orb_tables(oracle_api.orb_params())
    refs = [orc.stereo_compute(_orb_ref(orc, l), _orb_ref(orc, r), tab["scale_factors"], tab["inv_scale_factors"], BF,
                               BASELINE) for l, r in zip(left, right)]
    return left, right, refs, tab


@pytest.mark.parametrize("pad", [0, 16], ids=["step_eq_cols", "pitched16"])
def test_stereo_batch_dev_matches_oracle(ctx, orc, plp, stereo_case, pad):
    """bench_stereo's layout: the right image's ORB on a second context, the left on the first, then the batched
    stereo matcher.  The extractors' max_batch is larger than the batch; level 0 is read from the caller's buffer."""
    from plpslam_b200.tracking import DeviceBuffer
    left, right, refs, tab = stereo_case
    N, H, W = left.shape
    step = W + pad
    lib = plp.lib()
    ctx_r = plp.Context(ctx.device)
    el, er = plp.OrbExtractor(ctx, H, W, max_batch=N + 4), plp.OrbExtractor(ctx_r, H, W, max_batch=N + 4)
    cap = el.capacity
    d_l, p_l = _pitched(ctx, left, step, seed=1)
    d_r, p_r = _pitched(ctx_r, right, step, seed=2)
    out_l, out_r = _OrbOut(plp, ctx, N, cap), _OrbOut(plp, ctx, N, cap)
    d_xr, d_dp, d_br = DeviceBuffer(ctx, N * cap * 4), DeviceBuffer(ctx, N * cap * 4), DeviceBuffer(ctx, N * cap * 4)
    out_r.run(er, p_r, N, step)
    out_l.run(el, p_l, N, step)
    ctx.wait(ctx_r)
    ctx._check(lib.plp_stereo_compute_batch_dev(ctx.handle, el.handle, er.handle, C.c_int(N), out_l.kp.ptr, out_l.desc.ptr,
                                                out_l.n.ptr, out_r.kp.ptr, out_r.desc.ptr, out_r.n.ptr, C.c_float(BF),
                                                C.c_float(BASELINE), d_xr.ptr, d_dp.ptr, d_br.ptr))
    xr = d_xr.download(np.float32, (N, cap))
    dp = d_dp.download(np.float32, (N, cap))
    br = d_br.download(np.int32, (N, cap))
    n_l = _check_orb(orc, plp, out_l, left, "left")
    n_r = _check_orb(orc, plp, out_r, right, "right")
    assert n_r[9] == 0 and len(np.unique(n_l)) > 3 and len(np.unique(n_r)) > 3
    n_ok = []
    assert np.array_equal(el.scale_factors, tab["scale_factors"])
    assert np.array_equal(el.inv_scale_factors, tab["inv_scale_factors"])
    for b in range(N):
        ox, od, ob = refs[b]
        k = n_l[b]
        assert np.array_equal(br[b, :k], ob), f"frame {b}: Hamming-closest right keypoint"
        assert np.array_equal(xr[b, :k], ox, equal_nan=True), f"frame {b}: stereo_x_right"
        assert np.array_equal(dp[b, :k], od, equal_nan=True), f"frame {b}: depths"
        n_ok.append(int((ox >= 0).sum()))
    assert n_ok[9] == 0 and n_ok[10] > 300 and min(n_ok[:9]) > 100, n_ok
    for d in (d_l, d_r, d_xr, d_dp, d_br):
        d.free()
    out_l.free()
    out_r.free()
    el.close()
    er.close()
    ctx_r.close()


def test_stereo_batch_dev_rejects_frames_beyond_last_extraction(ctx, plp):
    """A batch larger than either extractor's last batch would read stale pyramid frames: rejected on the host, no
    kernel launched."""
    from plpslam_b200.tracking import DeviceBuffer
    lib = plp.lib()
    H, W = 480, 752
    el, er = plp.OrbExtractor(ctx, H, W, max_batch=8), plp.OrbExtractor(ctx, H, W, max_batch=8)
    imgs = np.stack([synth.make_texture(5 + i, H, W) for i in range(3)])
    el.extract_batch(imgs)
    er.extract_batch(imgs[:2])
    cap = el.capacity
    bufs = [DeviceBuffer(ctx, 8 * cap * 64) for _ in range(8)]
    kl, dl, nl, kr, dr, nr, xr, dp = [b.ptr for b in bufs]
    for batch in (3, 4, 8):   # right ran 2 frames, left 3
        n0 = ctx.launch_count()
        with pytest.raises(plp.PlpError, match="last extraction"):
            ctx._check(lib.plp_stereo_compute_batch_dev(ctx.handle, el.handle, er.handle, C.c_int(batch), kl, dl, nl, kr, dr,
                                                        nr, C.c_float(BF), C.c_float(BASELINE), xr, dp, None))
        assert ctx.launch_count() == n0
    for b in bufs:
        b.free()
    el.close()
    er.close()


# ----------------------------------------------------------------------------------------------------- lines
def test_line_batch_dev_automatic_kernel_choice(ctx, orc, plp):
    """plp_line_extract_batch_dev with caller buffers, an odd pitch and a caller status array, at batches where the
    automatic mode picks each region-growing kernel in turn: the multi-warp kernel for at most half a wave of frames,
    the shared-memory image kernel up to half of what stays resident (two frames per SM at 640 x 480), the L2 image
    kernel above (the benchmark's 12 frames per SM).  A live frame through the host entry point takes the out-of-order
    kernel, the fastest for one frame."""
    from plpslam_b200.tracking import DeviceBuffer
    lib = plp.lib()
    sm = _sm_count(ctx.device)
    cases = [(sm // 2, "lsd_grow_mw_kernel"), (sm // 2 + 1, "lsd_grow_kernel<true>"), (12 * sm, "lsd_grow_kernel<false>")]
    grow = {name for _, name in cases} | {"lsd_grow_ooo_kernel"}
    max_b = cases[-1][0]
    rows, cols = 480, 640
    step = cols + 13
    frames = _bench().build_line_frames(max_b, 1234)
    trk = plp.LineFeatureTracker(ctx, rows, cols, max_batch=max_b)
    cap = trk.capacity
    d_img, ptr = _pitched(ctx, frames, step, seed=9)
    d_kl = DeviceBuffer(ctx, max_b * cap * plp.KEYLINE_DTYPE.itemsize)
    d_lbd, d_fn = DeviceBuffer(ctx, max_b * cap * 32), DeviceBuffer(ctx, max_b * cap * 24)
    d_n = DeviceBuffer(ctx, max_b * 4)
    for batch, want in cases:
        d_st = DeviceBuffer.from_array(ctx, np.full(batch, -1, np.int32))
        names = _kernels_run(ctx, lib, lambda: ctx._check(lib.plp_line_extract_batch_dev(
            trk.handle, ptr, C.c_int(batch), C.c_size_t(step), d_kl.ptr, d_lbd.ptr, d_fn.ptr, d_n.ptr, d_st.ptr)))
        assert names & grow == {want}, (batch, names)
        assert not d_st.download(np.int32, (batch,)).any()
        n = d_n.download(np.int32, (batch,))
        kl = d_kl.download(plp.KEYLINE_DTYPE, (batch, cap))
        lbd = d_lbd.download(np.uint8, (batch, cap, 32))
        fn = d_fn.download(np.float64, (batch, cap, 3))
        rng = np.random.default_rng(batch)
        pick = sorted({0, batch - 1} | set(rng.choice(batch, min(batch, 22), replace=False).tolist()))
        for b in pick:
            _compare_lines(trk, orc, frames[b], b=b, got=(kl[b, :n[b]], lbd[b, :n[b]], fn[b, :n[b]]))
        assert n.min() > 40
        d_st.free()
    live = []
    names = _kernels_run(ctx, lib, lambda: live.append(trk.extract_LSD_LBD(frames[0])))
    assert names & grow == {"lsd_grow_ooo_kernel"}, names
    _compare_lines(trk, orc, frames[0], got=live[0])
    for d in (d_img, d_kl, d_lbd, d_fn, d_n):
        d.free()
    trk.close()


# ----------------------------------------------------------------------------------------------------- pose optimiser
def _pose_dev(ctx, plp, cam, T_in, pts_list, lines_list, cfg):
    """plp_pose_optimize_batch_dev on caller buffers; every output starts as garbage so that the call must write it."""
    from plpslam_b200.tracking import DeviceBuffer
    B = len(pts_list)
    pts = np.concatenate([np.asarray(p, plp.PT_OBS_DTYPE) for p in pts_list])
    lines = np.concatenate([np.asarray(l, plp.LINE_OBS_DTYPE) for l in lines_list])
    po = np.concatenate([[0], np.cumsum([len(p) for p in pts_list])]).astype(np.int32)
    lo = np.concatenate([[0], np.cumsum([len(l) for l in lines_list])]).astype(np.int32)
    max_edges = int(max(np.diff(po) + np.diff(lo)))
    ins = [DeviceBuffer.from_array(ctx, a) for a in (np.asarray(T_in, np.float64), pts, po, lines, lo)]
    outs = [DeviceBuffer.from_array(ctx, a) for a in (np.full((B, 4, 4), np.nan), np.full(len(pts), 0xAB, np.uint8),
                                                      np.full(len(lines), 0xAB, np.uint8), np.full(B, -7, np.int32),
                                                      np.full(B, -7, np.int32))]
    ctx._check(plp.lib().plp_pose_optimize_batch_dev(ctx.handle, C.byref(cam), C.c_int(B), *[d.ptr for d in ins],
                                                     C.c_int(max_edges), C.byref(cfg), *[d.ptr for d in outs]))
    T = outs[0].download(np.float64, (B, 4, 4))
    pout = outs[1].download(np.uint8, (len(pts),))
    lout = outs[2].download(np.uint8, (len(lines),))
    ninl = outs[3].download(np.int32, (B,))
    iters = outs[4].download(np.int32, (B,))
    for d in ins + outs:
        d.free()
    return (T, [pout[po[b]:po[b + 1]] for b in range(B)], [lout[lo[b]:lo[b + 1]] for b in range(B)], ninl, iters)




def _check_pose_batch(orc, cam, scenes, got, tag, rel_tol=1e-8):
    """Pose, outlier flags and inlier count of every frame; returns the oracle's LM iteration counts."""
    T, pout, lout, ninl, iters = got
    want_iters = []
    for b, (T_init, pts, lines) in enumerate(scenes):
        To, po, lo, no, io = orc.pose_optimize(cam, T_init, pts, lines if len(lines) else None, 4, 10)
        rel = np.linalg.norm(T[b] - To) / np.linalg.norm(To)
        assert rel < rel_tol, f"{tag} frame {b}: pose {rel}"
        assert np.array_equal(pout[b], po), f"{tag} frame {b}: point outlier flags"
        if len(lines):
            assert np.array_equal(lout[b], lo), f"{tag} frame {b}: line outlier flags"
        assert ninl[b] == no, f"{tag} frame {b}: n_inliers {ninl[b]} vs {no}"
        want_iters.append(io)
    return want_iters


def test_pose_opt_config3_batch_dev(ctx, orc, plp):
    """bench_pose_opt_config3's inputs (264 frames, scene b % 37, 1000 point + 200 line edges, 4 x 10 LM iterations):
    pose, flags, inlier count and the LM iteration count behind the "LM iterations/s" figure, frame by frame."""
    cam = plp.capi.make_camera(synth.FX, synth.FY, synth.CX, synth.CY, synth.COLS, synth.ROWS)
    batch, n_base = 264, 37
    base = [synth.make_pose_opt_scene(s, n_pts=1000, n_lines=200)[1:] for s in range(n_base)]
    scenes = [base[b % n_base] for b in range(batch)]
    got = _pose_dev(ctx, plp, cam, [s[0] for s in scenes], [s[1] for s in scenes], [s[2] for s in scenes],
                    plp.capi.PoseOptCfg(4, 10))
    # frames with the same scene got identical inputs: one oracle solve per scene, compared with every copy
    want = np.zeros(batch, np.int64)
    for s in range(n_base):
        idx = list(range(s, batch, n_base))
        want[idx] = _check_pose_batch(orc, cam, [base[s]] * len(idx), tuple([g[i] for i in idx] for g in got), f"scene {s}")
    g = got[4]
    print(f"[config3] LM iterations: kernel {g.sum()}, oracle {want.sum()}, frames equal {(g == want).mean():.3f}, "
          f"max |diff| {np.abs(g - want).max()}")
    scene.check_lm_iters(g, want, "config 3")


def test_pose_opt_batch_dev_uneven_edge_counts(ctx, orc, plp):
    cam = plp.capi.make_camera(synth.FX, synth.FY, synth.CX, synth.CY, synth.COLS, synth.ROWS)
    sizes = [(1000, 200), (317, 0), (4, 0), (600, 37), (50, 200), (4, 12), (6, 0), (1500, 5), (5, 1), (90, 0)]
    scenes = [synth.make_pose_opt_scene(300 + i, n_pts=p, n_lines=l, outlier_frac=0.15 + 0.03 * (i % 4))[1:]
              for i, (p, l) in enumerate(sizes)]
    got = _pose_dev(ctx, plp, cam, [s[0] for s in scenes], [s[1] for s in scenes], [s[2] for s in scenes],
                    plp.capi.PoseOptCfg(4, 10))
    # frames of 5 or 6 observations are poorly conditioned: the pose agrees to ~1e-7 there
    want = _check_pose_batch(orc, cam, scenes, got, "uneven", rel_tol=1e-6)
    scene.check_lm_iters(got[4], want, "uneven")
    assert got[4][2] == 0 and got[3][2] == 0 and np.array_equal(got[0][2], scenes[2][0])   # < 5 points: untouched


# ----------------------------------------------------------------------------------------------------- front end
def test_front_end_two_streams_no_host_sync(ctx, orc, plp):
    """bench.py's headline layout: two FrontEnds, each with its own extraction context and a high-priority tracking
    context, 4 end-to-end steps (upload_inputs_async -> step -> download_outputs_async) with no host synchronisation in
    between.  Consecutive steps alternate between two input sets (the same problems in rotated order), so a missing
    cross-stream dependency reads the other step's data.  Every step's host results must equal the oracle chain."""
    from plpslam_b200.tracking import PinnedBuffer
    bench = _bench()
    Bs, S, K = 6, 2, 4
    perms = [np.arange(Bs), np.roll(np.arange(Bs), 1)]
    fes, sets, outs, problems = [], [], [], []
    ctxs = [ctx, plp.Context(ctx.device)]
    tctxs = [plp.Context(ctx.device, high_priority=True) for _ in range(S)]
    for c in range(S):
        fe, frames, aux = bench.setup_front_end(plp, ctxs[c], Bs, 777 + 37 * c, tctxs[c])
        seqs, t_idx = aux["seqs"], aux["t_idx"]
        problems.append([(seqs[s], {t - 1: _orb_ref(orc, seqs[s].frames[t - 1]), t: _orb_ref(orc, seqs[s].frames[t])}, t,
                          aux["preds"][b]) for b, (s, t) in enumerate(t_idx)])
        # two pinned input sets of equal sizes: the first staged by setup_front_end, the second its rotation.  The
        # FrontEnd frees what it staged before whenever it stages again, so each set is taken out of its hands.
        last_pinned = [fe._last_pinned]
        fe._last_pinned = []
        p = perms[1]
        fe.set_last_frames([aux["lasts"][i] for i in p], aux["preds"][p],
                           np.stack([seqs[t_idx[i][0]].poses[t_idx[i][1] - 1] for i in p]))
        last_pinned.append(fe._last_pinned)
        fe._last_pinned = []
        pin_imgs, blocks = [], []
        for p in perms:
            fe.stage_host_io(frames[p])
            pin_imgs.append(fe._pin_imgs)
            blocks.append(fe._pin_out)
            fe._pin_imgs, fe._pin_out = None, None
        blocks += [PinnedBuffer(ctxs[c], blocks[0].nbytes) for _ in range(K - 2)]   # one result block per step
        fes.append(fe)
        sets.append(list(zip(pin_imgs, last_pinned)))
        outs.append(blocks)
    for k in range(K):
        for c, fe in enumerate(fes):
            fe._pin_imgs, fe._last_pinned = sets[c][k % 2]
            fe._pin_out = outs[c][k]
            fe.upload_inputs_async()
            fe.step(Bs)
            fe.download_outputs_async()
    # FrontEnd.download_tracking straight after step(), without a barrier: it orders itself after the tracking stream
    direct = []
    for fe in fes:
        fe.step(Bs)
        direct.append(fe.download_tracking(Bs))
    for cx in ctxs + tctxs:
        cx.sync()
    for c, fe in enumerate(fes):
        oracle = [_oracle_track(orc, plp, seq, res, t, pred) for seq, res, t, pred in problems[c]]
        for k in range(K):
            fe._pin_out = outs[c][k]
            hr = fe.host_results()
            perm = perms[k % 2]
            for b in range(Bs):
                m, T, nv, n_inl, iters = oracle[perm[b]]
                _, res, t, _ = problems[c][perm[b]]
                n = hr["n_kp"][b]
                what = f"front end {c} step {k} frame {b}"
                assert np.array_equal(hr["kp"][b, :n], res[t]["kps"]), what
                assert np.array_equal(hr["desc"][b, :n], res[t]["desc"]), what
                assert np.array_equal(hr["matched"][b, :n], m), what
                assert hr["num_valid"][b] == nv and hr["n_inliers"][b] == n_inl, what
                assert np.linalg.norm(hr["pose"][b] - T) / np.linalg.norm(T) < 1e-4, what
                assert hr["status"][b] == 0 and nv >= 20, what
            scene.check_lm_iters(hr["lm_iters"], [oracle[i][4] for i in perm], f"front end {c} step {k}")
        # the direct download saw the input set of the last end-to-end step
        perm = perms[(K - 1) % 2]
        d = direct[c]
        for b in range(Bs):
            m, T, nv, n_inl, iters = oracle[perm[b]]
            assert np.array_equal(d["matched"][b], m) and d["num_valid"][b] == nv, b
            assert np.linalg.norm(d["pose"][b] - T) / np.linalg.norm(T) < 1e-4, b
        scene.check_lm_iters(d["lm_iters"], [oracle[i][4] for i in perm], f"front end {c} direct download")
    for c, fe in enumerate(fes):
        for pin_imgs, last_pinned in sets[c]:
            pin_imgs.free()
            for b in last_pinned:
                b.free()
        for b in outs[c]:
            b.free()
        fe._pin_imgs, fe._last_pinned, fe._pin_out = None, [], None
        fe.close()
    for cx in ctxs[1:] + tctxs:
        cx.close()


# ----------------------------------------------------------------------------------------------------- DBoW2
def test_bow_transform_dev(ctx, orc, plp):
    """plp_bow_transform_dev on the batched front end's layout: rows = frames x capacity, rows past a frame's keypoint
    count carry whatever the buffer held (computed, ignored by the caller) -- compared row by row with the oracle."""
    from plpslam_b200.tracking import DeviceBuffer
    k, L, levelsup = 10, 4, 2
    vocab = bow_data.make_vocab(1004, k=k, L=L)
    rng = np.random.default_rng(17)
    leaves = vocab["desc"][vocab["is_leaf"] > 0]
    n = 3 * 1100 + 7
    desc = np.concatenate([synth.rand_desc(rng, 500),
                           synth.flip_bits(rng, leaves[rng.integers(0, len(leaves), n - 500)], rng.integers(0, 30, n - 500))])
    gv = plp.BowVocabulary(ctx, k=k, L=L, parent=vocab["parent"], desc=vocab["desc"], weight=vocab["weight"],
                           is_leaf=vocab["is_leaf"])
    ov = orc.bow_vocab_create(k, L, vocab["parent"], vocab["desc"], vocab["weight"], vocab["is_leaf"])
    want = orc.bow_transform(ov, desc, levelsup)
    d_desc = DeviceBuffer.from_array(ctx, desc)
    outs = [DeviceBuffer.from_array(ctx, np.full(n, -3, dt)) for dt in (np.int32, np.int32, np.float32)]
    ctx._check(plp.lib().plp_bow_transform_dev(gv._h, d_desc.ptr, C.c_int(n), C.c_int(levelsup), *[d.ptr for d in outs]))
    got = [d.download(dt, (n,)) for d, dt in zip(outs, (np.int32, np.int32, np.float32))]
    for g, w, name in zip(got, want, ("word id", "node id", "weight")):
        assert np.array_equal(g, w), name
    assert (want[2] == 0).any() and (want[2] > 0).any()
    for d in [d_desc] + outs:
        d.free()
    gv.close()
    orc.bow_vocab_destroy(ov)
