"""Device-resident batched front-end: ORB extraction (+ the right image's and match::stereo::compute for a stereo camera)
+ motion-based tracking (+ optionally the keyframe and robust trackers and the local-map stage) without leaving HBM.

Thin ctypes layer over plp_orb_extract_batch_dev + plp_tracker_motion_track_batch_dev (+
plp_tracker_keyframe_track_batch_dev, plp_tracker_robust_track_batch_dev, plp_tracker_update_local_map_batch_dev,
plp_tracker_local_map_track_batch_dev); used
by bench.py and the pipeline parity
tests.  No compute here.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from .capi import (KP_DTYPE, Context, OrbExtractor, PlpError, _P, make_camera, make_distorted_camera,  # noqa: F401
                   make_grid)


class TrackLast(C.Structure):
    _fields_ = [("pos_w", _P), ("octave", _P), ("angle", _P), ("desc", _P), ("valid", _P), ("offsets", _P),
                ("pose_pred", _P), ("pose_last", _P)]


class TrackLocal(C.Structure):
    _fields_ = [("pos_w", _P), ("obs_mean_normal", _P), ("min_valid_dist", _P), ("max_valid_dist", _P),
                ("max_valid_dist_raw", _P), ("desc", _P), ("valid", _P), ("offsets", _P), ("last_local_idx", _P)]


class TrackKeyframe(C.Structure):
    _fields_ = [("num_keyframes", C.c_int32), ("kf_of_frame", _P), ("row_offsets", _P), ("desc", _P), ("angle", _P),
                ("valid", _P), ("pos_w", _P), ("fv_offsets", _P), ("node_ids", _P), ("node_begin", _P), ("indices", _P),
                ("local_idx", _P), ("local_idx_offsets", _P)]


class TrackMap(C.Structure):
    _fields_ = [(f, _P) for f in ("pos_w", "obs_mean_normal", "min_valid_dist", "max_valid_dist", "max_valid_dist_raw",
                                  "desc", "lm_erased", "obs_offsets", "obs_kf", "kf_erased", "row_offsets", "row_lm",
                                  "cov_offsets", "cov_kf", "child_offsets", "child_kf", "parent", "last_row_lm",
                                  "kf_row_lm")]


def _logf(x: float) -> float:
    """The C library's logf: frame::log_scale_factor_ = std::log(scale_factor_) on a float."""
    libm = C.CDLL("libm.so.6")
    libm.logf.restype = C.c_float
    libm.logf.argtypes = [C.c_float]
    return float(libm.logf(float(np.float32(x))))


class _Packed:
    """Per-item arrays end to end, as the C ABI takes a ragged list (one item per frame or keyframe): item i's rows are
    [offsets[i], offsets[i + 1]), and `count` is the key whose length gives an item's rows."""

    def __init__(self, items, count: str):
        self.items = items
        self.offsets = np.zeros(len(items) + 1, np.int32)
        self.offsets[1:] = np.cumsum([len(it[count]) for it in items])

    def cat(self, key: str, dtype, shape=(), fill=None) -> np.ndarray:
        """The items' `key` arrays (rows of `shape`) end to end; with `fill`, an item whose `key` is missing or None
        contributes its rows of that value."""
        parts = [np.full(n, fill, dtype) if fill is not None and it.get(key) is None else
                 np.asarray(it[key], dtype).reshape((-1,) + shape) for it, n in zip(self.items, np.diff(self.offsets))]
        return np.ascontiguousarray(np.concatenate(parts) if parts else np.zeros((0,) + shape, dtype))


def _by_frame(n, a: np.ndarray) -> list:
    """Frame b's first n[b] rows of a (frames x ...) array, for every frame b < len(n)."""
    return [a[b, :n[b]].copy() for b in range(len(n))]


def _unpack(offsets, a: np.ndarray) -> list:
    """Item i's rows [offsets[i], offsets[i + 1]) of a packed array, for every i < len(offsets) - 1."""
    return [a[offsets[i]:offsets[i + 1]].copy() for i in range(len(offsets) - 1)]


class DeviceBuffer:
    """A cudaMalloc'ed block owned through the C ABI (plp_dev_alloc / plp_dev_free)."""

    def __init__(self, ctx: Context, nbytes: int):
        self._ctx = ctx
        self.nbytes = int(nbytes)
        p = C.c_void_p()
        ctx._check(ctx._lib.plp_dev_alloc(ctx.handle, C.c_size_t(max(self.nbytes, 1)), C.byref(p)))
        self.ptr = p

    @classmethod
    def from_array(cls, ctx: Context, arr: np.ndarray) -> "DeviceBuffer":
        arr = np.ascontiguousarray(arr)
        buf = cls(ctx, arr.nbytes)
        buf.upload(arr)
        return buf

    def upload(self, arr: np.ndarray):
        arr = np.ascontiguousarray(arr)
        assert arr.nbytes <= self.nbytes
        self._ctx._check(self._ctx._lib.plp_dev_upload(self._ctx.handle, self.ptr, arr.ctypes.data_as(_P),
                                                       C.c_size_t(arr.nbytes)))

    def download(self, dtype, shape) -> np.ndarray:
        out = np.zeros(shape, dtype)
        assert out.nbytes <= self.nbytes
        self._ctx._check(self._ctx._lib.plp_dev_download(self._ctx.handle, out.ctypes.data_as(_P), self.ptr,
                                                         C.c_size_t(out.nbytes)))
        return out

    def free(self):
        if self.ptr is not None:
            self._ctx._lib.plp_dev_free(self._ctx.handle, self.ptr)
            self.ptr = None


class PinnedBuffer:
    """Page-locked host memory owned through the C ABI (plp_host_alloc_pinned): the source / destination of the
    asynchronous copies of the end-to-end path."""

    def __init__(self, ctx: Context, nbytes: int):
        self._lib = ctx._lib
        self.nbytes = int(nbytes)
        p = C.c_void_p()
        ctx._check(self._lib.plp_host_alloc_pinned(C.c_size_t(max(self.nbytes, 1)), C.byref(p)))
        self.ptr = p

    @classmethod
    def from_array(cls, ctx: Context, arr: np.ndarray) -> "PinnedBuffer":
        arr = np.ascontiguousarray(arr)
        buf = cls(ctx, arr.nbytes)
        C.memmove(buf.ptr, arr.ctypes.data, arr.nbytes)
        return buf

    def view(self, dtype, shape, offset: int = 0) -> np.ndarray:
        n = int(np.prod(shape)) * np.dtype(dtype).itemsize
        assert offset + n <= self.nbytes
        raw = (C.c_char * n).from_address(self.ptr.value + offset)
        return np.frombuffer(raw, dtype).reshape(shape)

    def free(self):
        if self.ptr is not None:
            self._lib.plp_host_free_pinned(self.ptr)
            self.ptr = None


class FrontEnd:
    """extract (orb_extractor::extract) -> motion_based_track for a batch of frames, all on the device."""

    def __init__(self, ctx: Context, rows: int, cols: int, cam, max_batch: int, max_last_points: int = 4096,
                 max_num_keypts=1000, scale_factor=1.2, num_levels=8, ini_fast_thr=20, min_fast_thr=7,
                 track_ctx: Context | None = None, distortion=None, right_ctx: Context | None = None):
        """track_ctx: optional second context (stream) for the tracking kernels; extraction stays on `ctx`.  The two
        streams are chained by plp_ctx_wait_ctx, so extract(k + 1) of ANOTHER FrontEnd can run under track(k).
        distortion: a capi.Distortion (make_distortion); the tracker then undistorts the keypoints before matching, and
        cam's bounds and the grid come from the undistorted image corners (capi.make_distorted_camera).  None: the
        camera has no distortion.
        A stereo camera (cam.setup_type 1, rectified pairs) adds a second extractor for the right images and the
        stereo_x_right_ / depths_ buffers that extract() fills with match::stereo::compute; the tracker reads x_right.
        right_ctx: optional context (stream) for the right image's ORB pass, which then runs beside the left one."""
        self.ctx = ctx
        self.track_ctx = track_ctx if track_ctx is not None else ctx
        self.lib = ctx._lib
        self.rows, self.cols, self.max_batch = rows, cols, max_batch
        self.distortion = distortion
        if distortion is not None:
            cam, self.grid = make_distorted_camera(cam.fx, cam.fy, cam.cx, cam.cy, cols, rows, distortion)
        else:
            self.grid = make_grid(cols, rows)
        self.cam = cam
        self.orb = OrbExtractor(ctx, rows, cols, max_num_keypts, scale_factor, num_levels, ini_fast_thr, min_fast_thr,
                                max_batch=max_batch)
        self.cap = self.orb.capacity
        self.max_last = max_last_points
        h = C.c_void_p()
        sf = np.ascontiguousarray(self.orb.scale_factors, np.float32)
        isig = np.ascontiguousarray(self.orb.inv_level_sigma_sq, np.float32)
        ctx._check(self.lib.plp_tracker_create_ex(self.track_ctx.handle, C.byref(cam), C.byref(self.grid),
                                                  sf.ctypes.data_as(_P), isig.ctypes.data_as(_P), C.c_int(num_levels),
                                                  C.c_int(max_batch), C.c_int(self.cap), C.c_int(max_last_points),
                                                  None if distortion is None else C.byref(distortion), C.byref(h)))
        self._trk = h
        self.stereo = cam.setup_type == 1
        self.orb_right = None
        self._stereo_out = None
        if self.stereo:
            self.right_ctx = right_ctx if right_ctx is not None else ctx
            self.orb_right = OrbExtractor(self.right_ctx, rows, cols, max_num_keypts, scale_factor, num_levels,
                                          ini_fast_thr, min_fast_thr, max_batch=max_batch)
            self._stereo_out = self._frame_buffers(imgs_right=rows * cols, kp_right=self.cap * KP_DTYPE.itemsize,
                                                   desc_right=self.cap * 32, n_kp_right=4, status_right=4,
                                                   x_right=self.cap * 4, depths=self.cap * 4)
            self.d_x_right = self._stereo_out["x_right"]
            ctx._check(self.lib.plp_tracker_bind_stereo(self._trk, self.d_x_right.ptr))
        self._motion_out = self._frame_buffers(imgs=rows * cols, kp=self.cap * KP_DTYPE.itemsize, desc=self.cap * 32,
                                               n_kp=4, status=4, matched=self.cap * 4, pose=128, num_valid=4,
                                               n_inliers=4, lm_iters=4)
        (self.d_imgs, self.d_kp, self.d_desc, self.d_n, self.d_status, self.d_matched, self.d_pose, self.d_num_valid,
         self.d_n_inl, self.d_lm) = self._motion_out.values()
        self.scale_factor = scale_factor
        self._local_bufs = []
        self._local = None
        self._local_out = None
        self._kf_bufs = []
        self._kf = None
        self._kf_out = None
        self._kf_bearings = None
        self._rb_out = None
        self._upd_out = None
        self._map_bufs = []
        self._map = None
        self._local_from_update = False
        self._last_bufs = []
        self._last = None
        self._last_pinned = []   # host copies of the last-frame arrays (end-to-end path: uploaded every step)
        self._pin_imgs = None
        self._pin_out = None
        self._out_layout = None

    def _frame_buffers(self, **frame_bytes) -> dict:
        """One device buffer of max_batch x `frame_bytes[name]` bytes per name; close() frees them."""
        return {name: DeviceBuffer(self.ctx, self.max_batch * n) for name, n in frame_bytes.items()}

    def close(self):
        """Frees the tracker and every device and pinned buffer this FrontEnd still holds; a buffer a caller has taken
        out of its hands (by replacing the attribute) is the caller's.  A second call does nothing."""
        outs = [o for o in (self._motion_out, self._local_out, self._kf_out, self._rb_out, self._upd_out,
                            self._stereo_out) if o]
        for b in ([b for o in outs for b in o.values()] + self._last_bufs + self._last_pinned + self._local_bufs +
                  self._kf_bufs + self._map_bufs + [self._pin_imgs, self._pin_out]):
            if b is not None:
                b.free()
        if self._trk is not None:
            self.lib.plp_tracker_destroy(self._trk)
            self._trk = None
        self.orb.close()
        if self.orb_right is not None:
            self.orb_right.close()
            self.orb_right = None

    # -- inputs ---------------------------------------------------------------------------------------
    def upload_images(self, imgs: np.ndarray, right: np.ndarray | None = None):
        """imgs: the (left) images; right: the right images of a stereo FrontEnd, required there."""
        if self.stereo != (right is not None):
            raise PlpError("a stereo FrontEnd takes left and right images, a monocular one left images only")
        self.d_imgs.upload(np.ascontiguousarray(imgs, np.uint8))
        if right is not None:
            self._stereo_out["imgs_right"].upload(np.ascontiguousarray(right, np.uint8))

    def set_last_frames(self, last_list, pose_pred, pose_last):
        """last_list[b]: dict(pos_w[m,3], octave[m], angle[m], desc[m,32], valid[m]|None)."""
        for b in self._last_bufs:
            b.free()
        last = _Packed(last_list, "octave")
        offs = last.offsets
        assert max(np.diff(offs)) <= self.max_last
        arrays = [last.cat("pos_w", np.float64, (3,)), last.cat("octave", np.int32), last.cat("angle", np.float32),
                  last.cat("desc", np.uint8, (32,)), last.cat("valid", np.uint8, fill=1), offs,
                  np.ascontiguousarray(pose_pred, np.float64), np.ascontiguousarray(pose_last, np.float64)]
        self._last_bufs = [DeviceBuffer.from_array(self.ctx, a) for a in arrays]
        self._last = TrackLast(*[b.ptr for b in self._last_bufs])
        self._last_offsets = offs
        for b in self._last_pinned:
            b.free()
        self._last_pinned = [PinnedBuffer.from_array(self.ctx, a) for a in arrays]

    def reserve_local_map(self, max_local_points: int):
        """Scratch for local maps of up to max_local_points landmarks per frame (outside the hot path), and the
        outputs of track_local_map."""
        self.ctx._check(self.lib.plp_tracker_reserve_local_map(self._trk, C.c_float(_logf(self.scale_factor)),
                                                           C.c_int(max_local_points)))
        self.max_local = int(max_local_points)
        if self._local_out is None:
            self._local_out = self._frame_buffers(matched=self.cap * 4, local=self.cap * 4, pose=128, num_tracked=4,
                                                  n_inliers=4, lm_iters=4, status=4)

    def set_local_maps(self, local_list):
        """local_list[b]: dict(pos_w[m,3], normal[m,3] (get_obs_mean_normal), min_valid_dist[m], max_valid_dist[m]
        (get_min/max_valid_distance), max_valid_dist_raw[m] (max_valid_dist_), desc[m,32], valid[m]|None
        (!will_be_erased), last_local_idx[rows of frame b in set_last_frames] (-1: not in the local list)), in
        local_landmarks_ order."""
        for b in self._local_bufs:
            b.free()
        loc = _Packed(local_list, "max_valid_dist")
        offs = loc.offsets
        arrays = [loc.cat("pos_w", np.float64, (3,)), loc.cat("normal", np.float64, (3,)),
                  loc.cat("min_valid_dist", np.float32), loc.cat("max_valid_dist", np.float32),
                  loc.cat("max_valid_dist_raw", np.float32), loc.cat("desc", np.uint8, (32,)),
                  loc.cat("valid", np.uint8, fill=1), offs, loc.cat("last_local_idx", np.int32)]
        self._local_bufs = [DeviceBuffer.from_array(self.ctx, a) for a in arrays]
        self._local = TrackLocal(*[b.ptr for b in self._local_bufs])
        self._local_offsets = offs
        self._d_observable = DeviceBuffer(self.ctx, max(int(offs[-1]), 1))
        self._local_bufs.append(self._d_observable)

    def reserve_keyframe_track(self, max_keyframes: int, max_keyframe_points: int):
        """Scratch for keyframe tables of up to max_keyframes keyframes of up to max_keyframe_points rows (outside the
        hot path), and the outputs of track_keyframe."""
        self.ctx._check(self.lib.plp_tracker_reserve_keyframe_track(self._trk, C.c_int(max_keyframes),
                                                                    C.c_int(max_keyframe_points)))
        if self._kf_out is None:
            self._kf_out = self._frame_buffers(stage=4, matched=self.cap * 4, num_bow=4, pose=128, num_valid=4,
                                               n_inliers=4, lm_iters=4, status=4, motion_valid=1)

    def set_keyframes(self, keyframes, kf_of_frame, local_idx=None):
        """keyframes[k]: dict(desc[n,32], angle[n] (keypts_[i].angle), valid[n]|None (lm && !will_be_erased()),
        pos_w[n,3], fv=(node_ids, offsets, indices) (bow_feat_vec_ flattened, as capi.fold_bow returns it),
        bearings[n,3] (keyfrm->bearings_; optional, read by track_robust only));
        kf_of_frame[b]: frame b's reference keyframe.  local_idx (optional, for track_local_map after track_keyframe):
        per frame, one entry per row of its keyframe -- that landmark's index in the frame's local list, or -1."""
        for b in self._kf_bufs:
            b.free()
        kfs = _Packed(keyframes, "desc")
        fv = _Packed([dict(zip(("node_ids", "node_offsets", "indices"), k["fv"])) for k in keyframes], "node_ids")
        node_begin, base = [], 0
        for f in fv.items:
            node_begin.append(np.asarray(f["node_offsets"][:-1], np.int64) + base)
            base += len(f["indices"])
        node_begin = np.concatenate(node_begin + [np.array([base])]).astype(np.int32)
        arrays = [np.ascontiguousarray(kf_of_frame, np.int32), kfs.offsets, kfs.cat("desc", np.uint8, (32,)),
                  kfs.cat("angle", np.float32), kfs.cat("valid", np.uint8, fill=1), kfs.cat("pos_w", np.float64, (3,)),
                  fv.offsets, fv.cat("node_ids", np.uint32), node_begin, fv.cat("indices", np.uint32)]
        if local_idx is not None:
            li = _Packed([dict(local_idx=x) for x in local_idx], "local_idx")
            arrays += [li.cat("local_idx", np.int32), li.offsets]
        self._kf_bufs = [DeviceBuffer.from_array(self.ctx, a) for a in arrays]
        ptrs = [b.ptr for b in self._kf_bufs] + [None] * (12 - len(self._kf_bufs))
        self._kf = TrackKeyframe(len(keyframes), *ptrs)
        self._kf_bearings = None
        if keyframes and all(k.get("bearings") is not None for k in keyframes):
            self._kf_bearings = DeviceBuffer.from_array(self.ctx, kfs.cat("bearings", np.float64, (3,)))
            self._kf_bufs.append(self._kf_bearings)

    def reserve_robust_track(self):
        """Scratch of track_robust (outside the hot path), and its outputs."""
        self.ctx._check(self.lib.plp_tracker_reserve_robust_track(self._trk))
        if self._rb_out is None:
            self._rb_out = self._frame_buffers(stage=4, matched=self.cap * 4, num_bf=4, num_robust=4, pose=128,
                                               num_valid=4, n_inliers=4, lm_iters=4, status=4)

    def reserve_local_map_update(self, max_local_keyframes: int = 128):
        """Scratch and list of update_local_map (outside the hot path; after reserve_local_map and, where the keyframe
        stage runs, reserve_keyframe_track), and its per-frame outputs."""
        self.ctx._check(self.lib.plp_tracker_reserve_local_map_update(self._trk, C.c_int(max_local_keyframes)))
        self.max_local_keyframes = int(max_local_keyframes)
        for b in (self._upd_out or {}).values():
            b.free()
        self._upd_out = self._frame_buffers(nearest=4, local_kf=max_local_keyframes * 4, num_local_kf=4,
                                            local_lm=self.max_local * 4, status=4, observable=self.max_local)

    def set_map(self, snapshot):
        """The map snapshot update_local_map reads (plp_track_map), keyframes and landmarks by table index:
        snapshot = dict(pos_w[L,3], normal[L,3], min_valid_dist[L], max_valid_dist[L], max_valid_dist_raw[L], desc[L,32],
        lm_erased[L], obs_offsets[L+1], obs_kf, kf_erased[K], row_offsets[K+1], row_lm, cov_offsets[K+1], cov_kf,
        child_offsets[K+1], child_kf, parent[K], last_row_lm (one per set_last_frames row), kf_row_lm (one per
        set_keyframes row; optional without track_keyframe))."""
        for b in self._map_bufs:
            b.free()
        spec = [("pos_w", np.float64), ("normal", np.float64), ("min_valid_dist", np.float32),
                ("max_valid_dist", np.float32), ("max_valid_dist_raw", np.float32), ("desc", np.uint8),
                ("lm_erased", np.uint8), ("obs_offsets", np.int32), ("obs_kf", np.int32), ("kf_erased", np.uint8),
                ("row_offsets", np.int32), ("row_lm", np.int32), ("cov_offsets", np.int32), ("cov_kf", np.int32),
                ("child_offsets", np.int32), ("child_kf", np.int32), ("parent", np.int32), ("last_row_lm", np.int32),
                ("kf_row_lm", np.int32)]
        self._map_bufs, ptrs = [], []
        for key, dt in spec:
            if snapshot.get(key) is None:
                ptrs.append(None)
                continue
            buf = DeviceBuffer.from_array(self.ctx, np.ascontiguousarray(snapshot[key], dt))
            self._map_bufs.append(buf)
            ptrs.append(buf.ptr)
        self._map = TrackMap(*ptrs)

    # -- end-to-end path: every input of a step comes from pinned host memory, every result goes back ----
    def stage_host_io(self, imgs: np.ndarray):
        """Pinned host staging of one step: the images (input) and one block for all results."""
        batch = imgs.shape[0]
        if self._pin_imgs is not None:
            self._pin_imgs.free()
            self._pin_out.free()
        self._pin_imgs = PinnedBuffer.from_array(self.ctx, np.ascontiguousarray(imgs, np.uint8))
        items = [("kp", self.d_kp, batch * self.cap * KP_DTYPE.itemsize), ("desc", self.d_desc, batch * self.cap * 32),
                 ("n_kp", self.d_n, batch * 4), ("status", self.d_status, batch * 4),
                 ("matched", self.d_matched, batch * self.cap * 4), ("pose", self.d_pose, batch * 128),
                 ("num_valid", self.d_num_valid, batch * 4), ("n_inliers", self.d_n_inl, batch * 4),
                 ("lm_iters", self.d_lm, batch * 4)]
        off, layout = 0, []
        for name, dbuf, nbytes in items:
            layout.append((name, dbuf, off, nbytes))
            off += (nbytes + 255) & ~255
        self._pin_out = PinnedBuffer(self.ctx, off)
        self._out_layout = layout
        self._io_batch = batch

    @property
    def h2d_bytes_per_step(self) -> int:
        return self._pin_imgs.nbytes + sum(b.nbytes for b in self._last_pinned)

    @property
    def d2h_bytes_per_step(self) -> int:
        return sum(nb for _, _, _, nb in self._out_layout)

    def upload_inputs_async(self):
        """H2D of this step's images AND of its last-frame landmarks / descriptors / predicted poses (extraction stream).
        The previous step's tracking kernels and result downloads (tracking stream) must have drained first."""
        lib = self.lib
        if self.track_ctx is not self.ctx:
            self.ctx.wait(self.track_ctx)
        self.ctx._check(lib.plp_dev_upload_async(self.ctx.handle, self.d_imgs.ptr, self._pin_imgs.ptr,
                                                 C.c_size_t(self._pin_imgs.nbytes)))
        for dbuf, pbuf in zip(self._last_bufs, self._last_pinned):
            self.ctx._check(lib.plp_dev_upload_async(self.ctx.handle, dbuf.ptr, pbuf.ptr, C.c_size_t(pbuf.nbytes)))

    def download_outputs_async(self):
        """D2H of everything the host-side data::frame needs from this step: keypoints, descriptors, counts, the
        landmark index kept on every keypoint, pose, valid / inlier counts (tracking stream, after track())."""
        cx = self.track_ctx
        for _, dbuf, off, nbytes in self._out_layout:
            cx._check(self.lib.plp_dev_download_async(cx.handle, C.c_void_p(self._pin_out.ptr.value + off), dbuf.ptr,
                                                      C.c_size_t(nbytes)))

    def host_results(self):
        """Views into the pinned result block (valid after the tracking stream has been synchronised)."""
        b, out = self._io_batch, {}
        shapes = {"kp": (KP_DTYPE, (b, self.cap)), "desc": (np.uint8, (b, self.cap, 32)), "n_kp": (np.int32, (b,)),
                  "status": (np.int32, (b,)), "matched": (np.int32, (b, self.cap)), "pose": (np.float64, (b, 4, 4)),
                  "num_valid": (np.int32, (b,)), "n_inliers": (np.int32, (b,)), "lm_iters": (np.int32, (b,))}
        for name, _, off, _ in self._out_layout:
            dt, shp = shapes[name]
            out[name] = self._pin_out.view(dt, shp, off)
        return out

    # -- the hot path (no host synchronisation) ---------------------------------------------------------
    def extract(self, batch: int):
        if self.track_ctx is not self.ctx:
            self.ctx.wait(self.track_ctx)  # the previous track() still reads the keypoint / descriptor arrays
        if self.stereo:  # frame.cc:456-457: the right image's ORB pass
            o, rc = self._stereo_out, self.right_ctx
            if rc is not self.ctx:
                rc.wait(self.ctx)  # the previous stereo match still reads the right keypoints and pyramid
            rc._check(self.lib.plp_orb_extract_batch_dev(self.orb_right.handle, o["imgs_right"].ptr, C.c_int(batch),
                                                         C.c_size_t(self.cols), o["kp_right"].ptr, o["desc_right"].ptr,
                                                         o["n_kp_right"].ptr, o["status_right"].ptr))
        self.ctx._check(self.lib.plp_orb_extract_batch_dev(self.orb.handle, self.d_imgs.ptr, C.c_int(batch),
                                                          C.c_size_t(self.cols), self.d_kp.ptr, self.d_desc.ptr,
                                                          self.d_n.ptr, self.d_status.ptr))
        if self.stereo:  # frame.cc:470-480: stereo_x_right_ and depths_ of the left keypoints
            if rc is not self.ctx:
                self.ctx.wait(rc)
            self.ctx._check(self.lib.plp_stereo_compute_batch_dev(
                self.ctx.handle, self.orb.handle, self.orb_right.handle, C.c_int(batch), self.d_kp.ptr,
                self.d_desc.ptr, self.d_n.ptr, o["kp_right"].ptr, o["desc_right"].ptr, o["n_kp_right"].ptr,
                C.c_float(self.cam.focal_x_baseline), C.c_float(self.cam.true_baseline), o["x_right"].ptr,
                o["depths"].ptr, None))

    def track(self, batch: int, margin: float = 20.0):
        if self.track_ctx is not self.ctx:
            self.track_ctx.wait(self.ctx)  # the extraction of this batch
        self.ctx._check(self.lib.plp_tracker_motion_track_batch_dev(
            self._trk, C.c_int(batch), self.d_kp.ptr, self.d_desc.ptr, self.d_n.ptr, C.byref(self._last),
            C.c_float(margin), self.d_matched.ptr, self.d_pose.ptr, self.d_num_valid.ptr, self.d_n_inl.ptr,
            self.d_lm.ptr))

    def step(self, batch: int, margin: float = 20.0):
        self.extract(batch)
        self.track(batch, margin)

    def track_local_map(self, batch: int, margin: float = 5.0, updated: bool = False):
        """optimize_current_frame_with_local_map for the batch of the preceding track() (tracking stream).  margin:
        5, or 20 for a recently relocalised frame (tracking_module.cc:976-981).  updated: take the list the preceding
        update_local_map() built on the device instead of the one set_local_maps() uploaded."""
        o = self._local_out
        if updated:
            local, observable = self._updated_list(), self._upd_out["observable"]
        else:
            if o is None or self._local is None:
                raise PlpError("track_local_map needs reserve_local_map() and set_local_maps() first")
            local, observable = self._local, self._d_observable
        self.ctx._check(self.lib.plp_tracker_local_map_track_batch_dev(
            self._trk, C.c_int(batch), C.byref(local), C.c_float(margin), o["matched"].ptr, o["local"].ptr,
            observable.ptr, o["pose"].ptr, o["num_tracked"].ptr, o["n_inliers"].ptr, o["lm_iters"].ptr,
            o["status"].ptr))
        self._local_from_update = updated

    def update_local_map(self, batch: int):
        """update_local_map for the batch of the preceding tracking calls, from the set_map() snapshot (tracking
        stream); its list feeds track_local_map(updated=True)."""
        o = self._upd_out
        if o is None or self._map is None:
            raise PlpError("update_local_map needs reserve_local_map_update() and set_map() first")
        self.ctx._check(self.lib.plp_tracker_update_local_map_batch_dev(
            self._trk, C.c_int(batch), C.byref(self._map), o["nearest"].ptr, o["local_kf"].ptr, o["num_local_kf"].ptr,
            o["local_lm"].ptr, o["status"].ptr))

    def track_keyframe(self, batch: int, vocab, motion_valid=None):
        """bow_match_based_track for the frames of the preceding track() whose motion model is not usable
        (motion_valid[b] == 0; None: all usable) or whose motion track failed (tracking stream)."""
        o = self._kf_out
        if o is None or self._kf is None:
            raise PlpError("track_keyframe needs reserve_keyframe_track() and set_keyframes() first")
        mv = None
        if motion_valid is not None:  # on the tracking stream: an earlier call there may still read the buffer
            flags = np.ascontiguousarray(motion_valid, np.uint8)
            assert flags.nbytes <= o["motion_valid"].nbytes
            tc = self.track_ctx
            tc._check(self.lib.plp_dev_upload(tc.handle, o["motion_valid"].ptr, flags.ctypes.data_as(_P),
                                              C.c_size_t(flags.nbytes)))
            mv = o["motion_valid"].ptr
        self.ctx._check(self.lib.plp_tracker_keyframe_track_batch_dev(
            self._trk, vocab.handle, C.c_int(batch), C.byref(self._kf), mv, o["stage"].ptr, o["matched"].ptr,
            o["num_bow"].ptr, o["pose"].ptr, o["num_valid"].ptr, o["n_inliers"].ptr, o["lm_iters"].ptr,
            o["status"].ptr))

    def track_robust(self, batch: int, seed: int = 0):
        """robust_match_based_track for the frames of the preceding track_keyframe() that ran that stage and failed,
        against the same keyframe table (whose keyframes need "bearings"); RANSAC samples drawn on the device from
        `seed` (tracking stream)."""
        o = self._rb_out
        if o is None or self._kf_bearings is None:
            raise PlpError("track_robust needs reserve_robust_track() and set_keyframes() with keyframe bearings first")
        self.ctx._check(self.lib.plp_tracker_robust_track_batch_dev(
            self._trk, C.c_int(batch), self._kf_bearings.ptr, C.c_uint64(seed), o["stage"].ptr, o["matched"].ptr,
            o["num_bf"].ptr, o["num_robust"].ptr, o["pose"].ptr, o["num_valid"].ptr, o["n_inliers"].ptr,
            o["lm_iters"].ptr, o["status"].ptr))

    # -- results --------------------------------------------------------------------------------------
    def _after_tracking(self):
        """The downloads below run on the extraction stream; the tracking outputs are written on the tracking stream."""
        if self.track_ctx is not self.ctx:
            self.ctx.wait(self.track_ctx)

    def _tail_results(self, batch: int, o: dict, valid: str = "num_valid") -> dict:
        """What every tracking call returns per frame, from its outputs `o`: pose, the valid count, n_inliers, LM
        iterations and status."""
        return dict(pose=o["pose"].download(np.float64, (batch, 4, 4)),
                    **{k: o[k].download(np.int32, (batch,)) for k in (valid, "n_inliers", "lm_iters", "status")})

    def _keypoint_rows(self, n, buf: DeviceBuffer, dtype=np.int32) -> list:
        """Per frame b < len(n), the values of its n[b] keypoints in a max_batch x cap buffer."""
        return _by_frame(n, buf.download(dtype, (self.max_batch, self.cap)))

    def _download_ptr(self, p, dtype, shape) -> np.ndarray:
        """An array of `shape` read from the device address p (an int or a c_void_p)."""
        a = np.zeros(shape, dtype)
        if a.nbytes:
            self.ctx._check(self.lib.plp_dev_download(self.ctx.handle, a.ctypes.data_as(_P), C.c_void_p(p),
                                                      C.c_size_t(a.nbytes)))
        return a

    def download_keypoints(self, batch: int):
        self._after_tracking()
        n = self.d_n.download(np.int32, (batch,))
        return list(zip(self._keypoint_rows(n, self.d_kp, KP_DTYPE),
                        _by_frame(n, self.d_desc.download(np.uint8, (self.max_batch, self.cap, 32)))))

    def download_stereo(self, batch: int):
        """Per frame (stereo_x_right_, depths_) of the last extract() of a stereo FrontEnd, one entry per left
        keypoint (-1: no stereo match)."""
        if not self.stereo:
            raise PlpError("FrontEnd without a stereo camera")
        self._after_tracking()
        n = self.d_n.download(np.int32, (batch,))
        return list(zip(self._keypoint_rows(n, self.d_x_right, np.float32),
                        self._keypoint_rows(n, self._stereo_out["depths"], np.float32)))

    def download_undistorted(self, batch: int):
        """Per frame (undistorted keypoints, bearings) of the last track() -- frame::undist_keypts_ and bearings_.
        Without a distortion the undistorted keypoints are the ORB keypoints and there is nothing to download."""
        if self.distortion is None:
            raise PlpError("FrontEnd without distortion: the ORB keypoints are the undistorted keypoints")
        kp_p, b_p = C.c_void_p(), C.c_void_p()
        self.ctx._check(self.lib.plp_tracker_undistorted(self._trk, C.byref(kp_p), C.byref(b_p)))
        self._after_tracking()
        n = self.d_n.download(np.int32, (batch,))
        return list(zip(_by_frame(n, self._download_ptr(kp_p.value, KP_DTYPE, (batch, self.cap))),
                        _by_frame(n, self._download_ptr(b_p.value, np.float64, (batch, self.cap, 3)))))

    def download_local_tracking(self, batch: int):
        """Results of track_local_map: per frame the last-frame row / local-list index held by each keypoint, the
        observable flag of every local row, pose, num_tracked, n_inliers, LM iterations and status."""
        self._after_tracking()
        n = self.d_n.download(np.int32, (batch,))
        o = self._local_out
        if self._local_from_update:
            offs = self._download_updated_offsets(batch)
            obs = self._upd_out["observable"].download(np.uint8, (max(int(offs[-1]), 1),))
        else:
            offs = self._local_offsets
            obs = self._d_observable.download(np.uint8, (max(int(offs[-1]), 1),))
        return dict(matched=self._keypoint_rows(n, o["matched"]), local=self._keypoint_rows(n, o["local"]),
                    observable=_unpack(offs[:batch + 1], obs),
                    **self._tail_results(batch, o, valid="num_tracked"))

    def _updated_list(self) -> TrackLocal:
        local = TrackLocal()
        self.ctx._check(self.lib.plp_tracker_updated_local_map(self._trk, C.byref(local)))
        return local

    def _download_updated_offsets(self, batch: int) -> np.ndarray:
        return self._download_ptr(self._updated_list().offsets, np.int32, (batch + 1,))

    def download_local_map_update(self, batch: int):
        """Results of update_local_map, per frame: status, nearest keyframe, local keyframes, the local list (landmark
        of every row and its plp_track_local fields), last_local_idx over the frame's set_last_frames rows, and the
        keyframe local_idx block (empty for a frame that does not start from the keyframe or robust stage)."""
        self._after_tracking()
        o = self._upd_out
        loc = self._updated_list()
        offs = self._download_ptr(loc.offsets, np.int32, (batch + 1,))
        n = int(offs[-1])
        lk = o["local_kf"].download(np.int32, (self.max_batch, self.max_local_keyframes))
        nlk = o["num_local_kf"].download(np.int32, (batch,))
        lm = o["local_lm"].download(np.int32, (max(n, 1),))[:n]
        rows = dict(pos_w=self._download_ptr(loc.pos_w, np.float64, (n, 3)),
                    normal=self._download_ptr(loc.obs_mean_normal, np.float64, (n, 3)),
                    min_valid_dist=self._download_ptr(loc.min_valid_dist, np.float32, (n,)),
                    max_valid_dist=self._download_ptr(loc.max_valid_dist, np.float32, (n,)),
                    max_valid_dist_raw=self._download_ptr(loc.max_valid_dist_raw, np.float32, (n,)),
                    desc=self._download_ptr(loc.desc, np.uint8, (n, 32)),
                    valid=self._download_ptr(loc.valid, np.uint8, (n,)))
        lo = self._last_offsets[:batch + 1]
        lli = self._download_ptr(loc.last_local_idx, np.int32, (int(lo[batch]),))
        li, lio = C.c_void_p(), C.c_void_p()
        self.ctx._check(self.lib.plp_tracker_updated_local_idx(self._trk, C.byref(li), C.byref(lio)))
        lio = self._download_ptr(lio.value, np.int32, (batch + 1,))
        li = self._download_ptr(li.value, np.int32, (int(lio[-1]),))
        rows = {k: _unpack(offs, v) for k, v in rows.items()}
        return dict(status=o["status"].download(np.int32, (batch,)), nearest=o["nearest"].download(np.int32, (batch,)),
                    local_kf=_by_frame(nlk, lk), offsets=offs, local_lm=_unpack(offs, lm),
                    rows=[{k: v[b] for k, v in rows.items()} for b in range(batch)],
                    last_local_idx=_unpack(lo, lli), local_idx=_unpack(lio, li))

    def download_keyframe_tracking(self, batch: int):
        """Results of track_keyframe: per frame the stage flag, the keyframe row kept on each keypoint, the BoW match
        count, pose, num_valid, n_inliers, LM iterations, status, and the BoW rows (word id, node id, weight per
        keypoint; meaningful for the frames that ran the stage)."""
        self._after_tracking()
        n = self.d_n.download(np.int32, (batch,))
        o = self._kf_out
        w, nd, wt = C.c_void_p(), C.c_void_p(), C.c_void_p()
        self.ctx._check(self.lib.plp_tracker_keyframe_bow(self._trk, C.byref(w), C.byref(nd), C.byref(wt)))
        bow = [_by_frame(n, self._download_ptr(p.value, dt, (batch, self.cap)))
               for p, dt in ((w, np.int32), (nd, np.int32), (wt, np.float32))]
        return dict(stage=o["stage"].download(np.int32, (batch,)), matched=self._keypoint_rows(n, o["matched"]),
                    num_bow_matches=o["num_bow"].download(np.int32, (batch,)), **self._tail_results(batch, o),
                    bow=list(zip(*bow)))

    def download_robust_tracking(self, batch: int):
        """Results of track_robust: per frame the stage flag, the keyframe row kept on each keypoint, the brute-force
        and robust (RANSAC inlier) match counts, pose, num_valid, n_inliers, LM iterations, status, and the 50 x 8
        RANSAC sample sets (indices into the frame's brute-force match list, -1 where none were drawn)."""
        self._after_tracking()
        n = self.d_n.download(np.int32, (batch,))
        o = self._rb_out
        p = C.c_void_p()
        self.ctx._check(self.lib.plp_tracker_robust_samples(self._trk, C.byref(p)))
        return dict(stage=o["stage"].download(np.int32, (batch,)), matched=self._keypoint_rows(n, o["matched"]),
                    num_bf_matches=o["num_bf"].download(np.int32, (batch,)),
                    num_robust_matches=o["num_robust"].download(np.int32, (batch,)), **self._tail_results(batch, o),
                    samples=self._download_ptr(p.value, np.int32, (batch, 50, 8)))

    def download_match_counts(self, batch: int):
        """The window matcher's per-frame match counts (uint32) of the last track() and track_local_map() (None before
        reserve_local_map); 0xffffffff: the frame has more keypoints than the matcher holds."""
        self._after_tracking()
        m, l = C.c_void_p(), C.c_void_p()
        self.ctx._check(self.lib.plp_tracker_match_counts(self._trk, C.byref(m), C.byref(l)))
        return {name: self._download_ptr(p.value, np.uint32, (batch,)) if p.value else None
                for name, p in (("motion", m), ("local", l))}

    def download_tracking(self, batch: int):
        self._after_tracking()
        n = self.d_n.download(np.int32, (batch,))
        return dict(matched=self._keypoint_rows(n, self.d_matched), **self._tail_results(batch, self._motion_out))
