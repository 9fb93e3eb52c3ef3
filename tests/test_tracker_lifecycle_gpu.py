"""What a FrontEnd and its tracker own: close() frees every buffer the FrontEnd still holds, and a reservation the device
cannot hold is refused once, leaving no stage bound to freed memory and no error behind for the next call."""
import ctypes as C

import numpy as np
import pytest

import local_map_update_data as lmu
import scene

pytestmark = pytest.mark.gpu
TS = [2, 3, 4, 5]


def _front_end(plp, ctx, seq):
    """A FrontEnd over frames TS of `seq`, its last frames set from its own extraction of frames TS - 1."""
    from plpslam_b200.tracking import FrontEnd
    fe = FrontEnd(ctx, seq.rows, seq.cols, seq.camera(plp), max_batch=len(TS))
    fe.upload_images(seq.frames[[t - 1 for t in TS]])
    fe.extract(len(TS))
    kps = fe.download_keypoints(len(TS))
    lasts = [seq.last_frame_landmarks(t - 1, k, d) for t, (k, d) in zip(TS, kps)]
    rng = np.random.default_rng(3)
    fe.set_last_frames(lasts, np.stack([seq.predicted_pose(t, rng) for t in TS]),
                       np.stack([seq.poses[t - 1] for t in TS]))
    fe.upload_images(seq.frames[TS])
    return fe, lasts


def test_close_frees_every_buffer(ctx, plp, monkeypatch):
    """Every stage reserved, every input set, the host I/O staged and one step run: close() frees every device and
    pinned buffer the FrontEnd made, and a second close() does nothing."""
    from plpslam_b200.tracking import DeviceBuffer, PinnedBuffer
    made = []
    for cls in (DeviceBuffer, PinnedBuffer):
        def init(self, *a, _init=cls.__init__, **kw):
            _init(self, *a, **kw)
            made.append(self)
        monkeypatch.setattr(cls, "__init__", init)
    seq = scene.PlanarSequence(seed=51, n_frames=max(TS) + 1)
    fe, lasts = _front_end(plp, ctx, seq)
    rng = np.random.default_rng(5)
    fe.reserve_local_map(1024)
    fe.reserve_keyframe_track(2, 64)
    fe.reserve_robust_track()
    fe.reserve_local_map_update(64)
    n = [len(last["octave"]) for last in lasts]
    fe.set_local_maps([dict(pos_w=rng.normal(size=(8, 3)), normal=rng.normal(size=(8, 3)),
                            min_valid_dist=np.ones(8, np.float32), max_valid_dist=np.full(8, 2, np.float32),
                            max_valid_dist_raw=np.full(8, 2, np.float32),
                            desc=rng.integers(0, 256, (8, 32), dtype=np.uint8), valid=None,
                            last_local_idx=np.full(m, -1, np.int32)) for m in n])
    keyframes = [dict(desc=rng.integers(0, 256, (10, 32), dtype=np.uint8), angle=np.zeros(10, np.float32),
                      valid=None, pos_w=rng.normal(size=(10, 3)), bearings=rng.normal(size=(10, 3)),
                      fv=(np.array([3, 7], np.uint32), np.array([0, 4, 10]), np.arange(10, dtype=np.uint32)))
                 for _ in range(2)]
    fe.set_keyframes(keyframes, [0, 1, 0, 1], local_idx=[np.full(10, -1, np.int32) for _ in TS])
    snap = lmu.synthetic_snapshot(3, 20, rng)
    snap["last_row_lm"] = np.full(sum(n), -1, np.int32)
    snap["kf_row_lm"] = np.full(20, -1, np.int32)
    fe.set_map(snap)
    fe.stage_host_io(seq.frames[TS])
    fe.step(len(TS))
    ctx.sync()
    assert any(isinstance(b, PinnedBuffer) for b in made) and len(made) > 30
    fe.close()
    assert [b for b in made if b.ptr is not None] == []
    fe.close()


def test_refused_reservation_leaves_nothing_behind(ctx, plp):
    """A local-map reservation far beyond the device's memory returns PLP_ERR_CUDA: the old reservation is gone (its
    match counts are no longer handed out), and the next step runs and computes what it computed before the refusal."""
    from plpslam_b200.tracking import _logf
    seq = scene.PlanarSequence(seed=52, n_frames=max(TS) + 1)
    fe, _ = _front_end(plp, ctx, seq)
    try:
        fe.reserve_local_map(4096)
        fe.step(len(TS))
        before = fe.download_tracking(len(TS))
        assert fe.download_match_counts(len(TS))["local"] is not None
        st = fe.lib.plp_tracker_reserve_local_map(fe._trk, C.c_float(_logf(fe.scale_factor)), C.c_int(2**31 - 1))
        assert st == 3, fe.lib.plp_last_error()  # PLP_ERR_CUDA
        m, loc = C.c_void_p(), C.c_void_p()
        assert fe.lib.plp_tracker_match_counts(fe._trk, C.byref(m), C.byref(loc)) == 0
        assert m.value and loc.value is None
        fe.step(len(TS))
        after = fe.download_tracking(len(TS))
        assert before.keys() == after.keys()
        for k in before:
            assert all(np.array_equal(x, y) for x, y in zip(before[k], after[k])), k
    finally:
        fe.close()
