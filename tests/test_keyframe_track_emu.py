"""The keyframe-tracker DEVICE code (structure-plp-slam_b200/csrc/keyframe_track_kernels.cuh, with bow_match_kernel
between the job and gather kernels) executed on the CPU through tests/cta_emu, against a numpy restatement:
capi.fold_bow for the frame's feature vector, a merge-join for the shared nodes, the oracle's bow_tree for the matches,
then the gather and discard_outliers.  The feature vectors are chosen by the test (the transform rows are given), so
that every case occurs: empty keyframe nodes, weight-0 words, a node shared by many rows, no shared node, frames that
do not run the stage, and both status cases.  A second test runs the transform of the active frames only."""
import ctypes as C

import numpy as np
import pytest

import emu_build
import oracle_api
import synth

_P = C.c_void_p
ISIG = synth.inv_level_sigma_sq()


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return emu_build.emu("kftrack_emu", tmp_path_factory, extra=("-Wno-subobject-linkage",))


def _a(x, dt):
    return np.ascontiguousarray(x, dt)


def _ptr(a):
    return None if a is None else a.ctypes.data_as(_P)


def _fold(plp, word, node, weight):
    return plp.capi.fold_bow(word, node, weight)[2]


def _keyframe(plp, rng, n, node_pool, extra_empty=()):
    """A keyframe of n rows: descriptors, angles, landmarks (10 % erased) and a feature vector folded from rows whose
    nodes come from node_pool (a tenth of them stop words), plus empty nodes with the ids in extra_empty."""
    desc = synth.rand_desc(rng, n)
    node = rng.choice(node_pool, n).astype(np.int32)
    weight = rng.uniform(0.1, 2.0, n).astype(np.float32)
    weight[rng.random(n) < 0.1] = 0.0
    ids, offs, idx = _fold(plp, np.arange(n), node, weight)
    if len(extra_empty):  # nodes without rows: the table allows them, they share nothing
        ids_all = np.union1d(ids, np.asarray(extra_empty, np.uint32))
        cnt = {int(i): int(offs[j + 1] - offs[j]) for j, i in enumerate(ids)}
        offs = np.concatenate([[0], np.cumsum([cnt.get(int(i), 0) for i in ids_all])]).astype(np.int32)
        ids = ids_all.astype(np.uint32)
    return dict(desc=desc, node=node, angle=rng.uniform(0, 360, n).astype(np.float32),
                valid=(rng.random(n) >= 0.1).astype(np.uint8), pos_w=rng.normal(0, 3, (n, 3)),
                fv=(ids.astype(np.uint32), offs.astype(np.int32), idx.astype(np.uint32)))


def _frame(rng, kf, n, n_common, node_offset=0, zero_weight=0.1, big_node=None):
    """A frame whose n_common rows are noisy copies of keyframe rows (same node, angle rotated by 20 degrees),
    the rest random; transform rows (word, node, weight) given directly."""
    src = rng.choice(len(kf["desc"]), n_common, replace=False)
    desc = np.concatenate([synth.flip_bits(rng, kf["desc"][src], rng.integers(0, 20, n_common)),
                           synth.rand_desc(rng, n - n_common)])
    node = np.concatenate([kf["node"][src], rng.choice(np.unique(kf["node"]), n - n_common)]).astype(np.int32)
    node += node_offset
    if big_node is not None:  # the random rows pile into one node
        node[n_common:n_common + big_node[1]] = big_node[0]
    angle = np.concatenate([(kf["angle"][src] - 20.0 + rng.normal(0, 2, n_common)) % 360,
                            rng.uniform(0, 360, n - n_common)]).astype(np.float32)
    weight = rng.uniform(0.1, 2.0, n).astype(np.float32)
    weight[rng.random(n) < zero_weight] = 0.0
    perm = rng.permutation(n)
    return dict(desc=desc[perm], node=node[perm], word=np.arange(n, dtype=np.int32), weight=weight[perm],
                angle=angle[perm], x=rng.uniform(0, 640, n).astype(np.float32),
                y=rng.uniform(0, 480, n).astype(np.float32), octave=rng.integers(0, 8, n).astype(np.int32))


def _run(emu, plp, frames, kfs, kf_of_frame, motion_num_valid, motion_valid, max_kf_points, cap, vocab=None, rng=None):
    B = len(frames)
    n_kp = _a([len(f["desc"]) for f in frames], np.int32)

    def pad(key, dt, shape=()):
        out = np.zeros((B, cap) + shape, dt)
        for b, f in enumerate(frames):
            if key in f:
                out[b, :len(f[key])] = f[key]
        return out
    X, Y, A, O, Dsc = pad("x", np.float32), pad("y", np.float32), pad("angle", np.float32), pad("octave", np.int32), \
        pad("desc", np.uint8, (32,))
    word, node, weight = pad("word", np.int32), pad("node", np.int32), pad("weight", np.float32)
    if vocab is not None:  # the transform fills them for the active frames; the others keep the sentinel
        word[:], node[:], weight[:] = -9, -9, -9.0
    rows = np.concatenate([[0], np.cumsum([len(k["desc"]) for k in kfs])]).astype(np.int32)
    fv_offs = np.concatenate([[0], np.cumsum([len(k["fv"][0]) for k in kfs])]).astype(np.int32)
    node_begin, base = [], 0
    for k in kfs:
        node_begin.append(k["fv"][1][:-1].astype(np.int64) + base)
        base += len(k["fv"][2])
    node_begin = np.concatenate(node_begin + [[base]]).astype(np.int32)
    cat = lambda key, dt: _a(np.concatenate([k[key] for k in kfs]), dt)
    kdesc, kang, kval, kpos = cat("desc", np.uint8), cat("angle", np.float32), cat("valid", np.uint8), cat("pos_w", np.float64)
    nids, kidx = _a(np.concatenate([k["fv"][0] for k in kfs]), np.uint32), _a(np.concatenate([k["fv"][2] for k in kfs]), np.uint32)
    pose_last = _a(np.tile(np.eye(4), (B, 1, 1)), np.float64)
    mnv, kof = _a(motion_num_valid, np.int32), _a(kf_of_frame, np.int32)
    mv = None if motion_valid is None else _a(motion_valid, np.uint8)
    stage, status = np.full(B, -3, np.int32), np.full(B, -3, np.int32)
    fidx = np.zeros((B, cap), np.uint32)
    num_nodes = np.zeros(B, np.int32)
    nb2, ne2, nb1, ne1 = (np.zeros((B, cap), np.int32) for _ in range(4))
    matched = np.full((B, cap), -5, np.int32)
    num_bow = np.zeros(B, np.uint32)
    obs = np.zeros((B, cap), oracle_api.PT_OBS_DTYPE)
    obs_kp, obs_row = np.zeros((B, cap), np.int32), np.zeros((B, cap), np.int32)
    n_obs = np.zeros(B, np.int32)
    isig = _a(ISIG, np.float32)
    if vocab is None:
        G, vargs, nid_level = 4, [None] * 5, 0
    else:
        child_begin, children, vdesc, vw, vword, G, nid_level = vocab
        vargs = [_ptr(vdesc), _ptr(child_begin), _ptr(children), _ptr(vw), _ptr(vword)]
    emu.emu_kf_begin(
        C.c_int(B), C.c_int(cap), C.c_int(len(kfs)), C.c_int(max_kf_points), _ptr(n_kp), _ptr(X), _ptr(Y), _ptr(A),
        _ptr(O), _ptr(Dsc), _ptr(mnv), _ptr(pose_last), _ptr(isig), C.c_int(len(isig)), _ptr(mv), _ptr(kof),
        _ptr(rows), _ptr(kdesc), _ptr(kang), _ptr(kval), _ptr(kpos), _ptr(fv_offs), _ptr(nids), _ptr(node_begin),
        _ptr(kidx), C.c_int(G), *vargs, C.c_int(nid_level), _ptr(word), _ptr(node), _ptr(weight), _ptr(stage),
        _ptr(status), _ptr(fidx), _ptr(num_nodes), _ptr(nb2), _ptr(ne2), _ptr(nb1), _ptr(ne1), _ptr(matched),
        _ptr(num_bow), _ptr(obs), _ptr(obs_kp), _ptr(obs_row), _ptr(n_obs))
    got = dict(stage=stage, status=status, fidx=fidx, num_nodes=num_nodes, nb1=nb1, ne1=ne1, nb2=nb2, ne2=ne2,
               matched_pre=matched.copy(), num_bow=num_bow, obs=obs, obs_kp=obs_kp, obs_row=obs_row, n_obs=n_obs,
               word=word, node=node, weight=weight, rows=rows, node_begin=node_begin, fv_offs=fv_offs, n_kp=n_kp)
    # the pose optimiser is not emulated: random outlier flags stand for its result
    outlier = (rng.random((B, cap)) < 0.2).astype(np.uint8)
    num_valid = np.full(B, -3, np.int32)
    emu.emu_tail_finish(_ptr(outlier), _ptr(num_valid))
    got.update(matched=matched, num_valid=num_valid, outlier=outlier)
    return got


def _expect_and_compare(orc, plp, got, frames, kfs, kf_of_frame, motion_num_valid, motion_valid, max_kf_points):
    """The numpy / oracle restatement of every kernel, frame by frame."""
    for b, f in enumerate(frames):
        n = len(f["desc"])
        mv = 1 if motion_valid is None else motion_valid[b]
        stage = int(mv == 0 or motion_num_valid[b] < 20)
        k = kf_of_frame[b]
        status = 0
        if stage:
            if not 0 <= k < len(kfs):
                status = 2
            elif len(kfs[k]["desc"]) > max_kf_points:
                status = 1
        assert (got["stage"][b], got["status"][b]) == (stage, status), b
        active = stage and status == 0
        if not active:
            assert got["num_nodes"][b] == 0 and got["num_bow"][b] == 0 and got["n_obs"][b] == 0, b
            assert (got["matched"][b, :n] == -1).all() and got["num_valid"][b] == 0, b
            continue
        # the frame's bow_feat_vec_ (capi.fold_bow over the rows the kernel read) and the shared nodes
        ids, offs, idx = _fold(plp, got["word"][b, :n], got["node"][b, :n], got["weight"][b, :n])
        assert np.array_equal(got["fidx"][b, :len(idx)], idx), b
        kfv = kfs[k]["fv"]
        shared = []
        i = j = 0
        while i < len(kfv[0]) and j < len(ids):
            if kfv[0][i] == ids[j]:
                a = got["fv_offs"][k] + i
                shared.append((got["node_begin"][a], got["node_begin"][a + 1], offs[j], offs[j + 1]))
                i += 1
                j += 1
            elif kfv[0][i] < ids[j]:
                i += 1
            else:
                j += 1
        nn = got["num_nodes"][b]
        assert nn == len(shared), (b, nn, len(shared))
        spans = list(zip(got["nb1"][b, :nn], got["ne1"][b, :nn], got["nb2"][b, :nn], got["ne2"][b, :nn]))
        assert spans == [(s[0], s[1], s[2], s[3]) for s in shared], b
        # match_frame_and_keyframe, then the gather and discard_outliers
        side1 = dict(desc=kfs[k]["desc"], angle=kfs[k]["angle"], valid=kfs[k]["valid"],
                     fv=(kfv[0], kfv[1], kfv[2]))
        side2 = dict(desc=f["desc"], angle=f["angle"], valid=None, fv=(ids, offs, idx))
        _, m12, num = orc.bow_tree_match(side1, side2, 0.7, True)
        assert got["num_bow"][b] == num, (b, got["num_bow"][b], num)
        assert np.array_equal(got["matched_pre"][b, :n], m12), b
        _expect_tail(got, b, num, m12, kfs[k]["pos_w"], f)


def _expect_tail(got, b, count, m12, pos_w, f):
    """The tail (track_common.cuh) of frame b: below 20 matches nothing is gathered and every match is dropped;
    otherwise one observation per matched keypoint in keypoint order (its row's pos_w), then discard_outliers."""
    n = len(f["x"])
    if count < 20:
        assert got["n_obs"][b] == 0 and (got["matched"][b, :n] == -1).all() and got["num_valid"][b] == 0, b
        return
    sel = np.nonzero(m12 >= 0)[0]
    no = len(sel)
    assert got["n_obs"][b] == no, b
    assert np.array_equal(got["obs_kp"][b, :no], sel) and np.array_equal(got["obs_row"][b, :no], m12[sel]), b
    o = got["obs"][b, :no]
    assert np.array_equal(o["pos_w"], pos_w[m12[sel]]), b
    assert np.array_equal(o["obs_x"], f["x"][sel]) and np.array_equal(o["obs_y"], f["y"][sel]), b
    assert (o["x_right"] == -1.0).all() and np.array_equal(o["inv_sigma_sq"], ISIG[f["octave"][sel]]), b
    post = m12.copy()
    post[sel[got["outlier"][b, :no] != 0]] = -1
    assert np.array_equal(got["matched"][b, :n], post) and got["num_valid"][b] == (post >= 0).sum(), b


def test_keyframe_track_kernels_on_cpu_equal_restatement(emu, orc, plp):
    rng = np.random.default_rng(61)
    pool = np.sort(rng.choice(100000, 40, replace=False))
    kfs = [_keyframe(plp, rng, 300, pool), _keyframe(plp, rng, 260, pool, extra_empty=pool[:5] + 1),
           _keyframe(plp, rng, 420, pool)]
    assert (np.diff(kfs[1]["fv"][1]) == 0).sum() >= 5
    frames = [
        _frame(rng, kfs[0], 330, 200, big_node=(int(pool[3]), 130)),  # 0: many rows in one node, weight-0 words
        _frame(rng, kfs[1], 280, 180),                                   # 1: keyframe with empty nodes, motion failed
        _frame(rng, kfs[0], 300, 200, node_offset=200000),               # 2: no node in common with the keyframe
        _frame(rng, kfs[0], 310, 200),                                   # 3: the motion result stands
        _frame(rng, kfs[1], 250, 150, zero_weight=1.0),                  # 4: every word weighs 0: an empty vector
        _frame(rng, kfs[0], 200, 100),                                   # 5: kf_of_frame out of range
        _frame(rng, kfs[2], 200, 100),                                   # 6: keyframe over the reservation
        _frame(rng, kfs[0], 320, 220),                                   # 7: shares keyframe 0 with frames 0, 2, 3
    ]
    # frame 1's empty nodes are also frame nodes: a shared node with no keyframe row
    frames[1]["node"][:10] = pool[0] + 1
    kf_of_frame = [0, 1, 0, 0, 1, 3, 2, 0]
    motion_num_valid = [300, 5, 300, 300, 300, 300, 300, 300]
    motion_valid = [0, 1, 0, 1, 0, 0, 0, 0]
    cap, max_kf = 352, 300
    got = _run(emu, plp, frames, kfs, kf_of_frame, motion_num_valid, motion_valid, max_kf, cap, rng=rng)
    _expect_and_compare(orc, plp, got, frames, kfs, kf_of_frame, motion_num_valid, motion_valid, max_kf)
    assert list(got["stage"]) == [1, 1, 1, 0, 1, 1, 1, 1] and list(got["status"]) == [0, 0, 0, 0, 0, 2, 1, 0]
    assert all(got["num_bow"][b] >= 20 for b in (0, 1, 7)) and got["num_valid"][0] > 0
    assert got["num_nodes"][2] == 0 and got["num_nodes"][4] == 0 and got["num_bow"][2] == 0
    # frame 1 shares one of keyframe 1's empty nodes
    spans = list(zip(got["nb1"][1, :got["num_nodes"][1]], got["ne1"][1, :got["num_nodes"][1]]))
    assert any(s == e for s, e in spans)


def test_keyframe_track_transform_runs_on_active_frames_only(emu, orc, plp):
    """The vocabulary descent of kf_transform_kernel on the active frames (equal to the oracle's transform); the rows of
    the other frames are left alone.  Motion validity left out (NULL) means every motion model is usable."""
    import bow_data
    from test_cta_emu import _csr_vocab
    rng = np.random.default_rng(62)
    vocab = bow_data.make_vocab(62, k=4, L=6)
    child_begin, children, vdesc, vw, vword, max_children = _csr_vocab(vocab)
    G = 4 if max_children <= 4 else 8
    ov = orc.bow_vocab_create(4, 6, vocab["parent"], vocab["desc"], vocab["weight"], vocab["is_leaf"])
    try:
        leaves = vocab["desc"][vocab["is_leaf"] > 0]
        kdesc = synth.flip_bits(rng, leaves[rng.integers(0, len(leaves), 200)], rng.integers(0, 20, 200))
        _, _, fv = plp.capi.fold_bow(*orc.bow_transform(ov, kdesc, 4))
        kf = dict(desc=kdesc, angle=rng.uniform(0, 360, 200).astype(np.float32), valid=np.ones(200, np.uint8),
                  pos_w=rng.normal(0, 3, (200, 3)), fv=fv, node=np.zeros(200, np.int32))
        frames = []
        for n in (150, 171, 97):
            src = rng.choice(200, n // 2, replace=False)
            desc = np.concatenate([synth.flip_bits(rng, kdesc[src], rng.integers(0, 10, len(src))),
                                   synth.rand_desc(rng, n - len(src))])
            frames.append(dict(desc=desc, angle=np.concatenate([kf["angle"][src], rng.uniform(0, 360, n - len(src))]).astype(np.float32),
                               x=rng.uniform(0, 640, n).astype(np.float32), y=rng.uniform(0, 480, n).astype(np.float32),
                               octave=rng.integers(0, 8, n).astype(np.int32)))
        motion_num_valid = [3, 300, 0]  # frames 0 and 2 failed their motion track
        got = _run(emu, plp, frames, [kf], [0, 0, 0], motion_num_valid, None, 200, 192,
                   vocab=(child_begin, children, vdesc, vw, vword, G, vocab["L"] - 4), rng=rng)
        for b in (0, 2):
            n = len(frames[b]["desc"])
            want = orc.bow_transform(ov, frames[b]["desc"], 4)
            for g, w in zip((got["word"][b, :n], got["node"][b, :n], got["weight"][b, :n]), want):
                assert np.array_equal(g, w), b
        assert (got["word"][1] == -9).all() and (got["node"][1] == -9).all() and (got["weight"][1] == -9.0).all()
        _expect_and_compare(orc, plp, got, frames, [kf], [0, 0, 0], motion_num_valid, None, 200)
        assert list(got["stage"]) == [1, 0, 1]
    finally:
        orc.bow_vocab_destroy(ov)


def test_track_tail_motion_form_on_cpu_equal_restatement(emu):
    """The shared tail with null stage / status, as the motion stage binds it: the gate is the match count alone, frame
    b's rows are block b of the last frames' rows, and the optimisation starts from frame b's predicted pose."""
    rng = np.random.default_rng(63)
    counts = [57, 19, 20, 0, 300, 21]
    B, cap = len(counts), 300
    sizes = [int(rng.integers(30, 200)) for _ in range(B)]
    offsets = _a(np.concatenate([[0], np.cumsum(sizes)]), np.int32)
    pos_w = _a(rng.normal(0, 3, (int(offsets[-1]), 3)), np.float64)
    frames, m12s = [], []
    for b in range(B):
        n = int(rng.integers(100, cap + 1))
        frames.append(dict(x=rng.uniform(0, 640, n).astype(np.float32), y=rng.uniform(0, 480, n).astype(np.float32),
                           octave=rng.integers(0, 8, n).astype(np.int32)))
        m12s.append(np.where(rng.random(n) < 0.4, rng.integers(0, sizes[b], n), -1).astype(np.int32))
    n_kp = _a([len(f["x"]) for f in frames], np.int32)
    X, Y, O = (np.zeros((B, cap), dt) for dt in (np.float32, np.float32, np.int32))
    matched = np.full((B, cap), -5, np.int32)
    for b, f in enumerate(frames):
        n = len(f["x"])
        X[b, :n], Y[b, :n], O[b, :n], matched[b, :n] = f["x"], f["y"], f["octave"], m12s[b]
    count = _a(counts, np.int32)
    pose_in = _a(rng.normal(0, 1, (B, 16)), np.float64)
    obs = np.zeros((B, cap), oracle_api.PT_OBS_DTYPE)
    obs_kp, obs_row = np.zeros((B, cap), np.int32), np.zeros((B, cap), np.int32)
    n_obs, t_in = np.full(B, -3, np.int32), np.full(B, -3, np.int32)
    isig = _a(ISIG, np.float32)
    emu.emu_tail_begin(C.c_int(B), C.c_int(cap), _ptr(n_kp), _ptr(X), _ptr(Y), _ptr(O), _ptr(isig), C.c_int(len(isig)),
                       _ptr(count), None, None, _ptr(pos_w), _ptr(offsets), None, _ptr(pose_in), _ptr(matched),
                       _ptr(obs), _ptr(obs_kp), _ptr(obs_row), _ptr(n_obs), _ptr(t_in))
    outlier = (rng.random((B, cap)) < 0.2).astype(np.uint8)
    num_valid = np.full(B, -3, np.int32)
    emu.emu_tail_finish(_ptr(outlier), _ptr(num_valid))
    got = dict(n_obs=n_obs, obs_kp=obs_kp, obs_row=obs_row, obs=obs, matched=matched, num_valid=num_valid,
               outlier=outlier)
    assert list(t_in) == list(range(B))
    for b, f in enumerate(frames):
        _expect_tail(got, b, counts[b], m12s[b], pos_w[offsets[b]:offsets[b + 1]], f)
    assert [int(n_obs[b] > 0) for b in range(B)] == [1, 0, 1, 0, 1, 1]
