"""describe_kernel takes runs of RUN consecutive output positions of a frame per warp and stages each keypoint's disc and
blurred window by 16-byte copies (plain loads for a level-0 buffer whose rows are not 16-byte aligned).  Keypoints and
descriptors must equal the oracle's bit for bit where the run logic and the staging have edges: runs crossing level
boundaries, partial last runs, frames without keypoints between full ones, frames with more keypoints than the grid
covers (warps stride), and keypoints at the outermost positions of every level, whose aligned chunks end at the row."""
import numpy as np
import pytest

import oracle_api
import synth
from test_batch_dev_gpu import _OrbOut, _pitched

pytestmark = pytest.mark.gpu
RUN, WARPS = 8, 4  # kDescRun, kDescWarps in csrc/orb.cu


@pytest.fixture
def own():
    objs = []
    yield lambda x: objs.append(x) or x
    for x in reversed(objs):
        (x.free if hasattr(x, "free") else x.close)()


def _extract(plp, ctx, own, imgs, step, offset=0):
    B, rows, cols = imgs.shape
    ext = own(plp.OrbExtractor(ctx, rows, cols, max_batch=B))
    out = own(_OrbOut(plp, ctx, B, ext.capacity))
    d_img, ptr = _pitched(ctx, imgs, step, offset=offset, seed=offset + step)
    own(d_img)
    out.run(ext, ptr, B, step)
    n, got, st = out.get(plp, B)
    assert not st.any(), st
    return n, got


def _check_oracle(orc, imgs, got, what):
    p = oracle_api.orb_params()
    for b, img in enumerate(imgs):
        r = orc.orb_extract(p, img)
        assert np.array_equal(got[b][0], r["kps"]), f"{what} frame {b}: keypoints"
        assert np.array_equal(got[b][1], r["desc"]), f"{what} frame {b}: descriptors"


def test_runs_empty_frames_and_stride(ctx, orc, plp, own):
    """Textured frames (partial last runs, runs across level boundaries), flat frames without a keypoint between them,
    and a noise frame with more keypoints than the grid's max_num_keypts positions, so that its warps stride."""
    rows, cols = 480, 640
    flat = np.full((rows, cols), 128, np.uint8)
    noise = np.random.default_rng(41).integers(0, 256, (rows, cols), dtype=np.uint8)
    imgs = np.stack([synth.make_texture(40), flat, synth.make_plp_texture(42), flat, flat, noise,
                     synth.make_texture(43)])
    n, got = _extract(plp, ctx, own, imgs, cols)
    _check_oracle(orc, imgs, got, "640x480")
    assert list(n[[1, 3, 4]]) == [0, 0, 0], n
    cover = -(-max(256, 1000) // (WARPS * RUN)) * WARPS * RUN  # output positions of one pass of the grid
    assert n[5] > cover, (n[5], cover)
    assert any(k % RUN for k in n), n
    cum = [np.cumsum(np.bincount(got[b][0]["octave"], minlength=8))[:-1] for b in (0, 2, 6)]
    assert any(c % RUN for cc in cum for c in cc), cum


def _border_frame(seed, band, rows=480, cols=752):
    """Noise in a band along the four borders around a flat centre: the quadtree keeps keypoints at the outermost
    positions of the levels the band reaches."""
    img = np.random.default_rng(seed).integers(0, 256, (rows, cols), dtype=np.uint8)
    img[band:-band, band:-band] = 128
    return img


@pytest.mark.parametrize("step,offset", [(752, 0), (752, 1), (760, 0)], ids=["aligned", "base_plus_1", "pitch_760"])
def test_border_keypoints_every_level(ctx, orc, plp, own, step, offset):
    """752 x 480 (EuRoC): no level above 0 is a multiple of 16 wide.  At every level and next to each border, some
    keypoint lies at the outermost position a keypoint can take (22 pixels in).  The aligned buffer copies level 0's
    disc in 16-byte chunks; a base one byte off, or a 760-byte pitch, takes the plain loads."""
    imgs = np.stack([_border_frame(5, 48), _border_frame(6, 120), _border_frame(7, 48), _border_frame(9, 90),
                     synth.make_texture(44, 480, 752)])
    n, got = _extract(plp, ctx, own, imgs, step, offset)
    _check_oracle(orc, imgs, got, f"752x480 step {step} offset {offset}")
    ws, hs = orc.orb_level_sizes(oracle_api.orb_params(), 480, 752)
    kps = np.concatenate([got[b][0] for b in range(4)])
    for l in range(8):
        k = kps[kps["octave"] == l]
        s = np.float32(1.2) ** l
        x, y = np.rint(k["x"] / s), np.rint(k["y"] / s)
        edge = (x.min(), ws[l] - 1 - x.max(), y.min(), hs[l] - 1 - y.max())
        assert max(edge) == 22, (l, edge)
