"""Pins oracle/orb.cc: the OpenCV primitives bit-exactly against cv2 4.13 (the third-party library the
reference calls -- SURVEY.md Appendix A), the reference's own ORB known-answer / behavioural tests, and the
whole extract() orchestration against a cv2-driven mirror of orb_extractor.cc."""
import math

import cv2
import numpy as np
import pytest

import oracle_api
import synth


@pytest.fixture(scope="module")
def tex():
    return synth.make_texture(1234)


# ---------------------------------------------------------------- cv::resize (orb_extractor.cc:324)
@pytest.mark.parametrize("rows,cols", [(480, 640), (480, 752), (333, 517)])
def test_resize_chain_matches_cv2(orc, rows, cols):
    rng = np.random.default_rng(rows + cols)
    img = rng.integers(0, 256, (rows, cols), dtype=np.uint8)
    p = oracle_api.orb_params()
    w, h = orc.orb_level_sizes(p, rows, cols)
    cur = img
    for l in range(1, 8):
        ref = cv2.resize(cur, (int(w[l]), int(h[l])), interpolation=cv2.INTER_LINEAR)
        got = orc.resize_linear(cur, int(w[l]), int(h[l]))
        assert np.array_equal(ref, got), f"level {l}"
        cur = ref


def test_level_sizes_match_survey(orc):
    p = oracle_api.orb_params()
    w, h = orc.orb_level_sizes(p, 480, 640)
    assert list(zip(w.tolist(), h.tolist())) == [(640, 480), (533, 400), (444, 333), (370, 278), (309, 231),
                                                 (257, 193), (214, 161), (179, 134)]
    assert int((w.astype(np.int64) * h).sum()) == 950532  # SURVEY.md section 8


# ---------------------------------------------------------------- cv::FAST (orb_extractor.cc:404-411)
@pytest.mark.parametrize("thr", [20, 7])
def test_fast_matches_cv2_on_cells(orc, tex, thr):
    det = cv2.FastFeatureDetector_create(thr, True)
    rng = np.random.default_rng(thr)
    total = 0
    for _ in range(40):
        w, h = int(rng.integers(8, 71)), int(rng.integers(8, 71))
        x0, y0 = int(rng.integers(0, 640 - w)), int(rng.integers(0, 480 - h))
        roi = tex[y0:y0 + h, x0:x0 + w]
        ref = det.detect(np.ascontiguousarray(roi))
        got = orc.fast(roi, thr, True)
        assert len(ref) == len(got)
        for a, b in zip(ref, got):
            assert (a.pt[0], a.pt[1], a.response) == (b["x"], b["y"], b["response"])
        total += len(got)
    assert total > 100


def test_fast_without_nms_and_noise_image(orc):
    rng = np.random.default_rng(5)
    img = rng.integers(0, 256, (60, 70), dtype=np.uint8)
    for thr, nms in [(20, False), (40, True), (7, True)]:
        ref = cv2.FastFeatureDetector_create(thr, nms).detect(img)
        got = orc.fast(img, thr, nms)
        assert [(k.pt[0], k.pt[1], k.response) for k in ref] == [(g["x"], g["y"], g["response"]) for g in got]


# ---------------------------------------------------------------- cv::GaussianBlur
def test_gaussian_blur_matches_cv2(orc, tex):
    rng = np.random.default_rng(1)
    for img in (tex, rng.integers(0, 256, (200, 300), dtype=np.uint8), rng.integers(0, 256, (39, 41), dtype=np.uint8)):
        ref = cv2.GaussianBlur(img, (7, 7), 2, sigmaY=2, borderType=cv2.BORDER_REFLECT_101)
        assert np.array_equal(ref, orc.blur7(img))
        ref5 = cv2.GaussianBlur(img, (5, 5), 1)
        assert np.array_equal(ref5, orc.blur5(img))


# ---------------------------------------------------------------- cv::fastAtan2 (orb_extractor.cc:734)
def test_fast_atan2_matches_cv2(orc):
    rng = np.random.default_rng(2)
    pts = rng.integers(-200000, 200001, (20000, 2))
    pts[:50] = [[0, 0], [1, 0], [0, 1], [-1, 0], [0, -1]] * 10
    for y, x in pts:
        assert orc.lib.orc_fast_atan2(float(y), float(x)) == cv2.fastAtan2(float(y), float(x))


# ---------------------------------------------------------------- test/PLPSLAM/util/trigonometric.cc:8-24
def test_trigonometric_tolerance(orc):
    for deg in range(0, 3601):
        rad = np.float32(np.float32(deg / np.float32(10.0)) * math.pi / np.float32(180.0))
        assert abs(math.cos(rad) - orc.lib.orc_util_cos(float(rad))) < 1e-3
        assert abs(math.sin(rad) - orc.lib.orc_util_sin(float(rad))) < 1e-3


# ---------------------------------------------------------------- test/PLPSLAM/feature/orb_params.cc:159-211
def test_scale_tables_known_answers(orc):
    p = oracle_api.orb_params(levels=10, sf=1.26)
    t = orc.orb_tables(p)
    sf = np.float32(1.26)
    s = np.float32(1.0)
    for level in range(10):
        assert t["scale_factors"][level] == pytest.approx(float(sf) ** level, rel=4e-7 * (level + 1))
        assert t["inv_scale_factors"][level] == pytest.approx((1.0 / float(sf)) ** level, rel=4e-7 * (level + 1))
        assert t["level_sigma_sq"][level] == np.float32(s * s)
        assert t["inv_level_sigma_sq"][level] == np.float32(np.float32(1.0) / np.float32(s * s))
        s = np.float32(sf * s)


def test_keypoint_budget_and_umax(orc):
    t = orc.orb_tables(oracle_api.orb_params())
    assert t["num_keypts_per_level"].tolist() == [217, 181, 151, 126, 105, 87, 73, 60]  # orb_extractor.cc:255-264
    assert t["u_max"].tolist() == [15, 15, 15, 15, 14, 14, 14, 13, 13, 12, 11, 10, 9, 8, 6, 3]  # SURVEY A5


# ---------------------------------------------------------------- test/PLPSLAM/feature/orb_extractor.cc:27-83
@pytest.mark.parametrize("variant", [1, 2])
def test_toy_corner_localisation(orc, variant):
    img, (cx, cy) = synth.make_toy_corner_image(variant)
    p = oracle_api.orb_params()  # feature::orb_params() defaults: 2000 kp, 1.2, 8 levels, 20/7
    p.max_num_keypts = 2000
    r = orc.orb_extract(p, img)
    sf = orc.orb_tables(p)["scale_factors"]
    assert len(r["kps"]) == len(r["desc"]) > 0
    for k in r["kps"]:
        tol = 2.0 * sf[k["octave"]]
        assert abs(k["x"] - cx) <= tol and abs(k["y"] - cy) <= tol


def test_mask_containment(orc, tex):
    # test/PLPSLAM/feature/orb_extractor.cc:125-359: no keypoint inside the masked (zero) region
    mask = np.full(tex.shape, 255, np.uint8)
    mask[:, :320] = 0
    r = orc.orb_extract(oracle_api.orb_params(), tex, mask=mask)
    assert len(r["kps"]) > 100
    assert np.all(r["kps"]["x"] >= 320 - 1e-3)


def test_empty_and_tiny_images(orc):
    p = oracle_api.orb_params()
    flat = np.full((480, 640), 128, np.uint8)
    r = orc.orb_extract(p, flat)
    assert len(r["kps"]) == 0


# ---------------------------------------------------------------- whole pipeline vs a cv2-driven mirror
def _cv2_mirror_extract(orc, p, img):
    """orb_extractor.cc:73-160 with the third-party stages done by cv2 itself."""
    t = orc.orb_tables(p)
    L = p.num_levels
    w, h = orc.orb_level_sizes(p, *img.shape)
    pyr = [img]
    for l in range(1, L):
        pyr.append(cv2.resize(pyr[-1], (int(w[l]), int(h[l])), interpolation=cv2.INTER_LINEAR))
    det_ini = cv2.FastFeatureDetector_create(int(p.ini_fast_thr), True)
    det_min = cv2.FastFeatureDetector_create(int(p.min_fast_thr), True)
    kps_all, desc_all = [], []
    for l in range(L):
        im = pyr[l]
        R = 19
        max_bx, max_by = im.shape[1] - R, im.shape[0] - R
        width, height = max_bx - R, max_by - R
        ncols, nrows = width // 64 + 1, height // 64 + 1
        cands = []
        for i in range(nrows):
            min_y = R + i * 64
            if max_by - 6 <= min_y:
                continue
            max_y = min(min_y + 70, max_by)
            for j in range(ncols):
                min_x = R + j * 64
                if max_bx - 6 <= min_x:
                    continue
                max_x = min(min_x + 70, max_bx)
                roi = np.ascontiguousarray(im[min_y:max_y, min_x:max_x])
                kk = det_ini.detect(roi)
                if not kk:
                    kk = det_min.detect(roi)
                for k in kk:
                    cands.append((k.pt[0] + j * 64, k.pt[1] + i * 64, 7.0, -1.0, k.response, 0, -1))
        if not cands:
            continue
        cands = np.array(cands, oracle_api.KP_DTYPE)
        kl = orc.orb_distribute(p, cands, R, max_bx, R, max_by, int(t["num_keypts_per_level"][l]))
        kl["x"] += R
        kl["y"] += R
        kl["octave"] = l
        kl["size"] = float(int(31 * t["scale_factors"][l]))
        blurred = cv2.GaussianBlur(im, (7, 7), 2, sigmaY=2, borderType=cv2.BORDER_REFLECT_101)
        for k in kl:
            xi, yi = int(k["x"]), int(k["y"])
            m01 = m10 = 0
            um = t["u_max"]
            rowc = im[yi].astype(np.int64)
            for u in range(-15, 16):
                m10 += u * int(rowc[xi + u])
            for v in range(1, 16):
                d = int(um[v])
                plus = im[yi + v, xi - d:xi + d + 1].astype(np.int64)
                minus = im[yi - v, xi - d:xi + d + 1].astype(np.int64)
                us = np.arange(-d, d + 1)
                m01 += v * int((plus - minus).sum())
                m10 += int((us * (plus + minus)).sum())
            k["angle"] = cv2.fastAtan2(float(m01), float(m10))
            desc_all.append(orc.orb_describe(p, blurred, k))
        if l:
            s = t["scale_factors"][l]
            kl["x"] = (kl["x"] * s).astype(np.float32)
            kl["y"] = (kl["y"] * s).astype(np.float32)
        kps_all.append(kl)
    # a small image can leave every level without a keypoint
    kps = np.concatenate(kps_all) if kps_all else np.zeros(0, oracle_api.KP_DTYPE)
    return kps, np.array(desc_all, np.uint8).reshape(-1, 32), pyr


@pytest.mark.parametrize("shape", [(40, 41), (41, 40), (48, 64), (75, 100), (120, 160)])
def test_small_images_match_cv2_mirror(orc, shape):
    """Upper levels of a small image have no FAST cell (w or h <= 38); 41 x 40 has no keypoint at any level."""
    img = synth.make_texture(9, *shape)
    p = oracle_api.orb_params()
    r = orc.orb_extract(p, img)
    kps, desc, pyr = _cv2_mirror_extract(orc, p, img)
    for a, b in zip(pyr, r["pyramid"]):
        assert np.array_equal(a, b)
    assert len(kps) == len(r["kps"]) and desc.shape == r["desc"].shape
    for f in ("x", "y", "size", "angle", "response", "octave"):
        assert np.array_equal(kps[f], r["kps"][f]), f
    assert np.array_equal(desc, r["desc"])
    if min(shape) >= 75:
        assert len(kps) > 10


@pytest.mark.parametrize("seed,shape", [(1234, (480, 640)), (77, (480, 752))])
def test_extract_matches_cv2_mirror(orc, seed, shape):
    img = synth.make_texture(seed, shape[0], shape[1])
    p = oracle_api.orb_params()
    r = orc.orb_extract(p, img)
    kps, desc, pyr = _cv2_mirror_extract(orc, p, img)
    for a, b in zip(pyr, r["pyramid"]):
        assert np.array_equal(a, b)
    assert len(kps) == len(r["kps"]) > 1000
    for f in ("x", "y", "size", "angle", "response", "octave"):
        assert np.array_equal(kps[f], r["kps"][f]), f
    assert np.array_equal(desc, r["desc"])
