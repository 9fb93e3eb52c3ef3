"""Generate the golden vectors under tests/golden/ (run in the authoring container; cv2 4.13 is the third-party library the
reference calls for these primitives, the reference binary itself cannot be built here -- see DESIGN.md section 4).

    python tools/gen_golden.py

cv2_primitives.npz  cv::resize / cv::FAST / cv::GaussianBlur 7x7 + 5x5 / cv::Sobel / cv::fastAtan2 on a seeded image
cv2_lsd.npz         cv::LineSegmentDetector(1, 0.5, 0.6, 2, 22.5, 1, 0.6, 1024) segments on two seeded images
orb_mirror.npz      orb_extractor::extract with every third-party stage done by cv2 (tests/test_orb_oracle.py mirror)
line_extract.npz    LineFeatureTracker::extract_LSD_LBD output of the oracle (whose LSD stage is pinned to cv2 above)
cv2_lsd_odd.npz     cv2's half-resolution LSD image and LSD segments at sizes with a dimension = 3 (mod 4)
The images are regenerated from their seeds by the tests; only the outputs are stored.

    python tools/gen_golden.py cv2_lsd_odd      # only the named files"""
import sys
from pathlib import Path

import cv2
import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests"))
import oracle_api  # noqa: E402
import synth  # noqa: E402
import test_golden  # noqa: E402
import test_orb_oracle  # noqa: E402

OUT = ROOT / "tests" / "golden"


def lsd_odd():
    lsd = cv2.createLineSegmentDetector(1, 0.5, 0.6, 2.0, 22.5, 1.0, 0.6, 1024)
    out = {}
    for kind, seed, h, w in test_golden.LSD_ODD:
        img, key = test_golden.lsd_odd_image(kind, seed, h, w), f"{kind}_{seed}"
        g = cv2.GaussianBlur(img, (11, 11), 1.2)
        out[key + "_scaled"] = cv2.resize(g, None, fx=0.5, fy=0.5, interpolation=cv2.INTER_LINEAR_EXACT)
        r = lsd.detect(img)[0]
        out[key] = np.zeros((0, 4), np.float32) if r is None else r.reshape(-1, 4)
    np.savez_compressed(OUT / "cv2_lsd_odd.npz", **out)


def main():
    OUT.mkdir(exist_ok=True)
    if sys.argv[1:]:
        for name in sys.argv[1:]:
            {"cv2_lsd_odd": lsd_odd}[name]()
        return
    orc = oracle_api.Oracle()
    tex = synth.make_texture(4321, 240, 320, n_rect=120, n_blob=500)      # the image of __graft_entry__.smoke()
    lines = synth.make_line_image(7, 240, 320, n_patch=16)
    # ---- third-party primitives
    lv1 = cv2.resize(tex, (267, 200), interpolation=cv2.INTER_LINEAR)      # round(320 / 1.2) x round(240 / 1.2)
    lv2 = cv2.resize(lv1, (222, 167), interpolation=cv2.INTER_LINEAR)
    roi = np.ascontiguousarray(tex[19:89, 83:153])
    fast = {}
    for thr in (20, 7):
        kk = cv2.FastFeatureDetector_create(thr, True).detect(roi)
        fast[thr] = np.array([(k.pt[0], k.pt[1], k.response) for k in kk], np.float32).reshape(-1, 3)
    blur7 = cv2.GaussianBlur(tex, (7, 7), 2, sigmaY=2, borderType=cv2.BORDER_REFLECT_101)
    blur5 = cv2.GaussianBlur(lines, (5, 5), 1.0)
    dx = cv2.Sobel(blur5, cv2.CV_16S, 1, 0, ksize=3)
    dy = cv2.Sobel(blur5, cv2.CV_16S, 0, 1, ksize=3)
    yy, xx = np.meshgrid(np.arange(-40, 41, 5, dtype=np.float32), np.arange(-40, 41, 5, dtype=np.float32), indexing="ij")
    at = np.array([cv2.fastAtan2(float(y), float(x)) for y, x in zip(yy.ravel(), xx.ravel())], np.float32)
    np.savez_compressed(OUT / "cv2_primitives.npz", resize1=lv1, resize2=lv2, fast20=fast[20], fast7=fast[7], blur7=blur7,
                        blur5=blur5, sobel_dx=dx, sobel_dy=dy, atan2_y=yy.ravel(), atan2_x=xx.ravel(), atan2=at,
                        cv2_version=np.array(cv2.__version__))
    # ---- LSD
    lsd = cv2.createLineSegmentDetector(1, 0.5, 0.6, 2.0, 22.5, 1.0, 0.6, 1024)
    seg = {}
    for name, img in (("lines", lines), ("texture", tex)):
        r = lsd.detect(img)[0]
        seg[name] = np.zeros((0, 4), np.float32) if r is None else r.reshape(-1, 4)
    np.savez_compressed(OUT / "cv2_lsd.npz", lines=seg["lines"], texture=seg["texture"])
    # ---- ORB through the cv2-driven mirror of orb_extractor.cc
    p = oracle_api.orb_params(500)
    kps, desc, _ = test_orb_oracle._cv2_mirror_extract(orc, p, tex)
    np.savez_compressed(OUT / "orb_mirror.npz", kps=kps, desc=desc)
    # ---- line extraction (oracle, LSD pinned to cv2)
    kl, lbd, fn = orc.line_extract(lines)
    np.savez_compressed(OUT / "line_extract.npz", keylines=kl, lbd=lbd, line_functions=fn)
    lsd_odd()
    for f in sorted(OUT.glob("*.npz")):
        print(f.name, f.stat().st_size, "bytes")


if __name__ == "__main__":
    main()
