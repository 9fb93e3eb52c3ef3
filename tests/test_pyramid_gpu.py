"""The ORB image pyramid at the edges of pyr_resize_kernel's work split, every level of every frame bit-exact against
the oracle.

pyr_resize_kernel builds a level in bands of destination rows from source rows staged in shared memory (16-byte copies
when the source level's base and pitch allow them, byte loads otherwise) and writes 8 bytes per store.  The cases: level
heights that are not a multiple of the band, widths that are not a multiple of 16, level 0 in a caller buffer whose pitch
rules out 16-byte copies, the largest accepted image (bands of fewer rows), two levels, and a scale factor of 1.5."""
import numpy as np
import pytest

import oracle_api
import synth
from test_batch_dev_gpu import _OrbOut, _kernels_run, _pitched

pytestmark = pytest.mark.gpu


# rows, cols, levels, scale factor, frames
CASES = {
    "479x641": (479, 641, 8, 1.2, 3),
    "2085x1061": (1061, 2085, 8, 1.2, 1),
    "640x480_2_levels": (480, 640, 2, 1.2, 3),
    "320x240": (240, 320, 8, 1.2, 3),
    "427x333_scale_1.5": (333, 427, 4, 1.5, 2),
}


# level 0's row pitch: odd (byte loads), the image width, a multiple of 16 (16-byte loads)
STEPS = {"step_cols_plus_1": lambda cols: cols + 1, "step_eq_cols": lambda cols: cols,
         "step_16": lambda cols: (cols + 31) // 16 * 16}


@pytest.mark.parametrize("step_kind", list(STEPS))
@pytest.mark.parametrize("case", list(CASES))
def test_pyramid_levels(ctx, orc, plp, case, step_kind):
    rows, cols, levels, scale, B = CASES[case]
    lib = plp.lib()
    step = STEPS[step_kind](cols)
    imgs = np.stack([synth.make_texture(500 + i, rows, cols) for i in range(B)])
    p = oracle_api.orb_params(500, scale, levels, 20, 7)  # a keypoint budget the 2-level quadtree holds
    orb = plp.OrbExtractor(ctx, rows, cols, 500, scale_factor=scale, num_levels=levels, max_batch=B)
    out = _OrbOut(plp, ctx, B, orb.capacity)
    d_img, ptr = _pitched(ctx, imgs, step, seed=step)
    try:
        names = _kernels_run(ctx, lib, lambda: out.run(orb, ptr, B, step))
        assert "pyr_resize_kernel" in names, names
        n, got, st = out.get(plp, B)
        assert not st.any()
        for b in range(B):
            ref = orc.orb_extract(p, imgs[b], debug=True)["pyramid"]
            assert len(ref) == levels
            for l in range(levels):
                assert np.array_equal(orb.pyramid_level(b, l), ref[l]), f"frame {b} level {l} ({ref[l].shape})"
    finally:
        d_img.free()
        out.free()
        orb.close()
