// rectify_emu.cc -- csrc/rectify_kernels.cuh executed on the host (see cta_emu.h): the fixed-point map conversion and
// rectify_kernel's tiling, batch loop, pitches and partial last words, against the oracle.
#include "cta_emu.h"

#include <vector>

#include "rectify_kernels.cuh"

using namespace plp;

// map_x, map_y: rows x cols float maps; frame b of in / out at b * rows * step
extern "C" void emu_rectify(const float *map_x, const float *map_y, int rows, int cols, int batch, const uint8_t *in,
                            size_t in_step, uint8_t *out, size_t out_step) {
    const int pitch = rect_map_pitch(cols);
    std::vector<short2> xy((size_t)rows * pitch);
    std::vector<uint16_t> frac((size_t)rows * pitch);
    rect_fixed_map(map_x, map_y, rows, cols, xy.data(), frac.data());
    RectJob J;
    J.xy = xy.data();
    J.frac = frac.data();
    J.rows = rows;
    J.cols = cols;
    J.map_pitch = pitch;
    J.batch = batch;
    unsigned gx, gy;
    rect_grid(rows, cols, batch, &gx, &gy, &J.frames_per_cta);
    J.in = in;
    J.in_step = in_step;
    J.out = out;
    J.out_step = out_step;
    emu_launch2(rectify_kernel, gx, gy, (unsigned)kRectThreads, (size_t)0, J);
}
