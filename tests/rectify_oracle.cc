// rectify_oracle.cc -- the CPU oracle of stereo rectification (TEST INFRASTRUCTURE ONLY; __graft_entry__.build() compiles it
// into oracle/_build/librectify_oracle.so, tests/rectify_data.py loads it).
//
//   orc_rect_maps: util::stereo_rectifier's maps, compiled from the library's rectmath.h text (pinned to cv2 by
//                  test_rectify_oracle.py).
//   orc_remap_linear_u8: cv::remap(INTER_LINEAR, BORDER_CONSTANT 0) of an 8-bit image with float maps, restated here from
//                  OpenCV's fixed-point rule without the kernel header's code.
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#include "rectmath.h"

extern "C" int orc_rect_maps(int model, const double *K, const double *D, const double *R, const double *Kr, int rows,
                             int cols, float *map_x, float *map_y) {
    return rect_build_maps(model, K, D, R, Kr, rows, cols, map_x, map_y);
}

// cvRound of a float as the x86 conversion does it: round half to even, INT_MIN for anything outside int (and NaN)
static long long cv_round_f(float v) {
    if (!(v >= -2147483648.0f && v < 2147483648.0f)) return -2147483648ll;
    return (long long)nearbyintf(v);
}

static int sat_short(long long v) { return v < -32768 ? -32768 : v > 32767 ? 32767 : (int)v; }

// src: rows x cols (row stride step); map_x, map_y, dst: out_rows x out_cols (dst row stride out_step)
extern "C" void orc_remap_linear_u8(const uint8_t *src, int rows, int cols, size_t step, const float *map_x,
                                    const float *map_y, int out_rows, int out_cols, uint8_t *dst, size_t out_step) {
    for (int i = 0; i < out_rows; ++i)
        for (int j = 0; j < out_cols; ++j) {
            const size_t m = (size_t)i * out_cols + j;
            const long long X = cv_round_f(map_x[m] * 32.0f), Y = cv_round_f(map_y[m] * 32.0f);
            const long long sx = sat_short(X >> 5), sy = sat_short(Y >> 5);
            const long long ax = X & 31, ay = Y & 31;
            const long long w[4] = {(32 - ax) * (32 - ay) * 32, ax * (32 - ay) * 32, (32 - ax) * ay * 32, ax * ay * 32};
            long long s = 0;
            for (int t = 0; t < 4; ++t) {
                const long long x = sx + (t & 1), y = sy + (t >> 1);
                const int v = (x >= 0 && x < cols && y >= 0 && y < rows) ? src[(size_t)y * step + (size_t)x] : 0;
                s += v * w[t];
            }
            long long o = (s + (1 << 14)) >> 15;
            dst[(size_t)i * out_step + j] = (uint8_t)(o < 0 ? 0 : o > 255 ? 255 : o);
        }
}
