// rectify_kernels.cuh -- device code of stereo rectification, util::stereo_rectifier::rectify (util/stereo_rectifier.cc:
// 87-92): cv::remap(src, dst, map_x, map_y, INTER_LINEAR) of 8-bit images with float maps and BORDER_CONSTANT 0.  camera.cu
// launches it; free of host-side CUDA runtime dependencies so that tests/cta_emu can compile the same text for the host.
//
// cv::remap turns float maps into fixed point before it interpolates, and so does the rectifier, once, when it is created:
//   X = cvRound(map_x * 32) (round half to even; a value outside int gives INT_MIN like the x86 conversion),
//   sx = saturate<short>(X >> 5), ax = X & 31, and the same for y.
// A pixel is then (sum of tap * w + 2^14) >> 15 with the exact integer weights (32 - ax)(32 - ay) * 32, ax (32 - ay) * 32,
// (32 - ax) ay * 32 and ax ay * 32 of the taps (sx, sy), (sx + 1, sy), (sx, sy + 1), (sx + 1, sy + 1); a tap outside the
// source reads 0.
#pragma once
#include <stddef.h>
#include <stdint.h>

namespace plp {

// one output pixel's source corner and fractions: frac = ay * 32 + ax (OpenCV's layout)
struct RectEntry {
    int16_t sx, sy;
    uint16_t frac;
};

__host__ __device__ inline int rect_fixed(float m) {
    const float v = m * 32.0f;
    if (!(v >= -2147483648.0f && v < 2147483648.0f)) return INT32_MIN;  // also NaN
    return (int)rintf(v);
}

__host__ __device__ inline int16_t rect_sat16(int v) { return (int16_t)(v < -32768 ? -32768 : v > 32767 ? 32767 : v); }

__host__ __device__ inline RectEntry rect_entry(float mx, float my) {
    const int X = rect_fixed(mx), Y = rect_fixed(my);
    RectEntry e;
    e.sx = rect_sat16(X >> 5);
    e.sy = rect_sat16(Y >> 5);
    e.frac = (uint16_t)((Y & 31) * 32 + (X & 31));
    return e;
}

constexpr int kRectPx = 4;                       // adjacent output pixels per thread: one 32-bit store
constexpr int kRectTileW = 64;                   // output tile: 64 x 8 pixels per CTA
constexpr int kRectTileH = 8;
constexpr int kRectThreads = (kRectTileW / kRectPx) * kRectTileH;  // 128
constexpr int kRectFramesPerCta = 16;            // frames of the batch one CTA rectifies through its tile's map entries

inline int rect_map_pitch(int cols) { return (cols + kRectPx - 1) / kRectPx * kRectPx; }

// The fixed-point map of one side from its rows x cols float maps: rows x rect_map_pitch(cols) entries, the padding past
// `cols` pointing outside every image.
inline void rect_fixed_map(const float *map_x, const float *map_y, int rows, int cols, short2 *xy, uint16_t *frac) {
    const int pitch = rect_map_pitch(cols);
    for (int i = 0; i < rows; ++i)
        for (int j = 0; j < pitch; ++j) {
            const size_t m = (size_t)i * cols + j, o = (size_t)i * pitch + j;
            const RectEntry e = j < cols ? rect_entry(map_x[m], map_y[m]) : RectEntry{-32768, -32768, 0};
            xy[o] = short2{e.sx, e.sy};
            frac[o] = e.frac;
        }
}

// The launch: grid (div_up(cols, 64), tiles_y * chunks); blockIdx.y = chunk * tiles_y + tile row, and chunk c owns frames
// [c * frames_per_cta, (c + 1) * frames_per_cta) of the batch.  A chunk is kRectFramesPerCta frames unless the batch needs
// more than grid.y allows.
inline void rect_grid(int rows, int cols, int batch, unsigned *grid_x, unsigned *grid_y, int *frames_per_cta) {
    const int tiles_y = (rows + kRectTileH - 1) / kRectTileH, max_chunks = 65535 / tiles_y;
    int f = (batch + max_chunks - 1) / max_chunks;
    f = f < kRectFramesPerCta ? kRectFramesPerCta : f;
    *frames_per_cta = f;
    *grid_x = (unsigned)((cols + kRectTileW - 1) / kRectTileW);
    *grid_y = (unsigned)(tiles_y * ((batch + f - 1) / f));
}

struct RectJob {
    const short2 *xy;      // map_rows x map_pitch corners (sx, sy)
    const uint16_t *frac;  // map_rows x map_pitch fractions
    int rows, cols, map_pitch;  // map_pitch = cols rounded up to kRectPx; padding entries lie outside every image
    int batch, frames_per_cta;  // see rect_grid
    const uint8_t *in;     // frame b at in + b * rows * in_step
    size_t in_step;
    uint8_t *out;          // frame b at out + b * rows * out_step; out and out_step multiples of 4
    size_t out_step;
};

namespace {

// One CTA owns one 64 x 8 output tile of one side and loops over a chunk of the batch's frames: all frames of a side
// share the map, so a tile's entries are read once per chunk.  Each thread forms 4 adjacent pixels and stores them as one
// word; the last word of a row whose width is not a multiple of 4 is stored byte by byte, so nothing past `cols` is
// written.
__global__ void __launch_bounds__(kRectThreads) rectify_kernel(RectJob J) {
    const int t = (int)threadIdx.x;
    const int tiles_y = (J.rows + kRectTileH - 1) / kRectTileH;
    const int chunk = (int)blockIdx.y / tiles_y;
    const int x0 = (int)blockIdx.x * kRectTileW + (t % (kRectTileW / kRectPx)) * kRectPx;
    const int y = ((int)blockIdx.y - chunk * tiles_y) * kRectTileH + t / (kRectTileW / kRectPx);
    if (x0 >= J.cols || y >= J.rows) return;
    const int b0 = chunk * J.frames_per_cta, b1 = min(J.batch, b0 + J.frames_per_cta);
    const size_t mi = (size_t)y * J.map_pitch + x0;
    int sx[kRectPx], sy[kRectPx], ax[kRectPx], ay[kRectPx];
#pragma unroll
    for (int k = 0; k < kRectPx; ++k) {
        const short2 c = __ldg(J.xy + mi + k);
        const int f = __ldg(J.frac + mi + k);
        sx[k] = c.x;
        sy[k] = c.y;
        ax[k] = f & 31;
        ay[k] = f >> 5;
    }
    const unsigned W = (unsigned)J.cols, H = (unsigned)J.rows;
    const size_t in_frame = (size_t)J.rows * J.in_step, out_frame = (size_t)J.rows * J.out_step;
    const bool full = x0 + kRectPx <= J.cols;
    for (int b = b0; b < b1; ++b) {
        const uint8_t *src = J.in + (size_t)b * in_frame;
        uint32_t word = 0;
#pragma unroll
        for (int k = 0; k < kRectPx; ++k) {
            const int x = sx[k], yy = sy[k];
            const bool x_in0 = (unsigned)x < W, x_in1 = (unsigned)(x + 1) < W;
            const bool y_in0 = (unsigned)yy < H, y_in1 = (unsigned)(yy + 1) < H;
            const uint8_t *r0 = src + (ptrdiff_t)yy * (ptrdiff_t)J.in_step + x;
            const uint8_t *r1 = r0 + J.in_step;
            const int v00 = (y_in0 && x_in0) ? __ldg(r0) : 0;
            const int v01 = (y_in0 && x_in1) ? __ldg(r0 + 1) : 0;
            const int v10 = (y_in1 && x_in0) ? __ldg(r1) : 0;
            const int v11 = (y_in1 && x_in1) ? __ldg(r1 + 1) : 0;
            const int bx = ax[k], by = ay[k];
            const int s = v00 * ((32 - bx) * (32 - by) * 32) + v01 * (bx * (32 - by) * 32) +
                          v10 * ((32 - bx) * by * 32) + v11 * (bx * by * 32);
            word |= (uint32_t)((s + (1 << 14)) >> 15) << (8 * k);
        }
        uint8_t *dst = J.out + (size_t)b * out_frame + (size_t)y * J.out_step + x0;
        if (full) {
            *reinterpret_cast<uint32_t *>(dst) = word;
        } else {
            for (int k = 0; x0 + k < J.cols; ++k) dst[k] = (uint8_t)(word >> (8 * k));
        }
    }
}

}  // namespace

}  // namespace plp
