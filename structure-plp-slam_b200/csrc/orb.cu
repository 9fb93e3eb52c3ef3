// orb.cu -- ORB extraction on sm_90a: pyramid -> per-cell FAST -> quadtree selection -> orientation ->
// 7x7 Gaussian -> steered BRIEF.  Replaces feature::orb_extractor::extract (feature/orb_extractor.cc:73-160
// and the helpers it calls, orb_extractor_node.cc:31-80, util/trigonometric.h:42-78) bit-exactly.
//
// Batched from day one: every kernel has the frame index as its outermost grid dimension, so one launch
// covers `batch` frames.  10 launches per batch:
//   7 x pyr_resize_kernel     level l from level l-1 (chained like orb_extractor.cc:315-326), OpenCV's
//                             11-bit fixed-point bilinear
//   1 x fast_cells_kernel     a run of 64-px cells per CTA (6-px overlap, orb_extractor.cc:338-437): tile -> smem,
//                             FAST-9/16 score, 3x3 NMS at the initial threshold, fallback to the minimum
//                             threshold if the cell is empty, ordered compaction (row-major inside the cell)
//   1 x quadtree_kernel       one CTA per (level, frame): data-parallel formulation of
//                             distribute_keypoints_via_tree (see tools/quadtree_parallel_model.py)
//   1 x describe_kernel       a run of keypoints per warp, disc and blurred window staged by cp.async:
//                             intensity-centroid angle on DP4A -> 256 steered comparisons, one descriptor byte per lane
// Compiled with -fmad=false: the f32 steering must round exactly like the oracle (no FMA).
#include "common.cuh"
#include <cuda.h>  // CUtensorMap (types only: the encoder is fetched with cudaGetDriverEntryPoint, no libcuda link)
#include <stdlib.h>
// describe_kernel reads the pattern tables as uint2, so they are 16-byte aligned
#define PLP_BRIEF_TABLE __device__ const signed char __align__(16)
#include "brief_pattern.inc"
#include "quadtree_kernels.cuh"

namespace plp {

namespace {

constexpr int kMaxLevels = 16;
constexpr int kHalfPatch = 15;     // orb_extractor.h:158 fast_half_patch_size_
constexpr int kCellSize = 64;      // orb_extractor.cc:339
constexpr int kOverlap = 6;        // orb_extractor.cc:338

struct LevelInfo {
    int w, h, pitch;
    size_t offset;        // byte offset of the level inside one frame's pyramid block (levels >= 1)
    size_t blur_offset;   // byte offset of the level inside one frame's blurred-pyramid block (all levels)
    int cells_x, cells_y; // number of cell columns/rows visited (orb_extractor.cc:356-357)
    int cell_base;        // index of this level's first cell in the per-frame cell list
    int num_cells;
    int budget;           // num_keypts_per_level_
    int slot_base;        // first output slot of this level (per-level keypoint lists)
    int slot_cap;
    float scale_factor;
    float size;           // keypoint size = (unsigned)(31 * scale)
};

struct CellDesc {
    short level, i, j, pad;
    short min_x, min_y, max_x, max_y;
};

struct BlurTile {  // one 64 x 32 output tile of the Gaussian-blurred pyramid
    short level, x0, y0, pad;
};

struct OrbDev {
    int num_levels, rows, cols;
    int num_cells;       // per frame
    int total_slots;     // per frame
    int out_cap;         // per frame capacity of the final kp/desc arrays
    int ini_thr, min_thr;
    LevelInfo lv[kMaxLevels];
    int u_max[16];
    // per-batch inputs
    const uint8_t *img0;  // level 0 = the caller's images
    size_t img0_step, img0_frame_stride;
    const uint8_t *mask;  // optional, level-0 resolution, shared by the batch
    size_t mask_step;
    // device work areas
    uint8_t *pyr;  // batch x pyr_frame_bytes (levels >= 1)
    size_t pyr_frame_bytes;
    uint8_t *blur;  // batch x blur_frame_bytes: GaussianBlur(7x7, sigma 2) of every level (orb_extractor.cc:148-149)
    size_t blur_frame_bytes;
    const BlurTile *blur_tiles;
    int num_blur_tiles;
    const CellDesc *cells;
    uint32_t *cell_buf;   // batch x num_cells x kCellCap packed (x:11 | y:10 | score:8)
    int *cell_cnt;        // batch x num_cells
    LevelKp *lvl_kp;      // batch x total_slots
    int *lvl_cnt;         // batch x num_levels
    uint8_t *qt_scratch;  // global fallback work area of the quadtree kernel
    size_t qt_scratch_per_job;
    int *status;          // batch: != 0 on capacity overflow
};

__device__ __forceinline__ const uint8_t *level_ptr(const OrbDev &P, int b, int l) {
    return l == 0 ? P.img0 + (size_t)b * P.img0_frame_stride : P.pyr + (size_t)b * P.pyr_frame_bytes + P.lv[l].offset;
}
__device__ __forceinline__ int level_pitch(const OrbDev &P, int l) { return l == 0 ? (int)P.img0_step : P.lv[l].pitch; }

// ---- TMA staging of pyramid tiles (Gaussian blur and FAST) -----------------------------------------------------------
// Every level is described as an (x, y, frame) uint8 tensor (plp_orb::maps) with one box shape, kBoxW x kBoxH x 1: the
// source box of a 64 x 32 blur tile.  The innermost coordinate of a tiled copy must be a multiple of 16 BYTES (an
// unaligned x is an illegal instruction); any y -- negative included -- is accepted, and out-of-image elements arrive
// as zeros.
constexpr int kBtW = 64, kBtH = 32;  // blur output tile
constexpr int kBoxW = 96, kBoxH = kBtH + 6, kBoxX = 16;  // the box starts kBoxX columns left of the blur tile
static_assert(kBoxW >= kBoxX + kBtW + 3 && kBoxW % 16 == 0 && kBoxX % 16 == 0 && kBtW % 16 == 0,
              "TMA box: 16-byte aligned start and extent covering the 3-pixel halo");
static_assert(kBoxH % 2 == 0 && kBtH % 2 == 0, "the blur passes work on pairs of rows");
constexpr int kBoxStage = (kBoxH * kBoxW + 127) & ~127;  // a box in a shared-memory ring (TMA destinations: 128-byte aligned)
// FAST tiles (section 2): a cell's 70 rows of up to 70 pixels in two boxes, tile rows at the box pitch
constexpr int kTilePitch = kBoxW;
constexpr int kTileRows = kCellSize + kOverlap;

struct BlurMaps {
    CUtensorMap m[kMaxLevels];
};

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar) { asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar)); }

// bounded wait for phase `parity` of an mbarrier; false if it did not complete (the copy never arrived)
__device__ __forceinline__ bool mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t done = 0;
    for (int spin = 0; spin < (1 << 14) && !done; ++spin)
        asm volatile(
            "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(bar), "r"(parity)
            : "memory");
    return done != 0;
}

// thread 0 arms `bar` for `bytes` of copies of the current phase (before issuing them)
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}

// one box at (x, y, frame) of tensor `tm` into shared memory at `dst` (128-byte aligned), completing on `bar`
__device__ __forceinline__ void tma_box_load(uint32_t dst, const CUtensorMap *tm, int x, int y, int f, uint32_t bar) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
        ::"r"(dst), "l"(tm), "r"(x), "r"(y), "r"(f), "r"(bar)
        : "memory");
}

// =====================================================================================================
// 1. pyramid: cv::resize(INTER_LINEAR) fixed-point model (SURVEY.md Appendix A.1)
// =====================================================================================================
// tables: per destination column {sx0, sx1, a0, a1}, per destination row {sy0, sy1, b0, b1}
// A thread owns four destination columns of kResizeRows consecutive rows: the column taps and weights are row-independent,
// so they are unpacked once per strip (round 1 redid the table loads, the unpacking and the 64-bit address arithmetic for
// every row: 58 instructions per pixel).
constexpr int kResizeRows = 8;
__global__ void __launch_bounds__(256) pyr_resize_kernel(OrbDev P, int l, const short4 *__restrict__ xtab,
                                                         const short4 *__restrict__ ytab) {
    const int b = blockIdx.y;
    const int dw = P.lv[l].w, dh = P.lv[l].h, dpitch = P.lv[l].pitch;
    const int quads = (dw + 3) >> 2, strips = (dh + kResizeRows - 1) / kResizeRows;
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= quads * strips) return;
    const int strip = q / quads, x0 = (q - strip * quads) * 4;
    const uint8_t *src = level_ptr(P, b, l - 1);
    const int spitch = level_pitch(P, l - 1);
    uint8_t *dst = const_cast<uint8_t *>(level_ptr(P, b, l));
    int sx0[4], sx1[4], a0[4], a1[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const short4 xt = xtab[min(x0 + k, dw - 1)];  // columns past dw are row padding: any value may be stored there
        sx0[k] = xt.x;
        sx1[k] = xt.y;
        a0[k] = xt.z;
        a1[k] = xt.w;
    }
    const int y_end = min(dh, (strip + 1) * kResizeRows);
    for (int y = strip * kResizeRows; y < y_end; ++y) {
        const short4 yt = ytab[y];
        const uint8_t *S0 = src + (size_t)yt.x * spitch, *S1 = src + (size_t)yt.y * spitch;
        const int b0 = yt.z, b1 = yt.w;
        uint32_t packed = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int r0 = S0[sx0[k]] * a0[k] + S0[sx1[k]] * a1[k];
            const int r1 = S1[sx0[k]] * a0[k] + S1[sx1[k]] * a1[k];
            const int v = (((b0 * (r0 >> 4)) >> 16) + ((b1 * (r1 >> 4)) >> 16) + 2) >> 2;
            packed |= (uint32_t)(v & 0xff) << (8 * k);
        }
        // pitch is a multiple of 64 so the 4-byte store is aligned; pad bytes past dw are never read
        *reinterpret_cast<uint32_t *>(dst + (size_t)y * dpitch + x0) = packed;
    }
}

// =====================================================================================================
// 2. FAST-9/16 per cell
// =====================================================================================================
// FAST-9/16 ring (SURVEY.md Appendix A.2): offsets (dx, dy) of ring pixel k = 0 .. 15, starting below the centre, counter-clockwise:
//   (0,3) (1,3) (2,2) (3,1) (3,0) (3,-1) (2,-2) (1,-3) (0,-3) (-1,-3) (-2,-2) (-3,-1) (-3,0) (-3,1) (-2,2) (-1,3)
// m = max over the sixteen 9-arcs of min(arc differences), both polarities (d = v - ring for dark arcs, e = ring - v for bright
// ones); the sliding minimum of length 9 over the circular ring is built by doubling (2, 4, 4 + 4 + 1).  Written with minima
// and a bias instead of negations: ptxas 12.9 for sm_100a was seen to drop the negation of max(a, -max(...)) when fusing
// it into VIMNMX3 (not re-checked for sm_90a, which has the same instruction), see DESIGN.md.
// The score of TWO pixels at once on packed 16-bit halves (DPX min / max, VIMNMX3.S16x2): every difference is biased
// by +256 so that both halves stay in [1, 511] -- plain 32-bit subtraction then never borrows across the halves and no
// negation is needed (e' = 512 - d').  Returns (m_a + 256) | (m_b + 256) << 16 with m = max over the sixteen 9-arcs of
// min(arc differences), both polarities; the pixel is a corner at threshold t  <=>  m > t  (a 9-arc whose pixels all
// differ by more than t has a minimum above t and vice versa), which is the FAST-9 arc test.
__device__ __forceinline__ uint32_t fast_m_pair(const uint8_t *pa, const uint8_t *pb) {
    const uint32_t v2 = ((uint32_t)pa[0] + 256u) | (((uint32_t)pb[0] + 256u) << 16);
    uint32_t d[16];
#define PLP_RING(k, off) d[k] = v2 - ((uint32_t)pa[off] | ((uint32_t)pb[off] << 16))
    PLP_RING(0, 3 * kTilePitch);
    PLP_RING(1, 3 * kTilePitch + 1);
    PLP_RING(2, 2 * kTilePitch + 2);
    PLP_RING(3, 1 * kTilePitch + 3);
    PLP_RING(4, 3);
    PLP_RING(5, -1 * kTilePitch + 3);
    PLP_RING(6, -2 * kTilePitch + 2);
    PLP_RING(7, -3 * kTilePitch + 1);
    PLP_RING(8, -3 * kTilePitch);
    PLP_RING(9, -3 * kTilePitch - 1);
    PLP_RING(10, -2 * kTilePitch - 2);
    PLP_RING(11, -1 * kTilePitch - 3);
    PLP_RING(12, -3);
    PLP_RING(13, 1 * kTilePitch - 3);
    PLP_RING(14, 2 * kTilePitch - 2);
    PLP_RING(15, 3 * kTilePitch - 1);
#undef PLP_RING
    uint32_t e[16], d2[16], e2[16], d4[16], e4[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) e[k] = 0x02000200u - d[k];
#pragma unroll
    for (int k = 0; k < 16; ++k) {
        d2[k] = __vimin3_s16x2(d[k], d[(k + 1) & 15], d[(k + 1) & 15]);
        e2[k] = __vimin3_s16x2(e[k], e[(k + 1) & 15], e[(k + 1) & 15]);
    }
#pragma unroll
    for (int k = 0; k < 16; ++k) {
        d4[k] = __vimin3_s16x2(d2[k], d2[(k + 2) & 15], d2[(k + 2) & 15]);
        e4[k] = __vimin3_s16x2(e2[k], e2[(k + 2) & 15], e2[(k + 2) & 15]);
    }
    uint32_t best = 0u;
#pragma unroll
    for (int k = 0; k < 16; ++k) {
        const uint32_t d9 = __vimin3_s16x2(d4[k], d4[(k + 4) & 15], d[(k + 8) & 15]);
        const uint32_t e9 = __vimin3_s16x2(e4[k], e4[(k + 4) & 15], e[(k + 8) & 15]);
        best = __vimax3_s16x2(best, d9, e9);
    }
    return best;
}

__device__ __forceinline__ bool masked(const OrbDev &P, unsigned y, unsigned x, float scale) {
    // orb_extractor.cc:333-336 is_in_mask
    return P.mask[(size_t)(int)(y * scale) * P.mask_step + (int)(x * scale)] == 0;
}


// ---------------------------------------------------------------------------------------------------------------
// FAST cells: same cell semantics as cv::FAST per cell, few instructions per pixel.
//   phase A  four tested pixels per lane, a row per 16 lanes; the pretest is a necessary condition for a FAST-9 corner
//            evaluated with the native VABSDIFF4 byte SIMD (even8_4, or compass4 for thresholds >= 128), phase B decides
//            exactly;
//   phase B  the exact score of the survivors, two per thread; corners set their bit in a corner bitmap;
//   NMS      only over the corners, reading the score of a neighbour only when its corner bit is set (the score tile is
//            never cleared); survivors set bits in the per-(row, half) masks with atomicOr -- a bit mask is order
//            independent, so the row-major output order is unchanged;
//   output   one thread per mask word walks its set bits at a position from a per-warp scan of the word counts.
// One tile layout for both ways a tile arrives (fast_cells_tma_kernel, fast_cells_kernel_v2): kTileRows x kTilePitch
// bytes, cell column 0 at tile column kTileX.  Cells start at x = 19 + 64 j, so a cell's row minus kTileX = 3 pixels
// starts on a 16-byte boundary (the alignment TMA needs), and tested column 0 (cell column 3) is tile column 6: the
// centre word of four tested pixels is a funnel shift of two aligned words.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kTileX = kPatchRadius % 16;
constexpr int kTestX = kTileX + 3;  // tile column of tested column 0
static_assert(kCellSize % 16 == 0 && kTestX % 4 == 2, "the pretests below form their words for tested x = 2 (mod 4)");
static_assert(kTileX + kCellSize + kOverlap <= kTilePitch, "a cell row fits a tile row");
constexpr int kFastBox2Row = kTileRows - kBoxH;  // the second box of a cell: tile rows kFastBox2Row .. kTileRows - 1
static_assert(kFastBox2Row > 0 && kFastBox2Row <= kBoxH && (kFastBox2Row * kTilePitch) % 128 == 0,
              "two boxes cover the tile rows; the second lands 128-byte aligned");
constexpr int kFastStage = (kTileRows * kTilePitch + 127) & ~127;
constexpr int kCornerWords = 4;  // corner bitmap words per tile row: kTilePitch bits + one word for the 3-bit windows
static_assert(kCornerWords * 32 >= kTilePitch + 32, "corner bitmap row");

// aligned 32-bit word k of tile row y
#define PLP_TW(y, k) T32[(y) * (kTilePitch / 4) + (k)]

// Compass pretest (thresholds >= 128): two ADJACENT compass pixels differ from the centre by more than t.  Pixels
// X .. X + 3 with X = 4 k + 2; returns their bits in a nibble.
__device__ __forceinline__ uint32_t compass4(const uint32_t *T32, int y, int k, uint32_t t4) {
    const uint32_t c = __funnelshift_r(PLP_TW(y, k), PLP_TW(y, k + 1), 16);
    const uint32_t up = __funnelshift_r(PLP_TW(y - 3, k), PLP_TW(y - 3, k + 1), 16);
    const uint32_t dn = __funnelshift_r(PLP_TW(y + 3, k), PLP_TW(y + 3, k + 1), 16);
    const uint32_t lf = __funnelshift_r(PLP_TW(y, k - 1), PLP_TW(y, k), 24);      // bytes X-3 .. X
    const uint32_t rt = __funnelshift_r(PLP_TW(y, k + 1), PLP_TW(y, k + 2), 8);   // bytes X+3 .. X+6
    const uint32_t a0 = __vcmpgtu4(__vabsdiffu4(c, dn), t4), a4 = __vcmpgtu4(__vabsdiffu4(c, rt), t4);
    const uint32_t a8 = __vcmpgtu4(__vabsdiffu4(c, up), t4), a12 = __vcmpgtu4(__vabsdiffu4(c, lf), t4);
    const uint32_t sv = (a4 | a12) & (a0 | a8);  // the four adjacent pairs (0,4) (4,8) (8,12) (12,0)
    const uint32_t m = sv & 0x01010101u;
    return (m | (m >> 7) | (m >> 14) | (m >> 21)) & 0xfu;
}

// Stronger byte-SIMD pretest (thresholds < 128): a 9-arc covers at least FOUR CONSECUTIVE of the eight even ring pixels
// (0, 2, .., 14), which must then all differ from the centre by more than t -- a necessary condition for a FAST-9 corner
// that rejects about three times as many pixels as the compass pair, so that the scalar arc test (250 instructions)
// runs on few of them.  |ring - c| with the native VABSDIFF4; "byte > t" as ((x & 0x7f) + (0x7f - t) | x) & 0x80.
// With X = 4 k + 2 the diagonal pixels (+-2, +-2) are aligned words.
__device__ __forceinline__ uint32_t even8_4(const uint32_t *T32, int y, int k, uint32_t k7) {
    const uint32_t c = __funnelshift_r(PLP_TW(y, k), PLP_TW(y, k + 1), 16);
    auto gt = [&](uint32_t ring) -> uint32_t {
        const uint32_t d = __vabsdiffu4(c, ring);
        return (((d & 0x7f7f7f7fu) + k7) | d) & 0x80808080u;
    };
    const uint32_t e0 = gt(__funnelshift_r(PLP_TW(y + 3, k), PLP_TW(y + 3, k + 1), 16));  // ( 0, +3)
    const uint32_t e2 = gt(PLP_TW(y + 2, k + 1));                                        // (+2, +2)
    const uint32_t e4 = gt(__funnelshift_r(PLP_TW(y, k + 1), PLP_TW(y, k + 2), 8));      // (+3,  0)
    const uint32_t e6 = gt(PLP_TW(y - 2, k + 1));                                        // (+2, -2)
    const uint32_t e8 = gt(__funnelshift_r(PLP_TW(y - 3, k), PLP_TW(y - 3, k + 1), 16));  // ( 0, -3)
    const uint32_t e10 = gt(PLP_TW(y - 2, k));                                           // (-2, -2)
    const uint32_t e12 = gt(__funnelshift_r(PLP_TW(y, k - 1), PLP_TW(y, k), 24));        // (-3,  0)
    const uint32_t e14 = gt(PLP_TW(y + 2, k));                                           // (-2, +2)
    const uint32_t p0 = e0 & e2, p2 = e2 & e4, p4 = e4 & e6, p6 = e6 & e8, p8 = e8 & e10, p10 = e10 & e12, p12 = e12 & e14,
                   p14 = e14 & e0;
    const uint32_t r = (p0 & p4) | (p2 & p6) | (p4 & p8) | (p6 & p10) | (p8 & p12) | (p10 & p14) | (p12 & p0) | (p14 & p2);
    return ((r >> 7) | (r >> 14) | (r >> 21) | (r >> 28)) & 0xfu;
}
#undef PLP_TW

struct FastSmem {
    uint8_t score[kTileRows * kTilePitch];  // valid where the corner bit is set
    unsigned corner[kTileRows * kCornerWords];
    unsigned short list[kCellSize * kCellSize];  // pretest survivors, (tile row << 7) | tile column
    unsigned rowbits[128];  // NMS survivors: one 32-bit mask per (tested row, 32-column half)
    int rowbase[128];       // exclusive prefix of the mask counts inside the mask's warp
    int wsum[4];            // mask counts per warp
    int nsurv;
};

// the state fast_cell_detect expects on entry and leaves for the next cell (fast_cell_emit clears the masks it reads)
__device__ __forceinline__ void fast_smem_clear(FastSmem &S) {
    for (int i = threadIdx.x; i < kTileRows * kCornerWords; i += blockDim.x) S.corner[i] = 0u;
    if (threadIdx.x < 128) S.rowbits[threadIdx.x] = 0u;
    if (threadIdx.x == 0) S.nsurv = 0;
}

// FAST-9 corners of cell ci of frame b after 3x3 NMS, with the initial threshold or, if that leaves none, the minimum
// one (orb_extractor.cc:395-437): the survivors' masks in S.rowbits, their scores in S.score and the warp-local prefix
// of the mask counts in S.rowbase / S.wsum.  The tile must be complete and visible to every thread.
__device__ __forceinline__ void fast_cell_detect(const OrbDev &P, int ci, const uint8_t *tile, FastSmem &S) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const CellDesc cell = P.cells[ci];
    const int w = cell.max_x - cell.min_x, h = cell.max_y - cell.min_y;
    const float scale = P.lv[cell.level].scale_factor;
    bool skip = (w < 7 || h < 7);
    if (!skip && P.mask) {  // orb_extractor.cc:395-401
        skip = masked(P, cell.min_y, cell.min_x, scale) || masked(P, cell.max_y, cell.min_x, scale) ||
               masked(P, cell.min_y, cell.max_x, scale) || masked(P, cell.max_y, cell.max_x, scale);
    }
    const int tw = w - 6, th = h - 6;  // tested area: rows 3 .. h-4, columns 3 .. w-4 (<= 64 x 64)
    const uint32_t *T32 = reinterpret_cast<const uint32_t *>(tile);
    for (int pass = 0; !skip; ++pass) {
        const int thr = pass == 0 ? P.ini_thr : P.min_thr;
        const uint32_t t4 = (uint32_t)min(thr, 255) * 0x01010101u;
        const bool strong = thr < 128;  // the SWAR "byte > t" of even8_4 needs t < 128
        const uint32_t k7 = (uint32_t)(0x7f - min(thr, 127)) * 0x01010101u;
        // phase A: a warp takes two rows, a lane the tested columns 4g .. 4g+3 (tile columns X = kTestX + 4g ..)
        for (int rp = warp; rp < (th + 1) / 2; rp += 8) {
            const int ry = 2 * rp + (lane >> 4), g = lane & 15;
            const int nv = tw - 4 * g;  // tested pixels of this lane
            if (ry >= th || nv <= 0) continue;
            const int y = 3 + ry, k = (kTestX >> 2) + g;
            uint32_t nib = (strong ? even8_4(T32, y, k, k7) : compass4(T32, y, k, t4)) & (nv >= 4 ? 0xfu : (1u << nv) - 1u);
            // the list order is irrelevant (scores and NMS bits are per pixel, the output order comes from the row
            // masks), so a lane reserves its slots with one shared-memory atomic (one atomic per warp, with ballots to
            // rank the lanes, measured slower)
            if (!nib) continue;
            int pos = atomicAdd(&S.nsurv, __popc(nib));
            const int p0 = (y << 7) + kTestX + 4 * g;
            while (nib) {
                const int bit = __ffs(nib) - 1;
                nib &= nib - 1;
                S.list[pos++] = (unsigned short)(p0 + bit);
            }
        }
        __syncthreads();
        // phase B: exact arc test / score, two survivors per thread (packed 16-bit halves)
        const int nsurv = S.nsurv;
        {
            const int half = (nsurv + 1) >> 1;
            for (int i = tid; i < half; i += 256) {
                const int pa = S.list[i];
                const bool has_b = i + half < nsurv;
                const int pb = has_b ? S.list[i + half] : pa;
                const int off_a = (pa >> 7) * kTilePitch + (pa & 127), off_b = (pb >> 7) * kTilePitch + (pb & 127);
                const uint32_t m2 = fast_m_pair(tile + off_a, tile + off_b);
                const int m_a = (int)(m2 & 0xffffu) - 256, m_b = (int)(m2 >> 16) - 256;
                if (m_a > thr) {
                    S.score[off_a] = (uint8_t)(m_a - 1);
                    atomicOr(&S.corner[(pa >> 7) * kCornerWords + ((pa & 127) >> 5)], 1u << (pa & 31));
                }
                if (has_b && m_b > thr) {
                    S.score[off_b] = (uint8_t)(m_b - 1);
                    atomicOr(&S.corner[(pb >> 7) * kCornerWords + ((pb & 127) >> 5)], 1u << (pb & 31));
                }
            }
        }
        __syncthreads();
        // 3x3 non-maximum suppression over the corners only; a neighbour without its corner bit scores 0
        bool any_local = false;
        for (int i = tid; i < nsurv; i += 256) {
            const int p = S.list[i];
            const int y = p >> 7, x = p & 127;
            uint32_t nb[3];  // bits x-1 .. x+1 of rows y-1 .. y+1
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                const unsigned *row = S.corner + (y - 1 + r) * kCornerWords + ((x - 1) >> 5);
                nb[r] = __funnelshift_r(row[0], row[1], (x - 1) & 31) & 7u;
            }
            if (!(nb[1] & 2u)) continue;
            const uint8_t *sp = S.score + y * kTilePitch + x;
            const int sc = sp[0];
            bool keep = true;
#pragma unroll
            for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
                for (int dx = -1; dx <= 1; ++dx) {
                    if (dx == 0 && dy == 0) continue;
                    if (nb[dy + 1] & (1u << (dx + 1))) keep = keep && (sc > (int)sp[dy * kTilePitch + dx]);
                }
            if (keep) {
                const int xx = x - kTestX;
                atomicOr(&S.rowbits[(y - 3) * 2 + (xx >> 5)], 1u << (xx & 31));
                any_local = true;
            }
        }
        const int any = __syncthreads_or(any_local);
        // the survivor list and the corner bitmap are free again: cleared for the next pass or cell
        for (int i = tid; i < kTileRows * kCornerWords; i += 256) S.corner[i] = 0u;
        if (tid == 0) S.nsurv = 0;
        if (any || pass == 1 || P.min_thr == P.ini_thr) break;
        __syncthreads();
    }
    // fast_cells_tma_kernel runs the previous cell's fast_cell_emit right before this call, and it reads S.wsum of
    // other warps: the barriers of the passes order those reads before the writes below, and a skipped cell (uniform
    // over the block) needs one of its own
    if (skip) __syncthreads();
    // per-keypoint mask test (orb_extractor.cc:429) and the warp-local scan of the counts: thread t < 128 owns mask t
    // (tested row t >> 1, half t & 1, i.e. row-major order)
    if (tid < 128) {
        unsigned bits = S.rowbits[tid];
        if (P.mask && bits) {
            unsigned keepbits = bits;
            while (bits) {
                const int bit = __ffs(bits) - 1;
                bits &= bits - 1;
                const int x = 3 + (tid & 1) * 32 + bit, y = 3 + (tid >> 1);
                const float kx = (float)x + (float)(cell.j * kCellSize), ky = (float)y + (float)(cell.i * kCellSize);
                if (masked(P, (unsigned)((float)kPatchRadius + ky), (unsigned)((float)kPatchRadius + kx), scale))
                    keepbits &= ~(1u << bit);
            }
            S.rowbits[tid] = bits = keepbits;
        }
        const int c = __popc(bits);
        int incl = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
        }
        S.rowbase[tid] = incl - c;
        if (lane == 31) S.wsum[warp] = incl;
    }
}

// ordered (row-major) output of the cell fast_cell_detect left in S, after a barrier; clears the masks it reads
__device__ __forceinline__ void fast_cell_emit(const OrbDev &P, int b, int ci, FastSmem &S) {
    const int tid = threadIdx.x;
    const CellDesc cell = P.cells[ci];
    if (tid < 128) {
        uint32_t *buf = P.cell_buf + ((size_t)b * P.num_cells + ci) * kCellCap;
        unsigned bits = S.rowbits[tid];
        S.rowbits[tid] = 0u;
        int pos = S.rowbase[tid];
        for (int k = 0; k < (tid >> 5); ++k) pos += S.wsum[k];
        while (bits) {
            const int bit = __ffs(bits) - 1;
            bits &= bits - 1;
            const int x = 3 + (tid & 1) * 32 + bit, y = 3 + (tid >> 1);
            const int sc = S.score[y * kTilePitch + x + kTileX];
            const int lx = x + cell.j * kCellSize, ly = y + cell.i * kCellSize;  // relative to the 19-px border
            if (pos < kCellCap) buf[pos] = (uint32_t)lx | ((uint32_t)ly << 11) | ((uint32_t)sc << 21);
            ++pos;
        }
    }
    if (tid == 0) P.cell_cnt[(size_t)b * P.num_cells + ci] = min(S.wsum[0] + S.wsum[1] + S.wsum[2] + S.wsum[3], kCellCap);
}

// one cell per CTA, the tile by plain loads: the path for caller buffers TMA cannot describe (a base or pitch that is
// not a multiple of 16 bytes).  Level pitches are 64-byte multiples, so with a 16-byte aligned level the
// tile rows are fetched as aligned 16-byte chunks from min_x - kTileX: they read [min_x - 3, min_x + w + 13) at most,
// left of which lie >= 16 border pixels, and max_x + 15 <= cols - 4, so no read leaves the image row.
__global__ void __launch_bounds__(256, 4) fast_cells_kernel_v2(OrbDev P) {
    __shared__ __align__(16) uint8_t tile[kTileRows * kTilePitch];
    __shared__ FastSmem S;
    const int b = blockIdx.y, ci = blockIdx.x, tid = threadIdx.x;
    const CellDesc cell = P.cells[ci];
    const int w = cell.max_x - cell.min_x, h = cell.max_y - cell.min_y;
    const uint8_t *img = level_ptr(P, b, cell.level);
    const int pitch = level_pitch(P, cell.level);
    if ((((uintptr_t)img | (uintptr_t)pitch) & 15) == 0) {
        const int nchunks = (kTileX + w + 15) >> 4;
        for (int idx = tid; idx < h * nchunks; idx += 256) {
            const int y = idx / nchunks, c = idx - y * nchunks;
            const uint4 v = __ldg(reinterpret_cast<const uint4 *>(img + (size_t)(cell.min_y + y) * pitch + (cell.min_x - kTileX)) + c);
            *reinterpret_cast<uint4 *>(tile + y * kTilePitch + 16 * c) = v;
        }
    } else {
        for (int y = tid >> 5; y < h; y += 8) {
            const uint8_t *src = img + (size_t)(cell.min_y + y) * pitch + cell.min_x;
            for (int x = tid & 31; x < w; x += 32) tile[y * kTilePitch + kTileX + x] = src[x];
        }
    }
    fast_smem_clear(S);
    __syncthreads();
    fast_cell_detect(P, ci, tile, S);
    __syncthreads();
    fast_cell_emit(P, b, ci, S);
}

// ---- the same cells with the tiles staged by TMA, a run of cells per CTA ----------------------------------------------
// A CTA takes `run` consecutive cells of one frame (the cell list is level-major, so a run may cross levels).  A cell's
// tile arrives by TWO bulk tensor copies through the level's descriptor (the blur's box, 96 x 38: tile rows 0 .. 37 and
// kFastBox2Row .. 69, the rows in between written twice with the same bytes) into a two-stage ring, one mbarrier per
// stage.  The copy of cell i + 1 is issued before cell i is waited for, and the output of cell i - 1 is written while the
// copy of cell i is in flight.  Out-of-image box elements arrive as zeros; no cell reads them.
// The grid is not persistent: short runs keep CTAs retiring, so that kernels of a concurrent higher-priority stream
// (the tracking of the other sub-batch in the front end) still get SMs.
constexpr int kFastRun = 4;
__global__ void __launch_bounds__(256, 4) fast_cells_tma_kernel(const __grid_constant__ BlurMaps M, OrbDev P, int run) {
    __shared__ __align__(128) uint8_t s_tile[2][kFastStage];
    __shared__ FastSmem S;
    __shared__ __align__(8) unsigned long long s_bar[2];
    const int b = blockIdx.y, tid = threadIdx.x;
    const int first = blockIdx.x * run, n = min(run, P.num_cells - first);
    if (tid == 0) {
        mbar_init(smem_u32(&s_bar[0]));
        mbar_init(smem_u32(&s_bar[1]));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    fast_smem_clear(S);
    __syncthreads();
    auto issue = [&](int i) {  // thread 0: the tile of cell first + i into stage i & 1
        const CellDesc c = P.cells[first + i];
        const uint32_t bar = smem_u32(&s_bar[i & 1]), dst = smem_u32(s_tile[i & 1]);
        const CUtensorMap *tm = &M.m[c.level];
        mbar_expect_tx(bar, 2 * kBoxH * kBoxW);
        tma_box_load(dst, tm, c.min_x - kTileX, c.min_y, b, bar);
        tma_box_load(dst + kFastBox2Row * kTilePitch, tm, c.min_x - kTileX, c.min_y + kFastBox2Row, b, bar);
    };
    if (tid == 0) issue(0);
    for (int i = 0; i < n; ++i) {
        // every thread is past cell i - 1's detection: its stage may be refilled (read through the generic proxy, so the
        // refill by the async proxy is ordered after a fence), and its masks and counts are complete
        __syncthreads();
        if (tid == 0 && i + 1 < n) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            issue(i + 1);
        }
        if (i > 0) fast_cell_emit(P, b, first + i - 1, S);
        // the copy never completed: report it instead of hanging the device
        if (!mbar_wait(smem_u32(&s_bar[i & 1]), (i >> 1) & 1)) P.status[b] = 3;
        fast_cell_detect(P, first + i, s_tile[i & 1], S);
    }
    __syncthreads();
    if (n > 0) fast_cell_emit(P, b, first + n - 1, S);
}

// =====================================================================================================
// 4. orientation + blur + steered BRIEF, a run of keypoints per warp
// =====================================================================================================
constexpr int kDescWarps = 4;
constexpr int kDescRun = 8;  // consecutive output positions per warp run
constexpr int kDescMinBlocks = 5;  // 96 registers, no spills: 20 warps per SM
// A warp stages each keypoint's pixels into a two-stage shared-memory ring, as 16-byte aligned supersets of its rows:
//   disc:   the radius-15 disc of the pyramid level, rows cy - 15 .. cy + 15, 3 chunks (48 B) from (cx - 15) & ~15;
//   window: the blurred level, rows cy - 18 .. cy + 18 (a steered test point is round(x sa + y ca) with |x|, |y| <= 13,
//           at most 18 from the centre), 4 chunks (64 B) from (cx - 18) & ~15.
constexpr int kDiscRows = 2 * kHalfPatch + 1, kDiscPitch = 48;
constexpr int kWinHalf = 18, kWinRows = 2 * kWinHalf + 1, kWinPitch = 64;
constexpr int kDiscBytes = kDiscRows * kDiscPitch;
constexpr int kDescStage = kDiscBytes + kWinRows * kWinPitch;
static_assert(kDiscBytes % 16 == 0 && kDescStage % 16 == 0, "16-byte copies into every row of the ring");
static_assert(15 + kDiscRows <= kDiscPitch && 15 + kWinRows <= kWinPitch, "the aligned supersets fit the rows");

__device__ __forceinline__ int reflect101(int p, int len) {
    if (p < 0) p = -p;
    if (p >= len) p = 2 * (len - 1) - p;
    return p;
}

// cv::fastAtan2 (SURVEY.md Appendix A.7), f32, no FMA
__device__ __forceinline__ float fast_atan2_deg(float y, float x) {
    const float scale = (float)(180.0 / 3.14159265358979323846);
    const float p1 = 0.9997878412794807f * scale, p3 = -0.3258083974640975f * scale,
                p5 = 0.1555786518463281f * scale, p7 = -0.04432655554792128f * scale;
    const float ax = fabsf(x), ay = fabsf(y);
    float a, c, c2;
    if (ax >= ay) {
        c = __fdiv_rn(ay, ax + (float)2.2204460492503131e-16);
        c2 = c * c;
        a = (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
    } else {
        c = __fdiv_rn(ax, ay + (float)2.2204460492503131e-16);
        c2 = c * c;
        a = 90.f - (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
    }
    if (x < 0) a = 180.f - a;
    if (y < 0) a = 360.f - a;
    return a;
}

// util/trigonometric.h:42-78
__device__ __forceinline__ float poly_cos(float v) {
    const float c1 = 0.99940307f, c2 = -0.49558072f, c3 = 0.03679168f;
    const float v2 = v * v;
    return c1 + v2 * (c2 + c3 * v2);
}
__device__ __forceinline__ float util_cos(float v) {
    const float PI = 3.14159265358979f, PI_2 = PI / 2.0f, TWO_PI = 2.0f * PI, INV_TWO_PI = 1.0f / TWO_PI,
                THREE_PI_2 = 3.0f * PI_2;
    v = v - (float)cv_floor((double)(v * INV_TWO_PI)) * TWO_PI;
    v = (0.0f < v) ? v : -v;
    if (v < PI_2) return poly_cos(v);
    if (v < PI) return -poly_cos(PI - v);
    if (v < THREE_PI_2) return -poly_cos(v - PI);
    return poly_cos(TWO_PI - v);
}
__device__ __forceinline__ float util_sin(float v) {
    const float PI_2 = 3.14159265358979f / 2.0f;
    return util_cos(PI_2 - v);
}

// cv::GaussianBlur(level, 7x7, sigma 2, BORDER_REFLECT_101) of every pyramid level (orb_extractor.cc:148-149) in
// OpenCV's fixed-point form: Q8 kernel [18 34 48 56 48 34 18], exact integer passes, (v + 32768) >> 16.
// A 64 x 32 output tile is made from a kBoxW x kBoxH source box in shared memory (box column kBoxX = tile column 0, box
// row 3 = tile row 0): horizontal pass into vertically paired u16 sums, vertical pass, 32-bit stores.  Two kernels fill
// the box: blur_tiles_tma_kernel by TMA bulk tensor copies, blur_tiles_kernel (buffers TMA cannot describe) by plain loads.

// horizontal pass: h2[rp * kBtW + x] = h(2 rp, x) | h(2 rp + 1, x) << 16, where h(py, x) is the 7-tap sum of box row py
// around output column x (<= 255 * 256, a u16).  Output x uses box bytes x + 13 .. x + 19 (image columns x0 + x - 3 ..
// x0 + x + 3); for the outputs 4j .. 4j + 3 that is byte 1 of word j + 3 up to byte 2 of word j + 5, weighted by DP4A with
// (18, 34, 48, 56) and (48, 34, 18, 0) after funnel shifts.  A thread makes 2 rows x 4 columns.
__device__ __forceinline__ void blur_row4(const uint32_t *w, uint32_t h[4]) {
    const uint32_t A = w[0], B = w[1], C = w[2];
    const uint32_t kW1 = 0x38302212u, kW2 = 0x00122230u;  // bytes (18, 34, 48, 56) and (48, 34, 18, 0)
    h[0] = __dp4a(__funnelshift_r(A, B, 8), kW1, __dp4a(__funnelshift_r(B, C, 8), kW2, 0u));
    h[1] = __dp4a(__funnelshift_r(A, B, 16), kW1, __dp4a(__funnelshift_r(B, C, 16), kW2, 0u));
    h[2] = __dp4a(__funnelshift_r(A, B, 24), kW1, __dp4a(__funnelshift_r(B, C, 24), kW2, 0u));
    h[3] = __dp4a(B, kW1, __dp4a(C, kW2, 0u));
}
__device__ __forceinline__ void blur_h_pass(const uint8_t *box, uint32_t *h2) {
    const uint32_t *src32 = reinterpret_cast<const uint32_t *>(box);
    for (int i = threadIdx.x; i < (kBoxH / 2) * (kBtW / 4); i += blockDim.x) {
        const int rp = i / (kBtW / 4), j = i % (kBtW / 4);
        const uint32_t *w = src32 + 2 * rp * (kBoxW / 4) + j + (kBoxX - 4) / 4;
        uint32_t e[4], o[4];
        blur_row4(w, e);
        blur_row4(w + kBoxW / 4, o);
        *reinterpret_cast<uint4 *>(h2 + rp * kBtW + 4 * j) =
            make_uint4(__byte_perm(e[0], o[0], 0x5410), __byte_perm(e[1], o[1], 0x5410), __byte_perm(e[2], o[2], 0x5410),
                       __byte_perm(e[3], o[3], 0x5410));
    }
}

// vertical pass: output rows 2q and 2q + 1 read the pairs q .. q + 3.  With the weights of an output row taken as byte
// pairs, a pixel is four DP2A (u16 pair x u8 pair) into one 32-bit sum started at OpenCV's rounding constant:
//   even row  (18, 34) (48, 56) (48, 34) (18, 0)        odd row  (0, 18) (34, 48) (56, 48) (34, 18)
// The sum is at most 65280 * 256 + 32768 < 2^24, so it is exact and its byte 2 is (acc + 32768) >> 16.  A thread makes
// 2 rows x 4 columns: the 256 threads of the CTA cover the tile in one go.
constexpr int kBlurThreads = 256;
static_assert((kBtH / 2) * (kBtW / 4) == kBlurThreads, "one vertical-pass job per thread");
__device__ __forceinline__ void blur_v_pass(const uint32_t *h2, uint8_t *dst, int dpitch, int x0, int y0, int W, int H) {
    const int q = threadIdx.x / (kBtW / 4), px = (threadIdx.x % (kBtW / 4)) * 4;
    const int y = y0 + 2 * q;
    if (y >= H || x0 + px >= W) return;
    uint32_t r[4][4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const uint4 v = *reinterpret_cast<const uint4 *>(h2 + (q + k) * kBtW + px);
        r[k][0] = v.x;
        r[k][1] = v.y;
        r[k][2] = v.z;
        r[k][3] = v.w;
    }
    auto row = [&](uint32_t k0, uint32_t k1, uint32_t k2, uint32_t k3) -> uint32_t {
        uint32_t a[4];
#pragma unroll
        for (int c = 0; c < 4; ++c)
            a[c] = __dp2a_lo(r[0][c], k0, __dp2a_lo(r[1][c], k1, __dp2a_lo(r[2][c], k2, __dp2a_lo(r[3][c], k3, 32768u))));
        return __byte_perm(__byte_perm(a[0], a[1], 0x0062), __byte_perm(a[2], a[3], 0x0062), 0x5410);
    };
    // pitch is a multiple of 64: aligned 4-byte stores; bytes past the image width are padding
    uint8_t *d = dst + (size_t)y * dpitch + x0 + px;
    *reinterpret_cast<uint32_t *>(d) = row(0x2212u, 0x3830u, 0x2230u, 0x0012u);
    if (y + 1 < H) *reinterpret_cast<uint32_t *>(d + dpitch) = row(0x1200u, 0x3022u, 0x3038u, 0x1222u);
}

// plain loads, one tile per CTA: the box columns the horizontal pass reads (kBoxX - 4 .. kBoxX + kBtW + 3) are gathered
// with BORDER_REFLECT_101 applied to the coordinates
__global__ void __launch_bounds__(kBlurThreads) blur_tiles_kernel(OrbDev P) {
    __shared__ __align__(16) uint8_t s_src[kBoxH * kBoxW];
    __shared__ __align__(16) uint32_t s_h2[(kBoxH / 2) * kBtW];
    const int b = blockIdx.y, tid = threadIdx.x;
    const BlurTile t = P.blur_tiles[blockIdx.x];
    const int l = t.level, W = P.lv[l].w, H = P.lv[l].h;
    const uint8_t *img = level_ptr(P, b, l);
    const int pitch = level_pitch(P, l);
    constexpr int kCols = kBtW + 8;
    for (int i = tid; i < kBoxH * kCols; i += kBlurThreads) {
        const int py = i / kCols, px = i - py * kCols;
        // rows / columns past the image edge + 3 only feed outputs that are never stored, and box column kBoxX - 4 only
        // meets DP4A weight 0: clamp before reflecting
        const int gy = reflect101(min(t.y0 - 3 + py, H + 2), H);
        const int gx = reflect101(min(max(t.x0 - 4 + px, -3), W + 2), W);
        s_src[py * kBoxW + kBoxX - 4 + px] = img[(size_t)gy * pitch + gx];
    }
    __syncthreads();
    blur_h_pass(s_src, s_h2);
    __syncthreads();
    blur_v_pass(s_h2, P.blur + (size_t)b * P.blur_frame_bytes + P.lv[l].blur_offset, P.lv[l].pitch, t.x0, t.y0, W, H);
}

// BORDER_REFLECT_101 inside a TMA box whose tile touches the image border (the mirrored pixels are part of the same box):
// only the (at most) 3 + 3 halo columns and 3 + 3 halo rows the stored outputs read are rebuilt
__device__ void blur_reflect_box(uint8_t *box, int bx0, int by0, int W, int H) {
    for (int i = threadIdx.x; i < kBoxH * 6; i += blockDim.x) {
        const int py = i / 6, k = i - py * 6;
        const int gx = k < 3 ? k - 3 : W + (k - 3), gy = by0 + py;   // image columns -3 .. -1 and W .. W + 2
        const int px = gx - bx0;
        if (gy < 0 || gy >= H || px < 0 || px >= kBoxW) continue;
        box[py * kBoxW + px] = box[py * kBoxW + (reflect101(gx, W) - bx0)];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 6 * kBoxW; i += blockDim.x) {
        const int k = i / kBoxW, px = i - k * kBoxW;
        const int gy = k < 3 ? k - 3 : H + (k - 3);                  // image rows -3 .. -1 and H .. H + 2
        const int py = gy - by0;
        if (py < 0 || py >= kBoxH) continue;
        box[py * kBoxW + px] = box[(reflect101(gy, H) - by0) * kBoxW + px];
    }
    __syncthreads();
}

// ---- the same blur with the source boxes staged by TMA, a run of tiles per CTA --------------------------------------
// A CTA makes `run` consecutive tiles of one frame (the tile list is level-major, row-major inside a level).  Each box
// arrives by ONE bulk tensor copy (box 96 x 38 x 1 of the (x, y, frame) tensor of the level, see tma_box_load) into a
// two-stage shared-memory ring; every stage completes on its own mbarrier.  The copy of tile i + 1 is issued before tile
// i is waited for, so it overlaps the passes of tile i.  The box is the 16-byte aligned superset [x0 - 16, x0 + 80) of
// the 70 columns the tile needs; tiles that touch the image border rebuild BORDER_REFLECT_101 inside the box.
// The grid is not persistent: short runs keep CTAs retiring, so that kernels of a concurrent higher-priority stream
// (the tracking of the other sub-batch in the front end) still get SMs.
// tiles per CTA: 4, 8 and 16 give the same blur time (0.34 ms per 256-frame sub-batch on one H100 80GB HBM3 at 400 W);
// 4 gave the best step time of the front end, whose tracking stream needs SMs while the blur runs
constexpr int kBlurRun = 4;
__global__ void __launch_bounds__(kBlurThreads) blur_tiles_tma_kernel(const __grid_constant__ BlurMaps M, OrbDev P, int run) {
    __shared__ __align__(128) uint8_t s_src[2][kBoxStage];
    __shared__ __align__(16) uint32_t s_h2[(kBoxH / 2) * kBtW];
    __shared__ __align__(8) unsigned long long s_bar[2];
    const int b = blockIdx.y, tid = threadIdx.x;
    const int first = blockIdx.x * run, n = min(run, P.num_blur_tiles - first);
    if (tid == 0) {
        mbar_init(smem_u32(&s_bar[0]));
        mbar_init(smem_u32(&s_bar[1]));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    auto issue = [&](int i) {  // thread 0: the box of tile first + i into stage i & 1
        const BlurTile t = P.blur_tiles[first + i];
        const uint32_t bar = smem_u32(&s_bar[i & 1]);
        mbar_expect_tx(bar, kBoxH * kBoxW);
        tma_box_load(smem_u32(s_src[i & 1]), &M.m[t.level], t.x0 - kBoxX, t.y0 - 3, b, bar);
    };
    if (tid == 0) issue(0);
    for (int i = 0; i < n; ++i) {
        // every thread is past the passes of tile i - 1: its stage and s_h2 may be overwritten.  The stage was read and
        // (border fix-up) written through the generic proxy, so the refill by the async proxy is ordered after a fence.
        __syncthreads();
        if (tid == 0 && i + 1 < n) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            issue(i + 1);
        }
        const BlurTile t = P.blur_tiles[first + i];
        const int l = t.level, W = P.lv[l].w, H = P.lv[l].h;
        const int bx0 = t.x0 - kBoxX, by0 = t.y0 - 3;  // image coordinates of box element (0, 0)
        uint8_t *box = s_src[i & 1];
        // the copy never completed: report it instead of hanging the device
        if (!mbar_wait(smem_u32(&s_bar[i & 1]), (i >> 1) & 1)) P.status[b] = 3;
        if (t.x0 < 3 || by0 < 0 || t.x0 + kBtW + 3 > W || by0 + kBoxH > H) blur_reflect_box(box, bx0, by0, W, H);
        blur_h_pass(box, s_h2);
        __syncthreads();
        blur_v_pass(s_h2, P.blur + (size_t)b * P.blur_frame_bytes + P.lv[l].blur_offset, P.lv[l].pitch, t.x0, t.y0, W, H);
    }
}

__device__ __forceinline__ void cp_async16(void *dst, const void *src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
// every commit group of this thread but the newest has landed
__device__ __forceinline__ void cp_async_wait_prev() { asm volatile("cp.async.wait_group 1;" ::: "memory"); }

// c + the sum of the four products of the unsigned bytes of a and the signed bytes of b
__device__ __forceinline__ int dp4a_us(uint32_t a, uint32_t b, int c) {
    int d;
    asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}

// intensity-centroid sums of one disc row: r = the 12 staged words of the row, whose disc pixel u = -15 is byte
// 4 J + sh / 8; wu / wm = the lane's column weights u and 1 (zero outside |u| <= u_max of the row), one byte per column
template <int J>
__device__ __forceinline__ void disc_row_sums(const uint32_t (&r)[12], int sh, const uint32_t (&wu)[8],
                                              const uint32_t (&wm)[8], int &su, int &si) {
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const uint32_t w = __funnelshift_r(r[J + k], r[J + k + 1], sh);
        su = dp4a_us(w, wu[k], su);
        si = dp4a_us(w, wm[k], si);
    }
}

// A warp describes runs of kDescRun consecutive output positions of one frame (level-major order, orb_extractor.cc:
// 137-159): a run may cross a level boundary and a frame's last run may be partial.  Warps stride on when the frame has
// more keypoints than the grid covers.  The grid is not persistent, so that kernels of a concurrent higher-priority
// stream (the tracking of the other sub-batch in the front end) still get SMs.  Each keypoint's disc and window arrive
// by cp.async into stage i & 1 of the warp's ring; the copies of keypoint i + 1 are issued before keypoint i is waited
// for, so they overlap its description.
__global__ void __launch_bounds__(kDescWarps * 32, kDescMinBlocks) describe_kernel(OrbDev P, plp_keypoint *__restrict__ kp_out,
                                                                    uint8_t *__restrict__ desc_out,
                                                                    int32_t *__restrict__ n_out) {
    __shared__ __align__(16) uint8_t s_ring[kDescWarps][2][kDescStage];
    __shared__ int s_cum[kMaxLevels + 1];
    __shared__ const uint8_t *s_img[kMaxLevels], *s_blur[kMaxLevels];
    __shared__ int s_pitch[kMaxLevels], s_bpitch[kMaxLevels], s_slot[kMaxLevels];
    __shared__ float s_scale[kMaxLevels], s_size[kMaxLevels];
    const int b = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp == 0) {  // per-level lookups: lane l holds level l, the output offsets are a warp scan of the counts
        const int l = lane;
        int c = l < P.num_levels ? P.lvl_cnt[(size_t)b * P.num_levels + l] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, c, o);
            if (lane >= o) c += t;
        }
        if (l == 0) s_cum[0] = 0;
        if (l < kMaxLevels) s_cum[l + 1] = c;
        if (l < P.num_levels) {
            s_img[l] = level_ptr(P, b, l);
            s_pitch[l] = level_pitch(P, l);
            s_blur[l] = P.blur + (size_t)b * P.blur_frame_bytes + P.lv[l].blur_offset;
            s_bpitch[l] = P.lv[l].pitch;
            s_slot[l] = P.lv[l].slot_base;
            s_scale[l] = P.lv[l].scale_factor;
            s_size[l] = P.lv[l].size;
        }
    }
    // the disc of level 0 (the caller's buffer) is copied in 16-byte chunks only if its rows start 16-byte aligned
    const bool vec0 = ((reinterpret_cast<uintptr_t>(P.img0) | P.img0_step | P.img0_frame_stride) & 15) == 0;
    // ic_angle weights of lane v, which owns disc row v - 15 (u_max of orb_extractor.cc:270-286)
    uint32_t wu[8], wm[8];
    {
        const int dv = lane - kHalfPatch, umax = lane < kDiscRows ? P.u_max[dv < 0 ? -dv : dv] : -1;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            wu[k] = wm[k] = 0;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const int u = 4 * k + c - kHalfPatch;
                if (u <= kHalfPatch && (u < 0 ? -u : u) <= umax) {
                    wu[k] |= (uint32_t)(u & 0xff) << (8 * c);
                    wm[k] |= 1u << (8 * c);
                }
            }
        }
    }
    // the lane's 8 BRIEF test pairs as floats (small integers, exact), for every keypoint of the warp; the tables live
    // in global memory: lane-dependent indices into __constant__ memory would serialise
    float x1[8], y1[8], x2[8], y2[8];
    {
        const uint2 px1 = __ldg(reinterpret_cast<const uint2 *>(kBriefX1) + lane), py1 = __ldg(reinterpret_cast<const uint2 *>(kBriefY1) + lane);
        const uint2 px2 = __ldg(reinterpret_cast<const uint2 *>(kBriefX2) + lane), py2 = __ldg(reinterpret_cast<const uint2 *>(kBriefY2) + lane);
#pragma unroll
        for (int bit = 0; bit < 8; ++bit) {
            const int sh = (bit & 3) * 8;
            x1[bit] = (float)(signed char)(((bit < 4 ? px1.x : px1.y) >> sh) & 0xff);
            y1[bit] = (float)(signed char)(((bit < 4 ? py1.x : py1.y) >> sh) & 0xff);
            x2[bit] = (float)(signed char)(((bit < 4 ? px2.x : px2.y) >> sh) & 0xff);
            y2[bit] = (float)(signed char)(((bit < 4 ? py2.x : py2.y) >> sh) & 0xff);
        }
    }
    __syncthreads();
    const int total = min(s_cum[kMaxLevels], P.out_cap);
    if (blockIdx.x == 0 && threadIdx.x == 0) n_out[b] = total;
    const LevelKp *frame_kp = P.lvl_kp + (size_t)b * P.total_slots;
    uint8_t(*ring)[kDescStage] = s_ring[warp];
    for (int p0 = (blockIdx.x * kDescWarps + warp) * kDescRun; p0 < total; p0 += gridDim.x * kDescWarps * kDescRun) {
        const int n = min(kDescRun, total - p0);
        // lane i < n holds keypoint i of the run
        int ml = 0, mx = 0, my = 0, mresp = 0;
        if (lane < n) {
            const int pos = p0 + lane;
            while (pos >= s_cum[ml + 1]) ++ml;
            const LevelKp kp = frame_kp[s_slot[ml] + pos - s_cum[ml]];
            mx = kp.x;
            my = kp.y;
            mresp = kp.response;
        }
        // the copies of keypoint i into stage i & 1, one commit group per keypoint.  Every chunk copied holds a byte the
        // keypoint reads, and keypoints lie in [19, w - 19) x [19, h - 19), so those bytes are inside the level.  Rows of
        // the blurred levels and of the pyramid levels >= 1 start 64-byte aligned at a 64-byte multiple pitch, and level
        // 0 takes this path only when its base and step are 16-byte multiples: an aligned 16-byte chunk holding a byte
        // of [row, row + w) then never leaves [row, row + pitch).
        auto stage = [&](int i) {
            const int cx = __shfl_sync(0xffffffffu, mx, i), cy = __shfl_sync(0xffffffffu, my, i),
                      l = __shfl_sync(0xffffffffu, ml, i);
            uint8_t *disc = ring[i & 1], *win = disc + kDiscBytes;
            const int xw = cx - kWinHalf, ow = xw & 15, nw = (ow + kWinRows + 15) >> 4, bpitch = s_bpitch[l];
            const uint8_t *bsrc = s_blur[l] + (size_t)(cy - kWinHalf) * bpitch + (xw - ow);
#pragma unroll
            for (int t = lane; t < kWinRows * 4; t += 32) {
                const int r = t >> 2, c = t & 3;
                if (c < nw) cp_async16(win + r * kWinPitch + 16 * c, bsrc + (size_t)r * bpitch + 16 * c);
            }
            const int xd = cx - kHalfPatch, od = xd & 15, pitch = s_pitch[l];
            const uint8_t *dsrc = s_img[l] + (size_t)(cy - kHalfPatch) * pitch;
            if (l > 0 || vec0) {
                const int nd = (od + kDiscRows + 15) >> 4;
                dsrc += xd - od;
#pragma unroll
                for (int t = lane; t < kDiscRows * 3; t += 32) {
                    const int r = t / 3, c = t - 3 * r;
                    if (c < nd) cp_async16(disc + r * kDiscPitch + 16 * c, dsrc + (size_t)r * pitch + 16 * c);
                }
            } else if (lane < kDiscRows) {  // plain loads into the same layout (lane = disc column)
#pragma unroll 8
                for (int r = 0; r < kDiscRows; ++r)
                    disc[r * kDiscPitch + od + lane] = __ldg(dsrc + (size_t)r * pitch + xd + lane);
            }
        };
        stage(0);
        cp_async_commit();
        float my_angle = 0.f;
        for (int i = 0; i < n; ++i) {
            if (i + 1 < n) stage(i + 1);
            cp_async_commit();
            cp_async_wait_prev();
            __syncwarp();
            const int cx = __shfl_sync(0xffffffffu, mx, i);
            const uint8_t *disc = ring[i & 1], *win = disc + kDiscBytes;

            // ---- ic_angle (orb_extractor.cc:708-735): integer moments over the radius-15 disc.  Lane v takes the words
            //      of row v - 15 from the disc start on (a funnel shift by the row's alignment offset) and forms
            //      sum u I and sum I of the row by DP4A; m10 and m01 are then exact integer sums over the lanes
            int su = 0, si = 0;
            {
                const uint4 *row = reinterpret_cast<const uint4 *>(disc + min(lane, kDiscRows - 1) * kDiscPitch);
                const uint4 q0 = row[0], q1 = row[1], q2 = row[2];
                const uint32_t r[12] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w, q2.x, q2.y, q2.z, q2.w};
                const int od = (cx - kHalfPatch) & 15, sh = 8 * (od & 3);
                switch (od >> 2) {  // warp-uniform
                    case 0: disc_row_sums<0>(r, sh, wu, wm, su, si); break;
                    case 1: disc_row_sums<1>(r, sh, wu, wm, su, si); break;
                    case 2: disc_row_sums<2>(r, sh, wu, wm, su, si); break;
                    default: disc_row_sums<3>(r, sh, wu, wm, su, si); break;
                }
            }
            int m10 = su, m01 = (lane - kHalfPatch) * si;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                m10 += __shfl_xor_sync(0xffffffffu, m10, o);
                m01 += __shfl_xor_sync(0xffffffffu, m01, o);
            }
            const float angle = fast_atan2_deg((float)m01, (float)m10);

            // ---- steered BRIEF (orb_extractor.cc:747-807) on the Gaussian-blurred level (blur_tiles_kernel): lane i
            //      produces descriptor byte i from 16 gathers in the staged window
            const float ang_rad = (float)((double)angle * 3.14159265358979323846 / 180.0);
            const float ca = util_cos(ang_rad), sa = util_sin(ang_rad);
            const uint8_t *center = win + kWinHalf * kWinPitch + kWinHalf + ((cx - kWinHalf) & 15);
            int val = 0;
#pragma unroll
            for (int bit = 0; bit < 8; ++bit) {
                const int r1 = __float2int_rn(x1[bit] * sa + y1[bit] * ca), c1 = __float2int_rn(x1[bit] * ca - y1[bit] * sa);
                const int r2 = __float2int_rn(x2[bit] * sa + y2[bit] * ca), c2 = __float2int_rn(x2[bit] * ca - y2[bit] * sa);
                val |= (center[r1 * kWinPitch + c1] < center[r2 * kWinPitch + c2]) << bit;
            }
            desc_out[((size_t)b * P.out_cap + p0 + i) * 32 + lane] = (uint8_t)val;
            if (lane == i) my_angle = angle;
            __syncwarp();  // stage i & 1 is refilled with keypoint i + 2
        }
        if (lane < n) {
            plp_keypoint o;
            const float s = s_scale[ml];
            o.x = ml == 0 ? (float)mx : (float)mx * s;  // orb_extractor.cc:695-706
            o.y = ml == 0 ? (float)my : (float)my * s;
            o.size = s_size[ml];
            o.angle = my_angle;
            o.response = (float)mresp;
            o.octave = ml;
            o.class_id = -1;
            kp_out[(size_t)b * P.out_cap + p0 + lane] = o;
        }
    }
}

}  // namespace

}  // namespace plp

// =========================================================================================================
// handle + C ABI
// =========================================================================================================
using namespace plp;

// the two quadtree instances (quadtree_kernels.cuh) and the job the kernel reads from the extractor's device state
constexpr auto kQtSmall = quadtree_kernel<kNodeCapSmall, kCandCapSmall, kQtThreadsSmall, kQtMinBlocksSmall>;
constexpr auto kQtLarge = quadtree_kernel<kNodeCap, kCandCapLarge, kQtThreadsLarge, kQtMinBlocksLarge>;
static_assert(kQtMaxLevels >= kMaxLevels, "the quadtree job holds every pyramid level");

static QtJob qt_job(const OrbDev &D) {
    QtJob J;
    J.num_levels = D.num_levels;
    J.num_cells = D.num_cells;
    J.total_slots = D.total_slots;
    for (int l = 0; l < D.num_levels; ++l) {
        const LevelInfo &V = D.lv[l];
        J.lv[l] = QtLevel{V.w, V.h, V.cell_base, V.num_cells, V.budget, V.slot_base, V.slot_cap};
    }
    J.cell_buf = D.cell_buf;
    J.cell_cnt = D.cell_cnt;
    J.lvl_kp = D.lvl_kp;
    J.lvl_cnt = D.lvl_cnt;
    J.scratch = D.qt_scratch;
    J.scratch_per_job = D.qt_scratch_per_job;
    J.status = D.status;
    return J;
}

struct plp_orb {
    plp_ctx *ctx = nullptr;
    plp_orb_params params;
    int rows = 0, cols = 0, max_batch = 0;
    OrbDev dev;  // device pointers filled in at create
    std::vector<float> scale_factors, inv_scale_factors, level_sigma_sq, inv_level_sigma_sq;
    std::vector<uint32_t> num_keypts_per_level;
    std::vector<CellDesc> cells;
    short4 *d_xtab[kMaxLevels] = {nullptr};
    short4 *d_ytab[kMaxLevels] = {nullptr};
    CellDesc *d_cells = nullptr;
    uint8_t *d_pyr = nullptr;
    uint8_t *d_blur = nullptr;
    BlurTile *d_blur_tiles = nullptr;
    std::vector<BlurTile> blur_tiles;
    uint8_t *d_img = nullptr;  // staging for host-pointer extraction (max_batch frames)
    uint8_t *d_mask = nullptr;
    uint32_t *d_cell_buf = nullptr;
    int *d_cell_cnt = nullptr;
    LevelKp *d_lvl_kp = nullptr;
    int *d_lvl_cnt = nullptr;
    uint8_t *d_qt_scratch = nullptr;
    int *d_status = nullptr;
    plp_keypoint *d_kp = nullptr;
    uint8_t *d_desc = nullptr;
    int32_t *d_n = nullptr;
    size_t qt_smem = 0;
    bool qt_small = false;  // the <1024 nodes> instance of quadtree_kernel serves this configuration
    // TMA descriptors of the pyramid levels as (x, y, frame) uint8 tensors; levels >= 1 live in d_pyr (encoded once),
    // level 0 is the caller's buffer (re-encoded when its address / pitch / batch changes)
    BlurMaps maps;
    bool maps_ok = false;       // levels >= 1 encoded
    const uint8_t *map0_img = nullptr;
    size_t map0_step = 0;
    int map0_batch = 0;
    int last_batch = 0;
    const uint8_t *last_img0 = nullptr;
    size_t last_step = 0;
};

// cuTensorMapEncodeTiled through the runtime's driver-entry-point lookup (no link-time dependency on libcuda)
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn tensor_map_encoder() {
    static EncodeTiledFn fn = []() -> EncodeTiledFn {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess)
            return nullptr;
        return (EncodeTiledFn)p;
    }();
    return fn;
}
// (x, y, frame) uint8 tensor of one pyramid level; box = the blur kernel's source tile.  false when the buffer does not
// meet TMA's alignment rules (16-byte base and strides) -- the caller then uses the plain-load kernel for this batch.
static bool encode_level_map(CUtensorMap *m, const uint8_t *base, int w, int h, int frames, size_t pitch, size_t frame_stride) {
    EncodeTiledFn enc = tensor_map_encoder();
    if (!enc || ((uintptr_t)base & 15) || (pitch & 15) || (frame_stride & 15) || w < 1 || h < 1 || frames < 1) return false;
    const cuuint64_t dims[3] = {(cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)frames};
    const cuuint64_t strides[2] = {(cuuint64_t)pitch, (cuuint64_t)frame_stride};
    const cuuint32_t box[3] = {(cuuint32_t)kBoxW, (cuuint32_t)kBoxH, 1u}, estr[3] = {1u, 1u, 1u};
    return enc(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, (void *)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}


static void build_resize_tables(int sw, int sh, int dw, int dh, std::vector<short4> &xt, std::vector<short4> &yt) {
    // cv::resize INTER_LINEAR 8U: 11-bit coefficients, rounded half-to-even (SURVEY.md Appendix A.1)
    const double inv_scale_x = (double)dw / sw, inv_scale_y = (double)dh / sh;
    const double scale_x = 1. / inv_scale_x, scale_y = 1. / inv_scale_y;
    xt.resize(dw);
    yt.resize(dh);
    for (int dx = 0; dx < dw; ++dx) {
        float fx = (float)((dx + 0.5) * scale_x - 0.5);
        int sx = cv_floor(fx);
        fx -= sx;
        if (sx < 0) {
            fx = 0;
            sx = 0;
        }
        if (sx >= sw - 1) {
            fx = 0;
            sx = sw - 1;
        }
        short4 t;
        t.x = (short)sx;
        t.y = (short)std::min(sx + 1, sw - 1);
        t.z = (short)lrintf((1.f - fx) * 2048);
        t.w = (short)lrintf(fx * 2048);
        xt[dx] = t;
    }
    for (int dy = 0; dy < dh; ++dy) {
        float fy = (float)((dy + 0.5) * scale_y - 0.5);
        int sy = cv_floor(fy);
        fy -= sy;
        short4 t;
        t.x = (short)std::min(std::max(sy, 0), sh - 1);
        t.y = (short)std::min(std::max(sy + 1, 0), sh - 1);
        t.z = (short)lrintf((1.f - fy) * 2048);
        t.w = (short)lrintf(fy * 2048);
        yt[dy] = t;
    }
}

extern "C" {

void plp_orb_destroy(plp_orb *o) {
    if (!o) return;
    cudaSetDevice(o->ctx->device);
    cudaStreamSynchronize(o->ctx->stream);
    for (int l = 0; l < kMaxLevels; ++l) {
        if (o->d_xtab[l]) cudaFree(o->d_xtab[l]);
        if (o->d_ytab[l]) cudaFree(o->d_ytab[l]);
    }
    void *ptrs[] = {o->d_blur, o->d_blur_tiles, o->d_cells, o->d_pyr, o->d_img, o->d_mask, o->d_cell_buf, o->d_cell_cnt, o->d_lvl_kp,
                    o->d_lvl_cnt, o->d_qt_scratch, o->d_status, o->d_kp, o->d_desc, o->d_n};
    for (void *p : ptrs)
        if (p) cudaFree(p);
    delete o;
}

plp_status plp_orb_create(plp_ctx *ctx, const plp_orb_params *params, int rows, int cols, int max_batch,
                          plp_orb **out) {
    PLP_REQUIRE(ctx && params && out, "null pointer");
    *out = nullptr;
    PLP_REQUIRE(rows > 0 && cols > 0 && max_batch > 0, "image size / batch");
    PLP_REQUIRE(params->num_levels >= 1 && params->num_levels <= kMaxLevels, "num_levels in [1,16]");
    PLP_REQUIRE(params->scale_factor > 1.0f || params->num_levels == 1, "scale_factor > 1");
    PLP_REQUIRE(cols <= 2047 + 2 * kPatchRadius && rows <= 1023 + 2 * kPatchRadius,
                "image larger than 2085 x 1061 (packed candidate coordinates)");
    PLP_REQUIRE(params->ini_fast_thr < 255 && params->min_fast_thr >= 1 && params->min_fast_thr <= params->ini_fast_thr,
                "FAST thresholds: 1 <= min <= ini < 255");
    PLP_CUDA_TRY(cudaSetDevice(ctx->device));
    plp_orb *o = new plp_orb();
    o->ctx = ctx;
    o->params = *params;
    o->rows = rows;
    o->cols = cols;
    o->max_batch = max_batch;
    const unsigned L = params->num_levels;
    // ---- orb_params.cc:86-128 scale tables
    o->scale_factors.assign(L, 1.0f);
    o->inv_scale_factors.assign(L, 1.0f);
    o->level_sigma_sq.assign(L, 1.0f);
    o->inv_level_sigma_sq.assign(L, 1.0f);
    for (unsigned l = 1; l < L; ++l) o->scale_factors[l] = params->scale_factor * o->scale_factors[l - 1];
    for (unsigned l = 1; l < L; ++l) o->inv_scale_factors[l] = (1.0f / params->scale_factor) * o->inv_scale_factors[l - 1];
    {
        float s = 1.0f;
        for (unsigned l = 1; l < L; ++l) {
            s = params->scale_factor * s;
            o->level_sigma_sq[l] = s * s;
            o->inv_level_sigma_sq[l] = 1.0f / (s * s);
        }
    }
    // ---- orb_extractor.cc:244-253 per-level budget
    o->num_keypts_per_level.resize(L);
    {
        double desired = params->max_num_keypts * (1.0 - 1.0 / params->scale_factor) /
                         (1.0 - std::pow(1.0 / params->scale_factor, static_cast<double>(L)));
        if (L == 1) desired = params->max_num_keypts;
        unsigned total = 0;
        for (unsigned l = 0; l + 1 < L; ++l) {
            o->num_keypts_per_level[l] = (unsigned)std::round(desired);
            total += o->num_keypts_per_level[l];
            desired *= 1.0 / params->scale_factor;
        }
        o->num_keypts_per_level[L - 1] = (unsigned)std::max((int)params->max_num_keypts - (int)total, 0);
    }
    OrbDev &D = o->dev;
    memset(&D, 0, sizeof(D));
    D.num_levels = (int)L;
    D.rows = rows;
    D.cols = cols;
    D.ini_thr = (int)params->ini_fast_thr;
    D.min_thr = (int)params->min_fast_thr;
    // ---- orb_extractor.cc:270-286 u_max
    {
        const unsigned vmax = (unsigned)std::floor(kHalfPatch * std::sqrt(2.0) / 2 + 1);
        const unsigned vmin = (unsigned)std::ceil(kHalfPatch * std::sqrt(2.0) / 2);
        for (unsigned v = 0; v <= vmax; ++v)
            D.u_max[v] = (int)std::round(std::sqrt((double)kHalfPatch * kHalfPatch - (double)v * v));
        for (unsigned v = kHalfPatch, v0 = 0; vmin <= v; --v) {
            while (D.u_max[v0] == D.u_max[v0 + 1]) ++v0;
            D.u_max[v] = (int)v0;
            ++v0;
        }
    }
    // ---- level geometry, cells (orb_extractor.cc:344-392)
    int qt_max_slots = 0, qt_max_cells = 0;
    size_t pyr_bytes = 0, blur_bytes = 0;
    int slot_base = 0, cell_base = 0;
    plp_status st = PLP_OK;
    for (unsigned l = 0; l < L; ++l) {
        LevelInfo &V = D.lv[l];
        if (l == 0) {
            V.w = cols;
            V.h = rows;
        } else {
            const double scale = o->scale_factors[l];
            V.w = (int)std::round(cols * 1.0 / scale);
            V.h = (int)std::round(rows * 1.0 / scale);
        }
        V.pitch = (V.w + 63) & ~63;
        V.offset = pyr_bytes;
        if (l > 0) pyr_bytes += (size_t)V.pitch * V.h + 256;
        pyr_bytes = (pyr_bytes + 255) & ~(size_t)255;
        V.blur_offset = blur_bytes;
        blur_bytes += (size_t)V.pitch * V.h + 256;
        blur_bytes = (blur_bytes + 255) & ~(size_t)255;
        for (int y0 = 0; y0 < V.h; y0 += kBtH)
            for (int x0 = 0; x0 < V.w; x0 += kBtW) o->blur_tiles.push_back(BlurTile{(short)l, (short)x0, (short)y0, 0});
        V.budget = (int)o->num_keypts_per_level[l];
        V.scale_factor = o->scale_factors[l];
        V.size = (float)(unsigned)(31 * o->scale_factors[l]);
        V.slot_base = slot_base;
        {
            // initial nodes of the quadtree (orb_extractor.cc:561-582): one sweep can quadruple them
            int g0 = 1;
            if (V.w > 2 * kPatchRadius && V.h > 2 * kPatchRadius) {
                const double ratio = (double)(V.w - 2 * kPatchRadius) / (V.h - 2 * kPatchRadius);
                g0 = ratio > 1 ? (int)std::round(ratio) : (int)std::round(1 / ratio);
            }
            V.slot_cap = 4 * std::max(V.budget, g0) + 8;
        }
        slot_base += V.slot_cap;
        V.cell_base = cell_base;
        V.num_cells = 0;
        qt_max_slots = std::max(qt_max_slots, V.slot_cap);
        if (V.slot_cap > kNodeCap) {
            set_error("orb: level %u budget %d exceeds the quadtree node capacity", l, V.budget);
            st = PLP_ERR_CAPACITY;
        }
        if (V.w > 2 * kPatchRadius && V.h > 2 * kPatchRadius && V.w >= 1 && V.h >= 1) {
            const unsigned min_bx = kPatchRadius, min_by = kPatchRadius;
            const unsigned max_bx = V.w - kPatchRadius, max_by = V.h - kPatchRadius;
            const unsigned width = max_bx - min_bx, height = max_by - min_by;
            const unsigned ncols = width / kCellSize + 1, nrows = height / kCellSize + 1;
            V.cells_x = (int)ncols;
            V.cells_y = (int)nrows;
            for (unsigned i = 0; i < nrows; ++i) {
                const unsigned min_y = min_by + i * kCellSize;
                if (max_by - kOverlap <= min_y || max_by < kOverlap) continue;
                unsigned max_y = min_y + kCellSize + kOverlap;
                if (max_by < max_y) max_y = max_by;
                for (unsigned j = 0; j < ncols; ++j) {
                    const unsigned min_x = min_bx + j * kCellSize;
                    if (max_bx - kOverlap <= min_x || max_bx < kOverlap) continue;
                    unsigned max_x = min_x + kCellSize + kOverlap;
                    if (max_bx < max_x) max_x = max_bx;
                    CellDesc c;
                    c.level = (short)l;
                    c.i = (short)i;
                    c.j = (short)j;
                    c.pad = 0;
                    c.min_x = (short)min_x;
                    c.min_y = (short)min_y;
                    c.max_x = (short)max_x;
                    c.max_y = (short)max_y;
                    o->cells.push_back(c);
                    V.num_cells++;
                }
            }
        }
        cell_base += V.num_cells;
        qt_max_cells = std::max(qt_max_cells, V.num_cells);
    }
    // the quadtree keeps the prefix of a level's cell counts in shared memory (2 ints per node of its capacity)
    if (st == PLP_OK && qt_max_cells + 1 > 2 * (qt_max_slots <= kNodeCapSmall ? kNodeCapSmall : kNodeCap)) {
        set_error("orb: a pyramid level of %d FAST cells exceeds the quadtree's cell capacity", qt_max_cells);
        st = PLP_ERR_CAPACITY;
    }
    if (st != PLP_OK) {
        delete o;
        return st;
    }
    D.num_cells = cell_base;
    D.total_slots = slot_base;
    D.out_cap = slot_base;
    D.pyr_frame_bytes = pyr_bytes ? pyr_bytes : 256;
    D.blur_frame_bytes = blur_bytes ? blur_bytes : 256;
    D.num_blur_tiles = (int)o->blur_tiles.size();
    const size_t B = (size_t)max_batch;
    // ---- device allocations
#define ORB_ALLOC(ptr, bytes)                                              \
    do {                                                                   \
        cudaError_t e_ = cudaMalloc((void **)&(ptr), (bytes) ? (bytes) : 256); \
        if (e_ != cudaSuccess) {                                           \
            set_error("orb: cudaMalloc(%zu) failed: %s", (size_t)(bytes), cudaGetErrorString(e_)); \
            plp_orb_destroy(o);                                            \
            return PLP_ERR_CUDA;                                           \
        }                                                                  \
    } while (0)
    for (unsigned l = 1; l < L; ++l) {
        std::vector<short4> xt, yt;
        build_resize_tables(D.lv[l - 1].w, D.lv[l - 1].h, D.lv[l].w, D.lv[l].h, xt, yt);
        ORB_ALLOC(o->d_xtab[l], xt.size() * sizeof(short4));
        ORB_ALLOC(o->d_ytab[l], yt.size() * sizeof(short4));
        cudaMemcpy(o->d_xtab[l], xt.data(), xt.size() * sizeof(short4), cudaMemcpyHostToDevice);
        cudaMemcpy(o->d_ytab[l], yt.data(), yt.size() * sizeof(short4), cudaMemcpyHostToDevice);
    }
    ORB_ALLOC(o->d_cells, o->cells.size() * sizeof(CellDesc));
    if (!o->cells.empty())
        cudaMemcpy(o->d_cells, o->cells.data(), o->cells.size() * sizeof(CellDesc), cudaMemcpyHostToDevice);
    ORB_ALLOC(o->d_pyr, B * D.pyr_frame_bytes);
    ORB_ALLOC(o->d_blur, B * D.blur_frame_bytes);
    ORB_ALLOC(o->d_blur_tiles, o->blur_tiles.size() * sizeof(BlurTile));
    if (!o->blur_tiles.empty())
        cudaMemcpy(o->d_blur_tiles, o->blur_tiles.data(), o->blur_tiles.size() * sizeof(BlurTile), cudaMemcpyHostToDevice);
    ORB_ALLOC(o->d_img, B * (size_t)rows * cols);
    ORB_ALLOC(o->d_mask, (size_t)rows * cols);
    ORB_ALLOC(o->d_cell_buf, B * (size_t)D.num_cells * kCellCap * sizeof(uint32_t));
    ORB_ALLOC(o->d_cell_cnt, B * (size_t)D.num_cells * sizeof(int));
    ORB_ALLOC(o->d_lvl_kp, B * (size_t)D.total_slots * sizeof(LevelKp));
    ORB_ALLOC(o->d_lvl_cnt, B * L * sizeof(int));
    D.qt_scratch_per_job = qt_scratch_bytes_per_job();
    ORB_ALLOC(o->d_qt_scratch, B * L * D.qt_scratch_per_job);
    ORB_ALLOC(o->d_status, B * sizeof(int));
    ORB_ALLOC(o->d_kp, B * (size_t)D.out_cap * sizeof(plp_keypoint));
    ORB_ALLOC(o->d_desc, B * (size_t)D.out_cap * 32);
    ORB_ALLOC(o->d_n, B * sizeof(int32_t));
#undef ORB_ALLOC
    D.pyr = o->d_pyr;
    D.blur = o->d_blur;
    D.blur_tiles = o->d_blur_tiles;
    D.cells = o->d_cells;
    D.cell_buf = o->d_cell_buf;
    D.cell_cnt = o->d_cell_cnt;
    D.lvl_kp = o->d_lvl_kp;
    D.lvl_cnt = o->d_lvl_cnt;
    D.qt_scratch = o->d_qt_scratch;
    D.status = o->d_status;
    // TMA descriptors of the levels that live in the handle's own pyramid block (level 0 follows the caller's buffer)
    o->maps_ok = true;
    memset(&o->maps, 0, sizeof(o->maps));
    for (unsigned l = 1; l < L && o->maps_ok; ++l)
        o->maps_ok = encode_level_map(&o->maps.m[l], o->d_pyr + D.lv[l].offset, D.lv[l].w, D.lv[l].h, max_batch, D.lv[l].pitch,
                                      D.pyr_frame_bytes);
    o->qt_small = qt_max_slots <= kNodeCapSmall;
    plp_status so;
    if (o->qt_small) {
        o->qt_smem = qt_smem_bytes<kNodeCapSmall, kCandCapSmall, kQtThreadsSmall>();
        so = ensure_smem_optin((const void *)kQtSmall, o->qt_smem, "quadtree_kernel<small>");
    } else {
        o->qt_smem = qt_smem_bytes<kNodeCap, kCandCapLarge, kQtThreadsLarge>();
        so = ensure_smem_optin((const void *)kQtLarge, o->qt_smem, "quadtree_kernel<large>");
    }
    if (so != PLP_OK) {
        plp_orb_destroy(o);
        return so;
    }
    *out = o;
    return PLP_OK;
}

int plp_orb_capacity(const plp_orb *o) { return o ? o->dev.out_cap : 0; }

plp_status plp_orb_get_tables(const plp_orb *o, float *sf, float *isf, float *ls, float *ils, uint32_t *nk) {
    PLP_REQUIRE(o, "orb");
    for (int l = 0; l < o->dev.num_levels; ++l) {
        if (sf) sf[l] = o->scale_factors[l];
        if (isf) isf[l] = o->inv_scale_factors[l];
        if (ls) ls[l] = o->level_sigma_sq[l];
        if (ils) ils[l] = o->inv_level_sigma_sq[l];
        if (nk) nk[l] = o->num_keypts_per_level[l];
    }
    return PLP_OK;
}

static plp_status orb_run(plp_orb *o, const uint8_t *d_imgs, int batch, size_t step, const uint8_t *d_mask,
                          size_t mask_step, plp_keypoint *d_kp, uint8_t *d_desc, int32_t *d_n, int32_t *d_status) {
    plp_ctx *ctx = o->ctx;
    OrbDev D = o->dev;
    D.img0 = d_imgs;
    D.img0_step = step;
    D.img0_frame_stride = step * (size_t)o->rows;
    D.mask = d_mask;
    D.mask_step = mask_step;
    D.status = d_status ? d_status : o->d_status;
    o->last_batch = batch;
    o->last_img0 = d_imgs;
    o->last_step = step;
    PLP_CUDA_TRY(cudaMemsetAsync(D.status, 0, (size_t)batch * sizeof(int), ctx->stream));
    for (int l = 1; l < D.num_levels; ++l) {
        const int quads = ((D.lv[l].w + 3) >> 2) * ((D.lv[l].h + kResizeRows - 1) / kResizeRows);  // threads: 4 columns x 8 rows each
        if (quads <= 0) continue;
        dim3 grid(div_up(quads, 256), batch);
        PLP_LAUNCH(ctx, pyr_resize_kernel, grid, 256, 0, D, l, o->d_xtab[l], o->d_ytab[l]);
    }
    // TMA descriptors for the FAST tiles and the blur boxes: level 0 is the caller's buffer
    bool tma = o->maps_ok;
    if (tma && (o->map0_img != d_imgs || o->map0_step != step || o->map0_batch != batch)) {
        tma = encode_level_map(&o->maps.m[0], d_imgs, D.lv[0].w, D.lv[0].h, batch, step, D.img0_frame_stride);
        o->map0_img = tma ? d_imgs : nullptr;
        o->map0_step = step;
        o->map0_batch = batch;
    }
    // without TMA (caller buffer not 16-byte aligned / pitched): plain loads
    if (D.num_cells > 0) {
        dim3 grid(D.num_cells, batch), grid_run(div_up(D.num_cells, kFastRun), batch);
        if (tma)
            PLP_LAUNCH(ctx, fast_cells_tma_kernel, grid_run, 256, 0, o->maps, D, kFastRun);
        else
            PLP_LAUNCH(ctx, fast_cells_kernel_v2, grid, 256, 0, D);
    }
    if (D.num_blur_tiles > 0) {
        dim3 grid(D.num_blur_tiles, batch), grid_run(div_up(D.num_blur_tiles, kBlurRun), batch);
        if (tma)
            PLP_LAUNCH(ctx, blur_tiles_tma_kernel, grid_run, kBlurThreads, 0, o->maps, D, kBlurRun);
        else
            PLP_LAUNCH(ctx, blur_tiles_kernel, grid, kBlurThreads, 0, D);
    }
    {
        dim3 grid(D.num_levels, batch);
        // (PLP_LAUNCH spelled out: the report names the instance by its node capacity)
        if (ctx->timing) plp::timing_begin(ctx, o->qt_small ? "quadtree_kernel<1024>" : "quadtree_kernel<2048>");
        const QtJob J = qt_job(D);
        if (o->qt_small)
            kQtSmall<<<grid, kQtThreadsSmall, o->qt_smem, ctx->stream>>>(J);
        else
            kQtLarge<<<grid, kQtThreadsLarge, o->qt_smem, ctx->stream>>>(J);
        if (ctx->timing) plp::timing_end(ctx);
        ctx->launches++;
    }
    {
        // the grid covers max_num_keypts output positions; warps stride over the quadtree's overshoot
        const int kp_est = std::max(256, (int)o->params.max_num_keypts);
        dim3 grid(div_up(std::min(D.total_slots, kp_est), kDescWarps * kDescRun), batch);
        PLP_LAUNCH(ctx, describe_kernel, grid, kDescWarps * 32, 0, D, d_kp, d_desc, d_n);
    }
    PLP_CHECK_LAUNCH();
    return PLP_OK;
}

plp_status plp_orb_extract_batch_dev(plp_orb *o, const uint8_t *d_imgs, int batch, size_t step, plp_keypoint *d_kp,
                                     uint8_t *d_desc, int32_t *d_n, int32_t *d_status) {
    PLP_REQUIRE(o && d_imgs && d_kp && d_desc && d_n, "null pointer");
    PLP_REQUIRE(batch >= 1 && batch <= o->max_batch, "batch exceeds the handle's max_batch");
    PLP_REQUIRE(step >= (size_t)o->cols, "step < cols");
    PLP_CUDA_TRY(cudaSetDevice(o->ctx->device));
    return orb_run(o, d_imgs, batch, step, nullptr, 0, d_kp, d_desc, d_n, d_status);
}

static plp_status orb_extract_host(plp_orb *o, const uint8_t *imgs, int batch, size_t step, const uint8_t *mask,
                                   size_t mask_step, plp_keypoint *kp_out, uint8_t *desc_out, int32_t *n_out) {
    plp_ctx *ctx = o->ctx;
    PLP_CUDA_TRY(cudaSetDevice(ctx->device));
    const size_t rows = o->rows, cols = o->cols;
    PLP_CUDA_TRY(cudaMemcpy2DAsync(o->d_img, cols, imgs, step, cols, rows * (size_t)batch, cudaMemcpyHostToDevice,
                                   ctx->stream));
    const uint8_t *d_mask = nullptr;
    if (mask) {
        PLP_CUDA_TRY(cudaMemcpy2DAsync(o->d_mask, cols, mask, mask_step, cols, rows, cudaMemcpyHostToDevice, ctx->stream));
        d_mask = o->d_mask;
    }
    PLP_TRY(orb_run(o, o->d_img, batch, cols, d_mask, cols, o->d_kp, o->d_desc, o->d_n, nullptr));
    const size_t cap = o->dev.out_cap;
    PLP_CUDA_TRY(cudaMemcpyAsync(n_out, o->d_n, (size_t)batch * 4, cudaMemcpyDeviceToHost, ctx->stream));
    PLP_CUDA_TRY(cudaMemcpyAsync(kp_out, o->d_kp, (size_t)batch * cap * sizeof(plp_keypoint), cudaMemcpyDeviceToHost,
                                 ctx->stream));
    PLP_CUDA_TRY(cudaMemcpyAsync(desc_out, o->d_desc, (size_t)batch * cap * 32, cudaMemcpyDeviceToHost, ctx->stream));
    std::vector<int> status(batch);
    PLP_CUDA_TRY(cudaMemcpyAsync(status.data(), o->d_status, (size_t)batch * 4, cudaMemcpyDeviceToHost, ctx->stream));
    PLP_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    for (int b = 0; b < batch; ++b)
        if (status[b] != 0) {
            set_error("orb: capacity overflow in frame %d (code %d)", b, status[b]);
            return PLP_ERR_CAPACITY;
        }
    return PLP_OK;
}

plp_status plp_orb_extract(plp_orb *o, const uint8_t *img, int rows, int cols, size_t step, const uint8_t *mask,
                           size_t mask_step, plp_keypoint *kp_out, uint8_t *desc_out, int *n_out) {
    PLP_REQUIRE(o && n_out, "null pointer");
    *n_out = 0;
    if (!img || rows == 0 || cols == 0) return PLP_OK;  // orb_extractor.cc:76-79
    PLP_REQUIRE(rows == o->rows && cols == o->cols, "image size differs from the handle's");
    PLP_REQUIRE(kp_out && desc_out, "null output");
    PLP_REQUIRE(step >= (size_t)cols && (!mask || mask_step >= (size_t)cols), "step < cols");
    int32_t n = 0;
    PLP_TRY(orb_extract_host(o, img, 1, step, mask, mask_step, kp_out, desc_out, &n));
    *n_out = n;
    return PLP_OK;
}

plp_status plp_orb_extract_batch(plp_orb *o, const uint8_t *imgs, int batch, size_t step, plp_keypoint *kp_out,
                                 uint8_t *desc_out, int32_t *n_out) {
    PLP_REQUIRE(o && imgs && kp_out && desc_out && n_out, "null pointer");
    PLP_REQUIRE(batch >= 1 && batch <= o->max_batch, "batch exceeds the handle's max_batch");
    PLP_REQUIRE(step >= (size_t)o->cols, "step < cols");
    return orb_extract_host(o, imgs, batch, step, nullptr, 0, kp_out, desc_out, n_out);
}

plp_status plp_orb_get_pyramid(const plp_orb *o, int b, int level, plp_image_view *out) {
    PLP_REQUIRE(o && out, "null pointer");
    PLP_REQUIRE(b >= 0 && b < o->last_batch && level >= 0 && level < o->dev.num_levels, "index");
    const LevelInfo &V = o->dev.lv[level];
    out->rows = V.h;
    out->cols = V.w;
    if (level == 0) {
        out->data = o->last_img0 + (size_t)b * o->last_step * o->rows;
        out->step = o->last_step;
    } else {
        out->data = o->d_pyr + (size_t)b * o->dev.pyr_frame_bytes + V.offset;
        out->step = V.pitch;
    }
    return PLP_OK;
}

plp_status plp_orb_debug_blurred(plp_orb *o, int b, int level, uint8_t *out) {
    PLP_REQUIRE(o && out, "null pointer");
    PLP_REQUIRE(b >= 0 && b < o->last_batch && level >= 0 && level < o->dev.num_levels, "index");
    plp_ctx *ctx = o->ctx;
    PLP_CUDA_TRY(cudaSetDevice(ctx->device));
    const LevelInfo &V = o->dev.lv[level];
    PLP_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    PLP_CUDA_TRY(cudaMemcpy2D(out, V.w, o->d_blur + (size_t)b * o->dev.blur_frame_bytes + V.blur_offset, V.pitch, V.w, V.h,
                              cudaMemcpyDeviceToHost));
    return PLP_OK;
}

plp_status plp_orb_debug_candidates(plp_orb *o, int b, int level, plp_keypoint *out, int cap, int *n_out) {
    PLP_REQUIRE(o && out && n_out, "null pointer");
    PLP_REQUIRE(b >= 0 && b < o->last_batch && level >= 0 && level < o->dev.num_levels, "index");
    plp_ctx *ctx = o->ctx;
    PLP_CUDA_TRY(cudaSetDevice(ctx->device));
    const LevelInfo &V = o->dev.lv[level];
    std::vector<int> cnt(V.num_cells);
    std::vector<uint32_t> buf((size_t)V.num_cells * kCellCap);
    PLP_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    if (V.num_cells) {
        PLP_CUDA_TRY(cudaMemcpy(cnt.data(), o->d_cell_cnt + (size_t)b * o->dev.num_cells + V.cell_base,
                                cnt.size() * 4, cudaMemcpyDeviceToHost));
        PLP_CUDA_TRY(cudaMemcpy(buf.data(), o->d_cell_buf + ((size_t)b * o->dev.num_cells + V.cell_base) * kCellCap,
                                buf.size() * 4, cudaMemcpyDeviceToHost));
    }
    int n = 0;
    for (int c = 0; c < V.num_cells; ++c)
        for (int k = 0; k < cnt[c]; ++k) {
            if (n < cap) {
                const uint32_t v = buf[(size_t)c * kCellCap + k];
                plp_keypoint kp;
                kp.x = (float)(v & 0x7ff);
                kp.y = (float)((v >> 11) & 0x3ff);
                kp.size = 7.f;
                kp.angle = -1.f;
                kp.response = (float)(v >> 21);
                kp.octave = 0;
                kp.class_id = -1;
                out[n] = kp;
            }
            ++n;
        }
    *n_out = n;
    return PLP_OK;
}

}  // extern "C"
