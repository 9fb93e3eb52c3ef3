// lines.cu -- LSD line segments + LBD descriptors for batches of frames, sm_90a.
//
// Replaces LineFeatureTracker::extract_LSD_LBD (feature/line_extractor.cc:88-160) and what it calls:
//   LSDDetectorC::detectImpl            feature/line_descriptor/LSDDetector_custom.cpp:225-320
//   cv::LineSegmentDetector::detect     third party (OpenCV imgproc lsd.cpp); LSD of Grompone von Gioi et al., IPOL 2012,
//                                       refine = LSD_REFINE_STD, options of line_extractor.cc:113-122
//   BinaryDescriptor::compute           feature/line_descriptor/binary_descriptor_custom.cpp:518-679, 1018-1364
//
// LSD is a sequential greedy algorithm per image (a seed grows a region over a shared `used` map, the running region
// angle decides every next pixel), so the parallel axes are (1) the frames of a batch -- one warp owns one frame's
// region growing -- and (2) inside the warp: the 3 x 8 neighbours of three queue entries are fetched by 27 lanes at once
// and tested against the current region angle in parallel; only the accepted pixels are applied in sequence (the first
// aligned lane is what the scalar loop would have taken; later lanes are re-tested against the updated angle), which
// reproduces the scalar visiting order exactly.  Rectangle fitting / refinement are warp reductions with a fixed
// summation order.  Everything around it (11x11 blur + 1/2 down-scale, gradient + level-line angle, the 1024-bin stable
// seed ordering, 5x5 blur + Sobel, the 63-row LBD band sums) is ordinary data-parallel work.
//
// Determinism rules (the parity checker restates the same rules and is itself pinned bit-exactly against cv2 4.13):
// seeds ordered by (bin desc, raster asc); cos/sin/atan2 from detmath.h; double sums as 32 strided partials + xor tree;
// order-preserving compaction in reduce_region_radius.  Compiled with -fmad=false.
#include <algorithm>
#include <cmath>
#include <vector>

#include "common.cuh"
#include "detmath.h"
#include "lsd_grow_kernels.cuh"

using namespace plp;
using namespace plp::lsd;

namespace {

__device__ __forceinline__ int reflect101(int p, int len) {
    if (len == 1) return 0;
    while (p < 0 || p >= len) {
        if (p < 0) p = -p;
        if (p >= len) p = 2 * (len - 1) - p;
    }
    return p;
}

// ------------------------------------------------------------------------------------------------------------------
// K1: GaussianBlur(11x11, sigma 1.2) in OpenCV's Q8 fixed point (taps 0 0 4 21 60 86 60 21 4 0 0) followed by
//     resize(0.5, INTER_LINEAR_EXACT) == rounded mean of each 2x2 block (of its existing pixels at an odd border).
//     One CTA = 64 x 16 source pixels.
// ------------------------------------------------------------------------------------------------------------------
constexpr int kScTw = 64, kScTh = 16;
__global__ void __launch_bounds__(256) lsd_scale_kernel(LineDev D) {
    __shared__ uint8_t s_src[kScTh + 6][kScTw + 8];
    __shared__ uint16_t s_h[kScTh + 6][kScTw];
    __shared__ uint8_t s_b[kScTh][kScTw];
    const int b = blockIdx.y;
    const int tiles_x = (D.w + kScTw - 1) / kScTw;
    const int tx = (blockIdx.x % tiles_x) * kScTw, ty = (blockIdx.x / tiles_x) * kScTh;
    const uint8_t *img = D.img + (size_t)b * D.img_frame_stride;
    for (int i = threadIdx.x; i < (kScTh + 6) * (kScTw + 6); i += blockDim.x) {
        const int r = i / (kScTw + 6), c = i - r * (kScTw + 6);
        const int y = reflect101(ty + r - 3, D.h), x = reflect101(tx + c - 3, D.w);
        s_src[r][c] = img[(size_t)y * D.img_step + x];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < (kScTh + 6) * kScTw; i += blockDim.x) {
        const int r = i / kScTw, c = i - r * kScTw;
        const uint8_t *s = &s_src[r][c];
        s_h[r][c] = (uint16_t)(4 * (s[0] + s[6]) + 21 * (s[1] + s[5]) + 60 * (s[2] + s[4]) + 86 * s[3]);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kScTh * kScTw; i += blockDim.x) {
        const int r = i / kScTw, c = i - r * kScTw;
        const uint32_t v = 4u * (s_h[r][c] + s_h[r + 6][c]) + 21u * (s_h[r + 1][c] + s_h[r + 5][c]) +
                           60u * (s_h[r + 2][c] + s_h[r + 4][c]) + 86u * s_h[r + 3][c];
        s_b[r][c] = (uint8_t)((v + 32768u) >> 16);
    }
    __syncthreads();
    uint8_t *out = D.scaled + (size_t)b * D.npx;
    for (int i = threadIdx.x; i < (kScTh / 2) * (kScTw / 2); i += blockDim.x) {
        const int r = i / (kScTw / 2), c = i - r * (kScTw / 2);
        const int ox = tx / 2 + c, oy = ty / 2 + r;
        if (ox >= D.sw || oy >= D.sh) continue;
        // a dimension = 3 (mod 4) has a last half-resolution row / column with one source row / column: cv2 averages
        // the pixels that exist there, s / 2 ties to even, and copies the corner (the oracle's scaled_image states it)
        const bool fx = tx + 2 * c + 1 < D.w, fy = ty + 2 * r + 1 < D.h;
        const int x0 = 2 * c, y0 = 2 * r;
        int v;
        if (fx && fy) {
            v = (s_b[y0][x0] + s_b[y0][x0 + 1] + s_b[y0 + 1][x0] + s_b[y0 + 1][x0 + 1] + 2) >> 2;
        } else if (fx || fy) {
            const int s = s_b[y0][x0] + (fx ? s_b[y0][x0 + 1] : s_b[y0 + 1][x0]);
            v = (s + ((s >> 1) & 1)) >> 1;
        } else {
            v = s_b[y0][x0];
        }
        out[(size_t)oy * D.sw + ox] = (uint8_t)v;
    }
}

// ------------------------------------------------------------------------------------------------------------------
// ll_angle helpers.  The level-line field is never materialised: every consumer recomputes the 2x2 gradient from the
// half-resolution image (4 byte reads), which is what lets one frame's working set (image + `used` bitmap) live in
// shared memory.  (gx, gy) in [-510, 510]^2 determines the angle, hence cos/sin come from a table indexed by (gx, gy)
// that is built once per handle and shared by every frame (8.3 MB, L2 resident).
// ------------------------------------------------------------------------------------------------------------------

// table entry: level-line angle in degrees (cv::fastAtan2(gx, -gy)) and cos / sin of float(angle) as lsd.cpp
// accumulates them: `sumdx += cos(float(angle))`
__global__ void __launch_bounds__(256) lsd_cs_table_kernel(float4 *tab) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= kGDim * kGDim) return;
    const int gy = i / kGDim - kGRange, gx = i - (gy + kGRange) * kGDim - kGRange;
    const float deg = fast_atan2_deg((float)gx, (float)-gy);
    const double a = (double)deg * kDegToRads;
    const float af = (float)a;
    tab[i] = make_float4(deg, (float)det_cos((double)af), (float)det_sin((double)af), 0.f);
}

// ------------------------------------------------------------------------------------------------------------------
// K3: pseudo-ordering of the seeds: bin = int(modgrad * 1023 / max_grad), descending bins, raster order inside a bin.
//     One CTA (32 warps) per frame: frame maximum, then each warp owns a contiguous raster range -> per-warp
//     histograms, a scan over (bin desc, warp asc), and a stable scatter with __match_any ranks.
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int seed_k(const uint8_t *img, int sw, int sh, int i, int kthr) {
    const int y = i / sw, x = i - y * sw;
    if (x >= sw - 1 || y >= sh - 1) return -1;
    int gx, gy;
    grad_at(img, sw, i, gx, gy);
    const int k = gx * gx + gy * gy;
    return k > kthr ? k : -1;  // norm <= rho  <=>  k <= kthr
}

__global__ void __launch_bounds__(kSortWarps * 32) lsd_sort_kernel(LineDev D) {
    extern __shared__ uint32_t s_dyn[];
    uint32_t *hist = s_dyn;                        // [kSortWarps][kBins]: counts, then running start offsets
    uint32_t *base = s_dyn + kSortWarps * kBins;   // [kBins] first output slot of each bin
    __shared__ uint32_t s_scan[kBins];
    __shared__ uint32_t s_warp_tot[32];
    __shared__ int s_kmax[32];
    const int b = blockIdx.x, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint8_t *img = D.scaled + (size_t)b * D.npx;
    // frame maximum of the squared norm over the defined pixels
    int kloc = 0;
    for (int i = threadIdx.x; i < D.npx; i += blockDim.x) kloc = max(kloc, seed_k(img, D.sw, D.sh, i, D.kthr));
    for (int off = 16; off >= 1; off >>= 1) kloc = max(kloc, __shfl_xor_sync(kFull, kloc, off));
    if (lane == 0) s_kmax[wid] = kloc;
    for (int i = threadIdx.x; i < kSortWarps * kBins; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    int kmax = 0;
    for (int wv = 0; wv < kSortWarps; ++wv) kmax = max(kmax, s_kmax[wv]);
    const double max_grad = kmax > 0 ? sqrt((double)kmax / 4.0) : -1.0;
    const double bin_coef = (max_grad > 0) ? (double)(kBins - 1) / max_grad : 0.0;
    const int per_warp = ((D.npx + kSortWarps * 32 - 1) / (kSortWarps * 32)) * 32;
    const int beg = wid * per_warp, end = min(beg + per_warp, D.npx);
    uint32_t *myhist = hist + wid * kBins;
    // pass 1: per-warp histogram (lanes of one warp may hit the same bin: one leader per bin adds the group size)
    for (int i0 = beg; i0 < end; i0 += 32) {
        const int i = i0 + lane;
        int bin = -1;
        if (i < end) {
            const int k = seed_k(img, D.sw, D.sh, i, D.kthr);
            if (k >= 0) bin = (int)(sqrt((double)k / 4.0) * bin_coef);
        }
        const unsigned act = __ballot_sync(kFull, bin >= 0);
        if (bin >= 0) {
            const unsigned peers = __match_any_sync(act, bin);
            if (lane == __ffs(peers) - 1) myhist[bin] += (uint32_t)__popc(peers);
        }
        __syncwarp();
    }
    __syncthreads();
    // pass 2: thread t owns bin t: per-warp exclusive starts inside the bin, bin total; then an exclusive scan over the
    // bins in DESCENDING order (rank = 1023 - bin)
    {
        const int bin = threadIdx.x;
        uint32_t run = 0;
        for (int wv = 0; wv < kSortWarps; ++wv) {
            const uint32_t c = hist[wv * kBins + bin];
            hist[wv * kBins + bin] = run;
            run += c;
        }
        s_scan[kBins - 1 - bin] = run;
    }
    __syncthreads();
    {
        const uint32_t v = s_scan[threadIdx.x];  // total of rank threadIdx.x
        uint32_t incl = v;
        for (int off = 1; off < 32; off <<= 1) {
            const uint32_t nb = __shfl_up_sync(kFull, incl, off);
            if (lane >= off) incl += nb;
        }
        if (lane == 31) s_warp_tot[wid] = incl;
        __syncthreads();
        if (wid == 0) {
            const uint32_t t = s_warp_tot[lane];
            uint32_t ti = t;
            for (int off = 1; off < 32; off <<= 1) {
                const uint32_t nb = __shfl_up_sync(kFull, ti, off);
                if (lane >= off) ti += nb;
            }
            s_warp_tot[lane] = ti - t;
            if (lane == 31) D.nseeds[b] = (int)ti;
        }
        __syncthreads();
        base[kBins - 1 - threadIdx.x] = incl - v + s_warp_tot[wid];
    }
    __syncthreads();
    // pass 3: stable scatter
    uint32_t *order = D.order + (size_t)b * D.npx;
    for (int i0 = beg; i0 < end; i0 += 32) {
        const int i = i0 + lane;
        int bin = -1;
        if (i < end) {
            const int k = seed_k(img, D.sw, D.sh, i, D.kthr);
            if (k >= 0) bin = (int)(sqrt((double)k / 4.0) * bin_coef);
        }
        const unsigned act = __ballot_sync(kFull, bin >= 0);
        if (bin >= 0) {
            const unsigned peers = __match_any_sync(act, bin);
            const int rank = __popc(peers & ((1u << lane) - 1));
            const uint32_t start = myhist[bin];
            const int y = i / D.sw, x = i - y * D.sw;
            order[base[bin] + start + rank] = ((uint32_t)y << 16) | (uint32_t)x;
            __syncwarp(act);
            if (lane == __ffs(peers) - 1) myhist[bin] = start + (uint32_t)__popc(peers);
        }
        __syncwarp();
    }
}

// ------------------------------------------------------------------------------------------------------------------
// K5: segments -> KeyLines (LSDDetector_custom.cpp:266-300) + 2-D line functions (line_extractor.cc:147-159)
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32) keyline_kernel(LineDev D, plp_keyline *kl_out, double *fn_out, int32_t *n_out) {
    const int b = blockIdx.x, lane = threadIdx.x;
    const float4 *segs = D.segs + (size_t)b * D.seg_cap;
    plp_keyline *kls = kl_out + (size_t)b * D.kl_cap;
    double *fns = fn_out + (size_t)b * D.kl_cap * 3;
    const int nseg = D.nseg[b];
    int nk = 0, nc = 0;
    for (int s0 = 0; s0 < nseg; s0 += 32) {
        const int s = s0 + lane;
        float e0 = 0, e1 = 0, e2 = 0, e3 = 0;
        double length = 0;
        bool pass = false;
        if (s < nseg) {
            const float4 v = segs[s];
            e0 = v.x; e1 = v.y; e2 = v.z; e3 = v.w;
            // checkLineExtremes
            if (e0 < 0) e0 = 0;
            if (e0 >= D.w) e0 = (float)D.w - 1.0f;
            if (e2 < 0) e2 = 0;
            if (e2 >= D.w) e2 = (float)D.w - 1.0f;
            if (e1 < 0) e1 = 0;
            if (e1 >= D.h) e1 = (float)D.h - 1.0f;
            if (e3 < 0) e3 = 0;
            if (e3 >= D.h) e3 = (float)D.h - 1.0f;
            const double ddx = (double)(e0 - e2), ddy = (double)(e1 - e3);
            length = (double)(float)sqrt(ddx * ddx + ddy * ddy);
            // LSDDetector_custom.cpp:270 length > min_length; line_extractor.cc:136 lineLength >= 60
            pass = (length > D.min_length) && ((float)length >= 60.f);
        }
        // class_id counts every segment with length > min_length (also those the >= 60 filter would drop); with
        // min_length = 0.125 * min(w, h) >= 60 both filters coincide for images of at least 480 rows
        const bool counted = (s < nseg) && (length > D.min_length);
        const unsigned cm = __ballot_sync(kFull, counted);
        const unsigned pm = __ballot_sync(kFull, pass);
        if (pass) {
            const int pos = nk + __popc(pm & ((1u << lane) - 1));
            if (pos < D.kl_cap) {
                plp_keyline k;
                k.start_x = e0; k.start_y = e1; k.end_x = e2; k.end_y = e3;
                k.s_oct_x = e0; k.s_oct_y = e1; k.e_oct_x = e2; k.e_oct_y = e3;
                k.line_length = (float)length;
                const int x0 = __float2int_rn(e0), y0 = __float2int_rn(e1), x1 = __float2int_rn(e2), y1 = __float2int_rn(e3);
                k.num_pixels = max(abs(x1 - x0), abs(y1 - y0)) + 1;
                const float ay = e3 - e1, ax = e2 - e0;
                k.angle = (float)det_atan2((double)ay, (double)ax);
                k.class_id = nc + __popc(cm & ((1u << lane) - 1));
                k.octave = 0;
                k.size = (e2 - e0) * (e3 - e1);
                k.response = k.line_length / (float)max(D.w, D.h);
                k.pt_x = (e2 + e0) / 2;
                k.pt_y = (e3 + e1) / 2;
                kls[pos] = k;
                const double sx = e0, sy = e1, ex = e2, ey = e3;
                const double l0 = sy - ey, l1 = ex - sx, l2 = sx * ey - sy * ex;
                const double nrm = sqrt(l0 * l0 + l1 * l1);
                fns[3 * pos] = l0 / nrm;
                fns[3 * pos + 1] = l1 / nrm;
                fns[3 * pos + 2] = l2 / nrm;
            } else {
                atomicOr(&D.status[b], 2);
            }
        }
        nk += __popc(pm);
        nc += __popc(cm);
    }
    if (lane == 0) n_out[b] = min(nk, D.kl_cap);
}

// ------------------------------------------------------------------------------------------------------------------
// K6: GaussianBlur(5x5, sigma 1) (Q8 taps 14 62 104 62 14) + Sobel 3x3 -> int16 (dx, dy); reflect-101 borders
//     (binary_descriptor_custom.cpp:347-395).  One CTA = 32 x 8 pixels.
// ------------------------------------------------------------------------------------------------------------------
constexpr int kGrTw = 32, kGrTh = 8;
__global__ void __launch_bounds__(256) lbd_gradient_kernel(LineDev D) {
    // The reflect-101 extension of the image is symmetric about every border, and so is its blur with a symmetric
    // kernel: blurred(reflect(p)) == blur of the extended image at p.  The tile is therefore staged by plain reflected
    // coordinates (blur halo 2 + Sobel halo 1) and filtered separably.
    __shared__ uint8_t s_src[kGrTh + 6][kGrTw + 8];
    __shared__ uint16_t s_h[kGrTh + 6][kGrTw + 2];
    __shared__ uint8_t s_b[kGrTh + 2][kGrTw + 2];
    const int b = blockIdx.y;
    const int tiles_x = (D.w + kGrTw - 1) / kGrTw;
    const int tx = (blockIdx.x % tiles_x) * kGrTw, ty = (blockIdx.x / tiles_x) * kGrTh;
    const uint8_t *img = D.img + (size_t)b * D.img_frame_stride;
    for (int i = threadIdx.x; i < (kGrTh + 6) * (kGrTw + 6); i += blockDim.x) {
        const int r = i / (kGrTw + 6), c = i - r * (kGrTw + 6);
        s_src[r][c] = img[(size_t)reflect101(ty + r - 3, D.h) * D.img_step + reflect101(tx + c - 3, D.w)];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < (kGrTh + 6) * (kGrTw + 2); i += blockDim.x) {
        const int r = i / (kGrTw + 2), c = i - r * (kGrTw + 2);
        const uint8_t *q = &s_src[r][c];
        s_h[r][c] = (uint16_t)(14 * (q[0] + q[4]) + 62 * (q[1] + q[3]) + 104 * q[2]);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < (kGrTh + 2) * (kGrTw + 2); i += blockDim.x) {
        const int r = i / (kGrTw + 2), c = i - r * (kGrTw + 2);
        const uint32_t v = 14u * (s_h[r][c] + s_h[r + 4][c]) + 62u * (s_h[r + 1][c] + s_h[r + 3][c]) + 104u * s_h[r + 2][c];
        s_b[r][c] = (uint8_t)((v + 32768u) >> 16);
    }
    __syncthreads();
    short2 *out = D.grad + (size_t)b * D.w * D.h;
    for (int i = threadIdx.x; i < kGrTh * kGrTw; i += blockDim.x) {
        const int r = i / kGrTw, c = i - r * kGrTw;
        const int x = tx + c, y = ty + r;
        if (x >= D.w || y >= D.h) continue;
        const int a00 = s_b[r][c], a01 = s_b[r][c + 1], a02 = s_b[r][c + 2];
        const int a10 = s_b[r + 1][c], a12 = s_b[r + 1][c + 2];
        const int a20 = s_b[r + 2][c], a21 = s_b[r + 2][c + 1], a22 = s_b[r + 2][c + 2];
        const int gx = (a02 - a00) + 2 * (a12 - a10) + (a22 - a20);
        const int gy = (a20 - a00) + 2 * (a21 - a01) + (a22 - a02);
        out[(size_t)y * D.w + x] = make_short2((short)gx, (short)gy);
    }
}

// ------------------------------------------------------------------------------------------------------------------
// K7: LBD (binary_descriptor_custom.cpp:1018-1364 + 398-408, 642-646): one CTA of 64 threads per line; thread = row
//     of the 63-row line support region (the row sums are sequential float accumulations along the line, kept in the
//     reference's order); 9 threads accumulate the bands in row order; thread 0 normalises and packs the 32 bytes.
// ------------------------------------------------------------------------------------------------------------------
__constant__ int c_comb[32][2] = {{0, 1}, {0, 2}, {0, 3}, {0, 4}, {0, 5}, {0, 6}, {1, 2}, {1, 3}, {1, 4}, {1, 5}, {1, 6},
                                  {2, 3}, {2, 4}, {2, 5}, {2, 6}, {2, 7}, {2, 8}, {3, 4}, {3, 5}, {3, 6}, {3, 7}, {3, 8},
                                  {4, 5}, {4, 6}, {4, 7}, {4, 8}, {5, 6}, {5, 7}, {5, 8}, {6, 7}, {6, 8}, {7, 8}};

__global__ void __launch_bounds__(64) lbd_kernel(LineDev D, const plp_keyline *kl_in, const int32_t *n_in, uint8_t *lbd_out) {
    __shared__ float s_row[kLspHeight][4];   // pl, nl, po, no of each row (already multiplied by the global weight)
    __shared__ float s_band[8][kBands];
    __shared__ float s_des[kBands * 8];
    const int b = blockIdx.y, t = threadIdx.x;
    const int n = n_in[b];
    const short2 *grad = D.grad + (size_t)b * D.w * D.h;
    for (int line = blockIdx.x; line < n; line += gridDim.x) {
        const plp_keyline kl = kl_in[(size_t)b * D.kl_cap + line];
        const short image_w = (short)(D.w - 1), image_h = (short)(D.h - 1);
        const short length_lsp = (short)kl.num_pixels;
        const short half_h = (kLspHeight - 1) / 2;
        const short half_w = (length_lsp - 1) / 2;
        const float mid_x = (float)(0.5 * (kl.s_oct_x + kl.e_oct_x));
        const float mid_y = (float)(0.5 * (kl.s_oct_y + kl.e_oct_y));
        const float dl0 = (float)det_cos((double)kl.angle), dl1 = (float)det_sin((double)kl.angle);
        const float do0 = -dl1, do1 = dl0;
        if (t < kLspHeight) {
            float scx0 = -dl0 * half_w + dl1 * half_h + mid_x;
            float scy0 = -dl1 * half_w - dl0 * half_h + mid_y;
            for (int hh = 0; hh < t; ++hh) {  // the reference walks the rows with running float sums
                scx0 -= dl1;
                scy0 += dl0;
            }
            float scx = scx0, scy = scy0;
            float pl = 0, nl = 0, po = 0, no = 0;
            for (short wid = 0; wid < length_lsp; ++wid) {
                short tc = (short)roundf(scx);
                const short xc = (tc < 0) ? 0 : (tc > image_w) ? image_w : tc;
                tc = (short)roundf(scy);
                const short yc = (tc < 0) ? 0 : (tc > image_h) ? image_h : tc;
                const short2 gd = grad[(size_t)yc * D.w + xc];
                const float gdl = gd.x * dl0 + gd.y * dl1;
                const float gdo = gd.x * do0 + gd.y * do1;
                if (gdl > 0) pl += gdl; else nl -= gdl;
                if (gdo > 0) po += gdo; else no -= gdo;
                scx += dl0;
                scy += dl1;
            }
            const float coef = D.gauss_g[t];
            s_row[t][0] = coef * pl;
            s_row[t][1] = coef * nl;
            s_row[t][2] = coef * po;
            s_row[t][3] = coef * no;
        }
        __syncthreads();
        if (t < kBands) {
            float bs[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            const int h0 = max(0, (t - 1) * kBandWidth), h1 = min(kLspHeight, (t + 2) * kBandWidth);
            for (int hid = h0; hid < h1; ++hid) {
                const int hb = hid / kBandWidth;
                // row of band hb contributes to band t with: own band -> gl[r + 7]; band above (t == hb - 1) -> gl[r + 14];
                // band below (t == hb + 1) -> gl[r]
                const int rr = hid % kBandWidth;
                const float c = (t == hb) ? D.gauss_l[rr + kBandWidth] : (t == hb - 1) ? D.gauss_l[rr + 2 * kBandWidth] : D.gauss_l[rr];
                const float pl = s_row[hid][0], nl = s_row[hid][1], po = s_row[hid][2], no = s_row[hid][3];
                const float pl2 = pl * pl, nl2 = nl * nl, po2 = po * po, no2 = no * no;
                bs[0] += c * pl;
                bs[1] += c * nl;
                bs[2] += c * c * pl2;
                bs[3] += c * c * nl2;
                bs[4] += c * po;
                bs[5] += c * no;
                bs[6] += c * c * po2;
                bs[7] += c * c * no2;
            }
#pragma unroll
            for (int q = 0; q < 8; ++q) s_band[q][t] = bs[q];
        }
        __syncthreads();
        if (t == 0) {
            const float inv_n2 = (float)(1.0 / (kBandWidth * 2.0)), inv_n3 = (float)(1.0 / (kBandWidth * 3.0));
            for (int bb = 0; bb < kBands; ++bb) {
                const float inv_n = (bb == 0 || bb == kBands - 1) ? inv_n2 : inv_n3;
                float *d = s_des + bb * 8;
                float tt = s_band[0][bb] * inv_n;
                d[0] = tt;
                d[4] = sqrtf(s_band[2][bb] * inv_n - tt * tt);
                tt = s_band[1][bb] * inv_n;
                d[1] = tt;
                d[5] = sqrtf(s_band[3][bb] * inv_n - tt * tt);
                tt = s_band[4][bb] * inv_n;
                d[2] = tt;
                d[6] = sqrtf(s_band[6][bb] * inv_n - tt * tt);
                tt = s_band[5][bb] * inv_n;
                d[3] = tt;
                d[7] = sqrtf(s_band[7][bb] * inv_n - tt * tt);
            }
            float tm = 0, ts = 0;
            for (int bb = 0; bb < kBands; ++bb) {
                const float *d = s_des + bb * 8;
                tm += d[0] * d[0];
                tm += d[1] * d[1];
                tm += d[2] * d[2];
                tm += d[3] * d[3];
                ts += d[4] * d[4];
                ts += d[5] * d[5];
                ts += d[6] * d[6];
                ts += d[7] * d[7];
            }
            tm = 1 / sqrtf(tm);
            ts = 1 / sqrtf(ts);
            for (int bb = 0; bb < kBands; ++bb) {
                float *d = s_des + bb * 8;
                for (int q = 0; q < 4; ++q) d[q] = d[q] * tm;
                for (int q = 4; q < 8; ++q) d[q] = d[q] * ts;
            }
            for (int q = 0; q < kBands * 8; ++q)
                if ((double)s_des[q] > 0.4) s_des[q] = (float)0.4;
            float tt = 0;
            for (int q = 0; q < kBands * 8; ++q) tt += s_des[q] * s_des[q];
            tt = 1 / sqrtf(tt);
            for (int q = 0; q < kBands * 8; ++q) s_des[q] = s_des[q] * tt;
        }
        __syncthreads();
        if (t < 32) {
            const float *f1 = s_des + 8 * c_comb[t][0], *f2 = s_des + 8 * c_comb[t][1];
            unsigned r = 0;
#pragma unroll
            for (int q = 0; q < 8; ++q)
                if (f1[q] > f2[q]) r |= (1u << q);
            lbd_out[((size_t)b * D.kl_cap + line) * 32 + t] = (uint8_t)r;
        }
        if (D.lbd_float)
            for (int q = t; q < kBands * 8; q += 64) D.lbd_float[((size_t)b * D.kl_cap + line) * 72 + q] = s_des[q];
        __syncthreads();
    }
}

}  // namespace

// ====================================================================================================================
struct plp_line {
    plp_ctx *ctx = nullptr;
    int rows = 0, cols = 0, max_batch = 0, last_batch = 0;
    LineDev dev{};
    uint8_t *d_img = nullptr;
    plp_keyline *d_kl = nullptr;
    uint8_t *d_lbd = nullptr;
    double *d_fn = nullptr;
    int32_t *d_n = nullptr;
    size_t sort_smem = 0, grow_smem = 0, grow_smem_noimg = 0;
    bool img_smem_ok = true;
    int resident_smem_frames = 0;
    bool force_global_image = false;
    int grow_variant = 0;  // 0 automatic, 1 one warp per frame, 2 multi-warp rounds (lsd_grow_mw_kernel), 3 out of order (lsd_grow_ooo_kernel)
    int ooo_warps = 0;
    bool host_call = false;   // inside the host-pointer entry point (a live frame): automatic mode may take the out-of-order kernel
    bool used_ooo = false;    // the last run did
    int ooo_fallbacks = 0;    // host calls that were re-run with the round protocol after an out-of-order timeout
    size_t ooo_smem = 0;
    int mw_warps = 0, mw_max_batch = 0;
    size_t mw_smem = 0;
    uint32_t *d_reg_mw = nullptr;
    float4 *d_cstab = nullptr;
    std::vector<void *> owned;
};

template <class T>
static plp_status dev_alloc(plp_line *h, T **p, size_t count) {
    void *q = nullptr;
    cudaError_t e = cudaMalloc(&q, std::max<size_t>(count, 1) * sizeof(T));
    if (e != cudaSuccess) {
        set_error("cudaMalloc(%zu bytes) failed: %s", count * sizeof(T), cudaGetErrorString(e));
        return PLP_ERR_CUDA;
    }
    h->owned.push_back(q);
    *p = (T *)q;
    return PLP_OK;
}

static plp_status line_run(plp_line *h, const uint8_t *d_imgs, int batch, size_t step, plp_keyline *d_kl, uint8_t *d_lbd,
                           double *d_fn, int32_t *d_n, int32_t *d_status) {
    plp_ctx *ctx = h->ctx;
    LineDev D = h->dev;
    D.img = d_imgs;
    D.img_step = step;
    D.img_frame_stride = step * (size_t)h->rows;
    if (d_status) D.status = d_status;
    h->last_batch = batch;
    PLP_CUDA_TRY(cudaMemsetAsync(D.status, 0, (size_t)batch * sizeof(int), ctx->stream));
    {
        dim3 grid(div_up(D.w, kScTw) * div_up(D.h, kScTh), batch);
        PLP_LAUNCH(ctx, lsd_scale_kernel, grid, 256, 0, D);
    }
    PLP_LAUNCH(ctx, lsd_sort_kernel, batch, kSortWarps * 32, h->sort_smem, D);
    // small batches (at most half of what stays resident, so that a second handle -- the right image of a stereo pair --
    // fits beside it): image in shared memory (latency); larger batches: image through L2, 3x the frames per SM
    // a wave of frames or less: the frame-level parallelism cannot fill the GPU, several warps per frame (speculative, in-order
    // commit) cut the latency of a live frame instead
    const bool mw = h->mw_warps >= 2 && batch <= h->mw_max_batch && h->grow_variant != 1 &&
                    (h->grow_variant >= 2 || 2 * batch <= ctx->sm_count);  // half a wave: a second handle (stereo) fits beside it
    // automatic mode takes the out-of-order kernel for a live frame or stereo pair through the host entry point (which re-runs
    // the frame with the round protocol should the kernel ever give up)
    const bool ooo = mw && h->ooo_warps >= 2 &&
                     (h->grow_variant == 3 || (h->grow_variant == 0 && h->host_call && batch <= 2));
    h->used_ooo = ooo;
    if (ooo) {
        PLP_LAUNCH(ctx, lsd_grow_ooo_kernel, batch, h->ooo_warps * 32, h->ooo_smem, D, h->d_reg_mw);
    } else if (mw) {
        PLP_LAUNCH(ctx, lsd_grow_mw_kernel, batch, h->mw_warps * 32, h->mw_smem, D, h->d_reg_mw);
    } else if (h->img_smem_ok && 2 * batch <= h->resident_smem_frames && !h->force_global_image) {
        PLP_LAUNCH(ctx, lsd_grow_kernel<true>, batch, 32, h->grow_smem, D);
    } else {
        PLP_LAUNCH(ctx, lsd_grow_kernel<false>, batch, 32, h->grow_smem_noimg, D);
    }
    PLP_LAUNCH(ctx, keyline_kernel, batch, 32, 0, D, d_kl, d_fn, d_n);
    {
        dim3 grid(div_up(D.w, kGrTw) * div_up(D.h, kGrTh), batch);
        PLP_LAUNCH(ctx, lbd_gradient_kernel, grid, 256, 0, D);
    }
    {
        dim3 grid(256, batch);
        PLP_LAUNCH(ctx, lbd_kernel, grid, 64, 0, D, d_kl, d_n, d_lbd);
    }
    PLP_CHECK_LAUNCH();
    return PLP_OK;
}

extern "C" {

void plp_line_destroy(plp_line *h) {
    if (!h) return;
    cudaSetDevice(h->ctx->device);
    cudaStreamSynchronize(h->ctx->stream);
    for (void *p : h->owned) cudaFree(p);
    delete h;
}

plp_status plp_line_create(plp_ctx *ctx, int rows, int cols, int max_batch, plp_line **out) {
    PLP_REQUIRE(ctx && out, "null pointer");
    *out = nullptr;
    PLP_REQUIRE(rows >= 16 && cols >= 16 && rows < 32768 && cols < 32768, "image size");
    PLP_REQUIRE(max_batch >= 1, "max_batch");
    PLP_CUDA_TRY(cudaSetDevice(ctx->device));
    plp_line *h = new plp_line();
    h->ctx = ctx;
    h->rows = rows;
    h->cols = cols;
    h->max_batch = max_batch;
    LineDev &D = h->dev;
    D.w = cols;
    D.h = rows;
    D.sw = (int)lrint(cols * 0.5);
    D.sh = (int)lrint(rows * 0.5);
    D.npx = D.sw * D.sh;
    // line_extractor.cc:113-122 / lsd.cpp flsd
    const double ang_th = 22.5, quant = 2.0;
    D.prec = kPi * ang_th / 180;
    D.p = ang_th / 180;
    D.rho = quant / std::sin(D.prec);
    D.density_th = 0.6;
    const double log_nt = 5 * (std::log10((double)D.sw) + std::log10((double)D.sh)) / 2 + std::log10(11.0);
    D.min_reg_size = (int)(size_t)(-log_nt / std::log10(D.p));
    D.min_length = 0.125 * std::min(cols, rows);
    D.seg_cap = D.npx / std::max(D.min_reg_size, 2) + 1;
    {  // largest squared norm with sqrt(k / 4.0) <= rho (lsd.cpp: `norm <= threshold` -> NOTDEF)
        int k = (int)std::floor(4.0 * D.rho * D.rho) + 2;
        while (k > 0 && !(std::sqrt((double)k / 4.0) <= D.rho)) --k;
        D.kthr = k;
    }
    D.kl_cap = 1024;
    {  // LBD weights, binary_descriptor_custom.cpp:229-257 (integer divisions kept)
        double u = (kBandWidth * 3 - 1) / 2;
        double sigma = (kBandWidth * 2 + 1) / 2;
        double inv = -1 / (2 * sigma * sigma);
        for (int i = 0; i < kBandWidth * 3; ++i) {
            const double dis = i - u;
            D.gauss_l[i] = (float)std::exp(dis * dis * inv);
        }
        u = (kBands * kBandWidth - 1) / 2;
        sigma = u;
        inv = -1 / (2 * sigma * sigma);
        for (int i = 0; i < kLspHeight; ++i) {
            const double dis = i - u;
            D.gauss_g[i] = (float)std::exp(dis * dis * inv);
        }
    }
    const size_t B = max_batch, npx = D.npx;
    plp_status st = PLP_OK;
#define A(call) if (st == PLP_OK) st = (call)
    A(dev_alloc(h, &D.scaled, B * npx));
    A(dev_alloc(h, &D.order, B * npx));
    A(dev_alloc(h, &D.nseeds, B));
    A(dev_alloc(h, &D.reg_xy, B * npx));
    A(dev_alloc(h, &D.segs, B * D.seg_cap));
    A(dev_alloc(h, &D.nseg, B));
    A(dev_alloc(h, &D.grad, B * (size_t)rows * cols));
    A(dev_alloc(h, &D.lbd_float, B * D.kl_cap * 72));
    A(dev_alloc(h, &D.status, B));
    A(dev_alloc(h, &h->d_img, B * (size_t)rows * cols));
    A(dev_alloc(h, &h->d_kl, B * D.kl_cap));
    A(dev_alloc(h, &h->d_lbd, B * D.kl_cap * 32));
    A(dev_alloc(h, &h->d_fn, B * D.kl_cap * 3));
    A(dev_alloc(h, &h->d_n, B));
    if (st != PLP_OK) {
        plp_line_destroy(h);
        return st;
    }
    A(dev_alloc(h, &h->d_cstab, (size_t)kGDim * kGDim));
    if (st != PLP_OK) {
        plp_line_destroy(h);
        return st;
    }
#undef A
    D.cstab = h->d_cstab;
    lsd_cs_table_kernel<<<div_up(kGDim * kGDim, 256), 256, 0, ctx->stream>>>(h->d_cstab);
    ctx->launches++;
    h->sort_smem = ((size_t)kSortWarps * kBins + kBins) * sizeof(uint32_t);
    const size_t used_bytes = (size_t)((((D.npx + 31) >> 5) + 3) & ~3) * 4;
    D.reg_cap_small = kRegCapSmall;
    h->grow_smem_noimg = used_bytes + (size_t)D.reg_cap_small * 4;
    h->grow_smem = (size_t)((D.npx + 15) & ~15) + used_bytes + (size_t)kRegCap * 4;
    h->img_smem_ok = h->grow_smem <= 227 * 1024;
    if (h->grow_smem_noimg > 227 * 1024) {
        set_error("line: a %d x %d image needs %zu bytes of shared memory per frame (limit 232448)", cols, rows,
                  h->grow_smem_noimg);
        plp_line_destroy(h);
        return PLP_ERR_CAPACITY;
    }
    h->resident_smem_frames = h->img_smem_ok ? ctx->sm_count * (int)std::max<size_t>(1, (227 * 1024) / (h->grow_smem + 1024)) : 0;
    plp_status so = PLP_OK;
    if (h->img_smem_ok) so = ensure_smem_optin((const void *)lsd_grow_kernel<true>, h->grow_smem, "lsd_grow_kernel<true>");
    if (so == PLP_OK) so = ensure_smem_optin((const void *)lsd_grow_kernel<false>, h->grow_smem_noimg, "lsd_grow_kernel<false>");
    if (so == PLP_OK) so = ensure_smem_optin((const void *)lsd_sort_kernel, h->sort_smem, "lsd_sort_kernel");
    {  // multi-warp variant: image + committed bitmap + per warp {private bitmap, region window}
        const size_t fixed = (size_t)((D.npx + 15) & ~15) + used_bytes + sizeof(MwCtl) + 64, per_warp = used_bytes + (size_t)kMwRegCap * 4;
        const size_t budget = 227 * 1024;
        h->mw_warps = fixed + 2 * per_warp <= budget ? (int)std::min<size_t>(kMwMaxWarps, (budget - fixed) / per_warp) : 0;
        h->mw_smem = fixed + (size_t)h->mw_warps * per_warp;
        h->mw_max_batch = h->mw_warps >= 2 ? std::min(max_batch, ctx->sm_count) : 0;
        if (h->mw_warps >= 2) {
            if (so == PLP_OK) so = ensure_smem_optin((const void *)lsd_grow_mw_kernel, h->mw_smem, "lsd_grow_mw_kernel");
            if (so == PLP_OK) so = dev_alloc(h, &h->d_reg_mw, (size_t)h->mw_max_batch * (kMwMaxWarps + 1) * D.npx);
            // out-of-order variant: one more private bitmap + window (execution at the head), the reorder buffer
            const size_t ofixed = (size_t)((D.npx + 15) & ~15) + 3 * used_bytes + (size_t)kOooRegCap * 4 + sizeof(OooEntry) * kOooRing +
                                  sizeof(OooCtl) + 64, oper = used_bytes + (size_t)kOooRegCap * 4;
            h->ooo_warps = ofixed + 2 * oper <= budget ? (int)std::min<size_t>(kMwMaxWarps, (budget - ofixed) / oper) : 0;
            h->ooo_smem = ofixed + (size_t)h->ooo_warps * oper;
            if (h->ooo_warps >= 2 && so == PLP_OK)
                so = ensure_smem_optin((const void *)lsd_grow_ooo_kernel, h->ooo_smem, "lsd_grow_ooo_kernel");
            if (so == PLP_OK) so = dev_alloc(h, &h->dev.mw_stat, (size_t)8 * max_batch);
            if (so == PLP_OK && cudaMemsetAsync(h->dev.mw_stat, 0, (size_t)8 * max_batch * 8, ctx->stream) != cudaSuccess) so = PLP_ERR_CUDA;
        }
    }
    if (so != PLP_OK) {
        plp_line_destroy(h);
        return so;
    }
    *out = h;
    return PLP_OK;
}

int plp_line_capacity(const plp_line *h) { return h ? h->dev.kl_cap : 0; }

plp_status plp_line_extract_batch_dev(plp_line *h, const uint8_t *d_imgs, int batch, size_t step, plp_keyline *d_kl,
                                      uint8_t *d_lbd, double *d_fn, int32_t *d_n, int32_t *d_status) {
    PLP_REQUIRE(h && d_imgs && d_kl && d_lbd && d_fn && d_n, "null pointer");
    PLP_REQUIRE(batch >= 1 && batch <= h->max_batch, "batch exceeds the handle's max_batch");
    PLP_REQUIRE(step >= (size_t)h->cols, "step < cols");
    PLP_CUDA_TRY(cudaSetDevice(h->ctx->device));
    return line_run(h, d_imgs, batch, step, d_kl, d_lbd, d_fn, d_n, d_status);
}

static plp_status line_extract_host(plp_line *h, const uint8_t *imgs, int batch, size_t step, plp_keyline *kl_out,
                                    uint8_t *lbd_out, double *fn_out, int32_t *n_out) {
    plp_ctx *ctx = h->ctx;
    PLP_CUDA_TRY(cudaSetDevice(ctx->device));
    const size_t rows = h->rows, cols = h->cols, cap = h->dev.kl_cap;
    PLP_CUDA_TRY(cudaMemcpy2DAsync(h->d_img, cols, imgs, step, cols, rows * (size_t)batch, cudaMemcpyHostToDevice,
                                   ctx->stream));
    std::vector<int> status(batch);
    auto run_and_fetch = [&]() -> plp_status {
        h->host_call = true;
        const plp_status rs = line_run(h, h->d_img, batch, cols, h->d_kl, h->d_lbd, h->d_fn, h->d_n, nullptr);
        h->host_call = false;
        PLP_TRY(rs);
        PLP_CUDA_TRY(cudaMemcpyAsync(n_out, h->d_n, (size_t)batch * 4, cudaMemcpyDeviceToHost, ctx->stream));
        PLP_CUDA_TRY(cudaMemcpyAsync(kl_out, h->d_kl, (size_t)batch * cap * sizeof(plp_keyline), cudaMemcpyDeviceToHost, ctx->stream));
        PLP_CUDA_TRY(cudaMemcpyAsync(lbd_out, h->d_lbd, (size_t)batch * cap * 32, cudaMemcpyDeviceToHost, ctx->stream));
        PLP_CUDA_TRY(cudaMemcpyAsync(fn_out, h->d_fn, (size_t)batch * cap * 3 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        PLP_CUDA_TRY(cudaMemcpyAsync(status.data(), h->dev.status, (size_t)batch * 4, cudaMemcpyDeviceToHost, ctx->stream));
        PLP_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
        return PLP_OK;
    };
    PLP_TRY(run_and_fetch());
    bool gave_up = false;
    for (int b = 0; b < batch; ++b) gave_up = gave_up || (status[b] & 2) != 0;
    if (gave_up && h->used_ooo && h->grow_variant == 0) {
        // the out-of-order region growing bounds every wait; should it ever give up in automatic mode, the frames are run
        // again with the round protocol (still on the GPU) -- an explicitly selected variant 3 reports the failure instead
        h->ooo_fallbacks++;
        h->grow_variant = 2;
        const plp_status r2 = run_and_fetch();
        h->grow_variant = 0;
        PLP_TRY(r2);
    }
    for (int b = 0; b < batch; ++b)
        if (status[b] != 0) {
            set_error("line: capacity overflow in frame %d (code %d)", b, status[b]);
            return PLP_ERR_CAPACITY;
        }
    return PLP_OK;
}

plp_status plp_line_extract(plp_line *h, const uint8_t *img, int rows, int cols, size_t step, plp_keyline *kl_out,
                            uint8_t *lbd_out, double *fn_out, int *n_out) {
    PLP_REQUIRE(h && n_out, "null pointer");
    *n_out = 0;
    PLP_REQUIRE(img && kl_out && lbd_out && fn_out, "null pointer");
    PLP_REQUIRE(rows == h->rows && cols == h->cols, "image size differs from the handle's");
    PLP_REQUIRE(step >= (size_t)cols, "step < cols");
    int32_t n = 0;
    PLP_TRY(line_extract_host(h, img, 1, step, kl_out, lbd_out, fn_out, &n));
    *n_out = n;
    return PLP_OK;
}

plp_status plp_line_extract_batch(plp_line *h, const uint8_t *imgs, int batch, size_t step, plp_keyline *kl_out,
                                  uint8_t *lbd_out, double *fn_out, int32_t *n_out) {
    PLP_REQUIRE(h && imgs && kl_out && lbd_out && fn_out && n_out, "null pointer");
    PLP_REQUIRE(batch >= 1 && batch <= h->max_batch, "batch exceeds the handle's max_batch");
    PLP_REQUIRE(step >= (size_t)h->cols, "step < cols");
    return line_extract_host(h, imgs, batch, step, kl_out, lbd_out, fn_out, n_out);
}

plp_status plp_line_debug_force_global_image(plp_line *h, int on) {
    PLP_REQUIRE(h, "null pointer");
    h->force_global_image = on != 0;
    return PLP_OK;
}

plp_status plp_line_debug_grow_variant(plp_line *h, int variant) {
    PLP_REQUIRE(h && variant >= 0 && variant <= 3, "variant must be 0 (automatic), 1 (one warp per frame), 2 (multi-warp rounds) or 3 (out of order)");
    PLP_REQUIRE(variant < 2 || h->mw_warps >= 2, "the multi-warp variants do not fit the shared memory at this image size");
    PLP_REQUIRE(variant != 3 || h->ooo_warps >= 2, "the out-of-order variant does not fit the shared memory at this image size");
    h->grow_variant = variant;
    return PLP_OK;
}

int plp_line_debug_ooo_fallbacks(const plp_line *h) { return h ? h->ooo_fallbacks : 0; }

plp_status plp_line_debug_grow_stats(plp_line *h, int b, unsigned long long *out3) {
    PLP_REQUIRE(h && out3, "null pointer");
    PLP_REQUIRE(b >= 0 && b < h->max_batch, "index");
    for (int q = 0; q < 8; ++q) out3[q] = 0;
    if (!h->dev.mw_stat) return PLP_OK;
    plp_ctx *ctx = h->ctx;
    PLP_CUDA_TRY(cudaSetDevice(ctx->device));
    PLP_CUDA_TRY(cudaMemcpyAsync(out3, h->dev.mw_stat + 8 * (size_t)b, 64, cudaMemcpyDeviceToHost, ctx->stream));
    PLP_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return PLP_OK;
}

plp_status plp_line_debug_segments(plp_line *h, int b, float *segs_out, int cap, int *n_out) {
    PLP_REQUIRE(h && segs_out && n_out, "null pointer");
    PLP_REQUIRE(b >= 0 && b < h->last_batch, "index");
    plp_ctx *ctx = h->ctx;
    PLP_CUDA_TRY(cudaSetDevice(ctx->device));
    int n = 0;
    PLP_CUDA_TRY(cudaMemcpyAsync(&n, h->dev.nseg + b, 4, cudaMemcpyDeviceToHost, ctx->stream));
    PLP_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    *n_out = n;
    PLP_REQUIRE(n <= cap, "cap too small");
    PLP_CUDA_TRY(cudaMemcpyAsync(segs_out, h->dev.segs + (size_t)b * h->dev.seg_cap, (size_t)n * 16, cudaMemcpyDeviceToHost,
                                 ctx->stream));
    PLP_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return PLP_OK;
}

plp_status plp_line_debug_scaled(plp_line *h, int b, uint8_t *out) {
    PLP_REQUIRE(h && out, "null pointer");
    PLP_REQUIRE(b >= 0 && b < h->last_batch, "index");
    plp_ctx *ctx = h->ctx;
    PLP_CUDA_TRY(cudaSetDevice(ctx->device));
    PLP_CUDA_TRY(cudaMemcpyAsync(out, h->dev.scaled + (size_t)b * h->dev.npx, h->dev.npx, cudaMemcpyDeviceToHost, ctx->stream));
    PLP_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return PLP_OK;
}

plp_status plp_line_debug_lbd_float(plp_line *h, int b, float *out, int cap) {
    PLP_REQUIRE(h && out, "null pointer");
    PLP_REQUIRE(b >= 0 && b < h->last_batch && cap >= 0 && cap <= h->dev.kl_cap, "index");
    plp_ctx *ctx = h->ctx;
    PLP_CUDA_TRY(cudaSetDevice(ctx->device));
    PLP_CUDA_TRY(cudaMemcpyAsync(out, h->dev.lbd_float + (size_t)b * h->dev.kl_cap * 72, (size_t)cap * 72 * sizeof(float),
                                 cudaMemcpyDeviceToHost, ctx->stream));
    PLP_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return PLP_OK;
}

}  // extern "C"
