// match_common.cuh -- device building blocks of the Hamming matchers (match.cu, point_match_kernels.cuh,
// fuse_kernels.cuh, bow_kernels.cuh): descriptor loads, the orientation check of angle_checker.h, the grid window and
// cell order of data/common.cc, warp reductions of (distance, position) keys and the pinhole reprojection.  Free of
// host-side CUDA runtime dependencies so that tests/cta_emu can compile the same text for the host.
//
// The reprojection, window and bin arithmetic round like the oracle only in translation units compiled with
// -fmad=false (build.py FILE_FLAGS: match.cu, fuse.cu, bow.cu); a new user must be compiled the same way.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include "../../include/plpslam_b200.h"
#include "devmath.cuh"

namespace plp {

constexpr int kHistLen = 30;     // angle_checker.h:47
constexpr int kNumBinsThr = 3;   // angle_checker.h:48
constexpr int kNoOwner = 0x7fffffff;

__device__ __forceinline__ void load_desc(const uint8_t *p, uint4 &a, uint4 &b) {
    const uint4 *q = reinterpret_cast<const uint4 *>(p);
    a = __ldg(q);
    b = __ldg(q + 1);
}

// ---- orientation check (angle_checker.h:86-175)

// angle_checker.h:100-113: ORB-SLAM's round(delta / 30) bin
__device__ __forceinline__ int angle_bin(float delta_angle) {
    if (delta_angle < 0.0) delta_angle = (float)((double)delta_angle + 360.0);
    if (360.0 <= delta_angle) delta_angle = (float)((double)delta_angle - 360.0);
    const float inv_len = 1.0f / (float)kHistLen;
    return __float2int_rn(delta_angle * inv_len);
}

// angle_checker.h:163-175: rank bins by size (desc), ties by bin index (asc, the strict '<' of a stable sort); the
// first kNumBinsThr are valid.  One thread.
__device__ inline void rank_bins(const int *hist, uint8_t *bin_valid) {
    bool used[kHistLen];
    for (int b = 0; b < kHistLen; ++b) {
        used[b] = false;
        bin_valid[b] = 0;
    }
    for (int k = 0; k < kNumBinsThr; ++k) {
        int best = -1, best_cnt = -1;
        for (int b = 0; b < kHistLen; ++b)
            if (!used[b] && hist[b] > best_cnt) {
                best_cnt = hist[b];
                best = b;
            }
        used[best] = true;
        bin_valid[best] = 1;
    }
}

// Called by every thread of the CTA.  Adds the number of matches (choice[q] >= 0, q < m) to *num_matched and sets
// bin_valid[b]: with do_angle, the top kNumBinsThr bins of the histogram of angle_bin(delta(q, choice[q])); without,
// every bin.  A match q is kept iff !do_angle || bin_valid[angle_bin(delta(q, choice[q]))].  On entry hist (kHistLen)
// is zero and *num_matched holds its start value, both visible to every thread.
template <int Threads, class Delta>
__device__ __forceinline__ void orientation_check(int m, const int32_t *choice, bool do_angle, int *hist,
                                                  uint8_t *bin_valid, int *num_matched, Delta delta) {
    const int tid = threadIdx.x;
    for (int q = tid; q < m; q += Threads) {
        const int c = choice[q];
        if (c < 0) continue;
        atomicAdd(num_matched, 1);
        if (do_angle) atomicAdd(&hist[angle_bin(delta(q, c))], 1);
    }
    __syncthreads();
    if (tid == 0) {
        if (do_angle)
            rank_bins(hist, bin_valid);
        else
            for (int b = 0; b < kHistLen; ++b) bin_valid[b] = 1;
    }
    __syncthreads();
}

// ---- the keypoint grid (data/common.cc:205-313)

// the window of a query in grid cells (data/common.cc:249-272); false if it misses the grid
struct Window {
    int min_cx, max_cx, min_cy, max_cy;
};
__device__ __forceinline__ bool query_window(const plp_grid &grid, float ref_x, float ref_y, float r, Window &w) {
    w.min_cx = max(0, cv_floor((double)(ref_x - grid.min_x - r) * grid.inv_cell_width));
    w.max_cx = min(grid.num_cols - 1, cv_ceil((double)(ref_x - grid.min_x + r) * grid.inv_cell_width));
    w.min_cy = max(0, cv_floor((double)(ref_y - grid.min_y - r) * grid.inv_cell_height));
    w.max_cy = min(grid.num_rows - 1, cv_ceil((double)(ref_y - grid.min_y + r) * grid.inv_cell_height));
    return w.min_cx < grid.num_cols && w.max_cx >= 0 && w.min_cy < grid.num_rows && w.max_cy >= 0;
}

// Stable sort of the n keypoints (x, y) by (cell key, index), cell key = cell_x * num_rows + cell_y (data/common.h:
// 104-109): exactly the traversal order of get_keypoints_in_cell (data/common.cc:275-309).  Called by every thread of
// the CTA.  Cell histogram (shared-memory atomics), block-wide exclusive scan, scatter with per-cell cursors (any order),
// then every cell is put back into index order by one thread (cells hold ~0.4 keypoints on average, 10 x 10 px).
// Returns n_in, the number of keypoints inside the grid; out-of-grid keypoints take the positions [n_in, n) in no
// particular order and are never visited.  On return orig[p] is the index of the keypoint at sorted position p,
// key[i] the cell key of keypoint i (cells = num_cols * num_rows when outside), and cell_start[k] the first sorted
// position whose key >= k, so the cells [min_cy, max_cy] of one grid column are ONE contiguous span; cell_start[cells + 1]
// = n.  Scratch: cell_start and cursor hold cells + 2 entries, warp_sums Threads / 32.
template <int Threads>
__device__ __forceinline__ int sort_by_cell(const plp_grid &grid, int n, const float *x, const float *y, int *key,
                                            int *cell_start, int *cursor, int *warp_sums, int *orig) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = Threads / 32;
    const int cells = grid.num_cols * grid.num_rows;
    for (int k = tid; k < cells + 2; k += Threads) cell_start[k] = 0;
    __syncthreads();
    for (int i = tid; i < n; i += Threads) {
        const float px = x[i], py = y[i];
        const int cx = cv_floor((double)(px - grid.min_x) * grid.inv_cell_width);
        const int cy = cv_floor((double)(py - grid.min_y) * grid.inv_cell_height);
        const bool in = (0 <= cx && cx < grid.num_cols && 0 <= cy && cy < grid.num_rows);
        const int k = in ? cx * grid.num_rows + cy : cells;
        key[i] = k;
        atomicAdd(&cell_start[k], 1);
    }
    __syncthreads();
    {
        const int total = cells + 1;  // keys 0 .. cells
        const int per = (total + Threads - 1) / Threads;
        const int b0 = min(total, tid * per), b1 = min(total, b0 + per);
        int sum = 0;
        for (int k = b0; k < b1; ++k) sum += cell_start[k];
        int incl = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
        }
        if (lane == 31) warp_sums[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            const int v = lane < nwarps ? warp_sums[lane] : 0;
            int sc = v;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int u = __shfl_up_sync(0xffffffffu, sc, o);
                if (lane >= o) sc += u;
            }
            if (lane < nwarps) warp_sums[lane] = sc - v;  // exclusive prefix of the warp totals
        }
        __syncthreads();
        int run = warp_sums[warp] + incl - sum;
        for (int k = b0; k < b1; ++k) {
            const int v = cell_start[k];
            cell_start[k] = run;
            cursor[k] = run;
            run += v;
        }
        if (tid == 0) cell_start[cells + 1] = n;
    }
    __syncthreads();
    for (int i = tid; i < n; i += Threads) orig[atomicAdd(&cursor[key[i]], 1)] = i;
    __syncthreads();
    for (int k = tid; k < cells; k += Threads) {
        const int b0 = cell_start[k], b1 = cell_start[k + 1];
        for (int a = b0 + 1; a < b1; ++a) {  // insertion sort of the (few) indices of one cell
            const int v = orig[a];
            int b = a - 1;
            while (b >= b0 && orig[b] > v) {
                orig[b + 1] = orig[b];
                --b;
            }
            orig[b + 1] = v;
        }
    }
    __syncthreads();
    return cell_start[cells];
}

// ---- reductions of (distance, position) keys over groups of Width lanes (every lane of the warp calls them)

// smallest key: the reference's "first strictly smaller distance wins" when position is the traversal order
template <int Width, class K>
__device__ __forceinline__ K warp_min(K k) {
#pragma unroll
    for (int o = Width / 2; o > 0; o >>= 1) {
        const K other = __shfl_xor_sync(0xffffffffu, k, o);
        k = other < k ? other : k;
    }
    return k;
}

// two smallest keys (k1 <= k2) of the group, from each lane's own two smallest
template <int Width, class K>
__device__ __forceinline__ void warp_top2(K &k1, K &k2) {
#pragma unroll
    for (int o = Width / 2; o > 0; o >>= 1) {
        const K o1 = __shfl_xor_sync(0xffffffffu, k1, o);
        const K o2 = __shfl_xor_sync(0xffffffffu, k2, o);
        const K lo = k1 < o1 ? k1 : o1, hi = k1 < o1 ? o1 : k1;
        const K s2 = k2 < o2 ? k2 : o2;
        k1 = lo;
        k2 = hi < s2 ? hi : s2;
    }
}

// ---- camera/perspective.cc:190-209 with the pose [R | t] as a 3 x 4 row-major Rt.  A point behind the camera leaves
// (u, v) = (0, 0) (the reference leaves them unset).
struct Reproj {
    double u, v;
    float x_right;
    bool in_image;
    bool in_front;
};

__device__ __forceinline__ Reproj reproject(const plp_camera &cam, const double *Rt, const double *X) {
    Reproj r;
    const double pc0 = Rt[0] * X[0] + Rt[1] * X[1] + Rt[2] * X[2] + Rt[3];
    const double pc1 = Rt[4] * X[0] + Rt[5] * X[1] + Rt[6] * X[2] + Rt[7];
    const double pc2 = Rt[8] * X[0] + Rt[9] * X[1] + Rt[10] * X[2] + Rt[11];
    r.u = 0.0;
    r.v = 0.0;
    r.x_right = 0.0f;
    r.in_image = false;
    r.in_front = pc2 > 0.0;
    if (!r.in_front) return r;
    const double z_inv = 1.0 / pc2;
    r.u = cam.fx * pc0 * z_inv + cam.cx;
    r.v = cam.fy * pc1 * z_inv + cam.cy;
    r.x_right = (float)(r.u - cam.focal_x_baseline * z_inv);
    r.in_image = (cam.min_x < r.u && r.u < cam.max_x && cam.min_y < r.v && r.v < cam.max_y);
    return r;
}

}  // namespace plp
