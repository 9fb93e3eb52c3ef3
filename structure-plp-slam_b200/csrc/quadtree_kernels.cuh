// quadtree_kernels.cuh -- device code of the ORB keypoint quadtree (orb.cu launches it): one CTA per (level, frame) runs
// the array formulation of distribute_keypoints_via_tree (orb_extractor.cc:468-685, tools/quadtree_parallel_model.py)
// over the FAST candidates of its level.  Free of host-side CUDA runtime dependencies so that tests/cta_emu can compile
// the same text for the host.
#pragma once
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#include "devmath.cuh"

namespace plp {

namespace {

constexpr int kPatchRadius = 19;  // orb_extractor.h:161 orb_patch_radius_
constexpr int kCellCap = 1024;    // max NMS survivors of a 64x64 tested area (FAST cell buffer stride)
constexpr int kQtMaxLevels = 16;

// Two instances: <1024 nodes, 2048 candidates in shared memory, 256 threads, 3 CTAs per SM> serves every configuration
// whose levels need at most 1024 nodes (max_num_keypts up to 1171 at scale 1.2); <2048, 8192, 512 threads, 1 CTA per SM>
// serves the rest.  A level with more candidates than the shared-memory window works in its global scratch block (the
// window of the small instance holds every level of 640 x 480 frames at 1000 keypoints: at most ~1600 candidates).
constexpr int kNodeCapSmall = 1024, kCandCapSmall = 2048, kQtThreadsSmall = 256, kQtMinBlocksSmall = 3;
constexpr int kNodeCap = 2048, kCandCapLarge = 8192, kQtThreadsLarge = 512, kQtMinBlocksLarge = 1;
constexpr int kQtScratchCands = 65536;   // candidates of one (frame, level) in the global scratch block
constexpr int kQtCandBytes = 4 + 2 * 5 + 1;  // cand + perm[2] + owner[2] + rank + cls

struct LevelKp {  // quadtree output, level coordinates (border already added)
    short x, y;
    int response;
};

struct QtLevel {
    int w, h;
    int cell_base, num_cells;  // this level's cells in the per-frame cell list
    int budget;                // num_keypts_per_level_
    int slot_base, slot_cap;   // output slots of this level (per-level keypoint lists)
};

struct QtJob {
    int num_levels;
    int num_cells;    // per frame
    int total_slots;  // per frame
    QtLevel lv[kQtMaxLevels];
    const uint32_t *cell_buf;  // batch x num_cells x kCellCap packed (x:11 | y:10 | score:8)
    const int *cell_cnt;       // batch x num_cells
    LevelKp *lvl_kp;           // batch x total_slots
    int *lvl_cnt;              // batch x num_levels
    uint8_t *scratch;          // global fallback work area, batch x num_levels blocks of scratch_per_job bytes
    size_t scratch_per_job;
    int *status;               // batch: 1 = more than 65535 candidates (clipped), 3 = output slot overflow
};

__host__ __device__ constexpr size_t qt_scratch_bytes_per_job() { return (size_t)kQtScratchCands * kQtCandBytes + 256; }

struct QtArrays {
    uint32_t *cand;             // packed candidates in gather order
    unsigned short *perm[2];    // permutation (indices into cand), ping-pong
    unsigned short *owner[2];   // list position of the node owning each perm slot, ping-pong
};

__device__ __forceinline__ int cand_x(uint32_t c) { return (int)(c & 0x7ff); }
__device__ __forceinline__ int cand_y(uint32_t c) { return (int)((c >> 11) & 0x3ff); }
__device__ __forceinline__ int cand_score(uint32_t c) { return (int)(c >> 21); }

// [i0, i1): the contiguous share of thread threadIdx.x of n items split over T threads
template <int T>
__device__ __forceinline__ void qt_chunk(int n, int &i0, int &i1) {
    const int per = (n + T - 1) / T;
    i0 = min(n, (int)threadIdx.x * per);
    i1 = min(n, i0 + per);
}

// Block-wide exclusive scan of one value per thread: shuffles inside each warp, then every thread folds the T/32 warp
// totals itself (one barrier).  `wbuf` holds T/32 entries; the caller guarantees a barrier between the last reads of
// `wbuf` by the previous scan on it and this call (QtScan alternates two buffers for that).
template <int T, class V>
__device__ __forceinline__ V qt_block_scan(V v, V *wbuf, V *total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    V incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const V t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) wbuf[warp] = incl;
    __syncthreads();
    V pre = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < T / 32; ++w) {
        const V s = wbuf[w];
        if (w < warp) pre += s;
        tot += s;
    }
    *total = tot;
    return pre + incl - v;
}

// child class of a keypoint inside node rect (orb_extractor_node.cc:67-78)
__device__ __forceinline__ int classify(const short4 r, uint32_t c) {
    const unsigned half_x = (unsigned)cv_ceil((r.z - r.x) / 2.0);
    const unsigned half_y = (unsigned)cv_ceil((r.w - r.y) / 2.0);
    int q = 0;
    if ((float)((unsigned)r.x + half_x) <= (float)cand_x(c)) q += 1;
    if ((float)((unsigned)r.y + half_y) <= (float)cand_y(c)) q += 2;
    return q;
}

__device__ __forceinline__ short4 child_rect(const short4 r, int q) {
    const int half_x = cv_ceil((r.z - r.x) / 2.0), half_y = cv_ceil((r.w - r.y) / 2.0);
    short4 c;
    c.x = (q & 1) ? (short)(r.x + half_x) : r.x;
    c.z = (q & 1) ? r.z : (short)(r.x + half_x);
    c.y = (q & 2) ? (short)(r.y + half_y) : r.y;
    c.w = (q & 2) ? r.w : (short)(r.y + half_y);
    return c;
}

// NC = node capacity (>= 4 * budget + 8 of every level the kernel instance serves), T = threads per CTA
template <int NC, int T>
struct QtSharedT {
    short4 rect[2][NC];  // node lists, struct of arrays in list order, ping-pong
    unsigned short start[2][NC];  // segment start in perm
    unsigned short cnt[2][NC];
    uint8_t leaf[2][NC];
    uint8_t sel[NC];              // node is divided in this sweep
    unsigned short newpos[NC];    // new list position of a kept node / of the front-most child of a divided one
    unsigned short pool[NC];      // children with more than one keypoint, creation order
    unsigned short proc[NC];      // phase 2: the pool in processing order
    union {
        unsigned short tot[NC * 4];  // per divided node: keypoints of each child class
        int cell_pre[NC * 2];        // gather: exclusive prefix of the level's cell counts
    } u;
    unsigned long long wsum[2][T / 32];  // warp totals of qt_block_scan
    unsigned long long seg_tail[T / 32];  // warp aggregates of the segmented class scan
    int seg_head[T / 32];
    int misc[4];
};

// the two warp-total buffers of qt_block_scan (`stride` entries apart), used in turn
struct QtScan {
    unsigned long long *buf;
    int stride, next;
    __device__ unsigned long long *get() {
        unsigned long long *b = buf + next * stride;
        next ^= 1;
        return b;
    }
};

template <int T>
__device__ __forceinline__ int qt_block_scan_int(int v, QtScan &sc, int *total) {
    unsigned long long t;
    const unsigned long long pre = qt_block_scan<T, unsigned long long>((unsigned long long)v, sc.get(), &t);
    *total = (int)t;
    return (int)pre;
}

// Segmented scan of per-element class counters.  For every perm slot i whose node is selected (sel[owner]), computes
// cls[i] (child class), rank[i] = number of earlier slots of the same node with the same class, and per node the four
// class totals tot[node*4 + q].  Each thread walks a contiguous chunk; the carries between chunks (16-bit counters of the
// four classes packed into 64 bits, reset at segment heads) come from a segmented shuffle scan per warp and a fold over
// the warp aggregates.
template <int NC, int T>
__device__ __forceinline__ void segmented_class_scan(QtSharedT<NC, T> &S, const QtArrays &A, int cur, int n, int cur_n,
                                     unsigned short *rank, uint8_t *cls) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int i0, i1;
    qt_chunk<T>(n, i0, i1);
    const unsigned short *perm = A.perm[cur], *owner = A.owner[cur];
    const short4 *rect = S.rect[cur_n];
    // pass 1: local tail since the last segment head in this chunk.  The first element of a chunk starts a new segment
    // iff its owner differs from the previous slot's owner, hence prev_owner starts from owner[i0-1].
    unsigned long long acc = 0;
    int head = 0;
    int prev_owner = (i0 > 0 && i0 < n) ? owner[i0 - 1] : -1;
    for (int i = i0; i < i1; ++i) {
        const int o = owner[i];
        if (o != prev_owner) {
            head = 1;
            acc = 0;
        }
        prev_owner = o;
        int q = 0;
        if (S.sel[o]) {
            q = classify(rect[o], A.cand[perm[i]]);
            acc += 1ull << (16 * q);
        }
        cls[i] = (uint8_t)q;
    }
    // pass 2: carry-in of every chunk = segmented exclusive scan of the (tail, head) pairs in thread order
    unsigned long long v = acc;
    int f = head;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long pv = __shfl_up_sync(0xffffffffu, v, o);
        const int pf = __shfl_up_sync(0xffffffffu, f, o);
        if (lane >= o) {
            if (!f) v += pv;
            f |= pf;
        }
    }
    if (lane == 31) {
        S.seg_tail[warp] = v;
        S.seg_head[warp] = f;
    }
    unsigned long long ev = __shfl_up_sync(0xffffffffu, v, 1);
    int ef = __shfl_up_sync(0xffffffffu, f, 1);
    if (lane == 0) {
        ev = 0;
        ef = 0;
    }
    __syncthreads();
    unsigned long long carry = 0;
    for (int w = 0; w < warp; ++w) carry = S.seg_head[w] ? S.seg_tail[w] : carry + S.seg_tail[w];
    acc = ef ? ev : carry + ev;
    // pass 3: ranks and node totals
    prev_owner = (i0 > 0 && i0 < n) ? owner[i0 - 1] : -1;
    for (int i = i0; i < i1; ++i) {
        const int o = owner[i];
        if (o != prev_owner) acc = 0;
        prev_owner = o;
        if (S.sel[o]) {
            const int q = cls[i];
            rank[i] = (unsigned short)((acc >> (16 * q)) & 0xffff);
            acc += 1ull << (16 * q);
            const bool last = (i + 1 == n) || (owner[i + 1] != o);
            if (last) {
                unsigned short *t = S.u.tot + o * 4;
                t[0] = (unsigned short)(acc & 0xffff);
                t[1] = (unsigned short)((acc >> 16) & 0xffff);
                t[2] = (unsigned short)((acc >> 32) & 0xffff);
                t[3] = (unsigned short)((acc >> 48) & 0xffff);
            }
        }
    }
    __syncthreads();
}

// children of a divided node, and the children with more than one keypoint (pool entries), packed as
// bits 0-15 | bits 16-31
__device__ __forceinline__ unsigned long long qt_child_counts(const unsigned short *t) {
    const int nch = (t[0] > 0) + (t[1] > 0) + (t[2] > 0) + (t[3] > 0);
    const int npool = (t[0] > 1) + (t[1] > 1) + (t[2] > 1) + (t[3] > 1);
    return (unsigned long long)nch | ((unsigned long long)npool << 16);
}

// Divides the nodes with sel[p] != 0 of list `cur_n` (length len) and returns the new list length.  The new list holds
// the children of the divided nodes in front (later-divided first, classes reversed: orb_extractor.cc:639-657 pushes to
// the front), then the kept nodes in list order; the keypoints of each divided node are stably partitioned by class; the
// pool becomes the children with more than one keypoint in creation order (division order, classes ascending).
// Division order: `proc[0..num_proc)` when proc != nullptr (phase 2), else the selected nodes in list order (phase 1).
// One packed scan gives every output position: children (bits 0-15) and pool entries (16-31) over the division order,
// kept nodes (32-47) over the list.  Every total is below NC <= 2048 (the list before a sweep is shorter than the budget).
template <int NC, int T>
__device__ __forceinline__ int divide_nodes(QtSharedT<NC, T> &S, QtArrays &A, int &cur, int n_cand, int &cur_n, int len,
                            const unsigned short *proc, int num_proc, const unsigned short *rank, const uint8_t *cls,
                            int *pool_len_out, QtScan &sc) {
    const int tid = threadIdx.x;
    const int nxt_n = cur_n ^ 1;
    int p0, p1, k0, k1;
    qt_chunk<T>(len, p0, p1);
    if (proc) {
        qt_chunk<T>(num_proc, k0, k1);
    } else {
        k0 = p0;
        k1 = p1;
    }
    unsigned long long local = 0;
    for (int k = k0; k < k1; ++k) {
        const int p = proc ? proc[k] : k;
        if (proc || S.sel[p]) local += qt_child_counts(S.u.tot + p * 4);
    }
    for (int p = p0; p < p1; ++p)
        if (!S.sel[p]) local += 1ull << 32;
    unsigned long long total;
    const unsigned long long pre = qt_block_scan<T, unsigned long long>(local, sc.get(), &total);
    const int total_children = (int)(total & 0xffff), pool_len = (int)((total >> 16) & 0xffff);
    const int new_len = total_children + (int)(total >> 32);
    int cpre = (int)(pre & 0xffff), ppre = (int)((pre >> 16) & 0xffff), kpre = (int)(pre >> 32);
    // children: the divided node with cpre children before it (in division order) puts its own children at list
    // positions [total_children - cpre - nch, total_children - cpre), class order reversed
    for (int k = k0; k < k1; ++k) {
        const int p = proc ? proc[k] : k;
        if (!proc && !S.sel[p]) continue;
        const unsigned short *t = S.u.tot + p * 4;
        const int nch = (t[0] > 0) + (t[1] > 0) + (t[2] > 0) + (t[3] > 0);
        const int base = total_children - cpre - nch;
        const short4 r = S.rect[cur_n][p];
        int o = S.start[cur_n][p];
        int rnk = 0;
        for (int q = 0; q < 4; ++q) {
            if (t[q] == 0) continue;
            const int pos = base + (nch - 1 - rnk);
            S.rect[nxt_n][pos] = child_rect(r, q);
            S.start[nxt_n][pos] = (unsigned short)o;
            S.cnt[nxt_n][pos] = t[q];
            S.leaf[nxt_n][pos] = 0;
            if (t[q] > 1) S.pool[ppre++] = (unsigned short)pos;
            o += t[q];
            ++rnk;
        }
        S.newpos[p] = (unsigned short)base;  // class q child = base + (nch-1-rank_q)
        cpre += nch;
    }
    // kept nodes: positions after all children, in list order
    for (int p = p0; p < p1; ++p) {
        if (S.sel[p]) continue;
        const int pos = total_children + kpre++;
        S.rect[nxt_n][pos] = S.rect[cur_n][p];
        S.start[nxt_n][pos] = S.start[cur_n][p];
        S.cnt[nxt_n][pos] = S.cnt[cur_n][p];
        S.leaf[nxt_n][pos] = S.leaf[cur_n][p];
        S.newpos[p] = (unsigned short)pos;
    }
    __syncthreads();
    // keypoints: stable 4-way partition inside each divided node, owner update for everybody
    {
        const unsigned short *perm = A.perm[cur], *owner = A.owner[cur];
        unsigned short *perm2 = A.perm[cur ^ 1], *owner2 = A.owner[cur ^ 1];
        for (int i = tid; i < n_cand; i += T) {
            const int o = owner[i];
            if (S.sel[o]) {
                const unsigned short *t = S.u.tot + o * 4;
                const int q = cls[i];
                int off = 0, rnk = 0;
                for (int c = 0; c < q; ++c) {
                    off += t[c];
                    rnk += (t[c] > 0);
                }
                const int nch = (t[0] > 0) + (t[1] > 0) + (t[2] > 0) + (t[3] > 0);
                const int dst = S.start[cur_n][o] + off + rank[i];
                perm2[dst] = perm[i];
                owner2[dst] = (unsigned short)(S.newpos[o] + (nch - 1 - rnk));
            } else {
                perm2[i] = perm[i];
                owner2[i] = S.newpos[o];
            }
        }
    }
    __syncthreads();
    *pool_len_out = pool_len;
    cur ^= 1;
    cur_n = nxt_n;
    return new_len;
}

// One CTA per (level, frame): gather the level's candidates in cell order, initial nodes, phase 1 (whole-list sweeps),
// phase 2 (densest pool nodes first), the best keypoint of every node.
template <int NC, int CC, int T, int kMinBlocks>
__global__ void __launch_bounds__(T, kMinBlocks) quadtree_kernel(QtJob P) {
    PLP_DYNAMIC_SMEM(qsmem);
    using QtShared = QtSharedT<NC, T>;
    QtShared &S = *reinterpret_cast<QtShared *>(qsmem);
    const int l = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    const QtLevel &LV = P.lv[l];
    int *lvl_cnt = P.lvl_cnt + (size_t)b * P.num_levels + l;
    LevelKp *out = P.lvl_kp + (size_t)b * P.total_slots + LV.slot_base;
    QtScan sc{S.wsum[0], T / 32, 0};

    // ---- gather candidates of this level in cell order: exclusive prefix of the cell counts, then every candidate slot
    // finds its cell by binary search in the prefix (independent loads, several in flight per thread)
    const int *cc = P.cell_cnt + (size_t)b * P.num_cells + LV.cell_base;
    const int num_cells = LV.num_cells;
    int *cpre = S.u.cell_pre;
    int n;
    {
        int c0, c1;
        qt_chunk<T>(num_cells, c0, c1);
        int sum = 0;
        for (int c = c0; c < c1; ++c) {
            cpre[c] = cc[c];
            sum += cpre[c];
        }
        int run = qt_block_scan_int<T>(sum, sc, &n);
        for (int c = c0; c < c1; ++c) {
            const int k = cpre[c];
            cpre[c] = run;
            run += k;
        }
        if (tid == 0) cpre[num_cells] = n;
        __syncthreads();
    }
    if (n == 0) {
        if (tid == 0) *lvl_cnt = 0;
        return;
    }
    if (n > 65535) {
        n = 65535;
        if (tid == 0) P.status[b] = 1;
    }
    // work arrays: shared memory when they fit, else the global scratch block of this (frame, level)
    QtArrays A;
    unsigned short *rank;
    uint8_t *cls;
    {
        uint8_t *base;
        if (n <= CC) {
            base = qsmem + ((sizeof(QtShared) + 15) & ~(size_t)15);
        } else {
            base = P.scratch + ((size_t)b * P.num_levels + l) * P.scratch_per_job;
        }
        const size_t cap = n <= CC ? CC : kQtScratchCands;
        A.cand = reinterpret_cast<uint32_t *>(base);
        base += cap * 4;
        A.perm[0] = reinterpret_cast<unsigned short *>(base);
        base += cap * 2;
        A.perm[1] = reinterpret_cast<unsigned short *>(base);
        base += cap * 2;
        A.owner[0] = reinterpret_cast<unsigned short *>(base);
        base += cap * 2;
        A.owner[1] = reinterpret_cast<unsigned short *>(base);
        base += cap * 2;
        rank = reinterpret_cast<unsigned short *>(base);
        base += cap * 2;
        cls = base;
    }
    {
        constexpr int kBatch = 4;
        const uint32_t *cb = P.cell_buf + ((size_t)b * P.num_cells + LV.cell_base) * kCellCap;
        for (int i0 = tid; i0 < n; i0 += kBatch * T) {
            uint32_t v[kBatch];
#pragma unroll
            for (int j = 0; j < kBatch; ++j) {
                const int i = i0 + j * T;
                if (i < n) {
                    int lo = 0, hi = num_cells;  // cpre[lo] <= i < cpre[hi]
                    while (hi - lo > 1) {
                        const int mid = (lo + hi) >> 1;
                        if (cpre[mid] <= i) lo = mid;
                        else hi = mid;
                    }
                    v[j] = __ldg(cb + (size_t)lo * kCellCap + (i - cpre[lo]));
                }
            }
#pragma unroll
            for (int j = 0; j < kBatch; ++j)
                if (i0 + j * T < n) A.cand[i0 + j * T] = v[j];
        }
    }
    __syncthreads();

    // ---- initialize_nodes (orb_extractor.cc:557-637)
    const int min_x = kPatchRadius, max_x = LV.w - kPatchRadius, min_y = kPatchRadius, max_y = LV.h - kPatchRadius;
    const double ratio = (double)(max_x - min_x) / (max_y - min_y);
    int gx, gy;
    double dx, dy;
    if (ratio > 1) {
        gx = (int)round(ratio);
        gy = 1;
        dx = (double)(max_x - min_x) / gx;
        dy = max_y - min_y;
    } else {
        gx = 1;
        gy = (int)round(1 / ratio);
        dx = max_x - min_y;  // sic, orb_extractor.cc:580
        dy = (double)(max_y - min_y) / gy;
    }
    const int g = gx * gy;  // number of initial nodes (small)
    int cur = 0, cur_n = 0, len = 0;
    {
        // stable counting sort of the candidates by initial node; S.proc maps initial node -> list position and
        // S.newpos holds its segment start until phase 2
        int *cnts = S.u.cell_pre;  // g entries
        for (int i = tid; i < g; i += T) cnts[i] = 0;
        __syncthreads();
        for (int i = tid; i < n; i += T) {
            const uint32_t c = A.cand[i];
            const unsigned ix = (unsigned)((float)cand_x(c) / dx), iy = (unsigned)((float)cand_y(c) / dy);
            int node = (int)(ix + iy * gx);
            node = min(node, g - 1);
            A.owner[0][i] = (unsigned short)node;  // temporarily the initial node index
            atomicAdd(&cnts[node], 1);
        }
        __syncthreads();
        // node offsets + list (thread 0; g is tiny)
        if (tid == 0) {
            int off = 0, pos = 0;
            for (int i = 0; i < g; ++i) {
                const int c = cnts[i];
                S.newpos[i] = (unsigned short)off;
                if (c > 0) {
                    const int ix = i % gx, iy = i / gx;
                    short4 r;
                    r.x = (short)(int)(dx * ix);
                    r.y = (short)(int)(dy * iy);
                    r.z = (short)(int)(dx * (ix + 1));
                    r.w = (short)(int)(dy * (iy + 1));
                    S.rect[0][pos] = r;
                    S.start[0][pos] = (unsigned short)off;
                    S.cnt[0][pos] = (unsigned short)c;
                    S.leaf[0][pos] = (c == 1);
                    S.proc[i] = (unsigned short)pos;
                    ++pos;
                }
                off += c;
            }
            S.misc[0] = pos;
        }
        __syncthreads();
        len = S.misc[0];
        // stable placement: rank of element i inside its initial node = #earlier elements of the same node.
        // g is tiny, so do one ordered pass per initial node with a block scan of flags.
        int i0, i1;
        qt_chunk<T>(n, i0, i1);
        for (int node = 0; node < g; ++node) {
            if (cnts[node] == 0) continue;
            int c = 0;
            for (int i = i0; i < i1; ++i) c += (A.owner[0][i] == node);
            int tot;
            int run = qt_block_scan_int<T>(c, sc, &tot);
            const int base = S.newpos[node];
            const unsigned short lp = S.proc[node];
            for (int i = i0; i < i1; ++i)
                if (A.owner[0][i] == node) {
                    A.perm[1][base + run] = (unsigned short)i;
                    A.owner[1][base + run] = lp;
                    ++run;
                }
        }
        __syncthreads();
        cur = 1;
    }
    const int budget = LV.budget;
    int pool_len = 0;
    bool filled = false;

    // ---- phase 1 (orb_extractor.cc:482-518): every non-leaf node is divided, in list order
    while (true) {
        const int prev = len;
        for (int p = tid; p < len; p += T) S.sel[p] = S.leaf[cur_n][p] ? 0 : 1;
        __syncthreads();
        segmented_class_scan(S, A, cur, n, cur_n, rank, cls);
        len = divide_nodes(S, A, cur, n, cur_n, len, (const unsigned short *)nullptr, 0, rank, cls, &pool_len, sc);
        if (budget <= len || len == prev) {
            filled = true;
            break;
        }
        if (budget < len + pool_len) break;
    }
    // ---- phase 2 (orb_extractor.cc:520-552): the pool nodes by (cnt desc, creation desc) until the budget is reached
    while (!filled) {
        const int prev = len;
        for (int p = tid; p < len; p += T) S.sel[p] = 0;
        if (tid == 0) S.misc[1] = pool_len + 1;
        __syncthreads();
        for (int k = tid; k < pool_len; k += T) {
            S.sel[S.pool[k]] = 1;
            S.newpos[k] = S.cnt[cur_n][S.pool[k]];  // pool counts for the rank sort
        }
        __syncthreads();
        segmented_class_scan(S, A, cur, n, cur_n, rank, cls);
        // rank sort of the pool by (cnt desc, creation desc)
        for (int k = tid; k < pool_len; k += T) {
            const int ck = S.newpos[k];
            int r = 0;
            for (int j = 0; j < pool_len; ++j) {
                const int cj = S.newpos[j];
                r += (cj > ck) || (cj == ck && j > k);
            }
            S.proc[r] = S.pool[k];
        }
        __syncthreads();
        // cut: the first k with prev + sum_{j<=k}(nch_j - 1) >= budget ends the sweep
        int num_proc;
        bool reached;
        {
            int k0, k1;
            qt_chunk<T>(pool_len, k0, k1);
            int sum = 0;
            for (int k = k0; k < k1; ++k) sum += (int)(qt_child_counts(S.u.tot + S.proc[k] * 4) & 0xffff) - 1;
            int tot;
            int run = prev + qt_block_scan_int<T>(sum, sc, &tot);
            for (int k = k0; k < k1; ++k) {
                run += (int)(qt_child_counts(S.u.tot + S.proc[k] * 4) & 0xffff) - 1;
                if (run >= budget) {  // list size after dividing the k-th pool node
                    atomicMin(&S.misc[1], k + 1);
                    break;
                }
            }
            __syncthreads();
            reached = S.misc[1] <= pool_len;
            num_proc = reached ? S.misc[1] : pool_len;
        }
        // only the first num_proc pool nodes are divided
        for (int k = num_proc + tid; k < pool_len; k += T) S.sel[S.proc[k]] = 0;
        __syncthreads();
        len = divide_nodes(S, A, cur, n, cur_n, len, S.proc, num_proc, rank, cls, &pool_len, sc);
        if (reached) filled = true;
        if (filled || budget <= len || len == prev) break;
    }

    // ---- find_keypoints_with_max_response (orb_extractor.cc:659-685): first maximum wins
    const int n_out = min(len, LV.slot_cap);
    if (len > LV.slot_cap && tid == 0) P.status[b] = 3;
    for (int p = tid; p < n_out; p += T) {
        const int st = S.start[cur_n][p], c = S.cnt[cur_n][p];
        uint32_t best = A.cand[A.perm[cur][st]];
        for (int k = 1; k < c; ++k) {
            const uint32_t v = A.cand[A.perm[cur][st + k]];
            if (cand_score(v) > cand_score(best)) best = v;
        }
        LevelKp kp;
        kp.x = (short)(cand_x(best) + kPatchRadius);  // orb_extractor.cc:450-454
        kp.y = (short)(cand_y(best) + kPatchRadius);
        kp.response = cand_score(best);
        out[p] = kp;
    }
    if (tid == 0) *lvl_cnt = n_out;
}

// dynamic shared memory of an instance: the node arrays, then the candidate window
template <int NC, int CC, int T>
__host__ __device__ constexpr size_t qt_smem_bytes() {
    return ((sizeof(QtSharedT<NC, T>) + 15) & ~(size_t)15) + (size_t)CC * kQtCandBytes + 64;
}

}  // namespace

}  // namespace plp
