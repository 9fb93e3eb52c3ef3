// lsd_grow_kernels.cuh -- device code of LSD region growing (lsd.cpp region_grow / region2rect / refine /
// reduce_region_radius as OpenCV's LineSegmentDetector runs them, options of feature/line_extractor.cc:113-122): the
// one-warp-per-frame kernel, the multi-warp round protocol and the out-of-order variant (see lines.cu for the rest of the
// line front end).  Free of host-side CUDA runtime dependencies so that tests/cta_emu can compile the same text for the
// host (one host thread per CUDA thread) and compare all three variants with the oracle on the CPU.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>

#include "detmath.h"
#include "devmath.cuh"

namespace plp {
namespace lsd {

constexpr unsigned kFull = 0xffffffffu;
constexpr double kDegToRads = 0.017453292519943295769236907684;
constexpr double kPi = 3.14159265358979323846;
constexpr double k3_2Pi = 4.71238898038;  // literals of lsd.cpp
constexpr double k2Pi = 6.28318530718;
constexpr int kBins = 1024;
constexpr int kSortWarps = 32;
constexpr int kBands = 9, kBandWidth = 7, kLspHeight = kBands * kBandWidth;

struct LineDev {
    int w, h;          // full resolution
    int sw, sh, npx;   // half resolution LSD works on
    int seg_cap, kl_cap;
    int min_reg_size;
    double rho, prec, p, density_th, min_length;
    // per batch buffers (frame-major)
    const uint8_t *img;
    size_t img_step, img_frame_stride;
    uint8_t *scaled;     // npx
    const float4 *cstab; // (2*510+1)^2 x {deg, cos, sin} by (gx, gy), shared by all frames
    int kthr;            // level-line angle defined  <=>  gx^2+gy^2 > kthr  (norm > rho)
    uint32_t *order;     // npx packed (y<<16|x) seeds, bin desc / raster asc
    int *nseeds;
    uint32_t *reg_xy;    // npx: region entries beyond the shared-memory window
    int reg_cap_small;   // region window (entries) of lsd_grow_kernel<false>: kRegCapSmall
    unsigned long long *mw_stat;  // per frame {rounds, seeds run, seeds redone} of lsd_grow_mw_kernel (may be null)
    float4 *segs;        // seg_cap
    int *nseg;
    short2 *grad;        // w*h Sobel (dx, dy) of the 5x5-blurred frame
    float *lbd_float;    // kl_cap x 72
    int *status;
    float gauss_l[kBandWidth * 3];
    float gauss_g[kLspHeight];
};

// cv::fastAtan2 (degrees), f32 without FMA (SURVEY Appendix A.7)
__device__ __forceinline__ float fast_atan2_deg(float y, float x) {
    const float scale = (float)(180.0 / 3.14159265358979323846);
    const float p1 = 0.9997878412794807f * scale, p3 = -0.3258083974640975f * scale, p5 = 0.1555786518463281f * scale,
                p7 = -0.04432655554792128f * scale;
    const float ax = fabsf(x), ay = fabsf(y);
    // branch-free form of `if (ax >= ay) c = ay / (ax + eps) else c = ax / (ay + eps)`: one division for all lanes
    const bool steep = !(ax >= ay);
    const float mn = steep ? ax : ay, mx = steep ? ay : ax;
    const float c = mn / (mx + 2.220446049250313e-16f);
    const float c2 = c * c;
    float a = (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
    if (steep) a = 90.f - a;
    if (x < 0) a = 180.f - a;
    if (y < 0) a = 360.f - a;
    return a;
}

__device__ __forceinline__ void grad_at(const uint8_t *img, int sw, int idx, int &gx, int &gy) {
    const int a = img[idx], bq = img[idx + 1], c = img[idx + sw], d = img[idx + sw + 1];
    const int DA = d - a, BC = bq - c;
    gx = DA + BC;
    gy = DA - BC;
}

constexpr int kGRange = 510, kGDim = 2 * kGRange + 1;

// ------------------------------------------------------------------------------------------------------------------
// K4: region growing + rectangle + refinement: one warp per frame; half-resolution image, `used` bitmap and the region
//     list (= BFS queue) in shared memory.
// ------------------------------------------------------------------------------------------------------------------
constexpr int kRegCap = 6144;       // region entries kept in shared memory; longer regions spill to global memory
constexpr int kRegCapSmall = 2048;  // ... in the many-frames-per-SM variant

struct Rect {
    double x1, y1, x2, y2, width;
};

// kMw = false: one warp per frame, marks go straight into the frame's `used` bitmap.
// kMw = true (lsd_grow_mw_kernel): several warps of a CTA work on seeds of the SAME frame speculatively: `used` is the
// committed bitmap (read only while the warps grow), the warp's own marks live in its private bitmap `mark`, and the
// bounding box of every pixel the warp ever accepted is tracked for the conflict test.
template <bool kMw>
struct GrowT {  // per-warp state
    int sw, sh, kthr;
    double density_th;
    const uint8_t *img;    // shared: half-resolution image
    uint32_t *used;        // shared: bitmap (kMw: committed marks of the frame)
    uint32_t *mark;        // shared: where this warp sets / clears marks (= used unless kMw)
    uint32_t *reg;         // shared: first reg_cap region entries (packed y<<16|x)
    uint32_t *reg_ovf;     // global: all entries beyond reg_cap (indexed by absolute position)
    const float4 *tab;     // global: {deg, cos, sin} by (gx, gy)
    int lane, reg_cap;
    mutable int bx0, by0, bx1, by1;  // kMw: per-lane bounding box of the pixels this lane accepted (reduced by the caller)
    // out-of-order kernel only (claim == nullptr otherwise): `claim` = union of the private marks of every context in flight;
    // a region that is about to accept a pixel claimed by an EARLIER ticket stops at once (`aborted`) and is decided at the head
    uint32_t *claim;
    const uint32_t *priv_base;   // the contexts' private bitmaps, `ctx_words` words apart
    const int *ctx_ticket;       // ticket each context is working on (INT_MAX: idle)
    int nctx, self, my_ticket, ctx_words;
    mutable bool aborted;
    __device__ __forceinline__ uint32_t get(int e) const { return e < reg_cap ? reg[e] : reg_ovf[e]; }
    __device__ __forceinline__ void put(int e, uint32_t v) const {
        if (e < reg_cap) reg[e] = v;
        else reg_ovf[e] = v;
    }
    __device__ __forceinline__ bool is_used(int idx) const {
        uint32_t w = used[idx >> 5];
        if (kMw) w |= mark[idx >> 5];
        return (w >> (idx & 31)) & 1u;
    }
    __device__ __forceinline__ bool claimed_by_earlier(int idx) const {
        if (!kMw || !claim || !((claim[idx >> 5] >> (idx & 31)) & 1u)) return false;
        bool earlier = false;
        for (int w = 0; w < nctx; ++w)
            if (w != self && ((priv_base[(size_t)w * ctx_words + (idx >> 5)] >> (idx & 31)) & 1u))
                earlier = earlier || *reinterpret_cast<const volatile int *>(&ctx_ticket[w]) < my_ticket;
        return earlier;
    }
    __device__ __forceinline__ void unclaim(int idx) const {
        if (kMw && claim) atomicAnd(&claim[idx >> 5], ~(1u << (idx & 31)));
    }
    __device__ __forceinline__ void accept(int idx, uint32_t xy) const {  // one lane: mark a pixel of the region
        mark[idx >> 5] |= 1u << (idx & 31);
        if (kMw && claim) atomicOr(&claim[idx >> 5], 1u << (idx & 31));
        if (kMw) {
            const int x = (int)(xy & 0xffff), y = (int)(xy >> 16);
            bx0 = min(bx0, x);
            bx1 = max(bx1, x);
            by0 = min(by0, y);
            by1 = max(by1, y);
        }
    }
};
using Grow = GrowT<false>;

__device__ __forceinline__ bool is_aligned(double a, double theta, double prec) {
    double n_theta = theta - a;
    if (n_theta < 0) n_theta = -n_theta;
    if (n_theta > k3_2Pi) {
        n_theta -= k2Pi;
        if (n_theta < 0) n_theta = -n_theta;
    }
    return n_theta <= prec;
}

__device__ __forceinline__ double warp_sum_tree(double p) {
    for (int off = 16; off >= 1; off >>= 1) p = p + __shfl_xor_sync(kFull, p, off);
    return p;
}
__device__ __forceinline__ double warp_max(double p) {
    for (int off = 16; off >= 1; off >>= 1) p = fmax(p, __shfl_xor_sync(kFull, p, off));
    return p;
}
__device__ __forceinline__ double warp_min(double p) {
    for (int off = 16; off >= 1; off >>= 1) p = fmin(p, __shfl_xor_sync(kFull, p, off));
    return p;
}

// immutable data of one neighbour pixel (does not depend on the `used` map)
struct Nb {
    int nidx;     // -1: outside / no gradient defined
    uint32_t xy;
    float4 t;     // {deg, cos, sin}
};

// neighbour jj (0..7, centre skipped) of queue entry e
template <bool kMw>
__device__ __forceinline__ Nb load_nb(const GrowT<kMw> &G, int e, int ddx, int ddy) {
    Nb r;
    r.nidx = -1;
    r.xy = 0;
    r.t = make_float4(0.f, 0.f, 0.f, 0.f);
    const uint32_t pxy = G.get(e);
    const int nx = (int)(pxy & 0xffff) + ddx, ny = (int)(pxy >> 16) + ddy;
    // the last row / column carry no gradient (NOTDEF)
    if (nx >= 0 && nx < G.sw - 1 && ny >= 0 && ny < G.sh - 1) {
        const int idx = ny * G.sw + nx;
        int gx, gy;
        grad_at(G.img, G.sw, idx, gx, gy);
        if (gx * gx + gy * gy > G.kthr) {
            r.nidx = idx;
            r.xy = ((uint32_t)ny << 16) | (uint32_t)nx;
            r.t = G.tab[(gy + kGRange) * kGDim + gx + kGRange];
        }
    }
    return r;
}

// lsd.cpp region_grow.  Returns the region size; the region list lives in G.reg (+ overflow).
// 32 lanes = 4 queue entries x 8 neighbours, in the scalar visiting order (entry, then yy, then xx).  The immutable data
// of the next four entries is fetched while the current four are resolved; every candidate lane keeps the region sums
// and angle it WOULD produce if it were accepted next, so an acceptance is one shuffle away.
template <bool kMw>
__device__ int region_grow(const GrowT<kMw> &G, uint32_t seed_xy, float seed_deg, double prec, double &reg_angle_out) {
    const int sw = G.sw, lane = G.lane;
    double reg_angle = (double)seed_deg * kDegToRads;
    float sumdx = (float)det_cos(reg_angle);
    float sumdy = (float)det_sin(reg_angle);
    if (lane == 0) {
        const int sidx = (int)(seed_xy >> 16) * sw + (int)(seed_xy & 0xffff);
        G.accept(sidx, seed_xy);
        G.reg[0] = seed_xy;
    }
    __syncwarp();
    int n = 1, i = 0;
    const int g = lane >> 3, jj = lane & 7;
    const int j = jj + (jj >= 4);  // skip the centre
    const int ddx = j % 3 - 1, ddy = j / 3 - 1;
    Nb cur;
    cur.nidx = -1;
    cur.xy = 0;
    cur.t = make_float4(0.f, 0.f, 0.f, 0.f);
    int loaded = 0;  // groups of `cur` that hold valid data
    while (i < n) {
        const int take = min(4, n - i);
        if (g >= loaded && g < take) cur = load_nb(G, i + g, ddx, ddy);  // entries that were not known one round ago
        // prefetch the entries already known for the next round
        const int nxt_avail = min(4, n - (i + take));
        Nb nxt;
        nxt.nidx = -1;
        nxt.xy = 0;
        nxt.t = make_float4(0.f, 0.f, 0.f, 0.f);
        if (g < nxt_avail) nxt = load_nb(G, i + take + g, ddx, ddy);
        // resolve the current entries
        bool cand = (g < take) && (cur.nidx >= 0) && !G.is_used(cur.nidx);
        const bool ce = cand && G.claimed_by_earlier(cur.nidx);  // (false unless the out-of-order kernel runs)
        const double a = (double)cur.t.x * kDegToRads;
        float my_sdx = sumdx + cur.t.y, my_sdy = sumdy + cur.t.z;
        double my_theta = (double)fast_atan2_deg(my_sdy, my_sdx) * kDegToRads;
        for (;;) {
            const bool al = cand && is_aligned(a, reg_angle, prec);
            const unsigned m = __ballot_sync(kFull, al);
            if (!m) break;
            const int l = __ffs(m) - 1;
            if (kMw && __shfl_sync(kFull, ce ? 1 : 0, l)) {  // the next pixel of the sequential order belongs to an earlier region in flight
                G.aborted = true;
                reg_angle_out = reg_angle;
                return n;
            }
            sumdx = __shfl_sync(kFull, my_sdx, l);
            sumdy = __shfl_sync(kFull, my_sdy, l);
            reg_angle = __shfl_sync(kFull, my_theta, l);
            const int q = __shfl_sync(kFull, cur.nidx, l);
            if (lane == l) {
                G.accept(cur.nidx, cur.xy);
                G.put(n, cur.xy);
            }
            ++n;
            cand = cand && (lane > l) && (cur.nidx != q);
            my_sdx = sumdx + cur.t.y;
            my_sdy = sumdy + cur.t.z;
            my_theta = (double)fast_atan2_deg(my_sdy, my_sdx) * kDegToRads;
        }
        __syncwarp();
        i += take;
        cur = nxt;
        loaded = nxt_avail;
    }
    reg_angle_out = reg_angle;
    return n;
}

__device__ __forceinline__ double angle_diff_signed(double a, double b) {
    double diff = a - b;
    while (diff <= -kPi) diff += k2Pi;
    while (diff > kPi) diff -= k2Pi;
    return diff;
}
__device__ __forceinline__ double dist2(double x1, double y1, double x2, double y2) {
    return (x2 - x1) * (x2 - x1) + (y2 - y1) * (y2 - y1);
}
// modgrad of a region pixel, recomputed from the image
template <bool kMw>
__device__ __forceinline__ double px_weight(const GrowT<kMw> &G, uint32_t xy) {
    int gx, gy;
    grad_at(G.img, G.sw, (int)(xy >> 16) * G.sw + (int)(xy & 0xffff), gx, gy);
    return sqrt((double)(gx * gx + gy * gy) / 4.0);
}

// lsd.cpp region2rect + get_theta
template <bool kMw>
__device__ void region2rect(const GrowT<kMw> &G, int n, double reg_angle, double prec, Rect &R) {
    const int lane = G.lane;
    double sx = 0, sy = 0, ss = 0;
    for (int i = lane; i < n; i += 32) {
        const uint32_t xy = G.get(i);
        const double wgt = px_weight(G, xy);
        sx += (double)(int)(xy & 0xffff) * wgt;
        sy += (double)(int)(xy >> 16) * wgt;
        ss += wgt;
    }
    sx = warp_sum_tree(sx);
    sy = warp_sum_tree(sy);
    ss = warp_sum_tree(ss);
    const double x = sx / ss, y = sy / ss;
    double ixx = 0, iyy = 0, ixy = 0;
    for (int i = lane; i < n; i += 32) {
        const uint32_t xy = G.get(i);
        const double wgt = px_weight(G, xy);
        const double dx = (double)(int)(xy & 0xffff) - x, dy = (double)(int)(xy >> 16) - y;
        ixx += dy * dy * wgt;
        iyy += dx * dx * wgt;
        ixy += dx * dy * wgt;
    }
    const double Ixx = warp_sum_tree(ixx), Iyy = warp_sum_tree(iyy), Ixy = -warp_sum_tree(ixy);
    const double lambda = 0.5 * (Ixx + Iyy - sqrt((Ixx - Iyy) * (Ixx - Iyy) + 4.0 * Ixy * Ixy));
    double theta = (fabs(Ixx) > fabs(Iyy)) ? (double)fast_atan2_deg((float)(lambda - Ixx), (float)Ixy)
                                           : (double)fast_atan2_deg((float)Ixy, (float)(lambda - Iyy));
    theta *= kDegToRads;
    if (fabs(angle_diff_signed(theta, reg_angle)) > prec) theta += kPi;
    const double dx = det_cos(theta), dy = det_sin(theta);
    double l_min = 0, l_max = 0, w_min = 0, w_max = 0;
    for (int i = lane; i < n; i += 32) {
        const uint32_t xy = G.get(i);
        const double rdx = (double)(int)(xy & 0xffff) - x, rdy = (double)(int)(xy >> 16) - y;
        const double l = rdx * dx + rdy * dy;
        const double wv = -rdx * dy + rdy * dx;
        l_max = fmax(l_max, l);
        l_min = fmin(l_min, l);
        w_max = fmax(w_max, wv);
        w_min = fmin(w_min, wv);
    }
    l_max = warp_max(l_max);
    l_min = warp_min(l_min);
    w_max = warp_max(w_max);
    w_min = warp_min(w_min);
    R.x1 = x + l_min * dx;
    R.y1 = y + l_min * dy;
    R.x2 = x + l_max * dx;
    R.y2 = y + l_max * dy;
    R.width = w_max - w_min;
    if (R.width < 1.0) R.width = 1.0;
}

__device__ __forceinline__ double rect_density(int n, const Rect &R) {
    return (double)n / (sqrt(dist2(R.x1, R.y1, R.x2, R.y2)) * R.width);
}

// lsd.cpp refine + reduce_region_radius; n is updated; returns false when the region is rejected
template <bool kMw>
__device__ bool refine(const GrowT<kMw> &G, int &n, float seed_deg, double reg_angle, double prec, Rect &R) {
    const int lane = G.lane, sw = G.sw;
    double density = rect_density(n, R);
    if (density >= G.density_th) return true;
    const uint32_t seed_xy = G.reg[0];
    const double xc = (double)(int)(seed_xy & 0xffff), yc = (double)(int)(seed_xy >> 16);
    const double ang_c = (double)seed_deg * kDegToRads;
    double sum = 0, s_sum = 0;
    int cnt = 0;
    for (int i = lane; i < n; i += 32) {
        const uint32_t xy = G.get(i);
        const int px = xy & 0xffff, py = xy >> 16;
        const int pidx = py * sw + px;
        atomicAnd(&G.mark[pidx >> 5], ~(1u << (pidx & 31)));  // NOTUSED again
        G.unclaim(pidx);
        if (sqrt(dist2(xc, yc, (double)px, (double)py)) < R.width) {
            int gx, gy;
            grad_at(G.img, sw, pidx, gx, gy);
            const double ang = (double)fast_atan2_deg((float)gx, (float)-gy) * kDegToRads;
            const double d = angle_diff_signed(ang, ang_c);
            sum += d;
            s_sum += d * d;
            ++cnt;
        }
    }
    sum = warp_sum_tree(sum);
    s_sum = warp_sum_tree(s_sum);
    for (int off = 16; off >= 1; off >>= 1) cnt += __shfl_xor_sync(kFull, cnt, off);
    const double mean_angle = sum / (double)cnt;
    const double tau = 2.0 * sqrt((s_sum - 2.0 * mean_angle * sum) / (double)cnt + mean_angle * mean_angle);
    __syncwarp();
    n = region_grow(G, seed_xy, seed_deg, tau, reg_angle);
    if (kMw && G.aborted) return false;
    if (n < 2) return false;
    region2rect(G, n, reg_angle, prec, R);
    density = rect_density(n, R);
    if (density >= G.density_th) return true;
    // reduce_region_radius
    const double r1 = dist2(xc, yc, R.x1, R.y1), r2 = dist2(xc, yc, R.x2, R.y2);
    double rad_sq = r1 > r2 ? r1 : r2;
    while (density < G.density_th) {
        rad_sq *= 0.75 * 0.75;
        int o = 0;
        for (int i0 = 0; i0 < n; i0 += 32) {
            const int i = i0 + lane;
            uint32_t xy = 0;
            bool keep = false;
            if (i < n) {
                xy = G.get(i);
                const int px = xy & 0xffff, py = xy >> 16;
                keep = !(dist2(xc, yc, (double)px, (double)py) > rad_sq);
                if (!keep) {
                    const int pidx = py * sw + px;
                    atomicAnd(&G.mark[pidx >> 5], ~(1u << (pidx & 31)));
                    G.unclaim(pidx);
                }
            }
            const unsigned km = __ballot_sync(kFull, keep);
            __syncwarp();
            if (keep) G.put(o + __popc(km & ((1u << lane) - 1)), xy);
            o += __popc(km);
            __syncwarp();
        }
        n = o;
        if (n < 2) return false;
        region2rect(G, n, reg_angle, prec, R);
        density = rect_density(n, R);
    }
    return true;
}

// kImgSmem: the half-resolution image is staged in shared memory (lowest latency, 2 frames per SM at VGA) or read from
// global memory through L1 / L2 (34 KB of shared memory per frame -> 6 frames per SM: more frames in flight for big
// batches; the images of a batch, 77 KB each, stay L2 resident)
template <bool kImgSmem>
__global__ void __launch_bounds__(32) lsd_grow_kernel(LineDev D) {
    PLP_DYNAMIC_SMEM(s_grow_raw);
    uint4 *s_grow = reinterpret_cast<uint4 *>(s_grow_raw);
    uint8_t *s_img = reinterpret_cast<uint8_t *>(s_grow);
    const int img_bytes = kImgSmem ? ((D.npx + 15) & ~15) : 0;
    uint32_t *s_used = reinterpret_cast<uint32_t *>(s_img + img_bytes);
    const int used_words = (D.npx + 31) >> 5;
    uint32_t *s_reg = s_used + ((used_words + 3) & ~3);
    const int b = blockIdx.x, lane = threadIdx.x;
    {  // stage the frame
        const uint8_t *src = D.scaled + (size_t)b * D.npx;
        if (!kImgSmem) {
            // nothing to stage
        } else if (((size_t)src & 15) == 0) {
            const uint4 *s4 = reinterpret_cast<const uint4 *>(src);
            for (int i = lane; i < D.npx / 16; i += 32) s_grow[i] = s4[i];
            for (int i = (D.npx / 16) * 16 + lane; i < D.npx; i += 32) s_img[i] = src[i];
        } else {
            for (int i = lane; i < D.npx; i += 32) s_img[i] = src[i];
        }
        for (int i = lane; i < used_words; i += 32) s_used[i] = 0;
    }
    __syncwarp();
    Grow G;
    G.sw = D.sw;
    G.sh = D.sh;
    G.kthr = D.kthr;
    G.density_th = D.density_th;
    G.img = kImgSmem ? s_img : D.scaled + (size_t)b * D.npx;
    G.reg_cap = kImgSmem ? kRegCap : D.reg_cap_small;
    G.used = s_used;
    G.mark = s_used;
    G.reg = s_reg;
    G.reg_ovf = D.reg_xy + (size_t)b * D.npx;
    G.tab = D.cstab;
    G.claim = nullptr;
    G.aborted = false;
    G.lane = lane;
    const uint32_t *order = D.order + (size_t)b * D.npx;
    float4 *segs = D.segs + (size_t)b * D.seg_cap;
    const int nseeds = D.nseeds[b];
    const int sw = D.sw;
    int nseg = 0;
    for (int s0 = 0; s0 < nseeds; s0 += 32) {
        const int s = s0 + lane;
        const uint32_t oxy = s < nseeds ? order[s] : 0;
        const int oidx = (int)(oxy >> 16) * sw + (int)(oxy & 0xffff);
        unsigned m = __ballot_sync(kFull, s < nseeds && !((s_used[oidx >> 5] >> (oidx & 31)) & 1u));
        while (m) {
            const int l = __ffs(m) - 1;
            const uint32_t seed_xy = __shfl_sync(kFull, oxy, l);
            const int sidx = __shfl_sync(kFull, oidx, l);
            int gx, gy;
            grad_at(G.img, sw, sidx, gx, gy);
            const float seed_deg = fast_atan2_deg((float)gx, (float)-gy);
            double reg_angle;
            int n = region_grow(G, seed_xy, seed_deg, D.prec, reg_angle);
            if (n >= D.min_reg_size) {
                Rect R;
                region2rect(G, n, reg_angle, D.prec, R);
                const bool okr = refine(G, n, seed_deg, reg_angle, D.prec, R);
                if (okr) {
                    if (nseg < D.seg_cap) {
                        if (lane == 0) {
                            // + 0.5 offset, then / scale (0.5)
                            segs[nseg] = make_float4((float)((R.x1 + 0.5) / 0.5), (float)((R.y1 + 0.5) / 0.5),
                                                     (float)((R.x2 + 0.5) / 0.5), (float)((R.y2 + 0.5) / 0.5));
                        }
                    } else if (lane == 0) {
                        atomicOr(&D.status[b], 1);
                    }
                    ++nseg;
                }
            }
            __syncwarp();
            m = __ballot_sync(kFull, s < nseeds && !((s_used[oidx >> 5] >> (oidx & 31)) & 1u)) & ~((2u << l) - 1u);
        }
    }
    if (lane == 0) D.nseg[b] = min(nseg, D.seg_cap);
}

// ------------------------------------------------------------------------------------------------------------------
// K4': the same region growing for a SINGLE live frame (small batches): kMwWarps warps of one CTA work on consecutive
//      seeds of the frame speculatively and commit in seed order, so the result is the sequential one bit for bit.
//
// The sequential algorithm visits the seeds in order; what it does with a seed depends on the `used` map only through the
// pixels it ACCEPTS into a region (a neighbour that is not aligned is rejected whether it is used or not, a used one is
// never accepted).  One round: every warp takes the next not-yet-used seed (warp w the w-th), grows / refines it against
// the committed map plus a private mark bitmap, and records the bounding box of every pixel it accepted at any time.  The
// round's seeds e < w come earlier in the sequential order: if the box of w is disjoint from the boxes of all of them,
// nothing they mark can be a pixel w accepted, so w saw exactly the map the sequential run would have shown it.  The
// longest conflict-free prefix of the round commits (marks are OR-ed into the committed map, segments are emitted in
// seed order); the first conflicting seed and everything after it is redone in the next round, where it is first (and
// therefore commits): every round makes progress.  Marks of a committed region are final (refinement only ever clears a
// region's OWN pixels, before it commits), which is why skipping a seed that is used in the committed map is exact.
// ------------------------------------------------------------------------------------------------------------------
constexpr int kMwMaxWarps = 8;
constexpr int kMwRegCap = 1024;  // region entries per warp in shared memory (longer regions continue in global memory)

struct MwCtl {
    int bbox[kMwMaxWarps][4];
    int nfinal[kMwMaxWarps];
    int ok[kMwMaxWarps];
    float4 seg[kMwMaxWarps];
    unsigned long long stat[8];  // rounds, seeds run, seeds redone, cycles of warp 0: scan, own seed, wait, commit (tuning aid)
};

__global__ void __launch_bounds__(kMwMaxWarps * 32) lsd_grow_mw_kernel(LineDev D, uint32_t *reg_ovf_mw) {
    PLP_DYNAMIC_SMEM(s_grow_raw);
    uint4 *s_grow = reinterpret_cast<uint4 *>(s_grow_raw);
    const int W = blockDim.x >> 5;
    uint8_t *s_img = reinterpret_cast<uint8_t *>(s_grow);
    const int img_bytes = (D.npx + 15) & ~15;
    const int used_words = (D.npx + 31) >> 5, used_pad = (used_words + 3) & ~3;
    uint32_t *s_used = reinterpret_cast<uint32_t *>(s_img + img_bytes);  // committed marks
    uint32_t *s_priv = s_used + used_pad;                                // W private bitmaps
    uint32_t *s_reg = s_priv + (size_t)W * used_pad;                     // W region windows
    MwCtl &C = *reinterpret_cast<MwCtl *>(s_reg + (size_t)W * kMwRegCap);
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    {  // stage the frame
        const uint8_t *src = D.scaled + (size_t)b * D.npx;
        if (((size_t)src & 15) == 0) {
            const uint4 *s4 = reinterpret_cast<const uint4 *>(src);
            for (int i = tid; i < D.npx / 16; i += blockDim.x) s_grow[i] = s4[i];
            for (int i = (D.npx / 16) * 16 + tid; i < D.npx; i += blockDim.x) s_img[i] = src[i];
        } else {
            for (int i = tid; i < D.npx; i += blockDim.x) s_img[i] = src[i];
        }
        for (int i = tid; i < used_pad * (W + 1); i += blockDim.x) s_used[i] = 0;
        if (tid < 8) C.stat[tid] = 0;
    }
    __syncthreads();
    GrowT<true> G;
    G.sw = D.sw;
    G.sh = D.sh;
    G.kthr = D.kthr;
    G.density_th = D.density_th;
    G.img = s_img;
    G.reg_cap = kMwRegCap;
    G.used = s_used;
    G.mark = s_priv + (size_t)warp * used_pad;
    G.reg = s_reg + (size_t)warp * kMwRegCap;
    G.reg_ovf = reg_ovf_mw + ((size_t)b * kMwMaxWarps + warp) * D.npx;
    G.tab = D.cstab;
    G.claim = nullptr;
    G.aborted = false;
    G.lane = lane;
    const uint32_t *order = D.order + (size_t)b * D.npx;
    float4 *segs = D.segs + (size_t)b * D.seg_cap;
    const int nseeds = D.nseeds[b];
    const int sw = D.sw;
    int nseg = 0, cursor = 0;  // identical in every warp
    for (;;) {
        const long long tc0 = clock64();
        // ---- the next W seeds that are not used in the committed map (every warp scans for itself: same result)
        int my_pos = -1;       // lane i < W: position of the round's i-th seed in the order list
        uint32_t my_xy = 0;
        int found = 0, scan = cursor;
        while (found < W && scan < nseeds) {
            const int sidx_l = scan + lane;
            const uint32_t oxy = sidx_l < nseeds ? order[sidx_l] : 0;
            const int oidx = (int)(oxy >> 16) * sw + (int)(oxy & 0xffff);
            unsigned m = __ballot_sync(kFull, sidx_l < nseeds && !((s_used[oidx >> 5] >> (oidx & 31)) & 1u));
            while (m && found < W) {
                const int l = __ffs(m) - 1;
                m &= m - 1;
                const uint32_t xy = __shfl_sync(kFull, oxy, l);
                if (lane == found) {
                    my_pos = scan + l;
                    my_xy = xy;
                }
                ++found;
            }
            scan += 32;
        }
        if (found == 0) break;  // uniform over the CTA
        const long long tc1 = clock64();
        // ---- phase 1: warp w runs the w-th seed
        if (warp < found) {
            const uint32_t seed_xy = __shfl_sync(kFull, my_xy, warp);
            const int sidx = (int)(seed_xy >> 16) * sw + (int)(seed_xy & 0xffff);
            G.bx0 = G.by0 = 0x7fffffff;
            G.bx1 = G.by1 = -1;
            int gx, gy;
            grad_at(G.img, sw, sidx, gx, gy);
            const float seed_deg = fast_atan2_deg((float)gx, (float)-gy);
            double reg_angle;
            int n = region_grow(G, seed_xy, seed_deg, D.prec, reg_angle);
            bool okr = false;
            Rect R;
            if (n >= D.min_reg_size) {
                region2rect(G, n, reg_angle, D.prec, R);
                okr = refine(G, n, seed_deg, reg_angle, D.prec, R);
            }
            int x0 = G.bx0, y0 = G.by0, x1 = G.bx1, y1 = G.by1;
            for (int off = 16; off >= 1; off >>= 1) {
                x0 = min(x0, __shfl_xor_sync(kFull, x0, off));
                y0 = min(y0, __shfl_xor_sync(kFull, y0, off));
                x1 = max(x1, __shfl_xor_sync(kFull, x1, off));
                y1 = max(y1, __shfl_xor_sync(kFull, y1, off));
            }
            if (lane == 0) {
                C.bbox[warp][0] = x0;
                C.bbox[warp][1] = y0;
                C.bbox[warp][2] = x1;
                C.bbox[warp][3] = y1;
                C.nfinal[warp] = n;
                C.ok[warp] = okr ? 1 : 0;
                if (okr)  // + 0.5 offset, then / scale (0.5)
                    C.seg[warp] = make_float4((float)((R.x1 + 0.5) / 0.5), (float)((R.y1 + 0.5) / 0.5),
                                              (float)((R.x2 + 0.5) / 0.5), (float)((R.y2 + 0.5) / 0.5));
            }
        }
        const long long tc2 = clock64();
        __syncthreads();
        const long long tc3 = clock64();
        // ---- phase 2 (every warp, same result): first seed whose box meets the box of an earlier seed of the round
        int first_bad = found;
        {
            // lane = pair (v, e), e < v < found: at most 28 pairs
            int v = 1, e = lane;
            while (v < kMwMaxWarps && e >= v) {
                e -= v;
                ++v;
            }
            bool hit = false;
            if (v < found) {
                const int *bv = C.bbox[v], *be = C.bbox[e];
                hit = !(bv[2] < be[0] || be[2] < bv[0] || bv[3] < be[1] || be[3] < bv[1]);
            }
            for (int q = 1; q < found; ++q) {
                const unsigned mq = __ballot_sync(kFull, hit && v == q);
                if (mq && first_bad == found) first_bad = q;
            }
        }
        // ---- phase 3: commit the prefix, forget the rest
        if (warp < found) {
            const int n = C.nfinal[warp];
            const bool commit = warp < first_bad;
            for (int i = lane; i < n; i += 32) {
                const uint32_t xy = G.get(i);
                const int pidx = (int)(xy >> 16) * sw + (int)(xy & 0xffff);
                atomicAnd(&G.mark[pidx >> 5], ~(1u << (pidx & 31)));
                if (commit) atomicOr(&s_used[pidx >> 5], 1u << (pidx & 31));
            }
            if (commit && C.ok[warp] && lane == 0) {
                int slot = nseg;
                for (int e = 0; e < warp; ++e) slot += C.ok[e];
                if (slot < D.seg_cap) segs[slot] = C.seg[warp];
                else atomicOr(&D.status[b], 1);
            }
        }
        for (int e = 0; e < first_bad; ++e) nseg += C.ok[e];
        {
            const int pos_bad = __shfl_sync(kFull, my_pos, min(first_bad, found - 1));
            cursor = first_bad < found ? pos_bad : pos_bad + 1;
        }
        __syncthreads();
        if (tid == 0) {
            C.stat[0] += 1;
            C.stat[1] += (unsigned long long)found;
            C.stat[2] += (unsigned long long)(found - first_bad);
            C.stat[3] += (unsigned long long)(tc1 - tc0);
            C.stat[4] += (unsigned long long)(tc2 - tc1);
            C.stat[5] += (unsigned long long)(tc3 - tc2);
            C.stat[6] += (unsigned long long)(clock64() - tc3);
        }
    }
    if (tid == 0) {
        D.nseg[b] = min(nseg, D.seg_cap);
        if (D.mw_stat) {
            for (int q = 0; q < 7; ++q) D.mw_stat[8 * b + q] = C.stat[q];
        }
    }
}

// ------------------------------------------------------------------------------------------------------------------
// K4'': region growing for one live frame, OUT OF ORDER with in-order commit (a reorder buffer, as in a CPU core).
//
// The round protocol above loses much of its time waiting for the slowest seed of a round: 72 % of the seeds grow fewer
// than 5 pixels, 10 % grow a few hundred, and a round costs its slowest member.  Here a warp that has finished a small
// region PARKS it (its <= kOooPark pixels and its bounding box go into the ticket's reorder-buffer entry, the private marks
// are cleared) and takes the next seed at once, so the warps that draw small seeds run ahead -- up to kOooWindow tickets --
// while the long regions of several lines are grown concurrently by the other warps (a region too large to park is HELD by
// its warp until it commits).  Tickets = seeds in gradient order.  A ticket runs against the committed `used` map plus its
// own private marks only; it records `start_head` = the commit pointer when it started.  Commit is strictly in ticket
// order, by whichever warp finds the head entry finished: the entry is valid if the bounding box of everything it accepted
// is disjoint from the final boxes of the tickets in [start_head, ticket) -- the tickets before start_head were committed,
// hence fully visible, when it started; the others can only matter through pixels it accepted (see K4').  An invalid entry,
// and an entry that was DEFERRED because its seed lay inside a region another warp was growing (most likely about to be
// absorbed), is simply executed AT THE HEAD, where the committed map is exactly the sequential state -- so every decision that
// is not provably the sequential one is redone sequentially, and the segments come out in ticket order, bit for bit.
// ------------------------------------------------------------------------------------------------------------------
constexpr int kOooRing = 128;    // reorder-buffer entries (ticket % kOooRing)
constexpr int kOooWindow = 64;   // tickets in flight (<= kOooRing / 2: an entry is not reused while a later ticket may still test it)
constexpr int kOooPark = 24;     // pixels of a region that can be parked in its entry
constexpr int kOooRegCap = 512;  // region window per warp in shared memory (longer regions continue in global memory)

enum { kOooRunning = 1, kOooVoid = 2, kOooDeferred = 3, kOooParked = 4, kOooHeld = 5, kOooCommitted = 6 };

struct OooEntry {
    float4 seg;
    uint32_t xy;
    int state, start_head, owner, n, ok;
    short bx0, by0, bx1, by1;
    uint32_t px[kOooPark];
};

struct OooCtl {
    int lock_dispatch, lock_commit;
    int head, next_ticket;
    int scan_pos, chunk_base;
    unsigned chunk_mask;
    int nseg;
    uint32_t chunk_xy[32];
    int ctx_ticket[kMwMaxWarps + 1];  // ticket every context (warps + the head-execution context) works on, INT_MAX: none
    int pad_[3];
    unsigned long long stat[8];  // tickets, void, deferred, parked, held, executed at the head, conflicts, aborted
};

// (every wait of this kernel is bounded: after ~2 s of SM cycles a warp gives up, raises status bit 2 and leaves -- a protocol
// bug must not hang the device)
#ifdef PLP_CTA_EMU
constexpr long long kOooTimeout = 1200000000000ll;  // the host emulation counts nanoseconds and is ~1000x slower
#else
constexpr long long kOooTimeout = 4000000000ll;
#endif
__device__ __forceinline__ bool ooo_expired(long long t_start) {  // one lane decides (the lanes' clocks differ by a few cycles)
    int e = 0;
    if ((threadIdx.x & 31) == 0) e = clock64() - t_start > kOooTimeout ? 1 : 0;
    return __shfl_sync(kFull, e, 0) != 0;
}
__device__ __forceinline__ bool ooo_lock(int *l, int lane, long long t_start) {
    int ok = 1;
    if (lane == 0) {
        while (atomicCAS(l, 0, 1) != 0) {
            __nanosleep(40);
            if (clock64() - t_start > kOooTimeout) {
                ok = 0;
                break;
            }
        }
        __threadfence_block();
    }
    return __shfl_sync(kFull, ok, 0) != 0;
}
__device__ __forceinline__ bool ooo_trylock(int *l, int lane) {
    int got = 0;
    if (lane == 0) {
        got = atomicCAS(l, 0, 1) == 0 ? 1 : 0;
        if (got) __threadfence_block();
    }
    return __shfl_sync(kFull, got, 0) != 0;
}
__device__ __forceinline__ void ooo_unlock(int *l, int lane) {
    __syncwarp();
    if (lane == 0) {
        __threadfence_block();
        atomicExch(l, 0);
    }
    __syncwarp();
}
// A word that another warp may change at any moment is read by ONE lane and broadcast: if every lane read it for itself the
// lanes of a warp could see different values and take different branches around warp-collective operations (this hung the
// first version of the kernel).
__device__ __forceinline__ int ooo_ld(const int *p) {
    int v = 0;
    if ((threadIdx.x & 31) == 0) v = *reinterpret_cast<const volatile int *>(p);
    return __shfl_sync(kFull, v, 0);
}

// one seed against `G.used | G.mark`: grow, rectangle, refinement.  Returns the final region size (marks left in G.mark, list in
// G.reg); ok / seg describe the segment; the bounding box of everything accepted is left in (x0, y0, x1, y1).
// (G by value: a private copy whose address never escapes, so that its fields -- the bounding box above all -- live in registers)
__device__ __forceinline__ int ooo_run_seed(const GrowT<true> G, const LineDev &D, uint32_t seed_xy, bool &okr, float4 &seg, int &x0,
                                            int &y0, int &x1, int &y1, bool &aborted) {
    const int sw = D.sw, lane = G.lane;
    const int sidx = (int)(seed_xy >> 16) * sw + (int)(seed_xy & 0xffff);
    G.bx0 = G.by0 = 0x7fffffff;
    G.bx1 = G.by1 = -1;
    int gx, gy;
    grad_at(G.img, sw, sidx, gx, gy);
    const float seed_deg = fast_atan2_deg((float)gx, (float)-gy);
    double reg_angle;
    G.aborted = false;
    int n = region_grow(G, seed_xy, seed_deg, D.prec, reg_angle);
    okr = false;
    Rect R;
    if (!G.aborted && n >= D.min_reg_size) {
        region2rect(G, n, reg_angle, D.prec, R);
        okr = refine(G, n, seed_deg, reg_angle, D.prec, R);
    }
    aborted = G.aborted;
    if (aborted) okr = false;
    x0 = G.bx0, y0 = G.by0, x1 = G.bx1, y1 = G.by1;
    for (int off = 16; off >= 1; off >>= 1) {
        x0 = min(x0, __shfl_xor_sync(kFull, x0, off));
        y0 = min(y0, __shfl_xor_sync(kFull, y0, off));
        x1 = max(x1, __shfl_xor_sync(kFull, x1, off));
        y1 = max(y1, __shfl_xor_sync(kFull, y1, off));
    }
    seg = make_float4(0.f, 0.f, 0.f, 0.f);
    if (okr)  // + 0.5 offset, then / scale (0.5)
        seg = make_float4((float)((R.x1 + 0.5) / 0.5), (float)((R.y1 + 0.5) / 0.5), (float)((R.x2 + 0.5) / 0.5),
                          (float)((R.y2 + 0.5) / 0.5));
    (void)lane;
    return n;
}

struct OooShared {
    OooCtl *C;
    OooEntry *ring;
    uint32_t *used;  // committed marks
    int used_pad, sw;
};

// region list of G (n entries) -> committed map; the private marks are cleared
__device__ __forceinline__ void ooo_commit_list(const GrowT<true> &G, uint32_t *used, int n, int sw, bool commit) {
    for (int i = G.lane; i < n; i += 32) {
        const uint32_t xy = G.get(i);
        const int pidx = (int)(xy >> 16) * sw + (int)(xy & 0xffff);
        atomicAnd(&G.mark[pidx >> 5], ~(1u << (pidx & 31)));
        G.unclaim(pidx);
        if (commit) atomicOr(&used[pidx >> 5], 1u << (pidx & 31));
    }
    __syncwarp();
}

// Commit finished tickets from the head, in order (warp-collective; returns at once if another warp is draining).
// `Gown`: the caller's context (its HELD region, if any, is committed from it); `Gsp`: the spare context that whoever holds the
// commit lock uses to execute a ticket at the head.
__device__ void ooo_drain(const OooShared &S, const LineDev &D, const GrowT<true> &Gown, const GrowT<true> &Gsp, int warp, float4 *segs,
                          int b) {
    OooCtl &C = *S.C;
    const int lane = Gown.lane;
    {  // look before locking: when the head entry is still running, or is held by another warp (only its owner commits it),
       // taking the lock is pointless -- and the warps that spin here while the window is full would keep it away from that
       // owner (the first GPU run of this kernel starved a HELD owner for its whole 2 s budget that way)
        const int h = ooo_ld(&C.head);
        if (h == ooo_ld(&C.next_ticket)) return;
        const OooEntry &E = S.ring[h & (kOooRing - 1)];
        const int st = ooo_ld(&E.state);
        if (st == kOooRunning || (st == kOooHeld && ooo_ld(&E.owner) != warp)) return;
    }
    if (!ooo_trylock(&C.lock_commit, lane)) return;
    for (;;) {
        const int h = ooo_ld(&C.head);
        if (h == ooo_ld(&C.next_ticket)) break;
        OooEntry &E = S.ring[h & (kOooRing - 1)];
        const int st = ooo_ld(&E.state);
        if (st == kOooRunning) break;
        const int owner = ooo_ld(&E.owner);
        if (st == kOooHeld && owner != warp) break;  // its owner commits it (it is spinning on this lock)
        bool exec = st == kOooDeferred;
        if (st == kOooParked || st == kOooHeld) {
            // valid  <=>  box disjoint from the final boxes of the tickets that were not yet committed when it started
            bool hit = false;
            const int bx0 = E.bx0, by0 = E.by0, bx1 = E.bx1, by1 = E.by1;
            for (int e = E.start_head + lane; e < h; e += 32) {
                const OooEntry &F = S.ring[e & (kOooRing - 1)];
                hit = hit || !(F.bx1 < bx0 || bx1 < F.bx0 || F.by1 < by0 || by1 < F.by0);  // (an empty box has bx1 = -1 < bx0)
            }
            if (__any_sync(kFull, hit)) {
                exec = true;
                if (lane == 0) C.stat[6]++;
            }
        }
        int nseg = ooo_ld(&C.nseg);
        if (st == kOooVoid) {
            // nothing
        } else if (exec) {
            if (st == kOooHeld) ooo_commit_list(Gown, S.used, E.n, S.sw, false);  // drop the caller's speculative region
            const uint32_t seed_xy = E.xy;
            const int sidx = (int)(seed_xy >> 16) * S.sw + (int)(seed_xy & 0xffff);
            int n = 0, x0 = 0x7fffffff, y0 = 0x7fffffff, x1 = -1, y1 = -1;
            bool okr = false;
            float4 seg = make_float4(0.f, 0.f, 0.f, 0.f);
            if (!((ooo_ld(reinterpret_cast<const int *>(&S.used[sidx >> 5])) >> (sidx & 31)) & 1)) {  // the committed map IS the sequential state here
                GrowT<true> Gh = Gsp;
                Gh.my_ticket = h;  // the lowest ticket in flight: nothing it meets can belong to an earlier one, it never stops
                if (lane == 0) *reinterpret_cast<volatile int *>(&C.ctx_ticket[Gsp.self]) = h;
                __syncwarp();
                bool ab;
                n = ooo_run_seed(Gh, D, seed_xy, okr, seg, x0, y0, x1, y1, ab);
                ooo_commit_list(Gsp, S.used, n, S.sw, true);
                if (lane == 0) *reinterpret_cast<volatile int *>(&C.ctx_ticket[Gsp.self]) = 0x7fffffff;
            }
            if (lane == 0) {
                E.bx0 = (short)min(x0, 32767);
                E.by0 = (short)min(y0, 32767);
                E.bx1 = (short)x1;
                E.by1 = (short)y1;
                C.stat[5]++;
                if (okr) {
                    if (nseg < D.seg_cap) segs[nseg] = seg;
                    else atomicOr(&D.status[b], 1);
                    C.nseg = nseg + 1;
                }
            }
        } else {  // a valid speculative result
            if (st == kOooParked) {
                if (lane < E.n) {
                    const uint32_t xy = E.px[lane];
                    const int pidx = (int)(xy >> 16) * S.sw + (int)(xy & 0xffff);
                    atomicOr(&S.used[pidx >> 5], 1u << (pidx & 31));
                }
            } else {
                ooo_commit_list(Gown, S.used, E.n, S.sw, true);
            }
            if (lane == 0 && E.ok) {
                if (nseg < D.seg_cap) segs[nseg] = E.seg;
                else atomicOr(&D.status[b], 1);
                C.nseg = nseg + 1;
            }
        }
        __syncwarp();
        if (lane == 0) {
            __threadfence_block();
            if (st == kOooHeld) *reinterpret_cast<volatile int *>(&E.state) = kOooCommitted;  // releases the owner (the caller)
            *reinterpret_cast<volatile int *>(&C.head) = h + 1;
        }
        __syncwarp();
    }
    ooo_unlock(&C.lock_commit, lane);
}

__global__ void __launch_bounds__(kMwMaxWarps * 32) lsd_grow_ooo_kernel(LineDev D, uint32_t *reg_ovf_mw) {
    PLP_DYNAMIC_SMEM(s_grow_raw);
    uint4 *s_grow = reinterpret_cast<uint4 *>(s_grow_raw);
    const int W = blockDim.x >> 5;
    uint8_t *s_img = reinterpret_cast<uint8_t *>(s_grow);
    const int img_bytes = (D.npx + 15) & ~15;
    const int used_words = (D.npx + 31) >> 5, used_pad = (used_words + 3) & ~3;
    uint32_t *s_used = reinterpret_cast<uint32_t *>(s_img + img_bytes);  // committed marks
    uint32_t *s_priv = s_used + used_pad;                                // W + 1 private bitmaps (the last one: head execution)
    uint32_t *s_claim = s_priv + (size_t)(W + 1) * used_pad;             // union of the private bitmaps (collision detector)
    uint32_t *s_reg = s_claim + used_pad;                                // W + 1 region windows
    OooEntry *ring = reinterpret_cast<OooEntry *>(s_reg + (size_t)(W + 1) * kOooRegCap);
    OooCtl &C = *reinterpret_cast<OooCtl *>(ring + kOooRing);
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    {  // stage the frame
        const uint8_t *src = D.scaled + (size_t)b * D.npx;
        if (((size_t)src & 15) == 0) {
            const uint4 *s4 = reinterpret_cast<const uint4 *>(src);
            for (int i = tid; i < D.npx / 16; i += blockDim.x) s_grow[i] = s4[i];
            for (int i = (D.npx / 16) * 16 + tid; i < D.npx; i += blockDim.x) s_img[i] = src[i];
        } else {
            for (int i = tid; i < D.npx; i += blockDim.x) s_img[i] = src[i];
        }
        for (int i = tid; i < used_pad * (W + 3); i += blockDim.x) s_used[i] = 0;
        uint32_t *z = reinterpret_cast<uint32_t *>(ring);
        for (int i = tid; i < (int)((sizeof(OooEntry) * kOooRing + sizeof(OooCtl)) / 4); i += blockDim.x) z[i] = 0;
    }
    __syncthreads();
    GrowT<true> G, Gsp;
    G.sw = D.sw;
    G.sh = D.sh;
    G.kthr = D.kthr;
    G.density_th = D.density_th;
    G.img = s_img;
    G.reg_cap = kOooRegCap;
    G.used = s_used;
    G.tab = D.cstab;
    G.lane = lane;
    G.claim = s_claim;
    G.priv_base = s_priv;
    G.ctx_ticket = C.ctx_ticket;
    G.nctx = W + 1;
    G.ctx_words = used_pad;
    G.my_ticket = 0x7fffffff;
    G.aborted = false;
    G.self = warp;
    Gsp = G;
    Gsp.self = W;
    G.mark = s_priv + (size_t)warp * used_pad;
    G.reg = s_reg + (size_t)warp * kOooRegCap;
    G.reg_ovf = reg_ovf_mw + ((size_t)b * (kMwMaxWarps + 1) + warp) * D.npx;
    Gsp.mark = s_priv + (size_t)W * used_pad;
    Gsp.reg = s_reg + (size_t)W * kOooRegCap;
    Gsp.reg_ovf = reg_ovf_mw + ((size_t)b * (kMwMaxWarps + 1) + kMwMaxWarps) * D.npx;
    OooShared S{&C, ring, s_used, used_pad, D.sw};
    const uint32_t *order = D.order + (size_t)b * D.npx;
    float4 *segs = D.segs + (size_t)b * D.seg_cap;
    const int nseeds = D.nseeds[b];
    const int sw = D.sw;
    if (tid <= W) C.ctx_ticket[tid] = 0x7fffffff;
    __syncthreads();
    const long long t_start = clock64();
    bool timed_out = false;
    for (;;) {
        if (ooo_expired(t_start)) {
            timed_out = true;
            break;
        }
        // ---- take the next ticket: the next seed (in order) that is not used in the committed map
        int t = -1;  // -1: no seed left, -2: the window is full
        if (!ooo_lock(&C.lock_dispatch, lane, t_start)) {
            timed_out = true;
            break;
        }
        {
            const int nt = ooo_ld(&C.next_ticket);
            if (nt - ooo_ld(&C.head) >= kOooWindow) {
                t = -2;
            } else {
                unsigned m = (unsigned)ooo_ld(reinterpret_cast<const int *>(&C.chunk_mask));
                int base = ooo_ld(&C.chunk_base), sp = ooo_ld(&C.scan_pos);
                uint32_t cxy = *reinterpret_cast<volatile uint32_t *>(&C.chunk_xy[lane]);
                while (m == 0u && sp < nseeds) {
                    const int p = sp + lane;
                    cxy = p < nseeds ? order[p] : 0u;
                    const int oidx = (int)(cxy >> 16) * sw + (int)(cxy & 0xffff);
                    m = __ballot_sync(kFull, p < nseeds && !((s_used[oidx >> 5] >> (oidx & 31)) & 1u));
                    base = sp;
                    sp += 32;
                }
                if (m != 0u) {
                    const int l = __ffs(m) - 1;
                    const uint32_t xy = __shfl_sync(kFull, cxy, l);
                    const int head_now = ooo_ld(&C.head);
                    t = nt;
                    if (lane == 0) {
                        OooEntry &E = ring[t & (kOooRing - 1)];
                        E.xy = xy;
                        E.start_head = head_now;
                        E.owner = warp;
                        E.n = 0;
                        E.ok = 0;
                        E.bx0 = E.by0 = 32767;
                        E.bx1 = E.by1 = -1;
                        *reinterpret_cast<volatile int *>(&E.state) = kOooRunning;
                        C.stat[0]++;
                    }
                    m &= m - 1;
                }
                C.chunk_xy[lane] = cxy;
                if (lane == 0) {
                    C.chunk_mask = m;
                    C.chunk_base = base;
                    C.scan_pos = sp;
                    if (t >= 0) {
                        __threadfence_block();
                        *reinterpret_cast<volatile int *>(&C.next_ticket) = t + 1;
                    }
                }
            }
        }
        ooo_unlock(&C.lock_dispatch, lane);
        if (t < 0) {
            if (t == -1 && ooo_ld(&C.head) == ooo_ld(&C.next_ticket)) {
                // every ticket is committed; a seed can only have been left behind if another warp is between its scan and
                // its ticket, which the dispatch lock excludes
                break;
            }
            ooo_drain(S, D, G, Gsp, warp, segs, b);
            __nanosleep(400);
            continue;
        }
        OooEntry &E = ring[t & (kOooRing - 1)];
        const uint32_t seed_xy = E.xy;
        const int sidx = (int)(seed_xy >> 16) * sw + (int)(seed_xy & 0xffff);
        int state;
        // (the committed map changes under our feet: one lane reads the word, see ooo_ld)
        if ((ooo_ld(reinterpret_cast<const int *>(&s_used[sidx >> 5])) >> (sidx & 31)) & 1) {
            state = kOooVoid;  // committed since the scan: by a ticket before this one, so the sequential run skips it too
        } else {
            // inside a region another warp is growing right now: most likely absorbed -- decided at the head instead
            bool other = false;
            if (lane < W && lane != warp) other = (s_priv[(size_t)lane * used_pad + (sidx >> 5)] >> (sidx & 31)) & 1u;
            if (__any_sync(kFull, other)) {
                state = kOooDeferred;
            } else {
                bool okr, aborted;
                float4 seg;
                int x0, y0, x1, y1;
                G.my_ticket = t;
                if (lane == 0) *reinterpret_cast<volatile int *>(&C.ctx_ticket[warp]) = t;
                __syncwarp();
                const int n = ooo_run_seed(G, D, seed_xy, okr, seg, x0, y0, x1, y1, aborted);
                if (aborted) {
                    // ran into a pixel of an earlier region in flight: most likely this seed is about to be absorbed -- forget the
                    // partial region and let the head decide
                    ooo_commit_list(G, s_used, n, sw, false);
                    if (lane == 0) {
                        *reinterpret_cast<volatile int *>(&C.ctx_ticket[warp]) = 0x7fffffff;
                        C.stat[7]++;
                    }
                    state = kOooDeferred;
                } else {
                if (lane == 0) {
                    E.n = n;
                    E.ok = okr ? 1 : 0;
                    E.seg = seg;
                    E.bx0 = (short)x0;
                    E.by0 = (short)y0;
                    E.bx1 = (short)x1;
                    E.by1 = (short)y1;
                }
                if (n <= kOooPark) {
                    if (lane < n) E.px[lane] = G.get(lane);
                    __syncwarp();
                    ooo_commit_list(G, s_used, n, sw, false);  // clears the private marks only
                    if (lane == 0) *reinterpret_cast<volatile int *>(&C.ctx_ticket[warp]) = 0x7fffffff;
                    state = kOooParked;
                } else {
                    state = kOooHeld;  // (the context keeps its ticket until the region is committed)
                }
                }
            }
        }
        __syncwarp();
        if (lane == 0) {
            C.stat[state - 1]++;  // (counted without the lock: a tuning aid, may lose increments)
            __threadfence_block();
            *reinterpret_cast<volatile int *>(&E.state) = state;
        }
        __syncwarp();
        if (state == kOooHeld) {
            while (ooo_ld(&E.state) == kOooHeld) {
                ooo_drain(S, D, G, Gsp, warp, segs, b);
                if (ooo_ld(&E.state) == kOooHeld) __nanosleep(100);
                if (ooo_expired(t_start)) {
                    timed_out = true;
                    break;
                }
            }
            if (timed_out) break;
            if (lane == 0) *reinterpret_cast<volatile int *>(&C.ctx_ticket[warp]) = 0x7fffffff;
        } else {
            ooo_drain(S, D, G, Gsp, warp, segs, b);
        }
    }
    if (timed_out && lane == 0) {
        atomicOr(&D.status[b], 2);
        const int h = C.head;
        const OooEntry &E = ring[h & (kOooRing - 1)];
        printf("[ooo timeout] frame %d warp %d: head %d next %d scan_pos %d/%d | head entry: state %d owner %d n %d start_head %d | my ctx ticket %d "
               "locks d%d c%d\n", b, warp, h, C.next_ticket, C.scan_pos, nseeds, E.state, E.owner, E.n, E.start_head, C.ctx_ticket[warp],
               C.lock_dispatch, C.lock_commit);
    }
    __syncthreads();
    if (tid == 0) {
        D.nseg[b] = min(C.nseg, D.seg_cap);
        if (D.mw_stat)
            for (int q = 0; q < 8; ++q) D.mw_stat[8 * b + q] = C.stat[q];
    }
}


}  // namespace lsd
}  // namespace plp
