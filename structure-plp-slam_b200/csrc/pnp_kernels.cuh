// pnp_kernels.cuh -- device code of the batched EPnP RANSAC (pnp.cu launches it).  Free of host-side CUDA runtime
// dependencies so that tests/cta_emu can compile the same text for the host (see essential_kernels.cuh).
#pragma once
#include <stddef.h>
#include <stdint.h>

#include "pnpmath.h"

namespace plp {

namespace {

constexpr int kPnpHypThreads = 32;  // one warp: thread 0 solves, the warp tests; ~8 CTAs per SM at 252 registers
constexpr int kPnpThreads = 160;     // select / recompute: >= 144, one thread per M^T M entry
constexpr int kPnpMinSet = 4;     // pnp_solver.cc:75

// P independent problems; problem p owns correspondences [offsets[p], offsets[p + 1]).  Every pointer is a device
// pointer, so a caller that already holds the correspondences on the device can fill the job directly.
struct PnpJob {
    const int32_t *offsets;   // P + 1
    const double *bearings;   // N x 3
    const double *pos_w;      // N x 3
    const float *max_cos;     // N
    const int32_t *samples;   // P x num_iter x 4, problem-local indices
    int num_problems, num_iter, min_num_inliers, recompute;
    // per hypothesis
    double *hyp_Rt;           // P x num_iter x 12: R row-major, t
    int32_t *hyp_count;       // P x num_iter: check_inliers' count
    // the recompute's working set (pws_ / us_ / alphas_ / pcs_ / signs_), sliced by the offsets
    double *pws, *us, *alphas, *pcs;
    int *signs;
    // results
    int32_t *valid;           // P
    int32_t *num_inliers;     // P
    double *pose;             // P x 16
    uint8_t *is_inlier;       // N
};

// find_via_ransac's early exit (:76-80)
__device__ __forceinline__ bool pnp_runs(const PnpJob &J, int p, int *off, int *n) {
    *off = J.offsets[p];
    *n = J.offsets[p + 1] - *off;
    return *n >= kPnpMinSet && *n >= J.min_num_inliers;
}

// One warp-sized CTA per (problem, hypothesis), grid (P, num_iter): thread 0 solves the minimal EPnP (:98-111), every
// thread tests a strided share of the problem's correspondences (:114, check_inliers), the count is an integer sum.
__global__ void __launch_bounds__(kPnpHypThreads, 1) pnp_hypothesis_kernel(PnpJob J) {
    __shared__ double sRt[12];
    __shared__ int s_cnt;
    const int p = blockIdx.x, iter = blockIdx.y, tid = threadIdx.x;
    int off, n;
    if (!pnp_runs(J, p, &off, &n)) return;
    const size_t h = (size_t)p * J.num_iter + iter;
    if (tid == 0) {
        double pws[3 * kPnpMinSet], us[2 * kPnpMinSet], alphas[4 * kPnpMinSet], pcs[3 * kPnpMinSet];
        int signs[kPnpMinSet];
        pnp_work w{pws, us, alphas, pcs, signs, 0};
        const int32_t *s = J.samples + h * kPnpMinSet;
        for (int k = 0; k < kPnpMinSet; ++k)
            pnp_add_correspondence(&w, J.pos_w + 3 * (size_t)(off + s[k]), J.bearings + 3 * (size_t)(off + s[k]));
        pnp_compute_pose(&w, sRt, sRt + 9);
        for (int k = 0; k < 12; ++k) J.hyp_Rt[h * 12 + k] = sRt[k];
        s_cnt = 0;
    }
    __syncthreads();
    int local = 0;
    for (int i = tid; i < n; i += kPnpHypThreads)
        local += pnp_is_inlier(sRt, sRt + 9, J.pos_w + 3 * (size_t)(off + i), J.bearings + 3 * (size_t)(off + i),
                               J.max_cos[off + i]);
    atomicAdd(&s_cnt, local);
    __syncthreads();
    if (tid == 0) J.hyp_count[h] = s_cnt;
}

// One CTA per problem: the ordered "max_num_inliers < num_inliers" replay (:117-123), the validity test (:126-129), the
// winner's inlier flags, and the optional recompute over the inliers in correspondence order (:136-152): thread 0 builds
// the control points and barycentric coordinates, one thread per entry sums M^T M in correspondence order, thread 0
// finishes the solve.  The flags are not re-tested after the recompute, as in the reference.
__global__ void __launch_bounds__(kPnpThreads, 1) pnp_select_kernel(PnpJob J) {
    __shared__ int s_best, s_valid;
    __shared__ pnp_work s_w;
    __shared__ double s_cws[4][3];
    __shared__ double s_mtm[144];
    const int p = blockIdx.x, tid = threadIdx.x;
    int off, n;
    if (!pnp_runs(J, p, &off, &n)) {
        if (tid == 0) J.valid[p] = J.num_inliers[p] = 0;
        return;
    }
    if (tid == 0) {
        int best = -1, max_num_inliers = 0;
        for (int it = 0; it < J.num_iter; ++it) {
            const int num = J.hyp_count[(size_t)p * J.num_iter + it];
            if (max_num_inliers < num) {
                max_num_inliers = num;
                best = it;
            }
        }
        s_best = best;
        s_valid = max_num_inliers > J.min_num_inliers;
        J.num_inliers[p] = max_num_inliers;
        J.valid[p] = s_valid;
    }
    __syncthreads();
    const int best = s_best;
    const double *Rt = J.hyp_Rt + ((size_t)p * J.num_iter + (best < 0 ? 0 : best)) * 12;
    for (int i = tid; i < n; i += kPnpThreads)
        J.is_inlier[off + i] = best < 0 ? 0 : (uint8_t)pnp_is_inlier(Rt, Rt + 9, J.pos_w + 3 * (size_t)(off + i),
                                                                      J.bearings + 3 * (size_t)(off + i), J.max_cos[off + i]);
    if (!s_valid) return;
    if (!J.recompute) {
        if (tid == 0) pnp_cam_pose(Rt, Rt + 9, J.pose + 16 * (size_t)p);
        return;
    }
    __syncthreads();  // the flags of this CTA are in global memory
    if (tid == 0) {
        s_w = pnp_work{J.pws + 3 * (size_t)off, J.us + 2 * (size_t)off, J.alphas + 4 * (size_t)off,
                       J.pcs + 3 * (size_t)off, J.signs + off, 0};
        for (int i = 0; i < n; ++i)
            if (J.is_inlier[off + i])
                pnp_add_correspondence(&s_w, J.pos_w + 3 * (size_t)(off + i), J.bearings + 3 * (size_t)(off + i));
        pnp_control_points(&s_w, s_cws);
    }
    __syncthreads();
    if (tid < 144) s_mtm[tid] = pnp_mtm_entry(&s_w, tid / 12, tid % 12);
    __syncthreads();
    if (tid == 0) {
        double R[9], t[3];
        pnp_compute_pose_from_mtm(&s_w, s_cws, s_mtm, R, t);
        pnp_cam_pose(R, t, J.pose + 16 * (size_t)p);
    }
}

}  // namespace

}  // namespace plp
