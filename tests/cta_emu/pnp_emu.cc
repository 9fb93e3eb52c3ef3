// pnp_emu.cc -- csrc/pnp_kernels.cuh executed on the host (see cta_emu.h), with the launch sequence of csrc/pnp.cu.
// Outputs use the C ABI's convention: a problem that does not run gets valid 0 / num_inliers 0 and nothing else.
#include "cta_emu.h"

#include <string.h>

#include "pnp_kernels.cuh"

using namespace plp;

extern "C" void emu_pnp_ransac(int num_problems, const int32_t *offsets, const double *bearings, const double *pos_w,
                               const float *max_cos, const int32_t *samples, int num_iter, int min_num_inliers,
                               int recompute, int32_t *valid_out, int32_t *num_inliers_out, double *pose_out,
                               uint8_t *is_inlier_out) {
    const size_t P = (size_t)num_problems, K = (size_t)num_iter, N = (size_t)offsets[num_problems];
    std::vector<double> hyp(P * K * 12 + 1), pws(3 * N + 3), us(2 * N + 2), alphas(4 * N + 4), pcs(3 * N + 3),
        pose(P * 16 + 1);
    std::vector<int32_t> cnt(P * K + 1);
    std::vector<int> signs(N + 1);
    std::vector<uint8_t> flags(N + 1);
    PnpJob J;
    J.offsets = offsets;
    J.bearings = bearings;
    J.pos_w = pos_w;
    J.max_cos = max_cos;
    J.samples = samples;
    J.num_problems = num_problems;
    J.num_iter = num_iter;
    J.min_num_inliers = min_num_inliers;
    J.recompute = recompute;
    J.hyp_Rt = hyp.data();
    J.hyp_count = cnt.data();
    J.pws = pws.data();
    J.us = us.data();
    J.alphas = alphas.data();
    J.pcs = pcs.data();
    J.signs = signs.data();
    J.valid = valid_out;
    J.num_inliers = num_inliers_out;
    J.pose = pose.data();
    J.is_inlier = flags.data();
    if (num_iter > 0)
        emu_launch2(pnp_hypothesis_kernel, (unsigned)num_problems, (unsigned)num_iter, (unsigned)kPnpHypThreads, (size_t)0, J);
    emu_launch(pnp_select_kernel, (unsigned)num_problems, (unsigned)kPnpThreads, J);
    for (int p = 0; p < num_problems; ++p) {
        const int off = offsets[p], n = offsets[p + 1] - off;
        if (n < kPnpMinSet || n < min_num_inliers) continue;
        memcpy(is_inlier_out + off, flags.data() + off, (size_t)n);
        if (valid_out[p]) memcpy(pose_out + 16 * (size_t)p, pose.data() + 16 * (size_t)p, sizeof(double) * 16);
    }
}
