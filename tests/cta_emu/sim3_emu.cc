// sim3_emu.cc -- csrc/sim3_kernels.cuh executed on the host (see cta_emu.h), with the launch sequence of csrc/sim3.cu.
// cams: P x 4 (fx, fy, cx, cy), as sim3.cu stages them.
#include "cta_emu.h"

#include "sim3_kernels.cuh"

using namespace plp;

extern "C" void emu_sim3_ransac(int num_problems, const int32_t *offsets, const double *cams, const double *pts_1,
                                const double *pts_2, const float *chi_sq_1, const float *chi_sq_2, const int32_t *samples,
                                int num_iter, int fix_scale, int min_num_inliers, int32_t *valid_out,
                                int32_t *num_inliers_out, double *rot_12_out, double *trans_12_out, float *scale_12_out) {
    const size_t P = (size_t)num_problems, K = (size_t)num_iter, N = (size_t)offsets[num_problems];
    std::vector<double> reproj_1(2 * N + 2), reproj_2(2 * N + 2), hyp(P * K * 12 + 1);
    std::vector<float> hyp_scale(P * K + 1);
    std::vector<int32_t> cnt(P * K + 1);
    Sim3Job J;
    J.offsets = offsets;
    J.cams = cams;
    J.pts_1 = pts_1;
    J.pts_2 = pts_2;
    J.chi_sq_1 = chi_sq_1;
    J.chi_sq_2 = chi_sq_2;
    J.samples = samples;
    J.num_problems = num_problems;
    J.num_iter = num_iter;
    J.fix_scale = fix_scale;
    J.min_num_inliers = min_num_inliers;
    J.reproj_1 = reproj_1.data();
    J.reproj_2 = reproj_2.data();
    J.hyp_Rt = hyp.data();
    J.hyp_scale = hyp_scale.data();
    J.hyp_count = cnt.data();
    J.valid = valid_out;
    J.num_inliers = num_inliers_out;
    J.rot_12 = rot_12_out;
    J.trans_12 = trans_12_out;
    J.scale_12 = scale_12_out;
    if (num_problems == 0) return;
    if (num_iter > 0) {
        emu_launch(sim3_reproject_kernel, (unsigned)num_problems, (unsigned)kSim3PrepThreads, J);
        emu_launch2(sim3_hypothesis_kernel, (unsigned)num_problems, (unsigned)num_iter, (unsigned)kSim3Threads, (size_t)0, J);
    }
    emu_launch(sim3_select_kernel, (unsigned)num_problems, (unsigned)kSim3Threads, J);
}
