// sim3opt_emu.cc -- csrc/sim3_opt_kernels.cuh (one 128-thread CTA per problem) executed on the host (see cta_emu.h), with
// the staging of csrc/sim3_opt.cu.  cams: P x 4 (fx, fy, cx, cy); poses: P x 12 (rot row-major, trans) per keyframe.
#include "cta_emu.h"

#include <math.h>

#include "sim3_opt_kernels.cuh"

using namespace plp;

extern "C" void emu_sim3_optimize(int num_problems, const int32_t *offsets, const double *cams, const double *pose_1w,
                                  const double *pose_2w, const double *rot_12_in, const double *trans_12_in,
                                  const double *scale_12_in, const double *pos_w_1, const double *pos_w_2,
                                  const float *obs_1, const float *obs_2, const float *inv_sigma_sq_1,
                                  const float *inv_sigma_sq_2, float chi_sq, int num_iter, int fix_scale,
                                  int32_t *num_inliers_out, double *rot_12_out, double *trans_12_out, double *scale_12_out,
                                  uint8_t *inlier_out) {
    s3opt::Sim3OptJob J;
    J.offsets = offsets;
    J.cams = cams;
    J.pose_1w = pose_1w;
    J.pose_2w = pose_2w;
    J.rot_12_in = rot_12_in;
    J.trans_12_in = trans_12_in;
    J.scale_12_in = scale_12_in;
    J.pos_w_1 = pos_w_1;
    J.pos_w_2 = pos_w_2;
    J.obs_1 = obs_1;
    J.obs_2 = obs_2;
    J.inv_sigma_sq_1 = inv_sigma_sq_1;
    J.inv_sigma_sq_2 = inv_sigma_sq_2;
    J.chi_sq = (double)chi_sq;
    J.delta = (double)sqrtf(chi_sq);
    J.num_iter = num_iter;
    J.fix_scale = fix_scale ? 1 : 0;
    J.num_inliers = num_inliers_out;
    J.rot_12 = rot_12_out;
    J.trans_12 = trans_12_out;
    J.scale_12 = scale_12_out;
    J.inlier = inlier_out;
    if (num_problems == 0) return;
    emu_launch(s3opt::sim3_opt_kernel, (unsigned)num_problems, (unsigned)s3opt::kThreads, J, num_problems);
}
