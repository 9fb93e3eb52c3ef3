// sim3_opt.cu -- optimize::transform_optimizer::optimize (optimize/transform_optimizer.cc:47-197) for P independent
// problems (sm_90a).
//
// One 128-thread CTA per problem runs both LM rounds, the outlier re-classifications and the inlier count in a single
// launch (sim3_opt_kernels.cuh).  The Sim3 algebra, the mutual reprojection errors and the numeric Jacobian come from
// sim3optmath.h, the text the oracle compiles.  FP64, compiled with -fmad=false.
#include <cmath>

#include "common.cuh"
#include "sim3_opt_kernels.cuh"

using namespace plp;

extern "C" {

plp_status plp_sim3_optimize(plp_ctx *ctx, int num_problems, const int32_t *match_offsets, const plp_camera *cams,
                             const double *rot_1w, const double *trans_1w, const double *rot_2w, const double *trans_2w,
                             const double *rot_12_in, const double *trans_12_in, const double *scale_12_in,
                             const double *pos_w_1, const double *pos_w_2, const float *obs_1, const float *obs_2,
                             const float *inv_sigma_sq_1, const float *inv_sigma_sq_2, float chi_sq, int num_iter,
                             int fix_scale, int32_t *num_inliers_out, double *rot_12_out, double *trans_12_out,
                             double *scale_12_out, uint8_t *inlier_out) {
    PLP_REQUIRE(ctx && match_offsets && num_inliers_out && rot_12_out && trans_12_out && scale_12_out, "null pointer");
    PLP_REQUIRE(num_problems >= 0 && num_iter >= 0, "sizes");
    PLP_REQUIRE(std::isfinite(chi_sq) && chi_sq > 0.0f, "chi_sq must be finite and positive");
    if (num_iter > s3opt::kMaxIter) {
        set_error("plp_sim3_optimize: num_iter %d exceeds %d", num_iter, s3opt::kMaxIter);
        return PLP_ERR_CAPACITY;
    }
    PLP_REQUIRE(match_offsets[0] == 0, "offsets start at 0");
    for (int p = 0; p < num_problems; ++p) PLP_REQUIRE(match_offsets[p + 1] >= match_offsets[p], "offsets are non-decreasing");
    const int N = match_offsets[num_problems];
    PLP_REQUIRE(num_problems == 0 || (cams && rot_1w && trans_1w && rot_2w && trans_2w && rot_12_in && trans_12_in &&
                                      scale_12_in),
                "null pointer");
    PLP_REQUIRE(N == 0 || (pos_w_1 && pos_w_2 && obs_1 && obs_2 && inv_sigma_sq_1 && inv_sigma_sq_2 && inlier_out),
                "null pointer");
    if (num_problems == 0) return PLP_OK;
    PLP_CUDA_TRY(cudaSetDevice(ctx->device));
    const size_t P = (size_t)num_problems, M = (size_t)N;
    std::vector<double> cam4(P * 4), pose_1(P * 12), pose_2(P * 12);  // the intrinsics the edges read; R | t per keyframe
    for (size_t p = 0; p < P; ++p) {
        cam4[4 * p] = cams[p].fx;
        cam4[4 * p + 1] = cams[p].fy;
        cam4[4 * p + 2] = cams[p].cx;
        cam4[4 * p + 3] = cams[p].cy;
        for (int k = 0; k < 9; ++k) {
            pose_1[12 * p + k] = rot_1w[9 * p + k];
            pose_2[12 * p + k] = rot_2w[9 * p + k];
        }
        for (int k = 0; k < 3; ++k) {
            pose_1[12 * p + 9 + k] = trans_1w[3 * p + k];
            pose_2[12 * p + 9 + k] = trans_2w[3 * p + k];
        }
    }
    DevLayout L;
    s3opt::Sim3OptJob J;
    L.in(J.offsets, match_offsets, P + 1);
    L.in(J.cams, cam4.data(), P * 4);
    L.in(J.pose_1w, pose_1.data(), P * 12);
    L.in(J.pose_2w, pose_2.data(), P * 12);
    L.in(J.rot_12_in, rot_12_in, P * 9);
    L.in(J.trans_12_in, trans_12_in, P * 3);
    L.in(J.scale_12_in, scale_12_in, P);
    L.in(J.pos_w_1, pos_w_1, M * 3);
    L.in(J.pos_w_2, pos_w_2, M * 3);
    L.in(J.obs_1, obs_1, M * 2);
    L.in(J.obs_2, obs_2, M * 2);
    L.in(J.inv_sigma_sq_1, inv_sigma_sq_1, M);
    L.in(J.inv_sigma_sq_2, inv_sigma_sq_2, M);
    J.chi_sq = (double)chi_sq;
    J.delta = (double)std::sqrt(chi_sq);  // transform_optimizer.cc:51, float
    J.num_iter = num_iter;
    J.fix_scale = fix_scale ? 1 : 0;
    L.out(J.num_inliers, P);
    L.out(J.rot_12, P * 9);
    L.out(J.trans_12, P * 3);
    L.out(J.scale_12, P);
    L.out(J.inlier, M + 1);
    PLP_TRY(stage(ctx, 0, L));
    PLP_LAUNCH(ctx, s3opt::sim3_opt_kernel, num_problems, s3opt::kThreads, 0, J, num_problems);
    PLP_CHECK_LAUNCH();
    PLP_CUDA_TRY(to_host(ctx, num_inliers_out, J.num_inliers, P));
    PLP_CUDA_TRY(to_host(ctx, rot_12_out, J.rot_12, P * 9));
    PLP_CUDA_TRY(to_host(ctx, trans_12_out, J.trans_12, P * 3));
    PLP_CUDA_TRY(to_host(ctx, scale_12_out, J.scale_12, P));
    if (M) PLP_CUDA_TRY(to_host(ctx, inlier_out, J.inlier, M));
    PLP_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return PLP_OK;
}

}  // extern "C"
