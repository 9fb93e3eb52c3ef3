// sim3.cu -- solve::sim3_solver::find_via_ransac (solve/sim3_solver.cc:121-191) for P independent problems (sm_90a).
//
// The constructor's same-image reprojections are computed once per problem.  Hypotheses are independent given their
// sample sets: one warp-sized CTA per (problem, hypothesis) solves Horn's method in one thread (sim3math.h -- the same
// text the oracle compiles, hence bit-identical) and counts the inliers across the warp.  One warp per problem then
// replays the reference's ordered best-model scan and writes the winner.  FP64, compiled with -fmad=false.
#include "common.cuh"
#include "sim3_kernels.cuh"

using namespace plp;

extern "C" {

plp_status plp_sim3_ransac(plp_ctx *ctx, int num_problems, const int32_t *corr_offsets, const plp_camera *cams,
                           const double *pts_1, const double *pts_2, const float *chi_sq_1, const float *chi_sq_2,
                           const int32_t *samples, int num_iter, int fix_scale, int min_num_inliers, int32_t *valid_out,
                           int32_t *num_inliers_out, double *rot_12_out, double *trans_12_out, float *scale_12_out) {
    PLP_REQUIRE(ctx && corr_offsets && valid_out && num_inliers_out && rot_12_out && trans_12_out && scale_12_out,
                "null pointer");
    PLP_REQUIRE(num_problems >= 0 && num_iter >= 0 && min_num_inliers >= 0, "sizes");
    if (num_iter > 65535) {  // the hypothesis grid's y extent
        set_error("plp_sim3_ransac: num_iter %d exceeds 65535", num_iter);
        return PLP_ERR_CAPACITY;
    }
    PLP_REQUIRE(corr_offsets[0] == 0, "offsets start at 0");
    bool any_runs = false;
    for (int p = 0; p < num_problems; ++p) {
        PLP_REQUIRE(corr_offsets[p + 1] >= corr_offsets[p], "offsets are non-decreasing");
        const int n = corr_offsets[p + 1] - corr_offsets[p];
        any_runs = any_runs || (n >= kSim3MinSet && n >= min_num_inliers);
    }
    const int N = corr_offsets[num_problems];
    PLP_REQUIRE(num_problems == 0 || cams, "null pointer");
    PLP_REQUIRE(N == 0 || (pts_1 && pts_2 && chi_sq_1 && chi_sq_2), "null pointer");
    PLP_REQUIRE(!any_runs || num_iter == 0 || samples, "samples");
    for (int p = 0; p < num_problems; ++p) {  // only the problems that run read their samples
        const int n = corr_offsets[p + 1] - corr_offsets[p];
        if (n < kSim3MinSet || n < min_num_inliers) continue;
        const int32_t *s = samples + (size_t)p * num_iter * kSim3MinSet;
        for (int k = 0; k < num_iter * kSim3MinSet; ++k) PLP_REQUIRE(s[k] >= 0 && s[k] < n, "sample index out of range");
    }
    if (!any_runs) {  // :130-134 for every problem
        for (int p = 0; p < num_problems; ++p) {
            valid_out[p] = num_inliers_out[p] = 0;
            memset(rot_12_out + 9 * (size_t)p, 0, sizeof(double) * 9);
            memset(trans_12_out + 3 * (size_t)p, 0, sizeof(double) * 3);
            scale_12_out[p] = 0.0f;
        }
        return PLP_OK;
    }
    PLP_CUDA_TRY(cudaSetDevice(ctx->device));
    const size_t P = (size_t)num_problems, K = (size_t)num_iter, M = (size_t)N;
    std::vector<double> cam4(P * 4);  // the intrinsics reproject_to_image reads
    for (size_t p = 0; p < P; ++p) {
        cam4[4 * p] = cams[p].fx;
        cam4[4 * p + 1] = cams[p].fy;
        cam4[4 * p + 2] = cams[p].cx;
        cam4[4 * p + 3] = cams[p].cy;
    }
    DevLayout L;
    Sim3Job J;
    L.in(J.offsets, corr_offsets, P + 1);
    L.in(J.cams, cam4.data(), P * 4);
    L.in(J.pts_1, pts_1, M * 3);
    L.in(J.pts_2, pts_2, M * 3);
    L.in(J.chi_sq_1, chi_sq_1, M);
    L.in(J.chi_sq_2, chi_sq_2, M);
    L.in(J.samples, samples, P * K * kSim3MinSet);
    J.num_problems = num_problems;
    J.num_iter = num_iter;
    J.fix_scale = fix_scale ? 1 : 0;
    J.min_num_inliers = min_num_inliers;
    L.out(J.reproj_1, M * 2);
    L.out(J.reproj_2, M * 2);
    L.out(J.hyp_Rt, P * K * 12);
    L.out(J.hyp_scale, P * K);
    L.out(J.hyp_count, P * K);
    L.out(J.valid, P);
    L.out(J.num_inliers, P);
    L.out(J.rot_12, P * 9);
    L.out(J.trans_12, P * 3);
    L.out(J.scale_12, P);
    PLP_TRY(stage(ctx, 0, L));
    if (num_iter > 0) {
        PLP_LAUNCH(ctx, sim3_reproject_kernel, num_problems, kSim3PrepThreads, 0, J);
        PLP_CHECK_LAUNCH();
        PLP_LAUNCH(ctx, sim3_hypothesis_kernel, dim3(num_problems, num_iter), kSim3Threads, 0, J);
        PLP_CHECK_LAUNCH();
    }
    PLP_LAUNCH(ctx, sim3_select_kernel, num_problems, kSim3Threads, 0, J);
    PLP_CHECK_LAUNCH();
    PLP_CUDA_TRY(to_host(ctx, valid_out, J.valid, P));
    PLP_CUDA_TRY(to_host(ctx, num_inliers_out, J.num_inliers, P));
    PLP_CUDA_TRY(to_host(ctx, rot_12_out, J.rot_12, P * 9));
    PLP_CUDA_TRY(to_host(ctx, trans_12_out, J.trans_12, P * 3));
    PLP_CUDA_TRY(to_host(ctx, scale_12_out, J.scale_12, P));
    PLP_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return PLP_OK;
}

}  // extern "C"
