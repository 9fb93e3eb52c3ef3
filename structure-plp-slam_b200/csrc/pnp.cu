// pnp.cu -- solve::pnp_solver::find_via_ransac (solve/pnp_solver.cc:70-153) for P independent problems (sm_90a).
//
// Hypotheses are independent given their sample sets: one warp-sized CTA per (problem, hypothesis) solves the minimal
// EPnP in one thread (pnpmath.h -- the same text the oracle compiles, hence bit-identical) and counts the inliers across the CTA.
// One CTA per problem then replays the reference's ordered best-model scan, writes the winner's flags and, for a valid
// problem, optionally recomputes the pose over the inliers (M^T M summed one entry per thread).  FP64, compiled with
// -fmad=false.
#include "common.cuh"
#include "pnp_kernels.cuh"

using namespace plp;

extern "C" {

plp_status plp_pnp_ransac(plp_ctx *ctx, int num_problems, const int32_t *corr_offsets, const double *bearings,
                          const double *pos_w, const float *max_cos_error, const int32_t *samples, int num_iter,
                          int min_num_inliers, int recompute, int32_t *valid_out, int32_t *num_inliers_out,
                          double *pose_cw_out, uint8_t *is_inlier_out) {
    PLP_REQUIRE(ctx && corr_offsets && valid_out && num_inliers_out && pose_cw_out, "null pointer");
    PLP_REQUIRE(num_problems >= 0 && num_iter >= 0 && min_num_inliers >= 0, "sizes");
    if (num_iter > 65535) {  // the hypothesis grid's y extent
        set_error("plp_pnp_ransac: num_iter %d exceeds 65535", num_iter);
        return PLP_ERR_CAPACITY;
    }
    PLP_REQUIRE(corr_offsets[0] == 0, "offsets start at 0");
    bool any_runs = false;
    for (int p = 0; p < num_problems; ++p) {
        PLP_REQUIRE(corr_offsets[p + 1] >= corr_offsets[p], "offsets are non-decreasing");
        const int n = corr_offsets[p + 1] - corr_offsets[p];
        any_runs = any_runs || (n >= kPnpMinSet && n >= min_num_inliers);
    }
    const int N = corr_offsets[num_problems];
    PLP_REQUIRE(N == 0 || (bearings && pos_w && max_cos_error && is_inlier_out), "null pointer");
    PLP_REQUIRE(!any_runs || num_iter == 0 || samples, "samples");
    for (int p = 0; p < num_problems; ++p) {  // only the problems that run read their samples
        const int n = corr_offsets[p + 1] - corr_offsets[p];
        if (n < kPnpMinSet || n < min_num_inliers) continue;
        const int32_t *s = samples + (size_t)p * num_iter * kPnpMinSet;
        for (int k = 0; k < num_iter * kPnpMinSet; ++k) PLP_REQUIRE(s[k] >= 0 && s[k] < n, "sample index out of range");
    }
    if (!any_runs) {  // :76-80 for every problem
        for (int p = 0; p < num_problems; ++p) valid_out[p] = num_inliers_out[p] = 0;
        return PLP_OK;
    }
    PLP_CUDA_TRY(cudaSetDevice(ctx->device));
    const size_t P = (size_t)num_problems, K = (size_t)num_iter, M = (size_t)N;
    DevLayout L;
    PnpJob J;
    L.in(J.offsets, corr_offsets, P + 1);
    L.in(J.bearings, bearings, M * 3);
    L.in(J.pos_w, pos_w, M * 3);
    L.in(J.max_cos, max_cos_error, M);
    L.in(J.samples, samples, P * K * kPnpMinSet);
    J.num_problems = num_problems;
    J.num_iter = num_iter;
    J.min_num_inliers = min_num_inliers;
    J.recompute = recompute ? 1 : 0;
    L.out(J.hyp_Rt, P * K * 12);
    L.out(J.hyp_count, P * K);
    L.out(J.pws, recompute ? M * 3 : 0);
    L.out(J.us, recompute ? M * 2 : 0);
    L.out(J.alphas, recompute ? M * 4 : 0);
    L.out(J.pcs, recompute ? M * 3 : 0);
    L.out(J.signs, recompute ? M : 0);
    L.out(J.valid, P);
    L.out(J.num_inliers, P);
    L.out(J.pose, P * 16);
    L.out(J.is_inlier, M);
    PLP_TRY(stage(ctx, 0, L));
    if (num_iter > 0) {
        PLP_LAUNCH(ctx, pnp_hypothesis_kernel, dim3(num_problems, num_iter), kPnpHypThreads, 0, J);
        PLP_CHECK_LAUNCH();
    }
    PLP_LAUNCH(ctx, pnp_select_kernel, num_problems, kPnpThreads, 0, J);
    PLP_CHECK_LAUNCH();
    std::vector<double> pose(P * 16);
    std::vector<uint8_t> flags(M);
    PLP_CUDA_TRY(to_host(ctx, valid_out, J.valid, P));
    PLP_CUDA_TRY(to_host(ctx, num_inliers_out, J.num_inliers, P));
    PLP_CUDA_TRY(to_host(ctx, pose.data(), J.pose, P * 16));
    PLP_CUDA_TRY(to_host(ctx, flags.data(), J.is_inlier, M));
    PLP_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    // nothing but valid / num_inliers for a problem that did not run; the pose only for a valid one
    for (int p = 0; p < num_problems; ++p) {
        const int off = corr_offsets[p], n = corr_offsets[p + 1] - off;
        if (n < kPnpMinSet || n < min_num_inliers) continue;
        memcpy(is_inlier_out + off, flags.data() + off, (size_t)n);
        if (valid_out[p]) memcpy(pose_cw_out + 16 * (size_t)p, pose.data() + 16 * (size_t)p, sizeof(double) * 16);
    }
    return PLP_OK;
}

}  // extern "C"
