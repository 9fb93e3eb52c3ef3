// local_ba.cu -- Schur-complement Levenberg-Marquardt local bundle adjustment on sm_90a (FP64).
//
// Replaces optimize::local_bundle_adjuster::optimize (optimize/local_bundle_adjuster.cc:160-410),
// local_bundle_adjuster_extended_line::optimize (optimize/local_bundle_adjuster_extended_line.cc:190-640) and
// local_bundle_adjuster_extended_plane::optimize (optimize/local_bundle_adjuster_extended_plane.cc:300-430) from
// the point where the graph has been gathered: SE3 keyframe vertices (some fixed), marginalised point (3-dof,
// additive) and line (4-dof orthonormal Pluecker) landmark vertices, one binary reprojection edge per observation
// (Huber in the first optimize(5), none in the second optimize(10), outliers = chi2 > 5.991|7.815 or depth <= 0),
// optional unary point-to-plane edges.  g2o's BlockSolver + OptimizationAlgorithmLevenberg are restated.
//
// Work decomposition (one LM "try" = 5 kernels, no host synchronisation inside an optimize() chunk):
//   ba_decide_kernel   1 CTA    accept/reject of the previous try (rho test), lambda / nu update, iteration count
//   ba_linearize_kernel G CTAs  landmark-sharded: one warp per landmark evaluates its edges (residual, Jacobians,
//                               Huber weight), forms Hll, bl, (Hll+lambda I)^-1 and the per-edge blocks
//                               W = Hpl, Y = W Dinv; the CTA then accumulates its share of the reduced camera
//                               system S = Hpp - sum_l Hpl Dinv Hpl^T in SHARED MEMORY WITHOUT ATOMICS: every thread
//                               owns a fixed set of S entries and loops over the landmarks of the batch
//                               (deterministic summation order)
//   ba_reduce_kernel   n CTAs   sums the G per-CTA partial systems into the packed vector
//                               [S upper blocks | g | bp | chi2 | max-diag slots]   <- the ONLY data a multi-GPU run
//                               exchanges: one ncclAllReduce(sum) of this vector per try (ba_nccl.cu)
//   ba_solve_kernel    1 CTA    dense Cholesky of the 6N x 6N reduced system in shared memory, dp, trial poses
//   ba_update_kernel   G CTAs   back-substitution dl = Dinv (bl - W^T dp), trial landmarks, errors at the trial
//                               state (kept even if the step is rejected, like g2o), chi2 / scale partial sums; the CTA
//                               that finishes last adds the partials up (fixed order)
// Linearisation is recomputed on every try (also after a rejection) instead of being cached: the numbers are
// identical and it removes all bookkeeping.  Numeric Jacobians (delta = 1e-9 central differences) are used where
// the reference has no linearizeOplus (line edges, plane edges), see g2o BaseBinaryEdge::linearizeOplus.
#include "common.cuh"
#include "se3.cuh"
#include "ba_kernels.cuh"
#include "ba_lm_kernels.cuh"

namespace plp {

namespace {

using namespace balm;

}  // namespace

size_t ba_linearize_smem(int n_free, int n_pairs, int pool_cap) {
    const bool large = n_free > kBaMaxFree;  // large path: the reduced system is in HBM, not in the CTA
    return ((sizeof(BaSmem) + 15) & ~(size_t)15) + (size_t)pool_cap * sizeof(BaPoolEntry) +
           (large ? 0 : (size_t)(n_pairs * 36 + 12 * n_free) * 8) + 64;
}
// pool entries per batch: enough for kBaWarps landmarks of the maximum free degree if the 227 KB of shared memory allow
int ba_pool_capacity(int n_free, int n_pairs, int max_free_degree) {
    const size_t budget = 227 * 1024;
    const size_t fixed = ba_linearize_smem(n_free, n_pairs, 0);
    const int fit = fixed < budget ? (int)((budget - fixed) / sizeof(BaPoolEntry)) : 0;
    const int want = n_free > kBaMaxFree ? kBaWarps * max_free_degree : std::min(kBaWarps * max_free_degree, kPoolMax);
    return std::max(max_free_degree, std::min(want, fit));
}
size_t ba_solve_smem(int n_free) {
    const size_t n = 6 * (size_t)n_free;
    return (n * (n + 1) / 2 + 2 * n + 21 * (size_t)n_free) * 8 + 64;
}

plp_status ba_prepare_kernels(int n_free, int n_pairs, int pool_cap) {
    if (n_free > kBaMaxFree) {
        PLP_SMEM_OPTIN(ba_linearize_kernel<true>, ba_linearize_smem(n_free, n_pairs, pool_cap));
        PLP_SMEM_OPTIN(ba_update_kernel, (size_t)6 * n_free * 8);
        return PLP_OK;
    }
    PLP_SMEM_OPTIN(ba_linearize_kernel<false>, ba_linearize_smem(n_free, n_pairs, pool_cap));
    PLP_SMEM_OPTIN(ba_solve_kernel, ba_solve_smem(n_free));
    return PLP_OK;
}

// one LM try on the context stream; `between` (may be null) is called where the multi-GPU path all-reduces
// ba_decide_kernel also refreshes the 12 perturbed poses per keyframe (one se3::oplus each): one thread per pose
static int ba_decide_threads(const BaDev &B) { return std::max(64, std::min(512, (B.n_kf * 12 + 31) / 32 * 32)); }

plp_status ba_launch_try(plp_ctx *ctx, const BaDev &B, BaCollective *coll) {
    PLP_LAUNCH(ctx, ba_decide_kernel, 1, ba_decide_threads(B), 0, B);
    if (B.large) {
        // every landmark adds its blocks to the packed system in HBM with FP64 atomics: start from zero
        PLP_CUDA_TRY(cudaMemsetAsync(B.packed, 0, (size_t)(B.packed_sum_len + B.world) * sizeof(double), ctx->stream));
        PLP_LAUNCH(ctx, ba_linearize_kernel<true>, B.num_ctas, kBaThreads, ba_linearize_smem(B.n_free, B.n_pairs, B.pool_cap), B);
    } else {
        PLP_LAUNCH(ctx, ba_linearize_kernel<false>, B.num_ctas, kBaThreads, ba_linearize_smem(B.n_free, B.n_pairs, B.pool_cap), B);
        PLP_LAUNCH(ctx, ba_reduce_kernel, div_up((B.packed_sum_len + 1) * kReduceLanes, 256), 256, 0, B);
    }
    if (coll) PLP_TRY(coll->all_reduce(B.packed, B.packed_sum_len + B.world));
    if (B.large)
        PLP_TRY(ba_launch_solve_large(ctx, B));
    else
        PLP_LAUNCH(ctx, ba_solve_kernel, 1, kSolveThreads, ba_solve_smem(B.n_free), B);
    PLP_LAUNCH(ctx, ba_update_kernel, B.num_ctas, kBaThreads, (size_t)6 * B.n_free * sizeof(double), B);
    if (coll) PLP_TRY(coll->all_reduce(B.trial_sum, 2));
    PLP_CHECK_LAUNCH();
    return PLP_OK;
}

plp_status ba_launch_decide(plp_ctx *ctx, const BaDev &B) {
    PLP_LAUNCH(ctx, ba_decide_kernel, 1, ba_decide_threads(B), 0, B);
    PLP_CHECK_LAUNCH();
    return PLP_OK;
}
plp_status ba_launch_set_state(plp_ctx *ctx, const BaDev &B, int max_it, int robust, int reset_cur) {
    PLP_LAUNCH(ctx, ba_set_state_kernel, 1, 1, 0, B, max_it, robust, reset_cur);
    PLP_CHECK_LAUNCH();
    return PLP_OK;
}
plp_status ba_launch_classify(plp_ctx *ctx, const BaDev &B, int set_levels) {
    const int n = B.n_pt_edges + B.n_ln_edges;
    if (n > 0) PLP_LAUNCH(ctx, ba_classify_kernel, div_up(n, 256), 256, 0, B, set_levels);
    PLP_CHECK_LAUNCH();
    return PLP_OK;
}
plp_status ba_launch_init_poses(plp_ctx *ctx, const BaDev &B, const double *d_T_in) {
    PLP_LAUNCH(ctx, ba_init_poses_kernel, div_up(B.n_kf, 64), 64, 0, B, d_T_in);
    PLP_CHECK_LAUNCH();
    return PLP_OK;
}
plp_status ba_launch_export(plp_ctx *ctx, const BaDev &B, double *d_T_out, double *d_pts_out, double *d_lines_out) {
    int n = B.n_kf;
    n = max(n, 3 * B.n_pts);
    n = max(n, 6 * B.n_lines);
    PLP_LAUNCH(ctx, ba_export_kernel, div_up(n, 256), 256, 0, B, d_T_out, d_pts_out, d_lines_out);
    PLP_CHECK_LAUNCH();
    return PLP_OK;
}

}  // namespace plp
