// sim3_opt_kernels.cuh -- device code of the batched Sim3 optimiser (sim3_opt.cu launches it).  Free of host-side CUDA
// runtime dependencies so that tests/cta_emu can compile the same text for the host.
//
// optimize::transform_optimizer::optimize (optimize/transform_optimizer.cc:47-197): the g2o graph {1 Sim3 vertex, a
// forward and a backward reprojection edge per valid match, Huber delta = sqrt(chi_sq)} solved with
// OptimizationAlgorithmLevenberg; optimize(5), chi-square re-classification of both edges of every match, the "fewer than
// 10 survivors" return, optimize(num_iter) over the survivors, and the final inlier count.
//
// ONE 128-THREAD CTA PER PROBLEM, the whole optimize() in one launch, shaped like pose_opt_kernels.cuh:
//   * threads stride the matches; per match, both edges' errors and 2 x 7 numeric Jacobians in FP64 (sim3optmath.h, the
//     text the oracle compiles), 36 accumulators per thread (28 upper H, 7 b, 1 robust chi2), summed by a shuffle butterfly
//     per warp and a double-buffered shared-memory exchange between the 4 warps (one barrier), so every thread ends up with
//     the same totals in the same order;
//   * every thread runs the 7 x 7 Cholesky, the Sim3 exponential and the LM bookkeeping redundantly on identical inputs;
//   * the 14 estimates linearizeOplus visits (oplus(+-1e-9 e_d)) and their inverses are the same for every edge of one
//     buildSystem: 28 threads compute them once per LM iteration into shared memory, instead of once per edge as g2o does;
//     each edge's error and Jacobian arithmetic is unchanged;
//   * per-match state is only the g2o level, kept in the caller's inlier array (1 = level 0).  The chi2 an edge carries into
//     a re-classification is that of the LAST EVALUATED estimate -- also after a rejected step, as g2o's pop() does not
//     recompute -- and is recomputed from that estimate, which every thread holds.
// Every problem runs the same barrier sequence for its own iteration counts: a problem with no matches, or one that
// returns after round 1, takes the same path with empty strides, so nothing diverges around a __syncthreads().
#pragma once
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#include "sim3optmath.h"

namespace plp {

namespace s3opt {

constexpr int kWarps = 4;  // warps per problem (one CTA = one problem)
constexpr int kThreads = 32 * kWarps;
constexpr int kRed = 36;          // 28 (upper H) + 7 (b) + 1 (chi2)
constexpr int kMaxIter = 1000;    // num_iter cap (plp_sim3_optimize): bounds one CTA's running time
constexpr int kRound1Iter = 5;    // transform_optimizer.cc:132
constexpr int kMinSurvivors = 10; // :158

struct Sim3OptJob {
    const int32_t *offsets;   // P + 1
    const double *cams;       // P x 4 (fx, fy, cx, cy)
    const double *pose_1w;    // P x 12 (rot row-major, trans)
    const double *pose_2w;    // P x 12
    const double *rot_12_in;  // P x 9
    const double *trans_12_in;
    const double *scale_12_in;
    const double *pos_w_1;  // N x 3
    const double *pos_w_2;  // N x 3
    const float *obs_1;     // N x 2
    const float *obs_2;
    const float *inv_sigma_sq_1;  // N
    const float *inv_sigma_sq_2;
    double chi_sq;  // the float chi_sq as double
    double delta;   // sqrt_chi_sq (float sqrt) as double
    int num_iter;
    int fix_scale;
    int32_t *num_inliers;  // P
    double *rot_12;        // P x 9
    double *trans_12;      // P x 3
    double *scale_12;      // P
    uint8_t *inlier;       // N
};

struct Shared {
    double red[2][kWarps][kRed];  // per-warp partial sums of (H, b, chi2), double-buffered: one barrier per reduction
    double redc[2][kWarps];       // per-warp partial robust chi2 of a trial estimate
    s3o_sim3 fwd[14];             // the 14 estimates linearizeOplus visits (forward edges)
    s3o_sim3 bwd[14];             // their inverses (backward edges)
    double pose[24];              // rot_1w, trans_1w, rot_2w, trans_2w
    double cam[4];
    int cnt[2][kWarps];
};

__device__ __forceinline__ double warp_allsum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ int warp_allsum_int(int v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ double sumH(const Shared &S, int hp, int k) {
    double a = S.red[hp][0][k];
#pragma unroll
    for (int w = 1; w < kWarps; ++w) a += S.red[hp][w][k];
    return a;
}

// (H + lambda I) x = b by Cholesky in registers, with g2o_lite::cholesky_solve's operation order (divisions by the
// pivots); H is the upper triangle packed row-wise.  On failure x is left as it came (zeros), as cholesky_solve does.
__device__ __forceinline__ bool solve7(const Shared &S, int hp, double lambda, double *x) {
    double A[7][7], b[7];
    {
        int k = 0;
#pragma unroll
        for (int i = 0; i < 7; ++i)
#pragma unroll
            for (int j = i; j < 7; ++j) {
                A[j][i] = sumH(S, hp, k);  // lower triangle
                ++k;
            }
#pragma unroll
        for (int i = 0; i < 7; ++i) b[i] = sumH(S, hp, 28 + i);
    }
    bool ok = true;
#pragma unroll
    for (int j = 0; j < 7; ++j) {
        double d = A[j][j] + lambda;
#pragma unroll
        for (int q = 0; q < j; ++q) d -= A[j][q] * A[j][q];
        if (!(d > 0.0) || !isfinite(d)) ok = false;
        d = sqrt(d);
        A[j][j] = d;
#pragma unroll
        for (int i = j + 1; i < 7; ++i) {
            double s = A[i][j];
#pragma unroll
            for (int q = 0; q < j; ++q) s -= A[i][q] * A[j][q];
            A[i][j] = s / d;
        }
    }
    if (!ok) return false;
    double y[7];
#pragma unroll
    for (int i = 0; i < 7; ++i) {
        double s = b[i];
#pragma unroll
        for (int q = 0; q < i; ++q) s -= A[i][q] * y[q];
        y[i] = s / A[i][i];
    }
#pragma unroll
    for (int i = 6; i >= 0; --i) {
        double s = y[i];
#pragma unroll
        for (int q = i + 1; q < 7; ++q) s -= A[q][i] * x[q];
        x[i] = s / A[i][i];
    }
    return true;
}

// one match's camera-frame points and measurements
struct Match {
    double pc_2[3], pc_1[3];
    double obs_1[2], obs_2[2];
    double w_1, w_2;
};

__device__ __forceinline__ Match load_match(const Sim3OptJob &J, const Shared &S, size_t g) {
    Match m;
    const double X2[3] = {__ldg(&J.pos_w_2[3 * g]), __ldg(&J.pos_w_2[3 * g + 1]), __ldg(&J.pos_w_2[3 * g + 2])};
    const double X1[3] = {__ldg(&J.pos_w_1[3 * g]), __ldg(&J.pos_w_1[3 * g + 1]), __ldg(&J.pos_w_1[3 * g + 2])};
    s3o_to_cam(S.pose + 12, S.pose + 21, X2, m.pc_2);
    s3o_to_cam(S.pose, S.pose + 9, X1, m.pc_1);
    m.obs_1[0] = (double)__ldg(&J.obs_1[2 * g]);
    m.obs_1[1] = (double)__ldg(&J.obs_1[2 * g + 1]);
    m.obs_2[0] = (double)__ldg(&J.obs_2[2 * g]);
    m.obs_2[1] = (double)__ldg(&J.obs_2[2 * g + 1]);
    m.w_1 = (double)__ldg(&J.inv_sigma_sq_1[g]);
    m.w_2 = (double)__ldg(&J.inv_sigma_sq_2[g]);
    return m;
}

// constructQuadraticForm of one edge with its Huber weight: H += J^T w J (upper), b -= J^T w e, chi += rho(chi2)
__device__ __forceinline__ void accumulate(const double *Jm, const double *e, double w, double delta, double *acc) {
    const double chi2 = s3o_chi2(e, w);
    double rho0, rho1;
    se3::huber(chi2, delta, rho0, rho1);
    acc[35] += rho0;
    const double ww = w * rho1;
    int k = 0;
#pragma unroll
    for (int a = 0; a < 7; ++a) {
        const double wa = ww * Jm[a], wb = ww * Jm[7 + a];
#pragma unroll
        for (int c = a; c < 7; ++c) {
            acc[k] += wa * Jm[c] + wb * Jm[7 + c];
            ++k;
        }
        acc[28 + a] -= wa * e[0] + wb * e[1];
    }
}

// robust chi2 of both edges of one match at (S12, S21 = S12.inverse())
__device__ __forceinline__ double robust_pair(const Shared &S, const Match &m, const s3o_sim3 &S12, const s3o_sim3 &S21,
                                              double delta) {
    double e[2], rho0, rho1;
    s3o_error(S.cam, S12, m.pc_2, m.obs_1, e);
    se3::huber(s3o_chi2(e, m.w_1), delta, rho0, rho1);
    double chi = rho0;
    s3o_error(S.cam, S21, m.pc_1, m.obs_2, e);
    se3::huber(s3o_chi2(e, m.w_2), delta, rho0, rho1);
    return chi + rho0;
}

// SparseOptimizer::optimize(iterations) with OptimizationAlgorithmLevenberg over the level-0 matches; est is replicated in
// every thread, last_eval receives the estimate the edge errors were last computed at.
__device__ __forceinline__ void optimize(const Sim3OptJob &J, Shared &S, int off, int n, int iterations, s3o_sim3 &est,
                                         s3o_sim3 &last_eval, int &hp, int &cp) {
    const int tid = threadIdx.x;
    const uint8_t *level0 = J.inlier + off;
    double lambda = 0, ni = 2;
    for (int it = 0; it < iterations; ++it) {
        // the 14 visited estimates of linearizeOplus at this iteration's estimate; their last readers (the previous
        // buildSystem) are behind the previous reduction's barrier
        if (tid < 28) {
            const s3o_sim3 v = s3o_perturbed(est, tid % 14, J.fix_scale);
            if (tid < 14)
                S.fwd[tid] = v;
            else
                S.bwd[tid - 14] = s3o_inverse(v);
        }
        __syncthreads();
        // computeActiveErrors + buildSystem at the current estimate
        const s3o_sim3 est_inv = s3o_inverse(est);
        double acc[kRed];
#pragma unroll
        for (int k = 0; k < kRed; ++k) acc[k] = 0;
#pragma unroll 1
        for (int i = tid; i < n; i += kThreads) {
            if (!level0[i]) continue;
            const Match m = load_match(J, S, (size_t)off + i);
            double e[2], Jm[14];
            s3o_error(S.cam, est, m.pc_2, m.obs_1, e);
            s3o_numeric_jacobian(S.cam, S.fwd, m.pc_2, m.obs_1, Jm);
            accumulate(Jm, e, m.w_1, J.delta, acc);
            s3o_error(S.cam, est_inv, m.pc_1, m.obs_2, e);
            s3o_numeric_jacobian(S.cam, S.bwd, m.pc_1, m.obs_2, Jm);
            accumulate(Jm, e, m.w_2, J.delta, acc);
        }
        hp ^= 1;
#pragma unroll
        for (int k = 0; k < kRed; ++k) {
            const double v = warp_allsum(acc[k]);
            if ((tid & 31) == 0) S.red[hp][tid >> 5][k] = v;
        }
        __syncthreads();
        last_eval = est;
        double current_chi = sumH(S, hp, 35);
        if (it == 0) {  // computeLambdaInit: tau * max diag(H)
            double md = 0;
            const int diag[7] = {0, 7, 13, 18, 22, 25, 27};
#pragma unroll
            for (int j = 0; j < 7; ++j) md = fmax(fabs(sumH(S, hp, diag[j])), md);
            lambda = 1e-5 * md;
            ni = 2;
        }
        int qmax = 0;
        bool terminate = false;
        // Levenberg inner loop (<= 10 tries)
        while (true) {
            double x[7] = {0, 0, 0, 0, 0, 0, 0};
            const bool ok2 = solve7(S, hp, lambda, x);
            const s3o_sim3 trial = s3o_oplus(est, x, J.fix_scale);  // zeroes x[6] when fix_scale, as the reference
            const s3o_sim3 trial_inv = s3o_inverse(trial);
            double chi = 0;
#pragma unroll 1
            for (int i = tid; i < n; i += kThreads) {
                if (!level0[i]) continue;
                chi += robust_pair(S, load_match(J, S, (size_t)off + i), trial, trial_inv, J.delta);
            }
            cp ^= 1;
            chi = warp_allsum(chi);
            if ((tid & 31) == 0) S.redc[cp][tid >> 5] = chi;
            __syncthreads();
            last_eval = trial;  // the edge errors stay those of this estimate even if the step is rejected (pop())
            double temp_chi = S.redc[cp][0];
#pragma unroll
            for (int w = 1; w < kWarps; ++w) temp_chi += S.redc[cp][w];
            if (!ok2) temp_chi = 1.7976931348623157e308;
            double rho = current_chi - temp_chi;
            double scale = 0;
#pragma unroll
            for (int j = 0; j < 7; ++j) scale += x[j] * (lambda * x[j] + sumH(S, hp, 28 + j));
            scale += 1e-3;
            rho /= scale;
            bool lambda_finite = true;
            if (rho > 0 && isfinite(temp_chi)) {
                double alpha = 1. - pow((2 * rho - 1), 3);
                alpha = fmin(alpha, 2. / 3.);
                const double sf = fmax(1. / 3., alpha);
                lambda *= sf;
                ni = 2;
                current_chi = temp_chi;
                est = trial;
            } else {
                lambda *= ni;
                ni *= 2;
                if (!isfinite(lambda)) lambda_finite = false;
            }
            if (lambda_finite) qmax++;
            terminate = (qmax == 10 || rho == 0 || !lambda_finite);
            if (!(lambda_finite && rho < 0 && qmax < 10)) break;
        }
        if (terminate) break;
    }
}

__global__ void __launch_bounds__(kThreads, 1) sim3_opt_kernel(Sim3OptJob J, int num_problems) {
    __shared__ Shared S;
    const int tid = threadIdx.x;
    const int p = blockIdx.x;
    if (p >= num_problems) return;
    const int off = J.offsets[p], n = J.offsets[p + 1] - off;
    uint8_t *level0 = J.inlier + off;  // thread t only ever touches the matches t, t + kThreads, ...
    if (tid < 12) {
        S.pose[tid] = J.pose_1w[12 * (size_t)p + tid];
        S.pose[12 + tid] = J.pose_2w[12 * (size_t)p + tid];
    }
    if (tid < 4) S.cam[tid] = J.cams[4 * (size_t)p + tid];
    for (int i = tid; i < n; i += kThreads) level0[i] = 1;
    // g2o::Sim3(R, t, s) of the caller's estimate, replicated in every thread
    s3o_sim3 est = s3o_from_Rts(J.rot_12_in + 9 * (size_t)p, J.trans_12_in + 3 * (size_t)p, J.scale_12_in[p]);
    s3o_sim3 last_eval = est;
    int hp = 0, cp = 0;
    __syncthreads();  // S.pose, S.cam
    // 3. optimize(5) over every match
    optimize(J, S, off, n, kRound1Iter, est, last_eval, hp, cp);
    // 4. outliers: either edge fails chi2 < chi_sq at the last evaluated estimate
    {
        const s3o_sim3 inv = s3o_inverse(last_eval);
        int bad = 0;
#pragma unroll 1
        for (int i = tid; i < n; i += kThreads) {
            const Match m = load_match(J, S, (size_t)off + i);
            double e12[2], e21[2];
            s3o_error(S.cam, last_eval, m.pc_2, m.obs_1, e12);
            s3o_error(S.cam, inv, m.pc_1, m.obs_2, e21);
            if (s3o_chi2(e12, m.w_1) < J.chi_sq && s3o_chi2(e21, m.w_2) < J.chi_sq) continue;
            level0[i] = 0;
            ++bad;
        }
        bad = warp_allsum_int(bad);
        if ((tid & 31) == 0) S.cnt[0][tid >> 5] = bad;
        __syncthreads();
        int num_outliers = 0;
#pragma unroll
        for (int w = 0; w < kWarps; ++w) num_outliers += S.cnt[0][w];
        if (n - num_outliers < kMinSurvivors) {  // return 0: the caller's Sim3 is untouched (uniform across the CTA)
            if (tid < 9) J.rot_12[9 * (size_t)p + tid] = J.rot_12_in[9 * (size_t)p + tid];
            if (tid < 3) J.trans_12[3 * (size_t)p + tid] = J.trans_12_in[3 * (size_t)p + tid];
            if (tid == 0) {
                J.scale_12[p] = J.scale_12_in[p];
                J.num_inliers[p] = 0;
            }
            return;
        }
    }
    // 5. optimize(num_iter) over the level-0 matches
    optimize(J, S, off, n, J.num_iter, est, last_eval, hp, cp);
    // 6. inliers: level-0 matches with neither chi_sq < chi2 (a NaN chi2 stays an inlier, as in the reference)
    const s3o_sim3 inv = s3o_inverse(last_eval);
    int good = 0;
#pragma unroll 1
    for (int i = tid; i < n; i += kThreads) {
        if (!level0[i]) continue;
        const Match m = load_match(J, S, (size_t)off + i);
        double e12[2], e21[2];
        s3o_error(S.cam, last_eval, m.pc_2, m.obs_1, e12);
        s3o_error(S.cam, inv, m.pc_1, m.obs_2, e21);
        if (J.chi_sq < s3o_chi2(e12, m.w_1) || J.chi_sq < s3o_chi2(e21, m.w_2)) {
            level0[i] = 0;
            continue;
        }
        ++good;
    }
    good = warp_allsum_int(good);
    if ((tid & 31) == 0) S.cnt[1][tid >> 5] = good;
    __syncthreads();
    // 7. the estimate
    if (tid == 0) {
        int num_inliers = 0;
#pragma unroll
        for (int w = 0; w < kWarps; ++w) num_inliers += S.cnt[1][w];
        J.num_inliers[p] = num_inliers;
        s3o_quat_to_R(est.q, J.rot_12 + 9 * (size_t)p);
        J.trans_12[3 * (size_t)p] = est.t[0];
        J.trans_12[3 * (size_t)p + 1] = est.t[1];
        J.trans_12[3 * (size_t)p + 2] = est.t[2];
        J.scale_12[p] = est.s;
    }
}

}  // namespace s3opt

}  // namespace plp
