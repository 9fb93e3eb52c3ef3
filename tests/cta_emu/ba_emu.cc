// ba_emu.cc -- csrc/ba_lm_kernels.cuh (Schur-complement Levenberg-Marquardt bundle adjustment: decide / linearize / reduce /
// solve / update / classify kernels) executed on the host.  The harness restates what ba_host.cu does around the kernels
// (CSR offsets, cost-balanced landmark ranges, the LM try loop, the two optimize() phases of local BA) with plain host
// memory, so whole solves can be compared with the oracle on a machine without a GPU.
#include "cta_emu.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "ba_lm_kernels.cuh"

using namespace plp;
using namespace plp::balm;

namespace {
size_t linearize_smem(int n_free, int n_pairs, int pool_cap) {
    return ((sizeof(BaSmem) + 15) & ~(size_t)15) + (size_t)pool_cap * sizeof(BaPoolEntry) + (size_t)(n_pairs * 36 + 12 * n_free) * 8 + 64;
}
size_t solve_smem(int n_free) {
    const size_t n = 6 * (size_t)n_free;
    return (n * (n + 1) / 2 + 2 * n + 21 * (size_t)n_free) * 8 + 64;
}
unsigned div_up_u(size_t a, size_t b) { return (unsigned)((a + b - 1) / b); }
// read-back of the first real try of the next emu_ba_solve (what plp_ba_debug_try downloads on the GPU)
double *g_cap_packed = nullptr, *g_cap_dp = nullptr, *g_cap_lambda = nullptr;
}  // namespace

// The next emu_ba_solve copies out, after its second try (the first after the lambda initialisation) and before that try's
// accept / reject decision: packed [S upper blocks | g | bp | chi2] (n_pairs * 36 + 12 n_free + 1), dp (6 n_free), lambda.
extern "C" void emu_ba_capture_try(double *packed, double *dp, double *lambda) {
    g_cap_packed = packed;
    g_cap_dp = dp;
    g_cap_lambda = lambda;
}

// mode 0: local BA (optimize(first) with Huber, classification, optimize(second) without, classification);
// mode 1 / 2: one optimize(first) with / without the Huber kernel (global BA).  num_ctas: landmark shards (CTAs) to emulate.
extern "C" int emu_ba_solve(double fx, double fy, double cx, double cy, double bf, int setup_type, int n_kf, const double *kf_pose_cw,
                            const uint8_t *kf_fixed, int n_pts, const double *pt_pos_w, int n_pe, const int32_t *pt_edge_kf,
                            const int32_t *pt_edge_lm, const float *pt_edge_obs, const float *pt_edge_info, int n_lines,
                            const double *line_plucker, int n_le, const int32_t *line_edge_kf, const int32_t *line_edge_lm,
                            const float *line_edge_obs, const float *line_edge_info, int n_plane_edges, const int32_t *plane_edge_lm,
                            const double *plane_edge_fn, int num_first, int num_second, int mode, int num_ctas, double *kf_out,
                            double *pts_out, double *lines_out, uint8_t *pt_outlier_out, uint8_t *ln_outlier_out, int32_t *iters_out) {
    std::vector<int> hidx(n_kf, -1);
    int n_free = 0;
    for (int k = 0; k < n_kf; ++k)
        if (!kf_fixed[k]) hidx[k] = n_free++;
    if (n_free < 1 || n_free > kBaMaxFree) return -1;
    std::vector<int> pt_off(n_pts + 1, 0), ln_off(n_lines + 1, 0);
    for (int e = 0; e < n_pe; ++e) pt_off[pt_edge_lm[e] + 1]++;
    for (int l = 0; l < n_pts; ++l) pt_off[l + 1] += pt_off[l];
    for (int e = 0; e < n_le; ++e) ln_off[line_edge_lm[e] + 1]++;
    for (int l = 0; l < n_lines; ++l) ln_off[l + 1] += ln_off[l];
    std::vector<int> pt_plane(std::max(n_pts, 1), -1);
    for (int i = 0; i < n_plane_edges; ++i) pt_plane[plane_edge_lm[i]] = i;
    const int n_lm = n_pts + n_lines;
    int max_deg = 1;
    std::vector<int> deg_e(n_lm + 1, 0);
    for (int l = 0; l < n_pts; ++l) {
        int d = 0;
        for (int e = pt_off[l]; e < pt_off[l + 1]; ++e) d += hidx[pt_edge_kf[e]] >= 0;
        max_deg = std::max(max_deg, d);
        deg_e[l + 1] = deg_e[l] + 4 * (1 + (pt_off[l + 1] - pt_off[l] - 1) / 32);
    }
    for (int l = 0; l < n_lines; ++l) {
        int d = 0;
        for (int e = ln_off[l]; e < ln_off[l + 1]; ++e) d += hidx[line_edge_kf[e]] >= 0;
        max_deg = std::max(max_deg, d);
        deg_e[n_pts + l + 1] = deg_e[n_pts + l] + 8 + (ln_off[l + 1] - ln_off[l]);
    }
    const int n_pairs = n_free * (n_free + 1) / 2;
    const size_t budget = 227 * 1024, fixed = linearize_smem(n_free, n_pairs, 0);
    const int fit = (int)((budget - fixed) / sizeof(BaPoolEntry));
    const int pool_cap = std::max(max_deg, std::min(std::min(kBaWarps * max_deg, kPoolMax), fit));
    const int LB = std::max(1, std::min(16, pool_cap / max_deg));
    const int G = std::max(1, std::min(num_ctas, std::max(1, n_lm)));
    std::vector<int> ranges(G + 1, n_lm);
    ranges[0] = 0;
    {
        const long total = deg_e[n_lm];
        int l = 0;
        for (int g = 1; g < G; ++g) {
            const long target = total * g / G;
            while (l < n_lm && deg_e[l] < target) ++l;
            ranges[g] = l;
        }
    }
    std::vector<int> pair_bi(n_pairs), pair_bj(n_pairs);
    for (int i = 0, q = 0; i < n_free; ++i)
        for (int j = i; j < n_free; ++j, ++q) {
            pair_bi[q] = i;
            pair_bj[q] = j;
        }
    const int packed_sum_len = n_pairs * 36 + 12 * n_free + 1;
    const int packed_len = (packed_sum_len + 1 + 31) & ~31;
    const size_t P1 = std::max(n_pts, 1), L1 = std::max(n_lines, 1), E1 = std::max(n_pe, 1), F1 = std::max(n_le, 1);
    std::vector<se3::Pose> pose0(n_kf), pose1(n_kf), pert((size_t)n_kf * 12);
    std::vector<double> pts0(P1 * 3), pts1(P1 * 3), ln0(L1 * 6), ln1(L1 * 6), pt_chi(E1), pt_W(E1 * 24), pt_D(P1 * 16), pt_bl(P1 * 4);
    std::vector<double> ln_chi(F1), ln_W(F1 * 24), ln_D(L1 * 16), ln_bl(L1 * 4), pl_err(std::max(n_plane_edges, 1));
    std::vector<double> partial((size_t)G * packed_len), packed(packed_sum_len + 1 + 8), dp(6 * kBaMaxFree), trial_partial((size_t)G * 2), trial_sum(8, 0.0);
    std::vector<uint8_t> pt_level(E1, 0), pt_outl(E1, 0), pt_act(P1, 0), ln_level(F1, 0), ln_outl(F1, 0), ln_act(L1, 0);
    std::vector<double> T_out((size_t)n_kf * 16), P_out(P1 * 3), L_out(L1 * 6);
    BaState state;
    memset(&state, 0, sizeof(state));
    BaDev D;
    memset(&D, 0, sizeof(D));
    D.fx = fx;
    D.fy = fy;
    D.cx = cx;
    D.cy = cy;
    D.bf = bf;
    D.delta_pt = setup_type == 0 ? (double)sqrtf(5.99146f) : (double)sqrtf(7.81473f);
    D.delta_ln = (double)sqrtf(5.99146f);
    D.n_kf = n_kf;
    D.n_free = n_free;
    D.n_pairs = n_pairs;
    D.n_pts = n_pts;
    D.n_lines = n_lines;
    D.n_pt_edges = n_pe;
    D.n_ln_edges = n_le;
    D.n_pl_edges = n_plane_edges;
    D.num_ctas = G;
    D.batch_landmarks = LB;
    D.pool_cap = pool_cap;
    D.packed_len = packed_len;
    D.packed_sum_len = packed_sum_len;
    D.rank = 0;
    D.world = 1;
    D.kf_hidx = hidx.data();
    D.poses[0] = pose0.data();
    D.poses[1] = pose1.data();
    D.pert_pose = pert.data();
    D.pair_bi = pair_bi.data();
    D.pair_bj = pair_bj.data();
    D.pts[0] = pts0.data();
    D.pts[1] = pts1.data();
    D.lines[0] = ln0.data();
    D.lines[1] = ln1.data();
    D.pt_off = pt_off.data();
    D.pt_kf = pt_edge_kf;
    D.pt_lm = pt_edge_lm;
    D.pt_obs = pt_edge_obs;
    D.pt_info = pt_edge_info;
    D.pt_level = pt_level.data();
    D.pt_outlier = pt_outl.data();
    D.pt_chi2 = pt_chi.data();
    D.pt_W = pt_W.data();
    D.pt_Dinv = pt_D.data();
    D.pt_bl = pt_bl.data();
    D.pt_active = pt_act.data();
    D.pt_plane = n_plane_edges ? pt_plane.data() : nullptr;
    D.pl_fn = plane_edge_fn;
    D.pl_err = pl_err.data();
    D.ln_off = ln_off.data();
    D.ln_kf = line_edge_kf;
    D.ln_lm = line_edge_lm;
    D.ln_obs = line_edge_obs;
    D.ln_info = line_edge_info;
    D.ln_level = ln_level.data();
    D.ln_outlier = ln_outl.data();
    D.ln_chi2 = ln_chi.data();
    D.ln_W = ln_W.data();
    D.ln_Dinv = ln_D.data();
    D.ln_bl = ln_bl.data();
    D.ln_active = ln_act.data();
    D.cta_ranges = ranges.data();
    D.partial = partial.data();
    D.packed = packed.data();
    D.dp = dp.data();
    D.trial_partial = trial_partial.data();
    D.trial_sum = trial_sum.data();
    D.state = &state;

    const size_t lin_smem = linearize_smem(n_free, n_pairs, pool_cap), sol_smem = solve_smem(n_free);
    const unsigned decide_threads = (unsigned)std::max(64, std::min(512, (n_kf * 12 + 31) / 32 * 32));
    int tries_launched = 0;
    auto launch_try = [&]() {
        if (getenv("EMU_BA_TRACE")) fprintf(stderr, "[emu ba] try: phase %d it %d tries %d lambda %g chi %g\n", state.phase, state.it, state.tries, state.lambda, state.current_chi);
        emu_launch2(ba_decide_kernel, 1u, 1u, decide_threads, (size_t)0, D);
        if (getenv("EMU_BA_TRACE")) fprintf(stderr, "  linearize\n");
        emu_launch2(ba_linearize_kernel<false>, (unsigned)G, 1u, (unsigned)kBaThreads, lin_smem, D);
        if (getenv("EMU_BA_TRACE")) fprintf(stderr, "  reduce\n");
        emu_launch2(ba_reduce_kernel, div_up_u((size_t)(packed_sum_len + 1) * kReduceLanes, 256), 1u, 256u, (size_t)0, D);
        if (getenv("EMU_BA_TRACE")) fprintf(stderr, "  solve\n");
        emu_launch2(ba_solve_kernel, 1u, 1u, (unsigned)kSolveThreads, sol_smem, D);
        if (getenv("EMU_BA_TRACE")) fprintf(stderr, "  update\n");
        emu_launch2(ba_update_kernel, (unsigned)G, 1u, (unsigned)kBaThreads, (size_t)6 * n_free * sizeof(double), D);
        if (++tries_launched == 2 && g_cap_packed) {
            memcpy(g_cap_packed, packed.data(), (size_t)packed_sum_len * sizeof(double));
            memcpy(g_cap_dp, dp.data(), (size_t)6 * n_free * sizeof(double));
            *g_cap_lambda = state.lambda;
            g_cap_packed = nullptr;
        }
    };
    auto run_optimize = [&](int n, int robust, bool first) {  // ba_host.cu run_optimize
        emu_launch2(ba_set_state_kernel, 1u, 1u, 1u, (size_t)0, D, n, robust, first ? 1 : 0);
        int launched = 0;
        const int hard_cap = n * 10 + 4;
        int chunk = n + 2;
        while (true) {
            for (int t = 0; t < chunk; ++t) launch_try();
            emu_launch2(ba_decide_kernel, 1u, 1u, decide_threads, (size_t)0, D);
            launched += chunk;
            if (state.phase == kBaDone || launched >= hard_cap) break;
            chunk = 2;
        }
        return state.it;
    };
    auto classify = [&](int set_levels) {
        const int n = n_pe + n_le;
        if (n > 0) emu_launch2(ba_classify_kernel, div_up_u(n, 256), 1u, 256u, (size_t)0, D, set_levels);
    };
    emu_launch2(ba_init_poses_kernel, div_up_u(n_kf, 64), 1u, 64u, (size_t)0, D, kf_pose_cw);
    if (n_pts) memcpy(pts0.data(), pt_pos_w, (size_t)n_pts * 24);
    if (n_lines) memcpy(ln0.data(), line_plucker, (size_t)n_lines * 48);
    iters_out[0] = run_optimize(num_first, mode == 2 ? 0 : 1, true);
    iters_out[1] = 0;
    if (mode == 0) {
        classify(1);
        iters_out[1] = run_optimize(num_second, 0, false);
        classify(0);
    }
    iters_out[2] = state.tries;
    int nmax = std::max(n_kf, std::max(3 * n_pts, 6 * n_lines));
    emu_launch2(ba_export_kernel, div_up_u(nmax, 256), 1u, 256u, (size_t)0, D, T_out.data(), P_out.data(), L_out.data());
    memcpy(kf_out, T_out.data(), (size_t)n_kf * 128);
    if (n_pts) memcpy(pts_out, P_out.data(), (size_t)n_pts * 24);
    if (n_lines) memcpy(lines_out, L_out.data(), (size_t)n_lines * 48);
    if (n_pe) memcpy(pt_outlier_out, pt_outl.data(), n_pe);
    if (n_le) memcpy(ln_outlier_out, ln_outl.data(), n_le);
    return 0;
}
