// fuse_emu.cc -- csrc/fuse_kernels.cuh (match::fuse search, GPU-verified) executed on the host: dynamic shared memory, the
// stable counting sort with shared-memory atomics, a 2-D grid (landmark chunks x targets).
#include "cta_emu.h"

#include <string.h>

#include "fuse_kernels.cuh"

using namespace plp;

extern "C" void emu_fuse_points(int num_targets, const int32_t *t_n, const float *const *t_x, const float *const *t_y,
                                const float *const *t_xr, const int32_t *const *t_oct, const uint8_t *const *t_desc,
                                const uint8_t *const *t_skip, const double *t_pose /*num_targets x 15: R, t, c*/,
                                const plp_grid *grid, const plp_camera *cam, const float *scale_factors,
                                const float *inv_sigma_sq, const float *level_thr, int num_levels, float margin, int mode,
                                int m, const double *pos_w, const double *normal, const float *min_d, const float *max_d,
                                const float *max_raw, const uint8_t *lm_desc, const uint8_t *lm_valid, int chunk,
                                int32_t *best_idx, uint16_t *best_dist) {
    std::vector<FusePointTarget> T(num_targets);
    int max_n = 0;
    for (int t = 0; t < num_targets; ++t) {
        memset(&T[t], 0, sizeof(T[t]));
        T[t].n = t_n[t];
        T[t].x = t_x[t];
        T[t].y = t_y[t];
        T[t].xr = t_xr[t];
        T[t].octave = t_oct[t];
        T[t].desc = t_desc[t];
        T[t].skip = t_skip[t];
        memcpy(T[t].R, t_pose + 15 * t, 9 * 8);
        memcpy(T[t].t, t_pose + 15 * t + 9, 3 * 8);
        memcpy(T[t].c, t_pose + 15 * t + 12, 3 * 8);
        if (t_n[t] > max_n) max_n = t_n[t];
    }
    FuseLandmarks L;
    L.m = m;
    L.pos_w = pos_w;
    L.normal = normal;
    L.min_d = min_d;
    L.max_d = max_d;
    L.max_raw = max_raw;
    L.desc = lm_desc;
    L.valid = lm_valid;
    FuseParams P;
    memset(&P, 0, sizeof(P));
    P.cam = *cam;
    P.grid = *grid;
    for (int l = 0; l < num_levels; ++l) {
        P.scale_factors[l] = scale_factors[l];
        P.inv_sigma_sq[l] = inv_sigma_sq[l];
        P.level_thr[l] = level_thr[l];
    }
    P.num_levels = num_levels;
    P.margin = margin;
    P.mode = mode;
    const int cap = max_n < 64 ? 64 : ((max_n + 63) / 64) * 64;
    const size_t smem = fuse_point_smem_bytes(cap, grid->num_cols * grid->num_rows);
    const FusePointTarget *targets = T.data();
    emu_launch2(fuse_points_kernel, (unsigned)((m + chunk - 1) / chunk), (unsigned)num_targets, (unsigned)kThreads, smem,
                targets, L, P, cap, chunk, best_idx, best_dist);
}
