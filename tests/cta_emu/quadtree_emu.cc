// quadtree_emu.cc -- csrc/quadtree_kernels.cuh executed on the host (see cta_emu.h): the ORB quadtree of one level of one
// frame, fed through the kernel's own gather (candidates split into cells of at most kCellCap), against the oracle.
#include "cta_emu.h"

struct short4 {
    short x, y, z, w;
};

#include "quadtree_kernels.cuh"

#include <algorithm>
#include <vector>

using namespace plp;

template <int NC, int CC, int T>
static int run(const uint32_t *cand, int n, int w, int h, int budget, int cell_size, LevelKp *out, int out_cap, int *status) {
    const int cells = std::max(1, (n + cell_size - 1) / cell_size);
    std::vector<uint32_t> cell_buf((size_t)cells * kCellCap, 0u);
    std::vector<int> cell_cnt(cells, 0);
    for (int i = 0; i < n; ++i) {
        cell_buf[(size_t)(i / cell_size) * kCellCap + i % cell_size] = cand[i];
        cell_cnt[i / cell_size]++;
    }
    std::vector<LevelKp> kp(out_cap);
    std::vector<uint8_t> scratch(qt_scratch_bytes_per_job());
    int lvl_cnt = -1;
    *status = 0;
    QtJob J{};
    J.num_levels = 1;
    J.num_cells = cells;
    J.total_slots = out_cap;
    J.lv[0] = QtLevel{w, h, 0, cells, budget, 0, out_cap};
    J.cell_buf = cell_buf.data();
    J.cell_cnt = cell_cnt.data();
    J.lvl_kp = kp.data();
    J.lvl_cnt = &lvl_cnt;
    J.scratch = scratch.data();
    J.scratch_per_job = scratch.size();
    J.status = status;
    emu_launch2(quadtree_kernel<NC, CC, T, 1>, 1u, 1u, (unsigned)T, qt_smem_bytes<NC, CC, T>(), J);
    std::copy(kp.begin(), kp.begin() + std::max(0, lvl_cnt), out);
    return lvl_cnt;
}

// instance: 0 = <1024> (small), 1 = <2048> (large), 2 = the large layout at 4096 nodes (budgets beyond both instances)
extern "C" int emu_quadtree(int instance, const uint32_t *cand, int n, int w, int h, int budget, int cell_size,
                            LevelKp *out, int out_cap, int *status) {
    switch (instance) {
        case 0: return run<kNodeCapSmall, kCandCapSmall, kQtThreadsSmall>(cand, n, w, h, budget, cell_size, out, out_cap, status);
        case 1: return run<kNodeCap, kCandCapLarge, kQtThreadsLarge>(cand, n, w, h, budget, cell_size, out, out_cap, status);
        default: return run<4096, kCandCapLarge, kQtThreadsLarge>(cand, n, w, h, budget, cell_size, out, out_cap, status);
    }
}

extern "C" int emu_quadtree_cand_cap(int instance) { return instance == 0 ? kCandCapSmall : kCandCapLarge; }
