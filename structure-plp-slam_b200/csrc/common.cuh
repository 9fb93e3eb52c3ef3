// common.cuh -- context, error plumbing and small device helpers shared by all kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <string.h>
#include <vector>

#include "../../include/plpslam_b200.h"
#include "devmath.cuh"
#include "layout.h"

namespace plp {

// thread-local last error message (never throws across the C ABI)
void set_error(const char *fmt, ...);

struct ScratchBuf {
    void *ptr = nullptr;
    size_t bytes = 0;
};

}  // namespace plp

struct plp_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    int sm_count = 0;
    uint64_t launches = 0;  // kernels launched by this library on this context
    // growable device scratch areas (index = purpose), never shrunk
    plp::ScratchBuf scratch[8];
    // growable pinned host staging area
    void *pinned = nullptr;
    size_t pinned_bytes = 0;
    // optional per-kernel timing (bench.py roofline leg): CUDA events recorded around every launch
    bool timing = false;
    struct TimedLaunch {
        const char *name;
        cudaEvent_t start, stop;
    };
    std::vector<TimedLaunch> timed;
};

namespace plp {

void timing_begin(plp_ctx *ctx, const char *name);
void timing_end(plp_ctx *ctx);
plp_status ctx_scratch(plp_ctx *ctx, int slot, size_t bytes, void **out);
plp_status ctx_pinned(plp_ctx *ctx, size_t bytes, void **out);
// The two backings of a DevLayout (layout.h).  stage: a call's layout in scratch slot `slot`, its inputs gathered in the
// pinned staging buffer and sent in ONE host-to-device copy (per-array copies would be launch-latency bound at these
// sizes).  alloc: a handle's layout in one cudaMalloc into *block, which the handle frees (null if the allocation
// failed); `zero` clears the whole block before the inputs are copied, and the copy is waited for.
plp_status stage(plp_ctx *ctx, int slot, DevLayout &L);
cudaError_t alloc(plp_ctx *ctx, DevLayout &L, uint8_t **block, bool zero);
// queues the copy of `count` elements of a device output into caller memory
template <class T>
cudaError_t to_host(plp_ctx *ctx, T *dst, const T *dev, size_t count) {
    return cudaMemcpyAsync(dst, dev, count * sizeof(T), cudaMemcpyDeviceToHost, ctx->stream);
}
// Opt a kernel in to the DEVICE MAXIMUM of dynamic shared memory, once per (kernel, device), and check that `need`
// fits.  cudaFuncAttributeMaxDynamicSharedMemorySize is global per kernel: setting it to the size of the current
// problem would lower it under a concurrent larger launch of another handle / thread, so it is only ever raised.
plp_status ensure_smem_optin(const void *kernel, size_t need, const char *name);
#define PLP_SMEM_OPTIN(kernel, need) PLP_TRY(plp::ensure_smem_optin((const void *)(kernel), (need), #kernel))

#define PLP_CUDA_TRY(expr)                                                                   \
    do {                                                                                     \
        cudaError_t _e = (expr);                                                             \
        if (_e != cudaSuccess) {                                                             \
            plp::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, \
                           __LINE__);                                                        \
            return PLP_ERR_CUDA;                                                             \
        }                                                                                    \
    } while (0)

#define PLP_TRY(expr)                     \
    do {                                  \
        plp_status _s = (expr);           \
        if (_s != PLP_OK) return _s;      \
    } while (0)

#define PLP_REQUIRE(cond, msg)                                     \
    do {                                                           \
        if (!(cond)) {                                             \
            plp::set_error("invalid argument: %s (%s)", msg, #cond); \
            return PLP_ERR_INVALID;                                \
        }                                                          \
    } while (0)

// every kernel launch goes through this so gpu_launches can be reported honestly
#define PLP_LAUNCH(ctx, kernel, grid, block, smem, ...)                          \
    do {                                                                         \
        if ((ctx)->timing) plp::timing_begin((ctx), #kernel);                    \
        kernel<<<(grid), (block), (smem), (ctx)->stream>>>(__VA_ARGS__);         \
        if ((ctx)->timing) plp::timing_end((ctx));                               \
        (ctx)->launches++;                                                       \
    } while (0)

#define PLP_CHECK_LAUNCH()                                                              \
    do {                                                                                \
        cudaError_t _e = cudaGetLastError();                                            \
        if (_e != cudaSuccess) {                                                        \
            plp::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e),  \
                           __FILE__, __LINE__);                                         \
            return PLP_ERR_CUDA;                                                        \
        }                                                                               \
    } while (0)

}  // namespace plp
