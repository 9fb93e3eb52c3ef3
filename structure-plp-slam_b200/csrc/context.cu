// context.cu -- plp_ctx lifetime, error string, device-memory helpers of the C ABI.
#include "common.cuh"

#include <map>
#include <mutex>
#include <utility>

namespace plp {

static thread_local char g_err[512] = "";

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

void timing_begin(plp_ctx *ctx, const char *name) {
    plp_ctx::TimedLaunch t;
    t.name = name;
    cudaEventCreate(&t.start);
    cudaEventCreate(&t.stop);
    cudaEventRecord(t.start, ctx->stream);
    ctx->timed.push_back(t);
}

void timing_end(plp_ctx *ctx) { cudaEventRecord(ctx->timed.back().stop, ctx->stream); }

plp_status ctx_scratch(plp_ctx *ctx, int slot, size_t bytes, void **out) {
    ScratchBuf &b = ctx->scratch[slot];
    if (b.bytes < bytes) {
        if (b.ptr) {
            PLP_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
            PLP_CUDA_TRY(cudaFree(b.ptr));
            b.ptr = nullptr;
            b.bytes = 0;
        }
        size_t want = bytes + bytes / 2 + 256;
        PLP_CUDA_TRY(cudaMalloc(&b.ptr, want));
        b.bytes = want;
    }
    *out = b.ptr;
    return PLP_OK;
}

plp_status ctx_pinned(plp_ctx *ctx, size_t bytes, void **out) {
    if (ctx->pinned_bytes < bytes) {
        if (ctx->pinned) {
            PLP_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
            PLP_CUDA_TRY(cudaFreeHost(ctx->pinned));
            ctx->pinned = nullptr;
            ctx->pinned_bytes = 0;
        }
        size_t want = bytes + bytes / 2 + 256;
        PLP_CUDA_TRY(cudaMallocHost(&ctx->pinned, want));
        ctx->pinned_bytes = want;
    }
    *out = ctx->pinned;
    return PLP_OK;
}

plp_status stage(plp_ctx *ctx, int slot, DevLayout &L) {
    const size_t want = L.bytes() ? L.bytes() : 256;
    void *d = nullptr, *h = nullptr;
    PLP_TRY(ctx_scratch(ctx, slot, want, &d));
    PLP_TRY(ctx_pinned(ctx, want, &h));
    const size_t n = L.place((uint8_t *)d, (uint8_t *)h);
    if (n) PLP_CUDA_TRY(cudaMemcpyAsync(d, h, n, cudaMemcpyHostToDevice, ctx->stream));
    return PLP_OK;
}

cudaError_t alloc(plp_ctx *ctx, DevLayout &L, uint8_t **block, bool zero) {
    cudaError_t e = cudaMalloc((void **)block, L.bytes());
    if (e != cudaSuccess) {
        cudaGetLastError();  // the caller reports the refusal; a later launch check must not report it again
        *block = nullptr;
        return e;
    }
    std::vector<uint8_t> image(L.in_bytes());
    const size_t n = L.place(*block, image.data());
    if (zero) e = cudaMemsetAsync(*block, 0, L.bytes(), ctx->stream);
    if (e == cudaSuccess && n) e = cudaMemcpyAsync(*block, image.data(), n, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess && (zero || n)) e = cudaStreamSynchronize(ctx->stream);  // the image dies with this scope
    return e;
}

plp_status ensure_smem_optin(const void *kernel, size_t need, const char *name) {
    static std::mutex mu;
    static std::map<std::pair<const void *, int>, size_t> done;  // (kernel, device) -> opted-in bytes
    int dev = 0;
    PLP_CUDA_TRY(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lock(mu);
    auto it = done.find({kernel, dev});
    if (it == done.end()) {
        int optin = 0;
        PLP_CUDA_TRY(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
        cudaFuncAttributes fa;
        PLP_CUDA_TRY(cudaFuncGetAttributes(&fa, kernel));
        const int dyn_max = optin - (int)fa.sharedSizeBytes;  // static shared memory counts against the same limit
        PLP_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn_max));
        it = done.emplace(std::make_pair(kernel, dev), (size_t)dyn_max).first;
    }
    if (need > it->second) {
        set_error("%s needs %zu bytes of dynamic shared memory, the device offers %zu", name, need, it->second);
        return PLP_ERR_CAPACITY;
    }
    return PLP_OK;
}

}  // namespace plp

extern "C" {

const char *plp_last_error(void) { return plp::g_err; }

int plp_version(void) { return 100; }

int plp_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

plp_status plp_ctx_create(int device, plp_ctx **out) { return plp_ctx_create_ex(device, 0, out); }

plp_status plp_ctx_create_ex(int device, int high_priority, plp_ctx **out) {
    PLP_REQUIRE(out != nullptr, "out");
    *out = nullptr;
    int n = plp_device_count();
    if (n <= 0 || device < 0 || device >= n) {
        plp::set_error("no usable CUDA device (count=%d, requested=%d): this library has no CPU fallback", n,
                       device);
        return PLP_ERR_NO_DEVICE;
    }
    PLP_CUDA_TRY(cudaSetDevice(device));
    // everything that can fail comes before the allocation: no error path leaks the handle
    cudaDeviceProp prop;
    PLP_CUDA_TRY(cudaGetDeviceProperties(&prop, device));
    int prio_lo = 0, prio_hi = 0;
    PLP_CUDA_TRY(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));  // numerically lower = higher priority
    cudaStream_t stream = nullptr;
    PLP_CUDA_TRY(cudaStreamCreateWithPriority(&stream, cudaStreamNonBlocking, high_priority ? prio_hi : prio_lo));
    plp_ctx *c = new plp_ctx();
    c->device = device;
    c->sm_count = prop.multiProcessorCount;
    c->stream = stream;
    *out = c;
    return PLP_OK;
}

void plp_ctx_destroy(plp_ctx *ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    for (auto &b : ctx->scratch)
        if (b.ptr) cudaFree(b.ptr);
    if (ctx->pinned) cudaFreeHost(ctx->pinned);
    cudaStreamDestroy(ctx->stream);
    delete ctx;
}

plp_status plp_ctx_sync(plp_ctx *ctx) {
    PLP_REQUIRE(ctx != nullptr, "ctx");
    PLP_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return PLP_OK;
}

void *plp_ctx_stream(plp_ctx *ctx) { return ctx ? (void *)ctx->stream : nullptr; }

uint64_t plp_ctx_launch_count(plp_ctx *ctx) { return ctx ? ctx->launches : 0; }

plp_status plp_ctx_kernel_timing(plp_ctx *ctx, int enable) {
    PLP_REQUIRE(ctx != nullptr, "ctx");
    PLP_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    for (auto &t : ctx->timed) {
        cudaEventDestroy(t.start);
        cudaEventDestroy(t.stop);
    }
    ctx->timed.clear();
    ctx->timing = enable != 0;
    return PLP_OK;
}

plp_status plp_ctx_kernel_timing_report(plp_ctx *ctx, char *buf, size_t buf_bytes) {
    PLP_REQUIRE(ctx != nullptr && buf != nullptr && buf_bytes > 2, "ctx/buf");
    PLP_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    struct Agg {
        const char *name;
        double ms;
        long count;
    };
    std::vector<Agg> agg;
    for (auto &t : ctx->timed) {
        float ms = 0;
        if (cudaEventElapsedTime(&ms, t.start, t.stop) != cudaSuccess) continue;
        bool found = false;
        for (auto &a : agg)
            if (strcmp(a.name, t.name) == 0) {
                a.ms += ms;
                a.count++;
                found = true;
                break;
            }
        if (!found) agg.push_back({t.name, ms, 1});
    }
    size_t off = 0;
    off += snprintf(buf + off, buf_bytes - off, "{");
    for (size_t i = 0; i < agg.size() && off + 160 < buf_bytes; ++i)
        off += snprintf(buf + off, buf_bytes - off, "%s\"%s\": {\"count\": %ld, \"total_ms\": %.6f}", i ? ", " : "",
                        agg[i].name, agg[i].count, agg[i].ms);
    snprintf(buf + off, buf_bytes - off, "}");
    return PLP_OK;
}

plp_status plp_dev_alloc(plp_ctx *ctx, size_t bytes, void **out) {
    PLP_REQUIRE(ctx != nullptr && out != nullptr, "ctx/out");
    PLP_CUDA_TRY(cudaSetDevice(ctx->device));
    PLP_CUDA_TRY(cudaMalloc(out, bytes ? bytes : 1));
    return PLP_OK;
}

plp_status plp_dev_free(plp_ctx *ctx, void *ptr) {
    PLP_REQUIRE(ctx != nullptr, "ctx");
    if (ptr) {
        PLP_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
        PLP_CUDA_TRY(cudaFree(ptr));
    }
    return PLP_OK;
}

plp_status plp_dev_upload(plp_ctx *ctx, void *dst_dev, const void *src_host, size_t bytes) {
    PLP_REQUIRE(ctx != nullptr, "ctx");
    if (bytes == 0) return PLP_OK;
    PLP_CUDA_TRY(cudaMemcpyAsync(dst_dev, src_host, bytes, cudaMemcpyHostToDevice, ctx->stream));
    PLP_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return PLP_OK;
}

plp_status plp_dev_download(plp_ctx *ctx, void *dst_host, const void *src_dev, size_t bytes) {
    PLP_REQUIRE(ctx != nullptr, "ctx");
    if (bytes == 0) return PLP_OK;
    PLP_CUDA_TRY(cudaMemcpyAsync(dst_host, src_dev, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    PLP_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return PLP_OK;
}

plp_status plp_dev_upload_async(plp_ctx *ctx, void *dst_dev, const void *src_host, size_t bytes) {
    PLP_REQUIRE(ctx != nullptr, "ctx");
    if (bytes == 0) return PLP_OK;
    PLP_CUDA_TRY(cudaMemcpyAsync(dst_dev, src_host, bytes, cudaMemcpyHostToDevice, ctx->stream));
    return PLP_OK;
}

plp_status plp_dev_download_async(plp_ctx *ctx, void *dst_host, const void *src_dev, size_t bytes) {
    PLP_REQUIRE(ctx != nullptr, "ctx");
    if (bytes == 0) return PLP_OK;
    PLP_CUDA_TRY(cudaMemcpyAsync(dst_host, src_dev, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    return PLP_OK;
}

plp_status plp_ctx_wait_ctx(plp_ctx *waiter, plp_ctx *other) {
    PLP_REQUIRE(waiter != nullptr && other != nullptr, "ctx");
    if (waiter == other) return PLP_OK;
    cudaEvent_t ev;
    PLP_CUDA_TRY(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    PLP_CUDA_TRY(cudaEventRecord(ev, other->stream));
    PLP_CUDA_TRY(cudaStreamWaitEvent(waiter->stream, ev, 0));
    PLP_CUDA_TRY(cudaEventDestroy(ev));  // released once the recorded work has completed
    return PLP_OK;
}

plp_status plp_host_alloc_pinned(size_t bytes, void **out) {
    PLP_REQUIRE(out != nullptr, "out");
    PLP_CUDA_TRY(cudaMallocHost(out, bytes ? bytes : 1));
    return PLP_OK;
}

plp_status plp_host_free_pinned(void *ptr) {
    if (ptr) PLP_CUDA_TRY(cudaFreeHost(ptr));
    return PLP_OK;
}

}  // extern "C"
