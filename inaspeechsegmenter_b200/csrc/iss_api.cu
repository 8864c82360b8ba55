// iss_api.cu -- context, error reporting, version.
#include <stdarg.h>
#include <string.h>

#include <atomic>
#include <map>
#include <mutex>
#include <utility>

#include "iss_common.cuh"

static thread_local char g_err[1024] = "";

void iss_set_error(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

static std::atomic<long long> g_launches{0};
void iss_count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
extern "C" int64_t iss_launch_count(void) { return (int64_t)g_launches.load(std::memory_order_relaxed); }

cudaError_t iss_optin_smem(const void *func, int bytes)
{
    static std::mutex mu;
    static std::map<std::pair<const void *, int>, int> done;          // (kernel, device) -> bytes opted in
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    std::lock_guard<std::mutex> lk(mu);
    auto it = done.find({func, dev});
    if (it != done.end() && it->second >= bytes) return cudaSuccess;
    e = cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess) done[{func, dev}] = bytes;
    return e;
}

extern "C" int iss_version(void) { return ISS_ABI_VERSION; }

extern "C" const char *iss_last_error(void) { return g_err; }

extern "C" int iss_ctx_create(int device, iss_ctx **out)
{
    ISS_REQUIRE(out != nullptr, ISS_ERR_INVALID, "iss_ctx_create: out is NULL");
    int n = 0;
    ISS_CUDA_OK(cudaGetDeviceCount(&n));
    ISS_REQUIRE(device >= 0 && device < n, ISS_ERR_INVALID, "iss_ctx_create: device %d of %d", device, n);
    cudaDeviceProp prop;
    ISS_CUDA_OK(cudaGetDeviceProperties(&prop, device));
    // The library is compiled for sm_90a only: no PTX fallback, no other arch.
    ISS_REQUIRE(prop.major == 9 && prop.minor == 0, ISS_ERR_CUDA,
                "iss_ctx_create: device %d is sm_%d%d; libiss_b200 holds sm_90a code only",
                device, prop.major, prop.minor);
    ISS_CUDA_OK(cudaSetDevice(device));
    iss_ctx *c = new iss_ctx();
    c->device = device;
    c->sm_count = prop.multiProcessorCount;
    c->d_tables = nullptr;
    c->tables_ready = false;
    c->d_partials = nullptr;
    c->partials_cap = 0;
    c->d_recs = nullptr;
    c->recs_cap = 0;
    c->d_vbx_recs = nullptr;
    c->vbx_recs_cap = 0;
    c->resample = nullptr;
    *out = c;
    return ISS_OK;
}

extern "C" int iss_ctx_destroy(iss_ctx *ctx)
{
    if (!ctx) return ISS_OK;
    cudaSetDevice(ctx->device);
    if (ctx->d_tables) cudaFree(ctx->d_tables);
    if (ctx->d_partials) cudaFree(ctx->d_partials);
    if (ctx->d_recs) cudaFree(ctx->d_recs);
    if (ctx->d_vbx_recs) cudaFree(ctx->d_vbx_recs);
    iss_resample_free(ctx);
    delete ctx;
    return ISS_OK;
}
