// gx_ctx.cu — context, error reporting, timing, L2 flush.
#include <stdarg.h>
#include "gx_internal.cuh"

static char g_global_err[512] = "";

void gx_set_global_err(const char *fmt, ...)
{
    va_list ap; va_start(ap, fmt);
    vsnprintf(g_global_err, sizeof(g_global_err), fmt, ap);
    va_end(ap);
}

extern "C" int gx_abi_version(void) { return GX_ABI_VERSION; }

extern "C" const char *gx_last_error(gx_ctx *ctx) { return ctx ? ctx->err : g_global_err; }

extern "C" int gx_init(int device, gx_ctx **out)
{
    if (!out) return GX_ERR_ARG;
    *out = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev <= 0) {
        gx_set_global_err("gx_init: no CUDA device (%s); the GPU executor path is unavailable and has no CPU fallback",
                          e != cudaSuccess ? cudaGetErrorString(e) : "device count 0");
        return GX_ERR_NODEVICE;
    }
    if (device < 0 || device >= ndev) { gx_set_global_err("gx_init: device %d out of range [0,%d)", device, ndev); return GX_ERR_ARG; }
    cudaDeviceProp prop;
    if ((e = cudaGetDeviceProperties(&prop, device)) != cudaSuccess) { gx_set_global_err("gx_init: %s", cudaGetErrorString(e)); return GX_ERR_CUDA; }
    if (prop.major != 9 || prop.minor != 0) {   // an sm_90a cubin loads on compute capability 9.0 and nothing else
        gx_set_global_err("gx_init: device %d is sm_%d%d; libgpuexec is built for sm_90a only", device, prop.major, prop.minor);
        return GX_ERR_NODEVICE;
    }
    if ((e = cudaSetDevice(device)) != cudaSuccess) { gx_set_global_err("gx_init: cudaSetDevice: %s", cudaGetErrorString(e)); return GX_ERR_CUDA; }

    gx_ctx *ctx = (gx_ctx *) calloc(1, sizeof(gx_ctx));
    ctx->device = device;
    ctx->sm_count = prop.multiProcessorCount;
    ctx->cc_major = prop.major; ctx->cc_minor = prop.minor;
    ctx->hbm_bytes = prop.totalGlobalMem;
    ctx->smem_optin = prop.sharedMemPerBlockOptin;
    { int l2 = 0; cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, device); ctx->l2_bytes = (size_t) l2; }
    // L2 fetch granularity: a random 32-byte sector miss may otherwise drag in 64 bytes
    {
        const char *g = getenv("GX_L2_FETCH");
        size_t gran = g ? (size_t) atoi(g) : 0;      // opt-in only
        if (gran == 32 || gran == 64 || gran == 128) cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, gran);
        cudaGetLastError();
    }
    ctx->prof = new std::map<std::string, gx_prof_entry>();
    ctx->nnodes = 1; ctx->rank = 0; ctx->nranks = 1;
    {   // keep freed temporaries cached in the default pool instead of returning them to the OS
        cudaMemPool_t pool; unsigned long long thresh = ~0ULL;
        if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thresh);
        cudaGetLastError();
    }
    GX_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
    for (int i = 0; i < GX_NCOPY; i++) {
        GX_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->copy_streams[i], cudaStreamNonBlocking));
        for (int k = 0; k < 2; k++) GX_CUDA(ctx, cudaEventCreateWithFlags(&ctx->copy_ev[k][i], cudaEventDisableTiming));
    }
    GX_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_alloc, cudaEventDisableTiming));
    GX_CUDA(ctx, cudaEventCreate(&ctx->ev_t0)); GX_CUDA(ctx, cudaEventCreate(&ctx->ev_t1));
    GX_CUDA(ctx, cudaMalloc(&ctx->d_scratch, 64 * sizeof(long long)));
    GX_CUDA(ctx, cudaMemset(ctx->d_scratch, 0, 64 * sizeof(long long)));
    GX_CUDA(ctx, cudaHostAlloc(&ctx->h_scratch, 64 * sizeof(long long), cudaHostAllocDefault));
    GX_CUDA(ctx, cudaMalloc(&ctx->d_shardmap, GX_SHARD_MAP_SHARD_NUM * sizeof(int32_t)));
    GX_CUDA(ctx, cudaMemset(ctx->d_shardmap, 0, GX_SHARD_MAP_SHARD_NUM * sizeof(int32_t)));
    *out = ctx;
    return GX_OK;
}

extern "C" void gx_comm_destroy(gx_ctx *ctx);

// Map `bytes` of HBM into the context's stream-ordered pool up front (one allocation, freed at once; 0 = everything that
// is free minus 8 GB of headroom for NCCL and the host runtime).  Without it the pool grows on demand, and a query whose
// temporaries do not fit the blocks already mapped waits for the driver to create and map physical memory in the middle
// of its critical path, and with several ranks every rank waits for the slowest.
extern "C" int gx_pool_reserve(gx_ctx *ctx, size_t bytes)
{
    if (!ctx) return GX_ERR_ARG;
    if (bytes == 0) {
        size_t fr = 0, tot = 0;
        GX_CUDA(ctx, cudaMemGetInfo(&fr, &tot));
        const size_t head = (size_t) 8 << 30;
        if (fr <= head) return GX_OK;
        bytes = fr - head;
    }
    void *p = nullptr;
    cudaError_t e = cudaMallocAsync(&p, bytes, ctx->stream);
    if (e != cudaSuccess) { cudaGetLastError(); GX_SET_ERR(ctx, "pool_reserve: %zu bytes: %s", bytes, cudaGetErrorString(e)); return GX_ERR_NOMEM; }
    GX_CUDA(ctx, cudaFreeAsync(p, ctx->stream));
    GX_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GX_OK;
}

extern "C" void gx_shutdown(gx_ctx *ctx)
{
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    gx_comm_destroy(ctx);
    if (ctx->l2flush_buf) cudaFree(ctx->l2flush_buf);
    if (ctx->prof_pool) { for (int i = 0; i < GX_PROF_POOL; i++) { cudaEventDestroy(ctx->prof_pool[i].a); cudaEventDestroy(ctx->prof_pool[i].b); } free(ctx->prof_pool); }
    for (int i = 0; i < GX_NCOPY; i++) {
        cudaStreamSynchronize(ctx->copy_streams[i]); cudaStreamDestroy(ctx->copy_streams[i]);
        for (int k = 0; k < 2; k++) cudaEventDestroy(ctx->copy_ev[k][i]);
    }
    cudaEventDestroy(ctx->ev_alloc);
    for (int i = 0; i < 2; i++) { if (ctx->stage[i]) cudaFreeHost(ctx->stage[i]); if (ctx->stage_ev[i]) cudaEventDestroy(ctx->stage_ev[i]); }
    cudaFree(ctx->d_scratch); cudaFreeHost(ctx->h_scratch); cudaFree(ctx->d_shardmap);
    cudaEventDestroy(ctx->ev_t0); cudaEventDestroy(ctx->ev_t1);
    cudaStreamDestroy(ctx->stream);
    delete ctx->prof;
    free(ctx);
}

extern "C" int gx_device_info(gx_ctx *ctx, int *sm_count, int *cc_major, int *cc_minor, int64_t *hbm_bytes)
{
    if (!ctx) return GX_ERR_ARG;
    if (sm_count) *sm_count = ctx->sm_count;
    if (cc_major) *cc_major = ctx->cc_major;
    if (cc_minor) *cc_minor = ctx->cc_minor;
    if (hbm_bytes) *hbm_bytes = (int64_t) ctx->hbm_bytes;
    return GX_OK;
}

extern "C" int gx_sync(gx_ctx *ctx)
{
    if (!ctx) return GX_ERR_ARG;
    for (int i = 0; i < GX_NCOPY; i++) GX_CUDA(ctx, cudaStreamSynchronize(ctx->copy_streams[i]));
    GX_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GX_OK;
}

extern "C" int64_t gx_launch_count(gx_ctx *ctx) { return ctx ? ctx->launches : 0; }

extern "C" int gx_timer_start(gx_ctx *ctx)
{
    if (!ctx) return GX_ERR_ARG;
    GX_CUDA(ctx, cudaEventRecord(ctx->ev_t0, ctx->stream));
    return GX_OK;
}
extern "C" int gx_timer_stop(gx_ctx *ctx, double *ms_out)
{
    if (!ctx) return GX_ERR_ARG;
    GX_CUDA(ctx, cudaEventRecord(ctx->ev_t1, ctx->stream));
    GX_CUDA(ctx, cudaEventSynchronize(ctx->ev_t1));
    float ms = 0;
    GX_CUDA(ctx, cudaEventElapsedTime(&ms, ctx->ev_t0, ctx->ev_t1));
    if (ms_out) *ms_out = (double) ms;
    return GX_OK;
}

static int prof_resolve(gx_ctx *ctx)
{
    if (ctx->prof_used == 0) return GX_OK;
    GX_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (int i = 0; i < ctx->prof_used; i++) {
        float ms = 0;
        if (cudaEventElapsedTime(&ms, ctx->prof_pool[i].a, ctx->prof_pool[i].b) == cudaSuccess) {
            gx_prof_entry &e = (*ctx->prof)[ctx->prof_pool[i].name];
            e.ms += ms; e.launches += 1;
        }
    }
    ctx->prof_used = 0;
    return GX_OK;
}
extern "C" int gx_profile(gx_ctx *ctx, int enable)
{
    if (!ctx) return GX_ERR_ARG;
    if (enable && !ctx->prof_pool) {
        ctx->prof_pool = (gx_prof_rec *) calloc(GX_PROF_POOL, sizeof(gx_prof_rec));
        for (int i = 0; i < GX_PROF_POOL; i++) { GX_CUDA(ctx, cudaEventCreate(&ctx->prof_pool[i].a)); GX_CUDA(ctx, cudaEventCreate(&ctx->prof_pool[i].b)); }
    }
    if (enable) { cudaGetLastError(); ctx->prof_used = 0; ctx->prof->clear(); }
    ctx->profile = enable;
    return GX_OK;
}
extern "C" int gx_profile_get(gx_ctx *ctx, const char *name, double *ms_total, int64_t *launches)
{
    if (!ctx || !name) return GX_ERR_ARG;
    int rc = prof_resolve(ctx); if (rc) return rc;
    auto it = ctx->prof->find(name);
    if (ms_total) *ms_total = it == ctx->prof->end() ? 0.0 : it->second.ms;
    if (launches) *launches = it == ctx->prof->end() ? 0 : it->second.launches;
    return GX_OK;
}

__global__ void gx_k_l2flush(uint4 *buf, size_t n16, unsigned int v)
{
    size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t) gridDim.x * blockDim.x;
    for (; i < n16; i += stride) buf[i] = make_uint4(v, v + 1, v + 2, v + 3);
}

// Writes a buffer several times the size of L2 (50 MB on H100) so the next timed
// iteration starts from cold caches.
extern "C" int gx_l2_flush(gx_ctx *ctx)
{
    if (!ctx) return GX_ERR_ARG;
    if (!ctx->l2flush_buf) {
        ctx->l2flush_bytes = (size_t) 256 << 20;
        GX_CUDA(ctx, cudaMalloc(&ctx->l2flush_buf, ctx->l2flush_bytes));
    }
    static unsigned int v = 1;
    gx_k_l2flush<<<ctx->sm_count * 4, 512, 0, ctx->stream>>>((uint4 *) ctx->l2flush_buf, ctx->l2flush_bytes / 16, v++);
    GX_CUDA(ctx, cudaGetLastError());
    return GX_OK;
}
