// gx_exec.cu — the one-call form used by the CustomScan provider and by
// bench.py's end-to-end leg: HOST column buffers in, partial result out.
// Host->HBM staging: every column is cut into 64 MB chunks that go round-robin
// over GX_NCOPY copy streams (several DMA engines, no single-queue limit); the
// inner table is queued first, so the join-table build (compute stream) runs
// while the outer columns are still arriving.  The probe+aggregate kernel needs
// the whole outer table and starts when its last chunk has landed: at SF100 the
// step is 11.4 GB over PCIe against a few ms of kernels, so e2e is a PCIe figure
// and bench.py reports it next to a same-run copy ceiling (gx_h2d_probe).
#include "gx_internal.cuh"
#include <unistd.h>
#include <sys/syscall.h>

// Pinned staging memory is placed on the NUMA node the GPU hangs off.  On a two-socket host a
// pinned buffer that happens to be allocated on the other socket is copied at a fraction of the
// PCIe rate, and
// which socket a backend's first touch lands on is a coin toss.  The node comes from sysfs
// (/sys/bus/pci/devices/<bus id>/numa_node); the allocation runs under a temporary
// MPOL_BIND policy (raw syscall, no libnuma), retried unbound if the node cannot hold it.  Anything that fails leaves the default policy.
static int gpu_numa_node(int device)
{
    char bus[32] = { 0 }, path[128];
    if (cudaDeviceGetPCIBusId(bus, (int) sizeof(bus), device) != cudaSuccess) { cudaGetLastError(); return -1; }
    for (char *c = bus; *c; c++) if (*c >= 'A' && *c <= 'Z') *c = (char) (*c - 'A' + 'a');
    snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/numa_node", bus);
    FILE *f = fopen(path, "r");
    if (!f) return -1;
    int node = -1;
    if (fscanf(f, "%d", &node) != 1) node = -1;
    fclose(f);
    return node;
}
extern "C" int gx_host_alloc(gx_ctx *ctx, size_t bytes, void **out)
{
    if (!ctx || !out) return GX_ERR_ARG;
    const char *off = getenv("GX_NO_NUMA_BIND");
    int node = (off && off[0] == '1') ? -1 : gpu_numa_node(ctx->device);
    bool bound = false;
    if (node >= 0 && node < 1024) {
        unsigned long mask[16] = { 0 };
        mask[node / (8 * sizeof(unsigned long))] |= 1UL << (node % (8 * sizeof(unsigned long)));
        // MPOL_BIND: "preferred" silently spills to the other node when the local one is full of page cache
        bound = syscall(SYS_set_mempolicy, 2 /* MPOL_BIND */, mask, (unsigned long) (8 * sizeof(mask))) == 0;
    }
    cudaError_t e = cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocDefault);
    if (bound) syscall(SYS_set_mempolicy, 0 /* MPOL_DEFAULT */, (unsigned long *) nullptr, 0UL);
    if (e != cudaSuccess && bound) { cudaGetLastError(); e = cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocDefault); }   // node full: anywhere
    GX_CUDA(ctx, e);
    return GX_OK;
}
extern "C" int gx_host_free(gx_ctx *ctx, void *p)
{
    if (!ctx) return GX_ERR_ARG;
    if (p) GX_CUDA(ctx, cudaFreeHost(p));
    return GX_OK;
}

#define GX_COPY_CHUNK ((size_t) 64 << 20)

// allocate the device table on the compute stream (stream-ordered pool) — no copies yet
// ---- pinned staging ring for the page loader ---------------------------------------------
// gx_stage_acquire() hands out one of two pinned buffers (NUMA-bound like gx_host_alloc); a slot
// that still has a copy in flight is waited for first.  gx_table_append_heap_pages() on such a
// buffer records the slot's event after enqueueing its copies (gx_stage_mark), so the caller can
// fill the other slot meanwhile: heapgetpage/memcpy on the host overlap DMA + deform on the device.
extern "C" int gx_stage_acquire(gx_ctx *ctx, size_t bytes, void **out)
{
    if (!ctx || !out || bytes == 0) return GX_ERR_ARG;
    const int s = ctx->stage_next; ctx->stage_next ^= 1;
    if (ctx->stage_busy[s]) { GX_CUDA(ctx, cudaEventSynchronize(ctx->stage_ev[s])); ctx->stage_busy[s] = 0; }
    if (ctx->stage_bytes[s] < bytes) {
        if (ctx->stage[s]) { GX_CUDA(ctx, cudaFreeHost(ctx->stage[s])); ctx->stage[s] = nullptr; ctx->stage_bytes[s] = 0; }
        int rc = gx_host_alloc(ctx, bytes, &ctx->stage[s]); if (rc) return rc;
        ctx->stage_bytes[s] = bytes;
        if (!ctx->stage_ev[s]) GX_CUDA(ctx, cudaEventCreateWithFlags(&ctx->stage_ev[s], cudaEventDisableTiming));
    }
    *out = ctx->stage[s];
    return GX_OK;
}
cudaError_t gx_stage_mark(gx_ctx *ctx, const void *host)
{
    for (int s = 0; s < 2; s++)
        if (ctx->stage[s] && host >= ctx->stage[s] && (const char *) host < (const char *) ctx->stage[s] + ctx->stage_bytes[s]) {
            cudaError_t e = cudaEventRecord(ctx->stage_ev[s], ctx->stream);
            if (e == cudaSuccess) ctx->stage_busy[s] = 1;
            return e;
        }
    return cudaSuccess;      // not a ring buffer: pageable or caller-owned pinned memory
}

static int upload_alloc(gx_ctx *ctx, const gx_host_table *h, gx_table **out)
{
    GX_CHECK_ARG(ctx, h->ncols > 0 && h->ncols <= GX_MAX_COLS && h->nrows >= 0 && h->types && h->cols, "exec_host: bad host table");
    bool hn[GX_MAX_COLS];
    for (int c = 0; c < h->ncols; c++) { hn[c] = h->nulls && h->nulls[c]; GX_CHECK_ARG(ctx, h->cols[c] != nullptr || h->nrows == 0, "exec_host: column %d is NULL", c); }
    return gx_table_alloc_like(ctx, h->ncols, h->types, hn, h->nrows, out);
}
// queue the H2D copies of one host table on the copy streams; which = 0 inner / 1 outer event set
static int upload_copy(gx_ctx *ctx, const gx_host_table *h, gx_table *t, int which, int *rr)
{
    for (int c = 0; c < h->ncols; c++) {
        const size_t sz = (size_t) gx_type_size(h->types[c]), total = (size_t) h->nrows * sz;
        for (size_t off = 0; off < total; off += GX_COPY_CHUNK) {
            const size_t n = total - off < GX_COPY_CHUNK ? total - off : GX_COPY_CHUNK;
            GX_CUDA(ctx, cudaMemcpyAsync((char *) t->cols[c] + off, (const char *) h->cols[c] + off, n, cudaMemcpyHostToDevice,
                                         ctx->copy_streams[(*rr)++ % GX_NCOPY]));
        }
        if (t->nulls[c])
            for (size_t off = 0; off < (size_t) h->nrows; off += GX_COPY_CHUNK) {
                const size_t n = (size_t) h->nrows - off < GX_COPY_CHUNK ? (size_t) h->nrows - off : GX_COPY_CHUNK;
                GX_CUDA(ctx, cudaMemcpyAsync(t->nulls[c] + off, h->nulls[c] + off, n, cudaMemcpyHostToDevice, ctx->copy_streams[(*rr)++ % GX_NCOPY]));
            }
    }
    for (int i = 0; i < GX_NCOPY; i++) GX_CUDA(ctx, cudaEventRecord(ctx->copy_ev[which][i], ctx->copy_streams[i]));
    t->nrows = h->nrows;
    return GX_OK;
}
static int wait_copies(gx_ctx *ctx, int which)
{
    for (int i = 0; i < GX_NCOPY; i++) GX_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ctx->copy_ev[which][i], 0));
    return GX_OK;
}

extern "C" int gx_exec_host(gx_ctx *ctx, const gx_host_table *outer, const gx_host_table *inner, int inner_key_col,
                            int n_inner_preds, const gx_pred *inner_preds, int n_payload, const int32_t *payload_cols,
                            int inner_unique, const gx_agg_plan *plan, gx_result **out)
{
    if (!ctx || !outer || !plan || !out) return GX_ERR_ARG;
    int rc = gx_check_agg_join_type(ctx, plan); if (rc) return rc;      // before any upload
    gx_table *to = nullptr, *ti = nullptr; gx_hash *h = nullptr;
    const bool join = inner && plan->outer_key_col >= 0;
    int rr = 0;
    if (join) rc = upload_alloc(ctx, inner, &ti);
    if (rc == GX_OK) rc = upload_alloc(ctx, outer, &to);
    if (rc == GX_OK) {
        // the copy streams may touch the tables once the stream-ordered allocations are reached
        cudaError_t e = cudaEventRecord(ctx->ev_alloc, ctx->stream);
        for (int i = 0; i < GX_NCOPY && e == cudaSuccess; i++) e = cudaStreamWaitEvent(ctx->copy_streams[i], ctx->ev_alloc, 0);
        if (e != cudaSuccess) { GX_SET_ERR(ctx, "exec_host: %s", cudaGetErrorString(e)); rc = GX_ERR_CUDA; }
    }
    // inner first: its copy is short, and the build then runs while the (much larger) outer columns stream in
    if (rc == GX_OK && join) rc = upload_copy(ctx, inner, ti, 0, &rr);
    if (rc == GX_OK) rc = upload_copy(ctx, outer, to, 1, &rr);
    if (rc == GX_OK && join) {
        rc = wait_copies(ctx, 0);
        if (rc == GX_OK) rc = gx_hash_build(ctx, ti, inner_key_col, n_inner_preds, inner_preds, n_payload, payload_cols, inner_unique, &h);
    }
    if (rc == GX_OK) rc = wait_copies(ctx, 1);
    if (rc == GX_OK) rc = gx_hash_agg(ctx, to, h, plan, out);
    if (rc != GX_OK) for (int i = 0; i < GX_NCOPY; i++) cudaStreamSynchronize(ctx->copy_streams[i]);   // nothing may still write the tables freed below
    if (h) gx_hash_free(h);
    if (ti) gx_table_free(ti);
    if (to) gx_table_free(to);
    return rc;
}

// What the host link delivers from THIS buffer right now: `bytes` copied host -> device in 64 MB
// chunks over nstreams copy streams, three times, best rate (GB/s).  bench.py prints it beside the
// e2e figure so a slow e2e can be attributed to the box or to the code.
extern "C" int gx_h2d_probe(gx_ctx *ctx, const void *host, size_t bytes, int nstreams, double *gb_per_s)
{
    if (!ctx || !host || !gb_per_s || bytes == 0) return GX_ERR_ARG;
    if (nstreams < 1) nstreams = 1;
    if (nstreams > GX_NCOPY) nstreams = GX_NCOPY;
    void *d = nullptr;
    GX_CUDA(ctx, gx_tmp_alloc(ctx, &d, bytes));
    GX_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    cudaEvent_t a, b;
    GX_CUDA(ctx, cudaEventCreate(&a)); GX_CUDA(ctx, cudaEventCreate(&b));
    double best = 0.0;
    for (int rep = 0; rep < 3; rep++) {
        GX_CUDA(ctx, cudaEventRecord(a, ctx->stream));
        for (int i = 0; i < nstreams; i++) GX_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_streams[i], a, 0));
        int rr = 0;
        for (size_t off = 0; off < bytes; off += GX_COPY_CHUNK) {
            const size_t n = bytes - off < GX_COPY_CHUNK ? bytes - off : GX_COPY_CHUNK;
            GX_CUDA(ctx, cudaMemcpyAsync((char *) d + off, (const char *) host + off, n, cudaMemcpyHostToDevice, ctx->copy_streams[rr++ % nstreams]));
        }
        for (int i = 0; i < nstreams; i++) {
            GX_CUDA(ctx, cudaEventRecord(ctx->copy_ev[1][i], ctx->copy_streams[i]));
            GX_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ctx->copy_ev[1][i], 0));
        }
        GX_CUDA(ctx, cudaEventRecord(b, ctx->stream));
        GX_CUDA(ctx, cudaEventSynchronize(b));
        float ms = 0; GX_CUDA(ctx, cudaEventElapsedTime(&ms, a, b));
        if (ms > 0) { double r = (double) bytes / (ms / 1e3) / 1e9; if (r > best) best = r; }
    }
    cudaEventDestroy(a); cudaEventDestroy(b);
    gx_tmp_free(ctx, d);
    *gb_per_s = best;
    return GX_OK;
}
