// gx_comm.cu — K5: SHARD routing, partition-by-datanode, NCCL all-to-all
// redistribute, and the cross-datanode combine of partial aggregate states.
//
// Replaces the reference's redistribute step: GetDataRouting / EvaluateHashkey /
// GetNodeIndexByHashValue (execFragment.c:2360, locator.c:1611, shardmap.c:1147),
// FragmentSendTuple -> FnPage -> FN sender process -> TCP -> FN receiver ->
// TupleQueueThread (execFragment.c:2148, src/backend/forward/, tqueueThread.c).
// One datanode per GPU; rows travel as column slices over NVLink, counts are
// exchanged first (they replace FragmentSendCompleteMsg, execFragment.c:2953).
#include <dlfcn.h>
#include "gx_internal.cuh"

// ---- NCCL through dlopen: the same libnccl.so.2 the host process already has
// (torch's bundled copy under torchrun; the system one in a PG backend).
typedef struct { char internal[128]; } gx_ncclUniqueId;
typedef int (*fn_ncclGetUniqueId)(gx_ncclUniqueId *);
typedef int (*fn_ncclCommInitRank)(void **, int, gx_ncclUniqueId, int);
typedef int (*fn_ncclCommDestroy)(void *);
typedef int (*fn_ncclSend)(const void *, size_t, int, int, void *, cudaStream_t);
typedef int (*fn_ncclRecv)(void *, size_t, int, int, void *, cudaStream_t);
typedef int (*fn_ncclGroup)(void);
typedef int (*fn_ncclAllGather)(const void *, void *, size_t, int, void *, cudaStream_t);
typedef const char *(*fn_ncclGetErrorString)(int);
enum { GX_NCCL_INT8 = 0, GX_NCCL_INT64 = 4 };

struct gx_nccl_api {
    void *dl;
    fn_ncclGetUniqueId GetUniqueId; fn_ncclCommInitRank CommInitRank; fn_ncclCommDestroy CommDestroy;
    fn_ncclSend Send; fn_ncclRecv Recv; fn_ncclGroup GroupStart, GroupEnd; fn_ncclAllGather AllGather;
    fn_ncclGetErrorString GetErrorString;
};
static gx_nccl_api g_nccl; static bool g_nccl_loaded = false;

static int load_nccl(gx_ctx *ctx)
{
    if (g_nccl_loaded) return GX_OK;
    void *dl = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!dl) dl = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!dl) { GX_SET_ERR(ctx, "cannot load libnccl.so.2: %s", dlerror()); return GX_ERR_NCCL; }
    g_nccl.dl = dl;
#define SYM(f) g_nccl.f = (fn_nccl##f) dlsym(dl, "nccl" #f); if (!g_nccl.f) { GX_SET_ERR(ctx, "libnccl lacks nccl" #f); return GX_ERR_NCCL; }
    SYM(GetUniqueId) SYM(CommInitRank) SYM(CommDestroy) SYM(Send) SYM(Recv) SYM(AllGather) SYM(GetErrorString)
#undef SYM
    g_nccl.GroupStart = (fn_ncclGroup) dlsym(dl, "ncclGroupStart");
    g_nccl.GroupEnd = (fn_ncclGroup) dlsym(dl, "ncclGroupEnd");
    if (!g_nccl.GroupStart || !g_nccl.GroupEnd) { GX_SET_ERR(ctx, "libnccl lacks ncclGroupStart/End"); return GX_ERR_NCCL; }
    g_nccl_loaded = true;
    return GX_OK;
}
#define GX_NCCL(ctx, call) do { int r__ = (call); if (r__ != 0) { \
    GX_SET_ERR(ctx, "NCCL error %d at %s:%d: %s", r__, __FILE__, __LINE__, g_nccl.GetErrorString(r__)); return GX_ERR_NCCL; } } while (0)

extern "C" int gx_comm_unique_id(void *uid_out)
{
    if (!uid_out) return GX_ERR_ARG;
    gx_ctx *noctx = nullptr;
    int rc = load_nccl(noctx); if (rc) return rc;
    gx_ncclUniqueId id;
    GX_NCCL(noctx, g_nccl.GetUniqueId(&id));
    memcpy(uid_out, &id, sizeof(id));
    return GX_OK;
}

extern "C" int gx_set_shardmap(gx_ctx *ctx, const int32_t *shardmap, int nnodes)
{
    if (!ctx) return GX_ERR_ARG;
    GX_CHECK_ARG(ctx, nnodes >= 1 && nnodes <= GX_MAX_NODES, "set_shardmap: nnodes %d out of range", nnodes);
    int32_t map[GX_SHARD_MAP_SHARD_NUM];
    for (int i = 0; i < GX_SHARD_MAP_SHARD_NUM; i++) {
        map[i] = shardmap ? shardmap[i] : i % nnodes;            // default: catalog/pgxc_shard_map.c:93
        GX_CHECK_ARG(ctx, map[i] >= 0 && map[i] < nnodes, "set_shardmap: shard %d -> node %d out of range", i, map[i]);
    }
    GX_CUDA(ctx, cudaMemcpyAsync(ctx->d_shardmap, map, sizeof(map), cudaMemcpyHostToDevice, ctx->stream));
    GX_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->nnodes = nnodes;
    return GX_OK;
}

static int peer_setup(gx_ctx *ctx);
static void peer_teardown(gx_ctx *ctx);

extern "C" int gx_comm_init(gx_ctx *ctx, int rank, int nranks, const void *uid)
{
    if (!ctx || !uid) return GX_ERR_ARG;
    GX_CHECK_ARG(ctx, nranks >= 1 && rank >= 0 && rank < nranks, "comm_init: bad rank %d/%d", rank, nranks);
    int rc = load_nccl(ctx); if (rc) return rc;
    gx_ncclUniqueId id; memcpy(&id, uid, sizeof(id));
    void *comm = nullptr;
    GX_CUDA(ctx, cudaSetDevice(ctx->device));
    GX_NCCL(ctx, g_nccl.CommInitRank(&comm, nranks, id, rank));
    ctx->nccl = &g_nccl; ctx->comm = comm; ctx->rank = rank; ctx->nranks = nranks;
    if (ctx->nnodes != nranks) { rc = gx_set_shardmap(ctx, nullptr, nranks); if (rc) return rc; }
    return peer_setup(ctx);
}
extern "C" int gx_comm_rank(const gx_ctx *ctx, int *rank, int *nranks)
{
    if (!ctx) return GX_ERR_ARG;
    if (rank) *rank = ctx->rank;
    if (nranks) *nranks = ctx->nranks;
    return GX_OK;
}
extern "C" void gx_comm_destroy(gx_ctx *ctx)
{
    if (ctx) peer_teardown(ctx);
    if (ctx && ctx->comm && ctx->nccl) { ctx->nccl->CommDestroy(ctx->comm); ctx->comm = nullptr; ctx->nranks = 1; ctx->rank = 0; }
}

// ------------------------------------------------------------- routing
struct gx_route_args {
    gx_dcol key; long long nrows; const int32_t *shardmap; int nnodes; int _pad;
    unsigned char *dest;            // per-row destination
    long long *hist;                // hist[node * nblocks + block]
};

__device__ __forceinline__ int route_row(const gx_route_args &a, long long r)
{
    bool isnull = gx_is_null(a.key, r);
    long long datum = isnull ? 0 : gx_load_int(a.key, r);
    return a.shardmap[gx_shard_index(gx_route_hash(a.key.type, datum, isnull))];
}

__global__ void __launch_bounds__(256) gx_k_route_hist(gx_route_args a)
{
    __shared__ unsigned int sh[GX_MAX_NODES];
    if (threadIdx.x < GX_MAX_NODES) sh[threadIdx.x] = 0;
    __syncthreads();
    long long per = (a.nrows + gridDim.x - 1) / gridDim.x, b = per * blockIdx.x, e = min(a.nrows, b + per);
    for (long long r = b + threadIdx.x; r < e; r += blockDim.x) {
        int d = route_row(a, r);
        a.dest[r] = (unsigned char) d;
        atomicAdd(&sh[d], 1u);
    }
    __syncthreads();
    if (threadIdx.x < a.nnodes) a.hist[(long long) threadIdx.x * gridDim.x + blockIdx.x] = sh[threadIdx.x];
}

struct gx_scatter_args {
    long long nrows; int ncols, nnodes;
    const unsigned char *dest; const long long *offs;
    gx_dcol in[GX_MAX_COLS]; void *out[GX_MAX_COLS]; uint8_t *out_nulls[GX_MAX_COLS];
};
// Row order inside a destination is unspecified (as with the reference's FN pages).
__global__ void __launch_bounds__(256) gx_k_route_scatter(gx_scatter_args a)
{
    __shared__ unsigned int cur[GX_MAX_NODES];
    if (threadIdx.x < GX_MAX_NODES) cur[threadIdx.x] = 0;
    __syncthreads();
    long long per = (a.nrows + gridDim.x - 1) / gridDim.x, b = per * blockIdx.x, e = min(a.nrows, b + per);
    const int lane = threadIdx.x & 31;
    for (long long r0 = b; r0 < e; r0 += blockDim.x) {
        long long r = r0 + threadIdx.x;
        bool valid = r < e;
        int d = valid ? a.dest[r] : -1;
        if (valid) {
            unsigned int m = __match_any_sync(__activemask(), d);
            int leader = __ffs(m) - 1;
            unsigned int base = 0;
            if (lane == leader) base = atomicAdd(&cur[d], (unsigned int) __popc(m));
            base = __shfl_sync(m, base, leader);
            long long dst = a.offs[(long long) d * gridDim.x + blockIdx.x] + base + __popc(m & ((1u << lane) - 1));
            for (int c = 0; c < a.ncols; c++) {
                switch (a.in[c].type) {
                    case GX_INT4: case GX_DATE: ((int *) a.out[c])[dst] = ((const int *) a.in[c].data)[r]; break;
                    case GX_CHAR: ((signed char *) a.out[c])[dst] = ((const signed char *) a.in[c].data)[r]; break;
                    default: ((long long *) a.out[c])[dst] = ((const long long *) a.in[c].data)[r]; break;
                }
                if (a.out_nulls[c]) a.out_nulls[c][dst] = a.in[c].nulls ? a.in[c].nulls[r] : 0;
            }
        }
    }
}

__global__ void gx_k_scan_i64(long long *v, long long n, long long *total);   // gx_agg.cu

static int route_setup(gx_ctx *ctx, const gx_table *in, int key_col, gx_route_args *a, unsigned *nblk_out)
{
    GX_CHECK_ARG(ctx, key_col >= 0 && key_col < in->ncols, "route: key column %d out of range", key_col);
    int kt = in->types[key_col];
    GX_CHECK_ARG(ctx, kt == GX_INT4 || kt == GX_INT8 || kt == GX_DATE, "route: distribution column type %d not supported (int4/int8/date)", kt);
    memset(a, 0, sizeof(*a));
    a->key.data = in->cols[key_col]; a->key.nulls = in->nulls[key_col]; a->key.type = kt;
    a->nrows = in->nrows; a->shardmap = ctx->d_shardmap; a->nnodes = ctx->nnodes;
    unsigned nblk = (unsigned) (ctx->sm_count * 4);
    if ((long long) nblk * 256 > in->nrows) nblk = (unsigned) ((in->nrows + 255) / 256);
    if (nblk == 0) nblk = 1;
    *nblk_out = nblk;
    GX_CUDA(ctx, gx_tmp_alloc(ctx, (void **) &a->dest, (size_t) (in->nrows > 0 ? in->nrows : 1)));
    GX_CUDA(ctx, gx_tmp_alloc(ctx, (void **) &a->hist, (size_t) ctx->nnodes * nblk * sizeof(long long)));
    return GX_OK;
}

extern "C" int gx_route(gx_ctx *ctx, const gx_table *in, int key_col, int32_t *host_dest_out)
{
    if (!ctx || !in || !host_dest_out) return GX_ERR_ARG;
    gx_route_args a; unsigned nblk;
    int rc = route_setup(ctx, in, key_col, &a, &nblk); if (rc) return rc;
    { gx_launch_scope ls(ctx, "route"); gx_k_route_hist<<<nblk, 256, 0, ctx->stream>>>(a); }
    unsigned char *h = (unsigned char *) malloc((size_t) in->nrows + 1);
    cudaError_t e = cudaMemcpyAsync(h, a.dest, (size_t) in->nrows, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    for (int64_t i = 0; i < in->nrows; i++) host_dest_out[i] = h[i];
    free(h); gx_tmp_free(ctx, a.dest); gx_tmp_free(ctx, a.hist);
    if (e != cudaSuccess) { GX_SET_ERR(ctx, "route: %s", cudaGetErrorString(e)); return GX_ERR_CUDA; }
    return GX_OK;
}

// partition rows by destination node into a new table; counts[node] on the host
static int partition_impl(gx_ctx *ctx, const gx_table *in, int key_col, gx_table **out, int64_t *host_counts)
{
    gx_route_args a; unsigned nblk;
    int rc = route_setup(ctx, in, key_col, &a, &nblk); if (rc) return rc;
    bool hn[GX_MAX_COLS];
    for (int c = 0; c < in->ncols; c++) hn[c] = in->nulls[c] != nullptr;
    gx_table *t;
    rc = gx_table_alloc_like(ctx, in->ncols, in->types, hn, in->nrows, &t);
    if (rc) { gx_tmp_free(ctx, a.dest); gx_tmp_free(ctx, a.hist); return rc; }
    gx_scatter_args s; memset(&s, 0, sizeof(s));
    s.nrows = in->nrows; s.ncols = in->ncols; s.nnodes = ctx->nnodes; s.dest = a.dest; s.offs = a.hist;
    for (int c = 0; c < in->ncols; c++) {
        s.in[c].data = in->cols[c]; s.in[c].nulls = in->nulls[c]; s.in[c].type = in->types[c];
        s.out[c] = t->cols[c]; s.out_nulls[c] = t->nulls[c];
    }
    long long *h_offs = (long long *) malloc((size_t) ctx->nnodes * sizeof(long long));
    {
        gx_launch_scope ls(ctx, "partition", 3);
        gx_k_route_hist<<<nblk, 256, 0, ctx->stream>>>(a);
        gx_k_scan_i64<<<1, 1024, 0, ctx->stream>>>(a.hist, (long long) ctx->nnodes * nblk, nullptr);
        // node offsets = scanned hist at (node, block 0)
        cudaMemcpy2DAsync(h_offs, sizeof(long long), a.hist, (size_t) nblk * sizeof(long long), sizeof(long long), ctx->nnodes,
                          cudaMemcpyDeviceToHost, ctx->stream);
        gx_k_route_scatter<<<nblk, 256, 0, ctx->stream>>>(s);
    }
    cudaError_t e = cudaStreamSynchronize(ctx->stream);
    gx_tmp_free(ctx, a.dest); gx_tmp_free(ctx, a.hist);
    if (e != cudaSuccess) { free(h_offs); gx_table_free(t); GX_SET_ERR(ctx, "partition: %s", cudaGetErrorString(e)); return GX_ERR_CUDA; }
    for (int n = 0; n < ctx->nnodes; n++)
        host_counts[n] = ((n + 1 < ctx->nnodes) ? h_offs[n + 1] : in->nrows) - h_offs[n];
    free(h_offs);
    t->nrows = in->nrows;
    *out = t;
    return GX_OK;
}

// ---- one pass: route + scatter into fixed-capacity per-destination regions ----------------
// The two-pass form above reads the key column twice and the rows once more (histogram, scan,
// scatter).  For the redistribute itself the destinations only have to be contiguous PER
// DESTINATION, not densely packed: region d starts at d * cap rows, so a tile can claim its
// ranges with one global atomic per destination as soon as it has its own counts.  A CTA takes
// tiles of 2048 rows: destination and tile-local position of every row (warp-aggregated shared
// atomics), one claim per destination, then the copy.  cap = rows / N * 1.25 (SHARD placement of
// the default map is balanced to a percent); a region that would overflow raises a flag and the
// caller falls back to the exact two-pass form.
#define RP_THREADS 256
#define RP_K 8
struct gx_route1_args {
    gx_dcol key; long long nrows; const int32_t *shardmap; int nnodes, ncols;
    gx_dcol in[GX_MAX_COLS]; void *out[GX_MAX_COLS]; uint8_t *out_nulls[GX_MAX_COLS];
    long long cap; unsigned long long *cursor;   // [nnodes] rows claimed per destination; [GX_MAX_NODES] overflow flag
};
__global__ void __launch_bounds__(RP_THREADS, 4) gx_k_route_onepass(gx_route1_args a)     // 4 CTAs/SM (64 registers)
{
    __shared__ unsigned int cur[GX_MAX_NODES];
    __shared__ long long tbase[GX_MAX_NODES];
    const int lane = threadIdx.x & 31;
    const long long tile_rows = (long long) RP_THREADS * RP_K;
    for (long long base = (long long) blockIdx.x * tile_rows; base < a.nrows; base += (long long) gridDim.x * tile_rows) {
        if (threadIdx.x < GX_MAX_NODES) cur[threadIdx.x] = 0;
        __syncthreads();
        int d[RP_K]; unsigned int lp[RP_K];
#pragma unroll
        for (int k = 0; k < RP_K; k++) {
            const long long r = base + k * RP_THREADS + threadIdx.x;
            d[k] = -1; lp[k] = 0;
            if (r < a.nrows) {
                const bool isnull = gx_is_null(a.key, r);
                const long long datum = isnull ? 0 : gx_load_int(a.key, r);
                d[k] = a.shardmap[gx_shard_index(gx_route_hash(a.key.type, datum, isnull))];
                const unsigned int m = __match_any_sync(__activemask(), d[k]);
                const int leader = __ffs(m) - 1;
                unsigned int off = 0;
                if (lane == leader) off = atomicAdd(&cur[d[k]], (unsigned int) __popc(m));
                lp[k] = __shfl_sync(m, off, leader) + __popc(m & ((1u << lane) - 1));
            }
        }
        __syncthreads();
        if (threadIdx.x < a.nnodes) {
            const unsigned int n = cur[threadIdx.x];
            long long b = n ? (long long) atomicAdd(&a.cursor[threadIdx.x], (unsigned long long) n) : 0;
            if (b + n > a.cap) { atomicExch(&a.cursor[GX_MAX_NODES], 1ULL); b = -1; }
            tbase[threadIdx.x] = b;
        }
        __syncthreads();
        long long rr[RP_K], dd[RP_K]; bool keep[RP_K];
#pragma unroll
        for (int k = 0; k < RP_K; k++) {
            keep[k] = d[k] >= 0 && tbase[d[k] < 0 ? 0 : d[k]] >= 0;
            rr[k] = base + k * RP_THREADS + threadIdx.x;
            dd[k] = keep[k] ? (long long) d[k] * a.cap + tbase[d[k]] + lp[k] : 0;
        }
        for (int c = 0; c < a.ncols; c++) gx_copy_rows<RP_K>(a.in[c], a.out[c], a.out_nulls[c], rr, dd, keep);
        __syncthreads();
    }
}

// regions of `cap` rows per destination; returns GX_OK with *overflowed = 1 when a region was too small
static int partition_regions(gx_ctx *ctx, const gx_table *in, int key_col, gx_table **out, int64_t *host_counts, long long *cap_out, int *overflowed)
{
    GX_CHECK_ARG(ctx, key_col >= 0 && key_col < in->ncols, "route: key column %d out of range", key_col);
    const int kt = in->types[key_col], N = ctx->nnodes;
    GX_CHECK_ARG(ctx, kt == GX_INT4 || kt == GX_INT8 || kt == GX_DATE, "route: distribution column type %d not supported (int4/int8/date)", kt);
    const long long cap = N == 1 ? (in->nrows > 0 ? in->nrows : 1) : in->nrows / N + in->nrows / (4 * N) + 4096;
    bool hn[GX_MAX_COLS];
    for (int c = 0; c < in->ncols; c++) hn[c] = in->nulls[c] != nullptr;
    gx_table *t;
    int rc = gx_table_alloc_like(ctx, in->ncols, in->types, hn, cap * N, &t); if (rc) return rc;
    gx_route1_args a; memset(&a, 0, sizeof(a));
    a.key.data = in->cols[key_col]; a.key.nulls = in->nulls[key_col]; a.key.type = kt;
    a.nrows = in->nrows; a.shardmap = ctx->d_shardmap; a.nnodes = N; a.ncols = in->ncols; a.cap = cap;
    for (int c = 0; c < in->ncols; c++) {
        a.in[c].data = in->cols[c]; a.in[c].nulls = in->nulls[c]; a.in[c].type = in->types[c];
        a.out[c] = t->cols[c]; a.out_nulls[c] = t->nulls[c];
    }
    unsigned long long *d_cur;
    GX_CUDA(ctx, gx_tmp_alloc(ctx, (void **) &d_cur, (GX_MAX_NODES + 1) * 8));
    GX_CUDA(ctx, cudaMemsetAsync(d_cur, 0, (GX_MAX_NODES + 1) * 8, ctx->stream));
    a.cursor = d_cur;
    if (in->nrows > 0) {
        const long long tiles = (in->nrows + RP_THREADS * RP_K - 1) / (RP_THREADS * RP_K), maxb = (long long) ctx->sm_count * 8;
        gx_launch_scope ls(ctx, "partition");
        gx_k_route_onepass<<<(unsigned) (tiles < maxb ? tiles : maxb), RP_THREADS, 0, ctx->stream>>>(a);
    }
    unsigned long long h_cur[GX_MAX_NODES + 1];
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(h_cur, d_cur, sizeof(h_cur), cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    gx_tmp_free(ctx, d_cur);
    if (e != cudaSuccess) { gx_table_free(t); GX_SET_ERR(ctx, "partition: %s", cudaGetErrorString(e)); return GX_ERR_CUDA; }
    *overflowed = h_cur[GX_MAX_NODES] != 0;
    if (*overflowed) { gx_table_free(t); *out = nullptr; return GX_OK; }
    for (int n = 0; n < N; n++) host_counts[n] = (int64_t) h_cur[n];
    t->nrows = N == 1 ? in->nrows : cap * N;
    *cap_out = cap;
    *out = t;
    return GX_OK;
}

extern "C" int gx_partition_by_node(gx_ctx *ctx, const gx_table *in, int key_col, gx_table **out, int64_t *host_counts)
{
    if (!ctx || !in || !out || !host_counts) return GX_ERR_ARG;
    return partition_impl(ctx, in, key_col, out, host_counts);
}

// all-to-all of byte slices: sendbuf split by sendcnt (bytes), recvbuf by recvcnt
static int alltoallv_bytes(gx_ctx *ctx, const char *sendbuf, const int64_t *sendoff, const int64_t *sendcnt,
                           char *recvbuf, const int64_t *recvoff, const int64_t *recvcnt)
{
    GX_NCCL(ctx, g_nccl.GroupStart());
    for (int p = 0; p < ctx->nranks; p++) {
        if (sendcnt[p]) GX_NCCL(ctx, g_nccl.Send(sendbuf + sendoff[p], (size_t) sendcnt[p], GX_NCCL_INT8, p, ctx->comm, ctx->stream));
        if (recvcnt[p]) GX_NCCL(ctx, g_nccl.Recv(recvbuf + recvoff[p], (size_t) recvcnt[p], GX_NCCL_INT8, p, ctx->comm, ctx->stream));
    }
    GX_NCCL(ctx, g_nccl.GroupEnd());
    return GX_OK;
}

// exchange a small int64 vector: every rank learns every rank's vector
static int allgather_i64(gx_ctx *ctx, const int64_t *mine, int n, int64_t *all /* nranks*n */)
{
    long long *d_in, *d_out;
    GX_CUDA(ctx, gx_tmp_alloc(ctx, (void **) &d_in, (size_t) n * 8));
    GX_CUDA(ctx, gx_tmp_alloc(ctx, (void **) &d_out, (size_t) n * 8 * ctx->nranks));
    GX_CUDA(ctx, cudaMemcpyAsync(d_in, mine, (size_t) n * 8, cudaMemcpyHostToDevice, ctx->stream));
    GX_NCCL(ctx, g_nccl.AllGather(d_in, d_out, (size_t) n, GX_NCCL_INT64, ctx->comm, ctx->stream));
    GX_CUDA(ctx, cudaMemcpyAsync(all, d_out, (size_t) n * 8 * ctx->nranks, cudaMemcpyDeviceToHost, ctx->stream));
    GX_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    gx_tmp_free(ctx, d_in); gx_tmp_free(ctx, d_out);
    return GX_OK;
}


// ------------------------------------------------------------- redistribute over peer memory
// The reference's sender copies each tuple into the destination's FnPage and hands the page to the
// forwarder (ExecSendRemoteFragment, execFragment.c:3505-3652; FnPageAddItem, fnbufpage.c:50-85).
// On one NVSwitch node the destination's memory is addressable: every rank owns a window, all windows
// are mapped into all processes (CUDA IPC), and the routing kernel stores each row straight into the
// destination's window - routing, serialisation and transport are one kernel, nothing is staged locally
// and no collective runs.  Window of rank d: N regions, region s written only by rank s (columnar, `cap`
// rows per column, cap chosen by the writer).  Control words of rank d: hdr[s] = {epoch, rows, cap,
// nullbits} written by s after its rows; ack[d'] written by d' once it has copied epoch's rows out of
// ITS window, so the writer knows the regions it owns there may be overwritten.
// All ranks see all headers, so "someone's region overflowed" is common knowledge and every rank takes
// the NCCL path for that call together.
#define PEER_CTL_BYTES 4096
#define PEER_HDR(base, s) ((unsigned long long *) (base) + (size_t) (s) * 4)
#define PEER_ACK(base, d) ((unsigned long long *) (base) + 256 + (d))
#define PEER_FALLBACK 0xffffffffffffffffULL

static inline long long peer_align(long long b) { return (b + 255) & ~255LL; }
// byte offset of column c (or of its NULL array) inside a region laid out for `cap` rows; c == ncols: region size
__host__ __device__ static inline long long peer_layout(long long cap, int ncols, const int *sizes, unsigned long long nullbits, int c, int want_null)
{
    long long off = 0;
    for (int i = 0; i < ncols; i++) { if (!want_null && i == c) return off; off += (cap * sizes[i] + 255) & ~255LL; }
    for (int i = 0; i < ncols; i++) if ((nullbits >> i) & 1ULL) { if (want_null && i == c) return off; off += (cap + 255) & ~255LL; }
    return off;
}

static int allgather_i64(gx_ctx *ctx, const int64_t *mine, int n, int64_t *all);

// Collective like the set-up: an exporter must not free its block while a peer still has it mapped (or has an
// acknowledgement store in flight towards it), so the ranks meet once before the imports are closed and once before
// the blocks are freed.  GX_PEER_TEARDOWN_SYNC=0 skips the two rendezvous (a rank that is known to be alone).
static void peer_teardown(gx_ctx *ctx)
{
    if (ctx->peer_ready != 1) { ctx->peer_ready = 0; return; }
    const char *ts = getenv("GX_PEER_TEARDOWN_SYNC");
    const bool meet = ctx->comm && !(ts && ts[0] == '0');
    int64_t one = 1, all[GX_MAX_NODES];
    cudaStreamSynchronize(ctx->stream);
    if (meet) allgather_i64(ctx, &one, 1, all);                 // every rank's stores into the peers' blocks have completed
    for (int p = 0; p < ctx->nranks; p++) if (p != ctx->rank && ctx->peer_base[p]) cudaIpcCloseMemHandle(ctx->peer_base[p]);
    if (meet) allgather_i64(ctx, &one, 1, all);                 // nobody has this rank's block mapped any more
    if (ctx->peer_base[ctx->rank]) cudaFree(ctx->peer_base[ctx->rank]);
    memset(ctx->peer_base, 0, sizeof(ctx->peer_base));
    ctx->peer_ready = 0;
}

// Collective (called from gx_comm_init): allocate the window, exchange IPC handles through the communicator,
// map the peers.  Any rank failing any step makes every rank give the windows up (peer_ready = -1): the
// decision must be the same everywhere.  GX_PEER_WINDOW_MB (default 4096; 0 = no windows), GX_NO_PEER=1.
static int peer_setup(gx_ctx *ctx)
{
    const int N = ctx->nranks;
    ctx->peer_ready = -1; ctx->peer_epoch = 0;
    if (N < 2) return GX_OK;
    const char *no = getenv("GX_NO_PEER"), *mb = getenv("GX_PEER_WINDOW_MB");
    long long win_mb = mb ? atoll(mb) : 4096;
    if ((no && no[0] == '1') || win_mb <= 0) win_mb = 0;
    int64_t mine[16], *all = (int64_t *) calloc((size_t) N * 16, 8);
    memset(mine, 0, sizeof(mine));
    char *own = nullptr;
    cudaIpcMemHandle_t h;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle travels as 8 int64");
    if (win_mb > 0 && cudaMalloc((void **) &own, PEER_CTL_BYTES + ((size_t) win_mb << 20)) == cudaSuccess &&
        cudaMemset(own, 0, PEER_CTL_BYTES) == cudaSuccess && cudaIpcGetMemHandle(&h, own) == cudaSuccess) {
        memcpy(mine, &h, 64); mine[8] = 1; mine[9] = win_mb;
    } else {
        cudaGetLastError();
        if (own) { cudaFree(own); own = nullptr; }
    }
    int rc = allgather_i64(ctx, mine, 16, all);
    if (rc) { if (own) cudaFree(own); free(all); return rc; }
    bool ok = true;
    for (int p = 0; p < N; p++) ok = ok && all[(size_t) p * 16 + 8] == 1 && all[(size_t) p * 16 + 9] == win_mb;
    memset(ctx->peer_base, 0, sizeof(ctx->peer_base));
    int64_t mapped = ok ? 1 : 0;
    if (ok) {
        ctx->peer_base[ctx->rank] = own;
        for (int p = 0; p < N && mapped; p++) {
            if (p == ctx->rank) continue;
            cudaIpcMemHandle_t hp; memcpy(&hp, all + (size_t) p * 16, 64);
            void *ptr = nullptr;
            if (cudaIpcOpenMemHandle(&ptr, hp, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); mapped = 0; }
            else ctx->peer_base[p] = (char *) ptr;
        }
    }
    // second round: did everybody map everybody?
    int64_t *all2 = (int64_t *) calloc((size_t) N, 8);
    rc = allgather_i64(ctx, &mapped, 1, all2);
    bool all_mapped = rc == GX_OK;
    for (int p = 0; p < N && all_mapped; p++) all_mapped = all2[p] == 1;
    free(all); free(all2);
    if (!all_mapped) {
        for (int p = 0; p < N; p++) if (p != ctx->rank && ctx->peer_base[p]) cudaIpcCloseMemHandle(ctx->peer_base[p]);
        if (own) cudaFree(own);
        memset(ctx->peer_base, 0, sizeof(ctx->peer_base));
        return rc;
    }
    ctx->peer_win_bytes = (size_t) win_mb << 20;
    ctx->peer_ready = 1;
    return GX_OK;
}

__device__ __forceinline__ unsigned long long peer_load(const unsigned long long *p)
{
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void peer_store(unsigned long long *p, unsigned long long v)
{
    asm volatile("st.release.sys.global.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long peer_now_ns()
{
    unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); return t;
}

struct gx_peer_ptrs { char *base[GX_MAX_NODES]; };

// thread i waits until word i of `words` (own control block) reaches `want`; *timed_out is raised instead of hanging
__global__ void gx_k_peer_wait(const unsigned long long *words, int stride, int n, unsigned long long want, unsigned long long timeout_ns,
                               int *timed_out, unsigned long long *hdr_out)
{
    const int i = threadIdx.x;
    if (i >= n) return;
    const unsigned long long *w = words + (size_t) i * stride;
    const unsigned long long t0 = peer_now_ns();
    unsigned int spins = 0;
    while (peer_load(w) < want) {
        if ((++spins & 1023u) == 0 && peer_now_ns() - t0 > timeout_ns) { atomicExch(timed_out, 1); return; }
        __nanosleep(200);
    }
    if (hdr_out) { hdr_out[i * 3 + 0] = w[1]; hdr_out[i * 3 + 1] = w[2]; hdr_out[i * 3 + 2] = w[3]; }
}

// after the routing kernel: thread d tells rank d how many rows of this rank lie in its window (or that this
// rank cannot use the windows for this call)
__global__ void gx_k_peer_publish(gx_peer_ptrs P, int n, int self, unsigned long long epoch, const unsigned long long *cursor, int feasible,
                                  unsigned long long cap, unsigned long long nullbits)
{
    const int d = threadIdx.x;
    if (d >= n) return;
    const bool bad = !feasible || cursor[GX_MAX_NODES] != 0;
    unsigned long long *h = PEER_HDR(P.base[d], self);
    h[1] = bad ? PEER_FALLBACK : cursor[d]; h[2] = cap; h[3] = nullbits;
    __threadfence_system();
    peer_store(h, epoch);
}

// after the copy-out: thread s tells rank s that its region in this rank's window is free again
__global__ void gx_k_peer_ack(gx_peer_ptrs P, int n, int self, unsigned long long epoch)
{
    const int s = threadIdx.x;
    if (s >= n) return;
    __threadfence_system();
    peer_store(PEER_ACK(P.base[s], self), epoch);
}

// Route + serialise + transport in one kernel.  Tiles of 2048 rows: destination and tile-local position of every
// row, one claim per destination in this rank's region there, then per column the tile is grouped by destination
// in shared memory and leaves as contiguous runs (full 128-byte lines on the NVLink side, not 8-byte scatters).
#define PR_THREADS 256
#define PR_K 8
struct gx_peer_route_args {
    gx_dcol key; long long nrows; const int32_t *shardmap; int nnodes, ncols;
    gx_dcol in[GX_MAX_COLS];
    long long coff[GX_MAX_COLS], noff[GX_MAX_COLS];     // byte offset of the column / its NULL array inside a region (noff < 0: none)
    char *dst[GX_MAX_NODES];                             // this rank's region in the window of each destination
    long long cap; unsigned long long *cursor;           // [nnodes] rows claimed per destination; [GX_MAX_NODES] overflow flag
};
__global__ void __launch_bounds__(PR_THREADS) gx_k_route_peer(const __grid_constant__ gx_peer_route_args a)
{
    __shared__ unsigned int cur[GX_MAX_NODES];
    __shared__ unsigned int toff[GX_MAX_NODES + 1];
    __shared__ long long tbase[GX_MAX_NODES];
    __shared__ long long stage[PR_THREADS * PR_K];
    const int lane = threadIdx.x & 31;
    const long long tile_rows = (long long) PR_THREADS * PR_K;
    for (long long base = (long long) blockIdx.x * tile_rows; base < a.nrows; base += (long long) gridDim.x * tile_rows) {
        if (threadIdx.x < GX_MAX_NODES) cur[threadIdx.x] = 0;
        __syncthreads();
        int d[PR_K]; unsigned int lp[PR_K];
#pragma unroll
        for (int k = 0; k < PR_K; k++) {
            const long long r = base + k * PR_THREADS + threadIdx.x;
            d[k] = -1; lp[k] = 0;
            if (r < a.nrows) {
                const bool isnull = gx_is_null(a.key, r);
                const long long datum = isnull ? 0 : gx_load_int(a.key, r);
                d[k] = a.shardmap[gx_shard_index(gx_route_hash(a.key.type, datum, isnull))];
                const unsigned int m = __match_any_sync(__activemask(), d[k]);
                const int leader = __ffs(m) - 1;
                unsigned int off = 0;
                if (lane == leader) off = atomicAdd(&cur[d[k]], (unsigned int) __popc(m));
                lp[k] = __shfl_sync(m, off, leader) + __popc(m & ((1u << lane) - 1));
            }
        }
        __syncthreads();
        if (threadIdx.x < a.nnodes) {
            const unsigned int n = cur[threadIdx.x];
            long long b = n ? (long long) atomicAdd(&a.cursor[threadIdx.x], (unsigned long long) n) : 0;
            if (b + n > a.cap) { atomicExch(&a.cursor[GX_MAX_NODES], 1ULL); b = -1; }
            tbase[threadIdx.x] = b;
        }
        if (threadIdx.x == 32) {
            unsigned int run = 0;
            for (int n = 0; n < a.nnodes; n++) { toff[n] = run; run += cur[n]; }
            toff[a.nnodes] = run;
        }
        __syncthreads();
        unsigned int si[PR_K];
#pragma unroll
        for (int k = 0; k < PR_K; k++) si[k] = d[k] >= 0 ? toff[d[k]] + lp[k] : 0xffffffffu;
        const unsigned int total = toff[a.nnodes];
        for (int c = 0; c < a.ncols; c++) {
            const int ty = a.in[c].type;
            const int sz = (ty == GX_INT4 || ty == GX_DATE) ? 4 : (ty == GX_CHAR ? 1 : 8);
            for (int pass = 0; pass < 2; pass++) {                  // 0: the column, 1: its NULL bytes
                if (pass == 1 && a.noff[c] < 0) break;
                const int esz = pass ? 1 : sz;
                if (pass == 0 && sz == 8) {
                    long long v[PR_K];
#pragma unroll
                    for (int k = 0; k < PR_K; k++) v[k] = d[k] >= 0 ? __ldg((const long long *) a.in[c].data + base + k * PR_THREADS + threadIdx.x) : 0;
#pragma unroll
                    for (int k = 0; k < PR_K; k++) if (d[k] >= 0) stage[si[k]] = v[k];
                } else if (pass == 0 && sz == 4) {
                    int v[PR_K];
#pragma unroll
                    for (int k = 0; k < PR_K; k++) v[k] = d[k] >= 0 ? __ldg((const int *) a.in[c].data + base + k * PR_THREADS + threadIdx.x) : 0;
#pragma unroll
                    for (int k = 0; k < PR_K; k++) if (d[k] >= 0) ((int *) stage)[si[k]] = v[k];
                } else {
                    const unsigned char *src = pass ? a.in[c].nulls : (const unsigned char *) a.in[c].data;
#pragma unroll
                    for (int k = 0; k < PR_K; k++) if (d[k] >= 0) ((unsigned char *) stage)[si[k]] = src ? src[base + k * PR_THREADS + threadIdx.x] : 0;
                }
                __syncthreads();
                const long long coff = pass ? a.noff[c] : a.coff[c];
                int n = 0;
                for (unsigned int i = threadIdx.x; i < total; i += PR_THREADS) {
                    while (i >= toff[n + 1]) n++;
                    const long long tb = tbase[n];
                    if (tb < 0) continue;
                    char *out = a.dst[n] + coff;
                    const long long pos = tb + (long long) (i - toff[n]);
                    if (esz == 8) ((long long *) out)[pos] = stage[i];
                    else if (esz == 4) ((int *) out)[pos] = ((const int *) stage)[i];
                    else ((unsigned char *) out)[pos] = ((const unsigned char *) stage)[i];
                }
                __syncthreads();
            }
        }
    }
}

// copy-out on the receiving side: region s of the own window -> rows [sum of earlier counts, +count[s]) of the table
struct gx_peer_gather_args {
    int nnodes, ncols; int sizes[GX_MAX_COLS];
    const char *win; long long region_stride;
    long long count[GX_MAX_NODES], cap[GX_MAX_NODES]; unsigned long long nullbits[GX_MAX_NODES];
    void *out[GX_MAX_COLS]; uint8_t *out_nulls[GX_MAX_COLS];
};
__global__ void __launch_bounds__(256) gx_k_peer_gather(const __grid_constant__ gx_peer_gather_args a)
{
    const int s = blockIdx.y, c = blockIdx.z % a.ncols, want_null = blockIdx.z / a.ncols;
    if (want_null && !a.out_nulls[c]) return;
    long long first = 0;
    for (int i = 0; i < s; i++) first += a.count[i];
    const long long n = a.count[s];
    const bool src_has = !want_null || ((a.nullbits[s] >> c) & 1ULL);
    const char *src = a.win + (long long) s * a.region_stride + peer_layout(a.cap[s], a.ncols, a.sizes, a.nullbits[s], c, want_null);
    const int sz = want_null ? 1 : a.sizes[c];
    const long long step = (long long) gridDim.x * blockDim.x, i0 = (long long) blockIdx.x * blockDim.x + threadIdx.x;
    if (sz == 8 || sz == 4) {
        // four independent loads in flight per thread
        long long i = i0;
        for (; i + 3 * step < n; i += 4 * step) {
            if (sz == 8) {
                long long v[4];
#pragma unroll
                for (int j = 0; j < 4; j++) v[j] = ((const long long *) src)[i + j * step];
#pragma unroll
                for (int j = 0; j < 4; j++) ((long long *) a.out[c])[first + i + j * step] = v[j];
            } else {
                int v[4];
#pragma unroll
                for (int j = 0; j < 4; j++) v[j] = ((const int *) src)[i + j * step];
#pragma unroll
                for (int j = 0; j < 4; j++) ((int *) a.out[c])[first + i + j * step] = v[j];
            }
        }
        for (; i < n; i += step) {
            if (sz == 8) ((long long *) a.out[c])[first + i] = ((const long long *) src)[i];
            else ((int *) a.out[c])[first + i] = ((const int *) src)[i];
        }
        return;
    }
    for (long long i = i0; i < n; i += step) {
        if (!want_null) ((unsigned char *) a.out[c])[first + i] = ((const unsigned char *) src)[i];
        else a.out_nulls[c][first + i] = src_has ? ((const unsigned char *) src)[i] : 0;
    }
}

// What the redistribute of table rows exchanges between ranks.  redistribute_run makes every decision and runs every
// device step; a transport only moves bytes and headers: through the peer windows and NCCL between processes, or in
// one process on one GPU, where it builds from the input tables of all ranks what the other ranks would have delivered
// to one of them (gx_debug_redistribute).
struct gx_redist_transport {
    int rank, nranks;
    size_t window_bytes;            // window of every rank; 0: no peer windows, every call takes the NCCL path
    // dst[d] = this rank's region in the window of rank d, once the rows of the previous call have left it
    virtual int window_open(gx_ctx *ctx, long long region_stride, char **dst) = 0;
    // after this rank's rows are in the windows (d_cur: its cursor, see peer_route): the header of every source s of
    // this rank's window, hdr[s * 3 + {0, 1, 2}] = {rows (PEER_FALLBACK: s cannot use the windows), cap, nullbits};
    // *win = this rank's window, region s at s * region_stride
    virtual int window_headers(gx_ctx *ctx, const unsigned long long *d_cur, int feasible, long long cap, unsigned long long nullbits,
                               unsigned long long *hdr, const char **win) = 0;
    // nothing more of this call is read from this rank's window
    virtual void window_release(gx_ctx *ctx) = 0;
    // all[p * n + i] = word i of rank p's `mine`
    virtual int gather_counts(gx_ctx *ctx, const int64_t *mine, int n, int64_t *all) = 0;
    // the bytes of column c (want_null: its NULL bytes) every rank addressed to this one, rank p's at ro[p] of recvbuf;
    // sendbuf, so and sc are this rank's
    virtual int exchange_column(gx_ctx *ctx, int c, int want_null, const char *sendbuf, const int64_t *so, const int64_t *sc,
                                char *recvbuf, const int64_t *ro, const int64_t *rcn) = 0;
};

// One rank's rows into its regions of the N destinations' windows (dst[d]).  d_cur[GX_MAX_NODES + 1], zeroed by the
// caller, receives the rows per destination and the overflow flag.  The rank chooses the layout of its regions itself
// (*cap, *nullbits); *feasible = 0 when a region of that layout does not fit region_stride, and nothing is routed.
static int peer_route(gx_ctx *ctx, const gx_table *in, int key_col, int N, long long region_stride, char *const *dst,
                      unsigned long long *d_cur, long long *cap_out, unsigned long long *nullbits_out, int *feasible_out)
{
    const int kt = in->types[key_col];
    int sizes[GX_MAX_COLS]; unsigned long long nullbits = 0;
    for (int c = 0; c < in->ncols; c++) { sizes[c] = gx_type_size(in->types[c]); if (in->nulls[c]) nullbits |= 1ULL << c; }
    const long long cap = in->nrows / N + in->nrows / (4 * N) + 4096;
    const int feasible = peer_layout(cap, in->ncols, sizes, nullbits, in->ncols, 0) <= region_stride;
    if (feasible && in->nrows > 0) {
        gx_peer_route_args a; memset(&a, 0, sizeof(a));
        a.key.data = in->cols[key_col]; a.key.nulls = in->nulls[key_col]; a.key.type = kt;
        a.nrows = in->nrows; a.shardmap = ctx->d_shardmap; a.nnodes = N; a.ncols = in->ncols; a.cap = cap; a.cursor = d_cur;
        for (int c = 0; c < in->ncols; c++) {
            a.in[c].data = in->cols[c]; a.in[c].nulls = in->nulls[c]; a.in[c].type = in->types[c];
            a.coff[c] = peer_layout(cap, in->ncols, sizes, nullbits, c, 0);
            a.noff[c] = in->nulls[c] ? peer_layout(cap, in->ncols, sizes, nullbits, c, 1) : -1;
        }
        for (int p = 0; p < N; p++) a.dst[p] = dst[p];
        const long long tiles = (in->nrows + PR_THREADS * PR_K - 1) / (PR_THREADS * PR_K), maxb = (long long) ctx->sm_count * 8;
        gx_launch_scope ls(ctx, "peer_scatter");
        gx_k_route_peer<<<(unsigned) (tiles < maxb ? tiles : maxb), PR_THREADS, 0, ctx->stream>>>(a);
    }
    *cap_out = cap; *nullbits_out = nullbits; *feasible_out = feasible;
    return GX_OK;
}

// Returns GX_OK with *done = 1 and *out set when the rows travelled through the windows; *done = 0 when the ranks
// agreed (through the headers) that this call must take the NCCL path.
static int redistribute_peer(gx_ctx *ctx, const gx_table *in, int key_col, gx_redist_transport &T, gx_table **out, int *done)
{
    *done = 0;
    const int N = T.nranks;
    const long long region_stride = (long long) (T.window_bytes / N) & ~255LL;
    char *dst[GX_MAX_NODES];
    int rc = T.window_open(ctx, region_stride, dst); if (rc) return rc;
    unsigned long long *d_cur;
    GX_CUDA(ctx, gx_tmp_alloc(ctx, (void **) &d_cur, (GX_MAX_NODES + 1) * 8));
    GX_CUDA(ctx, cudaMemsetAsync(d_cur, 0, (GX_MAX_NODES + 1) * 8, ctx->stream));
    long long cap = 0; unsigned long long nullbits = 0; int feasible = 0;
    rc = peer_route(ctx, in, key_col, N, region_stride, dst, d_cur, &cap, &nullbits, &feasible);
    unsigned long long h_hdr[GX_MAX_NODES * 3]; const char *win = nullptr;
    if (rc == GX_OK) rc = T.window_headers(ctx, d_cur, feasible, cap, nullbits, h_hdr, &win);
    gx_tmp_free(ctx, d_cur);
    if (rc) return rc;
    bool fallback = false; long long total = 0; unsigned long long anynull = 0;
    for (int s = 0; s < N; s++) {
        if (h_hdr[s * 3] == PEER_FALLBACK) fallback = true; else total += (long long) h_hdr[s * 3];
        anynull |= h_hdr[s * 3 + 2];
    }
    if (fallback) {
        // nothing of this call will be read from the windows: release them and let the caller take the NCCL path
        T.window_release(ctx);
        return GX_OK;
    }
    bool hn[GX_MAX_COLS];
    for (int c = 0; c < in->ncols; c++) hn[c] = (anynull >> c) & 1ULL;
    gx_table *t;
    rc = gx_table_alloc_like(ctx, in->ncols, in->types, hn, total, &t);
    if (rc == GX_OK && total > 0) {
        gx_peer_gather_args g; memset(&g, 0, sizeof(g));
        g.nnodes = N; g.ncols = in->ncols; g.win = win; g.region_stride = region_stride;
        long long most = 0;
        for (int s = 0; s < N; s++) { g.count[s] = (long long) h_hdr[s * 3]; g.cap[s] = (long long) h_hdr[s * 3 + 1]; g.nullbits[s] = h_hdr[s * 3 + 2]; if (g.count[s] > most) most = g.count[s]; }
        for (int c = 0; c < in->ncols; c++) { g.sizes[c] = gx_type_size(in->types[c]); g.out[c] = t->cols[c]; g.out_nulls[c] = t->nulls[c]; }
        long long bx = (most + 256 * 8 - 1) / (256 * 8); if (bx < 1) bx = 1; if (bx > ctx->sm_count * 2) bx = ctx->sm_count * 2;
        gx_launch_scope ls(ctx, "peer_gather");
        gx_k_peer_gather<<<dim3((unsigned) bx, (unsigned) N, (unsigned) (anynull ? 2 * in->ncols : in->ncols)), 256, 0, ctx->stream>>>(g);
    }
    // the release goes out even when the allocation failed: the peers must not wait for this rank
    T.window_release(ctx);
    if (rc) return rc;
    GX_CUDA(ctx, cudaGetLastError());
    t->nrows = total;
    *out = t; *done = 1;
    return GX_OK;
}

// One rank's rows partitioned by destination for the NCCL path: the one-pass regions of `cap` rows per destination, or
// (GX_PARTITION_TWO_PASS=1, or a region overflowed) the exact two-pass form, densely packed.  counts[N] tells which
// columns have a NULL array, so that every rank agrees on the columns of the result.
struct gx_redist_part {
    gx_table *t;
    int64_t counts[GX_MAX_NODES + 1], sendoff[GX_MAX_NODES];
    int path;                       // 1 one-pass regions, 2 two-pass
};
static int redist_partition(gx_ctx *ctx, const gx_table *in, int key_col, int N, gx_redist_part *s)
{
    const char *two = getenv("GX_PARTITION_TWO_PASS");
    long long cap = 0; int overflowed = 0, rc;
    s->t = nullptr;
    if (!(two && two[0] == '1')) { rc = partition_regions(ctx, in, key_col, &s->t, s->counts, &cap, &overflowed); if (rc) return rc; }
    if (!s->t) { rc = partition_impl(ctx, in, key_col, &s->t, s->counts); if (rc) return rc; cap = 0; }
    int64_t nullbits = 0;
    for (int c = 0; c < in->ncols; c++) if (in->nulls[c]) nullbits |= 1LL << c;
    s->counts[N] = nullbits;
    for (int p = 0; p < N; p++)
        s->sendoff[p] = cap ? (int64_t) p * cap : (p ? s->sendoff[p - 1] + s->counts[p - 1] : 0);   // regions, or densely packed
    s->path = cap ? 1 : 2;
    return GX_OK;
}

// the NULL bytes a partitioned part sends for column c: its own, or zeros when it has no NULL array for c but another
// rank has one (*tmp: the zeros, for the caller to free)
static int send_nulls(gx_ctx *ctx, const gx_table *part, int c, const uint8_t **src, uint8_t **tmp)
{
    *tmp = nullptr; *src = part->nulls[c];
    if (*src) return GX_OK;
    GX_CUDA(ctx, gx_tmp_alloc(ctx, (void **) tmp, (size_t) (part->nrows > 0 ? part->nrows : 1)));
    GX_CUDA(ctx, cudaMemsetAsync(*tmp, 0, (size_t) part->nrows, ctx->stream));
    *src = *tmp;
    return GX_OK;
}

// The redistribute of rank T.rank of T.nranks: *out receives the rows of every rank whose key routes to this rank.
// *path (may be NULL): 0 the rows travelled through the peer windows, 1 the NCCL path with this rank's rows in one-pass
// regions, 2 the NCCL path with them in the two-pass form.
static int redistribute_run(gx_ctx *ctx, const gx_table *in, int key_col, gx_redist_transport &T, gx_table **out, int *path)
{
    const int N = T.nranks;
    GX_CHECK_ARG(ctx, ctx->nnodes == N, "redistribute: shard map covers %d nodes but the communicator has %d ranks", ctx->nnodes, N);
    GX_CHECK_ARG(ctx, key_col >= 0 && key_col < in->ncols, "route: key column %d out of range", key_col);
    const int kt = in->types[key_col];
    GX_CHECK_ARG(ctx, kt == GX_INT4 || kt == GX_INT8 || kt == GX_DATE, "route: distribution column type %d not supported (int4/int8/date)", kt);
    int rc = GX_OK;
    if (N > 1 && T.window_bytes > 0) {
        int done = 0;
        rc = redistribute_peer(ctx, in, key_col, T, out, &done);
        if (rc || done) { if (path && done) *path = 0; return rc; }
    }
    gx_redist_part s;
    rc = redist_partition(ctx, in, key_col, N, &s); if (rc) return rc;
    if (path) *path = s.path;
    if (N == 1) { *out = s.t; return GX_OK; }
    int64_t *all = (int64_t *) malloc((size_t) N * (N + 1) * 8);
    rc = T.gather_counts(ctx, s.counts, N + 1, all);
    if (rc) { free(all); gx_table_free(s.t); return rc; }
    int64_t recvcnt[GX_MAX_NODES], recvoff[GX_MAX_NODES], total = 0, anynull = 0;
    for (int p = 0; p < N; p++) {
        recvcnt[p] = all[(size_t) p * (N + 1) + T.rank];
        recvoff[p] = total; total += recvcnt[p];
        anynull |= all[(size_t) p * (N + 1) + N];
    }
    free(all);
    bool hn[GX_MAX_COLS];
    for (int c = 0; c < in->ncols; c++) hn[c] = (anynull >> c) & 1;
    gx_table *t;
    rc = gx_table_alloc_like(ctx, in->ncols, in->types, hn, total, &t);
    if (rc) { gx_table_free(s.t); return rc; }
    {
        gx_launch_scope ls(ctx, "alltoall", in->ncols);
        for (int c = 0; c < in->ncols && rc == GX_OK; c++) {
            int sz = gx_type_size(in->types[c]);
            int64_t so[GX_MAX_NODES], sc[GX_MAX_NODES], ro[GX_MAX_NODES], rcn[GX_MAX_NODES];
            for (int p = 0; p < N; p++) { so[p] = s.sendoff[p] * sz; sc[p] = s.counts[p] * sz; ro[p] = recvoff[p] * sz; rcn[p] = recvcnt[p] * sz; }
            rc = T.exchange_column(ctx, c, 0, (const char *) s.t->cols[c], so, sc, (char *) t->cols[c], ro, rcn);
            if (rc == GX_OK && hn[c]) {
                const uint8_t *src; uint8_t *tmp;
                rc = send_nulls(ctx, s.t, c, &src, &tmp);
                if (rc == GX_OK) rc = T.exchange_column(ctx, c, 1, (const char *) src, s.sendoff, s.counts, (char *) t->nulls[c], recvoff, recvcnt);
                if (tmp) { cudaStreamSynchronize(ctx->stream); gx_tmp_free(ctx, tmp); }
            }
        }
    }
    cudaError_t e = cudaStreamSynchronize(ctx->stream);
    gx_table_free(s.t);
    if (rc) { gx_table_free(t); return rc; }
    if (e != cudaSuccess) { gx_table_free(t); GX_SET_ERR(ctx, "redistribute: %s", cudaGetErrorString(e)); return GX_ERR_CUDA; }
    t->nrows = total;
    *out = t;
    return GX_OK;
}

// Between processes: the peer windows mapped through CUDA IPC, their headers and acknowledgements, and NCCL.
struct gx_nccl_redist_transport : gx_redist_transport {
    unsigned long long epoch = 0, timeout_ns = 0;
    unsigned long long *d_ctl = nullptr;            // [0] timed-out flag, [1 ..] the headers of the sources
    int window_open(gx_ctx *ctx, long long region_stride, char **dst) override
    {
        epoch = ++ctx->peer_epoch;
        const char *tmo = getenv("GX_PEER_TIMEOUT_MS");
        timeout_ns = (unsigned long long) (tmo ? atoll(tmo) : 60000) * 1000000ULL;
        GX_CUDA(ctx, gx_tmp_alloc(ctx, (void **) &d_ctl, 8 + (size_t) GX_MAX_NODES * 3 * 8));
        GX_CUDA(ctx, cudaMemsetAsync(d_ctl, 0, 8, ctx->stream));
        // the regions this rank owns in the peers' windows must have been emptied (previous call)
        { gx_launch_scope ls(ctx, "peer_wait_ack"); gx_k_peer_wait<<<1, GX_MAX_NODES, 0, ctx->stream>>>(PEER_ACK(ctx->peer_base[rank], 0), 1, nranks, epoch - 1, timeout_ns, (int *) d_ctl, nullptr); }
        for (int p = 0; p < nranks; p++) dst[p] = ctx->peer_base[p] + PEER_CTL_BYTES + (long long) rank * region_stride;
        return GX_OK;
    }
    int window_headers(gx_ctx *ctx, const unsigned long long *d_cur, int feasible, long long cap, unsigned long long nullbits,
                       unsigned long long *hdr, const char **win) override
    {
        gx_peer_ptrs P; memset(&P, 0, sizeof(P));
        for (int p = 0; p < nranks; p++) P.base[p] = ctx->peer_base[p];
        char *own = ctx->peer_base[rank];
        { gx_launch_scope ls(ctx, "peer_publish"); gx_k_peer_publish<<<1, GX_MAX_NODES, 0, ctx->stream>>>(P, nranks, rank, epoch, d_cur, feasible, (unsigned long long) cap, nullbits); }
        { gx_launch_scope ls(ctx, "peer_wait"); gx_k_peer_wait<<<1, GX_MAX_NODES, 0, ctx->stream>>>(PEER_HDR(own, 0), 4, nranks, epoch, timeout_ns, (int *) d_ctl, d_ctl + 1); }
        int h_flag = 0;
        cudaError_t e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaMemcpyAsync(hdr, d_ctl + 1, (size_t) nranks * 3 * 8, cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(&h_flag, d_ctl, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
        gx_tmp_free(ctx, d_ctl); d_ctl = nullptr;
        if (e != cudaSuccess) { GX_SET_ERR(ctx, "redistribute (peer windows): %s", cudaGetErrorString(e)); return GX_ERR_CUDA; }
        if (h_flag) { GX_SET_ERR(ctx, "redistribute (peer windows): rank %d waited %llu ms for its peers", rank, timeout_ns / 1000000ULL); return GX_ERR_NCCL; }
        *win = own + PEER_CTL_BYTES;
        return GX_OK;
    }
    void window_release(gx_ctx *ctx) override
    {
        gx_peer_ptrs P; memset(&P, 0, sizeof(P));
        for (int p = 0; p < nranks; p++) P.base[p] = ctx->peer_base[p];
        gx_launch_scope ls(ctx, "peer_ack"); gx_k_peer_ack<<<1, GX_MAX_NODES, 0, ctx->stream>>>(P, nranks, rank, epoch);
    }
    int gather_counts(gx_ctx *ctx, const int64_t *mine, int n, int64_t *all) override { return allgather_i64(ctx, mine, n, all); }
    int exchange_column(gx_ctx *ctx, int, int, const char *sendbuf, const int64_t *so, const int64_t *sc,
                        char *recvbuf, const int64_t *ro, const int64_t *rcn) override
    {
        return alltoallv_bytes(ctx, sendbuf, so, sc, recvbuf, ro, rcn);
    }
};

// In one process: parts[p] is the input table of rank p.  The body redistributes parts[rank]; the other parts are
// routed or partitioned here by the body's own steps, as their ranks would, and what they address to this rank is
// copied out of their buffers.  The windows of all ranks are allocated here; no header is published or awaited.
struct gx_inproc_redist_transport : gx_redist_transport {
    const gx_table *const *parts; int key_col; gx_ctx *ctx;
    char *win[GX_MAX_NODES]; long long region_stride = 0;
    gx_redist_part sent[GX_MAX_NODES];              // what every other rank sends on the NCCL path
    gx_inproc_redist_transport(gx_ctx *c, const gx_table *const *p, int k) : parts(p), key_col(k), ctx(c)
    {
        memset(win, 0, sizeof(win));
        for (int i = 0; i < GX_MAX_NODES; i++) sent[i].t = nullptr;
    }
    ~gx_inproc_redist_transport()
    {
        window_release(ctx);
        for (int i = 0; i < GX_MAX_NODES; i++) if (sent[i].t) gx_table_free(sent[i].t);
    }
    int window_open(gx_ctx *ctx, long long stride, char **dst) override
    {
        region_stride = stride;
        for (int d = 0; d < nranks; d++) {
            GX_CUDA(ctx, gx_tmp_alloc(ctx, (void **) &win[d], window_bytes));
            dst[d] = win[d] + (long long) rank * region_stride;
        }
        return GX_OK;
    }
    int window_headers(gx_ctx *ctx, const unsigned long long *d_cur, int feasible, long long cap, unsigned long long nullbits,
                       unsigned long long *hdr, const char **own) override
    {
        unsigned long long *d_src = nullptr;
        GX_CUDA(ctx, gx_tmp_alloc(ctx, (void **) &d_src, (GX_MAX_NODES + 1) * 8));
        int rc = GX_OK;
        for (int s = 0; s < nranks && rc == GX_OK; s++) {
            long long c = cap; unsigned long long nb = nullbits; int f = feasible;
            const unsigned long long *cur = d_cur;
            if (s != rank) {
                char *dst[GX_MAX_NODES];
                for (int d = 0; d < nranks; d++) dst[d] = win[d] + (long long) s * region_stride;
                cudaError_t e = cudaMemsetAsync(d_src, 0, (GX_MAX_NODES + 1) * 8, ctx->stream);
                if (e != cudaSuccess) { GX_SET_ERR(ctx, "debug_redistribute: %s", cudaGetErrorString(e)); rc = GX_ERR_CUDA; break; }
                rc = peer_route(ctx, parts[s], key_col, nranks, region_stride, dst, d_src, &c, &nb, &f);
                cur = d_src;
            }
            unsigned long long h[GX_MAX_NODES + 1];
            cudaError_t e = cudaGetLastError();
            if (e == cudaSuccess) e = cudaMemcpyAsync(h, cur, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream);
            if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
            if (rc == GX_OK && e != cudaSuccess) { GX_SET_ERR(ctx, "debug_redistribute: %s", cudaGetErrorString(e)); rc = GX_ERR_CUDA; }
            // what gx_k_peer_publish of rank s writes into the header of this rank's window
            hdr[s * 3] = !f || h[GX_MAX_NODES] != 0 ? PEER_FALLBACK : h[rank]; hdr[s * 3 + 1] = (unsigned long long) c; hdr[s * 3 + 2] = nb;
        }
        gx_tmp_free(ctx, d_src);
        *own = win[rank];
        return rc;
    }
    void window_release(gx_ctx *ctx) override
    {
        for (int d = 0; d < GX_MAX_NODES; d++) { gx_tmp_free(ctx, win[d]); win[d] = nullptr; }
    }
    int gather_counts(gx_ctx *ctx, const int64_t *mine, int n, int64_t *all) override
    {
        for (int p = 0; p < nranks; p++) {
            if (p != rank) { int rc = redist_partition(ctx, parts[p], key_col, nranks, &sent[p]); if (rc) return rc; }
            memcpy(all + (size_t) p * n, p == rank ? mine : sent[p].counts, (size_t) n * 8);
        }
        return GX_OK;
    }
    int exchange_column(gx_ctx *ctx, int c, int want_null, const char *sendbuf, const int64_t *so, const int64_t *,
                        char *recvbuf, const int64_t *ro, const int64_t *rcn) override
    {
        for (int p = 0; p < nranks; p++) {
            if (!rcn[p]) continue;
            const char *src = sendbuf + so[rank];
            uint8_t *tmp = nullptr;
            if (p != rank) {
                const gx_table *part = sent[p].t;
                if (want_null) {
                    const uint8_t *nb;
                    int rc = send_nulls(ctx, part, c, &nb, &tmp); if (rc) return rc;
                    src = (const char *) nb + sent[p].sendoff[rank];
                } else {
                    src = (const char *) part->cols[c] + sent[p].sendoff[rank] * gx_type_size(part->types[c]);
                }
            }
            cudaError_t e = cudaMemcpyAsync(recvbuf + ro[p], src, (size_t) rcn[p], cudaMemcpyDeviceToDevice, ctx->stream);
            gx_tmp_free(ctx, tmp);
            if (e != cudaSuccess) { GX_SET_ERR(ctx, "debug_redistribute: %s", cudaGetErrorString(e)); return GX_ERR_CUDA; }
        }
        return GX_OK;
    }
};

extern "C" int gx_redistribute(gx_ctx *ctx, const gx_table *in, int key_col, gx_table **out)
{
    if (!ctx || !in || !out) return GX_ERR_ARG;
    gx_nccl_redist_transport T;
    T.rank = ctx->rank; T.nranks = ctx->nranks;
    T.window_bytes = ctx->comm && ctx->peer_ready == 1 ? ctx->peer_win_bytes : 0;
    return redistribute_run(ctx, in, key_col, T, out, nullptr);
}

#define GX_DEBUG_WINDOW_LIMIT (4ULL << 30)      // window_bytes * nparts of gx_debug_redistribute

extern "C" int gx_debug_redistribute(gx_ctx *ctx, int nparts, const gx_table *const *parts, int key_col, int rank,
                                     size_t window_bytes, gx_table **out, int *path_out)
{
    if (!ctx || !parts || !out) return GX_ERR_ARG;
    GX_CHECK_ARG(ctx, nparts >= 1 && nparts <= GX_MAX_NODES, "debug_redistribute: %d parts (1..%d)", nparts, GX_MAX_NODES);
    GX_CHECK_ARG(ctx, rank >= 0 && rank < nparts, "debug_redistribute: rank %d of %d parts", rank, nparts);
    for (int p = 0; p < nparts; p++) {
        const gx_table *a = parts[p], *b = parts[0];
        GX_CHECK_ARG(ctx, a != nullptr, "debug_redistribute: part %d is NULL", p);
        GX_CHECK_ARG(ctx, a->ncols == b->ncols && memcmp(a->types, b->types, sizeof(a->types[0]) * a->ncols) == 0,
                     "debug_redistribute: part %d has other columns than part 0", p);
    }
    GX_CHECK_ARG(ctx, window_bytes <= GX_DEBUG_WINDOW_LIMIT / (size_t) nparts, "debug_redistribute: %d windows of %zu bytes exceed %llu bytes",
                 nparts, window_bytes, GX_DEBUG_WINDOW_LIMIT);
    gx_inproc_redist_transport T(ctx, parts, key_col);
    T.rank = rank; T.nranks = nparts; T.window_bytes = window_bytes;
    return redistribute_run(ctx, parts[rank], key_col, T, out, path_out);
}

// ------------------------------------------- Finalize across datanodes
int gx_combine_records(gx_ctx *ctx, gx_result *r, unsigned long long *d_recs, long long nrec,
                       unsigned long long **d_out, long long *ngroups_out);   // gx_agg.cu
int gx_pack_partial(gx_ctx *ctx, gx_result *r, long long cap, unsigned long long *d_seg);
int gx_combine_gathered(gx_ctx *ctx, gx_result *r, const unsigned long long *d_gather, int nseg, long long cap, int rank, int nranks,
                        unsigned long long **d_out, long long *ngroups_out, int *anybig);

__global__ void gx_k_rec_dest_hist(const unsigned long long *recs, long long nrec, int RW, int nranks,
                                   unsigned char *dest, long long *hist)
{
    __shared__ unsigned int sh[GX_MAX_NODES];
    if (threadIdx.x < GX_MAX_NODES) sh[threadIdx.x] = 0;
    __syncthreads();
    long long per = (nrec + gridDim.x - 1) / gridDim.x, b = per * blockIdx.x, e = min(nrec, b + per);
    for (long long i = b + threadIdx.x; i < e; i += blockDim.x) {
        const unsigned long long *rec = recs + i * RW;
        unsigned long long h = gx_mix64(rec[1] ^ (rec[2] * 0x9E3779B97F4A7C15ULL) ^ (rec[0] << 56));
        int d = (int) (h % (unsigned long long) nranks);
        dest[i] = (unsigned char) d;
        atomicAdd(&sh[d], 1u);
    }
    __syncthreads();
    if (threadIdx.x < nranks) hist[(long long) threadIdx.x * gridDim.x + blockIdx.x] = sh[threadIdx.x];
}
__global__ void gx_k_rec_scatter(const unsigned long long *recs, long long nrec, int RW, const unsigned char *dest,
                                 const long long *offs, unsigned long long *out)
{
    __shared__ unsigned int cur[GX_MAX_NODES];
    if (threadIdx.x < GX_MAX_NODES) cur[threadIdx.x] = 0;
    __syncthreads();
    long long per = (nrec + gridDim.x - 1) / gridDim.x, b = per * blockIdx.x, e = min(nrec, b + per);
    for (long long i = b + threadIdx.x; i < e; i += blockDim.x) {
        int d = dest[i];
        unsigned int k = atomicAdd(&cur[d], 1u);
        unsigned long long *dst = out + (offs[(long long) d * gridDim.x + blockIdx.x] + k) * RW;
        const unsigned long long *src = recs + i * RW;
        for (int j = 0; j < RW; j++) dst[j] = src[j];
    }
}

// Records -> a send buffer grouped by destination rank (the owner of each record's key, by the hash
// gx_k_merge_gathered uses), with the offset and the number of records of every destination.
static int partition_records(gx_ctx *ctx, const unsigned long long *recs, long long nrec, int RW, int N,
                             unsigned long long **d_send_out, int64_t *sendoff, int64_t *counts)
{
    unsigned nblk = (unsigned) ctx->sm_count;
    if ((long long) nblk * 256 > nrec) nblk = (unsigned) ((nrec + 255) / 256);
    if (nblk == 0) nblk = 1;
    unsigned char *d_dest; long long *d_hist; unsigned long long *d_send;
    GX_CUDA(ctx, gx_tmp_alloc(ctx, (void **) &d_dest, (size_t) (nrec > 0 ? nrec : 1)));
    GX_CUDA(ctx, gx_tmp_alloc(ctx, (void **) &d_hist, (size_t) N * nblk * 8));
    GX_CUDA(ctx, gx_tmp_alloc(ctx, (void **) &d_send, (size_t) (nrec > 0 ? nrec : 1) * RW * 8));
    long long h_offs[GX_MAX_NODES];
    {
        gx_launch_scope ls(ctx, "combine_partition", 3);
        gx_k_rec_dest_hist<<<nblk, 256, 0, ctx->stream>>>(recs, nrec, RW, N, d_dest, d_hist);
        gx_k_scan_i64<<<1, 1024, 0, ctx->stream>>>(d_hist, (long long) N * nblk, nullptr);
        cudaMemcpy2DAsync(h_offs, 8, d_hist, (size_t) nblk * 8, 8, N, cudaMemcpyDeviceToHost, ctx->stream);
        gx_k_rec_scatter<<<nblk, 256, 0, ctx->stream>>>(recs, nrec, RW, d_dest, d_hist, d_send);
    }
    cudaError_t e = cudaStreamSynchronize(ctx->stream);
    gx_tmp_free(ctx, d_dest); gx_tmp_free(ctx, d_hist);
    if (e != cudaSuccess) { gx_tmp_free(ctx, d_send); GX_SET_ERR(ctx, "combine: %s", cudaGetErrorString(e)); return GX_ERR_CUDA; }
    for (int p = 0; p < N; p++) { sendoff[p] = h_offs[p]; counts[p] = ((p + 1 < N) ? h_offs[p + 1] : nrec) - h_offs[p]; }
    *d_send_out = d_send;
    return GX_OK;
}

// What the Finalize exchanges between ranks.  combine_run makes every decision and runs every device step; a
// transport only moves bytes: over NCCL between processes, or in one process on one GPU, where it builds from
// the partial results of all ranks what NCCL would have delivered to one of them (gx_debug_combine).
struct gx_combine_transport {
    int rank, nranks;
    // every rank's segment of seg_bytes, in rank order, into d_all; d_seg is this rank's, packed with capacity cap
    virtual int gather_segments(gx_ctx *ctx, const unsigned long long *d_seg, unsigned long long *d_all, long long cap, size_t seg_bytes) = 0;
    // all[p * nranks + q] = the number of records rank p sends to rank q; mine = this rank's row
    virtual int gather_counts(gx_ctx *ctx, const int64_t *mine, int64_t *all) = 0;
    // the records every rank addressed to this one, rank p's at record recvoff[p] of d_recv; d_send, sendoff and
    // counts are this rank's partitioned records
    virtual int exchange_records(gx_ctx *ctx, const unsigned long long *d_send, const int64_t *sendoff, const int64_t *counts, int RW,
                                 unsigned long long *d_recv, const int64_t *recvoff, const int64_t *recvcnt) = 0;
};

struct gx_nccl_transport : gx_combine_transport {
    int gather_segments(gx_ctx *ctx, const unsigned long long *d_seg, unsigned long long *d_all, long long, size_t seg_bytes) override
    {
        gx_launch_scope ls(ctx, "allgather");
        int nr = g_nccl.AllGather(d_seg, d_all, seg_bytes, GX_NCCL_INT8, ctx->comm, ctx->stream);
        if (nr != 0) { GX_SET_ERR(ctx, "NCCL error %d in ncclAllGather: %s", nr, g_nccl.GetErrorString(nr)); return GX_ERR_NCCL; }
        return GX_OK;
    }
    int gather_counts(gx_ctx *ctx, const int64_t *mine, int64_t *all) override { return allgather_i64(ctx, mine, nranks, all); }
    int exchange_records(gx_ctx *ctx, const unsigned long long *d_send, const int64_t *sendoff, const int64_t *counts, int RW,
                         unsigned long long *d_recv, const int64_t *recvoff, const int64_t *recvcnt) override
    {
        int64_t so[GX_MAX_NODES], sc[GX_MAX_NODES], ro[GX_MAX_NODES], rcn[GX_MAX_NODES];
        for (int p = 0; p < nranks; p++) { so[p] = sendoff[p] * RW * 8; sc[p] = counts[p] * RW * 8; ro[p] = recvoff[p] * RW * 8; rcn[p] = recvcnt[p] * RW * 8; }
        gx_launch_scope ls(ctx, "alltoall");
        return alltoallv_bytes(ctx, (const char *) d_send, so, sc, (char *) d_recv, ro, rcn);
    }
};

// parts[p] is the partial result of rank p; only parts[rank] is combined, the others are read
struct gx_inproc_transport : gx_combine_transport {
    gx_result *const *parts;
    unsigned long long *send[GX_MAX_NODES];
    int64_t sendoff[GX_MAX_NODES][GX_MAX_NODES];
    gx_ctx *ctx;
    gx_inproc_transport(gx_ctx *c, gx_result *const *p) : parts(p), ctx(c) { memset(send, 0, sizeof(send)); }
    ~gx_inproc_transport() { for (int p = 0; p < GX_MAX_NODES; p++) gx_tmp_free(ctx, send[p]); }
    int gather_segments(gx_ctx *ctx, const unsigned long long *, unsigned long long *d_all, long long cap, size_t seg_bytes) override
    {
        for (int p = 0; p < nranks; p++) { int rc = gx_pack_partial(ctx, parts[p], cap, d_all + (size_t) p * (seg_bytes / 8)); if (rc) return rc; }
        return GX_OK;
    }
    int gather_counts(gx_ctx *ctx, const int64_t *mine, int64_t *all) override
    {
        for (int p = 0; p < nranks; p++) {
            if (p == rank) { memcpy(all + (size_t) p * nranks, mine, (size_t) nranks * 8); continue; }
            int rc = partition_records(ctx, (const unsigned long long *) parts[p]->d_recs, parts[p]->ngroups, parts[p]->L.rec_words, nranks,
                                       &send[p], sendoff[p], all + (size_t) p * nranks);
            if (rc) return rc;
        }
        return GX_OK;
    }
    int exchange_records(gx_ctx *ctx, const unsigned long long *d_send, const int64_t *own_off, const int64_t *, int RW,
                         unsigned long long *d_recv, const int64_t *recvoff, const int64_t *recvcnt) override
    {
        gx_launch_scope ls(ctx, "alltoall");
        for (int p = 0; p < nranks; p++) {
            if (!recvcnt[p]) continue;
            const unsigned long long *src = p == rank ? d_send + own_off[rank] * RW : send[p] + sendoff[p][rank] * RW;
            GX_CUDA(ctx, cudaMemcpyAsync(d_recv + recvoff[p] * RW, src, (size_t) recvcnt[p] * RW * 8, cudaMemcpyDeviceToDevice, ctx->stream));
        }
        return GX_OK;
    }
};

// The Finalize of rank T.rank of T.nranks over r, its partial result.  The groups of the ranks' results
// partition the combined groups: each group is returned by the one rank that owns its key.  A plain aggregate's
// one row is returned by rank 0, which owns the empty key (it hashes to 0); every other rank returns no row.
static int combine_run(gx_ctx *ctx, gx_result *r, gx_combine_transport &T)
{
    const int N = T.nranks;
    GX_CHECK_ARG(ctx, N == 1 || !gx_result_has_distinct(r), "combine: count(DISTINCT) counts do not add across %d ranks", N);
    GX_CHECK_ARG(ctx, N == 1 || !gx_result_has_variance(r), "combine: variance states are not combined across %d ranks", N);
    GX_CHECK_ARG(ctx, N == 1 || !gx_result_has_regr(r), "combine: regression states are not combined across %d ranks", N);
    if (N == 1 || r->finalized_across) return GX_OK;
    const int RW = r->L.rec_words;
    long long nrec = r->ngroups;
    auto finish = [&](unsigned long long *d_groups, long long ngroups, long long cap) {
        gx_tmp_free(ctx, r->d_recs);
        r->d_recs = (long long *) d_groups; r->ngroups = ngroups; r->cap = cap; r->finalized_across = 1;
        r->plain_row_elsewhere = r->plan.n_group_cols == 0 && T.rank != 0;
    };
    // ---- few groups (Q1, GROUP BY date): one ncclAllGather of fixed-capacity segments and a
    // device-side merge; no partition, no count exchange, one host synchronisation (the group
    // count).  The capacity comes from the planner's estimate, which every datanode shares
    // (same plan), so all ranks issue the same collective; a rank whose partial result does
    // not fit says so in its segment header and everybody falls through to the general path.
    {
        const char *off = getenv("GX_NO_GATHER_COMBINE");
        long long est = r->plan.n_group_cols == 0 ? 1 : (r->plan.est_groups > 0 ? r->plan.est_groups : 1024);
        long long cap = gx_pow2_ceil(est * 2 < 1024 ? 1024 : est * 2);
        if (cap <= 65536 && !(off && off[0] == '1')) {
            const size_t seg_bytes = (size_t) (2 + cap * RW) * 8;
            unsigned long long *d_seg, *d_all;
            GX_CUDA(ctx, gx_tmp_alloc(ctx, (void **) &d_seg, seg_bytes));
            GX_CUDA(ctx, gx_tmp_alloc(ctx, (void **) &d_all, seg_bytes * N));
            int rc = gx_pack_partial(ctx, r, cap, d_seg);
            if (rc == GX_OK) rc = T.gather_segments(ctx, d_seg, d_all, cap, seg_bytes);
            unsigned long long *d_groups = nullptr; long long ngroups = 0; int anybig = 0;
            if (rc == GX_OK) rc = gx_combine_gathered(ctx, r, d_all, N, cap, T.rank, N, &d_groups, &ngroups, &anybig);
            gx_tmp_free(ctx, d_seg); gx_tmp_free(ctx, d_all);
            if (rc) return rc;
            if (!anybig) { finish(d_groups, ngroups, ngroups > 0 ? ngroups : 1); return GX_OK; }
        }
    }
    unsigned long long *d_send;
    int64_t counts[GX_MAX_NODES], sendoff[GX_MAX_NODES], recvcnt[GX_MAX_NODES], recvoff[GX_MAX_NODES], total = 0;
    int rc = partition_records(ctx, (const unsigned long long *) r->d_recs, nrec, RW, N, &d_send, sendoff, counts);
    if (rc) return rc;
    int64_t *all = (int64_t *) malloc((size_t) N * N * 8);
    rc = T.gather_counts(ctx, counts, all);
    if (rc == GX_OK) {
        for (int p = 0; p < N; p++) { recvcnt[p] = all[(size_t) p * N + T.rank]; recvoff[p] = total; total += recvcnt[p]; }
    }
    free(all);
    unsigned long long *d_recv = nullptr;
    if (rc == GX_OK) {
        cudaError_t e = gx_tmp_alloc(ctx, (void **) &d_recv, (size_t) (total > 0 ? total : 1) * RW * 8);
        if (e != cudaSuccess) { d_recv = nullptr; GX_SET_ERR(ctx, "combine: %s", cudaGetErrorString(e)); rc = GX_ERR_NOMEM; }
    }
    if (rc == GX_OK) rc = T.exchange_records(ctx, d_send, sendoff, counts, RW, d_recv, recvoff, recvcnt);
    if (rc == GX_OK) { cudaError_t e = cudaStreamSynchronize(ctx->stream); if (e != cudaSuccess) { GX_SET_ERR(ctx, "combine: %s", cudaGetErrorString(e)); rc = GX_ERR_CUDA; } }
    gx_tmp_free(ctx, d_send);
    if (rc) { if (d_recv) gx_tmp_free(ctx, d_recv); return rc; }
    unsigned long long *d_groups; long long ngroups;
    rc = gx_combine_records(ctx, r, d_recv, total, &d_groups, &ngroups);
    gx_tmp_free(ctx, d_recv);
    if (rc) return rc;
    if (!d_groups) { GX_CUDA(ctx, gx_tmp_alloc(ctx, (void **) &d_groups, 64)); }
    finish(d_groups, ngroups, ngroups);
    return GX_OK;
}

extern "C" int gx_result_combine(gx_ctx *ctx, gx_result *r)
{
    if (!ctx || !r) return GX_ERR_ARG;
    gx_nccl_transport T;
    T.rank = ctx->rank; T.nranks = ctx->comm ? ctx->nranks : 1;
    return combine_run(ctx, r, T);
}

extern "C" int gx_debug_combine(gx_ctx *ctx, int nparts, gx_result *const *parts, int rank)
{
    if (!ctx || !parts) return GX_ERR_ARG;
    GX_CHECK_ARG(ctx, nparts >= 1 && nparts <= GX_MAX_NODES, "debug_combine: %d parts (1..%d)", nparts, GX_MAX_NODES);
    GX_CHECK_ARG(ctx, rank >= 0 && rank < nparts, "debug_combine: rank %d of %d parts", rank, nparts);
    for (int p = 0; p < nparts; p++) {
        const gx_result *a = parts[p], *b = parts[0];
        GX_CHECK_ARG(ctx, a != nullptr, "debug_combine: part %d is NULL", p);
        GX_CHECK_ARG(ctx, !a->finalized_across, "debug_combine: part %d was combined already", p);
        GX_CHECK_ARG(ctx, memcmp(&a->plan, &b->plan, sizeof(a->plan)) == 0, "debug_combine: part %d has another plan than part 0", p);
        GX_CHECK_ARG(ctx, a->L.rec_words == b->L.rec_words && memcmp(a->L.agg_word, b->L.agg_word, sizeof(a->L.agg_word)) == 0 &&
                     memcmp(a->L.agg_cnt_word, b->L.agg_cnt_word, sizeof(a->L.agg_cnt_word)) == 0,
                     "debug_combine: part %d has another record layout than part 0", p);
    }
    gx_inproc_transport T(ctx, parts);
    T.rank = rank; T.nranks = nparts;
    return combine_run(ctx, parts[rank], T);
}

// ------------------------------------------------- debug hash entry point
__global__ void gx_k_debug_hash(int which, const long long *in, long long n, unsigned int *out)
{
    long long i = (long long) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    long long v = in[i];
    unsigned int h;
    switch (which) {
        case 1: h = gx_hashint4((int) v); break;
        case 2: h = gx_hashint8(v); break;
        case 3: h = gx_crc32c_u64((unsigned long long) (long long) (int) v); break;   // hashint4new: widen to int64
        case 4: h = gx_crc32c_u64((unsigned long long) v); break;                     // hashint8new
        default: h = gx_murmurhash32((unsigned int) v); break;
    }
    out[i] = h;
}
extern "C" int gx_debug_hash(gx_ctx *ctx, int which, const int64_t *host_in, int64_t n, uint32_t *host_out)
{
    if (!ctx || !host_in || !host_out || n < 0) return GX_ERR_ARG;
    if (n == 0) return GX_OK;
    long long *d_in; unsigned int *d_out;
    GX_CUDA(ctx, gx_tmp_alloc(ctx, (void **) &d_in, (size_t) n * 8));
    GX_CUDA(ctx, gx_tmp_alloc(ctx, (void **) &d_out, (size_t) n * 4));
    GX_CUDA(ctx, cudaMemcpyAsync(d_in, host_in, (size_t) n * 8, cudaMemcpyHostToDevice, ctx->stream));
    { gx_launch_scope ls(ctx, "debug_hash"); gx_k_debug_hash<<<(unsigned) ((n + 255) / 256), 256, 0, ctx->stream>>>(which, d_in, n, d_out); }
    GX_CUDA(ctx, cudaMemcpyAsync(host_out, d_out, (size_t) n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    GX_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    gx_tmp_free(ctx, d_in); gx_tmp_free(ctx, d_out);
    return GX_OK;
}
