// gx_table.cu — K0 columnar loader (host columns, raw heap pages, synthetic
// generator) and K1 scan/qual/projection.
#include "gx_internal.cuh"
#include "../../include/gx_tpch_gen.h"

// --------------------------------------------------------------- lifecycle
uint64_t gx_table_next_version()
{
    static unsigned long long next = 0;
    return (uint64_t) __atomic_add_fetch(&next, 1ULL, __ATOMIC_RELAXED);
}

int gx_table_alloc_like(gx_ctx *ctx, int ncols, const int32_t *types, const bool *has_nulls,
                        int64_t capacity, gx_table **out)
{
    GX_CHECK_ARG(ctx, ncols > 0 && ncols <= GX_MAX_COLS, "table: ncols %d out of range", ncols);
    gx_table *t = (gx_table *) calloc(1, sizeof(gx_table));
    t->ctx = ctx; t->ncols = ncols; t->capacity = capacity < 1 ? 1 : capacity; t->version = gx_table_next_version();
    for (int c = 0; c < ncols; c++) {
        int sz = gx_type_size(types[c]);
        if (!sz) { free(t); GX_SET_ERR(ctx, "table: column %d has unknown type %d", c, types[c]); return GX_ERR_ARG; }
        t->types[c] = types[c];
        cudaError_t e = gx_tmp_alloc(ctx, &t->cols[c], (size_t) t->capacity * sz + 32);
        if (e == cudaSuccess && has_nulls && has_nulls[c]) {
            e = gx_tmp_alloc(ctx, (void **) &t->nulls[c], (size_t) t->capacity + 32);
            if (e == cudaSuccess) e = cudaMemsetAsync(t->nulls[c], 0, (size_t) t->capacity, ctx->stream);
        }
        if (e != cudaSuccess) {
            GX_SET_ERR(ctx, "table: cudaMalloc of %lld rows failed: %s", (long long) t->capacity, cudaGetErrorString(e));
            gx_table_free(t);
            return GX_ERR_NOMEM;
        }
    }
    *out = t;
    return GX_OK;
}

extern "C" int gx_table_create(gx_ctx *ctx, int ncols, const int32_t *types, int64_t capacity_rows, gx_table **out)
{
    if (!ctx || !types || !out) return GX_ERR_ARG;
    return gx_table_alloc_like(ctx, ncols, types, nullptr, capacity_rows, out);
}

extern "C" void gx_table_free(gx_table *t)
{
    if (!t) return;
    gx_table_settle(t, true);
    for (int c = 0; c < t->ncols; c++) { if (t->cols[c]) gx_tmp_free(t->ctx, t->cols[c]); if (t->nulls[c]) gx_tmp_free(t->ctx, t->nulls[c]); }
    free(t);
}
extern "C" int64_t gx_table_nrows(const gx_table *t) { return t ? t->nrows : -1; }
extern "C" int gx_table_ncols(const gx_table *t) { return t ? t->ncols : -1; }
extern "C" int gx_table_truncate(gx_table *t)
{
    if (!t) return GX_ERR_ARG;
    int rc = gx_table_settle(t); if (rc) return rc;
    t->nrows = 0; t->version = gx_table_next_version(); return GX_OK;
}
// End of a load: wait for the enqueued appends and report a NULL that arrived in a column staged as NOT NULL
extern "C" int gx_table_load_finish(gx_table *t)
{
    if (!t) return GX_ERR_ARG;
    gx_ctx *ctx = t->ctx;
    GX_CUDA(ctx, cudaMemcpyAsync(ctx->h_scratch + 20, ctx->d_scratch + 20, sizeof(long long), cudaMemcpyDeviceToHost, ctx->stream));
    GX_CUDA(ctx, cudaMemsetAsync(ctx->d_scratch + 20, 0, sizeof(long long), ctx->stream));
    GX_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (ctx->h_scratch[20] != 0) { GX_SET_ERR(ctx, "heap pages: a NULL value arrived in a column declared NOT NULL (att_notnull)"); return GX_ERR_STATE; }
    return GX_OK;
}
extern "C" int gx_table_drop_column(gx_table *t, int col)
{
    if (!t || col < 0 || col >= t->ncols || t->ncols < 2) return GX_ERR_ARG;
    int rc = gx_table_settle(t); if (rc) return rc;
    gx_tmp_free(t->ctx, t->cols[col]); gx_tmp_free(t->ctx, t->nulls[col]);
    for (int c = col; c + 1 < t->ncols; c++) { t->cols[c] = t->cols[c + 1]; t->nulls[c] = t->nulls[c + 1]; t->types[c] = t->types[c + 1]; }
    t->ncols--;
    t->version = gx_table_next_version();
    t->cols[t->ncols] = nullptr; t->nulls[t->ncols] = nullptr; t->types[t->ncols] = 0;
    return GX_OK;
}
extern "C" int gx_table_column_devptr(gx_table *t, int col, void **dptr)
{
    if (!t || col < 0 || col >= t->ncols || !dptr) return GX_ERR_ARG;
    int rc = gx_table_settle(t); if (rc) return rc;      // the caller may write the column
    *dptr = t->cols[col];
    return GX_OK;
}

// grow the column arrays (stream-ordered): the loader does not know a heap relation's row count up front
extern "C" int gx_table_reserve(gx_table *t, int64_t capacity_rows)
{
    if (!t || capacity_rows < 0) return GX_ERR_ARG;
    if (capacity_rows <= t->capacity) return GX_OK;
    int rc = gx_table_settle(t); if (rc) return rc;
    gx_ctx *ctx = t->ctx;
    for (int c = 0; c < t->ncols; c++) {
        const int sz = gx_type_size(t->types[c]);
        void *nc = nullptr; uint8_t *nn = nullptr;
        cudaError_t e = gx_tmp_alloc(ctx, &nc, (size_t) capacity_rows * sz + 32);
        if (e == cudaSuccess && t->nulls[c]) e = gx_tmp_alloc(ctx, (void **) &nn, (size_t) capacity_rows + 32);
        if (e != cudaSuccess) { gx_tmp_free(ctx, nc); GX_SET_ERR(ctx, "table_reserve: %lld rows: %s", (long long) capacity_rows, cudaGetErrorString(e)); cudaGetLastError(); return GX_ERR_NOMEM; }
        if (t->nrows) GX_CUDA(ctx, cudaMemcpyAsync(nc, t->cols[c], (size_t) t->nrows * sz, cudaMemcpyDeviceToDevice, ctx->stream));
        gx_tmp_free(ctx, t->cols[c]); t->cols[c] = nc;
        if (nn) {
            GX_CUDA(ctx, cudaMemsetAsync(nn, 0, (size_t) capacity_rows, ctx->stream));
            if (t->nrows) GX_CUDA(ctx, cudaMemcpyAsync(nn, t->nulls[c], (size_t) t->nrows, cudaMemcpyDeviceToDevice, ctx->stream));
            gx_tmp_free(ctx, t->nulls[c]); t->nulls[c] = nn;
        }
    }
    t->capacity = capacity_rows;
    return GX_OK;
}

static int ensure_null_array(gx_table *t, int c)
{
    if (t->nulls[c]) return GX_OK;
    GX_CUDA(t->ctx, gx_tmp_alloc(t->ctx, (void **) &t->nulls[c], (size_t) t->capacity + 32));
    GX_CUDA(t->ctx, cudaMemsetAsync(t->nulls[c], 0, (size_t) t->capacity, t->ctx->stream));
    return GX_OK;
}

extern "C" int gx_table_append_columns(gx_table *t, const void *const *host_cols,
                                       const uint8_t *const *host_nulls, int64_t nrows)
{
    if (!t || !host_cols || nrows < 0) return GX_ERR_ARG;
    int rc = gx_table_settle(t); if (rc) return rc;
    gx_ctx *ctx = t->ctx;
    GX_CHECK_ARG(ctx, t->nrows + nrows <= t->capacity, "append_columns: %lld + %lld rows exceed capacity %lld",
                 (long long) t->nrows, (long long) nrows, (long long) t->capacity);
    if (nrows == 0) return GX_OK;
    for (int c = 0; c < t->ncols; c++) {
        int sz = gx_type_size(t->types[c]);
        GX_CHECK_ARG(ctx, host_cols[c] != nullptr, "append_columns: column %d is NULL", c);
        GX_CUDA(ctx, cudaMemcpyAsync((char *) t->cols[c] + (size_t) t->nrows * sz, host_cols[c], (size_t) nrows * sz,
                                     cudaMemcpyHostToDevice, ctx->stream));
        if (host_nulls && host_nulls[c]) {
            int rc = ensure_null_array(t, c); if (rc) return rc;
            GX_CUDA(ctx, cudaMemcpyAsync(t->nulls[c] + t->nrows, host_nulls[c], (size_t) nrows,
                                         cudaMemcpyHostToDevice, ctx->stream));
        }
    }
    t->nrows += nrows;
    t->version = gx_table_next_version();
    return GX_OK;
}

extern "C" int gx_table_read_column(gx_table *t, int col, int64_t row0, int64_t nrows, void *host_out, uint8_t *host_nulls_out)
{
    if (!t || col < 0 || col >= t->ncols || row0 < 0 || nrows < 0 || row0 + nrows > t->nrows) return GX_ERR_ARG;
    gx_ctx *ctx = t->ctx;
    int sz = gx_type_size(t->types[col]);
    if (host_out && nrows)
        GX_CUDA(ctx, cudaMemcpyAsync(host_out, (char *) t->cols[col] + (size_t) row0 * sz, (size_t) nrows * sz, cudaMemcpyDeviceToHost, ctx->stream));
    if (host_nulls_out && nrows) {
        if (t->nulls[col]) GX_CUDA(ctx, cudaMemcpyAsync(host_nulls_out, t->nulls[col] + row0, (size_t) nrows, cudaMemcpyDeviceToHost, ctx->stream));
        else memset(host_nulls_out, 0, (size_t) nrows);
    }
    GX_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GX_OK;
}

// ------------------------------------------------------------ permute (bench / test plumbing)
// out[i] = in[(i * A + B) mod n] with A coprime to n near n / golden ratio: a bijection that sends
// neighbouring rows far apart — what an UNCLUSTERED copy of a table looks like to the join kernels.
struct gx_permute_args { long long n, A, B; int ncols; gx_dcol in[GX_MAX_COLS]; void *out[GX_MAX_COLS]; uint8_t *out_nulls[GX_MAX_COLS]; };
__global__ void gx_k_permute(gx_permute_args a)
{
    const long long stride = (long long) gridDim.x * blockDim.x;
    for (long long i = (long long) blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += stride) {
        const long long r = (long long) (((unsigned __int128) (unsigned long long) i * (unsigned long long) a.A + (unsigned long long) a.B) % (unsigned long long) a.n);
        for (int c = 0; c < a.ncols; c++) {
            switch (a.in[c].type) {
                case GX_INT4: case GX_DATE: ((int *) a.out[c])[i] = ((const int *) a.in[c].data)[r]; break;
                case GX_CHAR: ((signed char *) a.out[c])[i] = ((const signed char *) a.in[c].data)[r]; break;
                default: ((long long *) a.out[c])[i] = ((const long long *) a.in[c].data)[r]; break;
            }
            if (a.out_nulls[c]) a.out_nulls[c][i] = a.in[c].nulls ? a.in[c].nulls[r] : 0;
        }
    }
}
static long long gcd_ll(long long a, long long b) { while (b) { long long t = a % b; a = b; b = t; } return a; }
extern "C" int gx_table_permute(gx_ctx *ctx, const gx_table *in, int64_t seed, gx_table **out)
{
    if (!ctx || !in || !out) return GX_ERR_ARG;
    bool hn[GX_MAX_COLS];
    for (int c = 0; c < in->ncols; c++) hn[c] = in->nulls[c] != nullptr;
    gx_table *t;
    int rc = gx_table_alloc_like(ctx, in->ncols, in->types, hn, in->nrows > 0 ? in->nrows : 1, &t); if (rc) return rc;
    if (in->nrows > 1) {
        gx_permute_args a; memset(&a, 0, sizeof(a));
        a.n = in->nrows; a.ncols = in->ncols;
        a.A = (long long) ((double) in->nrows * 0.6180339887498949) | 1;
        while (gcd_ll(a.A, a.n) != 1) a.A += 2;
        a.B = (long long) ((unsigned long long) seed * 0x9E3779B97F4A7C15ULL % (unsigned long long) a.n);
        for (int c = 0; c < in->ncols; c++) { a.in[c].data = in->cols[c]; a.in[c].nulls = in->nulls[c]; a.in[c].type = in->types[c]; a.out[c] = t->cols[c]; a.out_nulls[c] = t->nulls[c]; }
        gx_launch_scope ls(ctx, "permute");
        gx_k_permute<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(a);
        GX_CUDA(ctx, cudaGetLastError());
    } else if (in->nrows == 1) {
        for (int c = 0; c < in->ncols; c++) {
            GX_CUDA(ctx, cudaMemcpyAsync(t->cols[c], in->cols[c], (size_t) gx_type_size(in->types[c]), cudaMemcpyDeviceToDevice, ctx->stream));
            if (t->nulls[c]) GX_CUDA(ctx, cudaMemcpyAsync(t->nulls[c], in->nulls[c], 1, cudaMemcpyDeviceToDevice, ctx->stream));
        }
    }
    t->nrows = in->nrows;
    *out = t;
    return GX_OK;
}

// ------------------------------------------------------------ block scan
// exclusive scan of n int64 values in place; total written to *total
__global__ void gx_k_scan_inplace(long long *v, long long n, long long *total)
{
    __shared__ long long sm[33];
    long long carry = 0;
    for (long long base = 0; base < n; base += blockDim.x) {
        long long i = base + threadIdx.x;
        long long x = i < n ? v[i] : 0, tot;
        long long ex = gx_block_exscan(x, &tot, sm);
        if (i < n) v[i] = carry + ex;
        carry += tot;
    }
    if (threadIdx.x == 0) *total = carry;
}

// ------------------------------------------------------------- generator
struct gx_gen_args {
    int table_id, sf, node, nnodes;
    long long o0, o1, base_row;
    const int32_t *shardmap;
    void *cols[GXG_L_NCOLS];
};

__device__ __forceinline__ int gen_rows_of(const gx_gen_args &a, long long i)
{
    if (a.table_id == GXG_T_CUSTOMER) {
        if (a.nnodes > 1) {
            int node = a.shardmap[gx_shard_index(gx_route_hash(GX_INT4, gxg_c_custkey(i), false))];
            if (node != a.node) return 0;
        }
        return 1;
    }
    if (a.nnodes > 1) {
        int node = a.shardmap[gx_shard_index(gx_route_hash(GX_INT8, gxg_o_orderkey(i), false))];
        if (node != a.node) return 0;
    }
    return a.table_id == GXG_T_LINEITEM ? gxg_l_nlines(i) : 1;
}

__global__ void gx_k_gen_count(gx_gen_args a, long long *blocksums)
{
    __shared__ long long sm[33];
    long long i = a.o0 + (long long) blockIdx.x * blockDim.x + threadIdx.x;
    long long n = (i < a.o1) ? gen_rows_of(a, i) : 0, tot;
    gx_block_exscan(n, &tot, sm);
    if (threadIdx.x == 0) blocksums[blockIdx.x] = tot;
}

__global__ void gx_k_gen_write(gx_gen_args a, const long long *blockoffs)
{
    __shared__ long long sm[33];
    long long i = a.o0 + (long long) blockIdx.x * blockDim.x + threadIdx.x;
    int n = (i < a.o1) ? gen_rows_of(a, i) : 0;
    long long tot;
    long long row = a.base_row + blockoffs[blockIdx.x] + gx_block_exscan(n, &tot, sm);
    if (n == 0) return;
    if (a.table_id == GXG_T_ORDERS) {
        if (a.cols[GXG_O_ORDERKEY])     ((long long *) a.cols[GXG_O_ORDERKEY])[row] = gxg_o_orderkey(i);
        if (a.cols[GXG_O_CUSTKEY])      ((int *) a.cols[GXG_O_CUSTKEY])[row] = gxg_o_custkey(i, a.sf);
        if (a.cols[GXG_O_ORDERDATE])    ((int *) a.cols[GXG_O_ORDERDATE])[row] = gxg_o_orderdate(i);
        if (a.cols[GXG_O_SHIPPRIORITY]) ((int *) a.cols[GXG_O_SHIPPRIORITY])[row] = gxg_o_shippriority(i);
    } else if (a.table_id == GXG_T_CUSTOMER) {
        if (a.cols[GXG_C_CUSTKEY])    ((int *) a.cols[GXG_C_CUSTKEY])[row] = gxg_c_custkey(i);
        if (a.cols[GXG_C_MKTSEGMENT]) ((signed char *) a.cols[GXG_C_MKTSEGMENT])[row] = gxg_c_mktsegment(i);
    } else {
        long long key = gxg_o_orderkey(i);
        for (int j = 0; j < n; j++, row++) {
            if (a.cols[GXG_L_ORDERKEY])      ((long long *) a.cols[GXG_L_ORDERKEY])[row] = key;
            if (a.cols[GXG_L_QUANTITY])      ((double *) a.cols[GXG_L_QUANTITY])[row] = gxg_l_quantity(i, j);
            if (a.cols[GXG_L_EXTENDEDPRICE]) ((double *) a.cols[GXG_L_EXTENDEDPRICE])[row] = gxg_l_extendedprice(i, j, a.sf);
            if (a.cols[GXG_L_DISCOUNT])      ((double *) a.cols[GXG_L_DISCOUNT])[row] = gxg_l_discount(i, j);
            if (a.cols[GXG_L_TAX])           ((double *) a.cols[GXG_L_TAX])[row] = gxg_l_tax(i, j);
            if (a.cols[GXG_L_SHIPDATE])      ((int *) a.cols[GXG_L_SHIPDATE])[row] = gxg_l_shipdate(i, j);
            if (a.cols[GXG_L_RETURNFLAG])    ((signed char *) a.cols[GXG_L_RETURNFLAG])[row] = gxg_l_returnflag(i, j);
            if (a.cols[GXG_L_LINESTATUS])    ((signed char *) a.cols[GXG_L_LINESTATUS])[row] = gxg_l_linestatus(i, j);
        }
    }
}

static const int32_t k_schema_orders[GXG_O_NCOLS] = { GX_INT8, GX_INT4, GX_DATE, GX_INT4 };
static const int32_t k_schema_lineitem[GXG_L_NCOLS] = { GX_INT8, GX_FLOAT8, GX_FLOAT8, GX_FLOAT8, GX_FLOAT8, GX_DATE, GX_CHAR, GX_CHAR };
static const int32_t k_schema_customer[GXG_C_NCOLS] = { GX_INT4, GX_CHAR };

// The table's columns must be a prefix-compatible subset of the fixed schema:
// the table is created with the full schema's column count; columns whose
// type is passed as the schema type are materialised.  To skip a column the
// caller creates the table with capacity and then frees nothing — skipping is
// expressed through gx_table_generate_cols() below.
static int generate_impl(gx_table *t, int table_id, int sf, int64_t o0, int64_t o1, int node, int nnodes, const int32_t *colmap)
{
    gx_ctx *ctx = t->ctx;
    const int32_t *schema; int nschema;
    switch (table_id) {
        case GXG_T_ORDERS: schema = k_schema_orders; nschema = GXG_O_NCOLS; break;
        case GXG_T_LINEITEM: schema = k_schema_lineitem; nschema = GXG_L_NCOLS; break;
        case GXG_T_CUSTOMER: schema = k_schema_customer; nschema = GXG_C_NCOLS; break;
        default: GX_SET_ERR(ctx, "generate: unknown table id %d", table_id); return GX_ERR_ARG;
    }
    GX_CHECK_ARG(ctx, sf >= 1 && o0 >= 0 && o1 >= o0, "generate: bad range");
    GX_CHECK_ARG(ctx, nnodes >= 1 && node >= 0 && node < nnodes, "generate: bad node %d/%d", node, nnodes);
    GX_CHECK_ARG(ctx, nnodes == 1 || nnodes == ctx->nnodes, "generate: nnodes %d != installed shard map (%d); call gx_set_shardmap first", nnodes, ctx->nnodes);
    gx_gen_args a; memset(&a, 0, sizeof(a));
    a.table_id = table_id; a.sf = sf; a.node = node; a.nnodes = nnodes; a.o0 = o0; a.o1 = o1; a.base_row = t->nrows;
    a.shardmap = ctx->d_shardmap;
    for (int c = 0; c < t->ncols; c++) {
        int sc = colmap ? colmap[c] : c;
        GX_CHECK_ARG(ctx, sc >= 0 && sc < nschema && schema[sc] == t->types[c], "generate: table column %d does not match schema column %d", c, sc);
        a.cols[sc] = t->cols[c];
    }
    long long n = o1 - o0;
    if (n == 0) return GX_OK;
    const int BS = 256;
    long long nblocks = (n + BS - 1) / BS;
    long long *d_sums;
    GX_CUDA(ctx, gx_tmp_alloc(ctx, (void **) &d_sums, (size_t) nblocks * sizeof(long long)));
    {
        gx_launch_scope ls(ctx, "generate", 3);
        gx_k_gen_count<<<(unsigned) nblocks, BS, 0, ctx->stream>>>(a, d_sums);
        gx_k_scan_inplace<<<1, 1024, 0, ctx->stream>>>(d_sums, nblocks, ctx->d_scratch);
    }
    cudaError_t e = cudaMemcpyAsync(ctx->h_scratch, ctx->d_scratch, sizeof(long long), cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) { gx_tmp_free(ctx, d_sums); GX_SET_ERR(ctx, "generate: %s", cudaGetErrorString(e)); return GX_ERR_CUDA; }
    long long total = ctx->h_scratch[0];
    if (t->nrows + total > t->capacity) {
        gx_tmp_free(ctx, d_sums);
        GX_SET_ERR(ctx, "generate: %lld + %lld rows exceed capacity %lld", (long long) t->nrows, total, (long long) t->capacity);
        return GX_ERR_ARG;
    }
    gx_k_gen_write<<<(unsigned) nblocks, BS, 0, ctx->stream>>>(a, d_sums);
    e = cudaStreamSynchronize(ctx->stream);
    gx_tmp_free(ctx, d_sums);
    if (e != cudaSuccess) { GX_SET_ERR(ctx, "generate: %s", cudaGetErrorString(e)); return GX_ERR_CUDA; }
    t->nrows += total;
    t->version = gx_table_next_version();
    return GX_OK;
}

extern "C" int gx_table_generate(gx_table *t, int table_id, int sf, int64_t order0, int64_t order1, int node, int nnodes)
{
    if (!t) return GX_ERR_ARG;
    int rc = gx_table_settle(t); if (rc) return rc;
    return generate_impl(t, table_id, sf, order0, order1, node, nnodes, nullptr);
}
// colmap[c] = schema column number feeding table column c (bench: only the referenced columns)
extern "C" int gx_table_generate_cols(gx_table *t, int table_id, int sf, int64_t order0, int64_t order1,
                                      int node, int nnodes, const int32_t *colmap)
{
    if (!t || !colmap) return GX_ERR_ARG;
    int rc = gx_table_settle(t); if (rc) return rc;
    return generate_impl(t, table_id, sf, order0, order1, node, nnodes, colmap);
}

// ------------------------------------------------------------- K1 filter
struct gx_filter_args {
    int npreds, ncols;
    gx_dpred preds[GX_MAX_PREDS];
    gx_dcol in[GX_MAX_COLS];
    void *out[GX_MAX_COLS];
    uint8_t *out_nulls[GX_MAX_COLS];
    long long nrows;
};

// ---- one pass, order preserving: quals -> compaction -> projection ------------------------
// A CTA takes tiles of FT_ROWS rows in ticket order.  Per tile: evaluate the quals (8 rows per
// thread, coalesced), rank the survivors (warp ballots + a 64-entry scan of the per-warp
// counts), publish the tile's count, obtain the tile's output offset by decoupled look-back
// over the tile-status array (a tile never waits for a tile that has not started: tickets are
// handed out in order), then copy the surviving rows of every projected column.  One kernel, no
// count pass, no host round trip between counting and writing; the row order of the input is
// kept (a key-ordered table stays key-ordered, which the join build and the run kernels use).
#define FT_THREADS 256
#define FT_AGG     (1ULL << 62)        /* tile's own count is available */
#define FT_INC     (2ULL << 62)        /* inclusive prefix is available */
#define FT_VAL     ((1ULL << 62) - 1)

__device__ __forceinline__ bool filter_pass(const gx_filter_args &a, long long r)
{
    bool ok = true;
#pragma unroll
    for (int p = 0; p < GX_MAX_PREDS; p++) if (p < a.npreds) ok = ok && gx_eval_pred(a.preds[p], r);
    return ok;
}

// FT_K rows per thread and tile (8: tiles of 2048 rows; 16: tiles of 4096 rows, half the barriers and look-backs per row).
// MARK 0: the quals decide; 1: a row must also have its bit set in `mark` (one bit per input row); 2: its bit clear
template <int FT_K, int MARK>
__device__ __forceinline__ void filter_onepass(const gx_filter_args &a, const unsigned int *mark, unsigned long long *tile_state, unsigned int *ticket,
                                               long long ntiles, long long *total_out)
{
    constexpr int FT_ROWS = FT_THREADS * FT_K;
    constexpr int NCNT = FT_K * (FT_THREADS / 32);          // (k, warp) counts per tile: 64 or 128
    __shared__ unsigned int wc[FT_K][FT_THREADS / 32];
    __shared__ unsigned int woff[FT_K][FT_THREADS / 32];
    __shared__ long long s_tile, s_prefix;
    __shared__ unsigned int s_total;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned int lt = (1u << lane) - 1;
    for (;;) {
        if (threadIdx.x == 0) s_tile = (long long) atomicAdd(ticket, 1u);
        __syncthreads();
        const long long tile = s_tile;
        if (tile >= ntiles) return;
        const long long base = tile * FT_ROWS;
        bool keep[FT_K]; unsigned int rank[FT_K];
        {
            // quals column by column: a descriptor is decoded once per tile and its FT_K loads are in flight together
            long long rr[FT_K];
#pragma unroll
            for (int k = 0; k < FT_K; k++) { rr[k] = base + k * FT_THREADS + threadIdx.x; keep[k] = rr[k] < a.nrows; }
#pragma unroll
            for (int p = 0; p < GX_MAX_PREDS; p++) if (p < a.npreds) pred_tile<FT_K>(a.preds[p], rr, keep);
            if (MARK != 0) {
                // a warp's 32 rows share one bitmap word (tiles start at multiples of FT_ROWS): one broadcast load
#pragma unroll
                for (int k = 0; k < FT_K; k++)
                    if (keep[k]) keep[k] = ((__ldg(mark + (rr[k] >> 5)) >> (rr[k] & 31)) & 1u) == (MARK == 1 ? 1u : 0u);
            }
        }
#pragma unroll
        for (int k = 0; k < FT_K; k++) {
            const unsigned int m = __ballot_sync(0xffffffffu, keep[k]);
            rank[k] = __popc(m & lt);
            if (lane == 0) wc[k][warp] = __popc(m);
        }
        __syncthreads();
        if (threadIdx.x < 32) {                                 // exclusive scan of the NCNT (k, warp) counts, k-major
            constexpr int PER = NCNT / 32;                      // consecutive counts per lane: 2 or 4
            unsigned int cv[PER], x = 0;
#pragma unroll
            for (int q = 0; q < PER; q++) { cv[q] = ((unsigned int *) wc)[PER * lane + q]; x += cv[q]; }
            unsigned int inc = x;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { unsigned int y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
            unsigned int run = inc - x;
#pragma unroll
            for (int q = 0; q < PER; q++) { ((unsigned int *) woff)[PER * lane + q] = run; run += cv[q]; }
            const unsigned int total = __shfl_sync(0xffffffffu, inc, 31);
            // ---- publish, then look back (warp-parallel: 32 predecessors per round)
            long long prefix = 0;
            if (lane == 0) {
                s_total = total;
                __threadfence();
                atomicExch(&tile_state[tile], (tile == 0 ? FT_INC : FT_AGG) | (unsigned long long) total);
            }
            if (tile > 0) {
                long long look = tile - 1;
                for (;;) {
                    const long long t = look - lane;
                    unsigned long long st = FT_INC;                       // tiles before 0: inclusive prefix 0
                    if (t >= 0) { do { st = *(volatile unsigned long long *) &tile_state[t]; } while ((st >> 62) == 0); }
                    const unsigned int incm = __ballot_sync(0xffffffffu, (st >> 62) == 2);
                    const int first = incm ? __ffs((int) incm) - 1 : 32;  // nearest predecessor holding an inclusive prefix
                    unsigned long long v = lane <= first ? (st & FT_VAL) : 0ULL;
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
                    prefix += (long long) __shfl_sync(0xffffffffu, v, 0);
                    if (incm) break;
                    look -= 32;
                }
                if (lane == 0) { __threadfence(); atomicExch(&tile_state[tile], FT_INC | (unsigned long long) (prefix + total)); }
            }
            if (lane == 0) { s_prefix = prefix; if (tile == ntiles - 1) *total_out = prefix + total; }
        }
        __syncthreads();
        const long long prefix = s_prefix;
#pragma unroll
        for (int h8 = 0; h8 < FT_K; h8 += 8) {                  // eight rows at a time: their loads in flight together
            long long rr[8], dd[8]; bool kp[8];
#pragma unroll
            for (int k = 0; k < 8; k++) { rr[k] = base + (h8 + k) * FT_THREADS + threadIdx.x; dd[k] = prefix + woff[h8 + k][warp] + rank[h8 + k]; kp[k] = keep[h8 + k]; }
            for (int c = 0; c < a.ncols; c++) gx_copy_rows<8>(a.in[c], a.out[c], a.out_nulls[c], rr, dd, kp);
        }
        __syncthreads();                                        // wc / woff / s_* are reused by the next tile
    }
}
template <int FT_K>
__global__ void __launch_bounds__(FT_THREADS, 4) gx_k_filter_onepass(gx_filter_args a, unsigned long long *tile_state, unsigned int *ticket, long long ntiles, long long *total_out)
{
    filter_onepass<FT_K, 0>(a, nullptr, tile_state, ticket, ntiles, total_out);
}
// the same compaction restricted to the marked (MARK 1) or unmarked (MARK 2) rows: the build side of gx_hash_agg_right
template <int FT_K, int MARK>
__global__ void __launch_bounds__(FT_THREADS, 4) gx_k_filter_onepass(gx_filter_args a, unsigned long long *tile_state, unsigned int *ticket, long long ntiles, long long *total_out,
                                                                  const unsigned int *mark)
{
    filter_onepass<FT_K, MARK>(a, mark, tile_state, ticket, ntiles, total_out);
}

static gx_dcol make_dcol(const gx_table *t, int c)
{
    gx_dcol d; d.data = t->cols[c]; d.nulls = t->nulls[c]; d.type = t->types[c]; d._pad = 0; return d;
}
int gx_fill_dpreds(gx_ctx *ctx, const gx_table *t, int n_preds, const gx_pred *preds, gx_dpred *out)
{
    GX_CHECK_ARG(ctx, n_preds >= 0 && n_preds <= GX_MAX_PREDS, "too many predicates (%d)", n_preds);
    for (int i = 0; i < n_preds; i++) {
        GX_CHECK_ARG(ctx, preds[i].col >= 0 && preds[i].col < t->ncols, "predicate %d: column %d out of range", i, preds[i].col);
        GX_CHECK_ARG(ctx, preds[i].op >= GX_LT && preds[i].op <= GX_NE, "predicate %d: bad operator %d", i, preds[i].op);
        out[i].col = make_dcol(t, preds[i].col);
        out[i].op = preds[i].op; out[i]._pad = 0; out[i].ival = preds[i].ival; out[i].fval = preds[i].fval;
    }
    return GX_OK;
}

// mark_mode 0: quals only; 1 / 2: also the rows whose bit in `mark` is set / clear (gx_filter_marked)
static int scan_filter_run(gx_ctx *ctx, const gx_table *in, int n_preds, const gx_pred *preds,
                           int n_out_cols, const int32_t *out_cols, const unsigned int *mark, int mark_mode, gx_table **out)
{
    GX_CHECK_ARG(ctx, n_out_cols > 0 && n_out_cols <= GX_MAX_COLS, "scan_filter: bad output column count");
    gx_filter_args a; memset(&a, 0, sizeof(a));
    a.npreds = n_preds; a.ncols = n_out_cols; a.nrows = in->nrows;
    int rc = gx_fill_dpreds(ctx, in, n_preds, preds, a.preds); if (rc) return rc;
    int32_t types[GX_MAX_COLS]; bool hn[GX_MAX_COLS];
    for (int c = 0; c < n_out_cols; c++) {
        GX_CHECK_ARG(ctx, out_cols[c] >= 0 && out_cols[c] < in->ncols, "scan_filter: column %d out of range", out_cols[c]);
        a.in[c] = make_dcol(in, out_cols[c]); types[c] = in->types[out_cols[c]]; hn[c] = in->nulls[out_cols[c]] != nullptr;
    }
    // the output is sized for the worst case (every row survives): stream-ordered pool memory, untouched pages cost nothing
    gx_table *t;
    rc = gx_table_alloc_like(ctx, n_out_cols, types, hn, in->nrows > 0 ? in->nrows : 1, &t);
    if (rc) return rc;
    long long total = 0;
    if (in->nrows > 0) {
        for (int c = 0; c < n_out_cols; c++) { a.out[c] = t->cols[c]; a.out_nulls[c] = t->nulls[c]; }
        const char *k16 = getenv("GX_FILTER_K16");
        const bool big = mark_mode != 0 || !(k16 && k16[0] == '0');    // 4096-row tiles unless GX_FILTER_K16=0 (marked rows: always)
        const long long tile_rows = (long long) FT_THREADS * (big ? 16 : 8);
        const long long ntiles = (in->nrows + tile_rows - 1) / tile_rows;
        unsigned long long *d_state = nullptr;
        cudaError_t e = gx_tmp_alloc(ctx, (void **) &d_state, (size_t) (ntiles + 1) * sizeof(unsigned long long));
        if (e == cudaSuccess) e = cudaMemsetAsync(d_state, 0, (size_t) (ntiles + 1) * sizeof(unsigned long long), ctx->stream);
        if (e == cudaSuccess) {
            gx_launch_scope ls(ctx, "filter");
            gx_launch_scope which(ctx, mark_mode ? "filter_marked" : nullptr, 0);
            long long maxb = (long long) ctx->sm_count * 8;
            const unsigned fgrid = (unsigned) (ntiles < maxb ? ntiles : maxb);
            unsigned int *tk = (unsigned int *) (d_state + ntiles);
            if (mark_mode == 1) gx_k_filter_onepass<16, 1><<<fgrid, FT_THREADS, 0, ctx->stream>>>(a, d_state, tk, ntiles, ctx->d_scratch, mark);
            else if (mark_mode == 2) gx_k_filter_onepass<16, 2><<<fgrid, FT_THREADS, 0, ctx->stream>>>(a, d_state, tk, ntiles, ctx->d_scratch, mark);
            else if (big) gx_k_filter_onepass<16><<<fgrid, FT_THREADS, 0, ctx->stream>>>(a, d_state, tk, ntiles, ctx->d_scratch);
            else gx_k_filter_onepass<8><<<fgrid, FT_THREADS, 0, ctx->stream>>>(a, d_state, tk, ntiles, ctx->d_scratch);
            e = cudaGetLastError();
        }
        if (e == cudaSuccess) e = cudaMemcpyAsync(ctx->h_scratch, ctx->d_scratch, sizeof(long long), cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
        gx_tmp_free(ctx, d_state);
        if (e != cudaSuccess) { gx_table_free(t); GX_SET_ERR(ctx, "scan_filter: %s", cudaGetErrorString(e)); return GX_ERR_CUDA; }
        total = ctx->h_scratch[0];
    }
    t->nrows = total;
    *out = t;
    return GX_OK;
}
extern "C" int gx_scan_filter(gx_ctx *ctx, const gx_table *in, int n_preds, const gx_pred *preds,
                              int n_out_cols, const int32_t *out_cols, gx_table **out)
{
    if (!ctx || !in || !out || !out_cols) return GX_ERR_ARG;
    return scan_filter_run(ctx, in, n_preds, preds, n_out_cols, out_cols, nullptr, 0, out);
}
int gx_filter_marked(gx_ctx *ctx, const gx_table *in, int n_preds, const gx_pred *preds, int n_out_cols,
                     const int32_t *out_cols, const unsigned int *mark, bool keep_marked, gx_table **out)
{
    return scan_filter_run(ctx, in, n_preds, preds, n_out_cols, out_cols, mark, keep_marked ? 1 : 2, out);
}

// ------------------------------------------------- K0 heap-page deform
// Page / tuple layout constants of the reference build
// (storage/bufpage.h:153-175, access/htup_details.h:126-201, storage/itemid.h:24-29):
#define PG_BLCKSZ       8192
#define PG_PAGE_HDR     44      // offsetof(PageHeaderData, pd_linp); LocationIndex is uint32 (__OPENTENBASE_C__)
#define PG_PD_LOWER     16
#define PG_HTH_INFOMASK2 38     // low 11 bits: number of attributes in THIS tuple (HEAP_NATTS_MASK)
#define PG_HTH_INFOMASK 40
#define PG_HTH_HOFF     46
#define PG_HTH_BITS     47
#define PG_HEAP_HASNULL 0x0001

struct gx_deform_args {
    const uint8_t *pages; long long npages;
    const uint16_t *vis; const int32_t *vis_counts; int vis_stride;
    int natts, ncols, maxatt;
    short att_len[64]; signed char att_align[64];
    signed char col_of_att[64];          // table column fed by attribute a, or -1
    void *out[GX_MAX_COLS]; uint8_t *out_nulls[GX_MAX_COLS]; int out_type[GX_MAX_COLS];
    long long base_row;
    int *notnull_violation;              // a NULL arrived in a column declared NOT NULL
};

__device__ __forceinline__ int page_nvisible(const gx_deform_args &a, long long p)
{
    if (a.vis_counts) return a.vis_counts[p];
    const uint8_t *pg = a.pages + p * PG_BLCKSZ;
    int lines = ((int) *(const uint32_t *) (pg + PG_PD_LOWER) - PG_PAGE_HDR) / 4;
    int n = 0;
    for (int i = 0; i < lines; i++) { unsigned int lp = *(const unsigned int *) (pg + PG_PAGE_HDR + 4 * i); n += ((lp >> 15) & 3) == 1; }
    return n;
}
__global__ void gx_k_deform_count(gx_deform_args a, long long *counts)
{
    long long p = (long long) blockIdx.x * blockDim.x + threadIdx.x;
    if (p < a.npages) counts[p] = page_nvisible(a, p);
}

// One warp per page; lane l takes visible tuples l, l+32, ...  Each lane walks
// its tuple's attributes exactly as slot_deform_tuple does
// (access/common/heaptuple.c:1518-1614), storing only referenced columns.
__global__ void gx_k_deform(gx_deform_args a, const long long *pageoffs)
{
    long long p = ((long long) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int lane = threadIdx.x & 31;
    if (p >= a.npages) return;
    const uint8_t *pg = a.pages + p * PG_BLCKSZ;
    int lines = ((int) *(const uint32_t *) (pg + PG_PD_LOWER) - PG_PAGE_HDR) / 4;
    long long row0 = a.base_row + pageoffs[p];
    int nvis = a.vis_counts ? a.vis_counts[p] : -1;
    // without a visibility list: k-th LP_NORMAL item; find by scanning (lane-cooperative ballot)
    int seen = 0;
    for (int base = 0; (nvis >= 0) ? (base < nvis) : (base < lines); base += 32) {
        int idx = base + lane;
        int lineoff = -1, myrow = -1;
        if (nvis >= 0) {
            if (idx < nvis) { lineoff = a.vis[p * a.vis_stride + idx]; myrow = idx; }
        } else {
            bool normal = false;
            if (idx < lines) { unsigned int lp = *(const unsigned int *) (pg + PG_PAGE_HDR + 4 * idx); normal = ((lp >> 15) & 3) == 1; }
            unsigned int m = __ballot_sync(0xffffffffu, normal);
            if (normal) { lineoff = idx + 1; myrow = seen + __popc(m & ((1u << lane) - 1)); }
            seen += __popc(m);
        }
        if (lineoff < 0) continue;
        unsigned int lp = *(const unsigned int *) (pg + PG_PAGE_HDR + 4 * (lineoff - 1));
        const uint8_t *tup = pg + (lp & 0x7FFF);
        bool hasnulls = (*(const uint16_t *) (tup + PG_HTH_INFOMASK) & PG_HEAP_HASNULL) != 0;
        const uint8_t *bp = tup + PG_HTH_BITS;
        const uint8_t *tp = tup + tup[PG_HTH_HOFF];
        unsigned int off = 0;
        long long row = row0 + myrow;
        // a tuple written before ALTER TABLE ADD COLUMN carries fewer attributes than the descriptor:
        // natts = Min(HeapTupleHeaderGetNatts(tup), natts), the rest reads as NULL (heaptuple.c:1424,1497-1502;
        // relations with missing-value defaults are declined by the provider)
        const int tnatts = (int) (*(const uint16_t *) (tup + PG_HTH_INFOMASK2) & 0x07FF);
        for (int att = 0; att < a.maxatt; att++) {
            int c = a.col_of_att[att];
            if (att >= tnatts || (hasnulls && !(bp[att >> 3] & (1 << (att & 7))))) {
                if (c >= 0) {
                    if (a.out_nulls[c]) a.out_nulls[c][row] = 1; else *a.notnull_violation = 1;
                    switch (a.out_type[c]) { case GX_INT4: case GX_DATE: ((int *) a.out[c])[row] = 0; break;
                                             case GX_CHAR: ((signed char *) a.out[c])[row] = 0; break;
                                             default: ((long long *) a.out[c])[row] = 0; }
                }
                continue;
            }
            int len = a.att_len[att], al = a.att_align[att];
            long long v = 0;
            if (len > 0) {
                off = (off + al - 1) & ~(unsigned) (al - 1);                 // att_align_nominal
                if (c >= 0) {
                    switch (len) {
                        case 1: v = (long long) (signed char) tp[off]; break;
                        case 2: v = (long long) *(const short *) (tp + off); break;
                        case 4: v = (long long) *(const int *) (tp + off); break;
                        default: v = *(const long long *) (tp + off); break;
                    }
                }
                off += len;
            } else {
                if (tp[off] == 0) off = (off + al - 1) & ~(unsigned) (al - 1);   // att_align_pointer
                uint8_t h = tp[off];
                unsigned int vsz, hdr;
                if (h & 1) { vsz = (h >> 1) & 0x7F; hdr = 1; }
                else { vsz = (((unsigned) tp[off]) | ((unsigned) tp[off + 1] << 8) | ((unsigned) tp[off + 2] << 16) | ((unsigned) tp[off + 3] << 24)) >> 2; vsz &= 0x3FFFFFFF; hdr = 4; }
                if (c >= 0) v = vsz > hdr ? (long long) (signed char) tp[off + hdr] : 0;  // bpchar(1) -> its byte
                off += vsz;
            }
            if (c >= 0) {
                if (a.out_nulls[c]) a.out_nulls[c][row] = 0;
                switch (a.out_type[c]) { case GX_INT4: case GX_DATE: ((int *) a.out[c])[row] = (int) v; break;
                                         case GX_CHAR: ((signed char *) a.out[c])[row] = (signed char) v; break;
                                         default: ((long long *) a.out[c])[row] = v; }
            }
        }
    }
}

extern "C" int gx_table_append_heap_pages(gx_table *t, const void *pages, int64_t npages, const gx_heap_desc *desc,
                                          const uint16_t *vis_offsets, const int32_t *vis_counts, int32_t vis_stride)
{
    if (!t || !pages || !desc || npages < 0) return GX_ERR_ARG;
    int rc = gx_table_settle(t); if (rc) return rc;
    gx_ctx *ctx = t->ctx;
    GX_CHECK_ARG(ctx, desc->natts > 0 && desc->natts <= 64, "heap desc: natts %d out of range", desc->natts);
    GX_CHECK_ARG(ctx, desc->ncols == t->ncols, "heap desc: ncols %d != table ncols %d", desc->ncols, t->ncols);
    GX_CHECK_ARG(ctx, (vis_offsets == nullptr) == (vis_counts == nullptr), "heap pages: vis_offsets and vis_counts go together");
    if (npages == 0) return GX_OK;
    gx_deform_args a; memset(&a, 0, sizeof(a));
    a.npages = npages; a.natts = desc->natts; a.ncols = desc->ncols; a.vis_stride = vis_stride; a.base_row = t->nrows;
    a.notnull_violation = (int *) (ctx->d_scratch + 20);     // reported by gx_table_load_finish()
    for (int i = 0; i < desc->natts; i++) {
        a.att_len[i] = desc->att_len[i]; a.att_align[i] = desc->att_align[i]; a.col_of_att[i] = -1;
        GX_CHECK_ARG(ctx, a.att_len[i] == -1 || a.att_len[i] == 1 || a.att_len[i] == 2 || a.att_len[i] == 4 || a.att_len[i] == 8, "heap desc: attribute %d has unsupported attlen %d", i, a.att_len[i]);
        GX_CHECK_ARG(ctx, a.att_align[i] == 1 || a.att_align[i] == 2 || a.att_align[i] == 4 || a.att_align[i] == 8, "heap desc: attribute %d has bad attalign", i);
    }
    for (int c = 0; c < desc->ncols; c++) {
        int att = desc->attnums[c];
        GX_CHECK_ARG(ctx, att >= 0 && att < desc->natts, "heap desc: attnum %d out of range", att);
        a.col_of_att[att] = (signed char) c;
        if (att + 1 > a.maxatt) a.maxatt = att + 1;
        // a NOT NULL attribute gets no NULL array (unless the table already has one for it)
        if (!desc->att_notnull[att] || t->nulls[c]) { int rc = ensure_null_array(t, c); if (rc) return rc; }
        a.out[c] = t->cols[c]; a.out_nulls[c] = t->nulls[c]; a.out_type[c] = t->types[c];
    }
    // With visibility lists the host knows every page's row count: the row offsets are scanned here and
    // travel with the batch, so the call only ENQUEUES work (copies + one kernel) — no device round
    // trip per batch.  Without them the LP_NORMAL items are counted on the device (one synchronisation).
    const bool host_counts = vis_counts != nullptr;
    long long total = 0;
    long long *h_offs = nullptr;
    if (host_counts) {
        h_offs = (long long *) malloc((size_t) npages * sizeof(long long));
        for (int64_t p = 0; p < npages; p++) {
            GX_CHECK_ARG(ctx, vis_counts[p] >= 0 && vis_counts[p] <= vis_stride, "heap pages: page %lld has %d visible items (stride %d)", (long long) p, vis_counts[p], vis_stride);
            h_offs[p] = total; total += vis_counts[p];
        }
        if (t->nrows + total > t->capacity) {
            int64_t want = t->capacity * 2 > t->nrows + total ? t->capacity * 2 : t->nrows + total;
            int grc = gx_table_reserve(t, want); if (grc) { free(h_offs); return grc; }
            for (int c = 0; c < desc->ncols; c++) { a.out[c] = t->cols[c]; a.out_nulls[c] = t->nulls[c]; }
        }
    }
    // stage the raw pages (and visibility lists) in HBM
    uint8_t *d_pages = nullptr; uint16_t *d_vis = nullptr; int32_t *d_cnt = nullptr; long long *d_offs = nullptr;
    cudaError_t e = gx_tmp_alloc(ctx, (void **) &d_pages, (size_t) npages * PG_BLCKSZ);
    if (e == cudaSuccess) e = gx_tmp_alloc(ctx, (void **) &d_offs, (size_t) npages * sizeof(long long));
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_pages, pages, (size_t) npages * PG_BLCKSZ, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess && vis_offsets) {
        e = gx_tmp_alloc(ctx, (void **) &d_vis, (size_t) npages * vis_stride * sizeof(uint16_t));
        if (e == cudaSuccess) e = gx_tmp_alloc(ctx, (void **) &d_cnt, (size_t) npages * sizeof(int32_t));
        if (e == cudaSuccess) e = cudaMemcpyAsync(d_vis, vis_offsets, (size_t) npages * vis_stride * sizeof(uint16_t), cudaMemcpyHostToDevice, ctx->stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(d_cnt, vis_counts, (size_t) npages * sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream);
    }
    rc = GX_OK;
    if (e == cudaSuccess && host_counts) {
        a.pages = d_pages; a.vis = d_vis; a.vis_counts = d_cnt;
        // h_offs is pageable: the copy is staged by the driver before the call returns
        e = cudaMemcpyAsync(d_offs, h_offs, (size_t) npages * sizeof(long long), cudaMemcpyHostToDevice, ctx->stream);
        if (e == cudaSuccess) {
            gx_launch_scope ls(ctx, "deform", 1);
            long long nthreads = npages * 32;
            gx_k_deform<<<(unsigned) ((nthreads + 255) / 256), 256, 0, ctx->stream>>>(a, d_offs);
            e = cudaGetLastError();
        }
        if (e == cudaSuccess) { t->nrows += total; t->version = gx_table_next_version(); e = gx_stage_mark(ctx, pages); }
    } else if (e == cudaSuccess) {
        a.pages = d_pages; a.vis = d_vis; a.vis_counts = d_cnt;
        {
            gx_launch_scope ls(ctx, "deform", 2);
            gx_k_deform_count<<<(unsigned) ((npages + 255) / 256), 256, 0, ctx->stream>>>(a, d_offs);
            gx_k_scan_inplace<<<1, 1024, 0, ctx->stream>>>(d_offs, npages, ctx->d_scratch);
        }
        e = cudaMemcpyAsync(ctx->h_scratch, ctx->d_scratch, sizeof(long long), cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
        if (e == cudaSuccess) {
            total = ctx->h_scratch[0];
            if (t->nrows + total > t->capacity) {
                int64_t want = t->capacity * 2 > t->nrows + total ? t->capacity * 2 : t->nrows + total;
                rc = gx_table_reserve(t, want);
                for (int c = 0; c < desc->ncols; c++) { a.out[c] = t->cols[c]; a.out_nulls[c] = t->nulls[c]; }
            }
            if (rc == GX_OK) {
                {
                    gx_launch_scope ls(ctx, "deform", 1);
                    long long nthreads = npages * 32;
                    gx_k_deform<<<(unsigned) ((nthreads + 255) / 256), 256, 0, ctx->stream>>>(a, d_offs);
                }
                e = cudaStreamSynchronize(ctx->stream);
                if (e == cudaSuccess) { t->nrows += total; t->version = gx_table_next_version(); }
            }
        }
    }
    free(h_offs);
    gx_tmp_free(ctx, d_pages); gx_tmp_free(ctx, d_offs); if (d_vis) gx_tmp_free(ctx, d_vis); if (d_cnt) gx_tmp_free(ctx, d_cnt);
    if (e != cudaSuccess) { GX_SET_ERR(ctx, "append_heap_pages: %s", cudaGetErrorString(e)); return e == cudaErrorMemoryAllocation ? GX_ERR_NOMEM : GX_ERR_CUDA; }
    return rc;
}
