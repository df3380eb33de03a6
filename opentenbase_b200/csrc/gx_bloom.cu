// gx_bloom.cu — the reference's split block bloom filter on the device (SURVEY.md §8 row a8).
//
// Replaces BlockBloomFilterInit / Insert / Find (utils/misc/bloomfilter.c:54,140,162), which the hash join
// fills while it builds (nodeHash.c:717-726, one Insert per inner tuple with the tuple's hash value) and asks
// on the probe side before it touches a bucket (ExecHashJoinBloomFilter, nodeHashjoin.c:1862).  Same geometry,
// bit for bit: 32-byte buckets of eight 32-bit words, bucket = Rehash32to32(hash) & mask, one bit per word at
// position (REHASH[i] * hash) >> 27; sized by MinLogSpace(ndv, 0.05) and abandoned above 2^20 buckets
// (bloomfilter.c:20-35,68).  The hash is the join's own ExecHashGetHashValue for one key column with the
// default "new hash": CRC32C of the value widened to int64 (hashint4new/hashint8new, hashfunc.c:112-175).
// A filter is at most 32 MB, i.e. L2-resident on H100 (50 MB of L2): a Find costs one L2 sector, not a DRAM one.
#include <math.h>
#include "gx_internal.cuh"

struct gx_bloom { gx_ctx *ctx; int log_num_buckets; unsigned int *words; int64_t ninsert; };

int gx_fill_dpreds(gx_ctx *ctx, const gx_table *t, int n_preds, const gx_pred *preds, gx_dpred *out);

__device__ __forceinline__ unsigned int bloom_rehash(unsigned int hash)
{
    return (unsigned int) (((unsigned long long) hash * 0x7850f11ec6d14889ULL + 0x6773610597ca4c63ULL) >> 32);
}
__constant__ unsigned int k_bloom_rehash[8] = { 0x47b6137bU, 0x44974d91U, 0x8824ad5bU, 0xa2b7289dU, 0x705495c7U, 0x2df1424bU, 0x9efc4947U, 0x5c6bfb31U };

struct gx_bloom_args { gx_dcol key; long long nrows; int npreds, _pad; gx_dpred preds[GX_MAX_PREDS]; unsigned int *words; unsigned int mask; unsigned char *pass; };

__device__ __forceinline__ unsigned int bloom_key_hash(const gx_dcol &key, long long r)
{
    // hashint4new widens to int64 before hashing, so int4/date and int8 keys of equal value hash alike
    return gx_crc32c_u64((unsigned long long) gx_load_int(key, r));
}
__global__ void gx_k_bloom_insert(gx_bloom_args a)
{
    const long long stride = (long long) gridDim.x * blockDim.x;
    for (long long r = (long long) blockIdx.x * blockDim.x + threadIdx.x; r < a.nrows; r += stride) {
        if (gx_is_null(a.key, r)) continue;                         // hashStrict: NULL keys never reach the table
        bool ok = true;
        for (int p = 0; p < a.npreds; p++) ok = ok && gx_eval_pred(a.preds[p], r);
        if (!ok) continue;
        const unsigned int h = bloom_key_hash(a.key, r);
        unsigned int *bucket = a.words + (size_t) (bloom_rehash(h) & a.mask) * 8;
#pragma unroll
        for (int i = 0; i < 8; i++) atomicOr(&bucket[i], 1u << ((k_bloom_rehash[i] * h) >> 27));
    }
}
__global__ void gx_k_bloom_find(gx_bloom_args a)
{
    const long long stride = (long long) gridDim.x * blockDim.x;
    for (long long r = (long long) blockIdx.x * blockDim.x + threadIdx.x; r < a.nrows; r += stride) {
        bool pass = false;
        if (!gx_is_null(a.key, r)) {
            const unsigned int h = bloom_key_hash(a.key, r);
            const uint4 *b4 = (const uint4 *) (a.words + (size_t) (bloom_rehash(h) & a.mask) * 8);
            const uint4 lo = __ldg(b4), hi = __ldg(b4 + 1);       // the whole bucket: one 32-byte sector
            const unsigned int w[8] = { lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w };
            pass = true;
#pragma unroll
            for (int i = 0; i < 8; i++) pass = pass && ((w[i] >> ((k_bloom_rehash[i] * h) >> 27)) & 1u);
        }
        a.pass[r] = pass ? 1 : 0;
    }
}

// MinLogSpace, bloomfilter.c:20-35 (k = 8 hash functions)
static int min_log_space(int64_t ndv, double fpp)
{
    if (ndv <= 0) return 0;
    const double k = 8.0, m = -k * (double) ndv / log(1 - pow(fpp, 1.0 / k));
    int v = (int) ceil(log2(m / 8));
    return v > 0 ? v : 0;
}

// *out = NULL with GX_OK when the reference would "give up using bloom filter" (more than 2^20 buckets)
extern "C" int gx_bloom_build(gx_ctx *ctx, const gx_table *inner, int key_col, int n_preds, const gx_pred *preds, gx_bloom **out)
{
    if (!ctx || !inner || !out) return GX_ERR_ARG;
    *out = nullptr;
    GX_CHECK_ARG(ctx, key_col >= 0 && key_col < inner->ncols, "bloom_build: key column %d out of range", key_col);
    const int kt = inner->types[key_col];
    GX_CHECK_ARG(ctx, kt == GX_INT4 || kt == GX_INT8 || kt == GX_DATE, "bloom_build: key type %d not supported", kt);
    int lnb = min_log_space(inner->nrows, 0.05) - 5;              // BLOOM_ERROR_RATE (nodeHash.c:57); 32-byte buckets
    if (lnb < 1) lnb = 1;
    if (lnb > 20) return GX_OK;
    gx_bloom_args a; memset(&a, 0, sizeof(a));
    int rc = gx_fill_dpreds(ctx, inner, n_preds, preds, a.preds); if (rc) return rc;
    gx_bloom *b = (gx_bloom *) calloc(1, sizeof(gx_bloom));
    b->ctx = ctx; b->log_num_buckets = lnb; b->ninsert = inner->nrows;
    const size_t bytes = (size_t) 32 << lnb;
    cudaError_t e = gx_tmp_alloc(ctx, (void **) &b->words, bytes);
    if (e == cudaSuccess) e = cudaMemsetAsync(b->words, 0, bytes, ctx->stream);
    if (e != cudaSuccess) { free(b); GX_SET_ERR(ctx, "bloom_build: %s", cudaGetErrorString(e)); return GX_ERR_NOMEM; }
    a.key.data = inner->cols[key_col]; a.key.nulls = inner->nulls[key_col]; a.key.type = kt;
    a.nrows = inner->nrows; a.npreds = n_preds; a.words = b->words; a.mask = (1u << lnb) - 1;
    if (inner->nrows > 0) {
        gx_launch_scope ls(ctx, "bloom_build");
        long long nb = (inner->nrows + 255) / 256, maxb = (long long) ctx->sm_count * 8;
        gx_k_bloom_insert<<<(unsigned) (nb < maxb ? nb : maxb), 256, 0, ctx->stream>>>(a);
        GX_CUDA(ctx, cudaGetLastError());
    }
    *out = b;
    return GX_OK;
}
extern "C" int gx_bloom_log_num_buckets(const gx_bloom *b) { return b ? b->log_num_buckets : -1; }
extern "C" int gx_bloom_read_words(gx_bloom *b, uint32_t *host_out /* 8 << log_num_buckets */)
{
    if (!b || !host_out) return GX_ERR_ARG;
    gx_ctx *ctx = b->ctx;
    GX_CUDA(ctx, cudaMemcpyAsync(host_out, b->words, (size_t) 32 << b->log_num_buckets, cudaMemcpyDeviceToHost, ctx->stream));
    GX_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GX_OK;
}
// host_pass[i] = 1 when row i's key may be in the build side (BlockBloomFilterFind); b == NULL passes everything
extern "C" int gx_bloom_test(gx_ctx *ctx, const gx_bloom *b, const gx_table *outer, int key_col, uint8_t *host_pass)
{
    if (!ctx || !outer || !host_pass) return GX_ERR_ARG;
    GX_CHECK_ARG(ctx, key_col >= 0 && key_col < outer->ncols, "bloom_test: key column %d out of range", key_col);
    if (outer->nrows == 0) return GX_OK;
    if (!b) { memset(host_pass, 1, (size_t) outer->nrows); return GX_OK; }
    const int kt = outer->types[key_col];
    GX_CHECK_ARG(ctx, kt == GX_INT4 || kt == GX_INT8 || kt == GX_DATE, "bloom_test: key type %d not supported", kt);
    gx_bloom_args a; memset(&a, 0, sizeof(a));
    a.key.data = outer->cols[key_col]; a.key.nulls = outer->nulls[key_col]; a.key.type = kt;
    a.nrows = outer->nrows; a.words = b->words; a.mask = (1u << b->log_num_buckets) - 1;
    GX_CUDA(ctx, gx_tmp_alloc(ctx, (void **) &a.pass, (size_t) outer->nrows));
    {
        gx_launch_scope ls(ctx, "bloom_find");
        long long nb = (outer->nrows + 255) / 256, maxb = (long long) ctx->sm_count * 8;
        gx_k_bloom_find<<<(unsigned) (nb < maxb ? nb : maxb), 256, 0, ctx->stream>>>(a);
    }
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(host_pass, a.pass, (size_t) outer->nrows, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    gx_tmp_free(ctx, a.pass);
    if (e != cudaSuccess) { GX_SET_ERR(ctx, "bloom_test: %s", cudaGetErrorString(e)); return GX_ERR_CUDA; }
    return GX_OK;
}
extern "C" void gx_bloom_free(gx_bloom *b)
{
    if (!b) return;
    gx_tmp_free(b->ctx, b->words);
    free(b);
}
