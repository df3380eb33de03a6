// gx_internal.cuh — internal structures and device helpers of libgpuexec.so.
// sm_90a (H100) only.  No CPU fallback anywhere: every entry point needs a live ctx.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <stdlib.h>
#include <string>
#include <map>
#include "../../include/gpuexec.h"

#define GX_EMPTY_KEY   ((long long) 0x8000000000000000LL)   /* INT64_MIN marks an empty join slot */
#define GX_MAX_NODES   64
#define GX_SUB_LOG2    11                 /* join table: linear probing wraps inside 2048-slot (32 KB) sub-tables */
#define GX_SUB         (1 << GX_SUB_LOG2)
#define GX_NCOPY       4                  /* copy streams of the host-table loader */

// ---------------------------------------------------------------- host side
struct gx_prof_entry { double ms; int64_t launches; };
#define GX_PROF_POOL 2048
struct gx_prof_rec { cudaEvent_t a, b; const char *name; };

struct gx_nccl_api;   // gx_comm.cu

struct gx_ctx {
    int device;
    int sm_count, cc_major, cc_minor;
    size_t hbm_bytes;
    size_t smem_optin;           // max dynamic smem per block
    size_t l2_bytes;             // cudaDevAttrL2CacheSize
    cudaStream_t stream;         // all kernels
    cudaStream_t copy_streams[GX_NCOPY];   // H2D staging: chunks go round-robin over these (gx_exec.cu)
    cudaEvent_t copy_ev[2][GX_NCOPY];      // [0] inner table landed, [1] outer table landed (per copy stream)
    cudaEvent_t ev_alloc;                  // the copy streams wait for the stream-ordered allocations
    cudaEvent_t ev_t0, ev_t1;    // gx_timer_*
    char err[512];
    int64_t launches;
    int profile;
    std::map<std::string, gx_prof_entry> *prof;
    gx_prof_rec *prof_pool; int prof_used;      // events recorded, not yet resolved
    void *l2flush_buf; size_t l2flush_bytes;
    // pinned staging ring of the heap-page loader (gx_stage_acquire): the host fills one slot while the
    // DMA of the other is in flight
    void *stage[2]; size_t stage_bytes[2]; cudaEvent_t stage_ev[2]; int stage_busy[2]; int stage_next;
    // small device scratch (counters / flags)
    long long *d_scratch;        // 64 x int64
    long long *h_scratch;        // pinned mirror
    // routing
    int32_t *d_shardmap; int nnodes;
    // communicator
    gx_nccl_api *nccl; void *comm; int rank, nranks;
    // peer windows (gx_comm.cu): every rank's exchange block mapped into this process over NVLink;
    // peer_base[p] = rank p's block (control words, then the data window), peer_ready 1 = mapped, -1 = not available
    int peer_ready; size_t peer_win_bytes; char *peer_base[GX_MAX_NODES]; unsigned long long peer_epoch;
};

struct gx_table {
    gx_ctx *ctx;
    int ncols;
    int32_t types[GX_MAX_COLS];
    void *cols[GX_MAX_COLS];
    uint8_t *nulls[GX_MAX_COLS];     // NULL when the column has no NULLs
    int64_t nrows, capacity;
    uint64_t version;                // new, never reused value whenever the table is created or its rows or columns change
    struct gx_hash *deferred;        // join tables built on this table whose fill is deferred (gx_hash::next_deferred)
};
uint64_t gx_table_next_version();    // gx_table.cu
// Fill the join tables built on t whose fill was deferred, before t's rows, columns or storage change: each then answers
// for the table as it was at build time.  freeing: t goes away whatever happens (a table whose fill failed then reports
// that failure on every use).  gx_join.cu
int gx_table_settle(gx_table *t, bool freeing = false);

struct gx_slot { long long key; unsigned long long payload; };   // 16 B
// Compact slot (8 B).  With an order-preserving slot function the keys that can land in one
// 2048-slot sub-table lie within a few thousand key units of each other, so 31 bits of
// (key - kmin) identify a key inside its sub-table whatever the total key span is:
// d = ((key - kmin) << 1) | 1 truncated to 32 bits; d is never 0, which marks an empty slot.
// Half the bytes to write, read and keep in L2.  Needs a payload of at most 4 bytes and the
// exact kmin/kmax of the build side (probe keys outside [kmin, kmax] are rejected before the
// 31-bit compare).
#define GX_CSLOT_D(key, kmin) ((unsigned int) (((((unsigned long long) (key)) - ((unsigned long long) (kmin))) << 1) | 1ULL))
struct gx_cslot { unsigned int d; unsigned int payload; };
// Narrow slot (4 B): one uint32 w = tag | (payload - pbase) << tbits with tag = ((key - kmin) mod 2^(tbits-1)) << 1 | 1,
// so an occupied slot is never 0, which marks an empty one.  It serves the key-ordered build of an int8 key with one
// 4-byte payload column whose values span at most 2^pbits, pbits = 32 - tbits (o_orderdate: 2406 days).  tbits is the
// smallest width with 2^(tbits-1) >= 4 (keys_per_slot GX_SUB + 64) (gx_nslot_tbits):
//  * probes never leave their home sub-table, and the keys that home in one sub-table lie within keys_per_slot GX_SUB
//    (+ under 64 of interpolation rounding) of each other, so two different keys that can meet there differ by less
//    than the tag modulus 2^(tbits-1) and never share a tag;
//  * reconstruction (gx_k_expand_slots): an entry in slot i homes in the same sub-table, so its key offset lies within
//    one sub-table's key span of i keys_per_slot, at most a quarter of the modulus; the offset congruent to the tag
//    nearest that estimate is the key's (gx_tag_key).
// Placement (slot function, amask = 3) is that of gx_cslot, so the home group of four slots is 16 B.  As for gx_cslot,
// probe keys outside [kmin, kmax] are rejected before the tag compare.  The helpers below are the only code that knows
// the encoding.
enum { GX_SLOTS_WIDE = 0, GX_SLOTS_COMPACT = 1, GX_SLOTS_NARROW = 2 };      // gx_slot, gx_cslot, narrow uint32
static inline unsigned int gx_nslot_tbits(double keys_per_slot)
{
    const double need = 4.0 * (keys_per_slot * GX_SUB + 64.0);
    unsigned int t = 2;
    while (t < 32 && (double) (1ULL << (t - 1)) < need) t++;
    return t;
}

// the slot function of a join table (gx_slot_index); tbits / pbase: the narrow slot format's parameters (gx_nslot_*),
// 0 for the other forms
struct gx_slotfn { int mode; unsigned int win; long long kmin; unsigned long long scale; unsigned long long mask; unsigned int shift; unsigned int amask;
                   unsigned int tbits; int pbase; };

struct gx_hash {
    gx_ctx *ctx;
    gx_slot *slots;
    int64_t nslots;                 // power of two
    int64_t nentries;
    int key_type;
    int n_payload;                  // 0: payload = build row number
    int32_t payload_types[GX_MAX_PAYLOAD];
    int unique;
    int mode;                       // slot function: 0 mixing hash, 1 order-preserving interpolation (gx_slot_index)
    long long kmin; unsigned long long scale; unsigned int win; unsigned int shift;
    double avg_chain;               // measured while the table was filled
    int sorted_build;               // built by the partition-free key-ordered path
    // compact form (gx_cslot): produced by the key-ordered build when key range and payload allow;
    // the 16-byte form is materialised from it on demand for consumers that only read that one
    gx_cslot *cslots; unsigned long long cspan;   // cspan = kmax - kmin + 1
    unsigned int *narrow; unsigned int tbits; int pbase;   // narrow form (GX_SLOTS_NARROW) instead of cslots, same cspan
    double keys_per_slot;           // key range / slot range of the interpolation (compact -> wide reconstruction)
    unsigned int amask;             // home slots are aligned to amask + 1 (2 for 16 B slots, 4 for compact ones)
    // rows whose key equals GX_EMPTY_KEY cannot live in the table: side list
    unsigned long long *special_payload; int special_cap; int special_count;
    // what the build read, for gx_hash_agg_right: the table, its version then, and the build quals (applied again
    // when the build rows are compacted)
    const gx_table *src; uint64_t src_version; int n_preds; gx_pred preds[GX_MAX_PREDS];
    // Deferred key-ordered build (gx_join.cu, hash_materialize): the build rows themselves, not yet a table.  Set only for a
    // unique int8 key without NULLs over strictly ascending sampled keys, one int4/date payload column and no build quals,
    // whose narrowest table would not fit L2.  The merge probe (gx_agg.cu) reads bkey / bpay; every other reader fills the
    // table first.
    struct gx_deferred *deferred;   // nullptr: the table is filled
    const long long *bkey; const int *bpay; long long nbuild;
    gx_hash *next_deferred;         // src->deferred list
};

int gx_hash_wide(gx_ctx *ctx, gx_hash *h);
// fill a deferred table exactly as gx_hash_build would have (no-op for a filled one); gx_join.cu
int hash_materialize(gx_hash *h);
// strided sample of an int8 key column without NULLs: *order bit 0 = two sampled keys descend, bit 1 = two are equal
// (one launch and one synchronise); gx_join.cu
int gx_sample_order(gx_ctx *ctx, const long long *keys, long long nrows, int *order);
// the slot function (and slot format parameters) a table was built with
static inline gx_slotfn gx_hash_slotfn(const gx_hash *h)
{
    gx_slotfn f;
    f.mode = h->mode; f.win = h->win; f.kmin = h->kmin; f.scale = h->scale; f.mask = (unsigned long long) h->nslots - 1;
    f.shift = h->shift; f.amask = h->amask; f.tbits = h->tbits; f.pbase = h->pbase;
    return f;
}
cudaError_t gx_stage_mark(gx_ctx *ctx, const void *host);   // gx_exec.cu: record "copy of this staging slot enqueued"   // materialise the 16-byte slot array of a compact table

// A group-state record: [null bits][k0][k1][w0..w(nwords-1)], 8-byte words.
// w0 is always the group's row count.
#define GX_MAX_WORDS 18

// where a record keeps each group column and each aggregate's state, and how its state words merge
struct gx_rec_layout {
    int nkw;                         // key words (1 or 2)
    int nwords;                      // state words
    int rec_words;                   // 3 + nwords (the null bits, k0 and k1 are always present)
    int need_w0;                     // w0 (rows per group) is maintained
    int32_t group_types[GX_MAX_GROUP_COLS];
    int gword[GX_MAX_GROUP_COLS], gshift[GX_MAX_GROUP_COLS], gbytes[GX_MAX_GROUP_COLS];   // k0 or k1, bit offset, width
    int agg_word[GX_MAX_AGGS];       // first word of the aggregate's state
    int agg_cnt_word[GX_MAX_AGGS];   // word holding its non-NULL input count (may be 0 = row count)
    int agg_var_word[GX_MAX_AGGS];   // variance aggregates: the shift C, followed by S1 and S2 (0 = none)
    int wkind[GX_MAX_WORDS];         // merge kind of each state word (gx_agg.cu, WK_*)
    long long winit[GX_MAX_WORDS];   // initial value of each state word
};

struct gx_result {
    gx_ctx *ctx;
    gx_agg_plan plan;
    gx_rec_layout L;
    long long *d_recs;               // ngroups * L.rec_words (dense, partial states)
    unsigned int *d_nullmask;        // ngroups (group-key null bits)
    int64_t ngroups, cap;
    int finalized_across;            // combined over the communicator already
    int plain_row_elsewhere;         // combined plain aggregate: another rank returns its one row
};
// a plain aggregate over zero rows: this result returns the one row of initial states
static inline bool gx_result_plain_empty(const gx_result *r) { return r->plan.n_group_cols == 0 && r->ngroups == 0 && !r->plain_row_elsewhere; }

bool gx_result_has_distinct(const gx_result *r);      // some aggregate is GX_AGG_COUNT_DISTINCT: no partial states
bool gx_result_has_variance(const gx_result *r);      // some aggregate is GX_AGG_VAR_* / GX_AGG_STDDEV_*
bool gx_result_has_regr(const gx_result *r);          // some aggregate is GX_AGG_REGR_COUNT .. GX_AGG_CORR_F8
static inline bool gx_is_var_fn(int fn) { return fn >= GX_AGG_VAR_POP_F8 && fn <= GX_AGG_STDDEV_SAMP_F8; }
__host__ __device__ static inline bool gx_is_regr_fn(int fn) { return fn >= GX_AGG_REGR_COUNT && fn <= GX_AGG_CORR_F8; }

#define GX_SET_ERR(ctx, ...) do { if (ctx) snprintf((ctx)->err, sizeof((ctx)->err), __VA_ARGS__); \
                                  gx_set_global_err(__VA_ARGS__); } while (0)
void gx_set_global_err(const char *fmt, ...);

#define GX_CUDA(ctx, call) do { cudaError_t e__ = (call); if (e__ != cudaSuccess) { \
    GX_SET_ERR(ctx, "CUDA error %s at %s:%d: %s", cudaGetErrorName(e__), __FILE__, __LINE__, cudaGetErrorString(e__)); \
    return (e__ == cudaErrorMemoryAllocation) ? GX_ERR_NOMEM : GX_ERR_CUDA; } } while (0)

#define GX_CHECK_ARG(ctx, cond, ...) do { if (!(cond)) { GX_SET_ERR(ctx, __VA_ARGS__); return GX_ERR_ARG; } } while (0)

// launch accounting + optional per-kernel CUDA-event timing (name nullptr: nothing is recorded)
struct gx_launch_scope {
    gx_ctx *ctx; const char *name;
    int slot;
    gx_launch_scope(gx_ctx *c, const char *n, int nlaunch = 1) : ctx(c), name(n), slot(-1) {
        ctx->launches += nlaunch;
        // events are only recorded here (asynchronously); gx_profile_get() resolves them
        if (name && ctx->profile && ctx->prof_used < GX_PROF_POOL) {
            slot = ctx->prof_used++;
            ctx->prof_pool[slot].name = name;
            cudaEventRecord(ctx->prof_pool[slot].a, ctx->stream);
        }
    }
    ~gx_launch_scope() { if (slot >= 0) cudaEventRecord(ctx->prof_pool[slot].b, ctx->stream); }
};

static inline int gx_type_size(int t)
{
    switch (t) { case GX_INT4: case GX_DATE: return 4; case GX_INT8: case GX_FLOAT8: return 8; case GX_CHAR: return 1; }
    return 0;
}
static inline int64_t gx_pow2_ceil(int64_t x) { int64_t p = 1; while (p < x) p <<= 1; return p; }

// Stream-ordered, pool-cached device allocations for per-query temporaries (join table,
// bucket buffers, group tables): cudaMalloc/cudaFree of multi-GB blocks cost milliseconds per query.
static inline cudaError_t gx_tmp_alloc(gx_ctx *ctx, void **p, size_t bytes) { return cudaMallocAsync(p, bytes ? bytes : 8, ctx->stream); }
static inline void gx_tmp_free(gx_ctx *ctx, void *p) { if (p) cudaFreeAsync(p, ctx->stream); }

int gx_table_alloc_like(gx_ctx *ctx, int ncols, const int32_t *types, const bool *has_nulls,
                        int64_t capacity, gx_table **out);
// gx_scan_filter that also keeps only the rows whose bit in `mark` (one bit per input row) is set (keep_marked) or
// clear; gx_table.cu
int gx_filter_marked(gx_ctx *ctx, const gx_table *in, int n_preds, const gx_pred *preds, int n_out_cols,
                     const int32_t *out_cols, const unsigned int *mark, bool keep_marked, gx_table **out);
// GX_ERR_ARG unless the plan's join type is one gx_hash_agg runs (INNER, SEMI, ANTI)
int gx_check_agg_join_type(gx_ctx *ctx, const gx_agg_plan *plan);
// what gx_hash_agg(ctx, t, nullptr, plan) would reject before touching the device (GX_ERR_ARG), without running it; t's
// column types and NULL arrays are read, not its rows.  gx_agg.cu
int gx_check_agg_plan(gx_ctx *ctx, const gx_table *t, const gx_agg_plan *plan);

// device-side plan descriptors -------------------------------------------
struct gx_dcol { const void *data; const uint8_t *nulls; int type; int _pad; };

struct gx_dpred { gx_dcol col; int op; int _pad; long long ival; double fval; };

// chain-form expression: acc = term0; acc = acc (op) term_i
enum { GXT_COL = 1, GXT_CONST = 2, GXT_K_SUB_COL = 3, GXT_K_ADD_COL = 4, GXT_K_MUL_COL = 5, GXT_COL_SUB_K = 6 };
struct gx_dterm { int op; int kind; gx_dcol col; double k; };
struct gx_dexpr { int nterms; int _pad; gx_dterm t[4]; };

enum { GXU_NONE = 0, GXU_ADD_F64 = 1, GXU_ADD_I64 = 2, GXU_MIN_F64 = 3, GXU_MAX_F64 = 4, GXU_CNT = 5 };
struct gx_dagg {
    int kind;          // GXU_*
    int word;          // state word receiving the value
    int cnt_word;      // word receiving +1 per non-NULL input (0 = none: w0 row count serves)
    int is_int;        // value is an integer column (SUM_I4/I8, COUNT(col))
    int var_word;      // GXU_ADD_F64 only: first of the words {C, S1, S2} of a variance over the same value (0 = none)
    int _pad;
    gx_dexpr expr;     // float8 argument (kind F64) ...
    gx_dcol icol;      // ... or integer argument column
};

// The state every two-argument aggregate of a plan shares (one (Y, X) pair per plan): a row whose y and x are both
// non-NULL adds +1 to cnt_word (0: w0 counts the rows) and, when word != 0, updates the nine words from `word` on:
// {Sx, Sy, Cx, S1x, S2x, Cy, S1y, S2y, Sxy'} (gx_agg.cu, WK_REGR_C).  on == 0: the plan has no such aggregate.
struct gx_dregr { int on, word, cnt_word, _pad; gx_dexpr y, x; };

struct gx_dgroupcol { int side; int type; gx_dcol col; int payload_idx; int word; int shift; int bytes; int _pad; };

struct gx_dplan {
    int npreds, nagg, ngroup, nkw;
    int nwords, has_join, key_type, unique;
    gx_dpred preds[GX_MAX_PREDS];
    gx_dcol okey;                       // outer join key column
    gx_dgroupcol gcols[GX_MAX_GROUP_COLS];
    gx_dagg aggs[GX_MAX_AGGS];
    int payload_types[GX_MAX_PAYLOAD];
    int n_payload; int join_type;       // GX_JOIN_INNER / _SEMI / _ANTI
    gx_dregr regr;                      // the plan's one (Y, X) pair of the two-argument aggregates
};

#ifdef __CUDACC__
// ---------------------------------------------------------------- device side

__device__ __forceinline__ unsigned int gx_rotl32(unsigned int x, int k) { return __funnelshift_l(x, x, k); }

// final() of Bob Jenkins' lookup3 as used by hash_uint32()
// (reference: src/backend/access/hash/hashfunc.c:593-602, 1044-1058)
__device__ __forceinline__ unsigned int gx_hash_uint32(unsigned int k)
{
    unsigned int a, b, c;
    a = b = c = 0x9e3779b9u + 4u + 3923095u;
    a += k;
    c ^= b; c -= gx_rotl32(b, 14);
    a ^= c; a -= gx_rotl32(c, 11);
    b ^= a; b -= gx_rotl32(a, 25);
    c ^= b; c -= gx_rotl32(b, 16);
    a ^= c; a -= gx_rotl32(c, 4);
    b ^= a; b -= gx_rotl32(a, 14);
    c ^= b; c -= gx_rotl32(b, 24);
    return c;
}
// hashint8(): fold hi into lo (hashfunc.c:92-110)
__device__ __forceinline__ unsigned int gx_hashint8(long long v)
{
    unsigned int lo = (unsigned int) v, hi = (unsigned int) ((unsigned long long) v >> 32);
    lo ^= (v >= 0) ? hi : ~hi;
    return gx_hash_uint32(lo);
}
__device__ __forceinline__ unsigned int gx_hashint4(int v) { return gx_hash_uint32((unsigned int) v); }

// CRC32C of the 8 little-endian bytes of v, bitwise (hash_any_new, hashfunc.c:112)
__device__ __forceinline__ unsigned int gx_crc32c_u64(unsigned long long v)
{
    unsigned int crc = 0xFFFFFFFFu;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        crc ^= (unsigned int) (v >> (8 * i)) & 0xFFu;
#pragma unroll
        for (int j = 0; j < 8; j++) crc = (crc >> 1) ^ (0x82F63B78u & (0u - (crc & 1u)));
    }
    return crc ^ 0xFFFFFFFFu;
}
__device__ __forceinline__ unsigned int gx_murmurhash32(unsigned int h)
{
    h ^= h >> 16; h *= 0x85ebca6bu; h ^= h >> 13; h *= 0xc2b2ae35u; h ^= h >> 16; return h;
}
// internal bucket hash of the join / group tables (need not match the reference:
// SURVEY.md §2 row 7): murmur3 fmix64
__device__ __forceinline__ unsigned long long gx_mix64(unsigned long long h)
{
    h ^= h >> 33; h *= 0xff51afd7ed558ccdULL; h ^= h >> 33; h *= 0xc4ceb9fe1a85ec53ULL; h ^= h >> 33; return h;
}

// SHARD routing, bit-exact (locator.c:1611, shardmap.c:1147): one distribution column
__device__ __forceinline__ int gx_shard_index(unsigned int hashvalue)
{
    int h = (int) hashvalue;
    unsigned int mag = (h < 0) ? (0u - (unsigned int) h) : (unsigned int) h;
    int a = (int) mag;                       // abs(INT_MIN) stays INT_MIN
    return a % GX_SHARD_MAP_SHARD_NUM;       // INT_MIN % 4096 == 0
}
__device__ __forceinline__ unsigned int gx_route_hash(int type, long long datum, bool isnull)
{
    unsigned int hashkey = 0;                // rotl1(0) == 0
    if (!isnull) hashkey ^= (type == GX_INT8) ? gx_hashint8(datum) : gx_hashint4((int) datum);
    return hashkey;
}

// typed column access ------------------------------------------------------
__device__ __forceinline__ long long gx_load_int(const gx_dcol &c, long long r)
{
    switch (c.type) {
        case GX_INT4: case GX_DATE: return (long long) __ldg((const int *) c.data + r);
        case GX_INT8: return __ldg((const long long *) c.data + r);
        case GX_CHAR: return (long long) __ldg((const signed char *) c.data + r);
        default: return __ldg((const long long *) c.data + r);     // FLOAT8 bit pattern
    }
}
__device__ __forceinline__ double gx_load_f64(const gx_dcol &c, long long r)
{
    switch (c.type) {
        case GX_FLOAT8: return __ldg((const double *) c.data + r);
        case GX_INT4: case GX_DATE: return (double) __ldg((const int *) c.data + r);      // i4tod
        case GX_INT8: return (double) __ldg((const long long *) c.data + r);              // i8tod
        default: return (double) __ldg((const signed char *) c.data + r);
    }
}
__device__ __forceinline__ bool gx_is_null(const gx_dcol &c, long long r)
{
    return c.nulls != nullptr && __ldg(c.nulls + r) != 0;
}

// float8_cmp_internal: NaN sorts above everything and equals itself (float.c:1160)
__device__ __forceinline__ int gx_f8cmp(double a, double b)
{
    if (isnan(a)) return isnan(b) ? 0 : 1;
    if (isnan(b)) return -1;
    return a > b ? 1 : (a < b ? -1 : 0);
}
// does "x op y" hold, given c = sign(x - y)?  Branch-free: three bits per operator (c = -1, 0, +1), looked up in one word -
// the switch this replaces compiled to a jump table inside every tile loop (ncu: 8 % of gx_k_runagg's instructions)
#define GX_OP_BITS(op, lt, eq, gt) ((unsigned int) ((lt) | ((eq) << 1) | ((gt) << 2)) << (3 * (op)))
__device__ __forceinline__ bool gx_op_holds(int op, int c)
{
    constexpr unsigned int T = GX_OP_BITS(GX_LT, 1, 0, 0) | GX_OP_BITS(GX_LE, 1, 1, 0) | GX_OP_BITS(GX_EQ, 0, 1, 0) |
                               GX_OP_BITS(GX_GE, 0, 1, 1) | GX_OP_BITS(GX_GT, 0, 0, 1) | GX_OP_BITS(GX_NE, 1, 0, 1);
    return (T >> (3 * op + c + 1)) & 1u;
}
__device__ __forceinline__ bool gx_eval_pred(const gx_dpred &p, long long r)
{
    if (gx_is_null(p.col, r)) return false;          // strict operator: NULL fails the qual
    int c;
    if (p.col.type == GX_FLOAT8) c = gx_f8cmp(gx_load_f64(p.col, r), p.fval);
    else if (p.col.type == GX_CHAR) {                // charlt etc. compare as uint8
        unsigned char x = (unsigned char) gx_load_int(p.col, r), y = (unsigned char) p.ival;
        c = x > y ? 1 : (x < y ? -1 : 0);
    } else { long long x = gx_load_int(p.col, r); c = x > p.ival ? 1 : (x < p.ival ? -1 : 0); }
    return gx_op_holds(p.op, c);
}

// quals of a tile of K rows per lane: the predicate descriptor is decoded once, the K column loads are independent
template <int K>
__device__ __forceinline__ void pred_tile(const gx_dpred &p, const long long (&r)[K], bool (&ok)[K])
{
    if (p.col.nulls == nullptr && (p.col.type == GX_INT4 || p.col.type == GX_DATE)) {
        const int *c = (const int *) p.col.data; int x[K];
#pragma unroll
        for (int j = 0; j < K; j++) x[j] = ok[j] ? __ldg(c + r[j]) : 0;
#pragma unroll
        for (int j = 0; j < K; j++) ok[j] = ok[j] && gx_op_holds(p.op, (long long) x[j] > p.ival ? 1 : ((long long) x[j] < p.ival ? -1 : 0));
    } else if (p.col.nulls == nullptr && p.col.type == GX_FLOAT8) {
        const double *c = (const double *) p.col.data; double x[K];
#pragma unroll
        for (int j = 0; j < K; j++) x[j] = ok[j] ? __ldg(c + r[j]) : 0.0;
#pragma unroll
        for (int j = 0; j < K; j++) ok[j] = ok[j] && gx_op_holds(p.op, gx_f8cmp(x[j], p.fval));
    } else {
#pragma unroll
        for (int j = 0; j < K; j++) if (ok[j]) ok[j] = gx_eval_pred(p, r[j]);
    }
}

// IEEE fp64 ops that ptxas must never contract into FMA: the reference computes
// float8mul/float8pl/float8mi as separate correctly-rounded operations.
__device__ __forceinline__ double gx_apply(int op, double a, double b)
{
    return op == GX_OP_ADD ? __dadd_rn(a, b) : (op == GX_OP_SUB ? __dsub_rn(a, b) : __dmul_rn(a, b));
}
__device__ __forceinline__ double gx_eval_term(const gx_dterm &t, long long r, bool &isnull)
{
    switch (t.kind) {
        case GXT_CONST: return t.k;
        case GXT_COL: isnull |= gx_is_null(t.col, r); return gx_load_f64(t.col, r);
        case GXT_K_SUB_COL: isnull |= gx_is_null(t.col, r); return __dsub_rn(t.k, gx_load_f64(t.col, r));
        case GXT_K_ADD_COL: isnull |= gx_is_null(t.col, r); return __dadd_rn(t.k, gx_load_f64(t.col, r));
        case GXT_K_MUL_COL: isnull |= gx_is_null(t.col, r); return __dmul_rn(t.k, gx_load_f64(t.col, r));
        default: isnull |= gx_is_null(t.col, r); return __dsub_rn(gx_load_f64(t.col, r), t.k);
    }
}
__device__ __forceinline__ double gx_eval_expr(const gx_dexpr &e, long long r, bool &isnull)
{
    double acc = gx_eval_term(e.t[0], r, isnull);
#pragma unroll
    for (int i = 1; i < 4; i++)
        if (i < e.nterms) acc = gx_apply(e.t[i].op, acc, gx_eval_term(e.t[i], r, isnull));
    return acc;
}

// join-table probe -------------------------------------------------------
__device__ __forceinline__ unsigned long long gx_key_hash(long long key) { return gx_mix64((unsigned long long) key); }
// Slot function.  A probe that misses L2 costs a whole 128-byte line of DRAM traffic
// (four 32-byte sectors), i.e. eight 16-byte slots, so it pays
// to keep keys that are probed together in the same line.
//   mode 0: slot = fmix64(key) & mask                      (any keys)
//   mode 1: slot = floor((key - kmin) * scale / 2^64)       order-preserving interpolation:
//           keys spread near-uniformly over [kmin, kmax] (serial primary keys; TPC-H order
//           keys) land in key order, so a probe side clustered on the key walks the table
//           almost sequentially.  Picked from a key-density sample at build time and kept
//           only if the chains measured while filling stay short (else rebuilt with mode 0).
// mode 1 maps keys to slots in key order (probes of a key-ordered outer side then walk
// the table front to back); `win` (0 or 2^w - 1) additionally scatters the low w slot bits
// with a multiplicative hash, which breaks up the pile-ups that locally bunched keys
// (TPC-H order keys: 8 used of every 32) cause under pure interpolation while keeping
// every key inside the same few cache lines and the same sub-table.
__device__ __forceinline__ unsigned long long gx_slot_index(long long key, const gx_slotfn &f)
{
    // Home slots are aligned to amask + 1 slots (2 x 16 B or 4 x 8 B = one 32-byte sector), which a
    // prober fetches as one 32-byte sector; linear probing is unchanged.
    if (f.mode == 0) return gx_mix64((unsigned long long) key) & f.mask & ~(unsigned long long) f.amask;
    if (f.mode == 2) {
        // key range below 2^32: the same interpolation in 32-bit arithmetic (one wide multiply)
        const unsigned int d = (unsigned int) ((unsigned long long) key - (unsigned long long) f.kmin);
        const unsigned long long s = (((unsigned long long) d * (unsigned int) f.scale) >> f.shift) & f.mask;
        return (s ^ (unsigned long long) (((d * 0x9E3779B9u) >> 24) & f.win)) & ~(unsigned long long) f.amask;
    }
    unsigned long long s = __umul64hi((unsigned long long) key - (unsigned long long) f.kmin, f.scale) & f.mask;
    return (s ^ ((unsigned long long) (((unsigned long long) key * 0x9E3779B97F4A7C15ULL) >> 40) & f.win)) & ~(unsigned long long) f.amask;
}
// next aligned pair of a probe sequence (same wrapping rule as gx_next_slot)
__device__ __forceinline__ unsigned long long gx_next_pair(unsigned long long s, unsigned long long mask)
{
    const unsigned long long w = mask < (GX_SUB - 1) ? mask : (unsigned long long) (GX_SUB - 1);
    return (s & ~w) | ((s + 2) & w);
}
__device__ __forceinline__ unsigned long long gx_next_quad(unsigned long long s, unsigned long long mask)
{
    const unsigned long long w = mask < (GX_SUB - 1) ? mask : (unsigned long long) (GX_SUB - 1);
    return (s & ~w) | ((s + 4) & w);
}
// next slot of a probe sequence: wraps inside the slot's sub-table (or the whole table when it is smaller)
__device__ __forceinline__ unsigned long long gx_next_slot(unsigned long long s, unsigned long long mask)
{
    const unsigned long long w = mask < (GX_SUB - 1) ? mask : (unsigned long long) (GX_SUB - 1);
    return (s & ~w) | ((s + 1) & w);
}

// narrow slots (see gx_nslot_tbits) --------------------------------------
__device__ __forceinline__ unsigned int gx_nslot_tag(long long key, const gx_slotfn &f)
{
    return GX_CSLOT_D(key, f.kmin) & ((1u << f.tbits) - 1u);
}
// does a payload fit the slot's 32 - tbits bits above pbase?
__device__ __forceinline__ bool gx_nslot_fits(long long payload, const gx_slotfn &f)
{
    return (unsigned long long) (payload - (long long) f.pbase) < (1ULL << (32 - f.tbits));
}
__device__ __forceinline__ unsigned int gx_nslot_make(long long key, long long payload, const gx_slotfn &f)
{
    return gx_nslot_tag(key, f) | ((unsigned int) (payload - (long long) f.pbase) << f.tbits);
}
__device__ __forceinline__ int gx_nslot_payload(unsigned int w, const gx_slotfn &f) { return f.pbase + (int) (w >> f.tbits); }
// a home group of four narrow slots: one 16-byte load
__device__ __forceinline__ uint4 gx_nslot_ld(const unsigned int *p)
{
    uint4 v;
    asm volatile("ld.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
// one group of a probe walk: true when the walk ends here (a slot holds the tag, or a slot is empty - a table that is only
// ever filled has no match behind an empty slot); found and payload tell which
__device__ __forceinline__ bool gx_nslot_group(const uint4 &q, unsigned int tag, const gx_slotfn &f, bool &found, int &payload)
{
    const unsigned int tm = (1u << f.tbits) - 1u;
    const bool h0 = (q.x & tm) == tag, h1 = (q.y & tm) == tag, h2 = (q.z & tm) == tag, h3 = (q.w & tm) == tag;
    found = h0 | h1 | h2 | h3;
    payload = gx_nslot_payload(h0 ? q.x : h1 ? q.y : h2 ? q.z : q.w, f);
    return found | (q.x == 0u) | (q.y == 0u) | (q.z == 0u) | (q.w == 0u);
}
// two 16-byte slots (one 32-byte sector) as two 128-bit loads (sm_90 has no 256-bit load)
__device__ __forceinline__ void gx_ld_pair(const gx_slot *p, long long &k0, unsigned long long &p0, long long &k1, unsigned long long &p1)
{
    asm volatile("ld.global.v2.u64 {%0, %1}, [%4];\n\tld.global.v2.u64 {%2, %3}, [%4+16];"
                 : "=l"(k0), "=l"(p0), "=l"(k1), "=l"(p1) : "l"(p));
}
#define PT_K 4                            /* rows per lane of a probe tile (gx_k_hash_probe_unique, gx_k_agg_exist) */
// First-match walk of K probe keys per lane over a join table in the format the build wrote (F: gx_slot, gx_cslot or
// narrow), never the 16-byte expansion of a compact or narrow one.  Every row's home group is loaded before any walk
// starts, so the K loads are in flight together.  ok[j] = false: no probe, hit[j] = false.  hit[j] / pay[j]: the key has a
// partner / the first partner's payload.  A key INT64_MIN lives in the side list of a 16-byte table (the compact and
// narrow builds take no such key, and their span test rejects it).  TAB: an argument block carrying the join-table
// fields (slots, cslots, narrow, cspan, mask, sf, special, special_count).
template <int F, int K, class TAB>
__device__ __forceinline__ void gx_probe_first(const TAB &a, const bool (&ok)[K], const long long (&key)[K], bool (&hit)[K], unsigned long long (&pay)[K])
{
    unsigned long long s[K];
    long long k0[K], k1[K]; unsigned long long p0[K], p1[K];
    if (F == GX_SLOTS_NARROW) {
        // four 4-byte slots per 16-byte group, one load each (gx_nslot_group)
        uint4 q[K]; unsigned int tg[K];
#pragma unroll
        for (int j = 0; j < K; j++) {
            const bool inspan = ok[j] && ((unsigned long long) key[j] - (unsigned long long) a.sf.kmin) < a.cspan;   // outside the build side's key span: no partner
            s[j] = gx_slot_index(key[j], a.sf);
            tg[j] = gx_nslot_tag(key[j], a.sf);
            q[j] = inspan ? gx_nslot_ld(a.narrow + s[j]) : make_uint4(0u, 0u, 0u, 0u);    // an empty group ends the walk unmatched
        }
#pragma unroll
        for (int j = 0; j < K; j++) {
            hit[j] = false; pay[j] = 0;
            if (!ok[j]) continue;
            for (;;) {
                bool f; int pv;
                if (gx_nslot_group(q[j], tg[j], a.sf, f, pv)) { hit[j] = f; pay[j] = (unsigned long long) (unsigned int) pv; break; }
                s[j] = gx_next_quad(s[j], a.mask);
                q[j] = gx_nslot_ld(a.narrow + s[j]);
            }
        }
    } else if (F == GX_SLOTS_COMPACT) {
        // four 8-byte slots {d, payload} per 32-byte sector; d = ((key - kmin) << 1) | 1 truncated to 32 bits, 0 = empty
        unsigned int d[K];
#pragma unroll
        for (int j = 0; j < K; j++) {
            const bool inspan = ok[j] && ((unsigned long long) key[j] - (unsigned long long) a.sf.kmin) < a.cspan;   // outside the build side's key span: no partner
            s[j] = gx_slot_index(key[j], a.sf);
            d[j] = GX_CSLOT_D(key[j], a.sf.kmin);
            k0[j] = k1[j] = 0; p0[j] = p1[j] = 0;
            if (inspan) gx_ld_pair((const gx_slot *) (a.cslots + s[j]), k0[j], p0[j], k1[j], p1[j]);
            else d[j] = 0xfffffffeu;                               // even: matches no stored d (they are odd), the all-zero group ends the walk
        }
#pragma unroll
        for (int j = 0; j < K; j++) {
            hit[j] = false; pay[j] = 0;
            if (!ok[j]) continue;
            for (;;) {
                const unsigned int d0 = (unsigned int) k0[j], d1 = (unsigned int) p0[j], d2 = (unsigned int) k1[j], d3 = (unsigned int) p1[j];
                const unsigned long long m = d0 == d[j] ? (unsigned long long) k0[j] : d1 == d[j] ? p0[j] : d2 == d[j] ? (unsigned long long) k1[j] : p1[j];
                hit[j] = (d0 == d[j]) | (d1 == d[j]) | (d2 == d[j]) | (d3 == d[j]);
                pay[j] = m >> 32;
                if (hit[j] | (d0 == 0u) | (d1 == 0u) | (d2 == 0u) | (d3 == 0u)) break;
                s[j] = gx_next_quad(s[j], a.mask);
                gx_ld_pair((const gx_slot *) (a.cslots + s[j]), k0[j], p0[j], k1[j], p1[j]);
            }
        }
    } else {
#pragma unroll
        for (int j = 0; j < K; j++) {
            s[j] = gx_slot_index(key[j], a.sf);            k0[j] = k1[j] = GX_EMPTY_KEY; p0[j] = p1[j] = 0;
            if (ok[j] && key[j] != GX_EMPTY_KEY) gx_ld_pair(a.slots + s[j], k0[j], p0[j], k1[j], p1[j]);
        }
#pragma unroll
        for (int j = 0; j < K; j++) {
            hit[j] = false; pay[j] = 0;
            if (!ok[j]) continue;
            if (key[j] == GX_EMPTY_KEY) { hit[j] = a.special_count > 0; if (hit[j]) pay[j] = a.special[0]; continue; }
            for (;;) {
                if (k0[j] == key[j]) { hit[j] = true; pay[j] = p0[j]; break; }
                if (k0[j] == GX_EMPTY_KEY) break;
                if (k1[j] == key[j]) { hit[j] = true; pay[j] = p1[j]; break; }
                if (k1[j] == GX_EMPTY_KEY) break;
                s[j] = gx_next_pair(s[j], a.mask);
                gx_ld_pair(a.slots + s[j], k0[j], p0[j], k1[j], p1[j]);
            }
        }
    }
}

// One warp's search for the first row of [0, nrows) at which pred holds, pred false before it and true from it on (nrows:
// none): the 32 rows around the guess g decide it in one round when the guess is within 16 rows; otherwise a bracket is
// grown (x16 per round) and narrowed 32-ary.  Over rows that are not so ordered the result is some row in [0, nrows].
template <class PRED>
__device__ __forceinline__ long long gx_warp_lower_bound(long long nrows, long long g, int lane, PRED pred_in)
{
    auto pred = [&](long long r) -> bool {                      // true from the bound onwards
        if (r >= nrows) return true;
        if (r < 0) return false;
        return pred_in(r);
    };
    if (g > nrows) g = nrows;
    // one round when the guess is within 16 rows
    {
        const long long pos = g - 16;
        const unsigned int b = __ballot_sync(0xffffffffu, pred(pos + lane));
        if (b != 0u && b != 0xffffffffu) return pos + (__ffs((int) b) - 1);
    }
    // grow a bracket [lo, hi]: pred(lo - 1) false (or lo == 0), pred(hi) true (or hi == nrows)
    long long lo = 0, hi = nrows;
    for (long long e = 256; ; e *= 16) {
        const long long cl = g - e > 0 ? g - e : 0, ch = g + e < nrows ? g + e : nrows;
        const bool p = lane == 0 ? pred(cl - 1) : (lane == 1 ? pred(ch) : false);
        const unsigned int b = __ballot_sync(0xffffffffu, p);
        const bool lo_ok = cl == 0 || !(b & 1u), hi_ok = ch == nrows || (b & 2u);
        if (lo_ok) lo = cl;
        if (hi_ok) hi = ch;
        if ((lo_ok && hi_ok) || (cl == 0 && ch == nrows)) break;
    }
    // 32-ary narrowing
    for (int round = 0; round < 16 && hi - lo > 32; round++) {
        const long long step = (hi - lo + 31) / 32;
        const long long r = lo + (long long) lane * step;
        const unsigned int b = __ballot_sync(0xffffffffu, r >= hi ? true : pred(r));
        if (b == 0u) { lo = lo + 31 * step + 1; continue; }
        const int f = __ffs((int) b) - 1;
        hi = lo + (long long) f * step < hi ? lo + (long long) f * step : hi;
        if (f > 0) lo = lo + (long long) (f - 1) * step + 1;
    }
    {
        const long long r = lo + lane;
        const unsigned int b = __ballot_sync(0xffffffffu, r >= hi ? true : pred(r));
        return b ? lo + (__ffs((int) b) - 1) : hi;
    }
}
// lower_bound(s) of the key-ordered build = first row whose key maps to sub-table >= s (gx_k_sorted_bounds_search).  The guess:
// the global density, or — better — the previous bound plus one sub-table's worth of rows (a datanode's 1/N pseudo-random
// subset of the keys wanders off the global density by hundreds of rows, but only by a dozen per sub-table)
__device__ __forceinline__ long long sorted_lower_bound(const long long *__restrict__ keys, long long nrows, const gx_slotfn &sf,
                                                        long long s, long long nsub, double rows_per_sub, int lane, long long seed = -1)
{
    if (s <= 0) return 0;
    if (s >= nsub) return nrows;
    const long long g = seed >= 0 ? seed + (long long) rows_per_sub : (long long) ((double) s * rows_per_sub);
    return gx_warp_lower_bound(nrows, g, lane, [&](long long r) { return (long long) (gx_slot_index(__ldg(keys + r), sf) >> GX_SUB_LOG2) >= s; });
}

// the key of a compact or narrow entry in slot i from its tag bits v = (key - kmin) mod 2^mbits: the offset congruent to v
// nearest the interpolation's estimate i keys_per_slot
__device__ __forceinline__ long long gx_tag_key(long long i, unsigned long long v, int mbits, long long kmin, double keys_per_slot)
{
    const long long M = 1LL << mbits, est = (long long) ((double) i * keys_per_slot);
    long long off = (est & ~(M - 1)) | (long long) v;
    if (off - est > M / 2) off -= M;
    else if (est - off > M / 2) off += M;
    return kmin + off;
}

// mbarrier and bulk-async copy (TMA) helpers.  Every wait is bounded: a caller whose wait gives up raises a flag and
// the host redoes the work with a kernel that does not stage through the copy engine, instead of hanging the device.
#define GX_MBAR_SPIN_LIMIT (1u << 22)
__device__ __forceinline__ unsigned int gx_smem_u32(const void *p) { return (unsigned int) __cvta_generic_to_shared(p); }
__device__ __forceinline__ void gx_mbar_init(void *bar, unsigned int count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(gx_smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void gx_mbar_arrive(void *bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(gx_smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void gx_mbar_arrive_expect_tx(void *bar, unsigned int bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(gx_smem_u32(bar)), "r"(bytes) : "memory");
}
// false when the phase did not complete within the poll budget (try_wait itself sleeps in hardware between polls)
__device__ __forceinline__ bool gx_mbar_wait(void *bar, unsigned int parity)
{
    const unsigned int a = gx_smem_u32(bar);
#pragma unroll 1
    for (unsigned int n = 0; n < GX_MBAR_SPIN_LIMIT; n++) {
        unsigned int ok;
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(a), "r"(parity) : "memory");
        if (ok) return true;
    }
    return false;
}
// one bulk-async copy global -> shared (16-byte aligned addresses, size a multiple of 16); completion is counted on `bar`
__device__ __forceinline__ void gx_bulk_g2s(void *dst, const void *src, unsigned int bytes, void *bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(gx_smem_u32(dst)), "l"(src), "r"(bytes), "r"(gx_smem_u32(bar)) : "memory");
}

// Copy K selected rows of one column (row r[j] -> position dst[j]): the K loads are independent and issued together,
// the type is decoded once per column instead of once per row (projection / compaction / scatter kernels).
template <int K>
__device__ __forceinline__ void gx_copy_rows(const gx_dcol &in, void *out, uint8_t *out_nulls, const long long (&r)[K], const long long (&dst)[K], const bool (&keep)[K])
{
    if (in.type == GX_INT4 || in.type == GX_DATE) {
        int v[K];
#pragma unroll
        for (int j = 0; j < K; j++) v[j] = keep[j] ? __ldg((const int *) in.data + r[j]) : 0;
#pragma unroll
        for (int j = 0; j < K; j++) if (keep[j]) ((int *) out)[dst[j]] = v[j];
    } else if (in.type == GX_CHAR) {
        signed char v[K];
#pragma unroll
        for (int j = 0; j < K; j++) v[j] = keep[j] ? __ldg((const signed char *) in.data + r[j]) : 0;
#pragma unroll
        for (int j = 0; j < K; j++) if (keep[j]) ((signed char *) out)[dst[j]] = v[j];
    } else {
        long long v[K];
#pragma unroll
        for (int j = 0; j < K; j++) v[j] = keep[j] ? __ldg((const long long *) in.data + r[j]) : 0;
#pragma unroll
        for (int j = 0; j < K; j++) if (keep[j]) ((long long *) out)[dst[j]] = v[j];
    }
    if (out_nulls) {
#pragma unroll
        for (int j = 0; j < K; j++) if (keep[j]) out_nulls[dst[j]] = in.nulls ? in.nulls[r[j]] : 0;
    }
}

// block-wide exclusive scan of one value per thread (blockDim.x <= 1024)
__device__ __forceinline__ long long gx_block_exscan(long long v, long long *total, long long *smem /* 33 */)
{
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    long long x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { long long y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) smem[wid] = x;
    __syncthreads();
    if (wid == 0) {
        long long w = (lane < (int) ((blockDim.x + 31) >> 5)) ? smem[lane] : 0, z = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { long long y = __shfl_up_sync(0xffffffffu, z, o); if (lane >= o) z += y; }
        smem[lane] = z - w;
        if (lane == 31) smem[32] = z;
    }
    __syncthreads();
    long long res = smem[wid] + x - v;
    *total = smem[32];
    __syncthreads();
    return res;
}
#endif  // __CUDACC__
