/*
 * gpuexec.h — C ABI of libgpuexec.so, the H100-native (sm_90a) replacement for
 * OpenTenBase's per-DataNode SeqScan -> HashJoin -> HashAggregate pipeline and the
 * cross-datanode redistribute step.
 *
 * This is the drop-in boundary (SURVEY.md §8b).  The reference has no FFI for
 * this path: its operators are reached through ExecProcNode()/TupleTableSlot
 * inside the backend.  The CustomScan provider (opentenbase_b200/provider/,
 * plain C, compiled against the reference's own headers) implements the
 * reference's CustomExecMethods (src/include/nodes/extensible.h:120-154) and
 * calls ONLY the functions declared here.  Every entry point cites the
 * reference routine whose work it takes over.
 *
 * Rules of the ABI (they exist because ereport() is siglongjmp,
 * src/include/utils/elog.h:386-398, and a backend is a single-threaded process):
 *   - plain C, POD structs, raw pointers and sizes; no C++ types, no torch types;
 *   - every function returns an int status (GX_OK == 0) and never throws, never
 *     longjmps, never calls back into the host; the message for the last
 *     failure is available from gx_last_error();
 *   - the library owns all device memory; the caller frees handles explicitly
 *     (the provider does so from a ResourceOwner callback);
 *   - there is NO CPU fallback: if no sm_90a-capable device (H100) is present
 *     gx_init() fails and nothing else is callable.
 */
#ifndef GPUEXEC_H
#define GPUEXEC_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GX_ABI_VERSION 1

/* ---- status codes ------------------------------------------------------ */
enum {
    GX_OK            = 0,
    GX_ERR_CUDA      = 1,   /* CUDA runtime/driver failure                  */
    GX_ERR_ARG       = 2,   /* invalid argument / unsupported plan shape    */
    GX_ERR_NOMEM     = 3,   /* HBM or pinned host memory exhausted          */
    GX_ERR_NCCL      = 4,   /* NCCL failure / libnccl missing               */
    GX_ERR_STATE     = 5,   /* call sequence error                          */
    GX_ERR_OVERFLOW  = 6,   /* float8 overflow from finite inputs: reference
                               raises ERROR (CHECKFLOATVAL, float.c:970-981);
                               an infinite input may give an infinite result */
    GX_ERR_NODEVICE  = 7    /* no usable GPU: the path is unavailable       */
};

/* ---- column types (by-value Datums only; pg_type oids in comments) ------ */
enum {
    GX_INT4   = 1,  /* int4   (23)   4 B */
    GX_INT8   = 2,  /* int8   (20)   8 B */
    GX_FLOAT8 = 3,  /* float8 (701)  8 B */
    GX_DATE   = 4,  /* date   (1082) 4 B, days since 2000-01-01 (DateADT)   */
    GX_CHAR   = 5   /* "char" (18)   1 B; also bpchar(1) staged as 1 byte   */
};

/* comparison operators for scan quals (ExecQual, execScan.c:237-330) */
enum { GX_LT = 1, GX_LE = 2, GX_EQ = 3, GX_GE = 4, GX_GT = 5, GX_NE = 6 };

/* aggregate functions: transition/combine/final semantics of
 * include/catalog/pg_aggregate.h:178,188,191,251-252 */
enum {
    GX_AGG_COUNT_STAR = 1, /* int8inc            (utils/adt/int8.c:714)      */
    GX_AGG_COUNT      = 2, /* int8inc_any, skips NULL input                  */
    GX_AGG_SUM_F8     = 3, /* float8pl           (utils/adt/float.c:970)     */
    GX_AGG_AVG_F8     = 4, /* float8_accum/float8_avg (float.c:2823,2991)    */
    GX_AGG_SUM_I4     = 5, /* int4_sum -> int8   (utils/adt/numeric.c:6154)  */
    GX_AGG_MIN_F8     = 6, /* float8smaller                                  */
    GX_AGG_MAX_F8     = 7, /* float8larger                                   */
    GX_AGG_SUM_I8     = 8, /* sum(int8): declined with GX_ERR_ARG, the reference
                              returns numeric (see DESIGN.md §3.2)            */
    GX_AGG_COUNT_DISTINCT = 9, /* count(DISTINCT col): process_ordered_aggregate_single
                              (executor/nodeAgg.c:888) with int8inc_any; see below */
    GX_AGG_VAR_POP_F8     = 10, /* float8_accum/float8_var_pop     (float.c:3010)  */
    GX_AGG_VAR_SAMP_F8    = 11, /* float8_accum/float8_var_samp    (float.c:3032); variance() */
    GX_AGG_STDDEV_POP_F8  = 12, /* float8_accum/float8_stddev_pop  (float.c:3054)  */
    GX_AGG_STDDEV_SAMP_F8 = 13, /* float8_accum/float8_stddev_samp (float.c:3076); stddev() */
    /* SQL:2003 binary aggregates (pg_aggregate.h:304-316): two float8 arguments (Y, X), see below */
    GX_AGG_REGR_COUNT        = 14, /* int8inc_float8_float8 (int8.c:805), bit-cast as GX_AGG_COUNT */
    GX_AGG_REGR_SXX_F8       = 15, /* float8_regr_accum/float8_regr_sxx       (float.c:3386)  */
    GX_AGG_REGR_SYY_F8       = 16, /* float8_regr_accum/float8_regr_syy       (float.c:3407)  */
    GX_AGG_REGR_SXY_F8       = 17, /* float8_regr_accum/float8_regr_sxy       (float.c:3428)  */
    GX_AGG_REGR_AVGX_F8      = 18, /* float8_regr_accum/float8_regr_avgx      (float.c:3449)  */
    GX_AGG_REGR_AVGY_F8      = 19, /* float8_regr_accum/float8_regr_avgy      (float.c:3468)  */
    GX_AGG_REGR_R2_F8        = 20, /* float8_regr_accum/float8_regr_r2        (float.c:3554)  */
    GX_AGG_REGR_SLOPE_F8     = 21, /* float8_regr_accum/float8_regr_slope     (float.c:3587)  */
    GX_AGG_REGR_INTERCEPT_F8 = 22, /* float8_regr_accum/float8_regr_intercept (float.c:3614)  */
    GX_AGG_COVAR_POP_F8      = 23, /* float8_regr_accum/float8_covar_pop      (float.c:3487)  */
    GX_AGG_COVAR_SAMP_F8     = 24, /* float8_regr_accum/float8_covar_samp     (float.c:3506)  */
    GX_AGG_CORR_F8           = 25  /* float8_regr_accum/float8_corr           (float.c:3525)  */
};
/* GX_AGG_COUNT_DISTINCT counts the distinct non-NULL values of one column per group.  Its argument is a single
 * GX_OP_COL over an outer column of type INT4, INT8, DATE or CHAR, compared as int4eq / int8eq / date_eq do
 * (INT64_MIN is an ordinary value).  NULL inputs are skipped, so a group whose inputs are all NULL counts 0.
 * gx_result_fetch returns the count as a bit-cast int64, as for GX_AGG_COUNT.
 * It runs in two steps: the plan is aggregated with the argument appended as one more group column (one record per
 * distinct (group, value) pair, the plan's other aggregates as partial states), then the pairs are folded back into
 * the plan's own groups.  So est_groups of such a plan is read as the estimate of distinct (group, value) pairs, and
 * the float8 overflow rule of gx_result_combine applies to the fold.
 * GX_ERR_ARG, the context staying usable: a FLOAT8 argument (float8_cmp's "all NaNs are equal" is not the group
 * keys' equality), an expression argument, DISTINCT aggregates over two different columns, and a group key that
 * does not fit 16 bytes with the argument packed after it (first fit, GX_MAX_GROUP_COLS columns at most).  Such a
 * result has no partial states: gx_result_fetch_states is GX_ERR_ARG, and so is gx_result_combine with more than
 * one rank (distinct counts do not add across datanodes). */
/* GX_AGG_VAR_POP_F8 .. GX_AGG_STDDEV_SAMP_F8 take the float8 expression argument of GX_AGG_SUM_F8 / GX_AGG_AVG_F8 and
 * skip NULL inputs.  gx_result_fetch returns the finalized float8: NULL when N == 0 (pop) or N <= 1 (samp).  A group
 * with an infinite or NaN input gives NaN (float8_accum makes its Sxx NaN); a finite input whose state overflows is
 * GX_ERR_OVERFLOW.  The device keeps the sum of squared deviations as sums shifted by the group's first value, merged
 * with re-centring (DESIGN.md §3.2), so Sxx matches the exact value within 2^-30 Sxx + 16 N^2 2^-52 D^2, D the largest
 * deviation from the group mean; Sxx is never negative and a constant group gives exactly 0.  gx_result_fetch_states
 * returns {N, Sx} as for GX_AGG_AVG_F8 (never NULL, {0, 0} over zero rows) and gx_result_fetch_sxx the Sxx that
 * completes float8_combine's {N, Sx, Sxx}.  A plan whose state words exceed the library's limit is GX_ERR_ARG, and so
 * is gx_result_combine with more than one rank (a two-phase plan combines the states in the reference's Finalize). */
/* GX_AGG_REGR_COUNT .. GX_AGG_CORR_F8 take two float8 expressions in one gx_expr: the ops before GX_OP_ARG2 are Y,
 * the first SQL argument, the ops after it X (each a program a one-argument aggregate would take; GX_MAX_EXPR_OPS
 * counts both and the separator).  GX_OP_ARG2 in a one-argument aggregate, twice, with an empty side, or missing in
 * a two-argument aggregate is GX_ERR_ARG.  A row whose Y or X is NULL is skipped (the transition function is strict
 * in both); N counts the remaining pairs.  gx_result_fetch returns the final of float.c:3386-3642: NULL when N < 1
 * (N < 2 for covar_samp) and for a vertical line (Sxx == 0: regr_slope, regr_intercept, regr_r2); corr is NULL when
 * Sxx == 0 or Syy == 0, regr_r2 is 1.0 when Syy == 0.  regr_count is never NULL.  As float8_regr_accum does, a
 * non-finite X makes Sxx and Sxy NaN, a non-finite Y makes Syy and Sxy NaN, and Sx, Sy are ordinary sums; a finite
 * input whose state overflows is GX_ERR_OVERFLOW (the rule of the variances above, both arguments' inputs counting).
 * The device keeps {C, S1, S2} shifted sums for X and for Y plus the cross term sum((x - Cx)(y - Cy)), merged with
 * re-centring (DESIGN.md §3.2): Sxx and Syy meet the variance bound, Sxy is within
 * 2^-30 sqrt(Sxx Syy) + 16 N^2 2^-52 Dx Dy, and a constant X (Y) gives Sxx (Syy) exactly 0.
 * The regression aggregates over one (Y, X) pair share one state; a plan with two different pairs is GX_ERR_ARG
 * (two states do not fit the library's state words), and so is a plan whose state words exceed the limit.
 * gx_result_fetch_states returns cnt_out = N (never NULL; val_out = Sx, 0 for regr_count) and gx_result_fetch_regr
 * float8_regr_accum's six-element state.  gx_result_combine with more than one rank is GX_ERR_ARG for such a plan
 * (a two-phase plan combines the states in the reference's Finalize with float8_regr_combine / int8pl). */

/* expression opcodes: tiny postfix VM over float8 (the provider pattern-matches
 * Var/Const/+,-,* trees from the reference's expression tree and declines
 * anything else; execExpr.c is out of scope, SURVEY.md §2 row 14) */
enum {
    GX_OP_COL   = 1,  /* push outer column `col` converted to float8        */
    GX_OP_CONST = 2,  /* push k                                             */
    GX_OP_ADD   = 3,  /* float8pl  */
    GX_OP_SUB   = 4,  /* float8mi  */
    GX_OP_MUL   = 5,  /* float8mul */
    GX_OP_ARG2  = 6   /* two-argument aggregates only: ends Y's program, X's follows */
};

#define GX_MAX_PREDS      4
#define GX_MAX_EXPR_OPS   12
#define GX_MAX_AGGS       8
#define GX_MAX_GROUP_COLS 4
#define GX_MAX_PAYLOAD    2
#define GX_MAX_COLS       16

typedef struct gx_ctx    gx_ctx;     /* one per backend process and device    */
typedef struct gx_table  gx_table;   /* HBM-resident columnar relation        */
typedef struct gx_hash   gx_hash;    /* open-addressing join hash table       */
typedef struct gx_result gx_result;  /* aggregate result (group keys + states)*/

typedef struct gx_pred {
    int32_t col;        /* column number in the scanned table                */
    int32_t op;         /* GX_LT..GX_NE                                      */
    int64_t ival;       /* constant for INT4/INT8/DATE/CHAR columns          */
    double  fval;       /* constant for FLOAT8 columns                       */
} gx_pred;

typedef struct gx_expr_op { int32_t op; int32_t col; double k; } gx_expr_op;
typedef struct gx_expr {
    int32_t    nops;                     /* 0 = no argument (count(*))       */
    int32_t    _pad;
    gx_expr_op ops[GX_MAX_EXPR_OPS];
} gx_expr;

typedef struct gx_agg { int32_t fn; int32_t _pad; gx_expr arg; } gx_agg;

/* a group-by column: side 0 = outer (probe/scanned) table column,
 * side 1 = i-th payload column carried by the join hash table            */
typedef struct gx_colref { int32_t side; int32_t col; } gx_colref;

/* Scan [-> HashJoin probe] -> HashAggregate descriptor: what the provider
 * hands over instead of the reference's Agg/HashJoin/SeqScan plan nodes
 * (nodeAgg.c:3342 ExecInitAgg, nodeHashjoin.c:797 ExecInitHashJoin). */
typedef struct gx_agg_plan {
    int32_t   n_preds;                   /* ANDed quals on the outer scan    */
    int32_t   outer_key_col;             /* join key column; -1 = no join    */
    gx_pred   preds[GX_MAX_PREDS];
    int32_t   n_group_cols;              /* 0 = plain aggregate (one group)  */
    int32_t   n_aggs;
    gx_colref group_cols[GX_MAX_GROUP_COLS];
    gx_agg    aggs[GX_MAX_AGGS];
    int64_t   est_groups;                /* planner's numGroups estimate: picks
                                            shared-memory vs radix strategy  */
    int32_t   strategy;                  /* 0 = auto, 1 = force shared-memory
                                            privatised, 2 = force two-pass radix */
    int32_t   join_type;                 /* GX_JOIN_INNER (0), GX_JOIN_SEMI or
                                            GX_JOIN_ANTI; see below            */
} gx_agg_plan;
/* join_type of an aggregate over a hash join (ExecHashJoinImpl, nodeHashjoin.c:569-634):
 *   INNER  every (outer row, build row) pair with equal keys is one input row of the aggregate;
 *   SEMI   an outer row is consumed once if at least one build row has its key, however many do;
 *   ANTI   the outer rows without a partner are consumed, NULL keys included (HJ_FILL_OUTER_TUPLE).
 * The outer quals (preds) apply before the join, as for INNER; a NULL key has no partner.  SEMI and
 * ANTI carry no inner column: a group column of side 1 is GX_ERR_ARG.  Any other join type (LEFT
 * included) is GX_ERR_ARG, and the context stays usable. */

/* ---- context ------------------------------------------------------------ */
/* Lazily creates the CUDA context (never from postmaster's _PG_init: fork after
 * CUDA init is illegal; the provider calls this from BeginCustomScan). */
int  gx_abi_version(void);
int  gx_init(int device, gx_ctx **out);
void gx_shutdown(gx_ctx *ctx);                /* free every table/hash/result handle first: their
                                               * device memory is returned on the context's stream */
const char *gx_last_error(gx_ctx *ctx);      /* ctx may be NULL: global msg   */
int  gx_device_info(gx_ctx *ctx, int *sm_count, int *cc_major, int *cc_minor,
                    int64_t *hbm_bytes);
int  gx_sync(gx_ctx *ctx);
/* Map `bytes` of HBM into the context's stream-ordered memory pool now (0 = all that is free minus
 * 8 GB), so that per-query temporaries never wait for the driver to create physical memory
 * mid-query.  Call it once per context, after gx_comm_init (NCCL allocates its own buffers). */
int  gx_pool_reserve(gx_ctx *ctx, size_t bytes);

/* kernel launch counter (bench.py's gpu_launches) and CUDA-event timing of the
 * library's own stream (torch.cuda.Event cannot see it) */
int64_t gx_launch_count(gx_ctx *ctx);
int  gx_timer_start(gx_ctx *ctx);
int  gx_timer_stop(gx_ctx *ctx, double *ms_out);
/* per-kernel accumulated CUDA-event time for the named kernel family
 * ("probe_agg", "build", "agg", "partition", ...); enabled by gx_profile(1) */
int  gx_profile(gx_ctx *ctx, int enable);
int  gx_profile_get(gx_ctx *ctx, const char *name, double *ms_total, int64_t *launches);
int  gx_l2_flush(gx_ctx *ctx);              /* writes a >L2-sized buffer      */
/* pinned host memory for the staging buffers the loader DMA-copies from */
int  gx_host_alloc(gx_ctx *ctx, size_t bytes, void **out);
int  gx_host_free(gx_ctx *ctx, void *p);
/* host -> device copy rate (GB/s, best of 3) of `bytes` from `host` over
 * nstreams (1..4) copy streams: the same-run PCIe ceiling bench.py reports */
int  gx_h2d_probe(gx_ctx *ctx, const void *host, size_t bytes, int nstreams, double *gb_per_s);

/* ---- K0: columnar loader ------------------------------------------------
 * Replaces heap_getnext/heapgetpage + slot_deform_tuple + SeqNext
 * (access/heap/heapam.c:388,2198; access/common/heaptuple.c:1518;
 * executor/nodeSeqscan.c:60): only the referenced attributes are staged. */
int  gx_table_create(gx_ctx *ctx, int ncols, const int32_t *types,
                     int64_t capacity_rows, gx_table **out);
/* host_cols[c] points at nrows values of column c (pageable or pinned);
 * host_nulls[c] (may be NULL, as may host_nulls itself) points at nrows bytes,
 * 1 = NULL (the layout of tts_isnull, tuptable.h:199). */
int  gx_table_append_columns(gx_table *t, const void *const *host_cols,
                             const uint8_t *const *host_nulls, int64_t nrows);
/* Raw heap pages (BLCKSZ 8192, layout of storage/bufpage.h:153-175 and
 * access/htup_details.h:126-201) + per-page visible line-pointer lists as
 * produced by heapgetpage() (rs_vistuples/rs_ntuples, access/relscan.h:105).
 * vis_offsets == NULL means "every LP_NORMAL item is visible".  Deform runs
 * on the device. attnums[c] = 0-based attribute number feeding table column c;
 * att_len/att_align describe ALL natts attributes of the relation
 * (attlen: 1,2,4,8 or -1 varlena; attalign: 1,2,4,8). */
typedef struct gx_heap_desc {
    int32_t natts;
    int32_t ncols;
    int16_t att_len[64];
    int8_t  att_align[64];
    int32_t attnums[GX_MAX_COLS];
    int8_t  att_notnull[64];   /* pg_attribute.attnotnull: such a column is staged WITHOUT a NULL array (an
                                * error if a tuple nevertheless lacks the value), which keeps the no-NULL
                                * fast paths of the join and aggregate kernels open for heap-loaded tables */
} gx_heap_desc;
/* With vis_offsets the call only ENQUEUES (copies + the deform kernel; row offsets are
 * scanned on the host from vis_counts) and grows the table if needed; `pages`, if it came
 * from gx_stage_acquire(), may be refilled after the NEXT gx_stage_acquire() returns it. */
int  gx_table_append_heap_pages(gx_table *t, const void *pages, int64_t npages,
                                const gx_heap_desc *desc,
                                const uint16_t *vis_offsets, const int32_t *vis_counts,
                                int32_t vis_stride);
/* ---- forward-node pages: the reference's redistribute wire format --------------------------------
 * What FragmentSendAttrs writes and the forward receiver reads (executor/execFragment.c:2067-2136,
 * forward/fnbufpage.h:54-127, executor/tqueueThread.c:913-925): 8192-byte pages, a 32-byte header
 * (FnPageHeaderData) and MAXALIGNed minimal tuples (heap_form_minimal_tuple_ptr, heaptuple.c:1852).
 * These two calls are what a GPU datanode needs to exchange rows with stock CPU datanodes through their
 * forwarder; between GPU datanodes gx_redistribute() moves columns instead.
 * `desc` describes the tuple (att_len/att_align per attribute; attlen -1 = bpchar(1) carried in a GX_CHAR
 * column).  gx_fnpage_id is what FnPageInit/FragmentGetPage stamp on every page of the stream. */
typedef struct gx_fnpage_id {
    int64_t  qid_timestamp_nodeid, qid_sequence;   /* FNQueryId */
    uint16_t fid, nodeid, workerid;                /* fragment id, source node, source parallel worker */
    uint8_t  virtualid, _pad;                      /* destination virtual datanode */
} gx_fnpage_id;
/* Sender.  Every table column is attribute c of the tuple (desc->natts == ncols, attnums[c] == c).
 * host_pages == NULL: only *npages is computed.  end_marker adds FragmentSendNullTuple's MAX_UINT32 word and
 * FNPAGE_END.  Without NULL arrays the pages equal the reference's byte for byte; with NULLs the rows per page
 * are fixed at the worst-case tuple size (valid pages, not the reference's greedy fill).  Bytes past `lower`
 * are zero. */
int  gx_fnpage_pack(gx_ctx *ctx, const gx_table *t, const gx_heap_desc *desc, const gx_fnpage_id *id, int end_marker,
                    void *host_pages, int64_t cap_pages, int64_t *npages);
/* Receiver: pages of one stream (any fill, NULL bitmaps, short tuples, an end marker) -> a new table with
 * desc->ncols columns of col_types; attributes declared att_notnull get no NULL array.  GX_ERR_ARG for
 * FNPAGE_HUGE pages or a corrupt length chain. */
int  gx_fnpage_unpack(gx_ctx *ctx, const void *host_pages, int64_t npages, const gx_heap_desc *desc,
                      const int32_t *col_types, gx_table **out);

/* End of a load: waits for the enqueued appends; GX_ERR_STATE if a NULL arrived in a column
 * the descriptor declared NOT NULL. */
int  gx_table_load_finish(gx_table *t);
/* Pinned staging for the loader above: one of two library-owned buffers; the call waits
 * until the previous copy out of that buffer has completed.  Filling one buffer while the
 * other one's DMA and deform run is how the provider overlaps heapgetpage() with the GPU. */
int  gx_stage_acquire(gx_ctx *ctx, size_t bytes, void **out);
/* grow a table's capacity (the loader doubles it when a relation holds more rows than estimated) */
int  gx_table_reserve(gx_table *t, int64_t capacity_rows);
int64_t gx_table_nrows(const gx_table *t);
int  gx_table_ncols(const gx_table *t);
int  gx_table_read_column(gx_table *t, int col, int64_t row0, int64_t nrows,
                          void *host_out, uint8_t *host_nulls_out);
int  gx_table_truncate(gx_table *t);         /* keep capacity, nrows = 0      */
/* projection in place: forget column `col` (ExecProject of a narrower target
 * list, execScan.c:237); later columns move down by one */
int  gx_table_drop_column(gx_table *t, int col);
void gx_table_free(gx_table *t);
/* an UNCLUSTERED copy: out[i] = in[(i * A + B) mod n], A coprime to n (bench/test plumbing:
 * the layout the run-folding and key-ordered fast paths must not depend on) */
int  gx_table_permute(gx_ctx *ctx, const gx_table *in, int64_t seed, gx_table **out);
/* raw device pointer of a column (bench/test plumbing; not used by the provider) */
int  gx_table_column_devptr(gx_table *t, int col, void **dptr);

/* Synthetic TPC-H-shaped data generated on the device (SURVEY.md §8d; the same
 * integer recipe as oracle/ generates on the host).  table_id: 1 orders,
 * 2 lineitem, 3 customer.  Rows of orders [order0, order1) (for lineitem: the
 * lines of those orders) are generated at scale factor sf; only rows whose
 * distribution key routes to datanode `node` of `nnodes` under the reference's
 * SHARD rule are kept (nnodes == 1 keeps everything).  colmask selects which
 * columns of the table's fixed schema are materialised. */
int  gx_table_generate(gx_table *t, int table_id, int sf, int64_t order0,
                       int64_t order1, int node, int nnodes);
/* same, for a table holding only some columns of the fixed schema:
 * colmap[c] = schema column number feeding table column c */
int  gx_table_generate_cols(gx_table *t, int table_id, int sf, int64_t order0,
                            int64_t order1, int node, int nnodes, const int32_t *colmap);

/* ---- K1: scan + qual + projection into a new table -----------------------
 * ExecScan qual/projection (executor/execScan.c:237-330) */
int  gx_scan_filter(gx_ctx *ctx, const gx_table *in, int n_preds,
                    const gx_pred *preds, int n_out_cols, const int32_t *out_cols,
                    gx_table **out);

/* ---- K2: hash build ------------------------------------------------------
 * MultiExecPrivateHash + ExecHashTableInsert (executor/nodeHash.c:157,1828).
 * key_col must be INT4/INT8/DATE.  Up to two payload columns totalling <= 8
 * bytes are stored in the slot; n_payload == 0 stores the build row number.
 * NULL keys are dropped (hashStrict, nodeHash.c:2071-2079).  unique = 1 is the
 * planner's inner_unique (nodeHashjoin.c:859-861).
 * Skew limit: linear probing wraps inside 2048-slot sub-tables, and every sub-table
 * keeps at least one free slot so that a probe for a missing key ends.  A build side
 * whose rows cannot be spread that way — one key repeated about 700 to 2047 times
 * or more (the exact count depends on the load factor and on the keys sharing its
 * sub-table), or many distinct keys that collide under the hash — is declined with
 * GX_ERR_ARG, the message giving how many rows hashed into one sub-table.  The table
 * is freed and the context stays usable. */
int  gx_hash_build(gx_ctx *ctx, const gx_table *inner, int key_col,
                   int n_preds, const gx_pred *preds,
                   int n_payload, const int32_t *payload_cols, int unique,
                   gx_hash **out);
int64_t gx_hash_nentries(const gx_hash *h);
int64_t gx_hash_nslots(const gx_hash *h);
/* How the table was built — chosen per build from the data, never from hints:
 * slot_mode 0 = mixing hash; 1 = order-preserving interpolation (near-uniform keys,
 * two-level bucketing build); 2 = the same with the build side found stored in key
 * order and built without any bucketing pass.  avg_chain = average displacement of an
 * entry from its home slot, measured while the table was filled (a build whose chains
 * exceed 4 is redone with the mixing hash before this call returns). */
int  gx_hash_info(const gx_hash *h, int *slot_mode, double *avg_chain);
void gx_hash_free(gx_hash *h);

/* ---- the hash join's bloom filter ------------------------------------------
 * BlockBloomFilterInit / Insert / Find (utils/misc/bloomfilter.c:54,140,162), filled while
 * the join builds (nodeHash.c:717-726) and asked per outer tuple (ExecHashJoinBloomFilter,
 * nodeHashjoin.c:1862).  Bit-identical directory: same sizing (MinLogSpace at 0.05, given up
 * above 2^20 buckets: *out = NULL), same bucket and bit positions, hash = the join's
 * CRC32C "new hash" of the key (hashfunc.c:112-175).  NULL keys and rows failing the
 * build-side quals are not inserted. */
typedef struct gx_bloom gx_bloom;
int  gx_bloom_build(gx_ctx *ctx, const gx_table *inner, int key_col, int n_preds,
                    const gx_pred *preds, gx_bloom **out);
int  gx_bloom_log_num_buckets(const gx_bloom *b);
int  gx_bloom_read_words(gx_bloom *b, uint32_t *host_out /* 8 << log_num_buckets words */);
/* host_pass[i] = 1 when row i's key may have a partner; b == NULL passes every row */
int  gx_bloom_test(gx_ctx *ctx, const gx_bloom *b, const gx_table *outer, int key_col,
                   uint8_t *host_pass);
void gx_bloom_free(gx_bloom *b);

/* ---- K3: probe, materialising the join ----------------------------------
 * ExecHashJoinImpl INNER join (executor/nodeHashjoin.c:446-666) +
 * ExecScanHashBucket (nodeHash.c:2174).  Output columns: out_outer_cols of the
 * outer table followed by the hash table's payload columns. */
int  gx_hash_probe(gx_ctx *ctx, const gx_table *outer, int key_col,
                   int n_preds, const gx_pred *preds, const gx_hash *h,
                   int n_out_outer, const int32_t *out_outer_cols,
                   gx_table **out);
/* Join types of ExecHashJoinImpl beyond INNER (JoinType, nodes/nodes.h): LEFT emits an unmatched
 * outer row with a NULL inner side (HJ_FILL_OUTER_TUPLE, nodeHashjoin.c:668-689; unique build sides
 * only), SEMI emits an outer row once on its first match, ANTI emits the outer rows without a match
 * (nodeHashjoin.c:628-634); SEMI/ANTI output carries no inner columns.  A NULL outer key never
 * matches.  RIGHT/FULL (HJ_FILL_INNER_TUPLES) are declined. */
enum { GX_JOIN_INNER = 0, GX_JOIN_LEFT = 1, GX_JOIN_SEMI = 4, GX_JOIN_ANTI = 5,
       GX_JOIN_SEMI_RIGHT = 8, GX_JOIN_ANTI_RIGHT = 9 };   /* the last two: gx_hash_agg_right only */
int  gx_hash_probe_ex(gx_ctx *ctx, const gx_table *outer, int key_col,
                      int n_preds, const gx_pred *preds, const gx_hash *h, int join_type,
                      int n_out_outer, const int32_t *out_outer_cols, gx_table **out);

/* ---- K3+K4: [probe ->] hash aggregate ------------------------------------
 * agg_fill_hash_table / lookup_hash_entries / advance_aggregates /
 * finalize_aggregates (executor/nodeAgg.c:2609,2149,856,1363).
 * h may be NULL when plan->outer_key_col < 0.  The result holds PARTIAL states
 * (aggsplit INITIAL_SERIAL, planner.c:8743) until gx_result_finalize(). */
int  gx_hash_agg(gx_ctx *ctx, const gx_table *outer, const gx_hash *h,
                 const gx_agg_plan *plan, gx_result **out);

/* Aggregate over a chain of unique INNER hash joins in one probe pass, without an intermediate join
 * (a left-deep HashJoin(HashJoin(outer, d1), d2) ... whose every level has inner_unique, nodeHashjoin.c:859-861).
 * The outer table probes steps[0].h, then steps[1].h, ...; an outer row reaches the aggregate only when every
 * step finds its key, and at most once, since every table was built with unique = 1.
 *   steps[i].key   side 0: outer column key.col; side s (1 <= s <= i): payload column key.col of step s
 *                  (steps are numbered from 1).  The key column is INT4, INT8 or DATE; a payload key widens
 *                  as a column key does (INT4/DATE sign-extended, INT8 whole; INT64_MIN is an ordinary key).
 *                  A payload is never NULL: gx_hash_build declines a nullable payload column.
 *   plan           outer_key_col = -1, join_type = GX_JOIN_INNER; the preds apply to the outer table;
 *                  group_cols[c].side = 0 for an outer column or s (1..n_steps) for payload column col of
 *                  step s; aggregate arguments read outer columns only.
 * The result is an ordinary gx_result.  n_steps == 1 is gx_hash_agg with outer_key_col = steps[0].key.col.
 * Steps 2.. are probed in the 16-byte slot form: a table built compact or narrow gets that form materialised and
 * attached to it (as gx_hash_agg does for the single-join kernels that need it), nslots x 16 bytes of HBM held until
 * gx_hash_free.
 * GX_ERR_ARG, the context staying usable: n_steps outside 1..GX_MAX_JOINS, a NULL or non-unique table, a key
 * of its own or a later step, a key column not INT4/INT8/DATE, a payload index out of range, a group column
 * side past n_steps, plan->outer_key_col >= 0, or a join type other than GX_JOIN_INNER. */
#define GX_MAX_JOINS 3
typedef struct gx_join_step {
    const gx_hash *h;         /* built with unique = 1                                            */
    gx_colref      key;       /* side 0: outer column; side s (1 <= s < this step's number):
                                 payload column key.col of step s                                 */
    int32_t        join_type; /* GX_JOIN_INNER; anything else is GX_ERR_ARG                        */
    int32_t        _pad;
} gx_join_step;
int  gx_hash_agg_joins(gx_ctx *ctx, const gx_table *outer, int n_steps, const gx_join_step *steps,
                       const gx_agg_plan *plan, gx_result **out);

/* Aggregate over a right semi or right anti hash join (JOIN_SEMI_RIGHT / JOIN_ANTI_RIGHT, nodes/nodes.h:897-900): the
 * preserved relation is the BUILD side and the probe side only decides which of its rows survive (the bucket-delete
 * arms of nodeHashjoin.c:580-607; HJ_FILL_INNER for ANTI_RIGHT, nodeHashjoin.c:880-882).
 *   SEMI_RIGHT  a build row that passes the build quals and whose non-NULL key equals the key of at least one probe row
 *               passing probe_preds is consumed once, however many probe rows match it; every build row of a matched
 *               key is consumed.
 *   ANTI_RIGHT  the build rows that pass the build quals and have no such partner, NULL keys included.
 * An empty or fully filtered probe side gives SEMI_RIGHT nothing and ANTI_RIGHT every build row passing the build quals.
 * Keys compare as for the other joins (INT4/DATE widened to int64, INT64_MIN an ordinary key).
 *   h      gx_hash_build(build, key, build quals, n_payload = 0, ...): its payload is the build row number.
 *   plan   an aggregate over build's columns (group columns side 0, arguments, preds), outer_key_col = -1 and
 *          join_type = GX_JOIN_INNER; its preds are ANDed with the build quals.  Every aggregate, group key, NULL,
 *          overflow and partial-state rule of gx_hash_agg applies; the result is an ordinary gx_result.
 * The device marks the matched build rows (one bit per row; a unique table is read in the format its build wrote, a
 * non-unique one walked in its 16-byte form, materialised as gx_hash_agg_joins does), compacts the consumed rows'
 * plan columns in build row order, and aggregates them without a join.
 * GX_ERR_ARG, the context staying usable: a join type other than GX_JOIN_SEMI_RIGHT / GX_JOIN_ANTI_RIGHT, an h with
 * payload columns or not built from this build table at its current row count, a probe key column out of range or not
 * INT4/INT8/DATE, plan->outer_key_col >= 0, plan->join_type != GX_JOIN_INNER, a plan column outside the build table,
 * and whatever gx_hash_agg rejects for the plan.  gx_hash_agg, gx_hash_agg_joins and gx_exec_host reject these join
 * types. */
int  gx_hash_agg_right(gx_ctx *ctx, const gx_table *probe, int probe_key_col, int n_probe_preds, const gx_pred *probe_preds,
                       const gx_table *build, const gx_hash *h, int join_type, const gx_agg_plan *plan, gx_result **out);

/* Combine partial states across datanodes: redistribute groups on the group
 * key, then Finalize HashAggregate (xc_groupby.out:193-205; combine fns
 * int8pl / float8pl / float8_combine).  No-op when no communicator.
 * Afterwards every group is returned by exactly one rank, so the union of the
 * ranks' rows is the answer.  A plain aggregate (no group columns) has its one
 * row on rank 0; gx_result_ngroups is 0 on every other rank. */
int  gx_result_combine(gx_ctx *ctx, gx_result *r);
int64_t gx_result_ngroups(const gx_result *r);
/* Fetch finalized rows (output order unspecified, as in the reference:
 * nodeAgg.c:2879).  key_out[g*n_group_cols + c] holds group column c widened
 * to int64 (float8 keys bit-cast); agg_out[g*n_aggs + a] holds int64 results
 * bit-cast for COUNT/SUM_I4 and float8 otherwise; null_out (may be NULL)
 * [g*(n_group_cols+n_aggs) + i] = 1 for SQL NULL. */
int  gx_result_fetch(gx_result *r, int64_t max_groups, int64_t *key_out,
                     double *agg_out, uint8_t *null_out);
/* Partial (transition) states instead of finalized values, for a two-phase plan whose
 * Finalize Agg runs in the reference above a RemoteSubplan (aggsplit INITIAL_SERIAL,
 * planner.c:8743-8749): per aggregate cnt_out = N, val_out = Sx / min / max (float8) or the
 * int8 sum bit-cast; null_out = 1 while the transition value is NULL. */
int  gx_result_fetch_states(gx_result *r, int64_t max_groups, int64_t *key_out,
                            double *val_out, int64_t *cnt_out, uint8_t *null_out);
/* Sxx of the float8_accum state {N, Sx, Sxx} per group and aggregate, groups in the order of gx_result_fetch_states:
 * sxx_out[g*n_aggs + a] is the group's Sxx for GX_AGG_VAR_* / GX_AGG_STDDEV_* and 0 for any other aggregate. */
int  gx_result_fetch_sxx(gx_result *r, int64_t max_groups, double *sxx_out);
/* float8_regr_accum's state {N, Sx, Sxx, Sy, Syy, Sxy} per group and aggregate, groups in the order of
 * gx_result_fetch_states: out[(g*n_aggs + a)*6 .. +5] for GX_AGG_REGR_SXX_F8 .. GX_AGG_CORR_F8, zeros for any other
 * aggregate (regr_count's partial state is the int8 count of gx_result_fetch_states). */
int  gx_result_fetch_regr(gx_result *r, int64_t max_groups, double *out);
void gx_result_free(gx_result *r);

/* One-call form used by the provider and by bench.py's e2e leg: HOST column
 * buffers in, partial-state result handle out.  The columns are copied in 64 MB
 * chunks over several copy streams, inner table first, so the join-table build
 * overlaps the upload of the outer columns; the probe+aggregate kernel starts
 * when the outer table has landed.  inner_* may be NULL/0 when there is no join. */
typedef struct gx_host_table {
    int32_t ncols;
    int32_t _pad;
    int64_t nrows;
    const int32_t *types;
    const void *const *cols;
    const uint8_t *const *nulls;       /* may be NULL                        */
} gx_host_table;
int  gx_exec_host(gx_ctx *ctx, const gx_host_table *outer,
                  const gx_host_table *inner, int inner_key_col,
                  int n_inner_preds, const gx_pred *inner_preds,
                  int n_payload, const int32_t *payload_cols, int inner_unique,
                  const gx_agg_plan *plan, gx_result **out);

/* ---- K5: redistribute ----------------------------------------------------
 * GetDataRouting/EvaluateHashkey/GetNodeIndexByHashValue + FragmentSendTuple +
 * FN sender/receiver (executor/execFragment.c:2360,2515; pgxc/locator/
 * locator.c:1611; pgxc/shard/shardmap.c:1147; src/backend/forward/).
 * One datanode per GPU; NCCL all-to-all over NVLink. */
#define GX_SHARD_MAP_SHARD_NUM 4096     /* include/pgxc/shardmap.h:20-21      */
#define GX_NCCL_UID_BYTES 128
int  gx_comm_unique_id(void *uid_out /* GX_NCCL_UID_BYTES */);
int  gx_comm_init(gx_ctx *ctx, int rank, int nranks, const void *uid);
int  gx_comm_rank(const gx_ctx *ctx, int *rank, int *nranks);
void gx_comm_destroy(gx_ctx *ctx);
/* shardmap[i] = node index owning shard i; NULL installs the default map
 * shard i -> i % nnodes (catalog/pgxc_shard_map.c:93). */
int  gx_set_shardmap(gx_ctx *ctx, const int32_t *shardmap /* 4096 */, int nnodes);
/* dest_out[i] = datanode of row i under the SHARD rule (bit-exact with the
 * reference: Jenkins hashint4/hashint8, abs((int)h) % 4096, shardmap). */
int  gx_route(gx_ctx *ctx, const gx_table *in, int key_col, int32_t *host_dest_out);
/* Partition `in` by destination and exchange; *out receives this node's rows.
 * Without a communicator (single node) it degenerates to a local copy. */
int  gx_redistribute(gx_ctx *ctx, const gx_table *in, int key_col, gx_table **out);
/* Local half only (tests / profiling): rows grouped by destination, with
 * per-destination counts; out table has the same schema. */
int  gx_partition_by_node(gx_ctx *ctx, const gx_table *in, int key_col,
                          gx_table **out, int64_t *host_counts /* nnodes */);

/* ---- device-side hash primitives exposed for parity tests ---------------- */
/* which: 1 hashint4 (Jenkins), 2 hashint8 (Jenkins), 3 hashint4new (CRC32C),
 * 4 hashint8new (CRC32C), 5 murmurhash32(uint32 of low half) */
int  gx_debug_hash(gx_ctx *ctx, int which, const int64_t *host_in, int64_t n,
                   uint32_t *host_out);
/* gx_result_combine without a communicator, for tests on one GPU: parts[0..nparts-1] are the partial results of
 * nparts datanodes (same plan).  parts[rank] is combined in place exactly as gx_result_combine combines it on rank
 * `rank` of nparts ranks whose ranks hold those parts; the other parts are only read.  nparts 1..GX_MAX_NODES.
 * GX_ERR_ARG, the context staying usable: the plans or record layouts of the parts differ, a part was combined
 * already, or rank is out of range. */
int  gx_debug_combine(gx_ctx *ctx, int nparts, gx_result *const *parts, int rank);
/* gx_redistribute of rank `rank` of nparts, on one GPU: parts[p] is the input table of datanode p (same column
 * count and types).  window_bytes > 0 runs the peer-window path with windows of that size per rank, 0 the NCCL
 * path.  The context's shard map must cover nparts nodes.  *out receives the rows rank `rank` would receive;
 * *path_out (may be NULL) = 0 peer windows, 1 NCCL path with one-pass regions, 2 NCCL path with the two-pass
 * partition (this rank's own part).  GX_ERR_ARG, the context staying usable: nparts outside 1..GX_MAX_NODES,
 * rank out of range, parts whose column count or types differ, a key column out of range or not INT4/INT8/DATE,
 * a shard map for another node count, window_bytes * nparts above 4 GiB. */
int  gx_debug_redistribute(gx_ctx *ctx, int nparts, const gx_table *const *parts, int key_col, int rank,
                           size_t window_bytes, gx_table **out, int *path_out);

#ifdef __cplusplus
}
#endif
#endif /* GPUEXEC_H */
