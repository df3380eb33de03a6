/*
 * gpuexec_provider.c — OpenTenBase CustomScan provider for libgpuexec.so.
 *
 * The host side of the drop-in boundary (SURVEY.md §8b), in the reference's own
 * language (C) against the reference's own headers.  It plugs the H100 path in
 * where the planner would otherwise put
 *
 *      HashAggregate <- [Hash Join <- Seq Scan, Hash <- Seq Scan]
 *
 * on a datanode: create_upper_paths_hook (optimizer/planner.h:52-56) offers a
 * CustomPath for UPPERREL_GROUP_AGG; the CustomScan is shipped to the datanodes
 * by name (_outCustomScan / _readCustomScan, nodes/outfuncs.c:1288,
 * readfuncs.c:3473) — so this library must be in shared_preload_libraries on
 * the CN and on every DN; the executor methods below stage the relations'
 * visible tuples into HBM page by page (heapgetpage, access/heapam.h:126, one
 * visibility pass per 8 KB page — MVCC/GTS stays on the host) and hand the rest
 * to libgpuexec.so through the C ABI of include/gpuexec.h.  Nothing here throws
 * across the boundary: every gx_* status is turned into ereport(ERROR) on this
 * side, and every handle is released from a ResourceOwner callback because
 * ereport is siglongjmp (utils/elog.h:386-398).
 *
 * Build: against an OpenTenBase install (pg_config --includedir-server), or in
 * this repository against /root/reference/src/include with the stub
 * pg_config.h of oracle/ref (compile check only; `make -C opentenbase_b200/provider`).
 *
 * Status: the executor side (Begin/Exec/End/ReScan/Explain), the plan
 * (de)serialisation into custom_private and the heap-page loader are complete
 * and are EXECUTED by provider/harness (a stub-linked fake backend: fake EState,
 * heapgetpage() fed from heap-page images, real libgpuexec.so; see
 * tests/test_provider_harness.py).  The planner hook recognises the plan shapes
 * listed above gpuexec_match_plan, with the aggregates of gpuexec_aggs, and offers
 *   - the whole aggregation pushed down when the GROUP BY covers the input's
 *     distribution key (grouping_distribution_match, planner.c:8588-8668), or
 *   - PARTIAL states (AGGSPLIT_INITIAL_SERIAL) under the reference's own
 *     redistribute + Finalize Agg (create_redistribute_grouping_path,
 *     pathnode.c:6091; planner.c:9045-9075) otherwise.
 * The planner side compiles against the reference headers but has never run
 * inside a live backend (none can be built here: SURVEY.md §8c).
 */
#include "postgres.h"

#include "access/heapam.h"
#include "access/htup_details.h"
#include "access/relscan.h"
#include "audit/audit_fga.h"
#include "catalog/pg_type.h"
#include "commands/explain.h"
#include "executor/executor.h"
#include "fmgr.h"
#include "miscadmin.h"
#include "nodes/extensible.h"
#include "nodes/makefuncs.h"
#include "nodes/nodeFuncs.h"
#include "optimizer/clauses.h"
#include "optimizer/cost.h"
#include "optimizer/distribution.h"
#include "optimizer/pathnode.h"
#include "optimizer/paths.h"
#include "optimizer/planner.h"
#include "optimizer/tlist.h"
#include "parser/parsetree.h"
#include "pgxc/locator.h"
#include "utils/array.h"
#include "utils/builtins.h"
#include "utils/cls.h"
#include "utils/datamask.h"
#include "utils/fmgroids.h"
#include "utils/mls.h"
#include "storage/bufmgr.h"
#include "utils/guc.h"
#include "utils/memutils.h"
#include "utils/rel.h"
#include "utils/selfuncs.h"
#include "utils/resowner.h"
#include "utils/snapmgr.h"
#include "utils/syscache.h"

#include "gpuexec.h"
#include "gpuexec_cost.h"

PG_MODULE_MAGIC;

void		_PG_init(void);

static bool gpuexec_enabled = true;
static int	gpuexec_device = 0;
static int	gpuexec_pool_reserve_mb = 0;	/* HBM mapped into the library's pool when the backend's context is created */
static int	gpuexec_hbm_limit_mb = 64 * 1024;	/* decline plans whose staged columns + join table would not fit (80 GB H100) */
/* the cost model's rates (gpuexec_cost.h) */
static double gpuexec_cost_unit_us = 10.0;
static double gpuexec_host_page_us = 1.5;
static double gpuexec_pcie_gb_s = 50.0;
static double gpuexec_hbm_gb_s = 3000.0;
static double gpuexec_startup_us = 1500.0;
static create_upper_paths_hook_type prev_upper_paths_hook = NULL;

/* one CUDA context per backend process, created lazily (never in the postmaster:
 * fork after CUDA initialisation is illegal) */
static gx_ctx *backend_ctx = NULL;

#define GPUEXEC_NAME "GpuExecHashAgg"

/* ---------------------------------------------------------------- state */
typedef struct GpuRelInfo
{
	Index		rti;			/* range-table index of the scanned relation */
	int			ncols;			/* referenced attributes */
	int			attnums[GX_MAX_COLS];	/* 0-based attribute numbers */
	int32		types[GX_MAX_COLS];		/* GX_* */
} GpuRelInfo;

/* one hash join of the plan: step s (1..) of a left-deep chain builds its table over rel and probes it with the rows that
 * passed steps 1 .. s-1 */
typedef struct GpuJoinStep
{
	GpuRelInfo	rel;
	int			key_col;		/* build key column of rel */
	int			n_payload;
	int32		payload_cols[GX_MAX_PAYLOAD];
	bool		unique;			/* the build keys are unique (inner_unique) */
	int			n_preds;
	gx_pred		preds[GX_MAX_PREDS];
	gx_colref	probe;			/* steps 2..: probe key, side 0 an outer column, side s a payload column of step s;
								 * step 1 probes with plan.outer_key_col */
	double		tuples;			/* planner only (HBM estimate), not shipped */
	Relation	r;
	gx_table   *tab;
	gx_hash    *hash;
} GpuJoinStep;

/* the descriptor word after the version for a join chain: 0 is no join, 1 + GX_JOIN_* a single join */
#define GPUEXEC_DESC_CHAIN 100

/* a right semi / right anti join: the outer slot holds the hashed (preserved) relation, join[0] the probing one */
static inline bool
is_right_join(int jt)
{
	return jt == GX_JOIN_SEMI_RIGHT || jt == GX_JOIN_ANTI_RIGHT;
}

typedef struct GpuExecState
{
	CustomScanState css;
	/* decoded from custom_private */
	GpuRelInfo	outer;
	int			n_joins;		/* 0 no join, 1 a join of plan.join_type, 2.. a chain of unique INNER joins */
	GpuJoinStep join[GX_MAX_JOINS];
	bool		partial;		/* emit transition states (AGGSPLIT_INITIAL_SERIAL), not final values */
	gx_agg_plan plan;
	/* run time */
	Relation	outer_rel;
	gx_table   *outer_tab;
	gx_result  *result;
	int64		ngroups,
				next;
	int64	   *keys;
	double	   *aggs;
	int64	   *cnts;			/* partial mode: N of every transition state */
	double	   *sxx;			/* partial mode: Sxx of every variance state */
	double	   *regr;			/* partial mode: float8_regr_accum's six values of every regression state */
	uint8	   *nulls;
	double		load_ms,
				exec_ms;
	bool		done_exec;
} GpuExecState;

/* handles that must die with the query even when ereport() longjmps past us */
typedef struct GpuHandles
{
	struct GpuHandles *next;
	ResourceOwner owner;
	GpuExecState *state;
} GpuHandles;
static GpuHandles *live_handles = NULL;

static void
gpuexec_release_state(GpuExecState *st)
{
	if (st->result)
		gx_result_free(st->result);
	if (st->outer_tab)
		gx_table_free(st->outer_tab);
	st->result = NULL;
	st->outer_tab = NULL;
	for (int i = 0; i < st->n_joins; i++)
	{
		if (st->join[i].hash)
			gx_hash_free(st->join[i].hash);
		if (st->join[i].tab)
			gx_table_free(st->join[i].tab);
		st->join[i].hash = NULL;
		st->join[i].tab = NULL;
	}
}

static void
gpuexec_resowner_callback(ResourceReleasePhase phase, bool isCommit, bool isTopLevel, void *arg)
{
	GpuHandles **p = &live_handles;

	if (phase != RESOURCE_RELEASE_AFTER_LOCKS)
		return;
	while (*p)
	{
		GpuHandles *h = *p;

		if (h->owner == CurrentResourceOwner)
		{
			gpuexec_release_state(h->state);
			*p = h->next;
			free(h);
		}
		else
			p = &h->next;
	}
}

#define GX_CHECK(call) \
	do { \
		int			gx_status__ = (call); \
		if (gx_status__ != GX_OK) \
			ereport(ERROR, \
					(errcode(gx_status__ == GX_ERR_OVERFLOW ? ERRCODE_NUMERIC_VALUE_OUT_OF_RANGE : ERRCODE_EXTERNAL_ROUTINE_EXCEPTION), \
					 errmsg("gpuexec: %s", gx_last_error(backend_ctx)))); \
	} while (0)

static void
gpuexec_ensure_context(void)
{
	if (backend_ctx == NULL)
	{
		int			st = gx_init(gpuexec_device, &backend_ctx);

		if (st != GX_OK)
			ereport(ERROR,
					(errcode(ERRCODE_EXTERNAL_ROUTINE_EXCEPTION),
					 errmsg("gpuexec: %s", gx_last_error(NULL))));
		/* several backends share one GPU: each reserves only what the DBA grants it */
		if (gpuexec_pool_reserve_mb > 0)
			GX_CHECK(gx_pool_reserve(backend_ctx, (size_t) gpuexec_pool_reserve_mb << 20));
	}
}

/* --------------------------------------------------- type / expr mapping */
static int32
gpuexec_type_of(Oid typid)
{
	switch (typid)
	{
		case INT4OID:
			return GX_INT4;
		case INT8OID:
			return GX_INT8;
		case FLOAT8OID:
			return GX_FLOAT8;
		case DATEOID:
			return GX_DATE;
		case CHAROID:
			return GX_CHAR;
		case BPCHAROID:
			return GX_CHAR;		/* bpchar(1) only: checked by the planner hook */
		default:
			return 0;
	}
}

/* ------------------------------------------------------------ aggregates */
/* the argument an aggregate takes */
typedef enum
{
	AGG_ARG_NONE,				/* count(*) */
	AGG_ARG_COLUMN,				/* one column (or float8 constant), a program of one op */
	AGG_ARG_F8,					/* one float8 expression */
	AGG_ARG_F8_PAIR				/* (Y, X): Y's program, GX_OP_ARG2, X's program */
} GpuAggArg;

/* the transition value a partial (AGGSPLIT_INITIAL_SERIAL) aggregate emits: what the reference's combine function
 * expects (pg_aggregate.h:178-316) */
typedef enum
{
	PARTIAL_VALUE,				/* the final value: float8 for sum/min/max(float8), int8 for sum(int4) */
	PARTIAL_COUNT,				/* int8 N (int8pl) */
	PARTIAL_AVG,				/* float8[3] {N, Sx, 0}: only var/stddev read Sxx; float8_combine (float.c:2725) keeps it finite */
	PARTIAL_VAR,				/* float8_accum's float8[3] {N, Sx, Sxx}, Sxx from gx_result_fetch_sxx */
	PARTIAL_REGR				/* float8[6] {N, Sx, Sxx, Sy, Syy, Sxy} (float8_regr_combine, float.c:3244), gx_result_fetch_regr */
} GpuAggPartial;

typedef struct GpuAggDef
{
	Oid			aggfnoid;		/* pg_aggregate.aggfnoid */
	int			fn;				/* GX_AGG_* */
	GpuAggArg	arg;
	GpuAggPartial partial;
} GpuAggDef;

/* Every aggregate the planner hook pushes down; an Aggref of any other aggfnoid declines the plan.  count(DISTINCT x) is
 * count(any)'s row under stricter rules (GX_AGG_COUNT_DISTINCT, match_aggregates). */
static const GpuAggDef gpuexec_aggs[] = {
	{2803, GX_AGG_COUNT_STAR, AGG_ARG_NONE, PARTIAL_COUNT},			/* count(*) */
	{2147, GX_AGG_COUNT, AGG_ARG_COLUMN, PARTIAL_COUNT},			/* count(any) */
	{2108, GX_AGG_SUM_I4, AGG_ARG_COLUMN, PARTIAL_VALUE},			/* sum(int4) */
	{2111, GX_AGG_SUM_F8, AGG_ARG_F8, PARTIAL_VALUE},				/* sum(float8) */
	{2105, GX_AGG_AVG_F8, AGG_ARG_F8, PARTIAL_AVG},					/* avg(float8) */
	{2136, GX_AGG_MIN_F8, AGG_ARG_F8, PARTIAL_VALUE},				/* min(float8) */
	{2120, GX_AGG_MAX_F8, AGG_ARG_F8, PARTIAL_VALUE},				/* max(float8) */
	{2722, GX_AGG_VAR_POP_F8, AGG_ARG_F8, PARTIAL_VAR},				/* var_pop(float8) */
	{2645, GX_AGG_VAR_SAMP_F8, AGG_ARG_F8, PARTIAL_VAR},			/* var_samp(float8) */
	{2152, GX_AGG_VAR_SAMP_F8, AGG_ARG_F8, PARTIAL_VAR},			/* variance(float8) */
	{2728, GX_AGG_STDDEV_POP_F8, AGG_ARG_F8, PARTIAL_VAR},			/* stddev_pop(float8) */
	{2716, GX_AGG_STDDEV_SAMP_F8, AGG_ARG_F8, PARTIAL_VAR},			/* stddev_samp(float8) */
	{2158, GX_AGG_STDDEV_SAMP_F8, AGG_ARG_F8, PARTIAL_VAR},			/* stddev(float8) */
	{2818, GX_AGG_REGR_COUNT, AGG_ARG_F8_PAIR, PARTIAL_COUNT},		/* regr_count(float8, float8) */
	{2819, GX_AGG_REGR_SXX_F8, AGG_ARG_F8_PAIR, PARTIAL_REGR},		/* regr_sxx */
	{2820, GX_AGG_REGR_SYY_F8, AGG_ARG_F8_PAIR, PARTIAL_REGR},		/* regr_syy */
	{2821, GX_AGG_REGR_SXY_F8, AGG_ARG_F8_PAIR, PARTIAL_REGR},		/* regr_sxy */
	{2822, GX_AGG_REGR_AVGX_F8, AGG_ARG_F8_PAIR, PARTIAL_REGR},		/* regr_avgx */
	{2823, GX_AGG_REGR_AVGY_F8, AGG_ARG_F8_PAIR, PARTIAL_REGR},		/* regr_avgy */
	{2824, GX_AGG_REGR_R2_F8, AGG_ARG_F8_PAIR, PARTIAL_REGR},		/* regr_r2 */
	{2825, GX_AGG_REGR_SLOPE_F8, AGG_ARG_F8_PAIR, PARTIAL_REGR},	/* regr_slope */
	{2826, GX_AGG_REGR_INTERCEPT_F8, AGG_ARG_F8_PAIR, PARTIAL_REGR},	/* regr_intercept */
	{2827, GX_AGG_COVAR_POP_F8, AGG_ARG_F8_PAIR, PARTIAL_REGR},		/* covar_pop */
	{2828, GX_AGG_COVAR_SAMP_F8, AGG_ARG_F8_PAIR, PARTIAL_REGR},	/* covar_samp */
	{2829, GX_AGG_CORR_F8, AGG_ARG_F8_PAIR, PARTIAL_REGR},			/* corr */
};

static const GpuAggDef *
agg_by_oid(Oid aggfnoid)
{
	for (int i = 0; i < (int) lengthof(gpuexec_aggs); i++)
		if (gpuexec_aggs[i].aggfnoid == aggfnoid)
			return &gpuexec_aggs[i];
	return NULL;
}

/* the row of a descriptor's aggregate, which carries no OID (an alias has its function's row); NULL for count(DISTINCT) */
static const GpuAggDef *
agg_by_fn(int fn)
{
	for (int i = 0; i < (int) lengthof(gpuexec_aggs); i++)
		if (gpuexec_aggs[i].fn == fn)
			return &gpuexec_aggs[i];
	return NULL;
}

/* ------------------------------------------------ K0: heap page loader
 * One heapgetpage() per block (pins the buffer, runs HeapTupleSatisfiesMVCC once
 * per tuple, fills rs_vistuples[]); the raw page bytes and the visible line
 * pointers go to the device in batches, the deform runs there.  A batch lives in
 * one slot of the library's pinned staging ring (gx_stage_acquire): while the DMA
 * and the deform of batch i run, the host fills batch i+1 — the append call only
 * enqueues.  The ring belongs to the library, so an ereport() out of
 * heapgetpage() leaks nothing. */
#define LOAD_BATCH_PAGES 4096	/* 32 MB of pages per gx_table_append_heap_pages() */

static void
gpuexec_load_relation(Relation rel, EState *estate, GpuRelInfo *info, gx_table **out)
{
	TupleDesc	desc = RelationGetDescr(rel);
	HeapScanDesc scan = heap_beginscan(rel, estate->es_snapshot, 0, NULL);
	BlockNumber nblocks = scan->rs_nblocks;
	gx_heap_desc hd;
	const size_t pages_bytes = (size_t) LOAD_BATCH_PAGES * BLCKSZ;
	const size_t vis_bytes = sizeof(uint16) * (size_t) LOAD_BATCH_PAGES * MaxHeapTuplesPerPage;
	const size_t slot_bytes = pages_bytes + vis_bytes + sizeof(int32) * LOAD_BATCH_PAGES;
	char	   *slot = NULL;
	char	   *pages = NULL;
	uint16	   *vis = NULL;
	int32	   *cnt = NULL;
	double		reltuples = rel->rd_rel ? rel->rd_rel->reltuples : 0;
	int64		est_rows;
	BlockNumber blk;
	int			nbatch = 0;
	int			i;

	memset(&hd, 0, sizeof(hd));
	hd.natts = desc->natts;
	hd.ncols = info->ncols;
	if (desc->natts > 64)
		ereport(ERROR, (errmsg("gpuexec: relation has more than 64 attributes")));
	for (i = 0; i < desc->natts; i++)
	{
		Form_pg_attribute att = TupleDescAttr(desc, i);

		hd.att_len[i] = att->attlen;
		hd.att_align[i] = att->attalign == 'd' ? 8 : att->attalign == 'i' ? 4 : att->attalign == 's' ? 2 : 1;
		hd.att_notnull[i] = att->attnotnull ? 1 : 0;	/* no NULL array: the kernels' no-NULL fast paths stay open */
	}
	for (i = 0; i < info->ncols; i++)
	{
		hd.attnums[i] = info->attnums[i];
		/* the device deform reads attributes a tuple was written without as NULL; a
		 * fast default (atthasmissing, heaptuple.c:109-135) would need the value */
		if (TupleDescAttr(desc, info->attnums[i])->atthasmissing)
			ereport(ERROR, (errcode(ERRCODE_FEATURE_NOT_SUPPORTED),
							errmsg("gpuexec: column \"%s\" has a missing-value default", NameStr(TupleDescAttr(desc, info->attnums[i])->attname))));
	}

	/* sized from the statistics, never from MaxHeapTuplesPerPage (291 rows per page would be
	 * five to six times the real count); the table grows when the estimate was low */
	est_rows = (int64) (reltuples * 1.1) + 1024;
	if (est_rows < (int64) nblocks * 8)
		est_rows = (int64) nblocks * 8;
	GX_CHECK(gx_table_create(backend_ctx, info->ncols, info->types, est_rows, out));

	for (blk = 0; blk < nblocks; blk++)
	{
		CHECK_FOR_INTERRUPTS();
		if (nbatch == 0)
		{
			GX_CHECK(gx_stage_acquire(backend_ctx, slot_bytes, (void **) &slot));
			pages = slot;
			vis = (uint16 *) (slot + pages_bytes);
			cnt = (int32 *) (slot + pages_bytes + vis_bytes);
		}
		heapgetpage(scan, blk);
		LockBuffer(scan->rs_cbuf, BUFFER_LOCK_SHARE);
		memcpy(pages + (size_t) nbatch * BLCKSZ, BufferGetPage(scan->rs_cbuf), BLCKSZ);
		LockBuffer(scan->rs_cbuf, BUFFER_LOCK_UNLOCK);
		cnt[nbatch] = scan->rs_ntuples;
		memcpy(vis + (size_t) nbatch * MaxHeapTuplesPerPage, scan->rs_vistuples, sizeof(uint16) * scan->rs_ntuples);
		if (++nbatch == LOAD_BATCH_PAGES || blk + 1 == nblocks)
		{
			int			st = gx_table_append_heap_pages(*out, pages, nbatch, &hd, vis, cnt, MaxHeapTuplesPerPage);

			if (st != GX_OK)
			{
				heap_endscan(scan);
				GX_CHECK(st);
			}
			nbatch = 0;
		}
	}
	heap_endscan(scan);
	GX_CHECK(gx_table_load_finish(*out));
}

/* ------------------------------------------- custom_private (de)serialisation
 * A flat list of Integer / Float Value nodes — the only thing nodeToString()
 * is guaranteed to carry to the datanodes (nodes/outfuncs.c:1288-1310). */
static List *
put_int(List *l, int64 v)
{
	Assert(v == (int64) (int32) v);		/* small enumerations and column numbers only */
	return lappend(l, makeInteger((long) v));
}

/* 64-bit integers travel as decimal strings: nodeRead() turns any integer token that does
 * not fit int32 into a T_Float node anyway (nodes/read.c), and a double would round above 2^53 */
static List *
put_int64(List *l, int64 v)
{
	char		buf[32];

	snprintf(buf, sizeof(buf), INT64_FORMAT, v);
	return lappend(l, makeFloat(pstrdup(buf)));
}
/* ... and the other way round: a value that does fit int32 ("10") comes back from nodeRead() as a T_Integer node, whatever
 * node type it was sent as, so the reader takes both (tests/test_provider_ship_cpu.py runs the reference's read.c over it) */
static int64
get_int64(ListCell **lc)
{
	Value	   *n = (Value *) lfirst(*lc);
	int64		v = IsA(n, Integer) ? (int64) intVal(n) : (int64) strtoll(strVal(n), NULL, 10);

	*lc = lnext(*lc);
	return v;
}
/* doubles travel as their bit pattern (a decimal int64 string like the integers above): "%.17g" round-trips finite values, but
 * NaN and the infinities print as "nan" / "inf", which nodeRead() (nodes/read.c:nodeTokenType) does not take for a number —
 * a qual such as  x < 'Infinity'  would make every datanode fail to read the plan */
static List *
put_double(List *l, double v)
{
	int64		bits;

	memcpy(&bits, &v, sizeof(bits));
	return put_int64(l, bits);
}
static int
get_int(ListCell **lc)
{
	int			v = intVal(lfirst(*lc));

	*lc = lnext(*lc);
	return v;
}
static double
get_double(ListCell **lc)
{
	int64		bits = get_int64(lc);
	double		v;

	memcpy(&v, &bits, sizeof(v));
	return v;
}

static List *
serialise_rel(List *l, const GpuRelInfo *r)
{
	int			i;

	l = put_int(l, r->rti);
	l = put_int(l, r->ncols);
	for (i = 0; i < r->ncols; i++)
	{
		l = put_int(l, r->attnums[i]);
		l = put_int(l, r->types[i]);
	}
	return l;
}
static void
deserialise_rel(ListCell **lc, GpuRelInfo *r)
{
	int			i;

	r->rti = get_int(lc);
	r->ncols = get_int(lc);
	for (i = 0; i < r->ncols; i++)
	{
		r->attnums[i] = get_int(lc);
		r->types[i] = get_int(lc);
	}
}

/* n quals of four words each: column, operator, integer and float8 constant (their count travels ahead of them) */
static List *
put_preds(List *l, int n, const gx_pred *preds)
{
	int			i;

	for (i = 0; i < n; i++)
	{
		l = put_int(l, preds[i].col);
		l = put_int(l, preds[i].op);
		l = put_int64(l, preds[i].ival);
		l = put_double(l, preds[i].fval);
	}
	return l;
}
static void
get_preds(ListCell **lc, int n, gx_pred *preds)
{
	int			i;

	for (i = 0; i < n; i++)
	{
		preds[i].col = get_int(lc);
		preds[i].op = get_int(lc);
		preds[i].ival = get_int64(lc);
		preds[i].fval = get_double(lc);
	}
}

/* one join step's block: rel, key column, [step 2..: probe side and column,] payload, [step 1: unique,] quals */
static List *
serialise_step(List *l, const GpuJoinStep *j, bool first)
{
	int			i;

	l = serialise_rel(l, &j->rel);
	l = put_int(l, j->key_col);
	if (!first)
	{
		l = put_int(l, j->probe.side);
		l = put_int(l, j->probe.col);
	}
	l = put_int(l, j->n_payload);
	for (i = 0; i < j->n_payload; i++)
		l = put_int(l, j->payload_cols[i]);
	if (first)
		l = put_int(l, j->unique);
	l = put_int(l, j->n_preds);
	return put_preds(l, j->n_preds, j->preds);
}
static void
deserialise_step(ListCell **lc, GpuJoinStep *j, bool first)
{
	int			i;

	deserialise_rel(lc, &j->rel);
	j->key_col = get_int(lc);
	if (!first)
	{
		j->probe.side = get_int(lc);
		j->probe.col = get_int(lc);
	}
	j->n_payload = get_int(lc);
	for (i = 0; i < j->n_payload; i++)
		j->payload_cols[i] = get_int(lc);
	j->unique = first ? get_int(lc) != 0 : true;	/* every step of a chain is unique */
	j->n_preds = get_int(lc);
	get_preds(lc, j->n_preds, j->preds);
}

static List *
gpuexec_serialise(const GpuExecState *st)
{
	List	   *l = NIL;
	const gx_agg_plan *p = &st->plan;
	int			i,
				j;

	l = put_int(l, GX_ABI_VERSION);
	/* 0 = no join, 1 + GX_JOIN_* one join (an INNER join keeps the word it had before SEMI and ANTI existed), or the chain
	 * word; a chain's count of further steps and their blocks follow step 1's block */
	l = put_int(l, st->n_joins == 0 ? 0 : st->n_joins == 1 ? 1 + p->join_type : GPUEXEC_DESC_CHAIN);
	l = serialise_rel(l, &st->outer);
	for (j = 0; j < st->n_joins; j++)
	{
		if (j == 1)
			l = put_int(l, st->n_joins - 1);
		l = serialise_step(l, &st->join[j], j == 0);
	}
	l = put_int(l, st->partial);
	l = put_int(l, p->n_preds);
	l = put_int(l, p->outer_key_col);
	l = put_preds(l, p->n_preds, p->preds);
	l = put_int(l, p->n_group_cols);
	for (i = 0; i < p->n_group_cols; i++)
	{
		l = put_int(l, p->group_cols[i].side);
		l = put_int(l, p->group_cols[i].col);
	}
	l = put_int(l, p->n_aggs);
	for (i = 0; i < p->n_aggs; i++)
	{
		l = put_int(l, p->aggs[i].fn);
		l = put_int(l, p->aggs[i].arg.nops);
		for (j = 0; j < p->aggs[i].arg.nops; j++)
		{
			l = put_int(l, p->aggs[i].arg.ops[j].op);
			l = put_int(l, p->aggs[i].arg.ops[j].col);
			l = put_double(l, p->aggs[i].arg.ops[j].k);
		}
	}
	l = put_int64(l, p->est_groups);
	return l;
}

static void
gpuexec_deserialise(List *priv, GpuExecState *st)
{
	ListCell   *lc = list_head(priv);
	gx_agg_plan *p = &st->plan;
	int			i,
				j;

	if (get_int(&lc) != GX_ABI_VERSION)
		ereport(ERROR, (errmsg("gpuexec: coordinator and datanode run different provider versions")));
	memset(p, 0, sizeof(*p));
	i = get_int(&lc);
	p->join_type = i != 0 && i != GPUEXEC_DESC_CHAIN ? i - 1 : GX_JOIN_INNER;
	st->n_joins = i != 0;
	deserialise_rel(&lc, &st->outer);
	if (st->n_joins)
		deserialise_step(&lc, &st->join[0], true);
	if (i == GPUEXEC_DESC_CHAIN)
	{
		st->n_joins = 1 + get_int(&lc);
		if (st->n_joins < 2 || st->n_joins > GX_MAX_JOINS)
			ereport(ERROR, (errmsg("gpuexec: join chain of %d steps in the plan descriptor", st->n_joins)));
		for (j = 1; j < st->n_joins; j++)
			deserialise_step(&lc, &st->join[j], false);
	}
	st->partial = get_int(&lc);
	p->n_preds = get_int(&lc);
	p->outer_key_col = get_int(&lc);
	get_preds(&lc, p->n_preds, p->preds);
	p->n_group_cols = get_int(&lc);
	for (i = 0; i < p->n_group_cols; i++)
	{
		p->group_cols[i].side = get_int(&lc);
		p->group_cols[i].col = get_int(&lc);
	}
	p->n_aggs = get_int(&lc);
	for (i = 0; i < p->n_aggs; i++)
	{
		p->aggs[i].fn = get_int(&lc);
		p->aggs[i].arg.nops = get_int(&lc);
		for (j = 0; j < p->aggs[i].arg.nops; j++)
		{
			p->aggs[i].arg.ops[j].op = get_int(&lc);
			p->aggs[i].arg.ops[j].col = get_int(&lc);
			p->aggs[i].arg.ops[j].k = get_double(&lc);
		}
	}
	p->est_groups = get_int64(&lc);
}

/* ------------------------------------------------------ executor methods */
static void gpuexec_begin(CustomScanState *node, EState *estate, int eflags);
static TupleTableSlot *gpuexec_exec(CustomScanState *node);
static void gpuexec_end(CustomScanState *node);
static void gpuexec_rescan(CustomScanState *node);
static void gpuexec_explain(CustomScanState *node, List *ancestors, ExplainState *es);

static const CustomExecMethods gpuexec_exec_methods = {
	.CustomName = GPUEXEC_NAME,
	.BeginCustomScan = gpuexec_begin,
	.ExecCustomScan = gpuexec_exec,
	.EndCustomScan = gpuexec_end,
	.ReScanCustomScan = gpuexec_rescan,
	.ExplainCustomScan = gpuexec_explain,
};

static Node *
gpuexec_create_state(CustomScan *cscan)
{
	GpuExecState *st = (GpuExecState *) palloc0(sizeof(GpuExecState));

	NodeSetTag(st, T_CustomScanState);
	st->css.methods = &gpuexec_exec_methods;
	gpuexec_deserialise(cscan->custom_private, st);
	return (Node *) st;
}

static const CustomScanMethods gpuexec_scan_methods = {
	.CustomName = GPUEXEC_NAME,
	.CreateCustomScanState = gpuexec_create_state,
};

static void
gpuexec_begin(CustomScanState *node, EState *estate, int eflags)
{
	GpuExecState *st = (GpuExecState *) node;
	GpuHandles *h;

	if (eflags & EXEC_FLAG_EXPLAIN_ONLY)
		return;
	gpuexec_ensure_context();
	/* scanrelid == 0: ExecInitCustomScan built the scan slot from custom_scan_tlist
	 * (nodeCustom.c:81-94); we open the base relations ourselves */
	st->outer_rel = ExecOpenScanRelation(estate, st->outer.rti, eflags);
	for (int i = 0; i < st->n_joins; i++)
		st->join[i].r = ExecOpenScanRelation(estate, st->join[i].rel.rti, eflags);
	h = (GpuHandles *) malloc(sizeof(GpuHandles));
	h->owner = CurrentResourceOwner;
	h->state = st;
	h->next = live_handles;
	live_handles = h;
}

static void
gpuexec_run(GpuExecState *st, EState *estate)
{
	int64		n;
	int			ng = st->plan.n_group_cols,
				na = st->plan.n_aggs;
	instr_time	t0,
				t1;

	INSTR_TIME_SET_CURRENT(t0);
	for (int i = 0; i < st->n_joins; i++)
		gpuexec_load_relation(st->join[i].r, estate, &st->join[i].rel, &st->join[i].tab);
	gpuexec_load_relation(st->outer_rel, estate, &st->outer, &st->outer_tab);
	INSTR_TIME_SET_CURRENT(t1);
	INSTR_TIME_SUBTRACT(t1, t0);
	st->load_ms = INSTR_TIME_GET_MILLISEC(t1);

	INSTR_TIME_SET_CURRENT(t0);
	/* the tables in chain order; every one is in st before the next call, so an ERROR frees them all */
	for (int i = 0; i < st->n_joins && !is_right_join(st->plan.join_type); i++)
	{
		GpuJoinStep *j = &st->join[i];

		GX_CHECK(gx_hash_build(backend_ctx, j->tab, j->key_col, j->n_preds, j->preds, j->n_payload, j->payload_cols, j->unique, &j->hash));
		CHECK_FOR_INTERRUPTS();
	}
	if (is_right_join(st->plan.join_type))
	{
		/* the hashed relation is the outer table (its row numbers ride in the slots); join[0] probes it */
		GpuJoinStep *j = &st->join[0];
		gx_agg_plan cp = st->plan;

		GX_CHECK(gx_hash_build(backend_ctx, st->outer_tab, cp.outer_key_col, cp.n_preds, cp.preds, 0, NULL, j->unique, &j->hash));
		CHECK_FOR_INTERRUPTS();
		cp.outer_key_col = -1;
		cp.n_preds = 0;			/* applied by the build, and again when the consumed rows are compacted */
		cp.join_type = GX_JOIN_INNER;
		GX_CHECK(gx_hash_agg_right(backend_ctx, j->tab, j->key_col, j->n_preds, j->preds, st->outer_tab, j->hash,
								   st->plan.join_type, &cp, &st->result));
	}
	else if (st->n_joins >= 2)
	{
		gx_join_step steps[GX_MAX_JOINS];
		gx_agg_plan cp = st->plan;

		memset(steps, 0, sizeof(steps));
		for (int i = 0; i < st->n_joins; i++)
		{
			steps[i].h = st->join[i].hash;
			steps[i].key = st->join[i].probe;
			steps[i].join_type = GX_JOIN_INNER;
		}
		steps[0].key.side = 0;
		steps[0].key.col = st->plan.outer_key_col;
		cp.outer_key_col = -1;
		GX_CHECK(gx_hash_agg_joins(backend_ctx, st->outer_tab, st->n_joins, steps, &cp, &st->result));
	}
	else
		GX_CHECK(gx_hash_agg(backend_ctx, st->outer_tab, st->n_joins ? st->join[0].hash : NULL, &st->plan, &st->result));
	/* The result holds this datanode's groups only.  Whether they are final is the PLANNER's
	 * business: the hook offers the pushed-down path only when the GROUP BY covers the
	 * distribution key, and otherwise asks for partial states, which the reference's own
	 * RemoteSubplan + Finalize Agg above us combine (st->partial). */
	n = gx_result_ngroups(st->result);
	st->keys = (int64 *) palloc(sizeof(int64) * Max(n * ng, 1));
	st->aggs = (double *) palloc(sizeof(double) * Max(n * na, 1));
	st->nulls = (uint8 *) palloc(Max(n * (ng + na), 1));
	if (st->partial)
	{
		bool		sxx = false,
					regr = false;

		for (int a = 0; a < na; a++)
		{
			const GpuAggDef *def = agg_by_fn(st->plan.aggs[a].fn);

			sxx |= def && def->partial == PARTIAL_VAR;
			regr |= def && def->arg == AGG_ARG_F8_PAIR;
		}
		st->cnts = (int64 *) palloc(sizeof(int64) * Max(n * na, 1));
		GX_CHECK(gx_result_fetch_states(st->result, n, st->keys, st->aggs, st->cnts, st->nulls));
		if (sxx)
		{
			st->sxx = (double *) palloc(sizeof(double) * Max(n * na, 1));
			GX_CHECK(gx_result_fetch_sxx(st->result, n, st->sxx));
		}
		if (regr)
		{
			st->regr = (double *) palloc(sizeof(double) * 6 * Max(n * na, 1));
			GX_CHECK(gx_result_fetch_regr(st->result, n, st->regr));
		}
	}
	else
		GX_CHECK(gx_result_fetch(st->result, n, st->keys, st->aggs, st->nulls));
	st->ngroups = n;
	st->next = 0;
	INSTR_TIME_SET_CURRENT(t1);
	INSTR_TIME_SUBTRACT(t1, t0);
	st->exec_ms = INSTR_TIME_GET_MILLISEC(t1);
	/* the device copies are no longer needed */
	gpuexec_release_state(st);
	st->done_exec = true;
}

/* Returns one group per call as a virtual tuple.  The SCAN tuple is described by
 * custom_scan_tlist, which PlanCustomPath builds as (group columns in GROUP BY order,
 * aggregates in descriptor order) — whatever order the query's own target list has; the
 * plan's targetlist is projected over it (ExecAssignScanProjectionInfoWithVarno,
 * nodeCustom.c:100-101) below.  In partial mode an aggregate column carries the transition
 * value its row of gpuexec_aggs names. */
static TupleTableSlot *
gpuexec_exec(CustomScanState *node)
{
	GpuExecState *st = (GpuExecState *) node;
	TupleTableSlot *slot = node->ss.ss_ScanTupleSlot;
	TupleDesc	desc = slot->tts_tupleDescriptor;
	ExprContext *econtext = node->ss.ps.ps_ExprContext;
	int			ng = st->plan.n_group_cols,
				na = st->plan.n_aggs;
	int			i;
	int64		g;

	if (!st->done_exec)
		gpuexec_run(st, node->ss.ps.state);
	ExecClearTuple(slot);
	if (st->next >= st->ngroups)
		return slot;			/* empty slot = end of scan */
	if (econtext)
		ResetExprContext(econtext);	/* by-reference datums of the previous row die here */
	g = st->next++;
	for (i = 0; i < ng + na; i++)
	{
		bool		isnull = st->nulls[g * (ng + na) + i] != 0;
		Oid			typid = TupleDescAttr(desc, i)->atttypid;

		slot->tts_isnull[i] = isnull;
		if (isnull)
		{
			slot->tts_values[i] = (Datum) 0;
			continue;
		}
		if (i < ng)
		{
			int64		v = st->keys[g * ng + i];

			switch (typid)
			{
				case FLOAT8OID:
					{
						double		d;

						memcpy(&d, &v, sizeof(d));
						slot->tts_values[i] = Float8GetDatum(d);
						break;
					}
				case INT8OID:
					slot->tts_values[i] = Int64GetDatum(v);
					break;
				case CHAROID:
					slot->tts_values[i] = CharGetDatum((char) v);
					break;
				case BPCHAROID:
					{
						/* bpchar(1) was staged as its one byte: rebuild the varlena */
						MemoryContext old = MemoryContextSwitchTo(econtext->ecxt_per_tuple_memory);
						char		c = (char) v;

						slot->tts_values[i] = PointerGetDatum(cstring_to_text_with_len(&c, 1));
						MemoryContextSwitchTo(old);
						break;
					}
				default:
					slot->tts_values[i] = Int32GetDatum((int32) v);
					break;
			}
		}
		else
		{
			int			a = i - ng;
			double		d = st->aggs[g * na + a];
			const GpuAggDef *def = agg_by_fn(st->plan.aggs[a].fn);
			GpuAggPartial form = st->partial && def ? def->partial : PARTIAL_VALUE;

			if (form == PARTIAL_AVG || form == PARTIAL_VAR)
			{
				MemoryContext old = MemoryContextSwitchTo(econtext->ecxt_per_tuple_memory);
				Datum		elems[3];

				elems[0] = Float8GetDatum((double) st->cnts[g * na + a]);
				elems[1] = Float8GetDatum(d);
				elems[2] = Float8GetDatum(form == PARTIAL_AVG ? 0.0 : st->sxx[g * na + a]);
				slot->tts_values[i] = PointerGetDatum(construct_array(elems, 3, FLOAT8OID, sizeof(float8), FLOAT8PASSBYVAL, 'd'));
				MemoryContextSwitchTo(old);
			}
			else if (form == PARTIAL_REGR)
			{
				MemoryContext old = MemoryContextSwitchTo(econtext->ecxt_per_tuple_memory);
				Datum		elems[6];
				int			k;

				for (k = 0; k < 6; k++)
					elems[k] = Float8GetDatum(st->regr[(g * na + a) * 6 + k]);
				slot->tts_values[i] = PointerGetDatum(construct_array(elems, 6, FLOAT8OID, sizeof(float8), FLOAT8PASSBYVAL, 'd'));
				MemoryContextSwitchTo(old);
			}
			else if (form == PARTIAL_COUNT)
				slot->tts_values[i] = Int64GetDatum(st->cnts[g * na + a]);
			else if (typid == INT8OID)
			{
				int64		v;

				memcpy(&v, &d, sizeof(v));
				slot->tts_values[i] = Int64GetDatum(v);
			}
			else
				slot->tts_values[i] = Float8GetDatum(d);
		}
	}
	ExecStoreVirtualTuple(slot);
	if (node->ss.ps.ps_ProjInfo)
	{
		econtext->ecxt_scantuple = slot;
		return ExecProject(node->ss.ps.ps_ProjInfo);
	}
	return slot;
}

static void
gpuexec_end(CustomScanState *node)
{
	GpuExecState *st = (GpuExecState *) node;
	GpuHandles **p = &live_handles;

	gpuexec_release_state(st);
	while (*p)
	{
		if ((*p)->state == st)
		{
			GpuHandles *h = *p;

			*p = h->next;
			free(h);
		}
		else
			p = &(*p)->next;
	}
	if (st->outer_rel)
		ExecCloseScanRelation(st->outer_rel);
	for (int i = 0; i < st->n_joins; i++)
		if (st->join[i].r)
			ExecCloseScanRelation(st->join[i].r);
}

static void
gpuexec_rescan(CustomScanState *node)
{
	GpuExecState *st = (GpuExecState *) node;

	/* the result does not depend on parameters: replay it */
	st->next = 0;
}

static void
gpuexec_explain(CustomScanState *node, List *ancestors, ExplainState *es)
{
	GpuExecState *st = (GpuExecState *) node;
	int			i;

	ExplainPropertyText("GPU Strategy", st->n_joins ? "hash build + fused probe/aggregate" : "scan + hash aggregate", es);
	if (st->n_joins)
		ExplainPropertyText("GPU Join Type", st->plan.join_type == GX_JOIN_SEMI ? "Semi" : st->plan.join_type == GX_JOIN_ANTI ? "Anti"
							: st->plan.join_type == GX_JOIN_SEMI_RIGHT ? "Right Semi" : st->plan.join_type == GX_JOIN_ANTI_RIGHT ? "Right Anti"
							: "Inner", es);
	if (st->n_joins > 1)
		ExplainPropertyInteger("GPU Joins", NULL, st->n_joins, es);
	for (i = 0; i < st->plan.n_aggs; i++)
		if (st->plan.aggs[i].fn == GX_AGG_COUNT_DISTINCT)
		{
			int			att = st->outer.attnums[st->plan.aggs[i].arg.ops[0].col];
			char		name[NAMEDATALEN + 16];

			if (st->outer_rel && st->outer_rel->rd_att && att < st->outer_rel->rd_att->natts)
				snprintf(name, sizeof(name), "%s", NameStr(TupleDescAttr(st->outer_rel->rd_att, att)->attname));
			else
				snprintf(name, sizeof(name), "attribute %d", att + 1);
			ExplainPropertyText("GPU Distinct Column", name, es);
			break;
		}
	ExplainPropertyText("GPU Output", st->partial ? "partial states (Finalize above the redistribute)" : "final values (GROUP BY covers the distribution key)", es);
	if (es->analyze && st->done_exec)
	{
		ExplainPropertyFloat("GPU Load", "ms", st->load_ms, 3, es);
		ExplainPropertyFloat("GPU Exec", "ms", st->exec_ms, 3, es);
		ExplainPropertyInteger("GPU Groups", NULL, st->ngroups, es);
	}
}

/* ------------------------------------------------------- planner side */
static Plan *gpuexec_plan_path(PlannerInfo *root, RelOptInfo *rel, CustomPath *best_path,
				  List *tlist, List *clauses, List *custom_plans);

static const CustomPathMethods gpuexec_path_methods = {
	.CustomName = GPUEXEC_NAME,
	.PlanCustomPath = gpuexec_plan_path,
};

/* PlanCustomPath.  CustomPath.custom_private = (serialised descriptor, scan-tuple expressions):
 * the second list holds the GROUP BY expressions in groupClause order followed by the
 * (final or partial) Aggrefs in descriptor order — exactly the columns gpuexec_exec() fills —
 * and becomes custom_scan_tlist.  The plan's own targetlist (SELECT order, resjunk entries,
 * whatever) is then resolved against it by set_customscan_references (setrefs.c:1805) and
 * projected at run time; nothing relies on the two orders coinciding. */
static Plan *
gpuexec_plan_path(PlannerInfo *root, RelOptInfo *rel, CustomPath *best_path,
				  List *tlist, List *clauses, List *custom_plans)
{
	CustomScan *cscan = makeNode(CustomScan);
	List	   *scan_exprs = (List *) lsecond(best_path->custom_private);
	List	   *stl = NIL;
	ListCell   *lc;
	AttrNumber	resno = 1;

	foreach(lc, scan_exprs)
		stl = lappend(stl, makeTargetEntry((Expr *) copyObject(lfirst(lc)), resno++, NULL, false));
	cscan->scan.plan.targetlist = tlist;
	cscan->scan.plan.qual = NIL;	/* HAVING is declined by the hook */
	cscan->scan.scanrelid = 0;
	cscan->flags = best_path->flags;
	cscan->custom_plans = NIL;
	cscan->custom_exprs = NIL;
	cscan->custom_private = (List *) linitial(best_path->custom_private);
	cscan->custom_scan_tlist = stl;
	cscan->custom_relids = NULL;
	cscan->methods = &gpuexec_scan_methods;
	return &cscan->scan.plan;
}

/* ---- plan-shape analysis -------------------------------------------------
 * Accepts:   Agg(HASHED/PLAIN) over  SeqScan(R)                       (configs 1, 2, Q1)
 *            Agg over HashJoin[INNER, one int4/int8 equi-key](SeqScan(R), SeqScan(S))   (config 3)
 *            Agg over HashJoin[SEMI / ANTI, the same key shape]  (EXISTS / NOT EXISTS: TPC-H Q4, Q21, Q22 shapes),
 *            with GROUP BY columns and aggregate arguments from the outer side only
 *            Agg over a left-deep chain of 2..GX_MAX_JOINS such INNER joins with unique build sides (star joins:
 *            TPC-H Q3), GROUP BY columns from any relation, aggregate arguments from the outer one (match_joins)
 * with "Var op Const" quals on the scans, Var group keys, no HAVING / grouping sets /
 * ORDER BY aggregates / FILTER, and the aggregates of gpuexec_aggs; every target-list entry must be a group Var or a
 * bare Aggref.  Anything else returns false and the CPU paths stay untouched — the same
 * "eligibility test" idea as jit_compile_hashjoin (jit/jit.c:253-303). */

/* what the matcher learns besides the descriptor: the planner hook reads the Aggrefs and the estimates */
typedef struct GpuPlanMatch
{
	List	   *agg_refs;		/* the Aggrefs, in descriptor order */
	int32		key_types[GX_MAX_GROUP_COLS + 1];	/* staged types of the group columns, then of the DISTINCT column */
	Var		   *distinct_arg;	/* the column of the query's count(DISTINCT) aggregates */
	double		outer_rows;		/* rows of the relation in the descriptor's outer slot */
	double		pages;			/* heap pages of every relation the plan scans */
	double		groups;
	double		pairs;			/* count(DISTINCT): the (group, value) pairs of its first stage; 0 without one */
	double		bytes;			/* HBM the plan needs */
} GpuPlanMatch;

/* column number of (rti, attno) in the descriptor, appended on first use */
static int
rel_column(GpuRelInfo *r, Index rti, AttrNumber attno, Oid typid, int32 typmod)
{
	int32		gxt = gpuexec_type_of(typid);
	int			i;

	if (r->rti != rti || attno <= 0 || gxt == 0)
		return -1;
	if (typid == BPCHAROID && typmod != VARHDRSZ + 1)
		return -1;				/* only bpchar(1) is staged as one byte */
	for (i = 0; i < r->ncols; i++)
		if (r->attnums[i] == attno - 1)
			return i;
	if (r->ncols >= GX_MAX_COLS)
		return -1;
	r->attnums[r->ncols] = attno - 1;
	r->types[r->ncols] = gxt;
	return r->ncols++;
}

/* float8 expression -> postfix program over outer columns */
static bool
match_f8_expr(Node *n, GpuRelInfo *outer, gx_expr *e)
{
	if (n == NULL || e->nops >= GX_MAX_EXPR_OPS)
		return false;
	if (IsA(n, RelabelType))
		return match_f8_expr((Node *) ((RelabelType *) n)->arg, outer, e);
	if (IsA(n, Var))
	{
		Var		   *v = (Var *) n;
		int			c = rel_column(outer, v->varno, v->varattno, v->vartype, v->vartypmod);

		if (c < 0 || v->varlevelsup != 0 || (v->vartype != FLOAT8OID && v->vartype != INT4OID && v->vartype != INT8OID))
			return false;
		e->ops[e->nops].op = GX_OP_COL;
		e->ops[e->nops].col = c;
		e->nops++;
		return true;
	}
	if (IsA(n, Const))
	{
		Const	   *c = (Const *) n;

		if (c->constisnull || c->consttype != FLOAT8OID)
			return false;
		e->ops[e->nops].op = GX_OP_CONST;
		e->ops[e->nops].k = DatumGetFloat8(c->constvalue);
		e->nops++;
		return true;
	}
	if (IsA(n, OpExpr))
	{
		OpExpr	   *o = (OpExpr *) n;
		int			op;

		if (list_length(o->args) != 2)
			return false;
		switch (o->opfuncid)
		{
			case F_FLOAT8PL:
				op = GX_OP_ADD;
				break;
			case F_FLOAT8MI:
				op = GX_OP_SUB;
				break;
			case F_FLOAT8MUL:
				op = GX_OP_MUL;
				break;
			default:
				return false;
		}
		if (!match_f8_expr(linitial(o->args), outer, e) || !match_f8_expr(lsecond(o->args), outer, e))
			return false;
		if (e->nops >= GX_MAX_EXPR_OPS)
			return false;
		e->ops[e->nops++].op = op;
		return true;
	}
	return false;
}

/* comparison function oid -> (GX_* operator, operand class: 'i' integer-like, 'f' float8, 'c' one byte) */
static bool
qual_operator(Oid funcid, int *op, char *cls)
{
	static const struct { Oid fn; int op; char cls; } tab[] = {
		{F_INT4LT, GX_LT, 'i'}, {F_INT4LE, GX_LE, 'i'}, {F_INT4EQ, GX_EQ, 'i'}, {F_INT4GE, GX_GE, 'i'}, {F_INT4GT, GX_GT, 'i'}, {F_INT4NE, GX_NE, 'i'},
		{F_INT8LT, GX_LT, 'i'}, {F_INT8LE, GX_LE, 'i'}, {F_INT8EQ, GX_EQ, 'i'}, {F_INT8GE, GX_GE, 'i'}, {F_INT8GT, GX_GT, 'i'}, {F_INT8NE, GX_NE, 'i'},
		{F_DATE_LT, GX_LT, 'i'}, {F_DATE_LE, GX_LE, 'i'}, {F_DATE_EQ, GX_EQ, 'i'}, {F_DATE_GE, GX_GE, 'i'}, {F_DATE_GT, GX_GT, 'i'}, {F_DATE_NE, GX_NE, 'i'},
		{F_FLOAT8LT, GX_LT, 'f'}, {F_FLOAT8LE, GX_LE, 'f'}, {F_FLOAT8EQ, GX_EQ, 'f'}, {F_FLOAT8GE, GX_GE, 'f'}, {F_FLOAT8GT, GX_GT, 'f'}, {F_FLOAT8NE, GX_NE, 'f'},
		{F_CHARLT, GX_LT, 'c'}, {F_CHARLE, GX_LE, 'c'}, {F_CHAREQ, GX_EQ, 'c'}, {F_CHARGE, GX_GE, 'c'}, {F_CHARGT, GX_GT, 'c'}, {F_CHARNE, GX_NE, 'c'},
		{F_BPCHAREQ, GX_EQ, 'b'}, {F_BPCHARNE, GX_NE, 'b'},
	};
	int			i;

	for (i = 0; i < (int) lengthof(tab); i++)
		if (tab[i].fn == funcid)
		{
			*op = tab[i].op;
			*cls = tab[i].cls;
			return true;
		}
	return false;
}

/* baserestrictinfo -> gx_pred[]: every clause must be "Var op Const" (either order) with both
 * sides of the SAME type (no cross-type int48/int84 operators); false = decline the plan */
static bool
match_quals(List *restrictinfo, GpuRelInfo *rel, gx_pred *preds, int *n_preds)
{
	ListCell   *lc;

	foreach(lc, restrictinfo)
	{
		RestrictInfo *ri = (RestrictInfo *) lfirst(lc);
		OpExpr	   *o = (OpExpr *) ri->clause;
		Node	   *l,
				   *r;
		Var		   *v;
		Const	   *k;
		int			op,
					c;
		char		cls;
		bool		flipped = false;

		if (ri->pseudoconstant || !IsA(o, OpExpr) || list_length(o->args) != 2 || *n_preds >= GX_MAX_PREDS)
			return false;
		l = (Node *) linitial(o->args);
		r = (Node *) lsecond(o->args);
		if (IsA(l, RelabelType))
			l = (Node *) ((RelabelType *) l)->arg;
		if (IsA(r, RelabelType))
			r = (Node *) ((RelabelType *) r)->arg;
		if (IsA(l, Const) && IsA(r, Var))
		{
			Node	   *t = l;

			l = r;
			r = t;
			flipped = true;
		}
		if (!IsA(l, Var) || !IsA(r, Const) || !qual_operator(o->opfuncid, &op, &cls))
			return false;
		v = (Var *) l;
		k = (Const *) r;
		if (k->constisnull || v->varlevelsup != 0 || k->consttype != v->vartype)
			return false;
		c = rel_column(rel, v->varno, v->varattno, v->vartype, v->vartypmod);
		if (c < 0)
			return false;
		if (flipped)			/* const op var  ==  var op' const */
			op = op == GX_LT ? GX_GT : op == GX_LE ? GX_GE : op == GX_GT ? GX_LT : op == GX_GE ? GX_LE : op;
		preds[*n_preds].col = c;
		preds[*n_preds].op = op;
		preds[*n_preds].ival = 0;
		preds[*n_preds].fval = 0;
		switch (cls)
		{
			case 'i':
				preds[*n_preds].ival = v->vartype == INT8OID ? DatumGetInt64(k->constvalue) : (int64) DatumGetInt32(k->constvalue);
				break;
			case 'f':
				preds[*n_preds].fval = DatumGetFloat8(k->constvalue);
				break;
			case 'c':
				preds[*n_preds].ival = (int64) (unsigned char) DatumGetChar(k->constvalue);
				break;
			default:			/* bpchar(1) = 'x' */
				{
					struct varlena *t = (struct varlena *) DatumGetPointer(k->constvalue);

					if (VARSIZE_ANY_EXHDR(t) != 1)
						return false;
					preds[*n_preds].ival = (int64) (unsigned char) VARDATA_ANY(t)[0];
					break;
				}
		}
		(*n_preds)++;
	}
	return true;
}

/* Relations the GPU path must not read around the row-level machinery ExecScan applies per
 * tuple (execScan.c:185-200,261,313-325): data masking, CLS policies, FGA audit policies. */
static bool
relation_is_protected(PlannerInfo *root, Index rti)
{
	RangeTblEntry *rte = planner_rt_fetch(rti, root);
	List	   *fga = NIL;

	if (rte->rtekind != RTE_RELATION)
		return true;
	if (g_enable_data_mask && datamask_check_table_has_datamask(rte->relid))
		return true;
	if (g_enable_cls && cls_check_table_has_policy(rte->relid))
		return true;
	if (enable_fga && get_audit_fga_quals(rte->relid, "select", root->parse->targetList, &fga) && fga != NIL)
		return true;
	return false;
}

/* GROUP BY covers the distribution key: groups on different datanodes cannot overlap, so the
 * whole aggregation may run below the RemoteSubplan.  Restates the rule of
 * grouping_distribution_match (planner.c:8588-8668) with plain equal() — stricter than the
 * reference's exprs_known_equal(), so it can only decline more often. */
static bool
grouping_covers_distribution(Query *parse, Distribution *d)
{
	int			j;

	if (d == NULL || IsLocatorReplicated(d->distributionType))
		return true;
	if (!IsValidDistribution(d))
		return false;
	for (j = 0; j < d->nExprs; j++)
	{
		ListCell   *lc;
		bool		found = false;

		foreach(lc, parse->groupClause)
		{
			TargetEntry *tle = get_sortgroupclause_tle((SortGroupClause *) lfirst(lc), parse->targetList);

			if (d->disExprs[j] && equal(tle->expr, d->disExprs[j]))
			{
				found = true;
				break;
			}
		}
		if (!found)
			return false;
	}
	return true;
}

/* bytes of a staged column */
static int
staged_type_bytes(int32 t)
{
	return (t == GX_INT8 || t == GX_FLOAT8) ? 8 : t == GX_CHAR ? 1 : 4;
}

/* pg_attribute.attnotnull of (relation of rti, attno): the join payload has no NULL representation */
static bool
column_is_not_null(PlannerInfo *root, Index rti, AttrNumber attno)
{
	RangeTblEntry *rte = planner_rt_fetch(rti, root);
	HeapTuple	tp = SearchSysCache2(ATTNUM, ObjectIdGetDatum(rte->relid), Int16GetDatum(attno));
	bool		res = false;

	if (HeapTupleIsValid(tp))
	{
		res = ((Form_pg_attribute) GETSTRUCT(tp))->attnotnull;
		ReleaseSysCache(tp);
	}
	return res;
}

/*
 * The library's state words per group (csrc/gx_agg.cu, compile_plan), restated so that a plan the library
 * would refuse with "too many state words" is declined here, at plan time.  Word 0 counts the group's rows; a count
 * of a nullable column takes one word, a sum(int4) two when its column is nullable; sum, avg, min and max of float8
 * take a value word and, over a nullable argument, a count word; sum, avg and the variances of one argument share
 * these, and the variances of one argument share three more {C, S1, S2}.  Before each aggregate the library wants
 * room for two words, or five for a variance; count(DISTINCT) is no aggregate of its first stage, and its fold adds
 * one word at the end.
 */
#define GPUEXEC_MAX_STATE_WORDS 18		/* GX_MAX_WORDS, csrc/gx_internal.cuh */

static bool
same_f8_expr(const gx_expr *x, const gx_expr *y)
{
	int			k;

	if (x->nops != y->nops)
		return false;
	for (k = 0; k < x->nops; k++)
		if (x->ops[k].op != y->ops[k].op || x->ops[k].col != y->ops[k].col || memcmp(&x->ops[k].k, &y->ops[k].k, sizeof(double)) != 0)
			return false;
	return true;
}

static bool
state_words_fit(PlannerInfo *root, const GpuRelInfo *outer, const gx_agg_plan *plan)
{
	bool		sum_words[GX_MAX_AGGS] = {false},
				var_words[GX_MAX_AGGS] = {false};
	bool		distinct = false,
				regr_full = false;
	int			nw = 1,
				regr_owner = -1,
				a,
				b,
				k;

	/* the two-argument aggregates share one state, over one (Y, X) pair: a second pair is declined */
	for (a = 0; a < plan->n_aggs; a++)
	{
		const GpuAggDef *def = agg_by_fn(plan->aggs[a].fn);

		if (def == NULL || def->arg != AGG_ARG_F8_PAIR)
			continue;
		if (def->partial == PARTIAL_REGR)
			regr_full = true;
		if (regr_owner < 0)
			regr_owner = a;
		else if (!same_f8_expr(&plan->aggs[a].arg, &plan->aggs[regr_owner].arg))
			return false;
	}

	for (a = 0; a < plan->n_aggs; a++)
	{
		const gx_agg *g = &plan->aggs[a];
		const GpuAggDef *def = agg_by_fn(g->fn);
		bool		nullable = false;
		int			twin = -1;

		if (def == NULL)		/* count(DISTINCT) */
		{
			distinct = true;
			continue;
		}
		for (k = 0; k < g->arg.nops; k++)
			if (g->arg.ops[k].op == GX_OP_COL && !column_is_not_null(root, outer->rti, outer->attnums[g->arg.ops[k].col] + 1))
				nullable = true;
		if (def->arg == AGG_ARG_F8_PAIR)
		{
			/* the first of them owns the pair count (when a side is nullable) and, unless all are regr_count,
			 * {Sx, Sy, Cx, S1x, S2x, Cy, S1y, S2y, Sxy'}; never shared with sum / avg */
			if (a == regr_owner)
				nw += (nullable ? 1 : 0) + (regr_full ? 9 : 0);
			if (nw > GPUEXEC_MAX_STATE_WORDS)
				return false;
			continue;
		}
		if (nw + (def->partial == PARTIAL_VAR ? 5 : 2) > GPUEXEC_MAX_STATE_WORDS)
			return false;
		switch (g->fn)
		{
			case GX_AGG_COUNT_STAR:
				break;
			case GX_AGG_COUNT:
				nw += nullable ? 1 : 0;
				break;
			case GX_AGG_SUM_I4:
			case GX_AGG_MIN_F8:
			case GX_AGG_MAX_F8:
				nw += nullable ? 2 : 1;
				break;
			default:			/* sum, avg and the variances of float8 */
				sum_words[a] = true;
				for (b = 0; b < a && twin < 0; b++)
					if (sum_words[b] && same_f8_expr(&plan->aggs[b].arg, &g->arg))
						twin = b;
				if (twin < 0)
				{
					twin = a;
					nw += nullable ? 2 : 1;
				}
				if (def->partial == PARTIAL_VAR && !var_words[twin])
				{
					var_words[twin] = true;
					nw += 3;
				}
				break;
		}
	}
	return nw + (distinct ? 1 : 0) <= GPUEXEC_MAX_STATE_WORDS;
}

/* payload slot of column c of a join's build side, appended on first use: a probe key of a later step and a group column
 * that read the same column share one slot */
static int
payload_slot(int32 *cols, int *n, int c)
{
	int			i;

	for (i = 0; i < *n; i++)
		if (cols[i] == c)
			return i;
	if (*n >= GX_MAX_PAYLOAD)
		return -1;
	cols[*n] = c;
	return (*n)++;
}

/* the join step (1..) whose build side scans rti, or 0 */
static int
join_step_of(const GpuExecState *st, Index rti)
{
	int			i;

	for (i = 0; i < st->n_joins; i++)
		if (st->join[i].rel.rti == rti)
			return 1 + i;
	return 0;
}

/* One level of a left-deep join: exactly one int4eq / int8eq hash clause that is its whole joinrestrictinfo, and a plain
 * SeqScan of an unprotected relation as the build side.  *iv = the clause's Var of the build side, *ov = the other one. */
static bool
join_level(PlannerInfo *root, HashPath *hp, Var **ov, Var **iv)
{
	Path	   *ip = hp->jpath.innerjoinpath;
	RestrictInfo *ri;
	OpExpr	   *clause;
	Var		   *a,
			   *b;

	if (list_length(hp->path_hashclauses) != 1 || list_length(hp->jpath.joinrestrictinfo) != 1)
		return false;
	if (ip->pathtype != T_SeqScan)		/* a RemoteSubplan below: the inputs are not co-located */
		return false;
	ri = (RestrictInfo *) linitial(hp->path_hashclauses);
	clause = (OpExpr *) ri->clause;
	if (!IsA(clause, OpExpr) || list_length(clause->args) != 2 || !IsA(linitial(clause->args), Var) || !IsA(lsecond(clause->args), Var))
		return false;
	if (clause->opfuncid != F_INT4EQ && clause->opfuncid != F_INT8EQ)
		return false;
	a = (Var *) linitial(clause->args);
	b = (Var *) lsecond(clause->args);
	if (b->varno != ip->parent->relid)
	{
		Var		   *t = a;

		a = b;
		b = t;
	}
	if (b->varno != ip->parent->relid || a->varno == b->varno || relation_is_protected(root, b->varno))
		return false;
	*ov = a;
	*iv = b;
	return true;
}

/* Agg over HashJoin(HashJoin(... SeqScan(F), SeqScan(D1)) ..., SeqScan(Dn)), 1 <= n <= GX_MAX_JOINS: step s builds Ds.
 * One join may be INNER, SEMI or ANTI (EXISTS / NOT EXISTS), or SEMI_RIGHT / ANTI_RIGHT; a chain (gx_hash_agg_joins) must
 * be INNER with a unique build side on every level.  LEFT, RIGHT, FULL and the JOIN_UNIQUE_* forms stay on the CPU.
 * A right semi / right anti join preserves its hashed (inner) relation: that relation takes the outer slot of the
 * descriptor (its key, quals, GROUP BY and argument columns), and the probing relation the join step, with its key and
 * quals only (gx_hash_agg_right).  Step 1's probe key is a
 * column of F; a later step's is a column of F or of an earlier D, carried in that step's payload (which has no NULL
 * flag: the column must be NOT NULL). */
static bool
match_joins(PlannerInfo *root, HashPath *top, GpuExecState *out, GpuPlanMatch *m)
{
	HashPath   *lv[GX_MAX_JOINS];
	Path	   *p = &top->jpath.path;
	gx_agg_plan *plan = &out->plan;
	int			n = 0,
				s;

	while (IsA(p, HashPath))
	{
		if (n == GX_MAX_JOINS)
			return false;
		lv[n++] = (HashPath *) p;
		p = ((HashPath *) p)->jpath.outerjoinpath;
	}
	if (p->pathtype != T_SeqScan)
		return false;
	out->outer.rti = p->parent->relid;
	if (relation_is_protected(root, out->outer.rti))
		return false;
	out->n_joins = n;
	m->outer_rows = p->parent->tuples;
	m->pages = p->parent->pages;
	for (s = 1; s <= n; s++)
	{
		HashPath   *hp = lv[n - s];
		JoinType	jt = hp->jpath.jointype;
		RelOptInfo *irel = hp->jpath.innerjoinpath->parent;
		GpuJoinStep *j = &out->join[s - 1];
		Var		   *ov,
				   *iv;
		int			c,
					t = 0;

		if (n == 1 ? (jt != JOIN_INNER && jt != JOIN_SEMI && jt != JOIN_ANTI && jt != JOIN_SEMI_RIGHT && jt != JOIN_ANTI_RIGHT)
			: (jt != JOIN_INNER || !hp->jpath.inner_unique))
			return false;
		if (!join_level(root, hp, &ov, &iv))
			return false;
		if (jt == JOIN_SEMI_RIGHT || jt == JOIN_ANTI_RIGHT)
		{
			/* the probe relation p (F so far) becomes the join step; the hashed relation the outer slot */
			plan->join_type = jt == JOIN_SEMI_RIGHT ? GX_JOIN_SEMI_RIGHT : GX_JOIN_ANTI_RIGHT;
			j->unique = hp->jpath.inner_unique;
			j->tuples = p->parent->tuples;
			j->rel.rti = out->outer.rti;
			out->outer.rti = iv->varno;
			m->outer_rows = irel->tuples;
			m->pages += irel->pages;
			plan->outer_key_col = rel_column(&out->outer, iv->varno, iv->varattno, iv->vartype, iv->vartypmod);
			j->key_col = rel_column(&j->rel, ov->varno, ov->varattno, ov->vartype, ov->vartypmod);
			return plan->outer_key_col >= 0 && j->key_col >= 0 &&
				match_quals(irel->baserestrictinfo, &out->outer, plan->preds, &plan->n_preds) &&
				match_quals(p->parent->baserestrictinfo, &j->rel, j->preds, &j->n_preds);
		}
		plan->join_type = jt == JOIN_SEMI ? GX_JOIN_SEMI : jt == JOIN_ANTI ? GX_JOIN_ANTI : GX_JOIN_INNER;
		j->unique = hp->jpath.inner_unique;
		j->tuples = irel->tuples;
		j->rel.rti = iv->varno;
		j->key_col = rel_column(&j->rel, iv->varno, iv->varattno, iv->vartype, iv->vartypmod);
		if (j->key_col < 0)
			return false;
		/* the probe key: a column of F, or the payload of the earlier step that scans ov's relation */
		if (ov->varno == out->outer.rti)
			c = rel_column(&out->outer, ov->varno, ov->varattno, ov->vartype, ov->vartypmod);
		else
		{
			t = join_step_of(out, ov->varno);
			if (t < 1 || t >= s || !column_is_not_null(root, ov->varno, ov->varattno))
				return false;
			c = rel_column(&out->join[t - 1].rel, ov->varno, ov->varattno, ov->vartype, ov->vartypmod);
			if (c >= 0)
				c = payload_slot(out->join[t - 1].payload_cols, &out->join[t - 1].n_payload, c);
		}
		if (c < 0)
			return false;
		if (s == 1)
		{
			/* the outer quals right after step 1's probe key: F's columns are numbered in the order they are first met */
			plan->outer_key_col = c;
			if (!match_quals(p->parent->baserestrictinfo, &out->outer, plan->preds, &plan->n_preds))
				return false;
		}
		else
		{
			j->probe.side = t;
			j->probe.col = c;
		}
		if (!match_quals(irel->baserestrictinfo, &j->rel, j->preds, &j->n_preds))
			return false;
		m->pages += irel->pages;
	}
	return true;
}

/* the outer relation: a base-relation scan, or a join (match_joins) */
static bool
match_input(PlannerInfo *root, RelOptInfo *input_rel, GpuExecState *out, GpuPlanMatch *m)
{
	Path	   *in = input_rel->cheapest_total_path;

	if (in->pathtype == T_SeqScan && input_rel->reloptkind == RELOPT_BASEREL)
	{
		out->outer.rti = input_rel->relid;
		if (relation_is_protected(root, input_rel->relid) ||
			!match_quals(input_rel->baserestrictinfo, &out->outer, out->plan.preds, &out->plan.n_preds))
			return false;
		m->outer_rows = input_rel->tuples;
		m->pages = input_rel->pages;
		return true;
	}
	return IsA(in, HashPath) && match_joins(root, (HashPath *) in, out, m);
}

/* GROUP BY: plain Vars of the outer side, or of a build side under INNER joins, riding in that join's payload */
static bool
match_group_by(PlannerInfo *root, GpuExecState *out, GpuPlanMatch *m)
{
	Query	   *parse = root->parse;
	gx_agg_plan *plan = &out->plan;
	ListCell   *lc;

	foreach(lc, parse->groupClause)
	{
		SortGroupClause *sgc = (SortGroupClause *) lfirst(lc);
		TargetEntry *tle = get_sortgroupclause_tle(sgc, parse->targetList);
		Var		   *v = (Var *) tle->expr;
		int			c,
					s = 0;

		if (!IsA(v, Var) || plan->n_group_cols >= GX_MAX_GROUP_COLS)
			return false;
		if (v->varno == out->outer.rti)
		{
			c = rel_column(&out->outer, v->varno, v->varattno, v->vartype, v->vartypmod);
			if (c < 0)
				return false;
			m->key_types[plan->n_group_cols] = out->outer.types[c];
		}
		else if (plan->join_type == GX_JOIN_INNER && (s = join_step_of(out, v->varno)) > 0)
		{
			/* a build-side column of step s, in that step's payload (a slot its probe key or another GROUP BY entry may share) */
			GpuJoinStep *j = &out->join[s - 1];

			c = rel_column(&j->rel, v->varno, v->varattno, v->vartype, v->vartypmod);
			if (c < 0 || !column_is_not_null(root, v->varno, v->varattno))
				return false;		/* gx_hash_build carries payload columns inside the slot: no room for a NULL flag */
			m->key_types[plan->n_group_cols] = j->rel.types[c];
			c = payload_slot(j->payload_cols, &j->n_payload, c);
			if (c < 0)
				return false;
		}
		else
			return false;
		plan->group_cols[plan->n_group_cols].side = s;
		plan->group_cols[plan->n_group_cols++].col = c;
	}
	return true;
}

/* the library's group key is two 8-byte words, filled first-fit in key order (compile_plan, csrc/gx_agg.cu): do columns
 * of these staged types fit? */
static bool
group_key_fits(const int32 *types, int n)
{
	int			used[2] = {0, 0};

	for (int i = 0; i < n; i++)
	{
		int			b = staged_type_bytes(types[i]),
					w = used[0] + b <= 8 ? 0 : 1;

		if (used[w] + b > 8)
			return false;
		used[w] += b;
	}
	return true;
}

/* Limits the library would only report at execution time (GX_ERR_ARG -> ERROR): decline here instead, the CPU plan stays.
 * A join's payload is one 8-byte word (gx_hash_build, csrc/gx_join.cu), and the GROUP BY key must fit the group key. */
static bool
within_library_limits(const GpuExecState *out, const GpuPlanMatch *m)
{
	for (int i = 0; i < out->n_joins; i++)
	{
		const GpuJoinStep *j = &out->join[i];
		int			payload_bytes = 0;

		for (int k = 0; k < j->n_payload; k++)
			payload_bytes += staged_type_bytes(j->rel.types[j->payload_cols[k]]);
		if (payload_bytes > 8)
			return false;
	}
	return group_key_fits(m->key_types, out->plan.n_group_cols);
}

/* every target-list entry is either one of the GROUP BY expressions or a bare Aggref of gpuexec_aggs; the Aggrefs, in
 * target-list order, are the descriptor's aggregates and the tail of the scan tuple */
static bool
match_aggregates(Query *parse, GpuExecState *out, GpuPlanMatch *m)
{
	gx_agg_plan *plan = &out->plan;
	ListCell   *lc;

	foreach(lc, parse->targetList)
	{
		TargetEntry *tle = (TargetEntry *) lfirst(lc);
		Aggref	   *a = (Aggref *) tle->expr;
		const GpuAggDef *def;
		gx_agg	   *g;

		if (IsA(a, Var))
		{
			ListCell   *gc;
			bool		is_group = false;

			foreach(gc, parse->groupClause)
				if (equal(get_sortgroupclause_tle((SortGroupClause *) lfirst(gc), parse->targetList)->expr, a))
					is_group = true;
			if (!is_group)
				return false;	/* functionally dependent column: not carried */
			continue;
		}
		if (!IsA(a, Aggref) || a->aggorder || a->aggfilter || a->aggdirectargs || plan->n_aggs >= GX_MAX_AGGS ||
			(def = agg_by_oid(a->aggfnoid)) == NULL)
			return false;
		g = &plan->aggs[plan->n_aggs];
		g->fn = def->fn;
		if (a->aggdistinct)
		{
			/* count(DISTINCT col) over a plain int4 / int8 / date column of the outer relation (GX_AGG_COUNT_DISTINCT):
			 * one sort clause, over the argument, and the same column in every DISTINCT aggregate of the query */
			TargetEntry *arg;
			SortGroupClause *sgc;
			Var		   *v;
			int			c;

			if (def->fn != GX_AGG_COUNT || list_length(a->args) != 1 || list_length(a->aggdistinct) != 1)
				return false;
			arg = (TargetEntry *) linitial(a->args);
			sgc = (SortGroupClause *) linitial(a->aggdistinct);
			v = (Var *) arg->expr;
			if (sgc->tleSortGroupRef != arg->ressortgroupref || !IsA(v, Var) || v->varlevelsup != 0 || v->varno != out->outer.rti ||
				(v->vartype != INT4OID && v->vartype != INT8OID && v->vartype != DATEOID))
				return false;
			c = rel_column(&out->outer, v->varno, v->varattno, v->vartype, v->vartypmod);
			if (c < 0 || (m->distinct_arg != NULL && !equal(m->distinct_arg, v)))
				return false;
			m->distinct_arg = v;
			m->key_types[plan->n_group_cols] = out->outer.types[c];	/* count(DISTINCT)'s first stage groups by it too */
			g->fn = GX_AGG_COUNT_DISTINCT;
			g->arg.nops = 1;
			g->arg.ops[0].op = GX_OP_COL;
			g->arg.ops[0].col = c;
		}
		else
			switch (def->arg)
			{
				case AGG_ARG_NONE:
					break;
				case AGG_ARG_COLUMN:
				case AGG_ARG_F8:
					if (list_length(a->args) != 1 ||
						!match_f8_expr((Node *) ((TargetEntry *) linitial(a->args))->expr, &out->outer, &g->arg))
						return false;
					if (def->arg == AGG_ARG_COLUMN && g->arg.nops != 1)
						return false;
					break;
				case AGG_ARG_F8_PAIR:
					/* Y's program, GX_OP_ARG2, X's program, within GX_MAX_EXPR_OPS */
					if (list_length(a->args) != 2 ||
						!match_f8_expr((Node *) ((TargetEntry *) linitial(a->args))->expr, &out->outer, &g->arg) ||
						g->arg.nops >= GX_MAX_EXPR_OPS)
						return false;
					g->arg.ops[g->arg.nops++].op = GX_OP_ARG2;
					if (!match_f8_expr((Node *) ((TargetEntry *) lsecond(a->args))->expr, &out->outer, &g->arg))
						return false;
					break;
			}
		m->agg_refs = lappend(m->agg_refs, a);
		plan->n_aggs++;
	}
	return plan->n_aggs > 0 || plan->n_group_cols > 0;
}

/* count(DISTINCT): the library groups by the key plus the DISTINCT column first, so that key must fit too (first fit, the
 * column packed last), and est_groups is read as the number of distinct (group, value) pairs */
static bool
size_distinct_pairs(PlannerInfo *root, double input_rows, GpuExecState *out, GpuPlanMatch *m)
{
	Query	   *parse = root->parse;
	gx_agg_plan *plan = &out->plan;
	List	   *exprs = NIL;
	ListCell   *lc;
	double		pairs;

	if (plan->n_group_cols >= GX_MAX_GROUP_COLS || !group_key_fits(m->key_types, plan->n_group_cols + 1))
		return false;
	foreach(lc, parse->groupClause)
		exprs = lappend(exprs, get_sortgroupclause_tle((SortGroupClause *) lfirst(lc), parse->targetList)->expr);
	exprs = lappend(exprs, m->distinct_arg);
	pairs = estimate_num_groups(root, exprs, input_rows, NULL);
	if (pairs > input_rows)
		pairs = input_rows;
	if (pairs < 1)
		pairs = 1;
	plan->est_groups = (int64) pairs;
	m->pairs = pairs;
	return true;
}

/* HBM the plan needs: the referenced columns of every row, plus 16 B x 2 per build row */
static double
hbm_bytes(const GpuExecState *out, const GpuPlanMatch *m)
{
	double		bytes = 0;
	int			i;

	for (i = 0; i < out->outer.ncols; i++)
		bytes += m->outer_rows * staged_type_bytes(out->outer.types[i]);
	if (is_right_join(out->plan.join_type))
	{
		double		probe_row = 0;

		for (i = 0; i < out->join[0].rel.ncols; i++)
			probe_row += staged_type_bytes(out->join[0].rel.types[i]);
		bytes = gpuexec_right_join_bytes(m->outer_rows, bytes / Max(m->outer_rows, 1), out->join[0].tuples, probe_row);
	}
	else
		for (i = 0; i < out->n_joins; i++)
		{
			const GpuJoinStep *j = &out->join[i];
			int			k;

			for (k = 0; k < j->rel.ncols; k++)
				bytes += j->tuples * staged_type_bytes(j->rel.types[k]);
			bytes += j->tuples * 32;
		}
	/* count(DISTINCT): one record of (3 + state words) 8-byte words per pair, held about three times over while the
	 * fold reads the stage-1 records and partitions its copy of them (csrc/gx_agg.cu, count_distinct_run) */
	if (m->distinct_arg)
		bytes += m->pairs * 8.0 * (3 + 1 + 2 * out->plan.n_aggs) * 3;
	return bytes * 1.25;
}

/* The steps run in this order: rel_column() numbers the descriptor's columns in the order they are first met. */
static bool
gpuexec_match_plan(PlannerInfo *root, RelOptInfo *input_rel, RelOptInfo *output_rel, GpuExecState *out, GpuPlanMatch *m)
{
	Query	   *parse = root->parse;
	Path	   *in = input_rel->cheapest_total_path;

	if (parse->groupingSets || parse->havingQual || parse->hasWindowFuncs || parse->hasTargetSRFs || in == NULL)
		return false;
	out->plan.outer_key_col = -1;
	if (!match_input(root, input_rel, out, m) || !match_group_by(root, out, m) || !within_library_limits(out, m) ||
		!match_aggregates(parse, out, m) || !state_words_fit(root, &out->outer, &out->plan))
		return false;
	m->groups = output_rel->rows > 0 ? output_rel->rows : 1;
	out->plan.est_groups = (int64) m->groups;
	if (m->distinct_arg && !size_distinct_pairs(root, in->rows, out, m))
		return false;
	m->bytes = hbm_bytes(out, m);
	return true;
}

static void
gpuexec_upper_paths_hook(PlannerInfo *root, UpperRelationKind stage, RelOptInfo *input_rel, RelOptInfo *output_rel)
{
	GpuExecState desc;
	GpuPlanMatch m = {0};
	Query	   *parse = root->parse;
	List	   *scan_exprs = NIL;
	ListCell   *lc;

	if (prev_upper_paths_hook)
		prev_upper_paths_hook(root, stage, input_rel, output_rel);
	if (!gpuexec_enabled || stage != UPPERREL_GROUP_AGG)
		return;
	memset(&desc, 0, sizeof(desc));
	if (!gpuexec_match_plan(root, input_rel, output_rel, &desc, &m))
		return;					/* decline: the CPU paths stay as they are */
	/* capacity (the analogue of ExecChooseHashTableSize deciding on batches, nodeHash.c:864): there is
	 * no spill path on the device, so a plan that would not fit is left to the CPU executor */
	if (m.bytes > (double) gpuexec_hbm_limit_mb * 1024.0 * 1024.0)
		return;
	{
		CustomPath *cpath = makeNode(CustomPath);
		Path	   *cheapest_in = input_rel->cheapest_total_path;
		bool		pushdown = grouping_covers_distribution(parse, cheapest_in->distribution);
		PathTarget *scan_target;

		desc.partial = !pushdown;
		/* a count(DISTINCT) result has no partial state, and distinct counts do not add across datanodes */
		if (desc.partial && m.pairs > 0)
			return;
		/* the scan tuple: GROUP BY expressions, then the aggregates (partial Aggrefs in two-phase mode) */
		scan_target = create_empty_pathtarget();
		foreach(lc, parse->groupClause)
		{
			SortGroupClause *sgc = (SortGroupClause *) lfirst(lc);
			TargetEntry *tle = get_sortgroupclause_tle(sgc, parse->targetList);

			scan_exprs = lappend(scan_exprs, tle->expr);
			add_column_to_pathtarget(scan_target, tle->expr, sgc->tleSortGroupRef);
		}
		foreach(lc, m.agg_refs)
		{
			Aggref	   *a = (Aggref *) lfirst(lc);

			if (desc.partial)
			{
				a = (Aggref *) copyObject(a);
				mark_partial_aggref(a, AGGSPLIT_INITIAL_SERIAL);
			}
			scan_exprs = lappend(scan_exprs, a);
			if (desc.partial)
				add_column_to_pathtarget(scan_target, (Expr *) a, 0);
		}

		cpath->path.pathtype = T_CustomScan;
		cpath->path.parent = output_rel;
		cpath->path.pathtarget = desc.partial ? scan_target : output_rel->reltarget;
		cpath->path.param_info = NULL;
		cpath->path.parallel_aware = false;
		cpath->path.parallel_safe = false;	/* the GPU replaces intra-node parallelism */
		cpath->path.rows = m.groups;
		/* the aggregate runs where the data lives */
		cpath->path.distribution = cheapest_in->distribution;
		/* priced like the reference's own paths — per datanode, in units of a sequential page fetch — so that add_path()
		 * compares like with like: the disk term of cost_seqscan (costsize.c:359), then per page on the host instead of
		 * per tuple, PCIe, HBM passes and a fixed start-up price (gpuexec_cost.h) */
		{
			gpuexec_cost_params cp;
			double		num_nodes = path_count_datanodes(cheapest_in);
			Cost		startup,
						total;

			cp.seq_page_cost = seq_page_cost;
			cp.cpu_tuple_cost = cpu_tuple_cost;
			cp.cost_unit_us = gpuexec_cost_unit_us;
			cp.host_page_us = gpuexec_host_page_us;
			cp.pcie_gb_s = gpuexec_pcie_gb_s;
			cp.hbm_gb_s = gpuexec_hbm_gb_s;
			cp.startup_us = gpuexec_startup_us;
			if (num_nodes < 1)
				num_nodes = 1;
			gpuexec_path_cost(&cp, m.pages / num_nodes, m.bytes / num_nodes, m.groups, &startup, &total);
			cpath->path.startup_cost = startup;
			cpath->path.total_cost = total;
		}
		cpath->flags = 0;
		cpath->custom_paths = NIL;
		cpath->custom_private = list_make2(gpuexec_serialise(&desc), scan_exprs);
		cpath->methods = &gpuexec_path_methods;
		if (pushdown)
			add_path(output_rel, &cpath->path);
		else
		{
			/* Partial GpuExecHashAgg -> Distribute results by the group key -> Finalize HashAggregate:
			 * the shape of planner.c:9045-9075 with our node in place of the partial AggPath
			 * (xc_groupby.out:193-205).  Aggregates whose transition state cannot travel decline. */
			AggClauseCosts final_costs;
			Path	   *remote;

			MemSet(&final_costs, 0, sizeof(final_costs));
			get_agg_clause_costs(root, (Node *) output_rel->reltarget->exprs, AGGSPLIT_FINAL_DESERIAL, &final_costs);
			if (final_costs.hasNonPartial || final_costs.hasNonSerial)
				return;
			remote = create_redistribute_grouping_path(root, parse, &cpath->path);
			if (remote == NULL)
				return;
			add_path(output_rel, (Path *)
					 create_agg_path(root, output_rel, remote, output_rel->reltarget,
									 parse->groupClause ? AGG_HASHED : AGG_PLAIN, AGGSPLIT_FINAL_DESERIAL,
									 parse->groupClause, NIL, &final_costs, m.groups));
		}
	}
}

void
_PG_init(void)
{
	DefineCustomBoolVariable("gpuexec.enabled", "Offer GPU paths for scan/join/aggregate sub-plans.", NULL,
							 &gpuexec_enabled, true, PGC_USERSET, 0, NULL, NULL, NULL);
	DefineCustomIntVariable("gpuexec.device", "CUDA device ordinal used by this datanode.", NULL,
							&gpuexec_device, 0, 0, 63, PGC_BACKEND, 0, NULL, NULL, NULL);
	DefineCustomIntVariable("gpuexec.pool_reserve_mb", "HBM (MB) mapped into the GPU memory pool when a backend first uses the GPU (0 = grow on demand).", NULL,
							&gpuexec_pool_reserve_mb, 0, 0, 1024 * 1024, PGC_BACKEND, 0, NULL, NULL, NULL);
	DefineCustomIntVariable("gpuexec.hbm_limit_mb", "Decline plans whose staged columns and join table are estimated above this many MB of HBM.", NULL,
							&gpuexec_hbm_limit_mb, 64 * 1024, 64, 1024 * 1024, PGC_USERSET, 0, NULL, NULL, NULL);
	DefineCustomRealVariable("gpuexec.cost_unit_us", "Microseconds one unit of planner cost (a sequential page fetch) stands for.", NULL,
							 &gpuexec_cost_unit_us, 10.0, 0.01, 1e6, PGC_USERSET, 0, NULL, NULL, NULL);
	DefineCustomRealVariable("gpuexec.host_page_us", "Host microseconds per heap page on the loader's path (visibility pass + copy into the pinned ring).", NULL,
							 &gpuexec_host_page_us, 1.5, 0.0, 1e6, PGC_USERSET, 0, NULL, NULL, NULL);
	DefineCustomRealVariable("gpuexec.pcie_gb_s", "Host-to-device copy rate of pinned memory in GB/s.", NULL,
							 &gpuexec_pcie_gb_s, 50.0, 0.1, 1e4, PGC_USERSET, 0, NULL, NULL, NULL);
	DefineCustomRealVariable("gpuexec.hbm_gb_s", "What the kernels sustain over the staged columns in GB/s.", NULL,
							 &gpuexec_hbm_gb_s, 3000.0, 1.0, 1e5, PGC_USERSET, 0, NULL, NULL, NULL);
	DefineCustomRealVariable("gpuexec.startup_us", "Fixed price of one GPU sub-plan in microseconds (plan compile, launches, result fetch).", NULL,
							 &gpuexec_startup_us, 1500.0, 0.0, 1e9, PGC_USERSET, 0, NULL, NULL, NULL);
	RegisterCustomScanMethods(&gpuexec_scan_methods);
	RegisterResourceReleaseCallback(gpuexec_resowner_callback, NULL);
	prev_upper_paths_hook = create_upper_paths_hook;
	create_upper_paths_hook = gpuexec_upper_paths_hook;
}
