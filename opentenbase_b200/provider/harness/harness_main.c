/*
 * harness_main.c — a stub-linked fake backend that EXECUTES the CustomScan provider.
 *
 * TEST INFRASTRUCTURE (tests/test_provider_harness.py).  The provider's source is included
 * verbatim (so its static functions are reachable); everything a live backend would supply
 * is faked here, the same way the reference's own unit tests link backend code against
 * stubs (src/backend/unittest/backend/stub/):
 *   - memory: palloc -> malloc; ereport(ERROR) prints and exits 3 (no PG_TRY is needed: the
 *     provider keeps no host resources across a longjmp);
 *   - relations: heap-page images read from a case file (built by the oracle's page writer,
 *     whose bytes are pinned against the reference's heaptuple.o / bufpage.o);
 *     heap_beginscan / heapgetpage / heap_endscan walk them with the REFERENCE's page and
 *     tuple macros (bufpage.h, itemid.h, htup_details.h) and fill rs_vistuples exactly as
 *     heapgetpage() does for an all-committed snapshot; BufferGetPage() resolves through the
 *     real macro (local-buffer branch of BufferGetBlock);
 *   - executor: what ExecInitCustomScan does around the provider (nodeCustom.c:32-115) is
 *     restated in main(): CreateCustomScanState, a scan slot with the scan tuple's
 *     descriptor, BeginCustomScan, ExecCustomScan until TupIsNull, EndCustomScan;
 *   - lists and Value nodes are the reference's own object code (nodes/list.c, nodes/value.c,
 *     compiled from where they lie).
 * libgpuexec.so is the real thing: executing a case needs a GPU.  Two modes need none (CPU tests):
 *   --ship-only <case file>   the plan descriptor as custom_private Value nodes, written as nodeToString() writes them and read
 *                             back by the reference's own nodes/read.c (tests/test_provider_ship_cpu.py)
 *   --plan <scenario file>    a hand-built Query through gpuexec_upper_paths_hook + PlanCustomPath; the planner-side helpers
 *                             are small restatements of the reference's (tests/test_provider_planner_cpu.py)
 *
 * usage: gpuexec_harness <case file>     -> one text line per result row on stdout
 */
#include "../gpuexec_provider.c"

#include "storage/itemid.h"
#include "storage/bufpage.h"

#include <stdio.h>
#include <stdlib.h>

#ifndef FLOAT8ARRAYOID
#define FLOAT8ARRAYOID 1022		/* _float8, catalog/pg_type.h */
#endif

/* ------------------------------------------------------------ fake backend */
void *palloc_internal(Size size, const char *file, int line) { return malloc(size ? size : 1); }
void *palloc0_internal(Size size, const char *file, int line) { return calloc(1, size ? size : 1); }
void *palloc_extended_internal(Size size, int flags, const char *file, int line) { return calloc(1, size ? size : 1); }
void *repallocInternal(void *p, Size size, const char *file, int line) { return realloc(p, size); }
void pfree(void *p) { free(p); }
void *MemoryContextAllocInternal(MemoryContext c, Size size, const char *file, int line) { return malloc(size ? size : 1); }
void *MemoryContextAllocZeroInternal(MemoryContext c, Size size, const char *file, int line) { return calloc(1, size ? size : 1); }
void *MemoryContextAllocZeroAlignedIternal(MemoryContext c, Size size, const char *file, int line) { return calloc(1, size ? size : 1); }
char *pstrdup(const char *in) { return strdup(in); }
void MemoryContextReset(MemoryContext c) { }
__thread MemoryContext CurrentMemoryContext = NULL;
__thread ResourceOwner CurrentResourceOwner = NULL;
volatile bool InterruptPending = false;
void ProcessInterrupts(void) { }
void pg_qsort(void *base, size_t nel, size_t elsize, int (*cmp) (const void *, const void *)) { qsort(base, nel, elsize, cmp); }
__thread bool am_sub_thread = false;
void CheckSubThreadContextInternal(MemoryContext context, const char *func) { }
bool enable_resource_queue = false;
void ResQUsageBackoffPriority(void) { }
char *BufferBlocks = NULL;
Block *LocalBufferBlockPointers = NULL;
bool g_enable_cls = false, g_enable_data_mask = false, enable_fga = false;
create_upper_paths_hook_type create_upper_paths_hook = NULL;

static char last_msg[1024];
bool errstart(int elevel, const char *filename, int lineno, const char *funcname, const char *domain)
{ return elevel >= ERROR; }
static ResourceReleaseCallback release_cb;
/* the transaction abort an ERROR causes: the resource owner's release callbacks run (they free every library handle of
 * the query), then the context goes away */
void errfinish(int dummy,...)
{
	fprintf(stderr, "harness: ereport(ERROR): %s\n", last_msg);
	if (release_cb)
		release_cb(RESOURCE_RELEASE_AFTER_LOCKS, false, true, NULL);
	if (backend_ctx)
		gx_shutdown(backend_ctx);
	exit(3);
}
int errmsg(const char *fmt,...) { va_list ap; va_start(ap, fmt); vsnprintf(last_msg, sizeof(last_msg), fmt, ap); va_end(ap); return 0; }
int errmsg_internal(const char *fmt,...) { return 0; }
int errcode(int sqlerrcode) { return 0; }
int errdetail(const char *fmt,...) { return 0; }
void elog_start(const char *filename, int lineno, const char *funcname) { }
void elog_finish(int elevel, const char *fmt,...) { if (elevel >= ERROR) { fprintf(stderr, "harness: elog(ERROR): %s\n", fmt); exit(3); } }
void ExceptionalCondition(const char *a, const char *b, const char *c, int d) { fprintf(stderr, "harness: Assert(%s) at %s:%d\n", a, c, d); abort(); }

/* planner-side entry points.  The executor test never reaches them; `--plan` mode does, so they are small working
 * restatements of what the reference does (file:line each), enough for a hand-built Query. */
#define NOT_REACHED(name) do { fprintf(stderr, "harness: %s() must not be reached\n", name); abort(); } while (0)
static List *added_paths = NIL;
static CustomPath *last_custom_path;
void add_path(RelOptInfo *r, Path *p) { added_paths = lappend(added_paths, p); if (IsA(p, CustomPath)) last_custom_path = (CustomPath *) p; }		/* pathnode.c:423: here, just remember it */
/* pathnode.c:3178 create_agg_path: only what the test inspects */
AggPath *create_agg_path(PlannerInfo *root, RelOptInfo *rel, Path *subpath, PathTarget *target, AggStrategy s, AggSplit sp, List *g, List *q,
						 const AggClauseCosts *c, double n)
{
	AggPath    *ap = makeNode(AggPath);

	ap->path.pathtype = T_Agg; ap->path.parent = rel; ap->path.pathtarget = target; ap->path.rows = n;
	ap->subpath = subpath; ap->aggstrategy = s; ap->aggsplit = sp; ap->groupClause = g; ap->numGroups = n;
	ap->path.startup_cost = subpath->total_cost; ap->path.total_cost = subpath->total_cost + cpu_tuple_cost * n;
	return ap;
}
/* tlist.c:create_empty_pathtarget / add_column_to_pathtarget (optimizer/util/tlist.c:608,647) */
PathTarget *create_empty_pathtarget(void) { return makeNode(PathTarget); }
void add_column_to_pathtarget(PathTarget *t, Expr *e, Index r)
{
	t->exprs = lappend(t->exprs, e);
	if (r)
	{
		int			n = list_length(t->exprs);

		t->sortgrouprefs = (Index *) realloc(t->sortgrouprefs, n * sizeof(Index));
		memset(t->sortgrouprefs, 0, (n - 1) * sizeof(Index));	/* good enough for a fresh target filled front to back */
		t->sortgrouprefs[n - 1] = r;
	}
}
/* the reference wraps the partial path in a RemoteSubplan distributed by the group key (pathnode.c:6091) */
Path *create_redistribute_grouping_path(PlannerInfo *root, Query *parse, Path *path)
{
	Path	   *p = makeNode(Path);

	if (IsA(path, CustomPath)) last_custom_path = (CustomPath *) path;
	p->pathtype = T_RemoteSubplan; p->parent = path->parent; p->pathtarget = path->pathtarget; p->rows = path->rows;
	p->startup_cost = path->startup_cost; p->total_cost = path->total_cost + 1.0;
	return p;
}
void get_agg_clause_costs(PlannerInfo *root, Node *clause, AggSplit s, AggClauseCosts *c) { }	/* all supported aggregates are partial + serial-free */
/* tlist.c:get_sortgroupref_tle (optimizer/util/tlist.c:367) */
TargetEntry *get_sortgroupclause_tle(SortGroupClause *s, List *t)
{
	ListCell   *l;

	foreach(l, t)
		if (((TargetEntry *) lfirst(l))->ressortgroupref == s->tleSortGroupRef)
			return (TargetEntry *) lfirst(l);
	fprintf(stderr, "harness: ORDER/GROUP BY expression not found in targetlist\n"); abort();
}
/* planner.c:mark_partial_aggref (optimizer/plan/planner.c): the partial aggregate returns its transition type */
void mark_partial_aggref(Aggref *a, AggSplit s)
{
	a->aggsplit = s;
	if (DO_AGGSPLIT_SKIPFINAL(s))
		a->aggtype = (DO_AGGSPLIT_SERIALIZE(s) && a->aggtranstype == INTERNALOID) ? BYTEAOID : a->aggtranstype;
}
/* makefuncs.c:237 */
TargetEntry *makeTargetEntry(Expr *e, AttrNumber r, char *n, bool j)
{
	TargetEntry *t = makeNode(TargetEntry);

	t->expr = e; t->resno = r; t->resname = n; t->resjunk = j;
	return t;
}
/* copyObject / equal for the handful of node types a hand-built Query holds (nodes/copyfuncs.c, equalfuncs.c): shallow copies -
 * the test only looks at the result */
static size_t fake_node_size(const void *o)
{
	switch (nodeTag(o))
	{
		case T_Var: return sizeof(Var);
		case T_Const: return sizeof(Const);
		case T_Aggref: return sizeof(Aggref);
		case T_OpExpr: return sizeof(OpExpr);
		case T_TargetEntry: return sizeof(TargetEntry);
		case T_RelabelType: return sizeof(RelabelType);
		default: fprintf(stderr, "harness: copyObject of node type %d\n", (int) nodeTag(o)); abort();
	}
}
void *copyObjectImpl(const void *o)
{
	void	   *c;

	if (o == NULL) return NULL;
	if (IsA(o, List)) return list_copy((const List *) o);
	c = malloc(fake_node_size(o));
	memcpy(c, o, fake_node_size(o));
	return c;
}
bool equal(const void *a, const void *b)
{
	if (a == b) return true;
	if (a == NULL || b == NULL || nodeTag(a) != nodeTag(b)) return false;
	if (IsA(a, Var))
	{
		const Var  *x = (const Var *) a, *y = (const Var *) b;

		return x->varno == y->varno && x->varattno == y->varattno && x->vartype == y->vartype && x->vartypmod == y->vartypmod && x->varlevelsup == y->varlevelsup;
	}
	return false;
}
static bool fake_cls_policy = false;		/* --plan scenario "protected": the relation has a CLS policy */
bool cls_check_table_has_policy(Oid r) { return fake_cls_policy; }
bool datamask_check_table_has_datamask(Oid r) { return false; }
bool get_audit_fga_quals(Oid rel, char *cmd, List *tl, List **out) { return false; }
void DefineCustomBoolVariable(const char *n, const char *s, const char *l, bool *v, bool b, GucContext c, int f, GucBoolCheckHook a, GucBoolAssignHook g, GucShowHook h) { }
void DefineCustomRealVariable(const char *n, const char *s, const char *l, double *v, double b, double mn, double mx, GucContext c, int f, GucRealCheckHook a, GucRealAssignHook g, GucShowHook h) { }
double		seq_page_cost = 1.0, cpu_tuple_cost = 0.01;		/* costsize.c:100-104 */
static double fake_datanodes = 1;
double path_count_datanodes(Path *p) { return fake_datanodes; }
/* selfuncs.c:3349 estimates from column statistics the harness does not have: the scenario's "pairs N" line stands in for
 * them (count(DISTINCT) asks for the GROUP BY columns plus its argument), else every input row is its own group */
static double fake_pairs = 0;
double estimate_num_groups(PlannerInfo *root, List *groupExprs, double input_rows, List **pgset) { return fake_pairs > 0 ? fake_pairs : input_rows; }
void DefineCustomIntVariable(const char *n, const char *s, const char *l, int *v, int b, int mn, int mx, GucContext c, int f, GucIntCheckHook a, GucIntAssignHook g, GucShowHook h) { }
static const CustomScanMethods *registered_methods = NULL;
void RegisterCustomScanMethods(const CustomScanMethods *m) { registered_methods = m; }
static ResourceReleaseCallback release_cb = NULL;
void RegisterResourceReleaseCallback(ResourceReleaseCallback cb, void *arg) { release_cb = cb; }
void ExplainPropertyText(const char *q, const char *v, ExplainState *es) { fprintf(stderr, "explain: %s: %s\n", q, v); }
void ExplainPropertyFloat(const char *q, const char *u, double v, int nd, ExplainState *es) { fprintf(stderr, "explain: %s: %.3f %s\n", q, v, u ? u : ""); }
void ExplainPropertyInteger(const char *q, const char *u, int64 v, ExplainState *es) { fprintf(stderr, "explain: %s: %ld\n", q, (long) v); }

/* text/array constructors the executor side uses for by-reference datums */
text *cstring_to_text_with_len(const char *s, int len)
{
	text	   *t = (text *) malloc(len + VARHDRSZ);

	SET_VARSIZE(t, len + VARHDRSZ);
	memcpy(VARDATA(t), s, len);
	return t;
}
/* construct_array for a 1-D array of pass-by-value float8 without NULLs (utils/adt/arrayfuncs.c:3306) */
ArrayType *construct_array(Datum *elems, int nelems, Oid elmtype, int elmlen, bool elmbyval, char elmalign)
{
	Size		nbytes = ARR_OVERHEAD_NONULLS(1) + (Size) nelems * elmlen;
	ArrayType  *a = (ArrayType *) calloc(1, nbytes);
	int			i;

	if (elmtype != FLOAT8OID || elmlen != 8 || !elmbyval) { fprintf(stderr, "harness: construct_array: only float8[]\n"); abort(); }
	SET_VARSIZE(a, nbytes);
	a->ndim = 1; a->dataoffset = 0; a->elemtype = elmtype;
	ARR_DIMS(a)[0] = nelems; ARR_LBOUND(a)[0] = 1;
	for (i = 0; i < nelems; i++)
		memcpy(ARR_DATA_PTR(a) + (Size) i * 8, &elems[i], 8);
	return a;
}

/* ------------------------------------------------------------ fake relations */
typedef struct FakeRel
{
	RelationData rd;
	FormData_pg_class cls;
	int64		npages;
	char	   *pages;
	int			buf_base;		/* index of page 0 in LocalBufferBlockPointers */
} FakeRel;
static FakeRel fake_rels[GX_MAX_JOINS + 1];		/* the outer relation and one per join of a chain */
static int	n_fake_rels = 0;

Relation ExecOpenScanRelation(EState *estate, Index scanrelid, int eflags)
{
	if ((int) scanrelid < 1 || (int) scanrelid > n_fake_rels) { fprintf(stderr, "harness: no relation with rti %u\n", scanrelid); exit(3); }
	return &fake_rels[scanrelid - 1].rd;
}
void ExecCloseScanRelation(Relation r) { }

HeapScanDesc heap_beginscan(Relation relation, Snapshot snapshot, int nkeys, ScanKey key)
{
	HeapScanDesc scan = (HeapScanDesc) calloc(1, sizeof(HeapScanDescData));
	FakeRel    *fr = (FakeRel *) relation;

	scan->rs_rd = relation;
	scan->rs_snapshot = snapshot;
	scan->rs_nblocks = (BlockNumber) fr->npages;
	scan->rs_cbuf = InvalidBuffer;
	scan->rs_pageatatime = true;
	return scan;
}
void heap_endscan(HeapScanDesc scan) { free(scan); }
void LockBuffer(Buffer b, int mode) { }

/* heapgetpage (access/heap/heapam.c:388-513) for a snapshot that sees every committed insert and
 * no in-progress transaction: a tuple is visible iff xmin is committed and xmax is invalid */
void heapgetpage(HeapScanDesc scan, BlockNumber page)
{
	FakeRel    *fr = (FakeRel *) scan->rs_rd;
	Page		dp;
	int			lines,
				ntup = 0;
	OffsetNumber lineoff;

	scan->rs_cbuf = -(fr->buf_base + (int) page + 1);		/* a "local buffer": BufferGetBlock's negative branch */
	scan->rs_cblock = page;
	dp = BufferGetPage(scan->rs_cbuf);
	lines = PageGetMaxOffsetNumber(dp);
	for (lineoff = FirstOffsetNumber; lineoff <= lines; lineoff++)
	{
		ItemId		lpp = PageGetItemId(dp, lineoff);

		if (ItemIdIsNormal(lpp))
		{
			HeapTupleHeader th = (HeapTupleHeader) PageGetItem(dp, lpp);

			if ((th->t_infomask & HEAP_XMIN_COMMITTED) && (th->t_infomask & HEAP_XMAX_INVALID))
				scan->rs_vistuples[ntup++] = lineoff;
		}
	}
	scan->rs_ntuples = ntup;
}

/* ------------------------------------------------------------ slots (executor/execTuples.c:612,679) */
TupleTableSlot *ExecClearTuple(TupleTableSlot *slot)
{
	slot->tts_tuple = NULL;
	slot->tts_flags |= TTS_FLAG_EMPTY;
	slot->tts_nvalid = 0;
	return slot;
}
TupleTableSlot *ExecStoreVirtualTuple(TupleTableSlot *slot)
{
	slot->tts_flags &= ~TTS_FLAG_EMPTY;
	slot->tts_nvalid = slot->tts_tupleDescriptor->natts;
	return slot;
}

/* ------------------------------------------------------------ case file */
static void rd(FILE *f, void *p, size_t n) { if (fread(p, 1, n, f) != n) { fprintf(stderr, "harness: short case file\n"); exit(2); } }
static int32 rd32(FILE *f) { int32 v; rd(f, &v, 4); return v; }
static int64 rd64(FILE *f) { int64 v; rd(f, &v, 8); return v; }

static void read_relinfo(FILE *f, GpuRelInfo *r)
{
	int			i;

	r->rti = (Index) rd32(f);
	r->ncols = rd32(f);
	for (i = 0; i < r->ncols; i++) { r->attnums[i] = rd32(f); r->types[i] = rd32(f); }
}

/* read.c calls this for '{' nodes; custom_private only ever holds Value nodes */
Node *parseNodeString(void) { NOT_REACHED("parseNodeString"); return NULL; }

/* What nodeToString() writes for a List of Value nodes: _outList (nodes/outfuncs.c:443-477) around _outValue (:5103-5117:
 * T_Integer as %d, T_Float as its string, unquoted). */
static char *
out_value_list(List *l)
{
	size_t		cap = 64 + (size_t) list_length(l) * 40, n = 0;
	char	   *buf = (char *) malloc(cap);
	ListCell   *lc;

	buf[n++] = '(';
	foreach(lc, l)
	{
		Value	   *v = (Value *) lfirst(lc);

		if (IsA(v, Integer))
			n += snprintf(buf + n, cap - n, "%d", (int) intVal(v));
		else if (IsA(v, Float))
			n += snprintf(buf + n, cap - n, "%s", strVal(v));
		else
			NOT_REACHED("out_value_list: node type");
		if (lnext(lc))
			buf[n++] = ' ';
	}
	buf[n++] = ')';
	buf[n] = 0;
	return buf;
}

/* the first of n quals whose constants did not come back bit for bit, or -1 */
static int
changed_pred(const gx_pred *sent, const gx_pred *got, int n)
{
	int			i;

	for (i = 0; i < n; i++)
		if (sent[i].ival != got[i].ival || memcmp(&sent[i].fval, &got[i].fval, 8) != 0)
			return i;
	return -1;
}

static char *out_value_list(List *l);
/* ------------------------------------------------------------ --plan: a hand-built Query through the planner hook
 * The scenario file (written by tests/test_provider_planner_cpu.py) describes base relations, the input path (SeqScan or
 * a left-deep chain of HashJoins over SeqScans), quals, GROUP BY, the target list and the input's distribution; this builds the PlannerInfo /
 * Query / RelOptInfo / Path nodes the hook reads, calls gpuexec_upper_paths_hook and PlanCustomPath, and prints what
 * came out: the path shape and costs, the descriptor as it would travel, and the scan tuple. */
typedef struct PlanRel { RelOptInfo *rel; RangeTblEntry *rte; int ncols; Oid types[GX_MAX_COLS * 2]; int32 typmods[GX_MAX_COLS * 2]; bool notnull[GX_MAX_COLS * 2]; } PlanRel;
#define PLAN_MAX_RELS (GX_MAX_JOINS + 2)			/* a chain one join longer than the provider takes */
static PlanRel plan_rels[PLAN_MAX_RELS + 1];

/* pg_attribute through the syscache, for column_is_not_null(): the scenario's "rel" line marks NOT NULL columns with a '!' */
static struct { HeapTupleData tup; HeapTupleHeaderData hdr; char pad[64]; FormData_pg_attribute att; } fake_att_tuple;
HeapTuple SearchSysCache2(int cacheId, Datum key1, Datum key2)
{
	int			r, a = DatumGetInt16(key2);

	if (cacheId != ATTNUM) NOT_REACHED("SearchSysCache2 of another cache");
	for (r = 1; r <= PLAN_MAX_RELS; r++)
		if (plan_rels[r].rte && plan_rels[r].rte->relid == DatumGetObjectId(key1) && a >= 1 && a <= plan_rels[r].ncols)
		{
			memset(&fake_att_tuple, 0, sizeof(fake_att_tuple));
			fake_att_tuple.hdr.t_hoff = (uint8) ((char *) &fake_att_tuple.att - (char *) &fake_att_tuple.hdr);
			fake_att_tuple.tup.t_data = &fake_att_tuple.hdr;
			fake_att_tuple.att.attnotnull = plan_rels[r].notnull[a - 1];
			fake_att_tuple.att.attnum = a;
			return &fake_att_tuple.tup;
		}
	return NULL;
}
void ReleaseSysCache(HeapTuple tuple) { }

static bool type_by_name(const char *n, Oid *t, int32 *m)
{
	*m = -1;
	if (!strcmp(n, "int8")) *t = INT8OID; else if (!strcmp(n, "int4")) *t = INT4OID; else if (!strcmp(n, "date")) *t = DATEOID;
	else if (!strcmp(n, "float8")) *t = FLOAT8OID; else if (!strcmp(n, "char")) *t = CHAROID; else if (!strcmp(n, "text")) *t = TEXTOID;
	else if (!strcmp(n, "numeric")) *t = NUMERICOID;
	else if (!strcmp(n, "bpchar1")) { *t = BPCHAROID; *m = VARHDRSZ + 1; } else if (!strcmp(n, "bpchar3")) { *t = BPCHAROID; *m = VARHDRSZ + 3; }
	else return false;
	return true;
}
static Var *plan_var(int rti, int att)
{
	Var		   *v = makeNode(Var);

	if (rti < 1 || rti > PLAN_MAX_RELS || att < 1 || att > plan_rels[rti].ncols) { fprintf(stderr, "harness: no column %d.%d\n", rti, att); exit(2); }
	v->varno = rti; v->varattno = att; v->vartype = plan_rels[rti].types[att - 1]; v->vartypmod = plan_rels[rti].typmods[att - 1];
	v->varnoold = rti; v->varoattno = att;
	return v;
}
static Const *plan_const(Oid t, const char *val)
{
	Const	   *c = makeNode(Const);

	c->consttype = t; c->consttypmod = -1; c->constlen = 8; c->constbyval = true;
	if (!strcmp(val, "null")) { c->constisnull = true; return c; }
	switch (t)
	{
		case INT8OID: c->constvalue = Int64GetDatum(strtoll(val, NULL, 10)); break;
		case INT4OID: case DATEOID: c->constvalue = Int32GetDatum((int32) strtol(val, NULL, 10)); break;
		case FLOAT8OID: c->constvalue = Float8GetDatum(strtod(val, NULL)); break;
		case CHAROID: c->constvalue = CharGetDatum(val[0]); break;
		default: c->constvalue = PointerGetDatum(cstring_to_text_with_len(val, (int) strlen(val))); c->constbyval = false; c->constlen = -1; break;
	}
	return c;
}
static Oid fn_by_name(const char *n)
{
	static const struct { const char *n; Oid f; } tab[] = {
		{"int4lt", F_INT4LT}, {"int4le", F_INT4LE}, {"int4eq", F_INT4EQ}, {"int4ge", F_INT4GE}, {"int4gt", F_INT4GT}, {"int4ne", F_INT4NE},
		{"int8lt", F_INT8LT}, {"int8le", F_INT8LE}, {"int8eq", F_INT8EQ}, {"int8ge", F_INT8GE}, {"int8gt", F_INT8GT}, {"int8ne", F_INT8NE},
		{"date_lt", F_DATE_LT}, {"date_le", F_DATE_LE}, {"date_eq", F_DATE_EQ}, {"date_ge", F_DATE_GE}, {"date_gt", F_DATE_GT}, {"date_ne", F_DATE_NE},
		{"float8lt", F_FLOAT8LT}, {"float8le", F_FLOAT8LE}, {"float8eq", F_FLOAT8EQ}, {"float8ge", F_FLOAT8GE}, {"float8gt", F_FLOAT8GT}, {"float8ne", F_FLOAT8NE},
		{"chareq", F_CHAREQ}, {"charlt", F_CHARLT}, {"bpchareq", F_BPCHAREQ}, {"bpcharne", F_BPCHARNE}, {"int84lt", F_INT84LT}, {"texteq", F_TEXTEQ},
	};
	int			i;

	for (i = 0; i < (int) lengthof(tab); i++) if (!strcmp(tab[i].n, n)) return tab[i].f;
	fprintf(stderr, "harness: unknown function %s\n", n); exit(2);
}
static Expr *plan_op(Oid fn, Node *l, Node *r) { OpExpr *o = makeNode(OpExpr); o->opfuncid = fn; o->args = list_make2(l, r); return (Expr *) o; }
/* postfix tokens: v<rti>.<att>  k<float>  + - *  */
static Node *plan_expr(char *toks)
{
	Node	   *stack[16];
	int			sp = 0;
	char	   *t;

	for (t = strtok(toks, " \n"); t; t = strtok(NULL, " \n"))
	{
		if (t[0] == 'v') { int r, a; sscanf(t + 1, "%d.%d", &r, &a); stack[sp++] = (Node *) plan_var(r, a); }
		else if (t[0] == 'k') stack[sp++] = (Node *) plan_const(FLOAT8OID, t + 1);
		else { Node *y = stack[--sp], *x = stack[--sp]; stack[sp++] = (Node *) plan_op(t[0] == '+' ? F_FLOAT8PL : t[0] == '-' ? F_FLOAT8MI : t[0] == '*' ? F_FLOAT8MUL : F_FLOAT8DIV, x, y); }
	}
	return sp == 1 ? stack[0] : NULL;
}
static int plan_main(const char *path)
{
	FILE	   *f = fopen(path, "r");
	char		line[1024];
	PlannerInfo *root = makeNode(PlannerInfo);
	Query	   *parse = makeNode(Query);
	RelOptInfo *input_rel = NULL, *output_rel = makeNode(RelOptInfo);
	Distribution *dist = NULL;
	List	   *groups = NIL;		/* Var per GROUP BY column */
	ListCell   *lc;
	int			i;

	if (!f) { perror(path); return 2; }
	root->parse = parse;
	root->simple_rel_array_size = PLAN_MAX_RELS + 1;
	root->simple_rte_array = (RangeTblEntry **) calloc(PLAN_MAX_RELS + 1, sizeof(RangeTblEntry *));
	output_rel->reltarget = makeNode(PathTarget);
	output_rel->rows = 100;
	_PG_init();
	while (fgets(line, sizeof(line), f))
	{
		char		w[64], ty[16][16];
		int			r, a, r2, a2, n, u;
		double		t, pg;

		if (line[0] == '#' || line[0] == '\n') continue;
		if (sscanf(line, "rel %d tuples %lf pages %lf cols %n", &r, &t, &pg, &n) == 3)
		{
			if (r < 1 || r > PLAN_MAX_RELS) { fprintf(stderr, "harness: rel %d\n", r); return 2; }
			PlanRel    *pr = &plan_rels[r];
			char	   *tok;

			pr->rel = makeNode(RelOptInfo); pr->rel->relid = r; pr->rel->reloptkind = RELOPT_BASEREL; pr->rel->tuples = t; pr->rel->pages = (BlockNumber) pg; pr->rel->rows = t;
			pr->rte = makeNode(RangeTblEntry); pr->rte->rtekind = RTE_RELATION; pr->rte->relid = 16384 + r;
			root->simple_rte_array[r] = pr->rte;
			for (tok = strtok(line + n, " \n"); tok; tok = strtok(NULL, " \n"))
			{
				size_t		L = strlen(tok);

				pr->notnull[pr->ncols] = L > 0 && tok[L - 1] == '!';
				if (pr->notnull[pr->ncols]) tok[L - 1] = 0;
				if (!type_by_name(tok, &pr->types[pr->ncols], &pr->typmods[pr->ncols])) { fprintf(stderr, "harness: type %s\n", tok); return 2; } else pr->ncols++;
			}
			(void) ty;
		}
		else if (sscanf(line, "scan %d", &r) == 1)
		{
			Path	   *p = makeNode(Path);

			input_rel = plan_rels[r].rel;
			p->pathtype = T_SeqScan; p->parent = input_rel; p->rows = input_rel->tuples; p->total_cost = input_rel->pages + 0.01 * input_rel->tuples;
			input_rel->cheapest_total_path = p;
		}
		else if (sscanf(line, "join %d.%d %d.%d unique %d %63s", &r, &a, &r2, &a2, &u, w) >= 5)
		{
			HashPath   *hp = makeNode(HashPath);
			/* a second "join" line joins the previous join's result: the left-deep chain HashJoin(HashJoin(..), S) */
			bool		chained = input_rel && input_rel->cheapest_total_path && IsA(input_rel->cheapest_total_path, HashPath);
			Path	   *op = chained ? input_rel->cheapest_total_path : makeNode(Path), *ip = makeNode(Path);
			RestrictInfo *ri = makeNode(RestrictInfo);
			Var		   *lv = plan_var(r, a), *rv = plan_var(r2, a2);
			bool		remote = strstr(line, "remote_inner") != NULL, swap = strstr(line, "swapped") != NULL;

			if (!chained) { op->pathtype = T_SeqScan; op->parent = plan_rels[r].rel; op->rows = op->parent->tuples; op->total_cost = op->parent->pages + 0.01 * op->rows; }
			ip->pathtype = remote ? T_RemoteSubplan : T_SeqScan; ip->parent = plan_rels[r2].rel; ip->rows = ip->parent->tuples; ip->total_cost = ip->parent->pages + 0.01 * ip->rows;
			ri->clause = plan_op(lv->vartype == INT8OID ? F_INT8EQ : lv->vartype == INT4OID ? F_INT4EQ : F_TEXTEQ, swap ? (Node *) rv : (Node *) lv, swap ? (Node *) lv : (Node *) rv);
			hp->jpath.path.pathtype = T_HashJoin; hp->jpath.inner_unique = u != 0;
			/* the right forms first: their words contain "semi", "anti" and "right" */
			hp->jpath.jointype = strstr(line, "semi_right") ? JOIN_SEMI_RIGHT : strstr(line, "anti_right") ? JOIN_ANTI_RIGHT :
				strstr(line, "left") ? JOIN_LEFT : strstr(line, "semi") ? JOIN_SEMI : strstr(line, "anti") ? JOIN_ANTI :
				strstr(line, "right") ? JOIN_RIGHT : strstr(line, "full") ? JOIN_FULL : JOIN_INNER;
			hp->jpath.outerjoinpath = op; hp->jpath.innerjoinpath = ip; hp->jpath.joinrestrictinfo = list_make1(ri); hp->path_hashclauses = list_make1(ri);
			if (strstr(line, "extra_clause"))
			{
				/* a second join clause next to the hash clause (a join filter the fused paths do not evaluate) */
				RestrictInfo *ri2 = makeNode(RestrictInfo);

				ri2->clause = ri->clause;
				hp->jpath.joinrestrictinfo = lappend(hp->jpath.joinrestrictinfo, ri2);
			}
			input_rel = makeNode(RelOptInfo); input_rel->reloptkind = RELOPT_JOINREL; input_rel->rows = op->rows;
			hp->jpath.path.parent = input_rel; hp->jpath.path.rows = op->rows; hp->jpath.path.total_cost = op->total_cost + ip->total_cost + 0.02 * op->rows;
			input_rel->cheapest_total_path = &hp->jpath.path;
		}
		else if (sscanf(line, "qual %d %d %63s %15s %n", &r, &a, w, ty[0], &n) == 4)
		{
			RestrictInfo *ri = makeNode(RestrictInfo);
			Oid			ct; int32 cm;
			char		val[128] = "";
			bool		flip = strstr(line + n, " flip") != NULL;

			sscanf(line + n, "%127s", val);
			type_by_name(ty[0], &ct, &cm);
			ri->clause = flip ? plan_op(fn_by_name(w), (Node *) plan_const(ct, val), (Node *) plan_var(r, a)) : plan_op(fn_by_name(w), (Node *) plan_var(r, a), (Node *) plan_const(ct, val));
			plan_rels[r].rel->baserestrictinfo = lappend(plan_rels[r].rel->baserestrictinfo, ri);
		}
		else if (sscanf(line, "group %d.%d", &r, &a) == 2)
			groups = lappend(groups, plan_var(r, a));
		else if (sscanf(line, "target var %d.%d", &r, &a) == 2)
			parse->targetList = lappend(parse->targetList, makeTargetEntry((Expr *) plan_var(r, a), list_length(parse->targetList) + 1, NULL, false));
		else if (sscanf(line, "target agg %63s %n", w, &n) == 1)
		{
			Aggref	   *ag = makeNode(Aggref);
			static const struct { const char *n; Oid fn, ty, tr; } tab[] = {
				{"count_star", 2803, INT8OID, INT8OID}, {"count", 2147, INT8OID, INT8OID}, {"sum_f8", 2111, FLOAT8OID, FLOAT8OID}, {"avg_f8", 2105, FLOAT8OID, FLOAT8ARRAYOID},
				{"min_f8", 2136, FLOAT8OID, FLOAT8OID}, {"max_f8", 2120, FLOAT8OID, FLOAT8OID}, {"sum_i4", 2108, INT8OID, INT8OID}, {"sum_numeric", 2114, NUMERICOID, INTERNALOID},
				{"stddev_f8", 2158, FLOAT8OID, FLOAT8ARRAYOID}, {"stddev_samp_f8", 2716, FLOAT8OID, FLOAT8ARRAYOID},
				{"stddev_pop_f8", 2728, FLOAT8OID, FLOAT8ARRAYOID}, {"variance_f8", 2152, FLOAT8OID, FLOAT8ARRAYOID},
				{"var_samp_f8", 2645, FLOAT8OID, FLOAT8ARRAYOID}, {"var_pop_f8", 2722, FLOAT8OID, FLOAT8ARRAYOID},
				{"stddev_f4", 2157, FLOAT8OID, FLOAT8ARRAYOID}, {"stddev_i8", 2154, NUMERICOID, INTERNALOID},
				{"regr_count", 2818, INT8OID, INT8OID}, {"regr_sxx", 2819, FLOAT8OID, FLOAT8ARRAYOID}, {"regr_syy", 2820, FLOAT8OID, FLOAT8ARRAYOID},
				{"regr_sxy", 2821, FLOAT8OID, FLOAT8ARRAYOID}, {"regr_avgx", 2822, FLOAT8OID, FLOAT8ARRAYOID}, {"regr_avgy", 2823, FLOAT8OID, FLOAT8ARRAYOID},
				{"regr_r2", 2824, FLOAT8OID, FLOAT8ARRAYOID}, {"regr_slope", 2825, FLOAT8OID, FLOAT8ARRAYOID}, {"regr_intercept", 2826, FLOAT8OID, FLOAT8ARRAYOID},
				{"covar_pop", 2827, FLOAT8OID, FLOAT8ARRAYOID}, {"covar_samp", 2828, FLOAT8OID, FLOAT8ARRAYOID}, {"corr", 2829, FLOAT8OID, FLOAT8ARRAYOID},
			};

			for (i = 0; i < (int) lengthof(tab); i++) if (!strcmp(tab[i].n, w)) break;
			if (i == (int) lengthof(tab)) { fprintf(stderr, "harness: aggregate %s\n", w); return 2; }
			ag->aggfnoid = tab[i].fn; ag->aggtype = tab[i].ty; ag->aggtranstype = tab[i].tr; ag->aggsplit = AGGSPLIT_SIMPLE; ag->aggkind = 'n';
			{
				/* "... filter" / "... order" after the arguments: a FILTER clause or an ORDER BY inside the call */
				char	   *kf = strstr(line + n, " filter"), *ko = strstr(line + n, " order");

				if (kf) ag->aggfilter = (Expr *) plan_const(INT4OID, "1");
				if (ko) ag->aggorder = list_make1(makeNode(SortGroupClause));
				if (kf) *kf = '\0';
				if (ko) *ko = '\0';
			}
			if (strstr(line + n, "distinct"))
			{
				/* "target agg count v1.2 distinct": the argument, and one sort clause over it (parse_agg.c transformAggregateCall) */
				*strstr(line + n, "distinct") = '\0';
				ag->aggdistinct = list_make1(makeNode(SortGroupClause));
			}
			if (tab[i].fn == 2803) ag->aggstar = true;
			else if (strstr(line + n, " , "))
			{
				/* "target agg corr Y , X": the two arguments of a binary aggregate, Y first */
				char	   *x = strstr(line + n, " , ");
				Node	   *ey, *ex;

				*x = '\0';
				ey = plan_expr(line + n); ex = plan_expr(x + 3);
				if (!ey || !ex) { fprintf(stderr, "harness: bad expression\n"); return 2; }
				ag->args = list_make2(makeTargetEntry((Expr *) ey, 1, NULL, false), makeTargetEntry((Expr *) ex, 2, NULL, false));
			}
			else { Node *e = plan_expr(line + n); if (!e) { fprintf(stderr, "harness: bad expression\n"); return 2; } ag->args = list_make1(makeTargetEntry((Expr *) e, 1, NULL, false)); }
			parse->targetList = lappend(parse->targetList, makeTargetEntry((Expr *) ag, list_length(parse->targetList) + 1, NULL, false));
		}
		else if (sscanf(line, "dist %63s", w) == 1)
		{
			if (strcmp(w, "none") != 0)
			{
				dist = makeNode(Distribution);
				dist->distributionType = !strcmp(w, "replicated") ? LOCATOR_TYPE_REPLICATED : LOCATOR_TYPE_SHARD;
				if (sscanf(line, "dist shard %d.%d nodes %d", &r, &a, &n) == 3)
				{
					dist->nExprs = 1; dist->disExprs = (Node **) calloc(1, sizeof(Node *)); dist->disExprs[0] = (Node *) plan_var(r, a);
					fake_datanodes = n;
				}
			}
		}
		else if (!strncmp(line, "having", 6)) parse->havingQual = (Node *) plan_const(INT4OID, "1");
		else if (!strncmp(line, "groupingsets", 12)) parse->groupingSets = list_make1(makeNode(GroupingSet));
		else if (sscanf(line, "groups %lf", &t) == 1) output_rel->rows = t;
		else if (sscanf(line, "pairs %lf", &t) == 1) fake_pairs = t;
		else if (!strncmp(line, "protected", 9)) { g_enable_cls = true; fake_cls_policy = true; }
		else { fprintf(stderr, "harness: scenario line not understood: %s", line); return 2; }
	}
	fclose(f);
	if (!input_rel) { fprintf(stderr, "harness: scenario without input\n"); return 2; }
	input_rel->cheapest_total_path->distribution = dist;
	/* GROUP BY columns: mark the matching target entry, or add a resjunk one (parse_clause.c:findTargetlistEntrySQL99) */
	i = 0;
	foreach(lc, groups)
	{
		Var		   *gv = (Var *) lfirst(lc);
		SortGroupClause *sgc = makeNode(SortGroupClause);
		ListCell   *tl;
		TargetEntry *found = NULL;

		sgc->tleSortGroupRef = ++i;
		foreach(tl, parse->targetList)
			if (equal(((TargetEntry *) lfirst(tl))->expr, gv) && ((TargetEntry *) lfirst(tl))->ressortgroupref == 0) { found = (TargetEntry *) lfirst(tl); break; }
		if (!found) { found = makeTargetEntry((Expr *) gv, list_length(parse->targetList) + 1, NULL, true); parse->targetList = lappend(parse->targetList, found); }
		found->ressortgroupref = sgc->tleSortGroupRef;
		parse->groupClause = lappend(parse->groupClause, sgc);
	}
	foreach(lc, parse->targetList)
		if (!((TargetEntry *) lfirst(lc))->resjunk)
			output_rel->reltarget->exprs = lappend(output_rel->reltarget->exprs, ((TargetEntry *) lfirst(lc))->expr);

	gpuexec_upper_paths_hook(root, UPPERREL_GROUP_AGG, input_rel, output_rel);
	if (added_paths == NIL) { printf("declined\n"); return 0; }
	{
		Path	   *top = (Path *) linitial(added_paths);
		CustomPath *cp;
		CustomScan *cs;
		AttrNumber	k = 0;

		if (IsA(top, AggPath))
		{
			AggPath    *ap = (AggPath *) top;

			if (ap->subpath->pathtype != T_RemoteSubplan) { fprintf(stderr, "harness: Finalize Agg without a redistribute below it\n"); return 3; }
			printf("path partial: Finalize Agg (split %d, strategy %d) <- RemoteSubplan <- CustomScan\n", (int) ap->aggsplit, (int) ap->aggstrategy);
			cp = NULL;
			/* the fake create_redistribute_grouping_path does not keep its input: the hook built exactly one CustomPath */
		}
		else printf("path pushdown: CustomScan\n");
		cp = last_custom_path;
		if (!cp) { fprintf(stderr, "harness: no CustomPath was built\n"); return 3; }
		printf("cost startup %.3f total %.3f rows %.0f\n", cp->path.startup_cost, cp->path.total_cost, cp->path.rows);
		cs = (CustomScan *) cp->methods->PlanCustomPath(root, output_rel, cp, parse->targetList, NIL, NIL);
		printf("desc %s\n", out_value_list(cs->custom_private));
		foreach(lc, cs->custom_scan_tlist)
		{
			TargetEntry *te = (TargetEntry *) lfirst(lc);

			if (te->resno != ++k) { fprintf(stderr, "harness: custom_scan_tlist resno %d at position %d\n", te->resno, k); return 3; }
			if (IsA(te->expr, Var)) printf("scan %d var %d.%d type %u\n", k, ((Var *) te->expr)->varno, ((Var *) te->expr)->varattno, ((Var *) te->expr)->vartype);
			else if (IsA(te->expr, Aggref)) printf("scan %d agg %u type %u split %d\n", k, ((Aggref *) te->expr)->aggfnoid, ((Aggref *) te->expr)->aggtype, (int) ((Aggref *) te->expr)->aggsplit);
			else printf("scan %d node %d\n", k, (int) nodeTag(te->expr));
		}
		printf("plan_tlist %d scanrelid %u\n", list_length(cs->scan.plan.targetlist), cs->scan.scanrelid);
	}
	return 0;
}

int main(int argc, char **argv)
{
	bool		ship_only = false;
	FILE	   *f;
	char		magic[4];
	int			nrels, i, r, nout, total_pages = 0;
	GpuExecState desc;
	Oid			out_types[GX_MAX_GROUP_COLS + GX_MAX_AGGS];
	CustomScan *cscan;
	CustomScanState *css;
	EState		estate;
	ExprContext econtext;
	TupleDesc	sdesc;
	TupleTableSlot *slot;
	int64		nrows = 0;

	if (argc >= 3 && strcmp(argv[1], "--plan") == 0) return plan_main(argv[2]);
	if (argc >= 3 && strcmp(argv[1], "--ship-only") == 0) { ship_only = true; argv++; argc--; }
	if (argc < 2) { fprintf(stderr, "usage: %s [--ship-only] <case file>\n", argv[0]); return 2; }
	f = fopen(argv[1], "rb");
	if (!f) { perror(argv[1]); return 2; }
	rd(f, magic, 4);
	if (memcmp(magic, "GXH1", 4) != 0) { fprintf(stderr, "harness: bad magic\n"); return 2; }
	nrels = rd32(f);
	if (nrels < 1 || nrels > GX_MAX_JOINS + 1) { fprintf(stderr, "harness: %d relations\n", nrels); return 2; }
	for (r = 0; r < nrels; r++)
	{
		FakeRel    *fr = &fake_rels[r];
		int			natts = rd32(f);
		TupleDesc	d = (TupleDesc) calloc(1, offsetof(struct tupleDesc, attrs) + natts * sizeof(FormData_pg_attribute));

		d->natts = natts;
		d->tdrefcount = -1;
		for (i = 0; i < natts; i++)
		{
			Form_pg_attribute a = TupleDescAttr(d, i);
			int32		len = rd32(f), align = rd32(f), typid = rd32(f), notnull = rd32(f);

			a->attlen = (int16) len;
			a->attalign = align == 8 ? 'd' : align == 4 ? 'i' : align == 2 ? 's' : 'c';
			a->atttypid = (Oid) typid;
			a->attnum = i + 1;
			a->attbyval = len > 0;
			a->attnotnull = notnull != 0;
			a->atttypmod = typid == BPCHAROID ? VARHDRSZ + 1 : -1;
			snprintf(NameStr(a->attname), NAMEDATALEN, "a%d", i + 1);
		}
		fr->npages = rd64(f);
		rd(f, &fr->cls.reltuples, 4);			/* float4, as in pg_class */
		fr->pages = (char *) malloc((size_t) fr->npages * BLCKSZ + 1);
		rd(f, fr->pages, (size_t) fr->npages * BLCKSZ);
		fr->rd.rd_att = d;
		fr->rd.rd_rel = &fr->cls;
		fr->buf_base = total_pages;
		total_pages += (int) fr->npages;
		n_fake_rels++;
	}
	LocalBufferBlockPointers = (Block *) calloc((size_t) total_pages + 1, sizeof(Block));
	for (r = 0; r < nrels; r++)
		for (i = 0; i < fake_rels[r].npages; i++)
			LocalBufferBlockPointers[fake_rels[r].buf_base + i] = (Block) (fake_rels[r].pages + (size_t) i * BLCKSZ);

	memset(&desc, 0, sizeof(desc));
	/* the number of joins (0 none); step 1's block carries its unique flag, the blocks of steps 2.. their probe key */
	desc.n_joins = rd32(f);
	if (desc.n_joins < 0 || desc.n_joins > GX_MAX_JOINS) { fprintf(stderr, "harness: %d joins\n", desc.n_joins); return 2; }
	read_relinfo(f, &desc.outer);
	for (r = 0; r < desc.n_joins; r++)
	{
		GpuJoinStep *j = &desc.join[r];

		read_relinfo(f, &j->rel);
		j->key_col = rd32(f);
		if (r > 0) { j->probe.side = rd32(f); j->probe.col = rd32(f); }
		j->n_payload = rd32(f);
		for (i = 0; i < j->n_payload; i++) j->payload_cols[i] = rd32(f);
		j->unique = r == 0 ? rd32(f) != 0 : true;	/* every step of a chain is unique */
		j->n_preds = rd32(f);
		rd(f, j->preds, sizeof(gx_pred) * j->n_preds);
	}
	desc.partial = rd32(f);
	rd(f, &desc.plan, sizeof(gx_agg_plan));
	nout = rd32(f);
	for (i = 0; i < nout; i++) out_types[i] = (Oid) rd32(f);
	fclose(f);

	if (ship_only)
	{
		/* CN -> DN plan shipping without a GPU: the descriptor as Value nodes, written the way nodeToString() writes them,
		 * read back by the reference's OWN nodes/read.c (stringToNode), deserialised and serialised again */
		List	   *priv = gpuexec_serialise(&desc);
		char	   *wire = out_value_list(priv);
		List	   *back = (List *) stringToNode(wire);
		GpuExecState got;
		char	   *again;

		if (!IsA(back, List) || list_length(back) != list_length(priv)) { fprintf(stderr, "harness: %d nodes sent, %d read back\n", list_length(priv), back ? list_length(back) : -1); return 3; }
		memset(&got, 0, sizeof(got));
		gpuexec_deserialise(back, &got);
		again = out_value_list(gpuexec_serialise(&got));
		if (strcmp(wire, again) != 0) { fprintf(stderr, "harness: descriptor changed in transit\n sent %s\n got  %s\n", wire, again); return 3; }
		if ((i = changed_pred(desc.plan.preds, got.plan.preds, desc.plan.n_preds)) >= 0) { fprintf(stderr, "harness: qual constant %d changed\n", i); return 3; }
		for (r = 0; r < desc.n_joins; r++)
			if ((i = changed_pred(desc.join[r].preds, got.join[r].preds, desc.join[r].n_preds)) >= 0) { fprintf(stderr, "harness: qual constant %d of join step %d changed\n", i, r + 1); return 3; }
		if (desc.plan.est_groups != got.plan.est_groups) { fprintf(stderr, "harness: est_groups changed\n"); return 3; }
		if (desc.plan.join_type != got.plan.join_type) { fprintf(stderr, "harness: join type changed\n"); return 3; }
		printf("ship ok: %d nodes, %zu bytes\n%s\n", list_length(priv), strlen(wire), wire);
		return 0;
	}
	/* ---- what the planner + ExecInitCustomScan would have done */
	_PG_init();
	if (!registered_methods) { fprintf(stderr, "harness: _PG_init registered nothing\n"); return 3; }
	cscan = makeNode(CustomScan);
	cscan->methods = registered_methods;
	cscan->custom_private = gpuexec_serialise(&desc);	/* the descriptor travels as Value nodes, as it would CN -> DN */
	css = (CustomScanState *) cscan->methods->CreateCustomScanState(cscan);
	memset(&estate, 0, sizeof(estate));
	memset(&econtext, 0, sizeof(econtext));
	css->ss.ps.plan = &cscan->scan.plan;
	css->ss.ps.state = &estate;
	css->ss.ps.ps_ExprContext = &econtext;
	css->ss.ps.ps_ProjInfo = NULL;		/* target list == scan tuple: no projection step */
	sdesc = (TupleDesc) calloc(1, offsetof(struct tupleDesc, attrs) + nout * sizeof(FormData_pg_attribute));
	sdesc->natts = nout;
	for (i = 0; i < nout; i++) { TupleDescAttr(sdesc, i)->atttypid = out_types[i]; TupleDescAttr(sdesc, i)->attnum = i + 1; }
	slot = (TupleTableSlot *) calloc(1, sizeof(TupleTableSlot));
	slot->type = T_TupleTableSlot;
	slot->tts_flags = TTS_FLAG_EMPTY;
	slot->tts_tupleDescriptor = sdesc;
	slot->tts_values = (Datum *) calloc(nout, sizeof(Datum));
	slot->tts_isnull = (bool *) calloc(nout, sizeof(bool));
	css->ss.ss_ScanTupleSlot = slot;

	css->methods->BeginCustomScan(css, &estate, 0);
	for (;;)
	{
		TupleTableSlot *res = css->methods->ExecCustomScan(css);

		if (TupIsNull(res))
			break;
		for (i = 0; i < nout; i++)
		{
			if (i) putchar('\t');
			if (res->tts_isnull[i]) { fputs("\\N", stdout); continue; }
			switch (out_types[i])
			{
				case FLOAT8OID: printf("%.17g", DatumGetFloat8(res->tts_values[i])); break;
				case INT8OID: printf("%ld", (long) DatumGetInt64(res->tts_values[i])); break;
				case CHAROID: printf("%d", (int) (signed char) DatumGetChar(res->tts_values[i])); break;
				case BPCHAROID: printf("%d", (int) (signed char) VARDATA_ANY(DatumGetPointer(res->tts_values[i]))[0]); break;
				case FLOAT8ARRAYOID:
					{
						ArrayType  *a = (ArrayType *) DatumGetPointer(res->tts_values[i]);
						double	   *v = (double *) ARR_DATA_PTR(a);
						int			k;

						for (k = 0; k < ARR_DIMS(a)[0]; k++)
							printf("%c%.17g", k ? ',' : '{', v[k]);
						putchar('}');
						break;
					}
				default: printf("%d", DatumGetInt32(res->tts_values[i])); break;
			}
		}
		putchar('\n');
		nrows++;
	}
	css->methods->ExplainCustomScan(css, NIL, &(ExplainState) {.analyze = true});
	css->methods->ReScanCustomScan(css);
	{
		TupleTableSlot *again = css->methods->ExecCustomScan(css);		/* TupIsNull() evaluates its argument twice */

		if (TupIsNull(again) != (nrows == 0)) { fprintf(stderr, "harness: rescan did not replay the result\n"); return 3; }
	}
	css->methods->EndCustomScan(css);
	if (live_handles != NULL) { fprintf(stderr, "harness: EndCustomScan left handles registered\n"); return 3; }
	gx_shutdown(backend_ctx);
	fprintf(stderr, "harness: %ld rows\n", (long) nrows);
	return 0;
}
