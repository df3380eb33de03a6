/*
 * gx_double.c — a TEST DOUBLE of the C ABI (include/gpuexec.h) for host-logic tests of the provider.
 *
 * TEST INFRASTRUCTURE ONLY.  It is linked into one binary, harness/gpuexec_harness_double, in place of libgpuexec.so,
 * so that the provider's host code — the heap-page loader's batching and visibility lists, the call sequence, the
 * Datum encoding of every result column type, NULL flags, partial transition states, ReScan/End bookkeeping — runs where
 * no GPU exists (tests/test_provider_host_logic_cpu.py).  It computes NOTHING: gx_hash_agg() hands back the groups the
 * test wrote into the file named by GX_DOUBLE_RESULT, after checking that the plan it was given has the announced
 * shape.  It is never installed, never loaded by the product, and is not a fallback: libgpuexec.so fails loudly without a
 * GPU (tests/test_abi.py::test_no_gpu_means_loud_failure_not_fallback).
 *
 * Every call appends one line to stderr ("double: ...") — the trace the test asserts on.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <stdint.h>

#include "gpuexec.h"

struct gx_ctx { int dummy; };
struct gx_table { int ncols; int32_t types[GX_MAX_COLS]; int64_t pages, rows, batches, est_rows; int finished; };
struct gx_hash { int key_col, n_payload, unique, n_preds; };
struct gx_result { int64_t ngroups; int ng, na; int64_t *keys; double *aggs; int64_t *cnts; uint8_t *nulls; double *sxx, *regr; };

static char last_error[256] = "";
static void *stage[2];
static size_t stage_bytes[2];
static int stage_next = 0;
static int live_tables = 0, live_hashes = 0, live_results = 0;

int gx_abi_version(void) { return GX_ABI_VERSION; }
const char *gx_last_error(gx_ctx *ctx) { return last_error; }
int gx_init(int device, gx_ctx **out) { *out = (gx_ctx *) calloc(1, sizeof(gx_ctx)); fprintf(stderr, "double: init device %d\n", device); return GX_OK; }
void gx_shutdown(gx_ctx *ctx)
{
	fprintf(stderr, "double: shutdown live tables %d hashes %d results %d\n", live_tables, live_hashes, live_results);
	free(ctx);
}
int gx_pool_reserve(gx_ctx *ctx, size_t bytes) { fprintf(stderr, "double: pool_reserve %zu\n", bytes); return GX_OK; }

int gx_table_create(gx_ctx *ctx, int ncols, const int32_t *types, int64_t capacity_rows, gx_table **out)
{
	gx_table   *t = (gx_table *) calloc(1, sizeof(gx_table));
	int			i;

	t->ncols = ncols; t->est_rows = capacity_rows;
	fprintf(stderr, "double: table_create ncols %d types", ncols);
	for (i = 0; i < ncols; i++) { t->types[i] = types[i]; fprintf(stderr, " %d", types[i]); }
	fprintf(stderr, " capacity %lld\n", (long long) capacity_rows);
	live_tables++;
	*out = t;
	return GX_OK;
}
void gx_table_free(gx_table *t) { if (t) { live_tables--; free(t); } }

int gx_stage_acquire(gx_ctx *ctx, size_t bytes, void **out)
{
	int			s = stage_next;

	stage_next ^= 1;
	if (stage_bytes[s] < bytes) { free(stage[s]); stage[s] = malloc(bytes); stage_bytes[s] = bytes; }
	memset(stage[s], 0xA5, bytes);			/* whatever the caller does not overwrite is recognisable */
	*out = stage[s];
	return GX_OK;
}

/* OpenTenBase page header: pd_lower at byte 16 (LocationIndex is uint32, bufpage.h:85-89), line pointers from byte 44 */
int gx_table_append_heap_pages(gx_table *t, const void *pages, int64_t npages, const gx_heap_desc *desc,
							   const uint16_t *vis_offsets, const int32_t *vis_counts, int32_t vis_stride)
{
	int64_t		p, rows = 0;
	int			i;

	if (npages < 1 || npages > 4096) { snprintf(last_error, sizeof(last_error), "double: batch of %lld pages", (long long) npages); return GX_ERR_ARG; }
	if (desc->ncols != t->ncols) { snprintf(last_error, sizeof(last_error), "double: descriptor has %d columns, table %d", desc->ncols, t->ncols); return GX_ERR_ARG; }
	for (p = 0; p < npages; p++)
	{
		const unsigned char *pg = (const unsigned char *) pages + p * 8192;
		uint32_t	lower;
		int			maxoff;

		memcpy(&lower, pg + 16, 4);
		maxoff = lower <= 44 ? 0 : (int) ((lower - 44) / 4);
		if (vis_counts[p] < 0 || vis_counts[p] > vis_stride || vis_counts[p] > maxoff)
		{ snprintf(last_error, sizeof(last_error), "double: page %lld: %d visible tuples, %d line pointers", (long long) p, vis_counts[p], maxoff); return GX_ERR_ARG; }
		for (i = 0; i < vis_counts[p]; i++)
		{
			int			off = vis_offsets[p * vis_stride + i];

			if (off < 1 || off > maxoff || (i > 0 && off <= vis_offsets[p * vis_stride + i - 1]))
			{ snprintf(last_error, sizeof(last_error), "double: page %lld: visible offset %d out of order or range", (long long) p, off); return GX_ERR_ARG; }
		}
		rows += vis_counts[p];
	}
	t->pages += npages; t->rows += rows; t->batches++;
	fprintf(stderr, "double: append_heap_pages pages %lld rows %lld natts %d attnums", (long long) npages, (long long) rows, desc->natts);
	for (i = 0; i < desc->ncols; i++) fprintf(stderr, " %d", desc->attnums[i]);
	fprintf(stderr, " notnull");
	for (i = 0; i < desc->ncols; i++) fprintf(stderr, " %d", (int) desc->att_notnull[desc->attnums[i]]);
	fprintf(stderr, "\n");
	return GX_OK;
}
int gx_table_load_finish(gx_table *t)
{
	t->finished = 1;
	fprintf(stderr, "double: load_finish pages %lld rows %lld batches %lld\n", (long long) t->pages, (long long) t->rows, (long long) t->batches);
	return GX_OK;
}

int gx_hash_build(gx_ctx *ctx, const gx_table *inner, int key_col, int n_preds, const gx_pred *preds,
				  int n_payload, const int32_t *payload_cols, int unique, gx_hash **out)
{
	gx_hash    *h = (gx_hash *) calloc(1, sizeof(gx_hash));
	int			i;

	if (!inner->finished) { snprintf(last_error, sizeof(last_error), "double: hash_build before load_finish"); return GX_ERR_STATE; }
	h->key_col = key_col; h->n_payload = n_payload; h->unique = unique; h->n_preds = n_preds;
	fprintf(stderr, "double: hash_build key %d unique %d payload", key_col, unique);
	for (i = 0; i < n_payload; i++) fprintf(stderr, " %d", payload_cols[i]);
	fprintf(stderr, " preds");
	for (i = 0; i < n_preds; i++) fprintf(stderr, " (%d %d %lld)", preds[i].col, preds[i].op, (long long) preds[i].ival);
	fprintf(stderr, "\n");
	live_hashes++;
	*out = h;
	return GX_OK;
}
void gx_hash_free(gx_hash *h) { if (h) { live_hashes--; free(h); } }

/* file: int64 ngroups, int32 ng, int32 na, keys[ngroups*ng] int64, aggs[ngroups*na] double, cnts[ngroups*na] int64, nulls[ngroups*(ng+na)],
 * then optionally sxx[ngroups*na] double and regr[ngroups*na*6] double (zeros when absent) */
int gx_hash_agg(gx_ctx *ctx, const gx_table *outer, const gx_hash *h, const gx_agg_plan *plan, gx_result **out)
{
	const char *path = getenv("GX_DOUBLE_RESULT");
	FILE	   *f = path ? fopen(path, "rb") : NULL;
	gx_result  *r = (gx_result *) calloc(1, sizeof(gx_result));
	int32_t		ng, na;
	size_t		n;

	if (!outer->finished) { snprintf(last_error, sizeof(last_error), "double: hash_agg before load_finish"); return GX_ERR_STATE; }
	if (!f) { snprintf(last_error, sizeof(last_error), "double: GX_DOUBLE_RESULT not readable"); return GX_ERR_ARG; }
	if (getenv("GX_DOUBLE_FAIL_AGG")) { fclose(f); free(r); snprintf(last_error, sizeof(last_error), "double: value out of range: overflow"); return GX_ERR_OVERFLOW; }
	n = fread(&r->ngroups, 8, 1, f); n += fread(&ng, 4, 1, f); n += fread(&na, 4, 1, f);
	if (n != 3 || ng != plan->n_group_cols || na != plan->n_aggs)
	{ snprintf(last_error, sizeof(last_error), "double: plan has %d group columns and %d aggregates, the canned result %d and %d", plan->n_group_cols, plan->n_aggs, ng, na); fclose(f); return GX_ERR_ARG; }
	r->ng = ng; r->na = na;
	r->keys = (int64_t *) calloc((size_t) r->ngroups * ng + 1, 8);
	r->aggs = (double *) calloc((size_t) r->ngroups * na + 1, 8);
	r->cnts = (int64_t *) calloc((size_t) r->ngroups * na + 1, 8);
	r->nulls = (uint8_t *) calloc((size_t) r->ngroups * (ng + na) + 1, 1);
	r->sxx = (double *) calloc((size_t) r->ngroups * na + 1, 8);
	r->regr = (double *) calloc((size_t) r->ngroups * na * 6 + 1, 8);
	n = fread(r->keys, 8, (size_t) r->ngroups * ng, f); n = fread(r->aggs, 8, (size_t) r->ngroups * na, f);
	n = fread(r->cnts, 8, (size_t) r->ngroups * na, f); n = fread(r->nulls, 1, (size_t) r->ngroups * (ng + na), f);
	n = fread(r->sxx, 8, (size_t) r->ngroups * na, f);
	n = fread(r->regr, 8, (size_t) r->ngroups * na * 6, f);
	fclose(f);
	fprintf(stderr, "double: hash_agg outer rows %lld join %d groups %d aggs %d preds %d outer_key %d est_groups %lld\n", (long long) outer->rows, h != NULL,
			plan->n_group_cols, plan->n_aggs, plan->n_preds, plan->outer_key_col, (long long) plan->est_groups);
	live_results++;
	*out = r;
	return GX_OK;
}
/* the chain's steps in order, then the canned result of gx_hash_agg */
int gx_hash_agg_joins(gx_ctx *ctx, const gx_table *outer, int n_steps, const gx_join_step *steps, const gx_agg_plan *plan, gx_result **out)
{
	int			i;

	if (n_steps < 1 || n_steps > GX_MAX_JOINS || plan->outer_key_col >= 0) { snprintf(last_error, sizeof(last_error), "double: join chain of %d steps, outer key %d", n_steps, plan->outer_key_col); return GX_ERR_ARG; }
	fprintf(stderr, "double: hash_agg_joins steps %d", n_steps);
	for (i = 0; i < n_steps; i++)
	{
		if (!steps[i].h || !steps[i].h->unique) { snprintf(last_error, sizeof(last_error), "double: step %d has no unique table", i + 1); return GX_ERR_ARG; }
		fprintf(stderr, " (key %d.%d table key %d)", steps[i].key.side, steps[i].key.col, steps[i].h->key_col);
	}
	fprintf(stderr, "\n");
	return gx_hash_agg(ctx, outer, steps[0].h, plan, out);
}
/* the probe side and the table, then the canned result of gx_hash_agg */
int gx_hash_agg_right(gx_ctx *ctx, const gx_table *probe, int probe_key_col, int n_probe_preds, const gx_pred *probe_preds,
					  const gx_table *build, const gx_hash *h, int join_type, const gx_agg_plan *plan, gx_result **out)
{
	int			i;

	if (!probe->finished) { snprintf(last_error, sizeof(last_error), "double: hash_agg_right before load_finish"); return GX_ERR_STATE; }
	if (!h || h->n_payload != 0 || plan->outer_key_col >= 0 || plan->join_type != GX_JOIN_INNER)
	{ snprintf(last_error, sizeof(last_error), "double: hash_agg_right with a payload or a join in the plan"); return GX_ERR_ARG; }
	fprintf(stderr, "double: hash_agg_right type %d probe rows %lld key %d table key %d preds", join_type, (long long) probe->rows,
			probe_key_col, h->key_col);
	for (i = 0; i < n_probe_preds; i++) fprintf(stderr, " (%d %d %lld)", probe_preds[i].col, probe_preds[i].op, (long long) probe_preds[i].ival);
	fprintf(stderr, "\n");
	return gx_hash_agg(ctx, build, NULL, plan, out);
}
int64_t gx_result_ngroups(const gx_result *r) { return r->ngroups; }
int gx_result_fetch(gx_result *r, int64_t max_groups, int64_t *key_out, double *agg_out, uint8_t *null_out)
{
	memcpy(key_out, r->keys, (size_t) r->ngroups * r->ng * 8);
	memcpy(agg_out, r->aggs, (size_t) r->ngroups * r->na * 8);
	if (null_out) memcpy(null_out, r->nulls, (size_t) r->ngroups * (r->ng + r->na));
	fprintf(stderr, "double: result_fetch (final values)\n");
	return GX_OK;
}
int gx_result_fetch_states(gx_result *r, int64_t max_groups, int64_t *key_out, double *val_out, int64_t *cnt_out, uint8_t *null_out)
{
	memcpy(key_out, r->keys, (size_t) r->ngroups * r->ng * 8);
	memcpy(val_out, r->aggs, (size_t) r->ngroups * r->na * 8);
	memcpy(cnt_out, r->cnts, (size_t) r->ngroups * r->na * 8);
	if (null_out) memcpy(null_out, r->nulls, (size_t) r->ngroups * (r->ng + r->na));
	fprintf(stderr, "double: result_fetch_states (transition states)\n");
	return GX_OK;
}
int gx_result_fetch_sxx(gx_result *r, int64_t max_groups, double *sxx_out)
{
	memcpy(sxx_out, r->sxx, (size_t) r->ngroups * r->na * 8);
	fprintf(stderr, "double: result_fetch_sxx\n");
	return GX_OK;
}
int gx_result_fetch_regr(gx_result *r, int64_t max_groups, double *out)
{
	memcpy(out, r->regr, (size_t) r->ngroups * r->na * 6 * 8);
	fprintf(stderr, "double: result_fetch_regr\n");
	return GX_OK;
}
void gx_result_free(gx_result *r)
{
	if (!r) return;
	live_results--;
	free(r->keys); free(r->aggs); free(r->cnts); free(r->nulls); free(r->sxx); free(r->regr); free(r);
}
