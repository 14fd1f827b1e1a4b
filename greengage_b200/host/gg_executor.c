/*
 * gg_executor.c — ExecInitNode / ExecProcNode / ExecEndNode for the GPU segment engine (include/gg_executor.h).
 *
 * Host C above the C-ABI of libggb200.so; no CUDA here.  What the reference does tuple-at-a-time through
 * ExecProcNode dispatch (execProcnode.c:925-1100), this layer does pipeline-at-a-time: ExecInitNode fuses the
 * slice into device pipelines, the first ExecProcNode call on a pipeline's top node runs it on the device, and
 * every call hands out one row of the result as a virtual tuple — the contract the node above sees is the
 * reference's (one TupleTableSlot per call, NULL at end of stream, ExecReScan restarts, ExecSquelchNode stops
 * early; nodeAgg.c:1123, nodeHashjoin.c:78, nodeSort.c:48, nodeMotion.c:180).
 *
 * Results stay on the device between the nodes of a slice:
 *     aggregate rows   as group records (gg_groups): Agg -> Motion -> FINAL Agg -> Gather move and combine them there
 *                      (gg_ic_motion_groups, gg_groups_final); the node at the top fetches once
 *     scanned rows     as datum rows (GG_FMT_DATUMROWS): SeqScan with a target list -> Redistribute Motion ->
 *                      Hash / HashJoin / Agg scan them with the same kernels (gg_motion_partition, gg_ic_exchange_rows)
 *     joined rows      as datum rows: a HashJoin with a target list writes them (gg_joinrows_create) for another HashJoin,
 *                      a Sort / Limit, a Motion or the caller
 * Host arrays of Datums appear only where a node has to hand tuples to its caller, or on the generic path (Sort, a
 * Motion over a transport callback).
 */
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../../include/gg_executor.h"
#include "../../include/gg_tupser.h"

int32_t gg_cdbhash_route(const int32_t *typids, const int64_t *vals, const int32_t *lens, const int32_t *isnull,
                         int nkeys, int nsegs);      /* gg_motion_host.c */

enum { K_SCANAGG = 1, K_JOINAGG, K_AGGFINAL, K_SORT, K_MOTION, K_SCANROWS, K_HASH, K_LIMIT, K_JOINROWS, K_WINDOW };

#define GG_NO_BOUND UINT64_MAX

/* The bounded sorts are referenced weakly, so this library still links and loads against a device library (or a stand-in for
 * one) that lacks them.  Without them, a Limit over a Sort is refused at ExecInitNode with GG_ERR_UNSUPPORTED, and the caller
 * keeps its CPU nodes for that subtree; no other sort takes their place. */
#pragma weak gg_sort_rows_bounded
#pragma weak gg_sort_datumrows_bounded
/* the same for the join that writes its rows: without them a HashJoin with a target list is refused (GG_ERR_UNSUPPORTED) */
#pragma weak gg_joinrows_create
#pragma weak gg_joinagg_rows
/* the same for the Agg that finalises its groups into datum rows: without them an Agg under a Sort or a Limit hands up host rows */
#pragma weak gg_scanagg_datumrows
#pragma weak gg_joinagg_datumrows
#pragma weak gg_groups_datumrows
/* the row filter of an Agg's HAVING: without it (or without the three above) an Agg with a qual is refused (GG_ERR_UNSUPPORTED);
 * no path runs the Agg with its qual dropped */
#pragma weak gg_rowfilter_create
#pragma weak gg_rowfilter_run
#pragma weak gg_rowfilter_free
/* and the upload of a FINAL Agg's host-finalised rows to such a filter or to a join */
#pragma weak gg_relation_load
/* the window functions: without them a WindowAgg is refused (GG_ERR_UNSUPPORTED); no other path runs it */
#pragma weak gg_window_create
#pragma weak gg_window_run
#pragma weak gg_window_free
#pragma weak gg_engine_last_kernel_ms

struct GgPlanState {
	int kind;
	GgPlan *plan;
	GgEState *estate;
	struct GgPlanState *child;          /* Sort / Motion / final Agg / Agg over rows: the pipeline below */
	struct GgPlanState *inner;          /* join: the rows node under the Hash (NULL: the inner SeqScan is fused) */
	int table_kept;                     /* K_JOINROWS: the hash table of one batch is built and kept for a rescan (never with a
	                                     * Motion on the inner side: every segment re-runs that exchange alike) */
	/* device pipelines */
	gg_scanagg *sa;
	gg_joinagg *ja;
	gg_relation *rel, *inner_rel;       /* base relations (not owned) */
	const void *host_pages;             /* K_SCANAGG over a relation in host memory */
	uint64_t host_nblocks;
	gg_agg agg;
	/* device-resident results */
	gg_groups *groups;                  /* aggregate rows */
	gg_relation *rows_rel;              /* datum rows (K_SCANROWS, K_MOTION over a scan): wraps rows_recv / rows_send; K_JOINROWS:
	                                     * wraps the join's output */
	gg_relation *rows_send, *rows_recv; /* raw device buffers (gg_relation_create) */
	uint64_t rows_cap;                  /* rows the send buffer holds over all destinations */
	uint64_t rows_n;
	int32_t rows_ncols;
	int32_t rows_targets[GG_MAX_OUTCOLS];
	gg_tupdesc rows_desc;               /* GG_FMT_DATUMROWS descriptor of what this node delivers */
	GgSeqScan *rows_scan;               /* the SeqScan the rows come from */
	int32_t rows_nsegs;                 /* destinations the rows are partitioned for (1: plain projection) */
	/* result set: filled on demand, then handed out row by row */
	int done;                           /* pipeline has run */
	int sort_runs;                      /* Sort over host rows: sorted runs the last execution merged (1: it fitted the operator's memory) */
	uint64_t sort_bound;                /* Sort: rows the Limit above wants (SortState.bound, set by pass_down_bound); GG_NO_BOUND: all */
	double instr_ntuples, instr_nloops; /* Instrumentation: tuples handed up, executions */
	int rows_ready;                     /* host arrays below are filled */
	int squelched;
	int nonreceiver;                    /* above a Gather, on a segment that is not its receiver: no rows at all */
	int dev_groups;                     /* decided at init, from the plan alone (so every segment decides alike): this node hands
	                                     * its aggregate rows up as device-resident group records */
	int agg_rows;                       /* decided at init, from the plan alone: an Agg directly under a Sort or a Limit, under a
	                                     * HashJoin, or with a HAVING qual hands up its groups finalised into device datum rows
	                                     * (rows_rel), which the node above sorts, windows or joins where they are */
	gg_rowfilter *having;               /* an Agg's plan.qual (HAVING), compiled at init over its rows_desc; a WindowAgg's qual */
	gg_window_obj *win;                 /* K_WINDOW: the window functions, created at init over the child's rows */
	float win_ms;                       /* K_WINDOW: CUDA-event time of the last gg_window_run */
	int rows_required;                  /* an Agg under a HashJoin: the join reads device rows only, so a FINAL Agg whose groups were
	                                     * finalised on the host uploads them */
	int lazy_fetch;                     /* set by a Motion above that moves this node's records on the device: the pipeline's result
	                                     * is not fetched to the host before it travels (no host synchronisation between the scan
	                                     * and the Motion); what a fetch would have decided travels as status flags */
	int32_t ncols;
	int64_t nrows, next, markpos;
	int64_t *values;
	uint8_t *isnull;
	int32_t typid[GG_MAX_OUTCOLS];
	int32_t *lens;                      /* [nrows][ncols], strings only */
	GgTupleTableSlot slot;
};

static _Thread_local char g_err[512];
static _Thread_local int g_errcode;
/* the first failure of THIS segment's own slice while it kept taking part in device Motions (so that its peers are never
 * left alone in a collective): what it reports in the end, rather than the flag that came back through the interconnect */
static _Thread_local char g_local_err[512];
static _Thread_local int g_local_code;

static void *exec_fail(int code, const char *fmt, ...)
{
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(g_err, sizeof g_err, fmt, ap);
	va_end(ap);
	g_errcode = code;
	return NULL;
}

const char *GgExecLastError(void) { return g_err; }
int GgExecLastErrorCode(void) { return g_errcode; }

const char *GgExecNodeKind(GgPlanState *s)
{
	if (!s) return "";
	switch (s->kind)
	{
		case K_SCANAGG: return "scanagg";
		case K_JOINAGG: return "joinagg";
		case K_AGGFINAL: return "aggfinal";
		case K_SORT: return "sort";
		case K_MOTION: return "motion";
		case K_SCANROWS: return "scanrows";
		case K_HASH: return "hash";
		case K_LIMIT: return "limit";
		case K_JOINROWS: return "joinrows";
		case K_WINDOW: return "windowagg";
	}
	return "";
}

/* where a node that has run keeps its result: "device-groups", "device-rows" or "host" (tests and EXPLAIN-style output) */
const char *GgExecNodeResultLocation(GgPlanState *s)
{
	if (!s || !s->done) return "";
	if (s->rows_rel && !s->rows_ready) return "device-rows";
	if (s->groups && !s->rows_ready) return "device-groups";
	return "host";
}

/* benchmarks: summed CUDA-event time of the scan / probe kernel launches of the pipeline at or below `s` since its last
 * rescan, their count, the kernel variant (gg_scanagg_variant), and for a join the build time */
int GgExecPipelineKernelMs(GgPlanState *s, float *ms, int *launches, int *variant, float *build_ms)
{
	for (; s; s = s->child)
	{
		if (s->sa)
		{
			if (variant) *variant = gg_scanagg_variant(s->sa);
			if (build_ms) *build_ms = 0;
			return gg_scanagg_scan_kernel_ms(s->sa, ms, launches);
		}
		if (s->ja)
		{
			uint64_t rb, tb;
			float b = 0;
			int rc = gg_joinagg_stats(s->ja, &rb, &tb, &b, ms);
			if (variant) *variant = gg_joinagg_variant(s->ja);
			if (build_ms) *build_ms = b;
			if (launches) *launches = 1;
			return rc;
		}
	}
	return GG_ERR_ARG;
}

GgPlanState *GgExecOuterPlanState(GgPlanState *s) { return s ? s->child : NULL; }
GgPlanState *GgExecInnerPlanState(GgPlanState *s) { return s ? s->inner : NULL; }

/* ---- output layout of an Agg node: group keys, then aggregates (a PARTIAL avg is its float8[3] state) ---- */
static int agg_ncols_of(const gg_agg *agg, int i)
{
	return (agg->aggs[i].aggfnoid == GG_AGG_AVG_FLOAT8 && agg->aggstage == GG_AGGSTAGE_PARTIAL) ? 3 : 1;
}

static int32_t agg_result_type(int32_t fn)
{
	switch (fn)
	{
		case GG_AGG_COUNT_ANY: case GG_AGG_COUNT_STAR: case GG_AGG_SUM_INT4: case GG_AGG_MAX_INT8: case GG_AGG_MIN_INT8:
			return GG_INT8OID;
		case GG_AGG_MAX_INT4: case GG_AGG_MIN_INT4: return GG_INT4OID;
		case GG_AGG_MAX_DATE: case GG_AGG_MIN_DATE: return GG_DATEOID;
		default: return GG_FLOAT8OID;
	}
}

static int64_t f8bits(double d) { int64_t v; memcpy(&v, &d, 8); return v; }
static double bitsf8(int64_t v) { double d; memcpy(&d, &v, 8); return d; }
static int is_string_type(int32_t t) { return t == GG_BPCHAROID || t == GG_VARCHAROID || t == GG_TEXTOID; }

/* the length of a string packed into a Datum word: string lengths do not travel with datum rows or host-row Motions */
static int32_t packed_len(uint64_t v)
{
	int32_t l = 0;
	while (l < 8 && ((v >> (8 * l)) & 0xff)) l++;
	return l;
}

static int alloc_result(GgPlanState *s, int64_t nrows, int32_t ncols)
{
	free(s->values); free(s->isnull); free(s->lens);
	s->nrows = nrows; s->ncols = ncols; s->next = 0; s->markpos = 0;
	s->values = calloc((size_t) (nrows > 0 ? nrows : 1) * (size_t) ncols, 8);
	s->isnull = calloc((size_t) (nrows > 0 ? nrows : 1) * (size_t) ncols, 1);
	s->lens = calloc((size_t) (nrows > 0 ? nrows : 1) * (size_t) ncols, 4);
	return (s->values && s->isnull && s->lens) ? 0 : -1;
}

/* the types of the grouping keys of the Agg whose rows a node hands up: at the FINAL stage grpCol holds type OIDs, at the
 * other stages expression roots */
static void agg_keytypes(const GgPlanState *s, int32_t *kt)
{
	int c;
	for (c = 0; c < s->agg.numCols; c++)
		kt[c] = s->agg.aggstage == GG_AGGSTAGE_FINAL ? s->agg.grpCol[c] : s->estate->pool->nodes[s->agg.grpCol[c]].rettype;
}

/* column count and types of an Agg node's output rows */
static int set_layout_types(GgPlanState *s)
{
	const gg_agg *agg = &s->agg;
	int ncols = agg->numCols, i, c;
	for (i = 0; i < agg->numAggs; i++) ncols += agg_ncols_of(agg, i);
	if (ncols > GG_MAX_OUTCOLS) { exec_fail(GG_ERR_UNSUPPORTED, "too many output columns"); return -1; }
	agg_keytypes(s, s->typid);
	for (i = 0, c = agg->numCols; i < agg->numAggs; i++)
	{
		int w = agg_ncols_of(agg, i), k;
		for (k = 0; k < w; k++) s->typid[c + k] = (w == 3) ? GG_FLOAT8OID : agg_result_type(agg->aggs[i].aggfnoid);
		c += w;
	}
	s->ncols = ncols;
	return 0;
}

/* gg_aggrow[] -> result columns */
static int rows_from_aggrows(GgPlanState *s, const gg_aggrow *rows, int n)
{
	const gg_agg *agg = &s->agg;
	int ncols, i, c, r;
	if (set_layout_types(s)) return -1;
	ncols = s->ncols;
	if (alloc_result(s, n, ncols)) { exec_fail(GG_ERR_NOMEM, "out of memory"); return -1; }
	for (r = 0; r < n; r++)
	{
		int64_t *v = s->values + (size_t) r * ncols;
		uint8_t *nl = s->isnull + (size_t) r * ncols;
		int32_t *ln = s->lens + (size_t) r * ncols;
		for (c = 0; c < agg->numCols; c++)
		{
			v[c] = rows[r].key[c]; nl[c] = (uint8_t) rows[r].keyisnull[c]; ln[c] = rows[r].keylen[c];
		}
		for (i = 0, c = agg->numCols; i < agg->numAggs; i++)
		{
			const gg_aggval *a = &rows[r].agg[i];
			int w = agg_ncols_of(agg, i);
			if (w == 3) { v[c] = f8bits(a->f[0]); v[c + 1] = f8bits(a->f[1]); v[c + 2] = f8bits(a->f[2]); }
			else
			{
				nl[c] = (uint8_t) a->isnull;
				v[c] = s->typid[c] == GG_FLOAT8OID ? f8bits(a->f[0]) : a->i;
			}
			c += w;
		}
	}
	s->rows_ready = 1;
	return 0;
}

/* result columns of a PARTIAL Agg (as they come out of a Motion) -> gg_aggrow[] for the FINAL stage */
static gg_aggrow *aggrows_from_rows(const GgPlanState *child, const gg_agg *agg)
{
	int64_t r;
	gg_aggrow *out = calloc((size_t) (child->nrows > 0 ? child->nrows : 1), sizeof *out);
	if (!out) return NULL;
	for (r = 0; r < child->nrows; r++)
	{
		const int64_t *v = child->values + (size_t) r * child->ncols;
		const uint8_t *nl = child->isnull + (size_t) r * child->ncols;
		const int32_t *ln = child->lens + (size_t) r * child->ncols;
		int c, i;
		for (c = 0; c < agg->numCols; c++)
		{
			out[r].key[c] = v[c]; out[r].keyisnull[c] = nl[c]; out[r].keylen[c] = ln[c];
		}
		for (i = 0, c = agg->numCols; i < agg->numAggs; i++)
		{
			gg_aggval *a = &out[r].agg[i];
			int32_t fn = agg->aggs[i].aggfnoid;
			if (fn == GG_AGG_AVG_FLOAT8)
			{
				a->f[0] = bitsf8(v[c]); a->f[1] = bitsf8(v[c + 1]); a->f[2] = bitsf8(v[c + 2]);
				c += 3;
			}
			else
			{
				a->isnull = nl[c];
				if (agg_result_type(fn) == GG_FLOAT8OID) a->f[0] = bitsf8(v[c]); else a->i = v[c];
				c += 1;
			}
		}
	}
	return out;
}

static void drop_device_results(GgPlanState *s)
{
	if (s->groups) { gg_groups_free(s->groups); s->groups = NULL; }
	if (s->rows_rel) { gg_relation_free(s->rows_rel); s->rows_rel = NULL; }
}

static void end_tree(GgPlanState *s)
{
	if (!s) return;
	end_tree(s->child);
	end_tree(s->inner);
	drop_device_results(s);
	if (s->rows_send) gg_relation_free(s->rows_send);
	if (s->rows_recv) gg_relation_free(s->rows_recv);
	if (s->sa) gg_scanagg_free(s->sa);
	if (s->ja) gg_joinagg_free(s->ja);
	if (s->having) gg_rowfilter_free(s->having);
	if (s->win) gg_window_free(s->win);
	free(s->values); free(s->isnull); free(s->lens);
	free(s);
}

#define GG_MAX_PLAN_DEPTH 32        /* the deepest accelerated slice is Motion <- Sort <- Agg <- Motion <- Agg <- HashJoin <- Hash <- Motion <- SeqScan */

static GgPlanState *init_node(GgPlan *node, GgEState *estate, int eflags, int depth);

GgPlanState *GgExecInitNode(GgPlan *node, GgEState *estate, int eflags)
{
	g_err[0] = 0; g_errcode = GG_OK;
	g_local_code = 0; g_local_err[0] = 0;
	return init_node(node, estate, eflags, 0);
}

static int multi_segment(const GgEState *es) { return es->nsegs > 1; }

/* a node that delivers device-resident datum rows: a SeqScan with a target list, a Motion over one, a HashJoin with a
 * target list, or a WindowAgg */
static int yields_rows(const GgPlan *p)
{
	if (!p) return 0;
	if (p->type == T_GgWindowAgg) return 1;
	if (p->type == T_GgSeqScan) return ((const GgSeqScan *) p)->numTargets > 0;
	if (p->type == T_GgHashJoin) return ((const GgHashJoin *) p)->numTargets > 0;
	if (p->type == T_GgMotion) return p->lefttree && p->lefttree->type == T_GgSeqScan && ((const GgSeqScan *) p->lefttree)->numTargets > 0;
	return 0;
}

/* the relation a SeqScan reads: resident on the device, or pages in host memory */
static int bind_relation(GgEState *es, const GgSeqScan *scan, gg_relation **rel, const void **host_pages, uint64_t *host_nblocks)
{
	*rel = NULL; *host_pages = NULL; *host_nblocks = 0;
	if (scan->scanrelid < 0 || scan->scanrelid >= GG_MAX_RELATIONS)
	{ exec_fail(GG_ERR_ARG, "SeqScan: relation %d out of range", scan->scanrelid); return -1; }
	if (es->relations[scan->scanrelid]) { *rel = es->relations[scan->scanrelid]; return 0; }
	if (es->host_pages[scan->scanrelid]) { *host_pages = es->host_pages[scan->scanrelid]; *host_nblocks = es->host_nblocks[scan->scanrelid]; return 0; }
	exec_fail(GG_ERR_ARG, "SeqScan: relation %d is neither resident on the device nor given as host pages", scan->scanrelid);
	return -1;
}

/* what a scan or join pipeline reads: a SeqScan's relation, or the datum rows of a row-producing node */
static int is_pipeline_input(const GgPlan *p) { return p && (p->type == T_GgSeqScan || yields_rows(p)); }

/* a join also reads the groups of an Agg, finalised into device datum rows (init_input checks that it can deliver them) */
static int is_join_input(const GgPlan *p) { return is_pipeline_input(p) || (p && p->type == T_GgAgg); }

static void mark_agg_rows(GgPlanState *ch);
static int agg_rows_desc(GgPlanState *s);

static int init_input(GgPlanState *s, GgPlan *p, int eflags, int depth, gg_scan *scan, GgPlanState **rows, gg_relation **rel)
{
	memset(scan, 0, sizeof *scan);
	if (p->type == T_GgAgg)
	{
		/* an Agg under a HashJoin hands up its groups as device rows, by the rule of an Agg under a Sort (mark_agg_rows) */
		GgPlanState *ch;
		if (!(ch = *rows = init_node(p, s->estate, eflags, depth))) return -1;
		mark_agg_rows(ch);
		if (!ch->agg_rows || !gg_relation_load)
		{
			exec_fail(GG_ERR_UNSUPPORTED, "HashJoin over an Agg: only a one-stage Agg over a scan or a join, or a FINAL Agg over device "
			          "group records, without numeric aggregates, delivers its groups as device rows");
			return -1;
		}
		if (!ch->having && agg_rows_desc(ch)) return -1;
		ch->rows_required = 1;
		scan->desc = ch->rows_desc; scan->qual = -1;
		return 0;
	}
	if (yields_rows(p))
	{
		if (!(*rows = init_node(p, s->estate, eflags, depth))) return -1;
		scan->desc = (*rows)->rows_desc; scan->qual = -1;
		return 0;
	}
	scan->desc = ((GgSeqScan *) p)->desc; scan->qual = p->qual;
	return bind_relation(s->estate, (GgSeqScan *) p, rel, &s->host_pages, &s->host_nblocks);
}

/* state of a rows-producing node (SeqScan with targets, optionally under a Redistribute Motion) */
static int init_rows_node(GgPlan *node, GgEState *estate, GgPlanState *s)
{
	GgSeqScan *sc = (GgSeqScan *) (node->type == T_GgMotion ? node->lefttree : node);
	const void *hp; uint64_t hn;
	int i;
	if (sc->numTargets < 1 || sc->numTargets > GG_MAX_OUTCOLS || sc->numTargets > 16)
	{ exec_fail(GG_ERR_UNSUPPORTED, "SeqScan projecting %d columns (1..16 travel as datum rows)", sc->numTargets); return -1; }
	if (bind_relation(estate, sc, &s->rel, &hp, &hn)) return -1;
	if (!s->rel) { exec_fail(GG_ERR_UNSUPPORTED, "a row-producing SeqScan needs its relation resident on the device"); return -1; }
	s->rows_scan = sc;
	s->rows_ncols = sc->numTargets;
	memset(&s->rows_desc, 0, sizeof s->rows_desc);
	s->rows_desc.natts = sc->numTargets;
	s->rows_desc.format = GG_FMT_DATUMROWS;
	for (i = 0; i < sc->numTargets; i++)
	{
		const int32_t root = sc->targets[i];
		const gg_expr *e;
		gg_attr *a = &s->rows_desc.attrs[i];
		if (root < 0 || root >= estate->pool->nnodes) { exec_fail(GG_ERR_ARG, "SeqScan target %d: node %d is not in the pool", i, root); return -1; }
		e = &estate->pool->nodes[root];
		s->rows_targets[i] = root;
		s->typid[i] = e->rettype;
		a->atttypid = e->rettype; a->atttypmod = -1; a->attlen = 8; a->attalign = 'd'; a->attbyval = 1;
		/* a plain Var of a NOT NULL column stays NOT NULL: lets the consumers run their NULL-free kernel variants */
		a->attnotnull = (e->kind == 1 /* GG_E_VAR */ && e->varattno >= 1 && e->varattno <= sc->desc.natts) ? sc->desc.attrs[e->varattno - 1].attnotnull : 0;
	}
	s->ncols = sc->numTargets;
	if (node->type == T_GgMotion)
	{
		GgMotion *mo = (GgMotion *) node;
		int c;
		if (mo->motionType != GG_MOTIONTYPE_HASH)
		{ exec_fail(GG_ERR_UNSUPPORTED, "only a Redistribute Motion moves scanned rows on the device"); return -1; }
		if (mo->numHashCols < 1 || mo->numHashCols > GG_MAX_KEYS)
		{ exec_fail(GG_ERR_UNSUPPORTED, "Redistribute Motion with %d hash columns", mo->numHashCols); return -1; }
		for (c = 0; c < mo->numHashCols; c++)
			if (mo->hashCol[c] < 0 || mo->hashCol[c] >= sc->numTargets)
			{ exec_fail(GG_ERR_ARG, "Motion hash column %d out of range (the scan projects %d columns)", mo->hashCol[c], sc->numTargets); return -1; }
		if (multi_segment(estate) && !estate->interconnect)
		{ exec_fail(GG_ERR_ARG, "Motion over a scan: %d segments but no device interconnect", estate->nsegs); return -1; }
		s->kind = K_MOTION;
		s->rows_nsegs = estate->nsegs > 0 ? estate->nsegs : 1;
	}
	else
	{
		s->kind = K_SCANROWS;
		s->rows_nsegs = 1;
	}
	return 0;
}

/* a HashJoin pipeline: fused with the Agg above it (agg != NULL, K_JOINAGG), or writing the rows of its target list (K_JOINROWS) */
static int init_join(GgPlanState *s, GgPlan *node, const gg_agg *agg, int eflags, int depth)
{
	GgEState *estate = s->estate;
	GgHashJoin *hj = (GgHashJoin *) node;
	GgPlan *outer = node->lefttree, *hash = node->righttree, *inner = hash ? hash->lefttree : NULL;
	gg_scan oscan, iscan;
	int rc, i;
	if (!agg && (!gg_joinrows_create || !gg_joinagg_rows))
	{ exec_fail(GG_ERR_UNSUPPORTED, "HashJoin with a target list: the device library has no join that writes its rows"); return -1; }
	if (!agg && (hj->numTargets > GG_MAX_OUTCOLS || hj->numTargets > 16))
	{ exec_fail(GG_ERR_UNSUPPORTED, "HashJoin projecting %d columns (1..16 travel as datum rows)", hj->numTargets); return -1; }
	if (!hash || hash->type != T_GgHash || !is_join_input(outer) || !is_join_input(inner))
	{
		exec_fail(GG_ERR_UNSUPPORTED, "HashJoin: both inputs must be a SeqScan, a Redistribute Motion over one, a HashJoin with a target "
		          "list or an Agg (Hash on the inner side)");
		return -1;
	}
	s->kind = agg ? K_JOINAGG : K_JOINROWS;
	if (init_input(s, outer, eflags, depth + 1, &oscan, &s->child, &s->rel)) return -1;
	if (!s->child && !s->rel) { exec_fail(GG_ERR_UNSUPPORTED, "HashJoin: the outer relation must be resident on the device"); return -1; }
	if (init_input(s, inner, eflags, depth + 2, &iscan, &s->inner, &s->inner_rel)) return -1;
	if (!s->inner && !s->inner_rel) { exec_fail(GG_ERR_UNSUPPORTED, "HashJoin: the inner relation must be resident on the device"); return -1; }
	if (agg)
	{
		rc = gg_joinagg_create(estate->engine, &oscan, &iscan, &hj->hj, agg, estate->pool, &s->ja);
		if (rc != GG_OK) { exec_fail(rc, "Agg <- HashJoin: %s", gg_last_error()); return -1; }
		s->dev_groups = 1;
		return 0;
	}
	rc = gg_joinrows_create(estate->engine, &oscan, &iscan, &hj->hj, hj->targets, hj->numTargets, estate->pool, &s->ja);
	if (rc != GG_OK) { exec_fail(rc, "HashJoin: %s", gg_last_error()); return -1; }
	/* the rows' descriptor: a column of the side a join null-extends is nullable; a plain Var of a NOT NULL column of the other
	 * side stays NOT NULL, as a scan's projection keeps it */
	s->rows_ncols = hj->numTargets;
	s->rows_nsegs = 1;
	s->ncols = hj->numTargets;
	memset(&s->rows_desc, 0, sizeof s->rows_desc);
	s->rows_desc.natts = hj->numTargets;
	s->rows_desc.format = GG_FMT_DATUMROWS;
	for (i = 0; i < hj->numTargets; i++)
	{
		const gg_expr *e = &estate->pool->nodes[hj->targets[i]];          /* checked by gg_joinrows_create */
		const int jt = hj->hj.jointype;
		const int nullext = e->varno == 0 ? (jt == GG_JOIN_RIGHT || jt == GG_JOIN_FULL) : (jt == GG_JOIN_LEFT || jt == GG_JOIN_FULL);
		const gg_tupdesc *d = e->varno == 0 ? &oscan.desc : &iscan.desc;
		gg_attr *a = &s->rows_desc.attrs[i];
		s->rows_targets[i] = hj->targets[i];
		s->typid[i] = e->rettype;
		a->atttypid = e->rettype; a->atttypmod = -1; a->attlen = 8; a->attalign = 'd'; a->attbyval = 1;
		a->attnotnull = (e->kind == 1 /* GG_E_VAR */ && !nullext && e->varattno >= 1 && e->varattno <= d->natts) ? d->attrs[e->varattno - 1].attnotnull : 0;
	}
	return 0;
}

static int has_numeric_agg(const gg_agg *agg)
{
	int i;
	for (i = 0; i < agg->numAggs; i++)
		if (agg->aggs[i].aggfnoid == GG_AGG_SUM_NUMERIC || agg->aggs[i].aggfnoid == GG_AGG_AVG_NUMERIC) return 1;
	return 0;
}

/* An Agg directly under a Sort or a Limit finalises its groups on the device into datum rows, which the node above sorts or
 * windows in place (only the Limit's window comes to the host).  Decided from the plan alone, so every segment decides alike:
 * a one-stage Agg over a scan or a join, or a FINAL Agg that combines device group records; no numeric aggregate (finalised on
 * the host only); and a device library with the entry points.  Otherwise the Agg hands up host rows, as it always did. */
static void mark_agg_rows(GgPlanState *ch)
{
	int ok;
	if (ch->having) return;                      /* decided at its own init: it always hands up (filtered) device rows */
	if (!gg_scanagg_datumrows || !gg_joinagg_datumrows || !gg_groups_datumrows) return;
	ok = ((ch->kind == K_SCANAGG || ch->kind == K_JOINAGG) && ch->agg.aggstage == GG_AGGSTAGE_NORMAL) ||
	     (ch->kind == K_AGGFINAL && ch->dev_groups);
	ch->agg_rows = ok && !has_numeric_agg(&ch->agg) && ch->agg.numCols + ch->agg.numAggs > 0;
}

/* The GG_FMT_DATUMROWS descriptor of an Agg's finalised rows: its output columns as set_layout_types types them.  NOT NULL
 * only where it is certain: count(*) and count(x) are never NULL; a key or any other aggregate may be (a NULL grouping value,
 * an aggregate over no non-NULL input).  A wrong NOT NULL would select a consumer's NULL-free kernel variant over NULLs. */
static int agg_rows_desc(GgPlanState *s)
{
	int c;
	if (set_layout_types(s)) return -1;
	if (s->ncols > GG_MAX_ATTS) { exec_fail(GG_ERR_UNSUPPORTED, "Agg with %d output columns (datum rows carry up to %d)", s->ncols, GG_MAX_ATTS); return -1; }
	memset(&s->rows_desc, 0, sizeof s->rows_desc);
	s->rows_desc.natts = s->ncols;
	s->rows_desc.format = GG_FMT_DATUMROWS;
	for (c = 0; c < s->ncols; c++)
	{
		gg_attr *a = &s->rows_desc.attrs[c];
		const int i = c - s->agg.numCols;
		a->atttypid = s->typid[c]; a->atttypmod = -1; a->attlen = 8; a->attalign = 'd'; a->attbyval = 1;
		a->attnotnull = i >= 0 && (s->agg.aggs[i].aggfnoid == GG_AGG_COUNT_STAR || s->agg.aggs[i].aggfnoid == GG_AGG_COUNT_ANY);
	}
	s->rows_ncols = s->ncols;
	return 0;
}

/* An Agg's HAVING (plan.qual; nodeAgg.c:1092 ExecQual over every finalised group).  Decided from the plan alone, so every
 * segment decides alike: the Agg always hands up its groups as device datum rows, filtered by the qual on the device
 * (gg_rowfilter); a FINAL Agg whose groups end up finalised on the host uploads them once and filters them the same way.  What
 * cannot take that path is refused: no path runs the Agg with its qual dropped. */
static int init_having(GgPlanState *s, int32_t qual)
{
	int rc;
	if (s->agg.aggstage == GG_AGGSTAGE_PARTIAL)
	{ exec_fail(GG_ERR_UNSUPPORTED, "a PARTIAL-stage Agg with a qual (HAVING belongs to the stage that finalises the groups)"); return -1; }
	if (has_numeric_agg(&s->agg))
	{ exec_fail(GG_ERR_UNSUPPORTED, "Agg with a qual: numeric aggregates have no device datum row to filter"); return -1; }
	if (s->agg.numCols + s->agg.numAggs < 1) { exec_fail(GG_ERR_UNSUPPORTED, "Agg with a qual and no output columns"); return -1; }
	if (!gg_rowfilter_create || !gg_rowfilter_run || !gg_rowfilter_free || !gg_relation_load || !gg_scanagg_datumrows || !gg_joinagg_datumrows ||
	    !gg_groups_datumrows)
	{ exec_fail(GG_ERR_UNSUPPORTED, "Agg with a qual: the device library has no row filter or no aggregate datum rows"); return -1; }
	if (agg_rows_desc(s)) return -1;
	rc = gg_rowfilter_create(s->estate->engine, &s->rows_desc, qual, s->estate->pool, &s->having);
	if (rc != GG_OK) { s->having = NULL; exec_fail(rc, "Agg qual: %s", gg_last_error()); return -1; }
	s->agg_rows = 1;
	if (s->kind != K_AGGFINAL) s->dev_groups = 0;     /* a FINAL Agg keeps dev_groups: it says how it combines its input */
	return 0;
}

/* The GG_FMT_DATUMROWS descriptor of the rows a node hands up, known at init: a row producer's own, an Agg's output columns,
 * and through a Sort, a Limit or a Motion that of the node below */
static int node_rows_desc(GgPlanState *s, gg_tupdesc *d)
{
	if (s->kind == K_SORT || s->kind == K_LIMIT || (s->kind == K_MOTION && !s->rows_scan)) return node_rows_desc(s->child, d);
	if (s->kind == K_SCANAGG || s->kind == K_JOINAGG || s->kind == K_AGGFINAL)
	{
		/* the descriptor of its output columns (a HAVING's init made it already); an Agg that hands up host rows keeps no row width */
		if (!s->having && agg_rows_desc(s)) return -1;
		if (!s->agg_rows) s->rows_ncols = 0;
	}
	else if (s->kind != K_SCANROWS && s->kind != K_MOTION && s->kind != K_JOINROWS && s->kind != K_WINDOW)
	{ exec_fail(GG_ERR_UNSUPPORTED, "WindowAgg: node kind %d below it delivers no rows", s->kind); return -1; }
	*d = s->rows_desc;
	return 0;
}

/* whether the plan below a WindowAgg delivers its order: a Sort whose leading keys are the partition columns, then the order
 * columns (possibly under other WindowAggs, which keep their input's order and columns); anything without keys */
static int window_order_ok(const GgPlan *child, const gg_window *w)
{
	const GgSort *so;
	int k;
	if (w->partNumCols + w->ordNumCols == 0) return 1;
	while (child && child->type == T_GgWindowAgg) child = child->lefttree;
	if (!child || child->type != T_GgSort) return 0;
	so = (const GgSort *) child;
	if (so->numCols < w->partNumCols + w->ordNumCols) return 0;
	for (k = 0; k < w->partNumCols; k++) if (so->keys[k].col != w->partColIdx[k]) return 0;
	for (k = 0; k < w->ordNumCols; k++) if (so->keys[w->partNumCols + k].col != w->ordColIdx[k]) return 0;
	return 1;
}

/* WindowAgg (nodeWindowAgg.c ExecInitWindowAgg): checked against the device's subset and created over the child's rows; its rows
 * are the child's columns followed by one column per function, handed up as device datum rows */
static int init_window(GgPlanState *s, GgPlan *node, int eflags, int depth)
{
	GgWindowAgg *wn = (GgWindowAgg *) node;
	const gg_window *w = &wn->win;
	GgEState *es = s->estate;
	gg_tupdesc in;
	int i, a, rc;
	s->kind = K_WINDOW;
	if (!gg_window_create || !gg_window_run || !gg_window_free || !gg_relation_load)
	{ exec_fail(GG_ERR_UNSUPPORTED, "WindowAgg: the device library has no window functions"); return -1; }
	if (node->qual != -1 && (!gg_rowfilter_create || !gg_rowfilter_run || !gg_rowfilter_free))
	{ exec_fail(GG_ERR_UNSUPPORTED, "WindowAgg with a qual: the device library has no row filter"); return -1; }
	if (w->numFuncs < 1 || w->numFuncs > GG_MAX_WINFUNCS)
	{ exec_fail(GG_ERR_UNSUPPORTED, "WindowAgg with %d window functions (1..%d)", w->numFuncs, GG_MAX_WINFUNCS); return -1; }
	for (i = 0; i < w->numFuncs; i++)
	{
		const int32_t fn = w->funcs[i].winfnoid;
		if (fn == GG_AGG_SUM_NUMERIC || fn == GG_AGG_AVG_NUMERIC)
		{ exec_fail(GG_ERR_UNSUPPORTED, "WindowAgg: numeric aggregates have no device datum row"); return -1; }
		for (a = 0; a < 3; a++)
		{
			const int32_t root = w->funcs[i].arg[a];
			const gg_expr *x;
			if (root < 0) continue;
			if (root >= es->pool->nnodes) { exec_fail(GG_ERR_ARG, "WindowAgg: argument node %d is not in the pool", root); return -1; }
			x = &es->pool->nodes[root];
			if (x->kind != GG_E_VAR && x->kind != GG_E_CONST)
			{ exec_fail(GG_ERR_UNSUPPORTED, "WindowAgg: argument %d of function %d is neither a Var nor a Const", a + 1, i + 1); return -1; }
			if (a == 0 && is_string_type(x->rettype) && fn != GG_AGG_COUNT_ANY && (fn < GG_WF_ROW_NUMBER || fn > GG_WF_NTH_VALUE))
			{ exec_fail(GG_ERR_UNSUPPORTED, "WindowAgg: string aggregates have no device datum row"); return -1; }
		}
	}
	if (!window_order_ok(node->lefttree, w))
	{
		exec_fail(GG_ERR_UNSUPPORTED, "WindowAgg: the node below must be a Sort on the partition columns, then the order columns");
		return -1;
	}
	if (!(s->child = init_node(node->lefttree, es, eflags, depth + 1))) return -1;
	mark_agg_rows(s->child);
	if (node_rows_desc(s->child, &in)) return -1;
	if (in.natts + w->numFuncs > GG_MAX_ATTS)
	{ exec_fail(GG_ERR_UNSUPPORTED, "WindowAgg with %d output columns (datum rows carry up to %d)", in.natts + w->numFuncs, GG_MAX_ATTS); return -1; }
	rc = gg_window_create(es->engine, &in, w, es->pool, &s->win);
	if (rc != GG_OK) { s->win = NULL; exec_fail(rc, "WindowAgg: %s", gg_last_error()); return -1; }
	s->rows_desc = in;
	for (i = 0; i < in.natts; i++) s->typid[i] = in.attrs[i].atttypid;
	for (i = 0; i < w->numFuncs; i++)
	{
		gg_attr *at = &s->rows_desc.attrs[in.natts + i];
		memset(at, 0, sizeof *at);
		at->atttypid = w->funcs[i].wintype; at->atttypmod = -1; at->attlen = 8; at->attalign = 'd'; at->attbyval = 1;
		s->typid[in.natts + i] = w->funcs[i].wintype;
	}
	s->rows_desc.natts = in.natts + w->numFuncs;
	s->ncols = s->rows_ncols = s->rows_desc.natts;
	s->rows_nsegs = 1;
	if (node->qual != -1)
	{
		rc = gg_rowfilter_create(es->engine, &s->rows_desc, node->qual, es->pool, &s->having);
		if (rc != GG_OK) { s->having = NULL; exec_fail(rc, "WindowAgg qual: %s", gg_last_error()); return -1; }
	}
	return 0;
}

static GgPlanState *init_node(GgPlan *node, GgEState *estate, int eflags, int depth)
{
	GgPlanState *s;
	if (!node) return NULL;                                   /* ExecInitNode(NULL) is NULL, execProcnode.c:268 */
	if (!estate || !estate->engine || !estate->pool) return exec_fail(GG_ERR_ARG, "EState without engine or expression pool");
	if (depth > GG_MAX_PLAN_DEPTH) return exec_fail(GG_ERR_ARG, "plan tree deeper than %d nodes (a cycle?)", GG_MAX_PLAN_DEPTH);
	s = calloc(1, sizeof *s);
	if (!s) return exec_fail(GG_ERR_NOMEM, "out of memory");
	s->plan = node; s->estate = estate;
	if (node->type == T_GgWindowAgg)
	{
		if (init_window(s, node, eflags, depth)) goto fail;
		return s;
	}
	if (yields_rows(node))
	{
		if (node->type == T_GgHashJoin ? init_join(s, node, NULL, eflags, depth) : init_rows_node(node, estate, s)) goto fail;
		return s;
	}
	switch (node->type)
	{
		case T_GgAgg:
		{
			GgAgg *an = (GgAgg *) node;
			GgPlan *below = node->lefttree;
			int rc;
			s->agg = an->agg;
			if (an->agg.numCols < 0 || an->agg.numCols > GG_MAX_KEYS || an->agg.numAggs < 0 || an->agg.numAggs > GG_MAX_AGGS)
			{
				exec_fail(GG_ERR_ARG, "Agg with %d grouping columns and %d aggregates", an->agg.numCols, an->agg.numAggs);
				goto fail;
			}
			if (an->agg.aggstage == GG_AGGSTAGE_FINAL)
			{
				/* the receiving half of a two-stage aggregate: combine what the Motion below delivers */
				s->kind = K_AGGFINAL;
				s->child = init_node(below, estate, eflags, depth + 1);
				if (!s->child) goto fail;
				{
					/* device path: the child delivers group records of a PARTIAL stage with these very aggregates */
					const GgPlanState *ch = s->child;
					int i, same = ch->dev_groups && ch->agg.aggstage == GG_AGGSTAGE_PARTIAL && ch->agg.numAggs == an->agg.numAggs && ch->agg.numCols == an->agg.numCols;
					for (i = 0; same && i < an->agg.numAggs; i++) same = ch->agg.aggs[i].aggfnoid == an->agg.aggs[i].aggfnoid;
					s->dev_groups = same;
				}
				goto agg_qual;
			}
			/* a HashJoin directly below stays fused with this Agg, whether it has a target list or not */
			if (below && below->type == T_GgHashJoin)
			{
				if (init_join(s, below, &an->agg, eflags, depth)) goto fail;
				goto agg_qual;
			}
			if (is_pipeline_input(below))
			{
				gg_scan scan;
				s->kind = K_SCANAGG;
				if (init_input(s, below, eflags, depth + 1, &scan, &s->child, &s->rel)) goto fail;
				rc = gg_scanagg_create(estate->engine, &scan, &an->agg, estate->pool, &s->sa);
				if (rc != GG_OK) { exec_fail(rc, "Agg <- SeqScan: %s", gg_last_error()); goto fail; }
				s->dev_groups = 1;
				goto agg_qual;
			}
			exec_fail(GG_ERR_UNSUPPORTED, "Agg: child node type %d is not on the accelerated path", below ? (int) below->type : 0);
			goto fail;
		agg_qual:
			if (node->qual != -1 && init_having(s, node->qual)) goto fail;
			return s;
		}
		case T_GgSort:
		{
			GgSort *so = (GgSort *) node;
			if (so->numCols < 1 || so->numCols > GG_MAX_SORTKEYS) { exec_fail(GG_ERR_UNSUPPORTED, "Sort with %d keys", so->numCols); goto fail; }
			s->kind = K_SORT;
			s->sort_bound = GG_NO_BOUND;
			s->child = init_node(node->lefttree, estate, eflags, depth + 1);
			if (!s->child) goto fail;
			mark_agg_rows(s->child);
			return s;
		}
		case T_GgLimit:
			if (!node->lefttree) { exec_fail(GG_ERR_ARG, "Limit without a child"); goto fail; }
			if (node->lefttree->type == T_GgSort && (!gg_sort_rows_bounded || !gg_sort_datumrows_bounded))
			{ exec_fail(GG_ERR_UNSUPPORTED, "Limit over a Sort: the device library has no bounded sort"); goto fail; }
			s->kind = K_LIMIT;
			s->child = init_node(node->lefttree, estate, eflags, depth + 1);
			if (!s->child) goto fail;
			mark_agg_rows(s->child);
			return s;
		case T_GgMotion:
		{
			GgMotion *mo = (GgMotion *) node;
			if (!estate->transport && !estate->interconnect && multi_segment(estate))
			{ exec_fail(GG_ERR_ARG, "Motion: %d segments but neither an interconnect nor a transport", estate->nsegs); goto fail; }
			if (mo->motionType == GG_MOTIONTYPE_HASH && (mo->numHashCols < 1 || mo->numHashCols > GG_MAX_KEYS))
			{ exec_fail(GG_ERR_UNSUPPORTED, "Redistribute Motion with %d hash columns", mo->numHashCols); goto fail; }
			s->kind = K_MOTION;
			s->child = init_node(node->lefttree, estate, eflags, depth + 1);
			if (!s->child) goto fail;
			s->agg = s->child->agg;
			{
				/* aggregate rows move as device-resident group records when the rows below are such records, the hash columns
				 * are grouping columns, and the receiver does not merge sorted streams */
				int c, ok = estate->interconnect != NULL && s->child->dev_groups && !s->child->having && mo->numSortCols == 0;
				for (c = 0; ok && mo->motionType == GG_MOTIONTYPE_HASH && c < mo->numHashCols; c++)
					ok = mo->hashCol[c] >= 0 && mo->hashCol[c] < s->child->agg.numCols;
				s->dev_groups = ok;
				if (ok && (s->child->kind == K_SCANAGG || s->child->kind == K_JOINAGG)) s->child->lazy_fetch = 1;
			}
			return s;
		}
		case T_GgSeqScan:
			exec_fail(GG_ERR_UNSUPPORTED, "a SeqScan without a target list is only accelerated underneath an Agg or a HashJoin");
			goto fail;
		case T_GgHashJoin:
			/* no target list: nothing says which columns its rows would have (one with a target list yields rows, above) */
			exec_fail(GG_ERR_UNSUPPORTED, "a HashJoin is only accelerated underneath an Agg (the join is never materialised)");
			goto fail;
		case T_GgHash:
			s->kind = K_HASH;          /* marker: the build is part of the join's pipeline */
			return s;
		case T_GgWindowAgg:
			break;                     /* handled above */
	}
	exec_fail(GG_ERR_UNSUPPORTED, "unknown node type %d", (int) node->type);
fail:
	end_tree(s);
	return NULL;
}

/* ---- external sort of host rows ----
 * tuplesort_mk.c: rows beyond the operator's memory go to sorted runs on tape (puttuple -> dumptuples, :1154,:2390) and the
 * runs are merged through a heap of their heads (mergeruns / mergeonerun, :2019).  Here a run is as many rows as the operator's
 * memory holds, sorted on the device (gg_sort_rows: the stable radix sort of gg_sort.cu); the runs stay in host memory — where
 * the reference writes its workfile — and a heap merges them.  The merge compares rows by the same order-preserving keys the
 * device sorts by, so the outcome is what one big sort would have produced, ties included (runs are consecutive input ranges,
 * a run's order is stable, and between runs the earlier one wins a tie). */
static uint64_t sort_radix_key(int64_t v, int32_t typid, int desc)
{
	uint64_t k;
	switch (typid)
	{
		case GG_INT4OID: case GG_DATEOID:
			k = (uint64_t) (int64_t) (int32_t) v ^ 0x8000000000000000ull;
			break;
		case GG_FLOAT8OID:
		{
			double d;
			memcpy(&d, &v, 8);
			if (d != d) k = ~0ull;                                   /* NaN sorts after everything (float8_cmp_internal, float.c:964) */
			else
			{
				if (d == 0.0) v = 0;                                 /* -0 = +0 */
				k = (uint64_t) v;
				k = (k >> 63) ? ~k : (k ^ 0x8000000000000000ull);
			}
			break;
		}
		case GG_BPCHAROID: case GG_VARCHAROID: case GG_TEXTOID:
			k = __builtin_bswap64((uint64_t) v);                     /* packed bytes, first character most significant */
			break;
		default:
			k = (uint64_t) v ^ 0x8000000000000000ull;
			break;
	}
	return desc ? ~k : k;
}

/* < 0, 0, > 0: row a against row b of the same row array under the sort keys */
static int sort_row_cmp(const gg_sortkey *keys, int nkeys, int ncols, const int64_t *values, const uint8_t *isnull, uint64_t a, uint64_t b)
{
	int k;
	for (k = 0; k < nkeys; k++)
	{
		const int c = keys[k].col;
		const int na = isnull[a * (uint64_t) ncols + c] != 0, nb = isnull[b * (uint64_t) ncols + c] != 0;
		const int da = na ? (keys[k].nulls_first ? 0 : 1) : (keys[k].nulls_first ? 1 : 0);
		const int db = nb ? (keys[k].nulls_first ? 0 : 1) : (keys[k].nulls_first ? 1 : 0);
		uint64_t ka, kb;
		if (da != db) return da < db ? -1 : 1;
		if (na) continue;                                         /* both NULL: equal on this key */
		ka = sort_radix_key(values[a * (uint64_t) ncols + c], keys[k].typid, keys[k].desc);
		kb = sort_radix_key(values[b * (uint64_t) ncols + c], keys[k].typid, keys[k].desc);
		if (ka != kb) return ka < kb ? -1 : 1;
	}
	return 0;
}

typedef struct { uint64_t pos, end; } SortRun;         /* the run's head and its end, as indices into perm[] */

/* perm[] = the sorted order of `n` rows: run by run through gg_sort_rows, then merged.  run_rows >= 1.  With a bound (a Limit
 * above), every run keeps only its first `bound` rows (gg_sort_rows_bounded) and the merge stops after `bound` rows. */
static int sort_rows_external(gg_engine *eng, const gg_sortkey *keys, int nkeys, int ncols, const int64_t *values, const uint8_t *isnull,
                              uint64_t n, uint64_t run_rows, uint64_t bound, uint64_t *perm, int *nruns_out)
{
	const uint64_t nruns = (n + run_rows - 1) / run_rows;
	uint64_t *runperm, r, i, out = 0;
	SortRun *runs;
	uint32_t *heap;                                             /* run numbers, smallest head on top */
	uint32_t hn = 0;
	int rc = GG_OK;
	if (nruns_out) *nruns_out = (int) nruns;
	if (nruns > 0x7FFFFFFFu) return GG_ERR_UNSUPPORTED;
	runperm = malloc(8 * (size_t) (n ? n : 1));
	runs = malloc(sizeof *runs * (size_t) (nruns ? nruns : 1));
	heap = malloc(4 * (size_t) (nruns ? nruns : 1));
	if (!runperm || !runs || !heap) { free(runperm); free(runs); free(heap); return GG_ERR_NOMEM; }
	for (r = 0; r < nruns && rc == GG_OK; r++)
	{
		const uint64_t first = r * run_rows, len = first + run_rows <= n ? run_rows : n - first;
		uint64_t kept = len;
		if (bound < len)
			rc = gg_sort_rows_bounded(eng, keys, nkeys, ncols, values + first * (uint64_t) ncols, isnull + first * (uint64_t) ncols, len, bound,
			                          runperm + first, &kept);
		else
			rc = gg_sort_rows(eng, keys, nkeys, ncols, values + first * (uint64_t) ncols, isnull + first * (uint64_t) ncols, len, runperm + first);
		for (i = 0; i < kept && rc == GG_OK; i++) runperm[first + i] += first;     /* row numbers of the whole input */
		runs[r].pos = first; runs[r].end = first + kept;
	}
	if (rc == GG_OK)
	{
		/* build the heap of run heads, then pop the smallest head, advance its run, sift down: mergeonerun */
		for (r = 0; r < nruns; r++)
		{
			uint32_t at;
			if (runs[r].pos == runs[r].end) continue;
			at = hn++;
			heap[at] = (uint32_t) r;
			while (at > 0)
			{
				const uint32_t up = (at - 1) / 2;
				const int c = sort_row_cmp(keys, nkeys, ncols, values, isnull, runperm[runs[heap[at]].pos], runperm[runs[heap[up]].pos]);
				if (c > 0 || (c == 0 && heap[at] > heap[up])) break;
				{ const uint32_t t = heap[at]; heap[at] = heap[up]; heap[up] = t; }
				at = up;
			}
		}
		while (hn > 0 && out < bound)
		{
			const uint32_t top = heap[0];
			uint32_t at = 0;
			perm[out++] = runperm[runs[top].pos++];
			if (runs[top].pos == runs[top].end) heap[0] = heap[--hn];
			for (;;)
			{
				uint32_t l = 2 * at + 1, rr = l + 1, m = at;
				if (l < hn)
				{
					const int c = sort_row_cmp(keys, nkeys, ncols, values, isnull, runperm[runs[heap[l]].pos], runperm[runs[heap[m]].pos]);
					if (c < 0 || (c == 0 && heap[l] < heap[m])) m = l;
				}
				if (rr < hn)
				{
					const int c = sort_row_cmp(keys, nkeys, ncols, values, isnull, runperm[runs[heap[rr]].pos], runperm[runs[heap[m]].pos]);
					if (c < 0 || (c == 0 && heap[rr] < heap[m])) m = rr;
				}
				if (m == at) break;
				{ const uint32_t t = heap[at]; heap[at] = heap[m]; heap[m] = t; }
				at = m;
			}
		}
	}
	free(runperm); free(runs); free(heap);
	return rc;
}

/* keys[] = a plan's sort keys, checked against the columns of the rows they sort; a key without a type takes its column's */
static int sort_keys(gg_sortkey *keys, const gg_sortkey *plan_keys, int nkeys, const GgPlanState *src, const char *what)
{
	int k;
	for (k = 0; k < nkeys; k++)
	{
		keys[k] = plan_keys[k];
		if (keys[k].col < 0 || keys[k].col >= src->ncols) { exec_fail(GG_ERR_ARG, "%s key column %d out of range", what, keys[k].col); return -1; }
		if (!keys[k].typid) keys[k].typid = src->typid[keys[k].col];
	}
	return 0;
}

/* the result of s = the host rows of src (s itself, or the node below) in the order of keys[]; with run_rows > 0 and more
 * rows than that, sorted externally and s->sort_runs counts the runs.  With a bound, only the first `bound` rows of that order. */
static int sort_host_rows(GgPlanState *s, const GgPlanState *src, const gg_sortkey *keys, int nkeys, uint64_t run_rows, uint64_t bound)
{
	const int64_t n = src->nrows > 0 && (uint64_t) src->nrows > bound ? (int64_t) bound : src->nrows;     /* rows of the result */
	const int32_t ncols = src->ncols;
	const size_t cells = (size_t) (n > 0 ? n : 1) * (size_t) ncols;
	uint64_t *perm = malloc(8 * (size_t) (n > 0 ? n : 1));
	int64_t *v = malloc(8 * cells);
	uint8_t *nl = malloc(cells);
	int32_t *ln = malloc(4 * cells);
	int64_t r;
	uint64_t kept = 0;
	int rc = GG_ERR_NOMEM;
	if (perm && v && nl && ln)
	{
		if (run_rows && (uint64_t) src->nrows > run_rows && bound > run_rows)
			rc = sort_rows_external(s->estate->engine, keys, nkeys, ncols, src->values, src->isnull, (uint64_t) src->nrows, run_rows, bound, perm, &s->sort_runs);
		else if (n < src->nrows)
			rc = gg_sort_rows_bounded(s->estate->engine, keys, nkeys, ncols, src->values, src->isnull, (uint64_t) src->nrows, bound, perm, &kept);
		else
			rc = gg_sort_rows(s->estate->engine, keys, nkeys, ncols, src->values, src->isnull, (uint64_t) n, perm);
	}
	if (rc != GG_OK)
	{
		exec_fail(rc, "%s", rc == GG_ERR_NOMEM ? "out of memory" : gg_last_error());
		free(perm); free(v); free(nl); free(ln);
		return -1;
	}
	for (r = 0; r < n; r++)
	{
		memcpy(v + (size_t) r * ncols, src->values + (size_t) perm[r] * ncols, 8 * (size_t) ncols);
		memcpy(nl + (size_t) r * ncols, src->isnull + (size_t) perm[r] * ncols, (size_t) ncols);
		memcpy(ln + (size_t) r * ncols, src->lens + (size_t) perm[r] * ncols, 4 * (size_t) ncols);
	}
	free(perm);
	free(s->values); free(s->isnull); free(s->lens);
	s->values = v; s->isnull = nl; s->lens = ln;
	s->nrows = n; s->ncols = ncols; s->next = 0; s->markpos = 0;
	return 0;
}

static int run_node(GgPlanState *s);
static int ensure_rows(GgPlanState *s);

static int run_child(GgPlanState *s)
{
	if (s->child && !s->child->done && run_node(s->child)) return -1;
	return 0;
}

/* ---- datum rows on the device: SeqScan projection, optionally partitioned for a Redistribute Motion ---- */
static int run_rows_node(GgPlanState *s)
{
	GgEState *es = s->estate;
	GgSeqScan *sc = s->rows_scan;
	const int N = s->rows_nsegs;
	const int W = 1 + s->rows_ncols;
	const uint64_t nblocks = gg_relation_nblocks(s->rel);
	gg_scan scan;
	int32_t hashkeys[GG_MAX_KEYS];
	int nkeys = 0, c, rc, attempt;
	uint64_t counts[1024], offs[1024];
	if (N > 1024) { exec_fail(GG_ERR_UNSUPPORTED, "more than 1024 segments"); return -1; }
	memset(&scan, 0, sizeof scan);
	scan.desc = sc->desc; scan.qual = sc->plan.qual;
	if (s->kind == K_MOTION)
	{
		GgMotion *mo = (GgMotion *) s->plan;
		for (c = 0; c < mo->numHashCols; c++) hashkeys[nkeys++] = s->rows_targets[mo->hashCol[c]];
	}
	else
		hashkeys[nkeys++] = s->rows_targets[0];          /* one destination: the key only feeds jump_consistent_hash(h, 1) = 0 */
	drop_device_results(s);
	for (attempt = 0; ; attempt++)
	{
		if (!s->rows_send)
		{
			uint64_t words;
			if (!s->rows_cap)
			{
				/* the line pointers bound the rows; a hash spreads them evenly over the destinations (10 % + 8192 slack each) */
				uint64_t nlp = 0;
				rc = gg_relation_count_rows(s->rel, &nlp);
				if (rc != GG_OK) { exec_fail(rc, "%s", gg_last_error()); return -1; }
				/* + 1/4: a hash does not spread perfectly, and the sending kernel leaves up to 1/8 of a region as dead slots */
				s->rows_cap = (nlp / (uint64_t) N + nlp / (uint64_t) (4 * N) + 8192) * (uint64_t) N;
			}
			words = s->rows_cap * (uint64_t) W + 8;
			rc = gg_relation_create(es->engine, (words * 8 + GG_BLCKSZ - 1) / GG_BLCKSZ, &s->rows_send);
			if (rc != GG_OK) { exec_fail(rc, "Motion send buffer: %s", gg_last_error()); return -1; }
		}
		rc = gg_motion_partition(es->engine, &scan, es->pool, hashkeys, nkeys, s->rows_targets, s->rows_ncols, N, s->rel, 0, nblocks,
		                         gg_relation_device_ptr(s->rows_send), s->rows_cap, counts, offs);
		if (rc != GG_ERR_NOMEM || attempt >= 2) break;
		gg_relation_free(s->rows_send); s->rows_send = NULL;
		s->rows_cap *= 2;
	}
	if (rc != GG_OK) { exec_fail(rc, "%s", gg_last_error()); return -1; }
	if (N == 1)
	{
		s->rows_n = counts[0];
		rc = gg_relation_attach_rows(es->engine, gg_relation_device_ptr(s->rows_send), s->rows_n, s->rows_ncols, &s->rows_rel);
		if (rc != GG_OK) { exec_fail(rc, "%s", gg_last_error()); return -1; }
		return 0;
	}
	for (attempt = 0; ; attempt++)
	{
		const uint64_t region_cap = (s->rows_cap / (uint64_t) N) & ~1ull;
		uint64_t recv_cap;
		if (!s->rows_recv)
		{
			rc = gg_relation_create(es->engine, ((s->rows_cap * (uint64_t) W + 8) * 8 + GG_BLCKSZ - 1) / GG_BLCKSZ, &s->rows_recv);
			if (rc != GG_OK) { exec_fail(rc, "Motion receive buffer: %s", gg_last_error()); return -1; }
		}
		recv_cap = gg_relation_nblocks(s->rows_recv) * (uint64_t) GG_BLCKSZ / 8 / (uint64_t) W - 2;
		rc = gg_ic_exchange_rows(es->interconnect, gg_relation_device_ptr(s->rows_send), counts, region_cap, W,
		                         gg_relation_device_ptr(s->rows_recv), recv_cap, &s->rows_n);
		if (rc != GG_ERR_NOMEM || attempt >= 1) break;
		/* every segment saw the overflow: all of them come back with a receive buffer twice the size */
		{
			const uint64_t nb = gg_relation_nblocks(s->rows_recv) * 2;
			gg_relation_free(s->rows_recv); s->rows_recv = NULL;
			rc = gg_relation_create(es->engine, nb, &s->rows_recv);
			if (rc != GG_OK) { exec_fail(rc, "Motion receive buffer: %s", gg_last_error()); return -1; }
		}
	}
	if (rc != GG_OK) { exec_fail(rc, "%s", gg_last_error()); return -1; }
	rc = gg_relation_attach_rows(es->engine, gg_relation_device_ptr(s->rows_recv), s->rows_n, s->rows_ncols, &s->rows_rel);
	if (rc != GG_OK) { exec_fail(rc, "%s", gg_last_error()); return -1; }
	return 0;
}

/* the device buffer that holds a rows node's datum rows */
static gg_relation *rows_buffer(const GgPlanState *s)
{
	if (s->kind == K_JOINROWS || s->kind == K_WINDOW || s->agg_rows) return s->rows_rel;   /* the join's / window's / Agg's own output */
	return s->rows_recv && s->rows_nsegs > 1 ? s->rows_recv : s->rows_send;
}

/* device rows -> host result arrays (only when a rows node sits at the top of what the caller drives) */
static int rows_to_host(GgPlanState *s)
{
	const int W = 1 + s->rows_ncols;
	const uint64_t n = s->rows_n;
	const uint64_t bytes = n * (uint64_t) W * 8;
	const uint64_t nb = (bytes + GG_BLCKSZ - 1) / GG_BLCKSZ;
	uint64_t *buf, r;
	int c, rc;
	if (alloc_result(s, (int64_t) n, s->rows_ncols)) { exec_fail(GG_ERR_NOMEM, "out of memory"); return -1; }
	if (n)
	{
		uint64_t live = 0;
		buf = malloc((size_t) nb * GG_BLCKSZ);
		if (!buf) { exec_fail(GG_ERR_NOMEM, "out of memory"); return -1; }
		rc = gg_relation_read(rows_buffer(s), 0, buf, nb);
		if (rc != GG_OK) { free(buf); exec_fail(rc, "%s", gg_last_error()); return -1; }
		for (r = 0; r < n; r++)
		{
			if (buf[r * W] & GG_DATUMROW_DEAD) continue;          /* a slot the sending kernel claimed and did not fill */
			for (c = 0; c < s->rows_ncols; c++)
			{
				const uint64_t v = buf[r * W + 1 + c];
				s->values[live * s->rows_ncols + c] = (int64_t) v;
				s->isnull[live * s->rows_ncols + c] = (uint8_t) ((buf[r * W] >> c) & 1);
				if (is_string_type(s->typid[c])) s->lens[live * s->rows_ncols + c] = packed_len(v);
			}
			live++;
		}
		s->nrows = (int64_t) live;
		free(buf);
	}
	s->rows_ready = 1;
	return 0;
}

/* a failure reading a node's aggregate rows: this segment's own earlier failure, when there was one, is the better message */
static void groups_fail(const GgPlanState *s, int rc)
{
	if (s->groups && g_local_code && rc != GG_ERR_RETRY_HOST) exec_fail(g_local_code, "%s", g_local_err);
	else exec_fail(rc, "%s", gg_last_error());
}

/* an Agg's s->rows_n finalised rows (a datum-row view) handed up as s->rows_rel: through its HAVING filter first, when it has one,
 * so that only the groups whose qual is TRUE reach the node above */
static int hand_up_rows(GgPlanState *s, gg_relation *rows)
{
	int rc = GG_OK;
	s->rows_ncols = s->ncols;
	s->rows_nsegs = 1;
	if (s->having) rc = gg_rowfilter_run(s->having, rows, s->rows_n, &rows, &s->rows_n);
	if (rc == GG_OK) rc = gg_relation_attach_rows(s->estate->engine, gg_relation_device_ptr(rows), s->rows_n, s->rows_ncols, &s->rows_rel);
	if (rc != GG_OK) { s->rows_rel = NULL; exec_fail(rc, "%s", gg_last_error()); return -1; }
	s->rows_ready = 0;
	return 0;
}

/* the Agg's groups as device datum rows (agg_rows): the view its pipeline or group set hands out, wrapped for the node above */
static int agg_datumrows(GgPlanState *s)
{
	gg_relation *out = NULL;
	int rc;
	if (set_layout_types(s)) return -1;
	if (s->groups) rc = gg_groups_datumrows(s->groups, &out, &s->rows_n);
	else if (s->kind == K_SCANAGG) rc = gg_scanagg_datumrows(s->sa, &out, &s->rows_n);
	else rc = gg_joinagg_datumrows(s->ja, &out, &s->rows_n);
	if (rc != GG_OK) { groups_fail(s, rc); return -1; }
	return hand_up_rows(s, out);
}

/* the host rows of src uploaded once as datum rows into s->rows_send; *view wraps them (the caller frees it) */
static int upload_host_rows(GgPlanState *s, const GgPlanState *src, gg_relation **view)
{
	GgEState *es = s->estate;
	const uint64_t n = src->nrows > 0 ? (uint64_t) src->nrows : 0, W = 1 + (uint64_t) src->ncols;
	const uint64_t nb = (n * W * 8 + 16 + GG_BLCKSZ - 1) / GG_BLCKSZ;
	uint64_t *buf, r;
	int c, rc;
	*view = NULL;
	if (s->rows_send && gg_relation_nblocks(s->rows_send) < nb) { gg_relation_free(s->rows_send); s->rows_send = NULL; }
	if (!s->rows_send && (rc = gg_relation_create(es->engine, nb, &s->rows_send)) != GG_OK)
	{ s->rows_send = NULL; exec_fail(rc, "rows: %s", gg_last_error()); return -1; }
	buf = calloc((size_t) nb, GG_BLCKSZ);
	if (!buf) { exec_fail(GG_ERR_NOMEM, "out of memory"); return -1; }
	for (r = 0; r < n; r++)
		for (c = 0; c < src->ncols; c++)
		{
			buf[r * W] |= (uint64_t) (src->isnull[r * (uint64_t) src->ncols + c] != 0) << c;
			buf[r * W + 1 + c] = (uint64_t) src->values[r * (uint64_t) src->ncols + c];
		}
	rc = gg_relation_load(s->rows_send, 0, buf, nb);              /* pageable: staged before the call returns, so buf can go */
	free(buf);
	if (rc == GG_OK) rc = gg_relation_attach_rows(es->engine, gg_relation_device_ptr(s->rows_send), n, src->ncols, view);
	if (rc != GG_OK) { *view = NULL; exec_fail(rc, "rows: %s", gg_last_error()); return -1; }
	return 0;
}

/* A FINAL Agg whose groups were finalised on the host (its child delivered host rows, or the slice was re-run with host-row
 * Motions), under a HAVING filter or a HashJoin: its host rows uploaded once as datum rows (into rows_send) and handed up as the
 * device path hands them up, so the qual is evaluated one way only */
static int upload_agg_rows(GgPlanState *s)
{
	gg_relation *view = NULL;
	int rc;
	if (upload_host_rows(s, s, &view)) return -1;
	s->rows_n = s->nrows > 0 ? (uint64_t) s->nrows : 0;
	rc = hand_up_rows(s, view);
	gg_relation_free(view);
	return rc;
}

/* WindowAgg: the child's sorted rows windowed where they are (or, when they ended up on the host, uploaded once), then through
 * the qual when there is one; the result stays on the device for the node above */
static int run_window(GgPlanState *s)
{
	GgEState *es = s->estate;
	GgPlanState *ch = s->child;
	gg_relation *in = NULL, *up = NULL, *out = NULL;
	uint64_t nin, nout = 0;
	int rc;
	drop_device_results(s);
	if (run_child(s)) return -1;
	s->nonreceiver = ch->nonreceiver;
	if (ch->rows_rel && !ch->rows_ready) { in = ch->rows_rel; nin = ch->rows_n; }
	else
	{
		if (ensure_rows(ch) || upload_host_rows(s, ch, &up)) return -1;
		in = up; nin = ch->nrows > 0 ? (uint64_t) ch->nrows : 0;
	}
	rc = gg_window_run(s->win, in, nin, &out, &nout);
	s->win_ms = 0.0f;
	if (rc == GG_OK && gg_engine_last_kernel_ms) (void) gg_engine_last_kernel_ms(es->engine, &s->win_ms);
	if (rc == GG_OK && s->having) rc = gg_rowfilter_run(s->having, out, nout, &out, &nout);
	if (rc == GG_OK) rc = gg_relation_attach_rows(es->engine, gg_relation_device_ptr(out), nout, s->rows_ncols, &s->rows_rel);
	if (up) gg_relation_free(up);
	if (rc != GG_OK) { s->rows_rel = NULL; exec_fail(rc, "%s", gg_last_error()); return -1; }
	s->rows_n = nout;
	s->rows_ready = 0;
	return 0;
}

/* a node's aggregate rows -> host result arrays, from its device group records (the one synchronisation of a
 * device-resident slice) or else from its scan / join pipeline */
static int aggrows_to_host(GgPlanState *s)
{
	gg_aggrow *rows = NULL;
	int cap, n = 0, rc;
	for (cap = 4096; ; cap *= 16)
	{
		free(rows);
		rows = malloc(sizeof(gg_aggrow) * (size_t) cap);
		if (!rows) { exec_fail(GG_ERR_NOMEM, "out of memory"); return -1; }
		if (s->groups) rc = gg_groups_fetch(s->groups, rows, cap, &n, NULL, NULL);
		else if (s->kind == K_SCANAGG) rc = gg_scanagg_fetch(s->sa, rows, cap, &n, NULL, NULL);
		else rc = gg_joinagg_fetch(s->ja, rows, cap, &n, NULL);
		if (rc != GG_ERR_NOMEM || cap >= (1 << 24)) break;
	}
	if (rc != GG_OK)
	{
		groups_fail(s, rc);
		free(rows);
		return -1;
	}
	rc = rows_from_aggrows(s, rows, n);
	free(rows);
	return rc;
}

/* the pipeline's result as device group records (none from the general HashAggregate, whose groups live in its hash table) */
static int pipeline_groups(GgPlanState *s)
{
	const int rc = s->kind == K_SCANAGG ? gg_scanagg_groups(s->sa, &s->groups) : gg_joinagg_groups(s->ja, &s->groups);
	if (rc != GG_OK) s->groups = NULL;
	return rc;
}

static int ensure_rows(GgPlanState *s)
{
	if (s->rows_ready) return 0;
	if (s->rows_rel || s->kind == K_SCANROWS || (s->kind == K_MOTION && s->rows_scan)) return rows_to_host(s);
	if (s->groups) return aggrows_to_host(s);
	exec_fail(GG_ERR_ARG, "node has no result");
	return -1;
}

/* the Agg description and key types of the rows a node hands up (for the nodes that pass rows through) */
static void inherit_layout(GgPlanState *s, const GgPlanState *ch)
{
	s->agg = ch->agg;
	s->ncols = ch->ncols;
	memcpy(s->typid, ch->typid, sizeof s->typid);
}

/* Motion of host rows: loopback, the C interconnect's staged exchange, or the transport callback */
static int motion_host_path(GgPlanState *s, int child_failed)
{
	GgEState *es = s->estate;
	GgMotion *mo = (GgMotion *) s->plan;
	GgPlanState *ch = s->child;
	int64_t r;
	int c, rc;
	if (!child_failed && ensure_rows(ch)) return -1;
	if (!multi_segment(es) || (!es->transport && !es->interconnect))
	{
		/* one segment: sender and receiver are the same process */
		if (alloc_result(s, ch->nrows, ch->ncols)) { exec_fail(GG_ERR_NOMEM, "out of memory"); return -1; }
		memcpy(s->values, ch->values, 8 * (size_t) ch->nrows * ch->ncols);
		memcpy(s->isnull, ch->isnull, (size_t) ch->nrows * ch->ncols);
		memcpy(s->lens, ch->lens, 4 * (size_t) ch->nrows * ch->ncols);
	}
	else
	{
		GgRowBatch send, recv;
		int32_t *dest;
		const int64_t nsend = child_failed ? 0 : ch->nrows;
		const int32_t ncols = child_failed ? 1 : ch->ncols;
		char child_err[sizeof g_err];
		int child_code = g_errcode;
		memcpy(child_err, g_err, sizeof child_err);
		if (!child_failed && mo->motionType == GG_MOTIONTYPE_HASH)
			for (c = 0; c < mo->numHashCols; c++)
				if (mo->hashCol[c] < 0 || mo->hashCol[c] >= ch->ncols)
				{ exec_fail(GG_ERR_ARG, "Motion hash column %d out of range (the node below has %d columns)", mo->hashCol[c], ch->ncols); return -1; }
		dest = malloc(4 * (size_t) (nsend > 0 ? nsend : 1));
		if (!dest) { exec_fail(GG_ERR_NOMEM, "out of memory"); return -1; }
		for (r = 0; r < nsend; r++)
		{
			if (mo->motionType == GG_MOTIONTYPE_HASH)
			{
				/* evalHashKey (nodeMotion.c:1481): cdbhash over the hash columns, reduced to a segment */
				int32_t t[GG_MAX_KEYS], ln[GG_MAX_KEYS], nn[GG_MAX_KEYS];
				int64_t v[GG_MAX_KEYS];
				for (c = 0; c < mo->numHashCols; c++)
				{
					int col = mo->hashCol[c];
					t[c] = ch->typid[col];
					v[c] = ch->values[(size_t) r * ch->ncols + col];
					ln[c] = ch->lens[(size_t) r * ch->ncols + col];
					nn[c] = ch->isnull[(size_t) r * ch->ncols + col];
				}
				dest[r] = gg_cdbhash_route(t, v, ln, nn, mo->numHashCols, es->nsegs);
			}
			else
				dest[r] = mo->motionType == GG_MOTIONTYPE_BROADCAST ? -1 : 0;
		}
		memset(&recv, 0, sizeof recv);
		if (es->interconnect)
		{
			rc = gg_ic_exchange_host(es->interconnect, ncols, nsend, child_failed ? NULL : ch->values, child_failed ? NULL : ch->isnull, dest,
			                         child_failed, &recv.nrows, &recv.values, &recv.isnull);
			free(dest);
			if (child_failed) { exec_fail(child_code, "%s", child_err); return -1; }        /* our own error is the better message */
			if (rc != GG_OK) { exec_fail(rc, "Motion %d: %s", mo->motionID, gg_last_error()); return -1; }
		}
		else
		{
			/* transport callback: nrows = -1 tells the peers that this segment failed */
			send.ncols = ncols; send.nrows = child_failed ? -1 : nsend;
			send.values = child_failed ? NULL : ch->values; send.isnull = child_failed ? NULL : ch->isnull;
			rc = es->transport->exchange(es->transport->ctx, mo->motionID, mo->motionType, &send, dest, &recv);
			free(dest);
			if (child_failed) { free(recv.values); free(recv.isnull); exec_fail(child_code, "%s", child_err); return -1; }
			if (rc) { exec_fail(rc == GG_ERR_PEER ? GG_ERR_PEER : GG_ERR_CUDA, "Motion %d: %s (%d)", mo->motionID, rc == GG_ERR_PEER ? "another segment reported an error" : "transport failed", rc); return -1; }
		}
		if (alloc_result(s, recv.nrows, ch->ncols)) { free(recv.values); free(recv.isnull); exec_fail(GG_ERR_NOMEM, "out of memory"); return -1; }
		if (recv.nrows)
		{
			memcpy(s->values, recv.values, 8 * (size_t) recv.nrows * ch->ncols);
			memcpy(s->isnull, recv.isnull, (size_t) recv.nrows * ch->ncols);
		}
		for (r = 0; r < recv.nrows; r++)
			for (c = 0; c < ch->ncols; c++)
				if (is_string_type(ch->typid[c])) s->lens[(size_t) r * ch->ncols + c] = packed_len((uint64_t) s->values[(size_t) r * ch->ncols + c]);
		free(recv.values); free(recv.isnull);
	}
	memcpy(s->typid, ch->typid, sizeof s->typid);
	if (mo->numSortCols > 0 && s->nrows > 1)
	{
		/* sorted receive: the merged order of sorted streams is the sorted order of their union; the comparator is
		 * the Sort node's (tuplesort_mk.c:2816), ties in unspecified order as in the reference's merge */
		gg_sortkey keys[GG_MAX_SORTKEYS];
		if (mo->numSortCols > GG_MAX_SORTKEYS) { exec_fail(GG_ERR_UNSUPPORTED, "Motion with %d merge keys", mo->numSortCols); return -1; }
		if (sort_keys(keys, mo->sortKeys, mo->numSortCols, s, "Motion merge") || sort_host_rows(s, s, keys, mo->numSortCols, 0, GG_NO_BOUND)) return -1;
	}
	s->rows_ready = 1;
	return 0;
}

/* a Motion in this subtree: rows cross segments there, so every segment has to run it whenever any does */
static int has_motion(const GgPlanState *s)
{
	return s && (s->kind == K_MOTION || has_motion(s->child) || has_motion(s->inner));
}

/* Agg <- SeqScan, Agg <- HashJoin, or a HashJoin writing its rows: one scan / join pipeline */
static int run_agg_pipeline(GgPlanState *s)
{
	GgEState *es = s->estate;
	int rc;
	drop_device_results(s);
	if (run_child(s)) return -1;
	if (s->kind == K_JOINROWS && s->table_kept)
	{
		/* ExecReScanHashJoin (nodeHashjoin.c:1015-1050): the table of the unchanged inner side is kept, only the outer side is
		 * probed again */
		gg_relation *outer = s->child ? s->child->rows_rel : s->rel;
		rc = gg_joinagg_probe(s->ja, outer, 0, gg_relation_nblocks(outer));
	}
	else
	{
		if (s->inner && !s->inner->done && run_node(s->inner)) return -1;
		if (s->kind == K_SCANAGG)
		{
			if (s->child) rc = gg_scanagg_run(s->sa, s->child->rows_rel, 0, gg_relation_nblocks(s->child->rows_rel));
			else if (s->rel) rc = gg_scanagg_run(s->sa, s->rel, 0, gg_relation_nblocks(s->rel));
			else rc = gg_scanagg_run_host(s->sa, s->host_pages, s->host_nblocks);
		}
		else
		{
			/* MultiExecHash + the probe loop; in batches when the table would not fit the operator's memory */
			rc = gg_joinagg_set_work_mem(s->ja, es->es_operator_mem);
			if (rc == GG_OK) rc = gg_joinagg_run(s->ja, s->inner ? s->inner->rows_rel : s->inner_rel, s->child ? s->child->rows_rel : s->rel);
		}
	}
	if (rc == GG_OK && s->kind == K_JOINROWS)
	{
		/* the joined rows stay on the device for the node above (or come to the host once, at the top) */
		gg_relation *out;
		uint64_t live;
		rc = gg_joinagg_rows(s->ja, &out, &s->rows_n, &live);
		if (rc == GG_OK) rc = gg_relation_attach_rows(es->engine, gg_relation_device_ptr(out), s->rows_n, s->rows_ncols, &s->rows_rel);
		if (rc != GG_OK) { s->rows_rel = NULL; exec_fail(rc, "%s", gg_last_error()); return -1; }
		/* whether a segment batched depends on its own inner rows; a Motion below the Hash is a plan property, the same on
		 * every segment, so a rescan re-runs that exchange everywhere or nowhere */
		s->table_kept = gg_joinagg_nbatch(s->ja) == 1 && !has_motion(s->inner);
		return 0;
	}
	if (rc != GG_OK) { exec_fail(rc, "%s", gg_last_error()); return -1; }
	/* under a Sort / Limit: the groups are settled (as a fetch settles them) and finalised into datum rows on the device */
	if (s->agg_rows) return agg_datumrows(s);
	if (s->lazy_fetch && !es->motion_on_host && pipeline_groups(s) == GG_OK)
	{
		/* the records go straight into the Motion above; a pipeline that would have to be replayed says so in its
		 * status, which makes that Motion (on every segment) fall back to host rows — where the fetch below runs */
		if (set_layout_types(s)) return -1;
		s->rows_ready = 0;
		return 0;
	}
	/* fetch decides whether the pipeline has to be replayed on a wider kernel variant (more groups than expected, a
	 * non-finite sum to attribute), so it runs before anything above consumes the records on the device */
	if (aggrows_to_host(s)) return -1;
	(void) pipeline_groups(s);                           /* the same rows as device records, for a Motion / FINAL Agg above */
	return 0;
}

/* FINAL Agg: combine the partial states the node below delivers */
static int run_final_agg(GgPlanState *s)
{
	GgEState *es = s->estate;
	GgPlanState *ch = s->child;
	gg_agg part = s->agg;
	gg_aggrow *in, *out;
	int n = 0, cap, i, rc, want;
	drop_device_results(s);
	if (run_child(s)) return -1;
	s->nonreceiver = ch->nonreceiver;
	if (s->dev_groups && !es->motion_on_host && ch->groups)
	{
		rc = gg_groups_final(es->engine, ch->groups, &s->groups);
		if (rc != GG_OK) { exec_fail(rc, "%s", gg_last_error()); return -1; }
		if (s->agg_rows) return agg_datumrows(s);
		if (set_layout_types(s)) return -1;
		s->rows_ready = 0;
		return 0;
	}
	if (ensure_rows(ch)) return -1;
	if (s->nonreceiver)
	{
		/* the slice above a Gather exists only on the receiving segment (the QD in the reference): no rows here, not
		 * even the empty-input row of a plain aggregate */
		if (alloc_result(s, 0, ch->ncols)) { exec_fail(GG_ERR_NOMEM, "out of memory"); return -1; }
		s->rows_ready = 1;
		if (s->having || s->rows_required) { if (set_layout_types(s)) return -1; s->nrows = 0; return upload_agg_rows(s); }
		return 0;
	}
	part.aggstage = GG_AGGSTAGE_PARTIAL;      /* layout of the incoming rows */
	for (i = 0, want = part.numCols; i < part.numAggs; i++) want += agg_ncols_of(&part, i);
	if (want != ch->ncols && ch->nrows > 0)
	{ exec_fail(GG_ERR_ARG, "FINAL Agg expects %d columns of partial state, the node below delivers %d", want, ch->ncols); return -1; }
	in = aggrows_from_rows(ch, &part);
	cap = ch->nrows > 0 ? (int) ch->nrows : 1;
	out = malloc(sizeof(gg_aggrow) * (size_t) cap);
	if (!in || !out) { free(in); free(out); exec_fail(GG_ERR_NOMEM, "out of memory"); return -1; }
	rc = gg_agg_final(es->engine, &s->agg, in, (int) ch->nrows, out, cap, &n);
	free(in);
	if (rc != GG_OK) { exec_fail(rc, "%s", gg_last_error()); free(out); return -1; }
	rc = rows_from_aggrows(s, out, n);
	free(out);
	if (rc == 0 && (s->having || s->rows_required)) rc = upload_agg_rows(s);
	return rc;
}

static int run_sort(GgPlanState *s)
{
	GgEState *es = s->estate;
	GgSort *so = (GgSort *) s->plan;
	GgPlanState *ch = s->child;
	gg_sortkey keys[GG_MAX_SORTKEYS];
	uint64_t rowbytes, run_rows;
	int rc;
	if (run_child(s)) return -1;
	s->nonreceiver = ch->nonreceiver;
	if (sort_keys(keys, so->keys, so->numCols, ch, "Sort")) return -1;
	if (ch->rows_rel && !ch->rows_ready)
	{
		/* the input is datum rows on the device (a row-producing SeqScan, or the Motion over one): sort them where they
		 * are; the sorted rows stay on the device for the node above, or come to the host once, at the top */
		const uint64_t W = 1 + (uint64_t) ch->rows_ncols;
		const uint64_t nout = ch->rows_n < s->sort_bound ? ch->rows_n : s->sort_bound;
		const uint64_t nb = (nout * W * 8 + 64 + GG_BLCKSZ - 1) / GG_BLCKSZ;
		uint64_t live = 0;
		drop_device_results(s);
		if (s->rows_send && gg_relation_nblocks(s->rows_send) < nb) { gg_relation_free(s->rows_send); s->rows_send = NULL; }
		if (!s->rows_send)
		{
			rc = gg_relation_create(es->engine, nb, &s->rows_send);
			if (rc != GG_OK) { exec_fail(rc, "Sort result: %s", gg_last_error()); return -1; }
		}
		/* bounded (a Limit above): only the first sort_bound rows of the order are selected, sorted and written */
		if (s->sort_bound != GG_NO_BOUND)
			rc = gg_sort_datumrows_bounded(es->engine, keys, so->numCols, ch->rows_ncols, gg_relation_device_ptr(ch->rows_rel), ch->rows_n,
			                               s->sort_bound, gg_relation_device_ptr(s->rows_send), &live, NULL);
		else
			rc = gg_sort_datumrows(es->engine, keys, so->numCols, ch->rows_ncols, gg_relation_device_ptr(ch->rows_rel), ch->rows_n,
			                       gg_relation_device_ptr(s->rows_send), &live, NULL);
		if (rc != GG_OK) { exec_fail(rc, "%s", gg_last_error()); return -1; }
		s->rows_n = live; s->rows_ncols = ch->rows_ncols; s->rows_nsegs = 1;
		s->ncols = ch->ncols;
		memcpy(s->typid, ch->typid, sizeof s->typid);
		rc = gg_relation_attach_rows(es->engine, gg_relation_device_ptr(s->rows_send), live, ch->rows_ncols, &s->rows_rel);
		if (rc != GG_OK) { exec_fail(rc, "%s", gg_last_error()); return -1; }
		return 0;
	}
	if (ensure_rows(ch)) return -1;
	memcpy(s->typid, ch->typid, sizeof s->typid);
	/* what the rows take in this node's memory: values, NULL flags, lengths — against the operator's memory
	 * (PlanStateOperatorMemKB, execnodes.h:1446): beyond it the sort goes external, never below 256 rows a run */
	rowbytes = (uint64_t) ch->ncols * 13u;
	run_rows = es->es_operator_mem ? es->es_operator_mem / (rowbytes ? rowbytes : 1) : 0;
	if (run_rows && run_rows < 256) run_rows = 256;
	s->sort_runs = 1;
	/* bounded: when the bound's rows fit the operator's memory, one bounded sort and no runs at all (tuplesort_mk's bounded
	 * heap never spills); otherwise each run keeps its first `bound` rows and the merge stops there */
	if (sort_host_rows(s, ch, keys, so->numCols, run_rows, s->sort_bound)) return -1;
	s->rows_ready = 1;
	return 0;
}

/* ---- Limit (nodeLimit.c): forward-only; the window [offset, offset + count) of the child's rows as host rows ---- */

/* s's result = live datum rows [skip, skip + take) of ch, copied from the device a few 32 KB blocks at a time: only the leading
 * blocks that hold them, never the whole buffer.  *pulled: live rows of ch read (skip + the rows taken). */
static int rows_window_to_host(GgPlanState *s, const GgPlanState *ch, uint64_t skip, uint64_t take, uint64_t *pulled)
{
	const uint64_t W = 1 + (uint64_t) ch->rows_ncols;
	const uint64_t total_nb = (ch->rows_n * W * 8 + GG_BLCKSZ - 1) / GG_BLCKSZ;
	const uint64_t need = skip + take < skip ? UINT64_MAX : skip + take;
	gg_relation *src = rows_buffer(ch);
	uint64_t *buf = NULL, have_nb = 0, r = 0, live = 0, out = 0;
	int c, rc;
	const uint64_t cap = take < (uint64_t) ch->rows_n ? take : (uint64_t) ch->rows_n;
	if (alloc_result(s, (int64_t) cap, ch->rows_ncols)) { exec_fail(GG_ERR_NOMEM, "out of memory"); return -1; }
	while (r < ch->rows_n && live < need)
	{
		/* every block so far held rows; ask for enough new blocks to hold the rows still wanted if none of them were dead */
		const uint64_t rows_wanted = need - live < ch->rows_n - r ? need - live : ch->rows_n - r;
		uint64_t want_nb = ((r + rows_wanted) * W * 8 + GG_BLCKSZ - 1) / GG_BLCKSZ;
		uint64_t *nbuf;
		if (want_nb <= have_nb) want_nb = have_nb + 1;
		if (want_nb > total_nb) want_nb = total_nb;
		nbuf = realloc(buf, (size_t) want_nb * GG_BLCKSZ);
		if (!nbuf) { free(buf); exec_fail(GG_ERR_NOMEM, "out of memory"); return -1; }
		buf = nbuf;
		rc = gg_relation_read(src, have_nb, (uint8_t *) buf + have_nb * GG_BLCKSZ, want_nb - have_nb);
		if (rc != GG_OK) { free(buf); exec_fail(rc, "%s", gg_last_error()); return -1; }
		have_nb = want_nb;
		for (; r < ch->rows_n && (r + 1) * W * 8 <= have_nb * GG_BLCKSZ && live < need; r++)
		{
			if (buf[r * W] & GG_DATUMROW_DEAD) continue;            /* a slot the sending kernel claimed and did not fill */
			if (live++ < skip) continue;
			for (c = 0; c < ch->rows_ncols; c++)
			{
				const uint64_t v = buf[r * W + 1 + c];
				s->values[out * ch->rows_ncols + c] = (int64_t) v;
				s->isnull[out * ch->rows_ncols + c] = (uint8_t) ((buf[r * W] >> c) & 1);
				if (is_string_type(ch->typid[c])) s->lens[out * ch->rows_ncols + c] = packed_len(v);
			}
			out++;
		}
	}
	free(buf);
	s->nrows = (int64_t) out;
	*pulled = live;
	return 0;
}

static int run_limit(GgPlanState *s)
{
	const GgLimit *lp = (const GgLimit *) s->plan;
	GgPlanState *ch = s->child;
	const int64_t offset = lp->hasOffset ? lp->limitOffset : 0;
	const int64_t count = lp->hasCount ? lp->limitCount : 0;
	uint64_t skip, take, pulled = 0;
	/* recompute_limits (nodeLimit.c:258), at the first run and at every ReScan */
	if (offset < 0) { exec_fail(GG_ERR_ARG, "OFFSET must not be negative"); return -1; }
	if (count < 0) { exec_fail(GG_ERR_ARG, "LIMIT must not be negative"); return -1; }
	/* pass_down_bound (nodeLimit.c:345): a Sort below needs only count + offset rows; no bound for LIMIT ALL, a sum that
	 * overflows, or one tuplesort_set_bound would not take (tuplesort_mk.c:1011) */
	if (ch->kind == K_SORT)
	{
		const int64_t needed = (int64_t) ((uint64_t) count + (uint64_t) offset);
		ch->sort_bound = (!lp->hasCount || needed < 0 || needed > INT32_MAX / 2) ? GG_NO_BOUND : (uint64_t) needed;
	}
	if (lp->hasCount && count <= 0)
	{
		/* an empty window: the child never runs; the squelch still runs a Motion below whose peers are in the exchange */
		GgExecSquelchNode(ch);
		inherit_layout(s, ch);
		if (alloc_result(s, 0, s->ncols > 0 ? s->ncols : 1)) { exec_fail(GG_ERR_NOMEM, "out of memory"); return -1; }
		s->nonreceiver = ch->nonreceiver;
		s->rows_ready = 1;
		return 0;
	}
	if (run_child(s)) return -1;
	s->nonreceiver = ch->nonreceiver;
	inherit_layout(s, ch);
	skip = (uint64_t) offset;
	take = lp->hasCount ? (uint64_t) count : UINT64_MAX;
	if (ch->rows_rel && !ch->rows_ready)
	{
		if (rows_window_to_host(s, ch, skip, take, &pulled)) return -1;
	}
	else
	{
		uint64_t n, first, len;
		if (ensure_rows(ch)) return -1;
		n = ch->nrows > 0 ? (uint64_t) ch->nrows : 0;
		first = skip < n ? skip : n;
		len = n - first < take ? n - first : take;
		if (alloc_result(s, (int64_t) len, ch->ncols)) { exec_fail(GG_ERR_NOMEM, "out of memory"); return -1; }
		memcpy(s->values, ch->values + first * (uint64_t) ch->ncols, 8 * (size_t) len * (size_t) ch->ncols);
		memcpy(s->isnull, ch->isnull + first * (uint64_t) ch->ncols, (size_t) len * (size_t) ch->ncols);
		memcpy(s->lens, ch->lens + first * (uint64_t) ch->ncols, 4 * (size_t) len * (size_t) ch->ncols);
		pulled = first + len;
	}
	/* the rows ExecLimit pulled through the child's ExecProcNode, for the child's Instrumentation */
	ch->instr_ntuples += (double) pulled;
	/* the window is complete: the node below will not be read again (ExecLimit, nodeLimit.c:239-247) */
	GgExecSquelchNode(ch);
	s->rows_ready = 1;
	return 0;
}

static int run_motion(GgPlanState *s)
{
	GgEState *es = s->estate;
	GgMotion *mo = (GgMotion *) s->plan;
	GgPlanState *ch = s->child;
	int32_t kt[GG_MAX_KEYS] = { 0 }, hashtyp[GG_MAX_KEYS] = { 0 };
	int child_failed = 0, c, rc;
	if (s->rows_scan) return run_rows_node(s);
	drop_device_results(s);
	if (run_child(s))
	{
		/* this segment's slice failed: it still takes part in the exchange (with no rows) so that no peer waits for
		 * it, and every segment comes back with an error (nodeMotion.c / cdbmotion.c:342 stop + error propagation) */
		if (!multi_segment(es) || (!es->interconnect && !es->transport)) return -1;
		child_failed = 1;
		if (!g_local_code) { g_local_code = g_errcode; memcpy(g_local_err, g_err, sizeof g_local_err); }
	}
	s->nonreceiver = (mo->motionType == GG_MOTIONTYPE_GATHER && multi_segment(es) && es->segindex != 0) || (!child_failed && ch->nonreceiver);
	if (!child_failed) inherit_layout(s, ch);
	if (!s->dev_groups || es->motion_on_host) return motion_host_path(s, child_failed);
	/* device path: aggregate rows move as group records, segment to segment, without touching the host.  Whether a
	 * Motion takes it was decided from the plan (every segment alike); a segment that cannot contribute records —
	 * its slice failed, or its aggregate keeps its groups in the general hash table — sends its status instead, and
	 * the flag reaches every segment's fetch with the data (an ERROR, or "run the slice again with host-row Motions"). */
	agg_keytypes(s, kt);
	for (c = 0; c < mo->numHashCols && mo->motionType == GG_MOTIONTYPE_HASH; c++) hashtyp[c] = kt[mo->hashCol[c]];
	rc = gg_ic_motion_groups(es->interconnect, mo->motionType, 0, mo->motionType == GG_MOTIONTYPE_HASH ? mo->numHashCols : 0,
	                         mo->hashCol, hashtyp, child_failed ? NULL : ch->groups, child_failed ? g_errcode : GG_OK, &s->groups);
	if (rc != GG_OK) { exec_fail(rc, "Motion %d: %s", mo->motionID, gg_last_error()); return -1; }
	if (s->nonreceiver) gg_groups_set_nonreceiver(s->groups);
	/* a failed child left no layout: the rows this node would have handed up take it from the plan */
	if (child_failed && set_layout_types(s)) return -1;
	s->rows_ready = 0;
	return 0;
}

static int run_node(GgPlanState *s)
{
	GgEState *es = s->estate;
	int rc;
	{
		/* GGB200_EXEC_TRACE=1: which node of which segment starts running (debugging a stuck slice) */
		static int trace = -1;
		if (trace < 0) { const char *t = getenv("GGB200_EXEC_TRACE"); trace = t && atoi(t) != 0; }
		if (trace) { fprintf(stderr, "[exec seg %d] run node kind %d (motion on host: %d)\n", es->segindex, (int) s->kind, es->motion_on_host); fflush(stderr); }
	}
	s->instr_nloops += 1.0;
	switch (s->kind)
	{
		case K_SCANROWS: rc = run_rows_node(s); break;
		case K_SCANAGG: case K_JOINAGG: case K_JOINROWS: rc = run_agg_pipeline(s); break;
		case K_AGGFINAL: rc = run_final_agg(s); break;
		case K_SORT: rc = run_sort(s); break;
		case K_MOTION: rc = run_motion(s); break;
		case K_LIMIT: rc = run_limit(s); break;
		case K_WINDOW: rc = run_window(s); break;
		default:
			exec_fail(GG_ERR_ARG, "bad plan state");
			return -1;
	}
	if (rc) return -1;
	s->done = 1;
	s->next = 0;
	return 0;
}


/* ---- rows on the wire: a CPU segment on the other side of a Motion (include/gg_tupser.h) ---- */
#define GG_FLOAT8ARRAYOID 1022

static void wire_attr(gg_attr *a, int32_t typid)
{
	memset(a, 0, sizeof *a);
	a->atttypid = typid; a->atttypmod = -1;
	switch (typid)
	{
		case GG_BOOLOID: a->attlen = 1; a->attalign = 'c'; a->attbyval = 1; break;
		case GG_INT4OID: case GG_DATEOID: a->attlen = 4; a->attalign = 'i'; a->attbyval = 1; break;
		case GG_BPCHAROID: case GG_VARCHAROID: case GG_TEXTOID: a->attlen = -1; a->attalign = 'i'; break;
		case GG_FLOAT8ARRAYOID: a->attlen = -1; a->attalign = 'd'; break;
		default: a->attlen = 8; a->attalign = 'd'; a->attbyval = 1; break;         /* int8, float8, timestamp */
	}
}

/* The tuple descriptor of a node's rows as the reference's nodes see them: one attribute per column, except that the three
 * columns {N, sumX, sumX2} of a PARTIAL-stage avg(float8) are ONE float8[] attribute — the transition value finalize_aggregate
 * hands up when there is no final function to run (nodeAgg.c:975-979; SURVEY App. A "two-stage interchange").
 * map[w] = first result column of wire attribute w; arr[w] = 1 for such an array. */
static int wire_layout(const GgPlanState *s, gg_attr *attrs, int *map, int *arr)
{
	int n = 0, c = 0, i;
	if (s->agg.aggstage == GG_AGGSTAGE_PARTIAL && (s->agg.numCols + s->agg.numAggs) > 0)
	{
		for (c = 0; c < s->agg.numCols; c++, n++) { wire_attr(&attrs[n], s->typid[c]); map[n] = c; arr[n] = 0; }
		for (i = 0; i < s->agg.numAggs; i++, n++)
		{
			const int w = agg_ncols_of(&s->agg, i);
			wire_attr(&attrs[n], w == 3 ? GG_FLOAT8ARRAYOID : s->typid[c]);
			map[n] = c; arr[n] = w == 3;
			c += w;
		}
		return c == s->ncols ? n : -1;
	}
	for (c = 0; c < s->ncols; c++) { wire_attr(&attrs[c], s->typid[c]); map[c] = c; arr[c] = 0; }
	return s->ncols;
}

/* the MemTuple binding of a row of these column types (what the reference builds from the node's result tuple descriptor) */
static int slot_binding(const int32_t *typids, int ncols, gg_memtuple_binding *b)
{
	gg_attr attrs[GG_MAX_OUTCOLS];
	int c;
	if (ncols < 1 || ncols > GG_MAX_OUTCOLS || ncols > GG_MT_MAX_ATTS) return GG_ERR_UNSUPPORTED;
	for (c = 0; c < ncols; c++)
	{
		if (typids[c] == GG_FLOAT8ARRAYOID) return GG_ERR_UNSUPPORTED;      /* a transition array is three slot columns, not one */
		wire_attr(&attrs[c], typids[c]);
	}
	return gg_memtuple_bind(attrs, ncols, b);
}

int GgExecSortRuns(GgPlanState *s) { return s && s->kind == K_SORT ? s->sort_runs : 0; }

/* the external sort's merge order on its own (tests hold it to the reference's comparators): < 0, 0, > 0 for row a against row b */
int GgExecDebugSortCompare(const gg_sortkey *keys, int nkeys, int ncols, const int64_t *values, const uint8_t *isnull, uint64_t a, uint64_t b)
{
	return sort_row_cmp(keys, nkeys, ncols, values, isnull, a, b);
}

int GgExecNodeInstrumentation(GgPlanState *s, GgInstrumentation *out)
{
	float ms = 0.0f, bms = 0.0f;
	int launches = 0, variant = 0;
	if (!s || !out) return GG_ERR_ARG;
	memset(out, 0, sizeof *out);
	out->ntuples = s->instr_ntuples;
	out->nloops = s->instr_nloops;
	out->sort_runs = s->kind == K_SORT ? s->sort_runs : 0;
	if ((s->kind == K_JOINAGG || s->kind == K_JOINROWS) && s->ja) out->hash_batches = gg_joinagg_nbatch(s->ja);
	if ((s->kind == K_SCANAGG && s->sa) || ((s->kind == K_JOINAGG || s->kind == K_JOINROWS) && s->ja))
		if (GgExecPipelineKernelMs(s, &ms, &launches, &variant, &bms) == GG_OK) out->kernel_ms = ms + bms;
	if (s->kind == K_WINDOW) out->kernel_ms = s->win_ms;
	return GG_OK;
}

int64_t GgExecFetchSlotMemTuple(const GgTupleTableSlot *slot, uint8_t *out, uint64_t cap, uint32_t *need)
{
	gg_memtuple_binding *b;
	uint32_t len = 0;
	int rc;
	if (!slot || slot->tts_isempty || slot->tts_nvalid < 1 || (!out && cap)) { exec_fail(GG_ERR_ARG, "empty slot"); return GG_ERR_ARG; }
	b = malloc(sizeof *b);
	if (!b) { exec_fail(GG_ERR_NOMEM, "out of memory"); return GG_ERR_NOMEM; }
	rc = slot_binding(slot->tts_typid, slot->tts_nvalid, b);
	if (rc == GG_OK)
		rc = gg_memtuple_form(b, slot->tts_values, slot->tts_isnull, slot->tts_len, NULL, out, cap > 0xFFFFFFFFu ? 0xFFFFFFFFu : (uint32_t) cap, &len);
	free(b);
	if (need) *need = len;
	if (rc != GG_OK) { exec_fail(rc, rc == GG_ERR_NOMEM ? "output buffer too small for the MemTuple" : "row layout has no MemTuple form"); return rc; }
	return (int64_t) len;
}

int GgExecStoreMemTuple(GgTupleTableSlot *slot, const int32_t *typids, int ncols, const uint8_t *mt, uint32_t len)
{
	gg_memtuple_binding *b;
	int32_t lens[GG_MAX_OUTCOLS];
	int rc, c;
	if (!slot || !typids || !mt) { exec_fail(GG_ERR_ARG, "bad arguments"); return GG_ERR_ARG; }
	b = malloc(sizeof *b);
	if (!b) { exec_fail(GG_ERR_NOMEM, "out of memory"); return GG_ERR_NOMEM; }
	rc = slot_binding(typids, ncols, b);
	if (rc == GG_OK) rc = gg_memtuple_deform(b, mt, len, slot->tts_values, slot->tts_isnull, lens);
	free(b);
	if (rc != GG_OK) { exec_fail(rc, "not a MemTuple of these %d columns", ncols); return rc; }
	for (c = 0; c < ncols; c++)
	{
		slot->tts_typid[c] = typids[c];
		slot->tts_len[c] = 0;
		if (slot->tts_isnull[c]) { slot->tts_values[c] = 0; continue; }
		if (is_string_type(typids[c]))
		{
			/* deform left the payload's offset and length: the slot keeps short strings packed in the Datum word */
			const int64_t off = slot->tts_values[c];
			uint64_t v = 0;
			int i;
			if (lens[c] < 0 || lens[c] > 8 || off < 0 || (uint64_t) off + (uint64_t) lens[c] > len)
			{ exec_fail(GG_ERR_UNSUPPORTED, "column %d: a string of %d bytes does not fit a slot", c, lens[c]); return GG_ERR_UNSUPPORTED; }
			for (i = 0; i < lens[c]; i++) v |= (uint64_t) mt[off + i] << (8 * i);
			slot->tts_values[c] = (int64_t) v;
			slot->tts_len[c] = lens[c];
		}
	}
	slot->tts_nvalid = ncols;
	slot->tts_isempty = 0;
	return GG_OK;
}

int64_t GgExecSendTupleChunks(GgPlanState *s, int max_chunk, uint8_t *out, uint64_t cap, int64_t *nrows)
{
	gg_attr attrs[GG_MAX_OUTCOLS];
	int map[GG_MAX_OUTCOLS], arr[GG_MAX_OUTCOLS], natts, w, rc;
	gg_memtuple_binding *b;
	uint64_t pos = 0;
	int64_t r;
	if (!s || !out) { exec_fail(GG_ERR_ARG, "bad arguments"); return GG_ERR_ARG; }
	if (!s->done) { g_err[0] = 0; g_errcode = GG_OK; if (run_node(s)) return g_errcode ? g_errcode : GG_ERR_ARG; }
	if (ensure_rows(s)) return g_errcode ? g_errcode : GG_ERR_ARG;
	natts = wire_layout(s, attrs, map, arr);
	if (natts < 0 || natts > GG_MT_MAX_ATTS) { exec_fail(GG_ERR_UNSUPPORTED, "row layout has no wire form"); return GG_ERR_UNSUPPORTED; }
	b = malloc(sizeof *b);
	if (!b) { exec_fail(GG_ERR_NOMEM, "out of memory"); return GG_ERR_NOMEM; }
	rc = gg_memtuple_bind(attrs, natts, b);
	for (r = 0; rc == GG_OK && r < s->nrows; r++)
	{
		int64_t v[GG_MAX_OUTCOLS];
		uint8_t nl[GG_MAX_OUTCOLS], arrbuf[GG_MAX_OUTCOLS][44];
		int32_t ln[GG_MAX_OUTCOLS];
		const void *ptrs[GG_MAX_OUTCOLS];
		int32_t nch = 0;
		int64_t got;
		for (w = 0; w < natts; w++)
		{
			const size_t at = (size_t) r * s->ncols + (size_t) map[w];
			ptrs[w] = NULL; ln[w] = 0;
			if (arr[w])
			{
				gg_float8_array3(bitsf8(s->values[at]), bitsf8(s->values[at + 1]), bitsf8(s->values[at + 2]), arrbuf[w]);
				v[w] = 0; nl[w] = 0; ptrs[w] = arrbuf[w]; ln[w] = 44;
			}
			else { v[w] = s->values[at]; nl[w] = s->isnull[at]; ln[w] = s->lens[at]; }
		}
		got = gg_tupser_serialize(b, v, nl, ln, ptrs, max_chunk, out + pos, cap - pos, &nch);
		if (got < 0) { rc = (int) got; break; }
		pos += (uint64_t) got;
	}
	if (rc == GG_OK)
	{
		const int e = gg_tupser_eos(out + pos, cap - pos);          /* SendEndOfStream, cdbmotion.c:532 */
		if (e < 0) rc = e; else pos += (uint64_t) e;
	}
	free(b);
	if (rc != GG_OK) { exec_fail(rc, "serialising rows: %s", rc == GG_ERR_NOMEM ? "output buffer too small" : "unsupported value"); return rc; }
	if (nrows) *nrows = s->nrows;
	return (int64_t) pos;
}

int GgExecRecvTupleChunks(GgPlanState *s, const uint8_t *chunks, uint64_t nbytes)
{
	gg_attr attrs[GG_MAX_OUTCOLS];
	int map[GG_MAX_OUTCOLS], arr[GG_MAX_OUTCOLS], natts, w, rc = GG_OK, pass;
	gg_memtuple_binding *b;
	int64_t nrows = 0;
	if (!s || s->kind != K_MOTION || !s->child || (!chunks && nbytes)) return (exec_fail(GG_ERR_ARG, "GgExecRecvTupleChunks takes a Motion node"), GG_ERR_ARG);
	/* the layout of what arrives is the child's: a Motion passes rows through */
	inherit_layout(s, s->child);
	if (!s->ncols && set_layout_types(s)) return g_errcode;
	natts = wire_layout(s, attrs, map, arr);
	if (natts < 0 || natts > GG_MT_MAX_ATTS) return (exec_fail(GG_ERR_UNSUPPORTED, "row layout has no wire form"), GG_ERR_UNSUPPORTED);
	b = malloc(sizeof *b);
	if (!b) return (exec_fail(GG_ERR_NOMEM, "out of memory"), GG_ERR_NOMEM);
	rc = gg_memtuple_bind(attrs, natts, b);
	/* two passes over the chunks: count the tuples, then fill the result */
	for (pass = 0; rc == GG_OK && pass < 2; pass++)
	{
		uint64_t pos = 0;
		int64_t r = 0;
		int eos = 0;
		if (pass == 1 && alloc_result(s, nrows, s->ncols)) { rc = GG_ERR_NOMEM; break; }
		while (pos < nbytes && !eos)
		{
			int64_t v[GG_MAX_OUTCOLS];
			uint8_t nl[GG_MAX_OUTCOLS], strbuf[4096];
			int32_t ln[GG_MAX_OUTCOLS];
			uint64_t used = 0;
			const int d = gg_tupser_deserialize(b, chunks + pos, nbytes - pos, &used, v, nl, ln, strbuf, sizeof strbuf);
			if (d == 1) { eos = 1; break; }
			if (d != GG_OK) { rc = d; break; }
			pos += used;
			if (pass == 1)
				for (w = 0; w < natts; w++)
				{
					const size_t at = (size_t) r * s->ncols + (size_t) map[w];
					if (arr[w])
					{
						double st[3] = { 0, 0, 0 };
						if (nl[w] || gg_float8_array3_read(strbuf + v[w], ln[w], st)) { rc = GG_ERR_ARG; break; }
						s->values[at] = f8bits(st[0]); s->values[at + 1] = f8bits(st[1]); s->values[at + 2] = f8bits(st[2]);
					}
					else if (attrs[w].attlen == -1)
					{
						uint64_t packed = 0;
						int k;
						if (!nl[w] && ln[w] > 8) { rc = GG_ERR_UNSUPPORTED; break; }      /* strings travel packed in 8 bytes on this path */
						for (k = 0; !nl[w] && k < ln[w]; k++) packed |= (uint64_t) strbuf[v[w] + k] << (8 * k);
						s->values[at] = (int64_t) packed; s->isnull[at] = nl[w]; s->lens[at] = nl[w] ? 0 : ln[w];
					}
					else { s->values[at] = v[w]; s->isnull[at] = nl[w]; }
				}
			r++;
		}
		if (rc == GG_OK && !eos) rc = GG_ERR_BADPAGE;              /* a stream ends with its end-of-stream chunk */
		nrows = r;
	}
	free(b);
	if (rc != GG_OK) return (exec_fail(rc, "reading tuple chunks failed (%d)", rc), rc);
	drop_device_results(s);
	s->rows_ready = 1; s->done = 1; s->next = 0;
	return GG_OK;
}

GgTupleTableSlot *GgExecProcNode(GgPlanState *s)
{
	int c;
	if (!s || s->squelched) return NULL;
	if (s->kind == K_HASH) { exec_fail(GG_ERR_ARG, "Hash node does not return tuples via ExecProcNode()"); return NULL; }     /* nodeHash.c:73 ExecHash */
	for (;;)
	{
		int failed = 0;
		if (!s->done)
		{
			g_err[0] = 0; g_errcode = GG_OK;
			/* the query's snapshot reaches every scan of the slice through the engine (heap_beginscan's argument,
			 * heapam.c:1573; EState.es_snapshot) */
			c = gg_engine_set_snapshot(s->estate->engine, s->estate->es_snapshot);
			if (c != GG_OK) { exec_fail(c, "%s", gg_last_error()); return NULL; }
			failed = run_node(s);                     /* the C wrapper on the Postgres side turns a failure into ereport(ERROR) */
		}
		if (!failed && !s->rows_ready)
		{
			g_err[0] = 0; g_errcode = GG_OK;
			failed = ensure_rows(s);
		}
		if (!failed) break;
		if (g_errcode == GG_ERR_RETRY_HOST && !s->estate->motion_on_host)
		{
			/* some segment could not keep its aggregate rows on the device; every segment learned it at its fetch, so all
			 * of them run the slice again, with the Motions moving host rows */
			s->estate->motion_on_host = 1;
			if (GgExecReScan(s) != GG_OK) return NULL;
			continue;
		}
		return NULL;
	}
	if (s->next >= s->nrows)
	{
		s->slot.tts_isempty = 1;                      /* ExecClearTuple: end of stream */
		return NULL;
	}
	s->slot.tts_isempty = 0;
	s->slot.tts_nvalid = s->ncols;
	for (c = 0; c < s->ncols; c++)
	{
		s->slot.tts_values[c] = s->values[(size_t) s->next * s->ncols + c];
		s->slot.tts_isnull[c] = s->isnull[(size_t) s->next * s->ncols + c];
		s->slot.tts_typid[c] = s->typid[c];
		s->slot.tts_len[c] = s->lens[(size_t) s->next * s->ncols + c];
	}
	s->next++;
	s->estate->es_processed++;
	s->instr_ntuples += 1.0;
	return &s->slot;
}

void *GgMultiExecProcNode(GgPlanState *s)
{
	/* execProcnode.c:1217: MultiExecHash is the only multi-exec node on this path, and its work — the build kernel — belongs
	 * to the join's pipeline (gg_joinagg_build), launched when the Agg above the join first runs */
	if (!s || s->kind != K_HASH) exec_fail(GG_ERR_ARG, "MultiExecProcNode on a node that is not a Hash");
	return NULL;
}

int GgExecReScan(GgPlanState *s)
{
	int rc = GG_OK;
	if (!s) return GG_ERR_ARG;
	g_local_code = 0; g_local_err[0] = 0;
	if (s->child && (rc = GgExecReScan(s->child)) != GG_OK) return rc;
	if (s->inner && (rc = GgExecReScan(s->inner)) != GG_OK) return rc;
	drop_device_results(s);
	if (s->sa) rc = gg_scanagg_reset(s->sa);
	if (s->ja && rc == GG_OK) rc = gg_joinagg_reset(s->ja);
	s->done = 0; s->squelched = 0; s->next = 0; s->nrows = 0; s->rows_ready = 0; s->markpos = 0;
	return rc;
}

void GgExecSquelchNode(GgPlanState *s)
{
	/* the node above needs no more rows (LIMIT satisfied, nodeLimit.c): stop handing them out.  A Motion between several
	 * segments that has not run yet still has to: its peers are (or will be) in the exchange, and a collective has no
	 * Stop message to send them (ExecSquelchMotion -> SendStopMessage, nodeMotion.c:1730) */
	for (; s; s = s->child)
	{
		if (s->kind == K_MOTION && !s->done && multi_segment(s->estate) && (s->estate->interconnect || s->estate->transport))
			(void) run_node(s);
		s->squelched = 1;
	}
}

void GgExecEndNode(GgPlanState *s)
{
	end_tree(s);
}

/* ---- per-node entry points (executor/node*.h names) ---- */
static GgPlanState *init_tagged(GgPlan *plan, GgNodeTag tag, GgEState *estate, int eflags)
{
	if (!plan || plan->type != tag) return exec_fail(GG_ERR_ARG, "node tag %d where %d was expected", plan ? (int) plan->type : 0, (int) tag);
	return GgExecInitNode(plan, estate, eflags);
}

GgPlanState *GgExecInitAgg(GgAgg *node, GgEState *estate, int eflags) { return init_tagged(&node->plan, T_GgAgg, estate, eflags); }
GgTupleTableSlot *GgExecAgg(GgPlanState *node) { return GgExecProcNode(node); }
void GgExecEndAgg(GgPlanState *node) { GgExecEndNode(node); }
int GgExecReScanAgg(GgPlanState *node) { return GgExecReScan(node); }
void GgExecSquelchAgg(GgPlanState *node) { GgExecSquelchNode(node); }

GgPlanState *GgExecInitSort(GgSort *node, GgEState *estate, int eflags) { return init_tagged(&node->plan, T_GgSort, estate, eflags); }
GgTupleTableSlot *GgExecSort(GgPlanState *node) { return GgExecProcNode(node); }
void GgExecEndSort(GgPlanState *node) { GgExecEndNode(node); }
int GgExecReScanSort(GgPlanState *node) { return GgExecReScan(node); }
void GgExecSquelchSort(GgPlanState *node) { GgExecSquelchNode(node); }
GgPlanState *GgExecInitLimit(GgLimit *node, GgEState *estate, int eflags) { return init_tagged(&node->plan, T_GgLimit, estate, eflags); }
GgTupleTableSlot *GgExecLimit(GgPlanState *node) { return GgExecProcNode(node); }
void GgExecEndLimit(GgPlanState *node) { GgExecEndNode(node); }
int GgExecReScanLimit(GgPlanState *node) { return GgExecReScan(node); }
void GgExecSquelchLimit(GgPlanState *node) { GgExecSquelchNode(node); }
/* ExecSortMarkPos / ExecSortRestrPos (nodeSort.c:444,462): the sorted result is materialised, so a position is an index */
void GgExecSortMarkPos(GgPlanState *node) { if (node && node->done) node->markpos = node->next; }
void GgExecSortRestrPos(GgPlanState *node) { if (node && node->done) node->next = node->markpos; }

GgPlanState *GgExecInitWindowAgg(GgWindowAgg *node, GgEState *estate, int eflags) { return init_tagged(&node->plan, T_GgWindowAgg, estate, eflags); }
GgTupleTableSlot *GgExecWindowAgg(GgPlanState *node) { return GgExecProcNode(node); }
void GgExecEndWindowAgg(GgPlanState *node) { GgExecEndNode(node); }
int GgExecReScanWindowAgg(GgPlanState *node) { return GgExecReScan(node); }
void GgExecSquelchWindowAgg(GgPlanState *node) { GgExecSquelchNode(node); }

GgPlanState *GgExecInitMotion(GgMotion *node, GgEState *estate, int eflags) { return init_tagged(&node->plan, T_GgMotion, estate, eflags); }
GgTupleTableSlot *GgExecMotion(GgPlanState *node) { return GgExecProcNode(node); }
void GgExecEndMotion(GgPlanState *node) { GgExecEndNode(node); }
int GgExecReScanMotion(GgPlanState *node) { return GgExecReScan(node); }
void GgExecSquelchMotion(GgPlanState *node) { GgExecSquelchNode(node); }

GgPlanState *GgExecInitHashJoin(GgHashJoin *node, GgEState *estate, int eflags) { return init_tagged(&node->plan, T_GgHashJoin, estate, eflags); }
GgTupleTableSlot *GgExecHashJoin(GgPlanState *node) { return GgExecProcNode(node); }
void GgExecEndHashJoin(GgPlanState *node) { GgExecEndNode(node); }
int GgExecReScanHashJoin(GgPlanState *node) { return GgExecReScan(node); }
void GgExecSquelchHashJoin(GgPlanState *node) { GgExecSquelchNode(node); }

GgPlanState *GgExecInitSeqScan(GgSeqScan *node, GgEState *estate, int eflags) { return init_tagged(&node->plan, T_GgSeqScan, estate, eflags); }
GgPlanState *GgExecInitSeqScanForPartition(GgSeqScan *node, GgEState *estate, int eflags, gg_relation *part)
{
	/* nodeSeqscan.c:221: the same scan over one partition's relation instead of the one the plan names */
	GgPlanState *s;
	gg_relation *saved;
	if (!node || !estate || node->scanrelid < 0 || node->scanrelid >= GG_MAX_RELATIONS || !part) return exec_fail(GG_ERR_ARG, "bad partition scan");
	saved = estate->relations[node->scanrelid];
	estate->relations[node->scanrelid] = part;
	s = init_tagged(&node->plan, T_GgSeqScan, estate, eflags);
	estate->relations[node->scanrelid] = saved;
	return s;
}
GgTupleTableSlot *GgExecSeqScan(GgPlanState *node) { return GgExecProcNode(node); }
void GgExecEndSeqScan(GgPlanState *node) { GgExecEndNode(node); }
int GgExecReScanSeqScan(GgPlanState *node) { return GgExecReScan(node); }

GgPlanState *GgExecInitHash(GgHash *node, GgEState *estate, int eflags) { return init_tagged(&node->plan, T_GgHash, estate, eflags); }
void *GgMultiExecHash(GgPlanState *node) { return GgMultiExecProcNode(node); }
GgTupleTableSlot *GgExecHash(GgPlanState *node) { return GgExecProcNode(node); }
void GgExecEndHash(GgPlanState *node) { GgExecEndNode(node); }
int GgExecReScanHash(GgPlanState *node) { return node ? GG_OK : GG_ERR_ARG; }

/* ---- the interconnect entry of the reference's per-type table (cdbinterconnect.h:500-533) ---- */
static int nccl_setup(GgEState *estate, const void *unique_id)
{
	if (!estate || estate->interconnect) return GG_ERR_ARG;
	return gg_ic_create(estate->engine, unique_id, estate->nsegs > 0 ? estate->nsegs : 1, estate->segindex, &estate->interconnect);
}

static void nccl_teardown(GgEState *estate, int hasErrors)
{
	if (!estate || !estate->interconnect) return;
	gg_ic_teardown(estate->interconnect, hasErrors);
	estate->interconnect = NULL;
}

const GgInterconnectOps GgInterconnectNCCL = {
	nccl_setup, nccl_teardown, gg_ic_motion_groups, gg_ic_exchange_rows, gg_ic_exchange_host
};
