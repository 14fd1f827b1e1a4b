/*
 * window_ref.c — TEST INFRASTRUCTURE: WindowAgg restated row at a time, the way nodeWindowAgg.c and windowfuncs.c compute it,
 * as the reference the device's gg_window_* (greengage_b200/csrc/gg_window.cu) is held to.  Compiled with gcc by the tests into
 * a temporary directory; never shipped.
 *
 * Input: datum rows (include/gg_plan.h GG_FMT_DATUMROWS: word 0 the NULL mask, then one word per column), sorted so that
 * partitions and peer groups are runs; slots marked GG_DATUMROW_DEAD are not rows.  Output: one row per live input row of the
 * input's words followed by one word per window function, NULL mask bits after the input's.
 *
 * What it restates:
 *   partitions and peers       execTuplesMatch (execGrouping.c:60-110) with each type's equality: float8eq (float.c:1010-1020:
 *                              NaN = NaN, -0 = +0), the others by value; two NULLs match
 *   frame head / tail          update_frameheadpos / update_frametailpos (nodeWindowAgg.c:1095-1300), ROWS and RANGE, the
 *                              UNBOUNDED and CURRENT ROW bounds
 *   aggregates                 eval_windowaggregates (nodeWindowAgg.c:380-620): the transition state is restarted whenever the
 *                              frame head moves, then advanced row by row up to the frame tail; strict transitions skip NULLs;
 *                              float8pl / float8_accum with CHECKFLOATVAL (float.c:782-800, 1878-1910), left to right
 *   window functions           windowfuncs.c: row_number :81, rank :99 (rank_up :60), dense_rank :118, percent_rank :140,
 *                              cume_dist :170, ntile :211-276 (its own loop), lag / lead :286-329, first / last / nth_value
 *                              :389-470
 */
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../include/ggb200.h"

typedef struct {
	const uint64_t *w;          /* the row's words */
} Row;

static int g_f8[GG_MAX_ATTS];

static int isnull_col(Row r, int c) { return (int) ((r.w[0] >> c) & 1); }
static double u2d(uint64_t u) { double d; memcpy(&d, &u, 8); return d; }
static uint64_t d2u(double d) { uint64_t u; memcpy(&u, &d, 8); return u; }

/* execTuplesMatch over the listed columns */
static int tuples_match(Row a, Row b, const int32_t *cols, int ncols)
{
	for (int k = 0; k < ncols; k++)
	{
		const int c = cols[k];
		const int na = isnull_col(a, c), nb = isnull_col(b, c);
		if (na != nb) return 0;
		if (na) continue;
		if (g_f8[c])
		{
			const double x = u2d(a.w[1 + c]), y = u2d(b.w[1 + c]);
			if (isnan(x) || isnan(y)) { if (!(isnan(x) && isnan(y))) return 0; }
			else if (x != y) return 0;
		}
		else if (a.w[1 + c] != b.w[1 + c]) return 0;
	}
	return 1;
}

/* float8_cmp_internal (float.c:964) */
static int f8cmp(double a, double b)
{
	if (isnan(a)) return isnan(b) ? 0 : 1;
	if (isnan(b)) return -1;
	return a > b ? 1 : (a < b ? -1 : 0);
}

typedef struct {
	int col, isnull_const, present;
	uint64_t v;
} Arg;

static uint64_t arg_value(const Arg *a, Row r, int *isnull)
{
	if (a->col < 0) { *isnull = a->isnull_const; return a->isnull_const ? 0 : a->v; }
	*isnull = isnull_col(r, a->col);
	return *isnull ? 0 : r.w[1 + a->col];
}

/* an aggregate's transition state */
typedef struct {
	int64_t count;              /* count(*) / count(x) / N of float8_accum */
	int has;                    /* strict state not NULL */
	uint64_t v;                 /* int8 sum, float8 sumX, or the extreme */
	double sumX2;
} AggState;

static int advance(int32_t fn, AggState *st, const Arg *a, Row r)
{
	int isnull;
	uint64_t x;
	if (fn == GG_AGG_COUNT_STAR) { st->count++; return 0; }
	x = arg_value(a, r, &isnull);
	if (isnull) return 0;                                        /* strict transition function: skipped */
	switch (fn)
	{
		case GG_AGG_COUNT_ANY: st->count++; return 0;
		case GG_AGG_SUM_INT4: st->v = st->has ? st->v + x : x; st->has = 1; return 0;   /* int4_sum */
		case GG_AGG_SUM_FLOAT8:
		{
			/* float8pl, state initially NULL: the first input becomes the state (nodeAgg.c advance_transition_function) */
			if (!st->has) { st->v = x; st->has = 1; return 0; }
			const double a1 = u2d(st->v), a2 = u2d(x), s = a1 + a2;
			if (isinf(s) && !(isinf(a1) || isinf(a2))) return GG_ERR_FLOAT_OVERFLOW;
			st->v = d2u(s);
			return 0;
		}
		case GG_AGG_AVG_FLOAT8:
		{
			/* float8_accum over "{0,0,0}" */
			const double v = u2d(x), sx = (st->has ? u2d(st->v) : 0.0) + v, sx2 = st->sumX2 + v * v;
			if (isinf(sx) && !(isinf(st->has ? u2d(st->v) : 0.0) || isinf(v))) return GG_ERR_FLOAT_OVERFLOW;
			if (isinf(sx2) && !(isinf(st->sumX2) || isinf(v))) return GG_ERR_FLOAT_OVERFLOW;
			st->count++; st->v = d2u(sx); st->sumX2 = sx2; st->has = 1;
			return 0;
		}
		case GG_AGG_MAX_INT4: case GG_AGG_MAX_INT8: case GG_AGG_MAX_DATE:
			if (!st->has || (int64_t) x > (int64_t) st->v) st->v = x;
			st->has = 1; return 0;
		case GG_AGG_MIN_INT4: case GG_AGG_MIN_INT8: case GG_AGG_MIN_DATE:
			if (!st->has || (int64_t) x < (int64_t) st->v) st->v = x;
			st->has = 1; return 0;
		case GG_AGG_MAX_FLOAT8:                                   /* float8larger: arg1 only if it is greater */
			if (!st->has || !(f8cmp(u2d(st->v), u2d(x)) > 0)) st->v = x;
			st->has = 1; return 0;
		case GG_AGG_MIN_FLOAT8:                                   /* float8smaller */
			if (!st->has || !(f8cmp(u2d(st->v), u2d(x)) < 0)) st->v = x;
			st->has = 1; return 0;
	}
	return GG_ERR_UNSUPPORTED;
}

static uint64_t finalize(int32_t fn, const AggState *st, int *isnull)
{
	*isnull = 0;
	switch (fn)
	{
		case GG_AGG_COUNT_STAR: case GG_AGG_COUNT_ANY: return (uint64_t) st->count;
		case GG_AGG_AVG_FLOAT8:                                   /* float8_avg: NULL when N = 0 */
			if (st->count == 0) { *isnull = 1; return 0; }
			return d2u(u2d(st->v) / (double) st->count);
	}
	if (!st->has) { *isnull = 1; return 0; }
	return st->v;
}

static int is_agg(int32_t fn) { return fn < GG_WF_ROW_NUMBER || fn > GG_WF_NTH_VALUE; }

int ref_window(const gg_window *win, const int32_t *types, int ncols, const gg_exprpool *pool, const uint64_t *rows, uint64_t n,
               uint64_t *out, uint64_t *nout, char *err, int errlen)
{
	const int W = 1 + ncols, nf = win->numFuncs, W2 = W + nf;
	const int opt = win->frameOptions;
	const int rowsmode = (opt & GG_FRAMEOPTION_ROWS) != 0;
	Row *R;
	Arg args[GG_MAX_WINFUNCS][3];
	uint64_t m = 0;
	int rc = 0;
	err[0] = 0;
	for (int c = 0; c < ncols; c++) g_f8[c] = types[c] == GG_FLOAT8OID;
	for (int i = 0; i < nf; i++)
		for (int a = 0; a < 3; a++)
		{
			const int32_t root = win->funcs[i].arg[a];
			Arg *x = &args[i][a];
			memset(x, 0, sizeof *x);
			x->col = -1;
			if (root < 0) continue;
			x->present = 1;
			if (pool->nodes[root].kind == GG_E_VAR) x->col = pool->nodes[root].varattno - 1;
			else { x->isnull_const = pool->nodes[root].constisnull != 0; x->v = (uint64_t) pool->nodes[root].constvalue; }
		}
	R = malloc(sizeof *R * (size_t) (n ? n : 1));
	if (!R) return GG_ERR_NOMEM;
	for (uint64_t s = 0; s < n; s++)
		if (!(rows[s * W] & GG_DATUMROW_DEAD)) R[m++].w = rows + s * W;
	*nout = m;
	for (uint64_t ps = 0; ps < m && !rc; )
	{
		/* the partition [ps, pe) */
		uint64_t pe = ps + 1;
		while (pe < m && tuples_match(R[pe], R[ps], win->partColIdx, win->partNumCols)) pe++;
		const int64_t total = (int64_t) (pe - ps);
		AggState st[GG_MAX_WINFUNCS];
		int64_t aggbase[GG_MAX_WINFUNCS], aggupto[GG_MAX_WINFUNCS];
		int64_t rank = 0, dense = 0;
		/* ntile's partition-local context (windowfuncs.c:26-32) */
		int32_t nt_ntile[GG_MAX_WINFUNCS] = { 0 };
		int64_t nt_rows[GG_MAX_WINFUNCS] = { 0 }, nt_boundary[GG_MAX_WINFUNCS] = { 0 }, nt_rem[GG_MAX_WINFUNCS] = { 0 };
		for (int i = 0; i < nf; i++) { aggbase[i] = -1; aggupto[i] = -1; }
		uint64_t gs = ps, ge = ps;
		for (uint64_t j = ps; j < pe && !rc; j++)
		{
			/* rank_up (windowfuncs.c:60-80); a new peer group [gs, ge) starts where the order columns change (without ORDER BY
			 * the whole partition is one) */
			if (j == ps) { rank = 1; dense = 1; }
			else if (!tuples_match(R[j - 1], R[j], win->ordColIdx, win->ordNumCols)) { rank = (int64_t) (j - ps) + 1; dense++; }
			if (j == ge)
			{
				gs = j; ge = j + 1;
				while (ge < pe && tuples_match(R[ge], R[j], win->ordColIdx, win->ordNumCols)) ge++;
			}
			const int64_t head = (opt & GG_FRAMEOPTION_START_UNBOUNDED_PRECEDING) ? (int64_t) ps : rowsmode ? (int64_t) j : (int64_t) gs;
			const int64_t tail = (opt & GG_FRAMEOPTION_END_UNBOUNDED_FOLLOWING) ? (int64_t) pe - 1 : rowsmode ? (int64_t) j : (int64_t) ge - 1;
			uint64_t *o = out + j * (uint64_t) W2;
			uint64_t mask = R[j].w[0];
			memcpy(o + 1, R[j].w + 1, 8 * (size_t) ncols);
			for (int i = 0; i < nf && !rc; i++)
			{
				const int32_t fn = win->funcs[i].winfnoid;
				const Arg *A = args[i];
				uint64_t v = 0;
				int isnull = 0;
				if (is_agg(fn))
				{
					/* eval_windowaggregates: restart when the frame head moved, then advance up to the tail */
					if (aggbase[i] != head) { memset(&st[i], 0, sizeof st[i]); aggbase[i] = head; aggupto[i] = head; }
					while (aggupto[i] <= tail && !rc) rc = advance(fn, &st[i], &A[0], R[aggupto[i]++]);
					if (rc) { snprintf(err, (size_t) errlen, "value out of range: overflow"); break; }
					v = finalize(fn, &st[i], &isnull);
				}
				else switch (fn)
				{
					case GG_WF_ROW_NUMBER: v = j - ps + 1; break;
					case GG_WF_RANK: v = (uint64_t) rank; break;
					case GG_WF_DENSE_RANK: v = (uint64_t) dense; break;
					case GG_WF_PERCENT_RANK: v = d2u(total <= 1 ? 0.0 : (double) (rank - 1) / (double) (total - 1)); break;
					case GG_WF_CUME_DIST: v = d2u((double) (ge - ps) / (double) total); break;
					case GG_WF_NTILE:
					{
						if (nt_ntile[i] == 0)
						{
							int nnull;
							const int32_t nb = (int32_t) arg_value(&A[0], R[j], &nnull);
							if (nnull) { isnull = 1; break; }
							if (nb <= 0) { snprintf(err, (size_t) errlen, "argument of ntile must be greater than zero"); rc = GG_ERR_WINDOW_ARG; break; }
							nt_ntile[i] = 1; nt_rows[i] = 0;
							nt_boundary[i] = total / nb;
							if (nt_boundary[i] <= 0) nt_boundary[i] = 1;
							else { nt_rem[i] = total % nb; if (nt_rem[i] != 0) nt_boundary[i]++; }
						}
						nt_rows[i]++;
						if (nt_boundary[i] < nt_rows[i])
						{
							if (nt_rem[i] != 0 && nt_ntile[i] == nt_rem[i]) { nt_rem[i] = 0; nt_boundary[i] -= 1; }
							nt_ntile[i] += 1;
							nt_rows[i] = 1;
						}
						v = (uint64_t) (int64_t) nt_ntile[i];
						break;
					}
					case GG_WF_LAG: case GG_WF_LAG_OFFSET: case GG_WF_LAG_DEFAULT:
					case GG_WF_LEAD: case GG_WF_LEAD_OFFSET: case GG_WF_LEAD_DEFAULT:
					{
						const int fwd = fn >= GG_WF_LEAD;
						int64_t off = 1, t;
						if (A[1].present)
						{
							int onull;
							off = (int32_t) arg_value(&A[1], R[j], &onull);
							if (onull) { isnull = 1; break; }
						}
						t = (int64_t) j + (fwd ? off : -off);
						if (t >= (int64_t) ps && t < (int64_t) pe) v = arg_value(&A[0], R[t], &isnull);
						else if (A[2].present) v = arg_value(&A[2], R[j], &isnull);
						else isnull = 1;
						break;
					}
					case GG_WF_FIRST_VALUE: v = arg_value(&A[0], R[head], &isnull); break;
					case GG_WF_LAST_VALUE: v = arg_value(&A[0], R[tail], &isnull); break;
					case GG_WF_NTH_VALUE:
					{
						int nnull;
						const int32_t nth = (int32_t) arg_value(&A[1], R[j], &nnull);
						if (nnull) { isnull = 1; break; }
						if (nth <= 0) { snprintf(err, (size_t) errlen, "argument of nth_value must be greater than zero"); rc = GG_ERR_WINDOW_ARG; break; }
						if (head + nth - 1 > tail) isnull = 1;
						else v = arg_value(&A[0], R[head + nth - 1], &isnull);
						break;
					}
					default:
						snprintf(err, (size_t) errlen, "function %d", fn);
						rc = GG_ERR_UNSUPPORTED;
				}
				if (isnull) { mask |= 1ull << (ncols + i); v = 0; }
				o[W + i] = v;
			}
			o[0] = mask;
		}
		ps = pe;
	}
	free(R);
	return rc;
}
