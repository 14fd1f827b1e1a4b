/*
 * or_agg.c — ORACLE (test infrastructure): restatement of Greengage's hybrid
 * hash aggregate and of the aggregate transition / combine / final functions.
 *
 *   ExecAgg (AGG_HASHED driver)          src/backend/executor/nodeAgg.c:1123-1244
 *   agg_hash_initial_pass                src/backend/executor/execHHashagg.c:905-1081
 *   calc_hash_value                      src/backend/executor/execHHashagg.c:157-188
 *   lookup_agg_hash_entry                src/backend/executor/execHHashagg.c:456-585
 *   BUCKET_IDX / BLOOMVAL                src/backend/executor/execHHashagg.c:110-113
 *   initialize_aggregates                src/backend/executor/nodeAgg.c:261-330
 *   advance_aggregates / invoke_agg_trans_func   src/backend/executor/nodeAgg.c:413-681
 *   finalize_aggregate                   src/backend/executor/nodeAgg.c:871-999
 *   stage -> transfn/combinefn choice    src/backend/executor/nodeAgg.c:2123-2148
 *   pg_aggregate rows                    src/include/catalog/pg_aggregate.h:156-220
 *   float8pl / float8_accum / float8_combine / float8_avg   src/backend/utils/adt/float.c:782,1842-1996
 *   float8larger/smaller                 src/backend/utils/adt/float.c:690-720
 *   int8inc / int8pl / int4_sum          src/backend/utils/adt/int8.c:513-531,677-720; numeric.c int4_sum
 *
 * Spill to workfiles (execHHashagg.c:1093-1455) is out of scope (SURVEY §8f);
 * the streaming bottom stage (execHHashagg.c:996-1002,1034-1040) is restated:
 * when max_entries is reached the table is emitted and restarted, so a partial
 * stage may emit one group several times.
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include <pthread.h>
#include "gg_oracle.h"
#include "or_internal.h"

#define GROUPS_PER_BUCKET 5			/* gp_hashagg_groups_per_bucket, guc_gp.c:4221 */

typedef struct or_aggstate {			/* AggStatePerGroupData, nodeAgg.h:192 (+float8[3] by-ref state) */
	double  f[3];
	int64_t i;
	int     transValueIsNull;
	int     noTransValue;
	/* numeric_avg_accum's state (numeric.c:3057): N and the exact running sum, here 128 bits at display scale nscale */
	int64_t nlo, nhi, nN;
	int     nscale;
} or_aggstate;

typedef struct or_entry {				/* HashAggEntry, execHHashagg.h:41 */
	struct or_entry *next;
	uint32_t hashvalue;
	int64_t  key[GG_MAX_KEYS];
	int32_t  keylen[GG_MAX_KEYS];
	int32_t  keyisnull[GG_MAX_KEYS];
	or_aggstate st[GG_MAX_AGGS];
	or_exact *x[GG_MAX_AGGS];			/* exact mode: one per float8 aggregate, NULL otherwise */
} or_entry;

struct or_aggtable {
	const gg_agg *agg;
	const gg_exprpool *pool;
	unsigned nbuckets;
	unsigned pshift;
	or_entry **buckets;
	uint64_t *bloom;
	long num_entries;
	long max_entries;					/* stands in for the operator memory quota */
	int32_t keytype[GG_MAX_KEYS];
	/* rows streamed out before the end (streaming bottom stage) */
	gg_aggrow *streamed;
	int nstreamed, capstreamed;
	/* plain aggregation (numCols == 0): exactly one group, even on empty input (nodeAgg.c:1247-1400) */
	or_entry *plain;
	/* exact mode: whether this table keeps the records, and those of the streamed rows (nfloat per row) */
	int exact, nfloat;
	or_exact *streamed_x;
};

double
or_now(void)
{
	struct timespec ts;

	clock_gettime(CLOCK_MONOTONIC, &ts);
	return ts.tv_sec + ts.tv_nsec * 1e-9;
}

static inline double as_f8(int64_t v) { double d; memcpy(&d, &v, 8); return d; }

/* ---- exact mode (gg_oracle.h): what any order of summation must be measured against ---- */

static int exact_on;
static or_exact *exact_out;
static long exact_nout, exact_cap;

void
or_exact_mode(int on)
{
	exact_on = on;
}

long
or_exact_fetch(or_exact *out, long cap)
{
	long n = exact_nout < cap ? exact_nout : cap;

	memcpy(out, exact_out, (size_t) n * sizeof *out);
	return exact_nout;
}

static int
is_f8_agg(int aggfnoid)
{
	return aggfnoid == GG_AGG_SUM_FLOAT8 || aggfnoid == GG_AGG_AVG_FLOAT8 ||
		aggfnoid == GG_AGG_MIN_FLOAT8 || aggfnoid == GG_AGG_MAX_FLOAT8;
}

static void
exact_init(or_exact *x)
{
	memset(x, 0, sizeof *x);
	x->lowbit = x->lowbit_sq = INT32_MAX;
}

/* finite x = m * 2^e with integer m, e >= -1074: add sign*m at bit e + 1074 of the fixed-point limbs */
static void
limbs_add(int64_t *limb, double x, int *lowbit)
{
	int e, k, sh;
	uint64_t m;
	unsigned __int128 w;
	double f;

	if (x == 0.0)
		return;
	f = frexp(fabs(x), &e);				/* |x| = f * 2^e, f in [0.5, 1) */
	if (e - 53 >= -1074)
	{
		m = (uint64_t) ldexp(f, 53);
		e -= 53;
	}
	else
	{
		m = (uint64_t) ldexp(f, e + 1074);	/* subnormal */
		e = -1074;
	}
	if (lowbit && e + __builtin_ctzll(m) < *lowbit)
		*lowbit = e + __builtin_ctzll(m);
	sh = e + 1074;
	k = sh >> 5;
	w = (unsigned __int128) m << (sh & 31);
	for (; w != 0; k++, w >>= 32)
		limb[k] += x < 0 ? -(int64_t) (uint32_t) w : (int64_t) (uint32_t) w;
}

static void
exact_add(int aggfnoid, or_exact *x, double v)
{
	x->n++;
	if (x->n == 1)
		x->flags |= OR_XF_ALL_NEGZERO;
	if (!(v == 0.0 && signbit(v)))
		x->flags &= ~OR_XF_ALL_NEGZERO;
	if (v == 0.0)
		x->flags |= signbit(v) ? OR_XF_NEGZERO : OR_XF_POSZERO;
	if (isnan(v))
		x->flags |= OR_XF_NAN;
	else if (isinf(v))
		x->flags |= v > 0 ? OR_XF_PINF : OR_XF_NINF;
	if (!isfinite(v) || aggfnoid == GG_AGG_MIN_FLOAT8 || aggfnoid == GG_AGG_MAX_FLOAT8)
		return;
	limbs_add(x->sum, v, &x->lowbit);
	limbs_add(x->abs, fabs(v), NULL);
	if (isfinite(v * v))
		limbs_add(x->sq, v * v, &x->lowbit_sq);
}

/* carries into 32-bit digits; the top limb keeps the sign */
static void
limbs_normalise(int64_t *limb)
{
	int k;

	for (k = 0; k < OR_XLIMBS - 1; k++)
	{
		int64_t c = limb[k] >> 32;			/* arithmetic shift: floor division by 2^32 */

		limb[k] -= c * ((int64_t) 1 << 32);
		limb[k + 1] += c;
	}
}

static void
exact_emit(const or_exact *x)
{
	or_exact *o;

	if (exact_nout == exact_cap)
	{
		exact_cap = exact_cap ? exact_cap * 2 : 64;
		exact_out = realloc(exact_out, (size_t) exact_cap * sizeof *exact_out);
	}
	o = &exact_out[exact_nout++];
	if (x == NULL)
		exact_init(o);
	else
		*o = *x;
	limbs_normalise(o->sum);
	limbs_normalise(o->abs);
	limbs_normalise(o->sq);
}

static void
entry_exact_init(const or_aggtable *t, or_entry *e)
{
	int i;

	for (i = 0; t->exact && i < t->agg->numAggs; i++)
		if (is_f8_agg(t->agg->aggs[i].aggfnoid))
		{
			e->x[i] = malloc(sizeof(or_exact));
			exact_init(e->x[i]);
		}
}

static void
entry_free(or_entry *e)
{
	int i;

	for (i = 0; i < GG_MAX_AGGS; i++)
		free(e->x[i]);
	free(e);
}

/* ---- transition machinery ---- */

/* initialize_aggregates (nodeAgg.c:261): initValue from pg_aggregate.agginitval */
static void
init_state(int aggfnoid, int stage, or_aggstate *st)
{
	memset(st, 0, sizeof *st);
	(void) stage;
	switch (aggfnoid)
	{
		case GG_AGG_AVG_FLOAT8:			/* "{0,0,0}" */
			st->transValueIsNull = 0;
			st->noTransValue = 0;
			break;
		case GG_AGG_COUNT_STAR:
		case GG_AGG_COUNT_ANY:			/* "0" */
			st->i = 0;
			st->transValueIsNull = 0;
			st->noTransValue = 0;
			break;
		default:						/* initval NULL: sum, min, max */
			st->transValueIsNull = 1;
			st->noTransValue = 1;
			break;
	}
}

static int
float8_cmp_internal(double a, double b)
{
	if (isnan(a))
		return isnan(b) ? 0 : 1;
	if (isnan(b))
		return -1;
	return (a > b) - (a < b);
}

/* One transition step (transfn).  `arg` is the evaluated aggregate argument. */
static int
advance_trans(int aggfnoid, or_aggstate *st, const or_datum *arg)
{
	switch (aggfnoid)
	{
		case GG_AGG_COUNT_STAR:			/* int8inc, int8.c:677: overflow => ERROR */
			if (st->i == INT64_MAX)
				return OR_ERR_INT_OVERFLOW;
			st->i++;
			return 0;
		case GG_AGG_COUNT_ANY:			/* int8inc_any is strict on its "any" argument */
			if (arg->isnull)
				return 0;
			if (st->i == INT64_MAX)
				return OR_ERR_INT_OVERFLOW;
			st->i++;
			return 0;
		case GG_AGG_SUM_FLOAT8:			/* float8pl, strict, initval NULL (nodeAgg.c:425-457) */
		{
			double x, r;

			if (arg->isnull)
				return 0;
			x = as_f8(arg->v);
			if (st->noTransValue)
			{
				st->f[0] = x;
				st->transValueIsNull = 0;
				st->noTransValue = 0;
				return 0;
			}
			r = st->f[0] + x;
			if (isinf(r) && !(isinf(st->f[0]) || isinf(x)))
				return OR_ERR_FLOAT_OVERFLOW;
			st->f[0] = r;
			return 0;
		}
		case GG_AGG_AVG_FLOAT8:			/* float8_accum (float.c:1878), strict */
		{
			double x, sumX, sumX2;

			if (arg->isnull)
				return 0;
			x = as_f8(arg->v);
			st->f[0] += 1.0;
			sumX = st->f[1] + x;
			if (isinf(sumX) && !(isinf(st->f[1]) || isinf(x)))
				return OR_ERR_FLOAT_OVERFLOW;
			sumX2 = st->f[2] + x * x;
			if (isinf(sumX2) && !(isinf(st->f[2]) || isinf(x)))
				return OR_ERR_FLOAT_OVERFLOW;
			st->f[1] = sumX;
			st->f[2] = sumX2;
			return 0;
		}
		case GG_AGG_SUM_NUMERIC:
		case GG_AGG_AVG_NUMERIC:		/* numeric_avg_accum: NULL inputs are skipped (numeric.c:3063) */
			if (arg->isnull)
				return 0;
			st->transValueIsNull = 0;
			st->noTransValue = 0;
			return or_numeric_accum(&st->nlo, &st->nhi, &st->nscale, &st->nN, arg);
		case GG_AGG_SUM_INT4:			/* int4_sum (numeric.c): not strict, NULL-aware, no overflow check */
			if (arg->isnull)
				return 0;
			if (st->transValueIsNull)
			{
				st->i = (int64_t) (int32_t) arg->v;
				st->transValueIsNull = 0;
				st->noTransValue = 0;
			}
			else
				st->i += (int64_t) (int32_t) arg->v;
			return 0;
		case GG_AGG_MAX_FLOAT8:
		case GG_AGG_MIN_FLOAT8:			/* float8larger/smaller (float.c:690-720), strict */
		{
			double x;

			if (arg->isnull)
				return 0;
			x = as_f8(arg->v);
			if (st->noTransValue)
			{
				st->f[0] = x;
				st->transValueIsNull = 0;
				st->noTransValue = 0;
				return 0;
			}
			if (aggfnoid == GG_AGG_MAX_FLOAT8)
				st->f[0] = float8_cmp_internal(st->f[0], x) > 0 ? st->f[0] : x;
			else
				st->f[0] = float8_cmp_internal(st->f[0], x) < 0 ? st->f[0] : x;
			return 0;
		}
		case GG_AGG_MAX_INT8: case GG_AGG_MIN_INT8:
		case GG_AGG_MAX_INT4: case GG_AGG_MIN_INT4:
		case GG_AGG_MAX_DATE: case GG_AGG_MIN_DATE:
		{
			int64_t x;
			int ismax = (aggfnoid == GG_AGG_MAX_INT8 || aggfnoid == GG_AGG_MAX_INT4 ||
						 aggfnoid == GG_AGG_MAX_DATE);

			if (arg->isnull)
				return 0;
			x = (aggfnoid == GG_AGG_MAX_INT8 || aggfnoid == GG_AGG_MIN_INT8) ? arg->v : (int64_t) (int32_t) arg->v;
			if (st->noTransValue)
			{
				st->i = x;
				st->transValueIsNull = 0;
				st->noTransValue = 0;
				return 0;
			}
			if (ismax ? x > st->i : x < st->i)
				st->i = x;
			return 0;
		}
	}
	return OR_ERR_UNSUPPORTED;
}

/* One combine step (combinefn, FINAL stage): the partial state arrives as a gg_aggval */
static int
advance_combine(int aggfnoid, or_aggstate *st, const gg_aggval *in)
{
	switch (aggfnoid)
	{
		case GG_AGG_COUNT_STAR:
		case GG_AGG_COUNT_ANY:
		case GG_AGG_SUM_INT4:			/* int8pl (int8.c:513), strict; count's state starts at 0, sum's at NULL */
		{
			int64_t r;

			if (in->isnull)
				return 0;
			if (st->noTransValue)
			{
				st->i = in->i;
				st->transValueIsNull = 0;
				st->noTransValue = 0;
				return 0;
			}
			if (__builtin_add_overflow(st->i, in->i, &r))
				return OR_ERR_INT_OVERFLOW;	/* "bigint out of range" */
			st->i = r;
			return 0;
		}
		case GG_AGG_SUM_FLOAT8:			/* float8pl */
		{
			double r;

			if (in->isnull)
				return 0;
			if (st->noTransValue)
			{
				st->f[0] = in->f[0];
				st->transValueIsNull = 0;
				st->noTransValue = 0;
				return 0;
			}
			r = st->f[0] + in->f[0];
			if (isinf(r) && !(isinf(st->f[0]) || isinf(in->f[0])))
				return OR_ERR_FLOAT_OVERFLOW;
			st->f[0] = r;
			return 0;
		}
		case GG_AGG_AVG_FLOAT8:			/* float8_combine, float.c:1842 */
		{
			double sumX, sumX2;

			if (in->isnull)
				return 0;
			st->f[0] += in->f[0];
			sumX = st->f[1] + in->f[1];
			if (isinf(sumX) && !(isinf(st->f[1]) || isinf(in->f[1])))
				return OR_ERR_FLOAT_OVERFLOW;
			sumX2 = st->f[2] + in->f[2];
			if (isinf(sumX2) && !(isinf(st->f[2]) || isinf(in->f[2])))
				return OR_ERR_FLOAT_OVERFLOW;
			st->f[1] = sumX;
			st->f[2] = sumX2;
			return 0;
		}
		case GG_AGG_MAX_FLOAT8: case GG_AGG_MIN_FLOAT8:
		{
			or_datum d;

			memset(&d, 0, sizeof d);
			d.isnull = in->isnull;
			memcpy(&d.v, &in->f[0], 8);
			return advance_trans(aggfnoid, st, &d);
		}
		case GG_AGG_MAX_INT8: case GG_AGG_MIN_INT8:
		case GG_AGG_MAX_INT4: case GG_AGG_MIN_INT4:
		case GG_AGG_MAX_DATE: case GG_AGG_MIN_DATE:
		{
			or_datum d;

			memset(&d, 0, sizeof d);
			d.isnull = in->isnull;
			d.v = in->i;
			return advance_trans(aggfnoid, st, &d);
		}
	}
	return OR_ERR_UNSUPPORTED;
}

/* combine's initial state for count differs from transfn's: the FINAL-stage count
 * still has initval "0" and combinefn int8pl is then called with a non-NULL state */
static void
init_state_final(int aggfnoid, or_aggstate *st)
{
	init_state(aggfnoid, GG_AGGSTAGE_FINAL, st);
}

/* finalize_aggregate (nodeAgg.c:871-999) */
static void
finalize(int aggfnoid, int stage, const or_aggstate *st, gg_aggval *out)
{
	memset(out, 0, sizeof *out);
	if (stage == GG_AGGSTAGE_PARTIAL)
	{
		/* no finalfn/serialfn in the partial stage: ship the transition value (nodeAgg.c:975-979) */
		out->isnull = st->transValueIsNull;
		out->f[0] = st->f[0];
		out->f[1] = st->f[1];
		out->f[2] = st->f[2];
		out->i = st->i;
		return;
	}
	switch (aggfnoid)
	{
		case GG_AGG_SUM_NUMERIC:		/* numeric_sum (numeric.c:3205): NULL without input */
		case GG_AGG_AVG_NUMERIC:		/* numeric_avg (numeric.c:3173): numeric_div(sum, N) */
		{
			int64_t lo = st->nlo, hi = st->nhi;
			int sc = st->nscale;

			if (st->nN == 0)
			{
				out->isnull = 1;
				return;
			}
			if (aggfnoid == GG_AGG_AVG_NUMERIC && or_numeric_avg(st->nlo, st->nhi, st->nscale, st->nN, &lo, &hi, &sc) != 0)
			{
				out->isnull = 1; out->pad = 1;		/* does not fit 128 bits */
				return;
			}
			out->i = lo;
			memcpy(&out->f[0], &hi, 8);
			out->f[1] = (double) sc;
			return;
		}
		case GG_AGG_AVG_FLOAT8:			/* float8_avg, float.c:1982 */
			if (st->f[0] == 0.0)
				out->isnull = 1;
			else
				out->f[0] = st->f[1] / st->f[0];
			return;
		default:
			out->isnull = st->transValueIsNull;
			out->f[0] = st->f[0];
			out->i = st->i;
			return;
	}
}

/* ---- the hash table ---- */

or_aggtable *
or_aggtable_create(const gg_agg *agg, const gg_exprpool *pool, long max_entries)
{
	or_aggtable *t = calloc(1, sizeof *t);
	int i;

	t->agg = agg;
	t->pool = pool;
	t->nbuckets = 1024;
	t->pshift = 0;
	t->buckets = calloc(t->nbuckets, sizeof *t->buckets);
	t->bloom = calloc(t->nbuckets, sizeof *t->bloom);
	t->max_entries = max_entries;
	t->exact = exact_on && agg->aggstage != GG_AGGSTAGE_FINAL;
	for (i = 0; i < agg->numAggs; i++)
		t->nfloat += is_f8_agg(agg->aggs[i].aggfnoid);
	for (i = 0; i < agg->numCols; i++)
		t->keytype[i] = pool ? pool->nodes[agg->grpCol[i]].rettype : 0;
	return t;
}

static void
free_entries(or_aggtable *t)
{
	unsigned b;

	for (b = 0; b < t->nbuckets; b++)
	{
		or_entry *e = t->buckets[b];

		while (e)
		{
			or_entry *n = e->next;

			entry_free(e);
			e = n;
		}
		t->buckets[b] = NULL;
		t->bloom[b] = 0;
	}
	t->num_entries = 0;
}

void
or_aggtable_free(or_aggtable *t)
{
	if (!t)
		return;
	free_entries(t);
	if (t->plain)
		entry_free(t->plain);
	free(t->streamed_x);
	free(t->buckets);
	free(t->bloom);
	free(t->streamed);
	free(t);
}

/* expand_hash_table (execHHashagg.c:1477-1540): double the bucket array, re-link */
static void
expand(or_aggtable *t)
{
	unsigned nb = t->nbuckets * 2, b;
	or_entry **nbk = calloc(nb, sizeof *nbk);
	uint64_t *nbl = calloc(nb, sizeof *nbl);

	for (b = 0; b < t->nbuckets; b++)
	{
		or_entry *e = t->buckets[b];

		while (e)
		{
			or_entry *n = e->next;
			unsigned idx = (e->hashvalue >> t->pshift) & (nb - 1);

			e->next = nbk[idx];
			nbk[idx] = e;
			nbl[idx] |= ((uint64_t) 1) << ((e->hashvalue >> 23) & 0x3f);
			e = n;
		}
	}
	free(t->buckets);
	free(t->bloom);
	t->buckets = nbk;
	t->bloom = nbl;
	t->nbuckets = nb;
}

static int
keys_equal(const or_aggtable *t, const or_entry *e, const int64_t *key, const int32_t *keylen,
		   const int32_t *keyisnull)
{
	int i;

	/* execHHashagg.c:500-531: both non-NULL and eqfn true, or both NULL */
	for (i = 0; i < t->agg->numCols; i++)
	{
		if (keyisnull[i] || e->keyisnull[i])
		{
			if (keyisnull[i] && e->keyisnull[i])
				continue;
			return 0;
		}
		switch (t->keytype[i])
		{
			case GG_BPCHAROID:		/* bpchareq on blank-stripped packed bytes */
			case GG_VARCHAROID:
			case GG_TEXTOID:
				if (keylen[i] != e->keylen[i] || key[i] != e->key[i])
					return 0;
				break;
			case GG_FLOAT8OID:		/* float8eq: NaN = NaN, -0 = +0 */
				if (float8_cmp_internal(as_f8(key[i]), as_f8(e->key[i])) != 0)
					return 0;
				break;
			case GG_INT4OID:
			case GG_DATEOID:
				if ((int32_t) key[i] != (int32_t) e->key[i])
					return 0;
				break;
			default:
				if (key[i] != e->key[i])
					return 0;
		}
	}
	return 1;
}

/* Evaluate the grouping columns of the current input row into packed key datums */
static int
eval_keys(or_aggtable *t, or_row *outer, or_row *inner, int64_t *key, int32_t *keylen, int32_t *keyisnull)
{
	int i, rc;

	for (i = 0; i < t->agg->numCols; i++)
	{
		or_datum d;

		if ((rc = or_eval(t->pool, t->agg->grpCol[i], outer, inner, &d)) != 0)
			return rc;
		keyisnull[i] = d.isnull;
		key[i] = 0;
		keylen[i] = 0;
		if (d.isnull)
			continue;
		if (d.ptr)
		{
			int len = d.len;

			if (t->keytype[i] == GG_BPCHAROID)
				len = or_bctruelen((const char *) d.ptr, len);
			if (len > 8)
				return OR_ERR_UNSUPPORTED;
			memcpy(&key[i], d.ptr, (size_t) len);
			keylen[i] = len;
		}
		else
			key[i] = d.v;
	}
	return 0;
}

/* calc_hash_value (execHHashagg.c:157): hash_any over the array of per-key hashes, NULL -> 0xdeadbeef */
static uint32_t
calc_hash_value(const or_aggtable *t, const int64_t *key, const int32_t *keylen, const int32_t *keyisnull)
{
	uint32_t buf[GG_MAX_KEYS];
	int i;

	for (i = 0; i < t->agg->numCols; i++)
		buf[i] = keyisnull[i] ? 0xdeadbeef : or_hash_datum(t->keytype[i], key[i], keylen[i]);
	return or_hash_any((const unsigned char *) buf, t->agg->numCols * (int) sizeof(uint32_t));
}

static void
row_from_entry(const or_aggtable *t, const or_entry *e, gg_aggrow *row)
{
	int i;

	memset(row, 0, sizeof *row);
	for (i = 0; i < t->agg->numCols; i++)
	{
		row->key[i] = e->key[i];
		row->keylen[i] = e->keylen[i];
		row->keyisnull[i] = e->keyisnull[i];
	}
	for (i = 0; i < t->agg->numAggs; i++)
		finalize(t->agg->aggs[i].aggfnoid, t->agg->aggstage, &e->st[i], &row->agg[i]);
}

/* streaming bottom stage: emit everything and start over (agg_hash_stream, execHHashagg.c:1832) */
static void
stream_out(or_aggtable *t)
{
	unsigned b;

	for (b = 0; b < t->nbuckets; b++)
	{
		or_entry *e;

		for (e = t->buckets[b]; e; e = e->next)
		{
			int i, f = 0;

			if (t->nstreamed == t->capstreamed)
			{
				t->capstreamed = t->capstreamed ? t->capstreamed * 2 : 64;
				t->streamed = realloc(t->streamed, (size_t) t->capstreamed * sizeof(gg_aggrow));
				if (t->exact)
					t->streamed_x = realloc(t->streamed_x, (size_t) t->capstreamed * t->nfloat * sizeof(or_exact));
			}
			for (i = 0; t->exact && i < t->agg->numAggs; i++)
				if (e->x[i])
					t->streamed_x[(size_t) t->nstreamed * t->nfloat + f++] = *e->x[i];
			row_from_entry(t, e, &t->streamed[t->nstreamed++]);
		}
	}
	free_entries(t);
}

static or_entry *
lookup(or_aggtable *t, uint32_t hashkey, const int64_t *key, const int32_t *keylen,
	   const int32_t *keyisnull, int final_stage, int *isnew)
{
	unsigned bucket_idx = (hashkey >> t->pshift) & (t->nbuckets - 1);
	uint64_t bloomval = ((uint64_t) 1) << ((hashkey >> 23) & 0x3f);
	or_entry *entry = (t->bloom[bucket_idx] & bloomval) == 0 ? NULL : t->buckets[bucket_idx];
	int i;

	*isnew = 0;
	while (entry != NULL)
	{
		if (hashkey == entry->hashvalue && keys_equal(t, entry, key, keylen, keyisnull))
			return entry;
		entry = entry->next;
	}
	if (t->max_entries > 0 && t->num_entries >= t->max_entries)
		return NULL;					/* no room (makeHashAggEntryForInput returned NULL) */
	entry = calloc(1, sizeof *entry);
	entry->hashvalue = hashkey;
	for (i = 0; i < t->agg->numCols; i++)
	{
		entry->key[i] = key[i];
		entry->keylen[i] = keylen[i];
		entry->keyisnull[i] = keyisnull[i];
	}
	entry_exact_init(t, entry);
	for (i = 0; i < t->agg->numAggs; i++)
	{
		if (final_stage)
			init_state_final(t->agg->aggs[i].aggfnoid, &entry->st[i]);
		else
			init_state(t->agg->aggs[i].aggfnoid, t->agg->aggstage, &entry->st[i]);
	}
	if (t->num_entries >= (long) t->nbuckets * GROUPS_PER_BUCKET)
	{
		expand(t);
		bucket_idx = (hashkey >> t->pshift) & (t->nbuckets - 1);
	}
	entry->next = t->buckets[bucket_idx];
	t->buckets[bucket_idx] = entry;
	t->bloom[bucket_idx] |= bloomval;
	t->num_entries++;
	*isnew = 1;
	return entry;
}

static or_entry *
plain_entry(or_aggtable *t, int final_stage)
{
	int i;

	if (!t->plain)
	{
		t->plain = calloc(1, sizeof(or_entry));
		entry_exact_init(t, t->plain);
		for (i = 0; i < t->agg->numAggs; i++)
		{
			if (final_stage)
				init_state_final(t->agg->aggs[i].aggfnoid, &t->plain->st[i]);
			else
				init_state(t->agg->aggs[i].aggfnoid, t->agg->aggstage, &t->plain->st[i]);
		}
	}
	return t->plain;
}

/* One input row of a NORMAL or PARTIAL stage: lookup + advance_aggregates (nodeAgg.c:545) */
int
or_aggtable_advance(or_aggtable *t, or_row *outer, or_row *inner)
{
	int64_t key[GG_MAX_KEYS];
	int32_t keylen[GG_MAX_KEYS], keyisnull[GG_MAX_KEYS];
	or_entry *e;
	int i, rc, isnew;

	if (t->agg->numCols == 0)
		e = plain_entry(t, 0);
	else
	{
		uint32_t h;

		if ((rc = eval_keys(t, outer, inner, key, keylen, keyisnull)) != 0)
			return rc;
		h = calc_hash_value(t, key, keylen, keyisnull);
		e = lookup(t, h, key, keylen, keyisnull, 0, &isnew);
		if (e == NULL)
		{
			stream_out(t);
			e = lookup(t, h, key, keylen, keyisnull, 0, &isnew);
		}
	}
	for (i = 0; i < t->agg->numAggs; i++)
	{
		const gg_aggref *ar = &t->agg->aggs[i];
		or_datum arg;

		memset(&arg, 0, sizeof arg);
		if (ar->arg >= 0 && (rc = or_eval(t->pool, ar->arg, outer, inner, &arg)) != 0)
			return rc;
		if ((rc = advance_trans(ar->aggfnoid, &e->st[i], &arg)) != 0)
			return rc;
		if (e->x[i] && !arg.isnull)
			exact_add(ar->aggfnoid, e->x[i], as_f8(arg.v));
	}
	return 0;
}

int
or_aggtable_emit(or_aggtable *t, gg_aggrow *out, int outcap, int *nout)
{
	unsigned b;
	int n = 0, i, j;

	if (t->exact)
		exact_nout = 0;
	for (i = 0; i < t->nstreamed; i++)
	{
		if (n >= outcap)
			return OR_ERR_NOMEM;
		out[n++] = t->streamed[i];
		for (j = 0; t->exact && j < t->nfloat; j++)
			exact_emit(&t->streamed_x[(size_t) i * t->nfloat + j]);
	}
	if (t->agg->numCols == 0)
	{
		or_entry *e = plain_entry(t, t->agg->aggstage == GG_AGGSTAGE_FINAL);

		if (n >= outcap)
			return OR_ERR_NOMEM;
		row_from_entry(t, e, &out[n++]);
		for (j = 0; t->exact && j < t->agg->numAggs; j++)
			if (e->x[j])
				exact_emit(e->x[j]);
	}
	for (b = 0; b < t->nbuckets; b++)
	{
		or_entry *e;

		for (e = t->buckets[b]; e; e = e->next)
		{
			if (n >= outcap)
				return OR_ERR_NOMEM;
			row_from_entry(t, e, &out[n++]);
			for (j = 0; t->exact && j < t->agg->numAggs; j++)
				if (e->x[j])
					exact_emit(e->x[j]);
		}
	}
	*nout = n;
	return 0;
}

/* ---- SeqScan -> qual -> Agg (ExecScan, execScan.c:111-214) ---- */

static int
scan_into_table(const gg_scan *scan, const gg_exprpool *pool, const uint8_t *pages, uint64_t nblocks,
				or_aggtable *t, uint64_t *rows_scanned, uint64_t *rows_passed)
{
	or_heapscan *hs = malloc(sizeof *hs);
	const uint8_t *tup;
	uint64_t nscan = 0, npass = 0;
	or_row row;
	int rc = 0;

	or_scan_begin(hs, &scan->desc, pages, nblocks);
	while ((tup = or_scan_next(hs, NULL)) != NULL)
	{
		nscan++;
		or_row_store(&row, &scan->desc, tup);
		if (scan->qual >= 0)
		{
			or_datum q;

			if ((rc = or_eval(pool, scan->qual, &row, NULL, &q)) != 0)
				break;
			if (q.isnull || !q.v)		/* ExecQual: NULL counts as false (execQual.c:6300) */
				continue;
		}
		npass++;
		if ((rc = or_aggtable_advance(t, &row, NULL)) != 0)
			break;
	}
	if (rc == 0 && hs->error)
		rc = hs->error;
	free(hs);
	if (rows_scanned)
		*rows_scanned = nscan;
	if (rows_passed)
		*rows_passed = npass;
	return rc;
}

int
or_seqscan_agg(const gg_scan *scan, const gg_agg *agg, const gg_exprpool *pool,
			   const uint8_t *pages, uint64_t nblocks,
			   gg_aggrow *out, int outcap, int *nout,
			   uint64_t *rows_scanned, uint64_t *rows_passed)
{
	or_aggtable *t = or_aggtable_create(agg, pool, 0);
	int rc = scan_into_table(scan, pool, pages, nblocks, t, rows_scanned, rows_passed);

	if (rc == 0)
		rc = or_aggtable_emit(t, out, outcap, nout);
	or_aggtable_free(t);
	return rc;
}

/* FINAL stage: group the partial rows again and run the combine functions */
int
or_agg_final(const gg_agg *agg, const gg_aggrow *in, int nin, gg_aggrow *out, int outcap, int *nout)
{
	gg_agg fin = *agg;
	or_aggtable *t;
	int r, i, rc = 0, isnew;

	fin.aggstage = GG_AGGSTAGE_FINAL;
	t = or_aggtable_create(&fin, NULL, 0);
	/* key types are not in a pool here: the caller passes them in grpCol[] as type OIDs */
	for (i = 0; i < agg->numCols; i++)
		t->keytype[i] = agg->grpCol[i];
	for (r = 0; r < nin && rc == 0; r++)
	{
		or_entry *e;

		if (agg->numCols == 0)
			e = plain_entry(t, 1);
		else
		{
			uint32_t h = calc_hash_value(t, in[r].key, in[r].keylen, in[r].keyisnull);

			e = lookup(t, h, in[r].key, in[r].keylen, in[r].keyisnull, 1, &isnew);
		}
		for (i = 0; i < agg->numAggs && rc == 0; i++)
			rc = advance_combine(agg->aggs[i].aggfnoid, &e->st[i], &in[r].agg[i]);
	}
	if (rc == 0)
		rc = or_aggtable_emit(t, out, outcap, nout);
	or_aggtable_free(t);
	return rc;
}

/* BASELINE config 0: SELECT count(*) — per segment SeqScan -> partial Agg(int8inc),
 * Gather Motion, final Agg(int8pl) on the QD */
int64_t
or_count_star_2stage(const uint8_t *const *seg_pages, const uint64_t *seg_nblocks, int nsegs)
{
	int64_t total = 0;
	int s;

	for (s = 0; s < nsegs; s++)
	{
		or_heapscan *hs = malloc(sizeof *hs);
		int64_t partial = 0;
		gg_tupdesc dummy;

		memset(&dummy, 0, sizeof dummy);
		or_scan_begin(hs, &dummy, seg_pages[s], seg_nblocks[s]);
		while (or_scan_next(hs, NULL) != NULL)
			partial++;					/* int8inc */
		free(hs);
		total += partial;				/* int8pl */
	}
	return total;
}

/* ---- multi-threaded CPU baseline: one thread per "segment" over a block range ---- */

typedef struct mt_arg {
	const gg_scan *scan;
	const gg_agg *partial;
	const gg_exprpool *pool;
	const uint8_t *pages;
	uint64_t nblocks;
	gg_aggrow rows[256];
	int nrows;
	int rc;
	uint64_t scanned;
} mt_arg;

static void *
mt_worker(void *p)
{
	mt_arg *a = p;

	a->rc = or_seqscan_agg(a->scan, a->partial, a->pool, a->pages, a->nblocks,
						   a->rows, 256, &a->nrows, &a->scanned, NULL);
	return NULL;
}

int
or_seqscan_agg_mt(const gg_scan *scan, const gg_agg *partial, const gg_agg *final,
				  const gg_exprpool *pool, const uint8_t *pages, uint64_t nblocks, int nthreads,
				  gg_aggrow *out, int outcap, int *nout, double *seconds, uint64_t *rows_scanned)
{
	mt_arg *args = calloc((size_t) nthreads, sizeof *args);
	pthread_t *th = calloc((size_t) nthreads, sizeof *th);
	gg_aggrow *all;
	gg_agg fin = *final;
	int i, nall = 0, rc = 0;
	double t0;
	uint64_t per = (nblocks + nthreads - 1) / nthreads, scanned = 0;

	t0 = or_now();
	for (i = 0; i < nthreads; i++)
	{
		uint64_t b0 = per * i, b1 = b0 + per;

		if (b0 > nblocks) b0 = nblocks;
		if (b1 > nblocks) b1 = nblocks;
		args[i].scan = scan;
		args[i].partial = partial;
		args[i].pool = pool;
		args[i].pages = pages + b0 * (uint64_t) GG_BLCKSZ;
		args[i].nblocks = b1 - b0;
		pthread_create(&th[i], NULL, mt_worker, &args[i]);
	}
	all = malloc(sizeof(gg_aggrow) * 256 * (size_t) nthreads);
	for (i = 0; i < nthreads; i++)
	{
		pthread_join(th[i], NULL);
		if (args[i].rc)
			rc = args[i].rc;
		memcpy(all + nall, args[i].rows, sizeof(gg_aggrow) * (size_t) args[i].nrows);
		nall += args[i].nrows;
		scanned += args[i].scanned;
	}
	if (rc == 0)
	{
		/* final stage: key types from the pool */
		for (i = 0; i < final->numCols; i++)
			fin.grpCol[i] = pool->nodes[partial->grpCol[i]].rettype;
		rc = or_agg_final(&fin, all, nall, out, outcap, nout);
	}
	if (seconds)
		*seconds = or_now() - t0;
	if (rows_scanned)
		*rows_scanned = scanned;
	free(all);
	free(args);
	free(th);
	return rc;
}
