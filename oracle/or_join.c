/*
 * or_join.c — ORACLE (test infrastructure): restatement of Hash + HashJoin.
 *
 *   MultiExecHash (build loop)            src/backend/executor/nodeHash.c:88-176
 *   ExecHashTableCreate / ChooseHashTableSize   src/backend/executor/nodeHash.c:270-659
 *   ExecHashGetHashValue                  src/backend/executor/nodeHash.c:1003-1096
 *   ExecHashGetBucketAndBatch             src/backend/executor/nodeHash.c:1132-1151
 *   ExecHashTableInsert                   src/backend/executor/nodeHash.c:906-986
 *   ExecScanHashBucket                    src/backend/executor/nodeHash.c:1164-1222
 *   ExecHashJoin_guts state machine       src/backend/executor/nodeHashjoin.c:78-509
 *   ExecHashJoinOuterGetTuple             src/backend/executor/nodeHashjoin.c:801-897
 *
 * Single batch only: multi-batch spill (nodeHash.c:713, nodeHashjoin.c:906) is
 * out of scope (SURVEY §8f).  Join types: inner, left, right, full, semi, anti, LASJ_NOTIN.
 */
#include <stdlib.h>
#include <string.h>
#include "gg_oracle.h"
#include "or_internal.h"

#define TUPLES_PER_BUCKET 5			/* gp_hashjoin_tuples_per_bucket, guc_gp.c:4210 */

typedef struct hj_tuple {				/* HashJoinTupleData {next, hashvalue} + tuple, hashjoin.h:70-88 */
	struct hj_tuple *next;
	uint32_t hashvalue;
	const uint8_t *tuple;
	uint64_t tid;
	int matched;					/* MemTupleSetMatch (HEAP_TUPLE_HAS_MATCH), nodeHashjoin.c:386 */
	int nullkey;					/* kept only for right/full joins: never matches */
} hj_tuple;

typedef struct hj_table {
	uint32_t nbuckets;
	hj_tuple **buckets;
	hj_tuple *arena;
	uint64_t ntuples, cap;
} hj_table;

/* nodeHash.c:1003 — h = rotl1(h) ^ hashfn(key); NULL key => reject unless keep_nulls */
static int
hash_keys(const gg_exprpool *pool, const int32_t *keys, int nkeys, or_row *row, int is_outer,
		  int keep_nulls, uint32_t *hashvalue, int *ok)
{
	uint32_t hashkey = 0;
	int i, rc;

	*ok = 1;
	for (i = 0; i < nkeys; i++)
	{
		or_datum d;

		hashkey = (hashkey << 1) | ((hashkey & 0x80000000) ? 1 : 0);
		if ((rc = or_eval(pool, keys[i], is_outer ? row : NULL, is_outer ? NULL : row, &d)) != 0)
			return rc;
		if (d.isnull)
		{
			if (!keep_nulls)
				*ok = 0;
		}
		else if (*ok)
		{
			int32_t typ = pool->nodes[keys[i]].rettype;
			int64_t v = d.v;
			int32_t len = d.len;

			if (d.ptr)
			{
				if (typ == GG_BPCHAROID)
					len = or_bctruelen((const char *) d.ptr, len);
				if (len > 8)
					return OR_ERR_UNSUPPORTED;
				v = 0;
				memcpy(&v, d.ptr, (size_t) len);
			}
			hashkey ^= or_hash_datum(typ, v, len);
		}
	}
	*hashvalue = hashkey;
	return 0;
}

/* hashqualclauses: outerkey[i] = innerkey[i] for all i (strict equality operators) */
static int
keys_match(const gg_exprpool *pool, const gg_hashjoin *hj, or_row *outer, or_row *inner, int *match)
{
	int i, rc;

	*match = 1;
	for (i = 0; i < hj->nkeys; i++)
	{
		or_datum a, b;
		int32_t typ = pool->nodes[hj->outerkey[i]].rettype;

		if ((rc = or_eval(pool, hj->outerkey[i], outer, NULL, &a)) != 0)
			return rc;
		if ((rc = or_eval(pool, hj->innerkey[i], NULL, inner, &b)) != 0)
			return rc;
		if (a.isnull || b.isnull)
		{
			*match = 0;
			return 0;
		}
		if (a.ptr || b.ptr)
		{
			if (typ == GG_BPCHAROID)
				*match = or_bpchareq((const char *) a.ptr, a.len, (const char *) b.ptr, b.len);
			else
				*match = (a.len == b.len && memcmp(a.ptr, b.ptr, (size_t) a.len) == 0);
		}
		else if (typ == GG_INT4OID || typ == GG_DATEOID || typ == GG_INT8OID)
		{
			/* int4eq / int48eq / int84eq / int8eq (integer_ops): each side widened from its own type, never truncated */
			int32_t ityp = pool->nodes[hj->innerkey[i]].rettype;
			int64_t x = (typ == GG_INT8OID) ? a.v : (int64_t) (int32_t) a.v;
			int64_t y = (ityp == GG_INT8OID || ityp == GG_TIMESTAMPOID) ? b.v : (int64_t) (int32_t) b.v;

			*match = x == y;
		}
		else if (typ == GG_FLOAT8OID)
		{
			double x, y;

			memcpy(&x, &a.v, 8);
			memcpy(&y, &b.v, 8);
			*match = (x == y) || (x != x && y != y);	/* float8eq: NaN = NaN */
		}
		else
			*match = a.v == b.v;
		if (!*match)
			return 0;
	}
	return 0;
}

typedef int (*hj_emit_fn)(void *ctx, or_row *outer, uint64_t otid, or_row *inner, uint64_t itid);

static int
run_join(const gg_scan *outer, const gg_scan *inner, const gg_hashjoin *hj, const gg_exprpool *pool,
		 const uint8_t *outer_pages, uint64_t outer_nblocks,
		 const uint8_t *inner_pages, uint64_t inner_nblocks, hj_emit_fn emit, void *ctx)
{
	or_heapscan *hs = malloc(sizeof *hs);
	hj_table tab;
	const uint8_t *tup;
	uint64_t tid;
	or_row row, irow;
	int rc = 0;
	uint32_t nb;
	const int fill_inner = (hj->jointype == GG_JOIN_RIGHT || hj->jointype == GG_JOIN_FULL);	/* HJ_FILL_INNER */
	const int fill_outer = (hj->jointype == GG_JOIN_LEFT || hj->jointype == GG_JOIN_FULL ||
							hj->jointype == GG_JOIN_ANTI || hj->jointype == GG_JOIN_LASJ_NOTIN);
	const int lasj = hj->jointype == GG_JOIN_LASJ_NOTIN;
	int inner_has_nullkey = 0;

	/* ---- HJ_BUILD_HASHTABLE: MultiExecHash drains the inner side ---- */
	memset(&tab, 0, sizeof tab);
	tab.cap = 1024;
	tab.arena = malloc(tab.cap * sizeof(hj_tuple));
	or_scan_begin(hs, &inner->desc, inner_pages, inner_nblocks);
	while ((tup = or_scan_next(hs, &tid)) != NULL)
	{
		uint32_t h;
		int ok;

		or_row_store(&row, &inner->desc, tup);
		if (inner->qual >= 0)
		{
			or_datum q;

			if ((rc = or_eval(pool, inner->qual, NULL, &row, &q)) != 0)
				goto done;
			if (q.isnull || !q.v)
				continue;
		}
		if ((rc = hash_keys(pool, hj->innerkey, hj->nkeys, &row, 0, 0, &h, &ok)) != 0)
			goto done;
		if (!ok)
		{
			/* NULL key never matches a strict operator (nodeHash.c:1070-1077): dropped, unless a right/full
			 * join must still emit the row (keepNulls, nodeHashjoin.c:209), or LASJ_NOTIN gives up (:223,238) */
			inner_has_nullkey = 1;
			if (!fill_inner)
				continue;
		}
		if (tab.ntuples == tab.cap)
		{
			tab.cap *= 2;
			tab.arena = realloc(tab.arena, tab.cap * sizeof(hj_tuple));
		}
		tab.arena[tab.ntuples].hashvalue = h;
		tab.arena[tab.ntuples].tuple = tup;
		tab.arena[tab.ntuples].tid = tid;
		tab.arena[tab.ntuples].matched = 0;
		tab.arena[tab.ntuples].nullkey = !ok;
		tab.ntuples++;
	}
	if (hs->error) { rc = hs->error; goto done; }
	/* ExecChooseHashTableSize: nbuckets = pow2 >= ntuples / tuples_per_bucket, at least 1024
	 * (the reference sizes from the planner's estimate; the exact count is the ideal estimate) */
	nb = 1024;
	while ((uint64_t) nb * TUPLES_PER_BUCKET < tab.ntuples && nb < (1u << 30))
		nb <<= 1;
	tab.nbuckets = nb;
	tab.buckets = calloc(nb, sizeof *tab.buckets);
	{
		uint64_t i;

		for (i = 0; i < tab.ntuples; i++)	/* ExecHashTableInsert: push on the bucket's chain */
		{
			hj_tuple *t = &tab.arena[i];
			uint32_t b = t->hashvalue & (nb - 1);

			t->next = tab.buckets[b];
			tab.buckets[b] = t;
		}
	}

	if (lasj && inner_has_nullkey)
		goto done;						/* x NOT IN (..., NULL, ...) is never true */

	/* ---- HJ_NEED_NEW_OUTER / HJ_SCAN_BUCKET ---- */
	or_scan_begin(hs, &outer->desc, outer_pages, outer_nblocks);
	while ((tup = or_scan_next(hs, &tid)) != NULL)
	{
		uint32_t h;
		int ok, matched = 0;
		int keep_nulls = fill_outer;
		hj_tuple *t;

		or_row_store(&row, &outer->desc, tup);
		if (outer->qual >= 0)
		{
			or_datum q;

			if ((rc = or_eval(pool, outer->qual, &row, NULL, &q)) != 0)
				goto done;
			if (q.isnull || !q.v)
				continue;
		}
		if ((rc = hash_keys(pool, hj->outerkey, hj->nkeys, &row, 1, keep_nulls, &h, &ok)) != 0)
			goto done;
		if (!ok)
			continue;
		if (lasj && tab.ntuples > 0)
		{
			/* OPT-3325: a NULL outer key against a non-empty inner side is dropped (nodeHashjoin.c:356-368) */
			int k, anynull = 0;

			for (k = 0; k < hj->nkeys; k++)
			{
				or_datum d;

				if ((rc = or_eval(pool, hj->outerkey[k], &row, NULL, &d)) != 0)
					goto done;
				anynull |= d.isnull;
			}
			if (anynull)
				continue;
		}
		for (t = tab.buckets[h & (nb - 1)]; t; t = t->next)
		{
			int m;

			if (t->hashvalue != h || t->nullkey)
				continue;
			or_row_store(&irow, &inner->desc, t->tuple);
			if ((rc = keys_match(pool, hj, &row, &irow, &m)) != 0)
				goto done;
			if (!m)
				continue;
			if (hj->joinqual >= 0)
			{
				or_datum q;

				if ((rc = or_eval(pool, hj->joinqual, &row, &irow, &q)) != 0)
					goto done;
				if (q.isnull || !q.v)
					continue;
			}
			matched = 1;
			t->matched = 1;
			if (hj->jointype == GG_JOIN_ANTI || lasj)
				break;
			if ((rc = emit(ctx, &row, tid, &irow, t->tid)) != 0)
				goto done;
			if (hj->jointype == GG_JOIN_SEMI)
				break;
		}
		if (!matched && fill_outer)
			if ((rc = emit(ctx, &row, tid, NULL, (uint64_t) -1)) != 0)	/* HJ_FILL_OUTER_TUPLE */
				goto done;
	}
	if (hs->error)
	{
		rc = hs->error;
		goto done;
	}
	if (fill_inner)
	{
		/* HJ_FILL_INNER_TUPLES: ExecScanHashTableForUnmatched, nodeHashjoin.c:460-490 */
		uint64_t i;

		for (i = 0; i < tab.ntuples; i++)
		{
			hj_tuple *u = &tab.arena[i];

			if (u->matched)
				continue;
			or_row_store(&irow, &inner->desc, u->tuple);
			if ((rc = emit(ctx, NULL, (uint64_t) -1, &irow, u->tid)) != 0)
				goto done;
		}
	}
done:
	free(tab.arena);
	free(tab.buckets);
	free(hs);
	return rc;
}

typedef struct agg_ctx { or_aggtable *t; uint64_t n; } agg_ctx;

static int
emit_agg(void *p, or_row *outer, uint64_t otid, or_row *inner, uint64_t itid)
{
	agg_ctx *c = p;

	(void) otid; (void) itid;
	c->n++;
	return or_aggtable_advance(c->t, outer, inner);
}

int
or_hashjoin_agg(const gg_scan *outer, const gg_scan *inner, const gg_hashjoin *hj,
				const gg_agg *agg, const gg_exprpool *pool,
				const uint8_t *outer_pages, uint64_t outer_nblocks,
				const uint8_t *inner_pages, uint64_t inner_nblocks,
				gg_aggrow *out, int outcap, int *nout, uint64_t *rows_joined)
{
	agg_ctx c;
	int rc;

	c.t = or_aggtable_create(agg, pool, 0);
	c.n = 0;
	rc = run_join(outer, inner, hj, pool, outer_pages, outer_nblocks, inner_pages, inner_nblocks,
				  emit_agg, &c);
	if (rc == 0)
		rc = or_aggtable_emit(c.t, out, outcap, nout);
	if (rows_joined)
		*rows_joined = c.n;
	or_aggtable_free(c.t);
	return rc;
}

typedef struct tid_ctx { int64_t *out; uint64_t cap, n; } tid_ctx;

static int
emit_tid(void *p, or_row *outer, uint64_t otid, or_row *inner, uint64_t itid)
{
	tid_ctx *c = p;

	(void) outer; (void) inner;
	if (c->n >= c->cap)
		return OR_ERR_NOMEM;
	c->out[2 * c->n] = (int64_t) otid;
	c->out[2 * c->n + 1] = (int64_t) itid;
	c->n++;
	return 0;
}

int
or_hashjoin_tids(const gg_scan *outer, const gg_scan *inner, const gg_hashjoin *hj,
				 const gg_exprpool *pool,
				 const uint8_t *outer_pages, uint64_t outer_nblocks,
				 const uint8_t *inner_pages, uint64_t inner_nblocks,
				 int64_t *out_pairs, uint64_t cap, uint64_t *npairs)
{
	tid_ctx c;
	int rc;

	c.out = out_pairs;
	c.cap = cap;
	c.n = 0;
	rc = run_join(outer, inner, hj, pool, outer_pages, outer_nblocks, inner_pages, inner_nblocks,
				  emit_tid, &c);
	*npairs = c.n;
	return rc;
}
