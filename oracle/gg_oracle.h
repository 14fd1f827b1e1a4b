/*
 * gg_oracle.h — CPU restatement of the Greengage executor hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing in the product (greengage_b200/, include/
 * ggb200.h) may link, import or call this library; only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
 * use it, as the checker and as the timed CPU arm.
 *
 * Every function restates one piece of the reference and cites it
 * (paths relative to /root/reference).  The restatement is pinned against the
 * reference itself: oracle/ref_build compiles the reference's own leaf objects
 * (hashfunc.c, heaptuple.c, cdbhash.c, float.c, int8.c, varchar.c, date.c)
 * into oracle/_ref/libggref.so, tests/golden/make_golden.py records their
 * outputs as committed golden vectors, and tests/test_oracle_*.py check this
 * library against those vectors (and against libggref.so directly when it is
 * present).  Node-level control flow (ExecAgg/ExecHashJoin/ExecSort/ExecMotion)
 * cannot be linked without the whole backend and is restated here, pinned by
 * the reference's own Q1 golden result (src/test/regress/output/rpt_tpch.source:309-315).
 */
#ifndef GG_ORACLE_H
#define GG_ORACLE_H

#include <stdint.h>
#include <stddef.h>
#include "../include/gg_plan.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---------------- hashing (access/hash/hashfunc.c, utils/adt/varchar.c, cdb/cdbhash.c) ------------- */
uint32_t or_hash_any(const unsigned char *k, int keylen);     /* hashfunc.c:302 */
uint32_t or_hash_uint32(uint32_t k);                          /* hashfunc.c:527 */
uint32_t or_hashint4(int32_t v);                              /* hashfunc.c:46 */
uint32_t or_hashint8(int64_t v);                              /* hashfunc.c:52 */
uint32_t or_hashfloat8(double v);                             /* hashfunc.c:110 */
uint32_t or_hashbpchar(const char *s, int len);               /* varchar.c:906 (+bcTruelen :653) */
int      or_bctruelen(const char *s, int len);                /* varchar.c:653 */
int      or_bpchareq(const char *a, int la, const char *b, int lb);   /* varchar.c:702 */
int      or_bpcharcmp(const char *a, int la, const char *b, int lb);  /* varchar.c:840, C locale */
uint32_t or_hash_datum(int32_t typid, int64_t datum, int32_t len);    /* per-type hash proc dispatch */

uint32_t or_cdbhash_init(void);                               /* cdbhash.c:173 */
uint32_t or_cdbhash_add(uint32_t h, uint32_t hkey, int isnull);      /* cdbhash.c:191-219 */
int32_t  or_jump_consistent_hash(uint64_t key, int32_t nsegs);       /* cdbhash.c:549-560 */
int32_t  or_cdbhash_reduce(uint32_t h, int32_t nsegs);               /* cdbhash.c:255-287 */

/* ---------------- heap tuples and pages (heaptuple.c, bufpage.c) ---------------- */
/* A row handed to the tuple former: by-value attrs carry Datum bits in val[];
 * varlena attrs carry a pointer to the PAYLOAD bytes (no header) in val[] and
 * the payload length in len[]. */
int  or_heap_compute_data_size(const gg_tupdesc *desc, const int64_t *val, const int32_t *len,
                               const uint8_t *isnull);                        /* heaptuple.c:68-129 */
int  or_heap_form_tuple(const gg_tupdesc *desc, const int64_t *val, const int32_t *len,
                        const uint8_t *isnull, uint8_t *out, int outcap);     /* heaptuple.c:664-760 */
void or_page_init(uint8_t *page);                                              /* bufpage.c:41 */
int  or_page_add_item(uint8_t *page, const uint8_t *item, int size);          /* bufpage.c:176; 0 = no room */
int  or_page_nitems(const uint8_t *page);                                      /* PageGetMaxOffsetNumber */
void or_page_set_all_visible(uint8_t *page);

/* deform: values[] get Datum bits for by-value attrs, and for varlenas the
 * byte OFFSET of the datum (header byte) from the tuple start.  heaptuple.c:1119-1213 */
int  or_heap_deform(const gg_tupdesc *desc, const uint8_t *tuple, int natts_wanted,
                    int64_t *values, uint8_t *isnull);
/* varlena accessors on a datum inside a tuple (postgres.h:158-300): payload pointer and length */
const uint8_t *or_varlena_payload(const uint8_t *datum, int *len);
/* visibility: HeapTupleSatisfiesMVCC fast path (tqual.c:997-1140); 1 visible, 0 invisible, -1 needs clog */
int  or_tuple_visible(const uint8_t *tuple);
/* the full rule against a snapshot (tqual.c:997-1238); or_set_snapshot makes the scans that follow use it */
int  or_tuple_satisfies_mvcc(const uint8_t *tuple, const gg_snapshot *snap);
void or_set_snapshot(const gg_snapshot *snap);

/* ---------------- expression evaluation (execQual.c) ---------------- */
/* numeric values: the 128-bit integer (hi:v), scaled by 10^dscale (or_numeric.c) */
typedef struct or_datum { int64_t v; int32_t len; int32_t isnull; const uint8_t *ptr; int64_t hi; int32_t dscale; int32_t pad; } or_datum;
typedef struct or_row {       /* a deformed tuple: one side of a (possibly joined) row */
	const gg_tupdesc *desc;
	const uint8_t *tuple;
	int64_t values[GG_MAX_ATTS];
	uint8_t isnull[GG_MAX_ATTS];
	int nvalid;
} or_row;
/* returns 0 ok, <0 error code (float overflow etc.: OR_ERR_*) */
int or_eval(const gg_exprpool *pool, int root, or_row *outer, or_row *inner, or_datum *res);

/* numeric (or_numeric.c) */
int or_numeric_decode(const uint8_t *payload, int len, or_datum *res);
void or_numeric_const(int64_t unscaled, int dscale, or_datum *res);
int or_numeric_func(int funcid, const or_datum *a, const or_datum *b, or_datum *res);
int or_numeric_accum(int64_t *sum_lo, int64_t *sum_hi, int *sum_dscale, int64_t *n, const or_datum *x);
int or_numeric_avg(int64_t sum_lo, int64_t sum_hi, int sum_dscale, int64_t n, int64_t *out_lo, int64_t *out_hi, int *rscale);

#define OR_ERR_FLOAT_OVERFLOW   (-2)   /* "value out of range: overflow"  float_utils.h:28 */
#define OR_ERR_FLOAT_UNDERFLOW  (-3)
#define OR_ERR_DIV_ZERO         (-4)
#define OR_ERR_INT_OVERFLOW     (-5)   /* "bigint out of range" int8.c:526,694 */
#define OR_ERR_UNSUPPORTED      (-6)
#define OR_ERR_VISIBILITY       (-7)
#define OR_ERR_NOMEM            (-8)

/* ---------------- operators ---------------- */
/* SeqScan -> qual -> (hash) Agg over heap pages resident in host memory.
 * Restates execScan.c:111-214, heapam.c:312-463,767-1006, execHHashagg.c:157-188,456-585,905-1081,
 * nodeAgg.c:413-681,871-999.  rows_scanned/rows_passed are optional. */
int or_seqscan_agg(const gg_scan *scan, const gg_agg *agg, const gg_exprpool *pool,
                   const uint8_t *pages, uint64_t nblocks,
                   gg_aggrow *out, int outcap, int *nout,
                   uint64_t *rows_scanned, uint64_t *rows_passed);

/* FINAL-stage Agg over partial rows (the receiving side of Q1's Redistribute):
 * combine functions float8pl / float8_combine / int8pl (nodeAgg.c:2123-2148). */
int or_agg_final(const gg_agg *agg, const gg_aggrow *in, int nin,
                 gg_aggrow *out, int outcap, int *nout);

/* SeqScan(outer) ⋈ Hash(SeqScan(inner)) -> Agg.  nodeHash.c:88-176,906-1222; nodeHashjoin.c:78-509 */
int or_hashjoin_agg(const gg_scan *outer, const gg_scan *inner, const gg_hashjoin *hj,
                    const gg_agg *agg, const gg_exprpool *pool,
                    const uint8_t *outer_pages, uint64_t outer_nblocks,
                    const uint8_t *inner_pages, uint64_t inner_nblocks,
                    gg_aggrow *out, int outcap, int *nout, uint64_t *rows_joined);

/* Joined row ids (block<<16|offnum) for small cases: out_pairs[2*i] outer tid, [2*i+1] inner tid (or -1) */
int or_hashjoin_tids(const gg_scan *outer, const gg_scan *inner, const gg_hashjoin *hj,
                     const gg_exprpool *pool,
                     const uint8_t *outer_pages, uint64_t outer_nblocks,
                     const uint8_t *inner_pages, uint64_t inner_nblocks,
                     int64_t *out_pairs, uint64_t cap, uint64_t *npairs);

/* Sort: comparator semantics of tuplesort_mk.c:2816-2850 + float.c:964-988 + varchar.c:840.
 * rows: n rows of ncols int64 Datum columns (strings packed), nulls: n*ncols bytes.
 * perm_out receives the sorted permutation (ties in unspecified order, like mk_qsort). */
int or_sort_perm(const gg_sortkey *keys, int nkeys, int ncols, const int64_t *rows,
                 const uint8_t *nulls, uint64_t n, uint64_t *perm_out);
int or_sort_compare(const gg_sortkey *keys, int nkeys, int ncols,
                    const int64_t *a, const uint8_t *an, const int64_t *b, const uint8_t *bn);

/* Motion routing: destination segment of every visible tuple of a relation for a hash
 * Redistribute on the given key expressions (nodeMotion.c:1481-1687, cdbhash.c:191-287). */
int or_motion_route(const gg_scan *scan, const gg_exprpool *pool, const int32_t *hashkeys, int nkeys,
                    int nsegs, const uint8_t *pages, uint64_t nblocks,
                    int32_t *dest_out, uint64_t cap, uint64_t *nrows);

/* Segment for one row of Datum keys (used for routing partial-agg rows) */
int32_t or_route_datums(const int32_t *typids, const int64_t *vals, const int32_t *lens,
                        const int32_t *isnull, int nkeys, int nsegs);

/* ---------------- column-oriented append-only (AOCS) column files, compresstype=none (or_aocs.c) ----------------
 * SURVEY §8f rank 1.  Storage blocks: cdbappendonlystorage_int.h:18-150, cdbappendonlystorageformat.c:26-321,1202-1417;
 * block content: datumstreamblock.h:68-81, datumstreamblock.c:150-330,1486-1748,3644-3710. */
uint32_t or_aocs_crc32c(const uint8_t *p, int64_t n);         /* port/pg_crc32c_sb8.c, not inverted at the end */
/* values[]: by-value Datums, or (attlen -1) pointers to payload bytes of lens[] bytes.  Returns the file length, <0 OR_ERR_* */
int64_t or_aocs_write_column(const gg_attr *att, const int64_t *values, const int32_t *lens, const uint8_t *nulls,
                             int64_t nrows, int blocksize, int checksum, int64_t first_rownum, uint8_t *out, int64_t outcap);
/* values[]: by-value Datums zero-extended from attlen bytes, or (attlen -1) byte offsets of the stored varlena in `file`.
 * firstrows/rowcounts: one entry per storage block.  Returns the row count, <0 OR_ERR_* (bad checksum, unknown block kind) */
int64_t or_aocs_read_column(const gg_attr *att, const uint8_t *file, int64_t nbytes, int checksum,
                            int64_t *values, uint8_t *nulls, int64_t cap,
                            int64_t *firstrows, int32_t *rowcounts, int blockcap, int *nblocks);
/* SeqScan (aocs_getnext, aocsam.c:700-800) -> qual -> Agg; colfiles[i] NULL = column not projected */
int or_aocs_seqscan_agg(const gg_scan *scan, const gg_agg *agg, const gg_exprpool *pool,
                        const uint8_t *const *colfiles, const int64_t *colbytes, int checksum, int64_t nrows_hint,
                        gg_aggrow *out, int outcap, int *nout, uint64_t *rows_scanned, uint64_t *rows_passed);

/* count(*) plumbing of BASELINE config 0: per-segment partial int8inc, Gather, final int8pl */
int64_t or_count_star_2stage(const uint8_t *const *seg_pages, const uint64_t *seg_nblocks, int nsegs);

/* multi-threaded timed runs for the CPU baseline: one thread per segment, pages split by block ranges */
int or_seqscan_agg_mt(const gg_scan *scan, const gg_agg *partial, const gg_agg *final,
                      const gg_exprpool *pool, const uint8_t *pages, uint64_t nblocks, int nthreads,
                      gg_aggrow *out, int outcap, int *nout, double *seconds, uint64_t *rows_scanned);

const char *or_strerror(int code);

/* ---------------- exact mode (checker only; or_agg.c) ----------------
 * Off by default.  When on, every hash/plain Agg of a NORMAL or PARTIAL stage keeps, beside its normal state, the exact
 * record of the float8 inputs of each aggregate: the exact sum, sum of absolute values and sum of fl(x*x) as fixed-point
 * integers in units of 2^-1074 (the least subnormal), so any double adds exactly.  or_aggtable_emit writes one or_exact per
 * (emitted row, aggregate), in its row order; or_exact_fetch copies them out.  The limbs are 32-bit two's-complement
 * digits, least significant first, carries resolved at emit.  Single-threaded operators only: the record is global. */
#define OR_XLIMBS            68      /* 2^-1074 .. 2^1024, times up to 2^31 inputs, and a sign */
#define OR_XF_NAN            0x01
#define OR_XF_PINF           0x02
#define OR_XF_NINF           0x04
#define OR_XF_ALL_NEGZERO    0x08    /* n > 0 and every input was -0 */
#define OR_XF_POSZERO        0x10    /* some input was +0 */
#define OR_XF_NEGZERO        0x20    /* some input was -0 */
typedef struct or_exact {
	int64_t  n;                      /* non-NULL inputs */
	int32_t  flags;                  /* OR_XF_* */
	int32_t  lowbit;                 /* exponent of the lowest set bit over the finite nonzero inputs (INT32_MAX: none) */
	int32_t  lowbit_sq;              /* the same over the finite nonzero fl(x*x) */
	int32_t  pad;
	int64_t  sum[OR_XLIMBS], abs[OR_XLIMBS], sq[OR_XLIMBS];
} or_exact;
void or_exact_mode(int on);
long or_exact_fetch(or_exact *out, long cap);     /* returns how many the last emit wrote */

#ifdef __cplusplus
}
#endif
#endif
