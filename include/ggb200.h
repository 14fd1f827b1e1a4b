/*
 * ggb200.h — C-ABI of the GPU segment engine (libggb200.so).
 *
 * This is the drop-in boundary for the Greengage executor hot path: plain
 * pointers, sizes and the PODs of gg_plan.h; no torch, no C++ types.  The
 * per-node C functions of src/backend/executor/execProcnode.c (ExecInitNode
 * :255, ExecProcNode :925, ExecEndNode :1315) are mirrored by the host layer in
 * greengage_b200/host/gg_executor.c, which drives the device through exactly
 * these entry points.  INTEGRATION.md shows the binding a maintainer adds on
 * the Postgres side.
 *
 * Conventions (SURVEY §8b):
 *   - every call returns 0 or a negative GG_ERR_* code; gg_last_error() has the
 *     text.  The C wrapper on the Postgres side turns a non-zero return into
 *     ereport(ERROR, ...) (utils/elog.h:190); nothing here longjmps or throws.
 *   - handles own device memory; gg_*_free() is what a
 *     MemoryContextRegisterResetCallback / ResourceReleaseCallback calls
 *     (utils/palloc.h:190, resowner.c:551).
 *   - one engine per process and GPU (one QE process per segment and slice,
 *     src/backend/cdb/dispatcher/README.md:9-18); calls are made from one thread.
 *   - there is NO CPU fallback: if no CUDA device is usable, gg_engine_create fails.
 */
#ifndef GGB200_H
#define GGB200_H

#include <stdint.h>
#include "gg_plan.h"

#ifdef __cplusplus
extern "C" {
#endif

#define GG_OK                   0
#define GG_ERR_CUDA            (-1)    /* CUDA runtime error (text in gg_last_error) */
#define GG_ERR_FLOAT_OVERFLOW  (-2)    /* "value out of range: overflow", float_utils.h:28 */
#define GG_ERR_FLOAT_UNDERFLOW (-3)
#define GG_ERR_DIV_ZERO        (-4)
#define GG_ERR_INT_OVERFLOW    (-5)    /* "bigint out of range", int8.c:526,694 */
#define GG_ERR_UNSUPPORTED     (-6)    /* plan shape outside the accelerated subset: caller keeps the CPU node */
#define GG_ERR_VISIBILITY      (-7)    /* a tuple needs clog/snapshot to decide visibility (tqual.c:997) */
#define GG_ERR_NOMEM           (-8)
#define GG_ERR_BADPAGE         (-9)    /* page header fails the PageAddItem sanity rules (bufpage.c:196-204) */
#define GG_ERR_ARG             (-10)
#define GG_ERR_DATE_RANGE      (-11)   /* "date out of range for timestamp", date.c:471 */
#define GG_ERR_PEER            (-12)   /* another segment of the Motion reported an ERROR (the QD cancels the query) */
#define GG_ERR_RETRY_HOST      (-13)   /* not an error of the query: some segment could not keep its aggregate rows on the device
                                        * (every segment gets this at its fetch): run the slice again with host-row Motions */

typedef struct gg_engine   gg_engine;     /* one GPU segment: device, streams, scratch */
typedef struct gg_relation gg_relation;   /* heap pages resident in HBM (replaces bufmgr/smgr for the scan) */
typedef struct gg_scanagg  gg_scanagg;    /* compiled SeqScan -> qual -> Agg pipeline */
typedef struct gg_joinagg  gg_joinagg;    /* compiled SeqScan ⋈ Hash(SeqScan) -> Agg pipeline */

const char *gg_last_error(void);
const char *gg_strerror(int code);

/* ---- engine (one per segment process) ---- */
int  gg_engine_create(int device, gg_engine **out);
void gg_engine_free(gg_engine *e);
int  gg_engine_sm_count(gg_engine *e);

/* ---- snapshot ----
 * The SnapshotData (utils/snapshot.h:36-100) heap_beginscan receives (heapam.c:1573), as far as HeapTupleSatisfiesMVCC
 * (tqual.c:997-1238) reads it, plus the transaction status bits the rule asks pg_clog for.  With a snapshot set, a tuple whose
 * hint bits do not decide alone is judged on the device by the full rule; without one such a tuple raises GG_ERR_VISIBILITY
 * (the relation stays on the CPU scan).  Still the CPU scan's: multixact xmax, combo command ids, sub-committed status,
 * HEAP_MOVED_*, xids outside [clog_base, clog_base + clog_n), and the three snapshot kinds flagged below. */
/* every scan the engine launches after this call uses `snap` (copied); NULL: back to hint bits only */
int  gg_engine_set_snapshot(gg_engine *e, const gg_snapshot *snap);
int  gg_engine_sync(gg_engine *e);
/* CUDA-event timing of the last *_run call on the engine's stream, in milliseconds */
int  gg_engine_last_kernel_ms(gg_engine *e, float *ms);
/* number of kernels the engine has launched since creation (bench.py's gpu_launches) */
uint64_t gg_engine_launch_count(gg_engine *e);
/* CUDA events on the engine's compute stream bracketing any number of calls (bench.py's timed region) */
int  gg_engine_timer_start(gg_engine *e);
int  gg_engine_timer_stop(gg_engine *e, float *ms);
/* the engine's compute stream (cudaStream_t), for callers that order their own work against it */
void *gg_engine_stream(gg_engine *e);

/* ---- relations: heap pages in device memory ----
 * Replaces heap_beginscan/heapgetpage's ReadBufferExtended path
 * (src/backend/access/heap/heapam.c:312-463, storage/buffer/bufmgr.c:315): the
 * segment's pages live in HBM as one contiguous array of 32 KB blocks. */
int  gg_relation_create(gg_engine *e, uint64_t nblocks, gg_relation **out);
/* wrap device memory owned by the caller (e.g. a torch tensor); not freed by gg_relation_free */
int  gg_relation_attach(gg_engine *e, void *device_pages, uint64_t nblocks, gg_relation **out);
/* wrap rows a receiving Motion delivered (GG_FMT_DATUMROWS, gg_plan.h): nrows rows of 1 + ncols 64-bit words.  Every
 * operator that scans heap pages also scans these, given a tuple descriptor with format = GG_FMT_DATUMROWS.  The
 * buffer must be 16-byte aligned and extend 16 bytes past the last row. */
int  gg_relation_attach_rows(gg_engine *e, void *device_rows, uint64_t nrows, int ncols, gg_relation **out);
/* host -> device copy of nblocks pages starting at first_block (async on the engine's copy stream
 * when host_pages is pinned; gg_engine_sync or the next *_run orders it) */
int  gg_relation_load(gg_relation *r, uint64_t first_block, const void *host_pages, uint64_t nblocks);
int  gg_relation_read(gg_relation *r, uint64_t first_block, void *host_pages, uint64_t nblocks);
/* device -> device copy of nblocks pages between two relations of one engine (async on the engine's stream): a partition
 * attached to its parent, a relation extended by pages another scan produced */
int  gg_relation_copy(gg_relation *dst, uint64_t dst_first, gg_relation *src, uint64_t src_first, uint64_t nblocks);
uint64_t gg_relation_nblocks(gg_relation *r);
/* upper bound on the tuples of the relation: its line pointers (one pass over the page headers), or the row count of datum rows */
int  gg_relation_count_rows(gg_relation *r, uint64_t *nrows);
void *gg_relation_device_ptr(gg_relation *r);
void gg_relation_free(gg_relation *r);

/* pinned host staging (cudaHostAlloc), for callers without their own pinned buffers */
int  gg_host_alloc(uint64_t bytes, void **out);
void gg_host_free(void *p);

/* ---- SeqScan -> qual -> Agg ----
 * Replaces ExecAgg(AGG_HASHED|AGG_PLAIN) over ExecSeqScan
 * (nodeAgg.c:1123, execHHashagg.c:905, nodeSeqscan.c:128, execScan.c:111).
 * Output rows follow gg_aggrow (group keys + aggregate values; PARTIAL stage
 * emits transition states).  Row order is unspecified, as for a hash aggregate. */
int  gg_scanagg_create(gg_engine *e, const gg_scan *scan, const gg_agg *agg, const gg_exprpool *pool,
                       gg_scanagg **out);
/* run over blocks [first_block, first_block+nblocks) of a resident relation; accumulates into the
 * pipeline's state, so several ranges (or relations) can be fed before fetching */
int  gg_scanagg_run(gg_scanagg *p, gg_relation *r, uint64_t first_block, uint64_t nblocks);
/* streamed variant: pages come from HOST memory (pinned or pageable); H2D copies are chunked and
 * overlapped with the kernel on two streams.  This is the end-to-end path bench.py's `e2e` times. */
int  gg_scanagg_run_host(gg_scanagg *p, const void *host_pages, uint64_t nblocks);
int  gg_scanagg_fetch(gg_scanagg *p, gg_aggrow *out, int outcap, int *nout,
                      uint64_t *rows_scanned, uint64_t *rows_passed);
int  gg_scanagg_reset(gg_scanagg *p);
void gg_scanagg_free(gg_scanagg *p);
/* introspection for benchmarks: summed CUDA-event duration of the scan kernel launches since the last reset and
 * their count; and which kernel variant runs (0 private accumulators, 1 transposed, 2 transposed+NULLs;
 * +16 plan-specialised at build time, +32 plan-specialised at run time) */
int  gg_scanagg_scan_kernel_ms(gg_scanagg *p, float *ms, int *launches);
int  gg_scanagg_variant(gg_scanagg *p);

/* FINAL-stage Agg over partial rows gathered from the segments (combine functions,
 * nodeAgg.c:2123-2148).  agg->grpCol[i] carries the key type OIDs. */
int  gg_agg_final(gg_engine *e, const gg_agg *agg, const gg_aggrow *in, int nin,
                  gg_aggrow *out, int outcap, int *nout);

/* ---- HashJoin (+ Agg on top) ----
 * Replaces MultiExecHash + ExecHashJoin (nodeHash.c:88, nodeHashjoin.c:512):
 * build from the inner relation, probe with the outer relation, feed matches
 * to the aggregate without materialising the join. */
int  gg_joinagg_create(gg_engine *e, const gg_scan *outer, const gg_scan *inner, const gg_hashjoin *hj,
                       const gg_agg *agg, const gg_exprpool *pool, gg_joinagg **out);
int  gg_joinagg_build(gg_joinagg *p, gg_relation *inner, uint64_t first_block, uint64_t nblocks);
int  gg_joinagg_probe(gg_joinagg *p, gg_relation *outer, uint64_t first_block, uint64_t nblocks);
int  gg_joinagg_probe_host(gg_joinagg *p, const void *host_pages, uint64_t nblocks);   /* outer pages in host memory, streamed */
/* Hybrid hash join (nodeHash.c:713 ExecHashIncreaseNumBatches, :1132 ExecHashGetBucketAndBatch; nodeHashjoin.c:906,1083):
 * `bytes` is the operator's memory (PlanStateOperatorMemKB, execnodes.h:1446) the hash table has to fit; 0 = no limit.
 * gg_joinagg_run builds and probes whole relations; when the table of the whole inner side would be larger than that, both
 * sides are split into nbatch = 2^k partitions by the batch bits of the reference's hash value (the partitions are datum rows
 * in device memory, not files) and the batches are joined one after the other into the same aggregate. */
int  gg_joinagg_set_work_mem(gg_joinagg *p, uint64_t bytes);
int  gg_joinagg_run(gg_joinagg *p, gg_relation *inner, gg_relation *outer);
int  gg_joinagg_nbatch(gg_joinagg *p);            /* batches of the last gg_joinagg_run (1: one hash table held everything) */
int  gg_joinagg_fetch(gg_joinagg *p, gg_aggrow *out, int outcap, int *nout, uint64_t *rows_joined);
int  gg_joinagg_reset(gg_joinagg *p);      /* ExecReScanHashJoin with the hash table kept (nodeHashjoin.c:1015-1050) */
int  gg_joinagg_stats(gg_joinagg *p, uint64_t *rows_built, uint64_t *table_bytes, float *build_ms, float *probe_ms);
int  gg_joinagg_variant(gg_joinagg *p);       /* kernel variant of the probe side, as gg_scanagg_variant */
void gg_joinagg_free(gg_joinagg *p);
/* HashJoin with a target list (ExecHashJoin -> ExecProject, nodeHashjoin.c:78-509): the same pipeline — build, table sizing,
 * batches, the fill-inner pass of right / full joins, reset, stats, set_work_mem and free are gg_joinagg_*'s — whose probe
 * writes every joined row as a datum row instead of feeding an aggregate.  targets: 1..16 expression roots in the pool, Vars
 * with varno 0 = outer, 1 = inner (outer only for SEMI / ANTI / LASJ_NOTIN); numeric targets are refused (GG_ERR_UNSUPPORTED).
 * The output is sized from the outer rows (+ the inner rows of a right / full join); a join that produces more is probed
 * once more against the kept table, into a buffer as large as the first probe found it needs. */
int  gg_joinrows_create(gg_engine *e, const gg_scan *outer, const gg_scan *inner, const gg_hashjoin *hj,
                        const int32_t *targets, int ntargets, const gg_exprpool *pool, gg_joinagg **out);
/* after gg_joinagg_run (or build + probe): the joined rows, GG_FMT_DATUMROWS of ntargets columns with the NULL mask of the
 * null-extended side set; *nrows slots of which some may be dead (GG_DATUMROW_DEAD); *nlive = rows joined.  The relation is
 * a view owned by the join, valid until gg_joinagg_reset / gg_joinagg_free; building, probing or running again needs a reset
 * first. */
int  gg_joinagg_rows(gg_joinagg *p, gg_relation **rows, uint64_t *nrows, uint64_t *nlive);

/* ---- Append-only column-oriented (AOCS) relations ----
 * Decode the projected columns of a segment file, resident in device memory together with the loader's block directories
 * and tile plans (include/gg_aocs.h), into GG_FMT_DATUMROWS rows: device_rows receives nrows rows of 1 + ncols 64-bit
 * words (NULL mask, then the columns in the order given) and is then scanned like any relation through
 * gg_relation_attach_rows.  What aocs_getnext does per row (src/backend/access/aocs/aocsam.c:700-800).  The pointers inside
 * cols[] are DEVICE pointers; cols itself is host memory.  device_rows: 16-byte aligned, 16 bytes of slack after the last
 * row.  GG_ERR_UNSUPPORTED: a projected column whose values have no common stride (strings longer than 8 bytes or of
 * mixed length); GG_ERR_BADPAGE: plan and directory disagree. */
struct gg_aocs_devcol;
/* The fused scan: SeqScan over the column files -> qual -> Agg in ONE kernel (aocs_getnext, aocsam.c:661, feeding the same
 * row program as heap pages): the kernel's producer warp walks the columns' block directories and bulk-copies each unit of
 * ~500 rows of every referenced column into shared memory, consumer lanes assemble their rows from there (a column whose
 * blocks carry NULL bitmaps or values of unequal size is read row by row from device memory instead); nothing is written
 * back to device memory, only the projected columns' bytes are read.  The pipeline must have been created over the
 * GG_FMT_DATUMROWS descriptor of the ncols projected columns (column i of the descriptor = cols[i]); tile_rows = the tile
 * size the tile plans were made for (a multiple of 32).  Accumulates like gg_scanagg_run; fetch as usual. */
int  gg_scanagg_run_aocs(gg_scanagg *p, const struct gg_aocs_devcol *cols, int ncols, uint64_t nrows, int32_t tile_rows);
/* the two-pass form: decode to rows any operator scans (joins, Motions) */
int  gg_aocs_decode_rows(gg_engine *e, const struct gg_aocs_devcol *cols, int ncols, uint64_t nrows, int32_t tile_rows,
                         void *device_rows);

/* ---- Sort ----
 * Replaces tuplesort_begin_heap_mk/puttupleslot/performsort/gettupleslot
 * (tuplesort_mk.c:771,1154,1378,1668) for fixed-width rows: rows is n x ncols
 * int64 Datum columns in device or host memory; perm receives the sorted order. */
int  gg_sort_rows(gg_engine *e, const gg_sortkey *keys, int nkeys, int ncols,
                  const int64_t *host_rows, const uint8_t *host_nulls, uint64_t n, uint64_t *host_perm);
/* the same sort over rows already resident on the device; dev_perm receives n uint32 row numbers,
 * passes (optional) the number of radix passes executed */
int  gg_sort_device(gg_engine *e, const gg_sortkey *keys, int nkeys, int ncols, const int64_t *dev_rows,
                    const uint8_t *dev_nulls, uint64_t n, uint32_t *dev_perm, int *passes);
/* Sort over what a row-producing SeqScan or a receiving Motion left on the device (nodeSort.c:48-256 with its input and its
 * result in device memory): dev_rows holds n GG_FMT_DATUMROWS rows of ncols columns (1 + ncols words each, NULLs in the mask
 * word; slots marked GG_DATUMROW_DEAD are dropped); dev_out_rows receives the *nlive rows in sorted order, same format.
 * keys[].col counts the row's columns from 0. */
int  gg_sort_datumrows(gg_engine *e, const gg_sortkey *keys, int nkeys, int ncols, const void *dev_rows, uint64_t n,
                       void *dev_out_rows, uint64_t *nlive, int *passes);
/* Bounded Sort (tuplesort_set_bound, tuplesort_mk.c:1000; a Limit above wants only the first `bound` rows): the first
 * min(bound, live) rows of what gg_sort_datumrows returns for the same input, byte for byte, in dev_out_rows; *nout = that
 * count.  A radix select on the first key keeps the rows that can be among them, in input order, and only those are sorted
 * (DESIGN §4.4).  bound == 0 launches nothing.  passes: histogram passes of the selection plus radix passes of the sort. */
int  gg_sort_datumrows_bounded(gg_engine *e, const gg_sortkey *keys, int nkeys, int ncols, const void *dev_rows, uint64_t n,
                               uint64_t bound, void *dev_out_rows, uint64_t *nout, int *passes);
/* the same for host rows: host_perm receives the first min(bound, n) entries of gg_sort_rows's permutation; *nperm = count */
int  gg_sort_rows_bounded(gg_engine *e, const gg_sortkey *keys, int nkeys, int ncols, const int64_t *host_rows,
                          const uint8_t *host_nulls, uint64_t n, uint64_t bound, uint64_t *host_perm, uint64_t *nperm);

/* ---- Motion ----
 * Sending side of a Redistribute Motion (nodeMotion.c:1481-1687, cdbhash.c:173-287) on the device: evaluates the
 * scan qual, the hash-key expressions and the expressions that travel for every tuple, computes the destination
 * segment bit-exactly (cdbhash + jump consistent hash), and writes GG_FMT_DATUMROWS rows of 1 + npayload words into
 * the destination's region of device_out_rows: region d = rows [d * cap, d * cap + host_counts[d]) with
 * cap = (out_cap_rows / nsegs) rounded down to even; host_offsets[d] = d * cap.  On large inputs the warps claim rows of a
 * region in windows; the few rows a warp claimed and did not fill are marked dead (bit 63 of the row's mask word) and are
 * skipped by every consumer, so host_counts[d] is the length of the region's run of rows, dead ones included: size
 * out_cap_rows with 1/8 of slack per region.  GG_ERR_NOMEM if a region overflows
 * (gg_last_error says how many rows the fullest destination receives).  The exchange itself is an all-to-all of the
 * regions over NCCL (greengage_b200/motion.py); the receiver wraps what it got with gg_relation_attach_rows. */
int  gg_motion_partition(gg_engine *e, const gg_scan *scan, const gg_exprpool *pool,
                         const int32_t *hashkeys, int nkeys, const int32_t *payload, int npayload,
                         int nsegs, gg_relation *r, uint64_t first_block, uint64_t nblocks,
                         void *device_out_rows, uint64_t out_cap_rows,
                         uint64_t *host_counts, uint64_t *host_offsets);

/* ---- device-resident aggregate rows ----
 * The rows an Agg pipeline produced, left on the device as group records so that the nodes above it in the slice
 * (Motion, FINAL Agg) consume them there; only the top of the slice fetches (SURVEY §8a rows 8, 15).  A gg_groups
 * obtained from a pipeline is a view: valid until that pipeline is reset or freed. */
typedef struct gg_groups gg_groups;
int  gg_scanagg_groups(gg_scanagg *p, gg_groups **out);      /* GG_ERR_UNSUPPORTED for the general HashAggregate: fetch rows */
int  gg_joinagg_groups(gg_joinagg *p, gg_groups **out);
/* FINAL-stage Agg over records a Motion delivered: the combine functions (nodeAgg.c:2123-2148) on the device */
int  gg_groups_final(gg_engine *e, gg_groups *in, gg_groups **out);
/* records + status -> rows: the one host synchronisation of a device-resident slice.  Rows read as the producing Agg's
 * stage says (PARTIAL: transition states; otherwise finalised values). */
int  gg_groups_fetch(gg_groups *g, gg_aggrow *out, int outcap, int *nout, uint64_t *rows_scanned, uint64_t *rows_passed);
int  gg_groups_info(gg_groups *g, int *sparse, int *cap);
/* ---- aggregate rows as datum rows ----
 * The groups of an Agg finalised on the device (finalize_aggregate, nodeAgg.c:871-999) into GG_FMT_DATUMROWS rows that a Sort
 * or a Limit above takes where they are (gg_sort_datumrows*): word 0 the NULL mask (bit c: grouping column c, bit numCols + i:
 * aggregate i), then the numCols grouping keys, then one word per aggregate — bit for bit what the *_fetch calls put into a
 * gg_aggrow's key[c] and agg[i].f[0] (float8 results) or agg[i].i.  No slot is dead.  Order: that of *_fetch for the merged
 * records of a block-table variant and for a group set; for the general HashAggregate a function of its table's contents
 * (unspecified, as for a hash aggregate).  A plain aggregate over no input still gives its one row (not on a segment that does
 * not receive a Gather).  The pipeline is settled first exactly as *_fetch settles it (kernel-variant escalation and replay,
 * the join's build error, the fill-inner pass of right / full joins), with fetch's error codes and messages.
 * *rows is a view owned by the pipeline or the set, valid until its reset or free; the buffer is 16-byte aligned with 16 bytes
 * of slack and grows as needed.  GG_ERR_UNSUPPORTED: a PARTIAL stage (its consumers read group records) or a numeric
 * aggregate (finalised on the host only). */
int  gg_scanagg_datumrows(gg_scanagg *p, gg_relation **rows, uint64_t *nrows);
int  gg_joinagg_datumrows(gg_joinagg *j, gg_relation **rows, uint64_t *nrows);
int  gg_groups_datumrows(gg_groups *g, gg_relation **rows, uint64_t *nrows);
/* ---- row filter: an Agg's HAVING over its datum rows ----
 * ExecQual of the Agg's plan.qual over every finalised group (nodeAgg.c:1092): a row passes only if the qual is TRUE (NULL
 * does not pass); AND / OR skip the arm the reference skips, so it raises nothing.  rows_desc is the GG_FMT_DATUMROWS descriptor
 * of the rows (for an Agg: its grouping keys, then one column per aggregate, typed as the Agg outputs them); qual is an
 * expression root in the pool whose Vars are varno 0, varattno = 1-based column of the rows.  create compiles the qual:
 * GG_ERR_UNSUPPORTED with a message for a function or a type the device does not evaluate (numeric columns have no datum
 * row), GG_ERR_ARG for a root outside the pool or a Var outside the columns.
 * run filters the first nrows rows of a datum-row relation of that many columns: *out_view receives the rows whose qual is
 * TRUE, in input order and in the same format, dead slots (GG_DATUMROW_DEAD) dropped; *nout their number.  The view is owned
 * by the filter, valid until its next run or free.  nrows == 0 launches nothing.  Errors of the qual (float8 overflow,
 * division by zero, date out of range, ...) are the reference's codes. */
typedef struct gg_rowfilter gg_rowfilter;
int  gg_rowfilter_create(gg_engine *e, const gg_tupdesc *rows_desc, int32_t qual, const gg_exprpool *pool, gg_rowfilter **out);
int  gg_rowfilter_run(gg_rowfilter *f, gg_relation *rows, uint64_t nrows, gg_relation **out_view, uint64_t *nout);
void gg_rowfilter_free(gg_rowfilter *f);
void gg_groups_set_nonreceiver(gg_groups *g);
void gg_groups_free(gg_groups *g);

/* ---- WindowAgg over datum rows (nodeWindowAgg.c, utils/adt/windowfuncs.c) ----
 * rows_desc is the GG_FMT_DATUMROWS descriptor of the input rows, which arrive sorted so that partitions (equal partition
 * columns) and peer groups (equal order columns within a partition) are runs: the planner's Sort below a WindowAgg.  Equality is
 * execTuplesMatch's: two NULLs match, float8 -0 = +0 and NaN = NaN, packed strings compare by bits.  win describes the node
 * (gg_plan.h gg_window); each function's arguments are Vars of the input row (varno 0, 1-based varattno) or Consts.
 * create checks the plan: GG_ERR_UNSUPPORTED with a message for a frame with value offsets, a numeric or unknown function, an
 * argument that is neither a Var nor a Const, a non-Const ntile / nth_value argument, or more than GG_MAX_ATTS output columns;
 * GG_ERR_ARG for a column or a root out of range.
 * run windows the first nrows slots of a datum-row relation of rows_desc's columns: *out_view receives one row per live input
 * row, in input order, of the input's columns followed by one column per function (word 0: the NULL mask over all of them);
 * dead slots (GG_DATUMROW_DEAD) get no number and no output row.  The view is owned by the window object, valid until its next
 * run or free.  nrows == 0 launches nothing.  Errors: GG_ERR_WINDOW_ARG for ntile / nth_value of a Const <= 0 over at least one
 * row (the reference's message), GG_ERR_FLOAT_OVERFLOW for a float8 sum / avg that becomes infinite with no infinite input. */
typedef struct gg_window_obj gg_window_obj;
#define GG_ERR_WINDOW_ARG      (-14)   /* "argument of ntile / nth_value must be greater than zero", SQLSTATE 22014 / 22016 */
int  gg_window_create(gg_engine *e, const gg_tupdesc *rows_desc, const gg_window *win, const gg_exprpool *pool, gg_window_obj **out);
int  gg_window_run(gg_window_obj *w, gg_relation *rows, uint64_t nrows, gg_relation **out_view, uint64_t *nout);
void gg_window_free(gg_window_obj *w);

/* ---- Interconnect: the Motion layer over NCCL ----
 * Replaces SetupInterconnect / TeardownInterconnect and the ChunkTransportState vtable of the UDP interconnect
 * (cdb/cdbinterconnect.h:500-533, cdb/motion/ic_common.c:522,560, cdbmotion.c:434,559) for GPU segments: one NCCL
 * communicator per query, rank = contentid, whole device-resident batches instead of tuple chunks.  The unique id is
 * what the dispatcher would ship in the slice table next to the listener addresses (cdbgang.h:121-137). */
typedef struct gg_interconnect gg_interconnect;
#define GG_IC_UNIQUE_ID_BYTES 128
#define GG_IC_MOTION_GATHER    0          /* = GgMotionType */
#define GG_IC_MOTION_HASH      1
#define GG_IC_MOTION_BROADCAST 2
int  gg_ic_available(void);                                   /* libnccl could be loaded */
int  gg_ic_unique_id(void *out, int len);                     /* on one segment (the QD's choice); len >= GG_IC_UNIQUE_ID_BYTES */
int  gg_ic_create(gg_engine *e, const void *unique_id, int nsegs, int segindex, gg_interconnect **out);   /* nsegs == 1: loopback, no NCCL */
void gg_ic_teardown(gg_interconnect *ic, int has_errors);     /* has_errors: ncclCommAbort instead of waiting for peers */
void gg_ic_free(gg_interconnect *ic);
int  gg_ic_nsegs(gg_interconnect *ic);
int  gg_ic_segindex(gg_interconnect *ic);
uint64_t gg_ic_collective_count(gg_interconnect *ic);
/* every segment contributes one word and learns everybody's (also a barrier on the engine's stream) */
int  gg_ic_allgather_u64(gg_interconnect *ic, uint64_t mine, uint64_t *all);
/* Motion of aggregate rows, device to device.  hashcol[] index the grouping columns of the rows, hashtypid[] their type
 * OIDs; routing is cdbhash + jump consistent hash, bit-exact with cdbhash.c:191-287.  The status (ERROR flags) of every
 * sender reaches every receiver with the data. */
int  gg_ic_motion_groups(gg_interconnect *ic, int motion_type, int root, int nhash, const int32_t *hashcol,
                         const int32_t *hashtypid, gg_groups *in, int local_error, gg_groups **out);
/* `in` == NULL: this segment has no device-resident records to send — its slice failed (local_error = the GG_ERR_* code) or
 * its aggregate keeps its groups elsewhere (local_error = GG_OK).  It still takes part, with an empty block whose status says
 * so; the flags travel with the data and every segment meets them at its fetch (an ERROR, or GG_ERR_RETRY_HOST).  A segment
 * never leaves its peers alone in a collective. */
/* Redistribute of datum rows: the all-to-all-v behind gg_motion_partition (send_rows = its regions, counts = its host_counts,
 * region_cap = out_cap_rows / nsegs rounded down to even).  recv_rows: device buffer of recv_cap rows (16-byte aligned,
 * 16 bytes of slack for gg_relation_attach_rows).  GG_ERR_NOMEM (on every segment) if any receive buffer is too small. */
int  gg_ic_exchange_rows(gg_interconnect *ic, const void *send_rows, const uint64_t *counts, uint64_t region_cap, int rowwords,
                         void *recv_rows, uint64_t recv_cap, uint64_t *nrecv);
/* Motion of host rows (the executor's generic path): dest[i] = receiving segment, -1 = all.  out_* are malloc'd.
 * my_error != 0: this segment's slice failed — it takes part with no rows and EVERY segment returns GG_ERR_PEER. */
int  gg_ic_exchange_host(gg_interconnect *ic, int ncols, int64_t nrows, const int64_t *values, const uint8_t *isnull,
                         const int32_t *dest, int my_error, int64_t *out_nrows, int64_t **out_values, uint8_t **out_isnull);

#ifdef __cplusplus
}
#endif
#endif /* GGB200_H */
