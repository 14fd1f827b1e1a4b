/*
 * gg_executor.h — the executor-node surface of the GPU segment engine (libggexec.so, host C).
 *
 * Mirrors what a Greengage QE runs for its slice of a plan (SURVEY §8b):
 *     ExecInitNode   src/backend/executor/execProcnode.c:255
 *     ExecProcNode   src/backend/executor/execProcnode.c:925   (one TupleTableSlot per call, NULL = end)
 *     ExecEndNode    src/backend/executor/execProcnode.c:1315
 *     ExecReScan     src/backend/executor/execAmi.c:76
 *     ExecSquelchNode src/backend/executor/execAmi.c:641
 * with the node types of the accelerated path (plannodes.h): SeqScan, Agg, Hash, HashJoin, Sort, Motion, Limit, WindowAgg.
 * Names keep the reference's, prefixed Gg.  The plan tree is what the Postgres-side translator of
 * INTEGRATION.md §2 builds from the real Plan tree; expressions live in one gg_exprpool.
 *
 * What ExecInitNode does differently from the reference: it FUSES the slice into device pipelines
 *     Agg <- SeqScan                         one scan+aggregate kernel      (gg_scanagg_*)
 *     Agg <- HashJoin(SeqScan, Hash(SeqScan)) build kernel + probe kernel   (gg_joinagg_*)
 *     HashJoin with a target list             build kernel + row-writing probe: datum rows (gg_joinrows_create)
 *     Sort <- any of the above                device radix sort             (gg_sort_rows)
 *     Sort / Limit <- Agg                      the groups finalised into device datum rows and sorted / windowed there
 *                                             (gg_scanagg_datumrows, gg_joinagg_datumrows, gg_groups_datumrows)
 *     Agg with HAVING (plan.qual)             its groups as device datum rows, filtered on the device (gg_rowfilter_run);
 *                                             refused (GG_ERR_UNSUPPORTED) where that cannot run, never run without its qual
 *     HashJoin <- Agg (either side)           the Agg's groups as device datum rows, scanned by the join like join rows
 *     WindowAgg <- Sort <- any row producer  the sorted rows windowed on the device (gg_window_run), its optional qual (a
 *                                             SubqueryScan's, e.g. rn <= 3) by gg_rowfilter_run; device datum rows for the
 *                                             caller, a Limit, a Sort, another WindowAgg, an Agg, a HashJoin or a Motion
 *     Motion <- any of the above              rows handed to the transport  (GgMotionTransport)
 * and returns NULL with GgExecLastError() set when a node or a shape is outside the accelerated subset, so the
 * caller keeps the CPU nodes for that subtree (there is no CPU implementation behind this API).
 */
#ifndef GG_EXECUTOR_H
#define GG_EXECUTOR_H

#include <stdint.h>
#include "ggb200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef enum GgNodeTag {            /* nodes/nodes.h NodeTag, the accelerated subset */
	T_GgSeqScan = 1,
	T_GgAgg,
	T_GgHash,
	T_GgHashJoin,
	T_GgSort,
	T_GgMotion,
	T_GgLimit,
	T_GgWindowAgg
} GgNodeTag;

typedef enum GgMotionType {         /* plannodes.h MotionType */
	GG_MOTIONTYPE_GATHER = 0,       /* all segments -> one receiver (MOTIONTYPE_FIXED with one target) */
	GG_MOTIONTYPE_HASH = 1,         /* Redistribute on hashExprs */
	GG_MOTIONTYPE_BROADCAST = 2
} GgMotionType;

/* Plan nodes (plannodes.h Plan and friends) */
typedef struct GgPlan {
	GgNodeTag type;
	struct GgPlan *lefttree;        /* outerPlan */
	struct GgPlan *righttree;       /* innerPlan */
	int32_t qual;                   /* implicit-AND qual folded into one expression root, -1 = none */
} GgPlan;

#define GG_MAX_SORTKEYS 4
#define GG_MAX_OUTCOLS (GG_MAX_KEYS + 3 * GG_MAX_AGGS)

typedef struct GgSeqScan {
	GgPlan plan;
	int32_t scanrelid;              /* index into GgEState.relations */
	gg_tupdesc desc;
	/* plan.targetlist (plannodes.h Plan): the expressions the scan projects (ExecProject, execScan.c:194), roots in the pool.
	 * 0 = the node above reads the relation's attributes directly (Agg <- SeqScan, HashJoin <- SeqScan: fused, nothing is
	 * projected).  > 0: the scan (or the Motion above it) produces rows of these columns — device-resident datum rows — and
	 * Vars of the nodes above refer to them by position. */
	int32_t numTargets;
	int32_t targets[GG_MAX_OUTCOLS];
} GgSeqScan;

typedef struct GgAgg {
	GgPlan plan;
	gg_agg agg;                     /* aggstrategy is implied: numCols == 0 plain, else hashed */
} GgAgg;

typedef struct GgHash {
	GgPlan plan;                    /* lefttree: the inner SeqScan */
} GgHash;

typedef struct GgHashJoin {
	GgPlan plan;                    /* lefttree: outer input; righttree: Hash over the inner input */
	gg_hashjoin hj;
	/* plan.targetlist: the expressions the join projects, roots in the pool, Vars with varno 0 = outer, 1 = inner (1..16).
	 * 0 = the Agg directly above reads the joined columns itself (fused, no row is written; refused anywhere else).  > 0: the
	 * join writes device-resident datum rows of these columns for the node above — another HashJoin, a Sort, a Limit, a
	 * Motion or the caller.  A join directly under an Agg stays fused whether it has targets or not. */
	int32_t numTargets;
	int32_t targets[GG_MAX_OUTCOLS];
} GgHashJoin;

typedef struct GgSort {
	GgPlan plan;
	int32_t numCols;
	gg_sortkey keys[GG_MAX_SORTKEYS];   /* col = 0-based output column of the child */
} GgSort;

typedef struct GgMotion {
	GgPlan plan;
	int32_t motionType;             /* GgMotionType */
	int32_t numHashCols;
	int32_t hashCol[GG_MAX_KEYS];   /* Redistribute: 0-based output columns of the child that are hashed */
	int32_t motionID;
	/* sendSorted (plannodes.h Motion.sendSorted + sort keys): every sender's stream is sorted on these keys and the
	 * receiver returns the merged order (execMotionSortedReceiver_mk, nodeMotion.c:636) — Q1's final
	 * "Gather Motion, Merge Key: l_returnflag, l_linestatus".  0 = arrival order. */
	int32_t numSortCols;
	gg_sortkey sortKeys[GG_MAX_SORTKEYS];
} GgMotion;

/* Limit (plannodes.h Limit): limitOffset / limitCount are the constants the translator evaluated the expressions to.
 * hasCount == 0: LIMIT ALL; hasOffset == 0: OFFSET 0.  Forward scans only.  The node's result is the window as host rows; a
 * Sort directly below it is told how many rows are wanted (pass_down_bound, nodeLimit.c:345) and sorts only those. */
typedef struct GgLimit {
	GgPlan plan;
	int32_t hasOffset, hasCount;
	int64_t limitOffset, limitCount;
} GgLimit;

/* WindowAgg (plannodes.h:1145): the child's rows, each followed by one column per window function (gg_plan.h gg_window).  The
 * child must deliver the window's order: a Sort whose leading keys are the partition columns, then the order columns (or a
 * WindowAgg over such a Sort); with neither partition nor order columns any row producer will do.  plan.qual (-1 = none) is a
 * qual over the output row, Vars varno 0 with 1-based varattno: what a translator folds in from a trivial SubqueryScan above.
 * Refused (GG_ERR_UNSUPPORTED) where the device cannot run it: value-offset frames, numeric aggregates, an argument that is
 * neither a Var nor a Const, more than GG_MAX_WINFUNCS functions or GG_MAX_ATTS output columns, an input in the wrong order, a
 * device library without gg_window_*. */
typedef struct GgWindowAgg {
	GgPlan plan;
	gg_window win;
} GgWindowAgg;

/* TupleTableSlot holding a virtual tuple (tuptable.h:117-175): Datums + null flags */
typedef struct GgTupleTableSlot {
	int32_t  tts_nvalid;
	int32_t  tts_isempty;
	int64_t  tts_values[GG_MAX_OUTCOLS];
	uint8_t  tts_isnull[GG_MAX_OUTCOLS];
	int32_t  tts_typid[GG_MAX_OUTCOLS];     /* Datum type per column (what the Motion / Sort above needs) */
	int32_t  tts_len[GG_MAX_OUTCOLS];       /* byte length for packed strings */
} GgTupleTableSlot;
#define GgTupIsNull(slot) ((slot) == NULL || (slot)->tts_isempty)

/* The interconnect behind a Motion node.  exchange() is called once by the sending half with every row this
 * segment produced, already routed (dest[i] = receiving segment); it returns the rows this segment receives.
 * greengage_b200/motion.py provides one over torch.distributed (NCCL / gloo); with nsegs == 1 the built-in
 * loopback is used. */
typedef struct GgRowBatch {
	int32_t ncols;
	int64_t nrows;
	int64_t *values;                /* [nrows][ncols] */
	uint8_t *isnull;                /* [nrows][ncols] */
} GgRowBatch;

typedef struct GgMotionTransport {
	void *ctx;
	/* 0 = ok.  `out` is filled with malloc'd arrays the executor frees. */
	int (*exchange)(void *ctx, int motionID, int motionType, const GgRowBatch *send, const int32_t *dest, GgRowBatch *out);
} GgMotionTransport;

#define GG_MAX_RELATIONS 16

/* EState (execnodes.h:360): per-query executor state */
typedef struct GgEState {
	gg_engine *engine;
	const gg_exprpool *pool;
	gg_relation *relations[GG_MAX_RELATIONS];   /* scanrelid -> heap pages resident on the device */
	int32_t nsegs, segindex;                    /* GpIdentity.numsegments / segindex */
	GgMotionTransport *transport;               /* host-row transport callback (tests over gloo); NULL: none */
	uint64_t es_processed;                      /* rows the top node has returned */
	/* the interconnect of this query (es_interconnect_is_setup / interconnect_context, execnodes.h:420): Motion nodes move
	 * device-resident batches through it (gg_ic_*, NCCL); with neither this nor `transport`, nsegs must be 1 */
	gg_interconnect *interconnect;
	/* a relation whose pages are in HOST memory (the segment's shared buffers): relations[i] == NULL and host_pages[i] set —
	 * the scan streams them to the device (gg_scanagg_run_host), H2D overlapped with the kernel */
	const void *host_pages[GG_MAX_RELATIONS];
	uint64_t host_nblocks[GG_MAX_RELATIONS];
	/* set by the executor when a slice had to be run again with its Motions moving host rows (some segment's aggregate did
	 * not fit the device-resident path); 0 at query start */
	int32_t motion_on_host;
	int32_t pad;
	/* the operator's share of statement_mem in bytes (PlanStateOperatorMemKB, execnodes.h:1446): a HashJoin whose table of
	 * the whole inner side would be larger runs as a hybrid hash join, in batches (gg_joinagg_run); 0 = no limit */
	uint64_t es_operator_mem;
	/* es_snapshot (execnodes.h:380): what heap_beginscan hands to HeapTupleSatisfiesMVCC.  NULL: the scans decide from hint
	 * bits alone and refuse a relation holding a tuple that needs more (GG_ERR_VISIBILITY).  ExecProcNode gives it to the
	 * engine before it runs the slice (gg_engine_set_snapshot). */
	const gg_snapshot *es_snapshot;
} GgEState;

typedef struct GgPlanState GgPlanState;        /* execnodes.h PlanState */

GgPlanState *GgExecInitNode(GgPlan *node, GgEState *estate, int eflags);
GgTupleTableSlot *GgExecProcNode(GgPlanState *node);
void *GgMultiExecProcNode(GgPlanState *node);     /* execProcnode.c:1217: only a Hash node answers (with NULL: the table lives in the join's pipeline) */
void GgExecEndNode(GgPlanState *node);
int  GgExecReScan(GgPlanState *node);
void GgExecSquelchNode(GgPlanState *node);
const char *GgExecLastError(void);
int  GgExecLastErrorCode(void);                /* GG_ERR_* of the failure, GG_OK if none */
/* introspection: which device pipeline a state node was fused into ("scanagg", "joinagg", "joinrows", "sort", "motion",
 * "limit", "windowagg", ...) */
const char *GgExecNodeKind(GgPlanState *node);
/* where a node that has run keeps its result: "device-groups" (aggregate rows as group records), "device-rows" (datum rows)
 * or "host" (Datum arrays); "" before it has run */
const char *GgExecNodeResultLocation(GgPlanState *node);
/* the state of a node's outer / inner child (outerPlanState / innerPlanState, execnodes.h:1441), NULL if fused away */
int GgExecPipelineKernelMs(GgPlanState *node, float *ms, int *launches, int *variant, float *build_ms);   /* benchmarks */
/* What EXPLAIN ANALYZE reads per node (Instrumentation, executor/instrument.h:38-66, filled by InstrStopNode; explain_gp.c turns
 * it into "Rows out", "Sort Method", "(slice...) ... batches"): counted by the node surface itself. */
typedef struct GgInstrumentation {
	double   ntuples;           /* tuples this node handed up through ExecProcNode, all executions */
	double   nloops;            /* executions: the first one plus every ExecReScan that ran the node again */
	float    kernel_ms;         /* GPU time of the node's own pipeline in its last execution (scan / probe kernels), 0 if it has none */
	int32_t  sort_runs;         /* Sort: runs the last execution merged (1 = in memory; GgExecSortRuns) */
	int32_t  hash_batches;      /* HashJoin pipeline: batches of the last execution (1 = one table; nodeHash.c:713), 0 otherwise */
	int32_t  pad;
} GgInstrumentation;
int GgExecNodeInstrumentation(GgPlanState *node, GgInstrumentation *out);

/* a Sort node over host rows: how many sorted runs its last execution merged (tuplesort's external path, taken when the rows
 * exceed GgEState.es_operator_mem: each run sorted on the device, the runs merged on the host); 1 = one in-memory sort */
int GgExecSortRuns(GgPlanState *node);
/* debugging / tests: the order that merge uses, for two rows of one [nrows][ncols] array */
int GgExecDebugSortCompare(const gg_sortkey *keys, int nkeys, int ncols, const int64_t *values, const uint8_t *isnull, uint64_t a, uint64_t b);
GgPlanState *GgExecOuterPlanState(GgPlanState *node);
GgPlanState *GgExecInnerPlanState(GgPlanState *node);

/* The per-node entry points of src/include/executor/node*.h (SURVEY §8b), for a build that replaces the node files
 * at link time instead of going through ExecProcNode's switch.  Each checks the node tag and delegates to the
 * functions above; the state they return is the state of the fused pipeline rooted at that node.
 *     nodeAgg.h:22-25,231   nodeSort.h:19-25   nodeMotion.h:20-27   nodeHashjoin.h:20-28   nodeSeqscan.h:19-24
 * A HashJoin or SeqScan without a target list is only accelerated underneath an Agg (its rows are never written), so
 * GgExecInitHashJoin / GgExecInitSeqScan on such a bare node return NULL with GG_ERR_UNSUPPORTED; with a target list they
 * produce device-resident rows.  The Hash node has no state of its own (MultiExecHash is the build kernel the join's
 * pipeline launches). */
GgPlanState *GgExecInitAgg(GgAgg *node, GgEState *estate, int eflags);
GgTupleTableSlot *GgExecAgg(GgPlanState *node);
void GgExecEndAgg(GgPlanState *node);
int  GgExecReScanAgg(GgPlanState *node);
void GgExecSquelchAgg(GgPlanState *node);
GgPlanState *GgExecInitSort(GgSort *node, GgEState *estate, int eflags);
GgTupleTableSlot *GgExecSort(GgPlanState *node);
void GgExecEndSort(GgPlanState *node);
int  GgExecReScanSort(GgPlanState *node);
void GgExecSquelchSort(GgPlanState *node);
GgPlanState *GgExecInitMotion(GgMotion *node, GgEState *estate, int eflags);
GgTupleTableSlot *GgExecMotion(GgPlanState *node);
void GgExecEndMotion(GgPlanState *node);
int  GgExecReScanMotion(GgPlanState *node);
void GgExecSquelchMotion(GgPlanState *node);
/* nodeLimit.h:19-23.  LIMIT / OFFSET must not be negative (GG_ERR_ARG, the reference's message); an empty window never runs
 * the child, and a window that ends squelches it (ExecLimit, nodeLimit.c:239-247) */
GgPlanState *GgExecInitLimit(GgLimit *node, GgEState *estate, int eflags);
GgTupleTableSlot *GgExecLimit(GgPlanState *node);
void GgExecEndLimit(GgPlanState *node);
int  GgExecReScanLimit(GgPlanState *node);
void GgExecSquelchLimit(GgPlanState *node);
/* nodeWindowAgg.h */
GgPlanState *GgExecInitWindowAgg(GgWindowAgg *node, GgEState *estate, int eflags);
GgTupleTableSlot *GgExecWindowAgg(GgPlanState *node);
void GgExecEndWindowAgg(GgPlanState *node);
int  GgExecReScanWindowAgg(GgPlanState *node);
void GgExecSquelchWindowAgg(GgPlanState *node);
void GgExecSortMarkPos(GgPlanState *node);      /* nodeSort.c:444 ExecSortMarkPos */
void GgExecSortRestrPos(GgPlanState *node);     /* nodeSort.c:462 ExecSortRestrPos */
GgPlanState *GgExecInitHashJoin(GgHashJoin *node, GgEState *estate, int eflags);
GgTupleTableSlot *GgExecHashJoin(GgPlanState *node);
void GgExecEndHashJoin(GgPlanState *node);
int  GgExecReScanHashJoin(GgPlanState *node);
void GgExecSquelchHashJoin(GgPlanState *node);
/* nodeSeqscan.h:19-24.  A SeqScan with a target list produces device-resident rows; returned as slots at the top of a slice */
GgPlanState *GgExecInitSeqScan(GgSeqScan *node, GgEState *estate, int eflags);
GgPlanState *GgExecInitSeqScanForPartition(GgSeqScan *node, GgEState *estate, int eflags, gg_relation *part);   /* nodeSeqscan.c:221 */
GgTupleTableSlot *GgExecSeqScan(GgPlanState *node);
void GgExecEndSeqScan(GgPlanState *node);
int  GgExecReScanSeqScan(GgPlanState *node);
/* nodeHash.h:23-27.  The Hash node has no pipeline of its own — MultiExecHash is the build kernel the join's pipeline
 * launches — so its state is a marker whose entry points say so the way the reference's do (ExecHash always ERRORs). */
GgPlanState *GgExecInitHash(GgHash *node, GgEState *estate, int eflags);
void *GgMultiExecHash(GgPlanState *node);
GgTupleTableSlot *GgExecHash(GgPlanState *node);
void GgExecEndHash(GgPlanState *node);
int  GgExecReScanHash(GgPlanState *node);

/* A CPU segment on the other side of a Motion (a CPU FINAL-stage Agg above this engine's PARTIAL stage, a mixed cluster).
 * GgExecSendTupleChunks: the rows `node` produces, as the reference's senders put them on the interconnect — SendTuple ->
 * SerializeTuple (cdbmotion.c:434, tupser.c:400): one MemTuple per row in tuple chunks of at most max_chunk bytes, then an
 * end-of-stream chunk (cdbmotion.c:532).  A PARTIAL-stage avg(float8) state travels as the float8[3] array the reference
 * ships (nodeAgg.c:975-979).  Returns the bytes written (< 0: GG_ERR_*).  The caller hands them to SendChunk.
 * GgExecRecvTupleChunks: the reverse for a Motion node's receiving half — what CPU senders produced (RecvTupleFrom ->
 * CvtChunksToTup, cdbmotion.c:559, tupser.c:609; MemTuple or heap-tuple form), up to and including the end-of-stream chunk,
 * becomes the node's result as if its exchange had delivered it. */
/* The other physical form of a slot (tuptable.h:117-175: a slot holds a virtual tuple, a MemTuple or a heap tuple; GPDB's
 * executor hands MemTuples to Sort, Hash spill files, Material and the Motion layer):
 * GgExecFetchSlotMemTuple = ExecFetchSlotMemTuple (execTuples.c:770): the slot's virtual tuple formed as a MemTuple under the
 * binding of its column types (create_memtuple_binding + memtuple_form_to, memtuple.c:420,551) — byte for byte what the
 * reference forms for the same Datums; returns its length, GG_ERR_NOMEM when cap is too small (*need then says how much).
 * GgExecStoreMemTuple = ExecStoreMemTuple + slot_getallattrs (execTuples.c:560, memtuple.c:917): a MemTuple of ncols columns
 * of the given types back into a virtual slot (strings come back packed: at most 8 bytes, else GG_ERR_UNSUPPORTED). */
int64_t GgExecFetchSlotMemTuple(const GgTupleTableSlot *slot, uint8_t *out, uint64_t cap, uint32_t *need);
int GgExecStoreMemTuple(GgTupleTableSlot *slot, const int32_t *typids, int ncols, const uint8_t *mt, uint32_t len);
int64_t GgExecSendTupleChunks(GgPlanState *node, int max_chunk, uint8_t *out, uint64_t cap, int64_t *nrows);
int GgExecRecvTupleChunks(GgPlanState *node, const uint8_t *chunks, uint64_t nbytes);

/* The interconnect as the reference selects it: a table of entry points per GpVars_Interconnect_Type
 * (cdbinterconnect.h:500-533, ic_common.c:522-575; UDPIFC / TCP / proxy there).  This is the NCCL entry: a 4th value of
 * that enum would install it. */
typedef struct GgInterconnectOps {
	int  (*SetupInterconnect)(GgEState *estate, const void *unique_id);       /* ic_common.c:522 */
	void (*TeardownInterconnect)(GgEState *estate, int hasErrors);            /* ic_common.c:560 */
	/* SendChunk + SendEos of a whole batch (cdbinterconnect.h:525,529): group records / datum rows / host rows */
	int  (*SendRecvGroups)(gg_interconnect *ic, int motionType, int root, int nhash, const int32_t *hashcol, const int32_t *hashtypid,
	                       gg_groups *in, int local_error, gg_groups **out);
	int  (*SendRecvRows)(gg_interconnect *ic, const void *send_rows, const uint64_t *counts, uint64_t region_cap, int rowwords,
	                     void *recv_rows, uint64_t recv_cap, uint64_t *nrecv);
	int  (*SendRecvHostRows)(gg_interconnect *ic, int ncols, int64_t nrows, const int64_t *values, const uint8_t *isnull,
	                         const int32_t *dest, int my_error, int64_t *out_nrows, int64_t **out_values, uint8_t **out_isnull);
} GgInterconnectOps;
extern const GgInterconnectOps GgInterconnectNCCL;

#ifdef __cplusplus
}
#endif
#endif /* GG_EXECUTOR_H */
