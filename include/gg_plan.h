/*
 * gg_plan.h — plain-C description of the slice of a Greengage plan that the
 * GPU executor accelerates.  These PODs are what crosses the C-ABI
 * (include/ggb200.h): no pointers, fixed-size arrays, so the same bytes can be
 * produced by the C host executor (greengage_b200/host), by ctypes, or by a
 * Postgres-side translator walking Plan/Expr trees.
 *
 * Everything here mirrors a reference structure; the citation says which:
 *   gg_attr / gg_tupdesc  <- Form_pg_attribute / TupleDesc
 *                            (src/include/catalog/pg_attribute.h, access/tupdesc.h)
 *   gg_expr               <- Var / Const / OpExpr / BoolExpr / NullTest
 *                            (src/include/nodes/primnodes.h), funcid = pg_proc OID
 *   gg_aggref             <- Aggref + pg_aggregate row (catalog/pg_aggregate.h:161-220)
 *   gg_scan / gg_agg / gg_hashjoin / gg_sort / gg_motion
 *                         <- SeqScan / Agg / HashJoin+Hash / Sort / Motion
 *                            (src/include/nodes/plannodes.h)
 * Type ids and function ids are the catalog OIDs, so a translator is a tree walk.
 */
#ifndef GG_PLAN_H
#define GG_PLAN_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- storage constants (configure.in:284-296, storage/bufpage.h:153-166) ---- */
#define GG_BLCKSZ            32768
#define GG_PAGE_HEADER_SIZE  24          /* SizeOfPageHeaderData */
#define GG_ITEMID_SIZE       4
#define GG_MAXALIGN(x)       (((uint64_t)(x) + 7) & ~(uint64_t)7)
#define GG_PD_ALL_VISIBLE    0x0004      /* bufpage.h:178 */
#define GG_PAGE_VERSION      14          /* PG_PAGE_LAYOUT_VERSION, bufpage.h:207 */
#define GG_LP_NORMAL         1           /* storage/itemid.h:34-40 */

/* heap tuple header (access/htup_details.h:139-196) */
#define GG_HEAP_HDR_SIZE       23        /* offsetof(HeapTupleHeaderData, t_bits) */
#define GG_HEAP_HASNULL        0x0001
#define GG_HEAP_HASVARWIDTH    0x0002
#define GG_HEAP_HASEXTERNAL    0x0004
#define GG_HEAP_XMIN_COMMITTED 0x0100
#define GG_HEAP_XMIN_INVALID   0x0200
#define GG_HEAP_XMIN_FROZEN    0x0300
#define GG_HEAP_XMAX_INVALID   0x0800
#define GG_HEAP_XMAX_COMMITTED 0x0400
#define GG_HEAP_XMAX_IS_MULTI  0x1000
#define GG_HEAP_XMAX_LOCK_ONLY 0x0080
#define GG_HEAP_XMAX_EXCL_LOCK 0x0040
#define GG_HEAP_XMAX_KEYSHR_LOCK 0x0010
#define GG_HEAP_COMBOCID       0x0020
#define GG_HEAP_MOVED          0xC000    /* HEAP_MOVED_OFF | HEAP_MOVED_IN: pre-9.0 VACUUM FULL leftovers */
#define GG_HEAP_NATTS_MASK     0x07FF
#define GG_FROZEN_XID          2         /* FrozenTransactionId, access/transam.h */

/* ---- the snapshot of a scan (utils/snapshot.h:36-100 as far as tqual.c:997-1238 reads it; see gg_engine_set_snapshot) ---- */
#define GG_SNAPSHOT_MAX_XIP 1024
typedef struct gg_snapshot {
	uint32_t xmin;                 /* all xids < xmin are finished */
	uint32_t xmax;                 /* all xids >= xmax are in progress */
	uint32_t xcnt;                 /* xids in progress at snapshot time, xmin <= xip[i] < xmax */
	uint32_t curcid;               /* command ids >= curcid of the own transaction are invisible */
	uint32_t own_xid;              /* GetCurrentTransactionIdIfAny() of the scanning backend; 0: none assigned */
	uint32_t clog_base, clog_n;    /* transaction status is given for xids clog_base .. clog_base + clog_n - 1 (clog_base % 4 == 0) */
	uint8_t  suboverflowed, takenDuringRecovery, haveDistribSnapshot, pad;      /* any of them set: GG_ERR_UNSUPPORTED */
	const uint32_t *xip;
	const uint8_t *clog;           /* 2 bits per xid exactly as pg_clog stores them (clog.h:25-28, clog.c:73-78) */
} gg_snapshot;

/* ---- type OIDs (src/include/catalog/pg_type.h) ---- */
#define GG_BOOLOID       16
#define GG_INT8OID       20
#define GG_INT4OID       23
#define GG_TEXTOID       25
#define GG_FLOAT8OID     701
#define GG_BPCHAROID     1042
#define GG_VARCHAROID    1043
#define GG_DATEOID       1082
#define GG_TIMESTAMPOID  1114
#define GG_NUMERICOID    1700     /* numeric(p,s) columns with a declared scale: evaluated as scaled 64-bit integers (exact), see
                                   * "numeric" below */

/* ---- function OIDs (pg_proc.h; values checked against the reference's generated fmgroids.h) ---- */
#define GG_F_INT4EQ 65
#define GG_F_INT4LT 66
#define GG_F_INT4NE 144
#define GG_F_INT4GT 147
#define GG_F_INT4LE 149
#define GG_F_INT4GE 150
#define GG_F_FLOAT8MUL 216
#define GG_F_FLOAT8DIV 217
#define GG_F_FLOAT8PL 218
#define GG_F_FLOAT8MI 219
#define GG_F_FLOAT8EQ 293
#define GG_F_FLOAT8NE 294
#define GG_F_FLOAT8LT 295
#define GG_F_FLOAT8LE 296
#define GG_F_FLOAT8GT 297
#define GG_F_FLOAT8GE 298
#define GG_F_I4TOD 316
#define GG_F_INT8EQ 467
#define GG_F_INT8NE 468
#define GG_F_INT8LT 469
#define GG_F_INT8GT 470
#define GG_F_INT8LE 471
#define GG_F_INT8GE 472
#define GG_F_INT48 481          /* int4 -> int8 cast */
#define GG_F_I8TOD 482
#define GG_F_BPCHAREQ 1048
#define GG_F_BPCHARNE 1053
#define GG_F_DATE_EQ 1086
#define GG_F_DATE_LT 1087
#define GG_F_DATE_LE 1088
#define GG_F_DATE_GT 1089
#define GG_F_DATE_GE 1090
#define GG_F_DATE_NE 1091
#define GG_F_NUMERIC_EQ 1718
#define GG_F_NUMERIC_NE 1719
#define GG_F_NUMERIC_GT 1720
#define GG_F_NUMERIC_GE 1721
#define GG_F_NUMERIC_LT 1722
#define GG_F_NUMERIC_LE 1723
#define GG_F_NUMERIC_ADD 1724
#define GG_F_NUMERIC_SUB 1725
#define GG_F_NUMERIC_MUL 1726
#define GG_F_DATE_LT_TIMESTAMP 2338
#define GG_F_DATE_LE_TIMESTAMP 2339
#define GG_F_DATE_EQ_TIMESTAMP 2340
#define GG_F_DATE_GT_TIMESTAMP 2341
#define GG_F_DATE_GE_TIMESTAMP 2342
#define GG_F_DATE_NE_TIMESTAMP 2343

/* aggregate OIDs (pg_aggregate.h:156-220) */
#define GG_AGG_AVG_NUMERIC  2103   /* numeric_avg_accum / numeric_avg: sum / N as numeric_div computes it (numeric.c:3173) */
#define GG_AGG_SUM_NUMERIC  2114   /* numeric_avg_accum / numeric_sum (numeric.c:3205) */
#define GG_AGG_AVG_FLOAT8   2105   /* float8_accum / float8_avg / float8_combine, state float8[3] "{0,0,0}" */
#define GG_AGG_SUM_INT4     2108   /* int4_sum / - / int8pl, state int8 init NULL */
#define GG_AGG_SUM_FLOAT8   2111   /* float8pl / - / float8pl, state float8 init NULL (strict: first value) */
#define GG_AGG_MAX_INT8     2115
#define GG_AGG_MAX_INT4     2116
#define GG_AGG_MAX_FLOAT8   2120
#define GG_AGG_MAX_DATE     2122
#define GG_AGG_MIN_INT8     2131
#define GG_AGG_MIN_INT4     2132
#define GG_AGG_MIN_FLOAT8   2136
#define GG_AGG_MIN_DATE     2138
#define GG_AGG_COUNT_ANY    2147   /* int8inc_any / - / int8pl, init 0 */
#define GG_AGG_COUNT_STAR   2803   /* int8inc / - / int8pl, init 0 */

/* ---- numeric ----
 * A numeric(p,s) column (atttypmod = ((p << 16) | s) + 4, utils/adt/numeric.c:650 numeric_typmod) is decoded from its on-disk
 * base-10000 digits (numeric.c:95-190) into a 64-bit integer scaled by 10^s; numeric_add / _sub / _mul and the comparisons run
 * on such integers with the result scales numeric.c gives them (add/sub: the larger display scale, :1659,1698; mul: their sum,
 * :1735) — exact, as the reference's arithmetic is.  sum() accumulates in 128 bits; avg() is numeric_div(sum, N) with
 * select_div_scale's result scale and div_var's rounding (numeric.c:3173, :6480 ff).  A value, product or sum outside 64 / 128
 * bits, a NaN, or a stored value with more fractional digits than its column's scale raises GG_ERR_UNSUPPORTED at fetch: the
 * caller runs the relation on the CPU path.
 * Constants: gg_expr.constvalue = the unscaled integer, constlen = its display scale.
 * Results (gg_aggval of sum / avg over numeric): the value is a 128-bit integer scaled by 10^dscale —
 * i = its low 64 bits, f[0] = the bit pattern of its high 64 bits, f[1] = dscale. */
#define GG_NUMERIC_TYPMOD(p, s) ((((int32_t) (p)) << 16 | (int32_t) (s)) + 4)

/* ---- limits of the accelerated subset ---- */
#define GG_MAX_ATTS        32
#define GG_MAX_EXPR_NODES  96
#define GG_MAX_AGGS        16
#define GG_MAX_KEYS        4       /* group / sort / hash key columns */
#define GG_MAX_TLIST       16

/* ---- tuple descriptor ---- */
typedef struct gg_attr {
	int32_t atttypid;
	int32_t atttypmod;      /* bpchar(n)/varchar(n): n + 4 (VARHDRSZ), else -1 */
	int16_t attlen;         /* >0 fixed, -1 varlena */
	int8_t  attalign;       /* 'c' 's' 'i' 'd' (tupmacs.h:121-130) */
	int8_t  attbyval;
	int8_t  attnotnull;
	int8_t  pad[3];
} gg_attr;                  /* 16 bytes */

/* How the tuples of a relation are laid out in device memory.
 *   GG_FMT_HEAP       32 KB heap pages (bufpage.h / htup_details.h), what SeqScan reads from storage
 *   GG_FMT_DATUMROWS  fixed-width rows of 64-bit words: word 0 = NULL mask (bit i: column i is NULL), word 1+i =
 *                     column i as a Datum in loaded form (int4/date sign-extended, float8 bits, short strings
 *                     packed LSB-first, bpchar blank-stripped).  This is what a receiving Motion hands to the
 *                     node above it — the device analogue of the MinimalTuples tupser.c serialises
 *                     (cdbmotion.c:378-470): every operator that scans heap pages also scans these rows.
 *                     Bit 63 of the mask word marks a slot that holds no row (a sending Motion claimed it and did not
 *                     fill it): consumers skip it. */
#define GG_FMT_HEAP      0
#define GG_FMT_DATUMROWS 1
#define GG_DATUMROW_DEAD 0x8000000000000000ull

typedef struct gg_tupdesc {
	int32_t natts;
	int32_t format;         /* GG_FMT_* */
	gg_attr attrs[GG_MAX_ATTS];
} gg_tupdesc;

/* ---- expressions: flat pool, children by index ----
 * A node's arguments have SMALLER indices than the node itself (children are appended before their parents, the way a
 * post-order walk of the Expr tree emits them); the plan compiler checks this, which is also what rules out cycles.
 * A malformed pool (index out of range, attribute number outside the descriptor, ...) is GG_ERR_ARG, never a crash. */
enum gg_expr_kind {
	GG_E_VAR = 1,      /* varno (0 = outer/scan, 1 = inner), varattno 1-based */
	GG_E_CONST = 2,    /* constvalue = Datum bits; strings: <=8 blank-stripped bytes packed LSB-first, constlen */
	GG_E_FUNC = 3,     /* OpExpr/FuncExpr with funcid (strict) */
	GG_E_AND = 4,      /* BoolExpr, 2 args (execQual.c ExecEvalAnd 3-valued logic) */
	GG_E_OR = 5,
	GG_E_NOT = 6,
	GG_E_ISNULL = 7,   /* NullTest IS NULL */
	GG_E_ISNOTNULL = 8
};

typedef struct gg_expr {
	int32_t kind;
	int32_t funcid;
	int32_t rettype;        /* type OID of the result */
	int16_t varno;
	int16_t varattno;
	int32_t nargs;
	int32_t args[2];
	int32_t constisnull;
	int32_t constlen;       /* string constants: blank-stripped length */
	int64_t constvalue;
} gg_expr;                  /* 48 bytes */

typedef struct gg_exprpool {
	int32_t nnodes;
	int32_t pad;
	gg_expr nodes[GG_MAX_EXPR_NODES];
} gg_exprpool;

/* ---- aggregates ---- */
enum gg_aggstage {          /* primnodes.h:257-264 AggStage */
	GG_AGGSTAGE_NORMAL = 0,
	GG_AGGSTAGE_PARTIAL = 1,   /* transfn, emit transition state (nodeAgg.c:975-979) */
	GG_AGGSTAGE_FINAL = 3      /* combinefn over partial states, then finalfn (nodeAgg.c:2123-2148) */
};

typedef struct gg_aggref {
	int32_t aggfnoid;       /* GG_AGG_* */
	int32_t arg;            /* root node of the argument expression; -1 for count(*).
	                         * FINAL stage: index of the input column carrying the partial state. */
} gg_aggref;

/* One aggregate value as it crosses the ABI.  NORMAL/FINAL: the SQL result
 * (f[0] for float8 results, i for int8 results).  PARTIAL: the transition
 * state exactly as the reference ships it through Motion (SURVEY App. A
 * "two-stage interchange"): sum(float8) -> f[0] (isnull if no input),
 * avg(float8) -> f[0..2] = {N, sumX, sumX2}, count -> i, sum(int4) -> i. */
typedef struct gg_aggval {
	double  f[3];
	int64_t i;
	int32_t isnull;
	int32_t pad;
} gg_aggval;                /* 40 bytes */

/* One output row of an Agg: group keys (Datum bits; strings packed like consts) + aggregate values. */
typedef struct gg_aggrow {
	int64_t   key[GG_MAX_KEYS];
	int32_t   keylen[GG_MAX_KEYS];     /* string keys: stripped length; else 0 */
	int32_t   keyisnull[GG_MAX_KEYS];
	gg_aggval agg[GG_MAX_AGGS];
} gg_aggrow;

/* ---- plan nodes ---- */
typedef struct gg_scan {            /* SeqScan + its qual (nodeSeqscan.c, execScan.c:111) */
	gg_tupdesc desc;
	int32_t    qual;                /* root in the pool, -1 = none; NULL result = not passed (execQual.c:6260) */
	int32_t    pad;
} gg_scan;

/* gg_agg.flags.  DEVICE_FINAL (PARTIAL stage only): the rows of this stage are combined by this engine's own FINAL stage
 * (gg_agg_final / the device-resident Motion), which like float8_avg never reads avg's sumX2 (float.c:1982-1996): the
 * stage then does not compute it and ships 0.  Leave it clear when a CPU FINAL stage consumes the rows — the reference's
 * float8_combine adds the sumX2 fields and its CHECKFLOATVAL sees them (float.c:1842-1876). */
#define GG_AGGF_DEVICE_FINAL 1

typedef struct gg_agg {             /* Agg (AGG_HASHED or AGG_PLAIN when numCols==0), nodeAgg.c */
	int32_t   aggstage;
	int32_t   numCols;
	int32_t   grpCol[GG_MAX_KEYS];      /* expr roots of the grouping columns (Vars of the input) */
	int32_t   numAggs;
	int32_t   flags;                    /* GG_AGGF_* */
	gg_aggref aggs[GG_MAX_AGGS];
	int64_t   numGroups;                /* planner's estimate (Agg.numGroups, plannodes.h); 0 = unknown.
	                                     * Sizes the hash table as in create_agg_hash_table (execHHashagg.c:810) */
} gg_agg;

enum gg_jointype {                  /* nodes/nodes.h JoinType */
	GG_JOIN_INNER = 0, GG_JOIN_LEFT = 1, GG_JOIN_FULL = 2, GG_JOIN_RIGHT = 3, GG_JOIN_SEMI = 4, GG_JOIN_ANTI = 5,
	GG_JOIN_LASJ_NOTIN = 6              /* NOT IN: any NULL inner key empties the result (nodeHashjoin.c:220-239,356-368) */
};

typedef struct gg_hashjoin {        /* HashJoin + Hash (nodeHashjoin.c, nodeHash.c) */
	int32_t jointype;
	int32_t nkeys;
	int32_t outerkey[GG_MAX_KEYS];      /* expr roots over the outer tuple (varno 0) */
	int32_t innerkey[GG_MAX_KEYS];      /* expr roots over the inner tuple (varno 1) */
	int32_t joinqual;                   /* extra join qual over both sides, -1 = none */
	int32_t pad;
} gg_hashjoin;

typedef struct gg_sortkey {         /* Sort.sortColIdx/sortOperators/nullsFirst (plannodes.h Sort) */
	int32_t col;                        /* 0-based column of the input row */
	int32_t typid;
	int32_t desc;                       /* 1 = DESC */
	int32_t nulls_first;
} gg_sortkey;

/* ---- window functions (WindowAgg, plannodes.h:1145; WindowFunc, primnodes.h) ---- */
/* frame_clause options (parsenodes.h:495-517) */
#define GG_FRAMEOPTION_NONDEFAULT                0x00001
#define GG_FRAMEOPTION_RANGE                     0x00002
#define GG_FRAMEOPTION_ROWS                      0x00004
#define GG_FRAMEOPTION_BETWEEN                   0x00008
#define GG_FRAMEOPTION_START_UNBOUNDED_PRECEDING 0x00010
#define GG_FRAMEOPTION_END_UNBOUNDED_PRECEDING   0x00020
#define GG_FRAMEOPTION_START_UNBOUNDED_FOLLOWING 0x00040
#define GG_FRAMEOPTION_END_UNBOUNDED_FOLLOWING   0x00080
#define GG_FRAMEOPTION_START_CURRENT_ROW         0x00100
#define GG_FRAMEOPTION_END_CURRENT_ROW           0x00200
#define GG_FRAMEOPTION_START_VALUE_PRECEDING     0x00400
#define GG_FRAMEOPTION_END_VALUE_PRECEDING       0x00800
#define GG_FRAMEOPTION_START_VALUE_FOLLOWING     0x01000
#define GG_FRAMEOPTION_END_VALUE_FOLLOWING       0x02000
#define GG_FRAMEOPTION_DEFAULTS (GG_FRAMEOPTION_RANGE | GG_FRAMEOPTION_START_UNBOUNDED_PRECEDING | GG_FRAMEOPTION_END_CURRENT_ROW)

/* window function OIDs (pg_proc.h:4874-4902); the aggregates allowed as window functions are the GG_AGG_* above, numeric excepted */
#define GG_WF_ROW_NUMBER        3100   /* int8 */
#define GG_WF_RANK              3101   /* int8 */
#define GG_WF_DENSE_RANK        3102   /* int8 */
#define GG_WF_PERCENT_RANK      3103   /* float8 */
#define GG_WF_CUME_DIST         3104   /* float8 */
#define GG_WF_NTILE             3105   /* int4; ntile(n), n a Const */
#define GG_WF_LAG               3106   /* lag(x) */
#define GG_WF_LAG_OFFSET        3107   /* lag(x, int4 offset) */
#define GG_WF_LAG_DEFAULT       3108   /* lag(x, int4 offset, default) */
#define GG_WF_LEAD              3109
#define GG_WF_LEAD_OFFSET       3110
#define GG_WF_LEAD_DEFAULT      3111
#define GG_WF_FIRST_VALUE       3112
#define GG_WF_LAST_VALUE        3113
#define GG_WF_NTH_VALUE         3114   /* nth_value(x, n), n a Const */

#define GG_MAX_WINFUNCS 8

typedef struct gg_winfunc {         /* WindowFunc (primnodes.h) */
	int32_t winfnoid;                   /* GG_WF_* or GG_AGG_* */
	int32_t wintype;                    /* type OID of the result */
	int32_t arg[3];                     /* expression roots in the pool, -1 = absent: a Var of the input row (varno 0) or a Const */
	int32_t pad;
} gg_winfunc;

typedef struct gg_window {          /* WindowAgg (plannodes.h:1145) */
	int32_t partNumCols;
	int32_t partColIdx[GG_MAX_KEYS];    /* 0-based columns of the input rows */
	int32_t ordNumCols;
	int32_t ordColIdx[GG_MAX_KEYS];
	int32_t frameOptions;               /* GG_FRAMEOPTION_* */
	int32_t numFuncs;
	gg_winfunc funcs[GG_MAX_WINFUNCS];
} gg_window;

enum gg_motiontype {                /* plannodes.h MotionType */
	GG_MOTION_HASH = 0,                 /* Redistribute */
	GG_MOTION_FIXED = 1,                /* Broadcast / Gather */
	GG_MOTION_EXPLICIT = 2
};

#ifdef __cplusplus
}
#endif
#endif /* GG_PLAN_H */
