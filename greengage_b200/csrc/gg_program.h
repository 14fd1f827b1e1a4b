/*
 * gg_program.h — the per-plan "device program" the host compiles from gg_plan.h
 * structures and hands to the kernels as a __grid_constant__ parameter.
 *
 * The reference evaluates Expr trees with one fmgr call per node per row
 * (execQual.c:2169,6260; SURVEY §8a rows 5,7).  Here the whole per-row work of
 * a SeqScan -> qual -> Agg slice — scan qual, grouping keys, every aggregate
 * argument — is flattened once per plan into ONE straight-line program for an
 * accumulator machine: a 64-bit accumulator + null flag and four temporaries
 * per lane, every lane of a warp running the same op on its own tuple.  Each
 * arithmetic op is a single IEEE/integer operation applied in the same order as
 * the tree, so per-row values are bit-identical to the reference's.
 */
#ifndef GG_PROGRAM_H
#define GG_PROGRAM_H

#include <stdint.h>
#include "../../include/gg_plan.h"

#define GGP_MAX_COLS    32     /* distinct referenced columns per side (= GG_MAX_ATTS) */
#define GGP_MAX_CONSTS  24
#define GGP_MAX_CODE    160
#define GGP_MAX_ACCS    16     /* accumulator columns (deduplicated aggregate arguments) */
#define GGP_MAX_SLOTS   24     /* value slots: columns + their sums of squares */
#define GGP_MAX_PAIRS   128    /* transposed kernel: (group, slot) pairs held in registers across a warp */
#define GGP_FAST_GROUPS 32     /* groups per block table */

/* how a referenced column is loaded into the 64-bit accumulator */
enum ggp_loadtype {
	GGP_LT_I4 = 1,       /* int4/date: sign-extended */
	GGP_LT_I8 = 2,       /* int8/timestamp/float8 bits */
	GGP_LT_BPCHAR = 3,   /* short string, trailing blanks stripped (bcTruelen), <= 8 bytes packed LSB-first */
	GGP_LT_VARCHAR = 4,  /* short string, not stripped */
	GGP_LT_BOOL = 5,
	GGP_LT_NUM = 6       /* numeric varlena -> 64-bit integer scaled by 10^scale (scale in the load op's aux, bits 0-3) */
};

/* Opcodes.  Operation and operand kind are fused into one opcode.  Operand suffixes: _C column (8-byte
 * load), _C4 int4/date column (sign-extended), _K constant, _T temporary.  idx = slot/const/temp index;
 * idx bit 7 on a column operand = inner tuple of a join.  aux bits 0-2 = ggp_cc for compares. */
enum ggp_opcode {
	GGP_END = 0,
	GGP_LD_C4, GGP_LD_C8, GGP_LD_BP, GGP_LD_VS, GGP_LD_BOOL, GGP_LD_K, GGP_LD_T,
	GGP_ADD_C, GGP_ADD_K, GGP_ADD_T,            /* float8pl   (float.c:782) */
	GGP_SUB_C, GGP_SUB_K, GGP_SUB_T,            /* float8mi   acc - x */
	GGP_RSUB_C, GGP_RSUB_K, GGP_RSUB_T,         /*            x - acc */
	GGP_MUL_C, GGP_MUL_K, GGP_MUL_T,            /* float8mul */
	GGP_DIV_C, GGP_DIV_K, GGP_DIV_T,            /* float8div  acc / x */
	GGP_RDIV_C, GGP_RDIV_K, GGP_RDIV_T,         /*            x / acc */
	GGP_CMPF_C, GGP_CMPF_K, GGP_CMPF_T,         /* float8_cmp_internal(acc, x) cc  (float.c:964) */
	GGP_CMPI_C4, GGP_CMPI_C8, GGP_CMPI_K, GGP_CMPI_T,   /* signed 64-bit compare */
	GGP_CMPS_K, GGP_CMPS_T,                     /* packed strings equal / not equal (bpchareq on stripped bytes) */
	GGP_DATE2TS,                                /* date2timestamp (date.c:457) */
	GGP_I2F8,                                   /* i4tod / i8tod */
	GGP_AND_T, GGP_OR_T,                        /* 3-valued (execQual.c:3404,3455) */
	GGP_NOT, GGP_ISNULL, GGP_ISNOTNULL,
	GGP_NOP,                                    /* carries post-actions only */
	/* short-circuit evaluation (ExecEvalAnd / ExecEvalOr, execQual.c:3321-3450): the second arm of AND / OR is not
	 * evaluated when the first decides the result, so it cannot raise.  The op stream stays warp-uniform: the arm still
	 * runs, but on lanes where the reference would have skipped it the lane is not `live`, and dead lanes raise nothing.
	 * GUARD pushes `live` and clears it where temp[idx] already decides (AND: non-NULL FALSE; OR: non-NULL TRUE);
	 * UNGUARD pops. */
	GGP_GUARD_AND, GGP_GUARD_OR, GGP_UNGUARD,
	/* numeric as scaled 64-bit integers (gg_plan.h "numeric"): exact integer arithmetic; a result that does not fit raises
	 * GGP_EF_NUMERIC_RANGE (the plan then runs on the CPU path), never a wrong value */
	GGP_LD_NUM,                                 /* acc = numeric column idx scaled by 10^(aux & 15) */
	GGP_IADD_K, GGP_IADD_T,                     /* acc + x */
	GGP_ISUB_K, GGP_ISUB_T,                     /* acc - x */
	GGP_IRSUB_K, GGP_IRSUB_T,                   /* x - acc */
	GGP_IMUL_K, GGP_IMUL_T,                     /* acc * x */
	GGP_LO32, GGP_SAR32,                        /* acc & 0xFFFFFFFF ; acc >> 32 (arithmetic): the two halves a 128-bit sum is kept in */
	GGP_NOPS
};

enum ggp_cc { GGP_LT = 0, GGP_LE, GGP_EQ, GGP_NE, GGP_GT, GGP_GE };

/* post-actions, applied to the accumulator after the op, in this order */
#define GGP_F_ST      0x01     /* temp[(aux >> 4) & 3] = acc */
#define GGP_F_FILTER  0x02     /* the row passes only if acc is TRUE (NULL is not true, execQual.c:6300) */
#define GGP_F_KEY     0x04     /* grouping key [(aux >> 6) & 3] = acc */
#define GGP_F_GROUP   0x08     /* all keys known: find/insert the group */
#define GGP_F_OUT     0x10     /* value slot[out] = acc */
#define GGP_F_OUTSQ   0x20     /* value slot[out2] = acc * acc  (float8_accum's sumX2, float.c:1878); out2 = GGP_OUTSQ_CHECK_ONLY:
                                * the square is only tested for overflow (a plan that does not ship sumX2 still raises what
                                * float8_accum's CHECKFLOATVAL raises for a single input, float.c:1895-1896) */
#define GGP_OUTSQ_CHECK_ONLY 0xFF
#define GGP_F_PROBE   0x40     /* join pipelines: the probing row's join keys are complete; what follows runs once per match */

typedef struct ggp_op {
	uint8_t  op;
	uint8_t  idx;
	uint8_t  aux;
	uint8_t  flags;
	uint16_t off;        /* column operand: constant offset (attcacheoff) usable when the tuple has no NULLs, else 0xFFFF */
	uint8_t  out, out2;
} ggp_op;                /* 8 bytes */

/* accumulator column kinds */
enum ggp_acckind {
	GGP_ACC_F8SUM = 1,   /* sum (and, through a second slot, sum of squares) of a float8 expression */
	GGP_ACC_F8MIN, GGP_ACC_F8MAX,
	GGP_ACC_I8SUM, GGP_ACC_I8MIN, GGP_ACC_I8MAX,
	GGP_ACC_COUNT        /* non-null count only (count(expr)); count(*) needs no column */
};

typedef struct ggp_attr {
	int16_t attlen;
	int8_t  attalign;    /* 'c','s','i','d' */
	int8_t  slot;        /* column slot if referenced, else -1 */
	int16_t cacheoff;    /* attcacheoff: constant offset while no NULL/varlena precedes, else -1 (heaptuple.c:1160) */
	int8_t  notnull;
	int8_t  pad;
} ggp_attr;

/* One side (scan tuple layout + the columns the program touches) */
typedef struct ggp_side {
	int32_t natts;           /* attributes in the descriptor */
	int32_t natts_walk;      /* walk attributes [0, natts_walk) : highest referenced attno */
	int32_t first_walk;      /* first attribute whose offset is not a constant (no-NULL tuples start walking at first_walk-1) */
	int32_t ncols;
	int32_t rowwords;        /* 0: heap pages; > 0: datum rows (GG_FMT_DATUMROWS) of this many 64-bit words */
	int32_t pad;
	ggp_attr att[GG_MAX_ATTS];
	uint8_t  coltype[GGP_MAX_COLS];   /* ggp_loadtype per slot */
	uint8_t  colatt[GGP_MAX_COLS];    /* 0-based attribute per slot */
} ggp_side;

typedef struct ggp_program {
	ggp_side outer;
	int32_t  nconst;
	int32_t  nullable;       /* 1: some referenced value can be NULL => null-tracking kernel variant */
	int64_t  consts[GGP_MAX_CONSTS];
	int32_t  constnull;      /* bit i: const i is NULL */
	int32_t  ncode;
	ggp_op   code[GGP_MAX_CODE];     /* qual (FILTER) ; keys (KEY.., GROUP) ; aggregate arguments (OUT/OUTSQ) ; END */
	int32_t  nkeys;
	uint8_t  keytype[GG_MAX_KEYS];    /* 1 int, 2 float8 (normalise -0/NaN), 3 string */
	int32_t  nacc;           /* accumulator columns */
	uint8_t  acckind[GGP_MAX_ACCS];
	int8_t   accsq[GGP_MAX_ACCS];     /* value slot of the column's sum of squares (avg's float8_accum state), or -1 */
	int32_t  nslots;         /* value slots = nacc + number of sum-of-squares slots; slot j < nacc is column j */
	int32_t  priv_ok;        /* 1: every column is a NOT NULL float8 sum => private-accumulator kernel applies */
} ggp_program;

/* HashJoin (+ Agg on top): two programs.
 *   build  runs over every inner tuple:  [inner qual FILTER]  join keys KEY k..  payload columns OUT p..
 *   probe  runs over every outer tuple:  [outer qual FILTER]  join keys KEY k.. PROBE
 *          and then once per matching inner row, with the payload visible as "inner columns":
 *          [join qual FILTER]  grouping keys KEY k.. GROUP  aggregate arguments OUT/OUTSQ
 * The payload is exactly the set of inner columns referenced above the join (Vars with varno 1). */
#define GGP_MAX_PAYLOAD 8
typedef struct ggp_joinprog {
	ggp_program build;
	ggp_program probe;       /* probe.nkeys/keytype describe the GROUPING keys of the aggregate above the join */
	int32_t nkeys;           /* join keys */
	int32_t npayload;
	int32_t jointype;        /* gg_jointype */
	int32_t probe_pc;        /* first op of the per-match segment of `probe` */
	uint8_t keytype[GG_MAX_KEYS];
} ggp_joinprog;

/* One partial group record: what a block (or a segment, for the FINAL stage) knows about one group.
 * The merge kernel folds records with equal keys in a fixed order, so results are deterministic. */
typedef struct ggp_grec {
	uint64_t key[GG_MAX_KEYS];
	uint32_t keynull;        /* bit i: key i is NULL */
	uint32_t valid;
	uint64_t count;          /* rows of the group (count(*)) */
	double   sum[GGP_MAX_ACCS];      /* F8SUM: sum ; F8MIN/MAX: value ; I8*: int64 bits */
	double   sumsq[GGP_MAX_ACCS];
	uint64_t n[GGP_MAX_ACCS];        /* non-null inputs */
} ggp_grec;

/* error flags raised by kernels (bit mask in a device word) */
#define GGP_EF_FLOAT_OVERFLOW   0x01
#define GGP_EF_FLOAT_UNDERFLOW  0x02
#define GGP_EF_DIV_ZERO         0x04
#define GGP_EF_VISIBILITY       0x08
#define GGP_EF_BADPAGE          0x10
#define GGP_EF_GROUP_OVERFLOW   0x20   /* more groups than the kernel variant holds: rerun on a wider variant */
#define GGP_EF_STRING_TOO_LONG  0x40
#define GGP_EF_DATE_RANGE       0x80
#define GGP_EF_NOTNULL_VIOLATED 0x100
#define GGP_EF_INT_OVERFLOW     0x200
#define GGP_EF_TABLE_FULL       0x400
#define GGP_EF_SAW_INF          0x800   /* informational: an aggregate input was +-Inf/NaN */
#define GGP_EF_RECHECK          0x1000  /* a fast variant saw a non-finite sum: replay on the checked variant */
#define GGP_EF_PEER_FAILED      0x2000  /* a segment's slice below a Motion failed with an error that has no flag of its own */
#define GGP_EF_HOSTPATH         0x4000  /* a segment could not contribute device-resident records to a Motion (its aggregate
                                         * spilled to the general hash table, or holds more groups than a block carries): every
                                         * segment sees it and the slice is run again with host-row Motions */
#define GGP_EF_NUMERIC_RANGE    0x8000  /* a numeric value / product outside the scaled 64-bit representation, a NaN, or more
                                         * fractional digits than the column's scale: not an ERROR of the query — CPU path */
#define GGP_EF_INFO_MASK        (GGP_EF_SAW_INF | GGP_EF_RECHECK)

/* how a Motion hash key is hashed (cdbhash.c:215-287: the type's default hash opclass function) */
enum ggp_hashtype { GGP_HT_INT4 = 1, GGP_HT_INT8, GGP_HT_FLOAT8, GGP_HT_STR, GGP_HT_BOOL };

typedef struct ggp_acckinds { uint8_t k[GGP_MAX_ACCS]; } ggp_acckinds;

#if defined(__cplusplus) && !defined(__CUDACC_RTC__)
/* host-side compiler (gg_compile.cpp) */
struct ggp_aggmap {          /* how each Aggref reads the accumulator columns */
	int32_t col;             /* accumulator column, -1 for count(*); numeric sum / avg: the low half, col + 1 the high half */
	int32_t scale;           /* numeric sum / avg: display scale of the summed expression */
};
/* the accumulator column an aggregate's transition state lives in (ggp_acckind); 0 for count(*), whose state is
 * ggp_grec::count and needs no column; -1 for an aggregate the device does not run */
static inline int ggp_acckind_of(int32_t aggfnoid)
{
	switch (aggfnoid)
	{
		case GG_AGG_COUNT_STAR: return 0;
		case GG_AGG_COUNT_ANY: return GGP_ACC_COUNT;
		case GG_AGG_SUM_FLOAT8: case GG_AGG_AVG_FLOAT8: return GGP_ACC_F8SUM;
		case GG_AGG_MIN_FLOAT8: return GGP_ACC_F8MIN;
		case GG_AGG_MAX_FLOAT8: return GGP_ACC_F8MAX;
		/* numeric: a 128-bit integer sum kept as two int64 sums of the inputs' halves (col, col + 1) */
		case GG_AGG_SUM_INT4: case GG_AGG_SUM_NUMERIC: case GG_AGG_AVG_NUMERIC: return GGP_ACC_I8SUM;
		case GG_AGG_MIN_INT4: case GG_AGG_MIN_INT8: case GG_AGG_MIN_DATE: return GGP_ACC_I8MIN;
		case GG_AGG_MAX_INT4: case GG_AGG_MAX_INT8: case GG_AGG_MAX_DATE: return GGP_ACC_I8MAX;
		default: return -1;
	}
}
/* the ggp_hashtype of a key type (cdb_hashproc_in_opfamily, cdbhash.c:135-165: date hashes as int4, timestamp as int8, bool as
 * hashchar, bpchar blank-stripped); 0 for a type the device cannot hash */
static inline int ggp_hashtype_of(int32_t typid)
{
	switch (typid)
	{
		case GG_INT4OID: case GG_DATEOID: return GGP_HT_INT4;
		case GG_INT8OID: case GG_TIMESTAMPOID: return GGP_HT_INT8;
		case GG_FLOAT8OID: return GGP_HT_FLOAT8;
		case GG_BPCHAROID: case GG_VARCHAROID: case GG_TEXTOID: return GGP_HT_STR;
		case GG_BOOLOID: return GGP_HT_BOOL;
		default: return 0;
	}
}
int ggp_compile_scanagg(const gg_scan *scan, const gg_agg *agg, const gg_exprpool *pool,
                        ggp_program *prog, ggp_aggmap *aggmap, char *err, int errlen);
int ggp_disasm(const ggp_program *p, char *buf, int cap);
/* Redistribute Motion: scan qual FILTER ; hash keys KEY.. GROUP (= route + claim an output row) ; payload OUT.. */
int ggp_compile_motion(const gg_scan *scan, const gg_exprpool *pool, const int32_t *hashkeys, int nkeys,
                       const int32_t *payload, int npayload, ggp_program *prog, uint8_t *hashtype /* [GG_MAX_KEYS] */,
                       char *err, int errlen);
int ggp_compile_join(const gg_scan *outer, const gg_scan *inner, const gg_hashjoin *hj, const gg_agg *agg,
                     const gg_exprpool *pool, ggp_joinprog *jp, ggp_aggmap *aggmap, char *err, int errlen);
/* HashJoin with a target list: the same build program; the probe's per-match piece is the join qual FILTER, then GROUP (= claim
 * an output row) and one OUT per target (1..16, Vars with varno 0 outer / 1 inner) */
int ggp_compile_joinrows(const gg_scan *outer, const gg_scan *inner, const gg_hashjoin *hj, const int32_t *targets, int ntargets,
                         const gg_exprpool *pool, ggp_joinprog *jp, char *err, int errlen);
#endif

#endif /* GG_PROGRAM_H */
