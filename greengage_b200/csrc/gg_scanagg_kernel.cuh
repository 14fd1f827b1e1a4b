/*
 * gg_scanagg_kernel.cuh — the scan kernel body of the GPU segment engine, in six roles.
 *
 * Replaces, for one segment, the per-tuple loops
 *   ExecAgg -> agg_hash_initial_pass -> ExecSeqScan -> heap_getnext -> heapgetpage
 *   MultiExecHash / ExecHashJoin_guts, the sending half of ExecMotion
 *   (nodeAgg.c:1123, execHHashagg.c:905, nodeSeqscan.c:128, heapam.c:312-463,767-1006, nodeHash.c:88,
 *    nodeHashjoin.c:78, nodeMotion.c:270; SURVEY §3.3 hot loops B and C)
 * with one persistent, warp-specialised kernel body (scanagg_body<MODE, PL, JOIN>):
 *
 *   producer warp    TMA bulk-copies whole 32 KB heap pages (or 32 KB chunks of datum rows) HBM -> shared-memory
 *                    ring (cp.async.bulk + mbarrier complete_tx; SASS UBLKCP)
 *   consumer warps   lane = one line pointer: ItemId decode, visibility, attribute walk (slot_deform_tuple
 *                    semantics), then ONE compiled program per row (gg_program.h); what the program's
 *                    post-actions do is the role:
 *     MODE_PRIV      scan qual -> grouping keys -> group lookup in a per-block key table -> aggregate arguments into
 *                    per-thread private accumulators: [group][slot][thread] float8 arrays in shared memory (a
 *                    warp's 32 read-modify-writes hit 32 banks: 3 instructions per value, no atomics, no
 *                    shuffles) and, in plan-specialised kernels, the last slots in registers (RegAcc)
 *     MODE_TR/TRN    the same with "lane owns (group, slot)": the warp's 32 values are transposed through shared
 *                    memory and folded by the owning lane into registers (<= 32 groups, <= 128 pairs; min/max/int
 *                    sums; TRN tracks NULLs)
 *     MODE_HASH      the general HashAggregate: groups in one HBM hash table, transition functions as atomics
 *     MODE_BUILD     Hash node: join keys + payload columns into the join hash table
 *     JOIN = true    (with PRIV / TR / TRN / HASH) the probe side: every outer row probes the table and each match
 *                    runs the per-match piece of the program; also the fill-inner pass of right / full joins
 *     MODE_PART      sending Motion: cdbhash + jump consistent hash, rows packed per destination; with JOIN = true the
 *                    probe of a join with a target list: every joined row written as a datum row (JoinRowSink)
 *   epilogue         PRIV / TR: threads -> one record per group and block -> global; a single-block merge kernel
 *                    folds records with equal keys.  Every reduction tree is fixed => sums are bit-identical run to
 *                    run.
 *   PL               how the kernel reaches the plan: DynPlan interprets the program table; a generated StaticPlan
 *                    (gg_jit.cpp) carries the same exec_op()/walk_step() calls with literal operands.
 *
 * HBM-bound by construction: algorithmic bytes = nblocks * 32768, each read exactly once.
 */
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "gg_device.cuh"
#include "gg_aocs_decode.h"

namespace ggd {

#define GG_NROUNDS (GGP_MAX_PAIRS / 32)
#define GG_REG_GROUPS 4        /* register-resident accumulators: groups ... */
#define GG_REG_SLOTS  3        /* ... x trailing value slots */
/* the 12 accumulators are separate scalars (arrays inside the sink end up in local memory): X(group, slot) */
#define GG_RQ_FOREACH(X) X(0, 0) X(0, 1) X(0, 2) X(1, 0) X(1, 1) X(1, 2) X(2, 0) X(2, 1) X(2, 2) X(3, 0) X(3, 1) X(3, 2)
struct RegAcc {
#define GG_RQ_DECL(G, J) double r##G##J;
	GG_RQ_FOREACH(GG_RQ_DECL)
#undef GG_RQ_DECL
	/* float8 sums start from -0, the identity of IEEE addition: a sum is -0 exactly when every input was -0, as
	 * float8pl's NULL initcond gives (the first input taken as it is) */
	__device__ __forceinline__ void zero()
	{
#define GG_RQ_ZERO(G, J) r##G##J = -0.0;
		GG_RQ_FOREACH(GG_RQ_ZERO)
#undef GG_RQ_ZERO
	}
	__device__ __forceinline__ void add(int g, int j, double v)
	{
#define GG_RQ_ADD(G, J) if (j == J && g == G) r##G##J = __dadd_rn(r##G##J, v);
		GG_RQ_FOREACH(GG_RQ_ADD)
#undef GG_RQ_ADD
	}
};

enum { MODE_PRIV = 0, MODE_TR = 1, MODE_TRN = 2,
       MODE_BUILD = 3,     /* Hash node: scan the inner relation into the join hash table (no aggregation) */
       MODE_PART = 4,      /* sending Motion: route every row by cdbhash and write it into its destination's region */
       MODE_HASH = 5 };    /* HashAggregate with any number of groups: one hash table in HBM, atomics */

/* The general HashAggregate (execHHashagg.c:456 lookup_agg_hash_entry, nodeAgg.c:545 advance_aggregates) for group
 * counts beyond what a block holds on chip: open addressing in HBM, capacity a power of two, one entry of `stride`
 * 64-bit words per slot (a multiple of 4 words, so entries start on 32-byte sectors and a row's lookup + transition
 * touch one or two sectors):
 *   [0]                    0 empty | 1 being written | bit 63 ready, bits 32..35 key-NULL mask, bits 0..31 hash tag
 *   [1 .. nkeys]           normalised grouping keys
 *   [off_cnt]              rows of the group
 *   [off_acc + j]          F8SUM/I8SUM: running sum; MIN/MAX: current extreme (bits)   -> atomicAdd / CAS / atomicMin,Max
 *   [off_accn + j]         non-NULL inputs (only when the plan can see NULLs; else it equals the row count)
 *   [off_sq + j]           float8_accum's sumX2 where the plan ships it
 * Float sums are accumulated with atomicAdd in arrival order: exact to the last few ulps, not run-to-run identical
 * (the reference's hash aggregate adds in scan order, also not an order the SQL result depends on). */
struct HashAggTable {
	unsigned long long *ent;
	uint64_t cap;                          /* slots */
	uint32_t stride;                       /* words per entry */
	uint32_t off_cnt, off_acc, off_accn, off_sq;   /* word offsets inside an entry; off_accn / off_sq = 0: not kept */
	uint8_t sqcol[GGP_MAX_SLOTS];          /* value slot -> accumulator column whose sum of squares it is (slots >= nacc) */
	uint8_t acckind[GGP_MAX_ACCS];
	int nacc, nkeys;
};
#define GG_HA_LOCKED 1ull

/* Redistribute Motion, sending side (nodeMotion.c:1481-1687 + cdbhash.c:173-287): output = nsegs regions of
 * `cap` datum rows (GG_FMT_DATUMROWS) each; cursor[d] counts the rows claimed for destination d. */
struct MotionOut {
	unsigned long long *rows;             /* [nsegs][cap][rowwords] */
	unsigned long long *cursor;           /* [nsegs] */
	uint64_t cap;
	int nsegs, rowwords;
	uint32_t hashtypes;                   /* 4 bits per hash key: ggp_hashtype */
	/* > 0: a warp claims rows of a destination's region `window` at a time and hands them out from shared memory, so the
	 * region cursors (a handful of addresses every warp of the grid would otherwise hit once per 32 rows) see 1 / window of
	 * the atomics.  What a warp has claimed and not used when the kernel ends is marked dead (GG_ROW_DEAD in the row's mask
	 * word): the region stays one contiguous run of rows, a few of which no consumer sees.  0: exact claims, no dead rows
	 * (small inputs, more than 32 destinations). */
	uint32_t window;
	/* how a row's hash value picks its region: 0 = a segment (cdbhashreduce: jump consistent hash, cdbhash.c:255-287);
	 * 1 = a hash-join batch, the reference's bit usage (ExecHashGetBucketAndBatch, nodeHash.c:1132-1151):
	 * batchno = (hashvalue >> log2_nbuckets) & (nbatch - 1), nsegs = nbatch a power of two, shift = log2_nbuckets */
	uint32_t route, shift;
};
#define GG_ROW_DEAD 0x8000000000000000ull  /* datum rows: mask word bit 63 = not a row (skipped by every consumer) */

/* Column files staged in a ring slot (the producer of an AOCS scan writes this, the consumers read it): the slot starts with
 * one 48-byte record per projected column slot, the copied byte ranges follow from GG_AOCS_DATA_OFF.  A unit's rows of one
 * column lie in at most four runs (one per storage block touched): run k holds the unit's rows [cum[k-1], cum[k]) at
 * base + rel[k] + (row - cum[k-1]) * stride[k]. */
#define GG_AOCS_META_BYTES  48
#define GG_AOCS_META_CUM    0        /* u32[4]: rows of the unit up to and including run k (0xFFFFFFFF: no such run) */
#define GG_AOCS_META_REL    16       /* u32[4]: byte offset of run k's first value from `base` */
#define GG_AOCS_META_STRIDE 32       /* u16[4]: bytes between the values of run k */
#define GG_AOCS_META_FLAGS  40       /* u32: bit 0 = not staged (consumers take gg_aocs_fetch), bits 8..15 = enum gg_aocs_kind */
#define GG_AOCS_META_BASE   44       /* u32: shared address of the column's copied range */
#define GG_AOCS_META_SLOW   1u
#define GG_AOCS_DATA_OFF    (32 * GG_AOCS_META_BYTES)

/* Join hash table (Hash / HashJoin, nodeHash.c:88-176,906-1222): open addressing, linear probing, one
 * slot per inner row (duplicate keys simply occupy successive slots), entries of `stride` 64-bit words:
 *   [0]            bit 63 occupied | bit 62 NULL join key (kept for right/full joins only: never matches) |
 *                  bit 61 matched (MemTupleSetMatch, nodeHashjoin.c:386; right/full joins) |
 *                  bits 32..39 payload-NULL mask | bits 0..31 hash
 *   [1 .. nkeys]   join keys, normalised so that bitwise equality is SQL equality
 *   [1+nkeys ..]   payload = the inner columns referenced above the join, loaded by the build program
 * Sized by the host to >= 2x the inner row count, so a probe always ends at an empty slot. */
struct JoinTable {
	unsigned long long *ent;
	uint32_t mask;                        /* slots - 1 (power of two) */
	uint32_t stride;                      /* 64-bit words per entry */
	int nkeys, npayload;
	int jointype;                         /* gg_jointype */
	int probe_pc;                         /* probe program: first op of the per-match segment */
	uint32_t keytypes;                    /* join keys, 2 bits each */
	unsigned long long *nbuilt;           /* [0] rows inserted, [1] inner rows with a NULL join key, [2] != 0: two inserted rows may
	                                       * share a join key (an insert passed an entry with its own hash tag) */
	int unique;                           /* probe side: the table's join keys are pairwise distinct (nbuilt[2] stayed 0), so a row's
	                                       * first key match is its only one and the probe need not run on to an empty slot */
	int keepnull;                         /* right / full join: rows with NULL keys are inserted too (nodeHashjoin.c:209) */
	int mark_matched;                     /* right / full join: a qualifying match marks the entry */
	int inner_empty;                      /* LASJ_NOTIN needs to know (nodeHashjoin.c:361) */
};
#define GG_HT_OCCUPIED 0x8000000000000000ull
#define GG_HT_NULLKEY  0x4000000000000000ull
#define GG_HT_MATCHED  0x2000000000000000ull

__device__ __forceinline__ uint64_t join_hash(uint64_t k0, uint64_t k1)
{
	uint64_t h = k0 ^ (k1 * 0x9E3779B97F4A7C15ull);
	h ^= h >> 33; h *= 0xff51afd7ed558ccdull; h ^= h >> 33; h *= 0xc4ceb9fe1a85ec53ull; h ^= h >> 33;
	return h;
}

struct ScanAggParams {
	const uint8_t *pages;
	uint64_t nblocks;
	ggp_grec *block_recs;                 /* [gridDim.x][GGP_FAST_GROUPS] */
	uint32_t *errflags;
	unsigned long long *counters;         /* [0] rows scanned (visible), [1] rows passed */
	int nstage;
	int gcap;                             /* groups this variant holds per block */
	int scratch_per_warp;                 /* bytes: column offsets (+ TR: transposed values, group ids, null masks) */
	uint32_t scratch_off;                 /* byte offsets from the start of dynamic shared memory */
	uint32_t cnt_off, acc_off;            /* MODE_PRIV: per-thread row counts [gcap][NT] u32, sums [gcap][nslots][NT] f64 */
	JoinTable jt;                         /* joins only */
	MotionOut mo;                         /* MODE_PART only */
	HashAggTable ha;                      /* MODE_HASH only */
	uint64_t nrows;                       /* datum-row input: total rows (pages/nblocks then describe 32 KB chunks of rows) */
	int fill_inner;                       /* join probe kernels: this launch is HJ_FILL_INNER_TUPLES — the "pages" are the hash
	                                       * table itself, every unmatched entry is emitted with a null-extended outer side */
	/* Append-only column-oriented input (aocsam.c:661 aocs_getnext): aocs_tile_rows > 0 — there are no pages; unit `it` of a
	 * block is a TILE of aocs_tile_rows rows (a multiple of 32), a lane loads the referenced columns of its row straight from
	 * the column files in device memory (aocs[a] = column a of the plan's descriptor; gg_aocs_fetch) into a staged datum row
	 * in shared memory and the row program runs over that: no attribute walk, no line pointers, only projected bytes read. */
	const gg_aocs_devcol *aocs;
	int32_t aocs_tile_rows;
	/* the scan's staging unit: `aocs_unit_rows` consecutive rows (a multiple of 32, at most 1024) of every projected column
	 * are bulk-copied into one ring slot; nblocks counts these units and every block takes a contiguous run of them */
	int32_t aocs_unit_rows;
	int nokeycache;                       /* experiments: 1 = every row looks its group up in the block table (no register cache) */
	const uint32_t *snap;                 /* the scan's snapshot in device memory (gg_device.cuh heap_tuple_satisfies_mvcc), or
	                                       * nullptr: visibility from hint bits only */
	int team;                             /* > 0: consumer warps work in teams of this many warps, one page per team at a time (a
	                                       * warp only visits its team's pages); 0: every warp visits every page and the chunks
	                                       * are dealt round-robin across pages */
};

__device__ __forceinline__ uint4 lds128(uint32_t a)
{
	uint4 v;
	asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a));
	return v;
}
/* gg_aocs_value (gg_aocs_decode.h) over a value staged in shared memory */
__device__ __forceinline__ uint32_t aocs_value_smem(int kind, uint32_t a, uint64_t &word)
{
	uint64_t v = 0;
	if (kind == GG_AOCS_K_W8) v = lds64(a);
	else if (kind == GG_AOCS_K_I4) v = (uint64_t) (int64_t) (int32_t) lds32(a);
	else if (kind == GG_AOCS_K_I2) v = (uint64_t) (int64_t) (int16_t) lds16(a);
	else if (kind == GG_AOCS_K_B1) v = lds8(a);
	else
	{
		int n = (int) (lds8(a) & 0x7F) - 1;                 /* payload bytes after the 1-byte header */
		if (kind == GG_AOCS_K_BPCHAR)
			while (n > 0 && lds8(a + (uint32_t) n) == ' ') n--;      /* bcTruelen (varchar.c:653) */
		if (n > 8) return GG_AOCS_E_IRREGULAR;
		for (int i = 0; i < n; i++) v |= (uint64_t) lds8(a + 1 + (uint32_t) i) << (8 * i);
	}
	word = v;
	return 0;
}

#define GG_MAX_TEAMS 6                    /* consumer teams per block (at most one per ring slot) */
#define GG_MAX_STAGES 6                   /* ring slots */
struct BlockTable {                       /* per-block group table in shared memory */
	/* teams only: the "page has landed" barriers, one set per team — [team][use of the team's barrier set mod nstage].  A parity
	 * wait tells a barrier's current phase from the one before it and no further, so it is exact only for a waiter that has
	 * itself seen every earlier phase of that barrier complete.  The per-slot barriers are that for a warp visiting every page;
	 * a team sees only its own pages, hence its own barriers, which nobody else waits on (the data still lands in ring slot
	 * page mod nstage, released through the slot's `empty` barrier as always). */
	unsigned long long teamfull[GG_MAX_TEAMS * GG_MAX_STAGES];
	uint64_t key[GGP_FAST_GROUPS][GG_MAX_KEYS];
	uint32_t keynull[GGP_FAST_GROUPS];
	volatile int n;
	int lock;
};

__device__ __forceinline__ bool key_eq(const BlockTable *T, int i, const uint64_t *k, uint32_t knull, int nkeys, uint32_t keytypes)
{
	if (T->keynull[i] != knull) return false;
	for (int c = 0; c < nkeys; c++)
		if (!key_same(T->key[i][c], k[c], (f8_keys(keytypes) >> (2 * c)) & 1)) return false;
	return true;
}

/* find the group of each lane's key, inserting new groups under a block-level lock
 * (lookup_agg_hash_entry, execHHashagg.c:456: NULL keys compare equal to each other) */
__device__ __forceinline__ int find_or_insert(BlockTable *T, const uint64_t *k, uint32_t knull, int nkeys, uint32_t keytypes,
                                              int gcap, bool want, int lane, uint32_t &err)
{
	int gid = -1;
	bool need = want;
	if (need)
	{
		int n = T->n;
		for (int i = 0; i < n; i++)
			if (key_eq(T, i, k, knull, nkeys, keytypes)) { gid = i; break; }
		need = gid < 0;
	}
	unsigned m = __ballot_sync(GG_FULL_MASK, need);
	while (m)
	{
		int leader = __ffs(m) - 1;
		if (lane == leader)
		{
			while (atomicCAS(&T->lock, 0, 1) != 0) { }
			__threadfence_block();
			int n = T->n, found = -1;
			for (int i = 0; i < n; i++)
				if (key_eq(T, i, k, knull, nkeys, keytypes)) { found = i; break; }
			if (found < 0)
			{
				if (n < gcap)
				{
					for (int c = 0; c < GG_MAX_KEYS; c++) T->key[n][c] = c < nkeys ? k[c] : 0;
					T->keynull[n] = knull;
					__threadfence_block();
					T->n = n + 1;
					found = n;
				}
				else
					err |= GGP_EF_GROUP_OVERFLOW;
			}
			__threadfence_block();
			atomicExch(&T->lock, 0);
			gid = found;
			need = false;
		}
		__syncwarp();
		if (need)
		{
			int n = T->n;
			for (int i = 0; i < n; i++)
				if (key_eq(T, i, k, knull, nkeys, keytypes)) { gid = i; break; }
			need = gid < 0;
		}
		m = __ballot_sync(GG_FULL_MASK, need);
	}
	return gid;
}

/* post-action sink shared by the kernel variants */
template <int MODE, bool JOIN = false>
struct RowSink {
	uint32_t keytypes;           /* 2 bits per key: 1 int, 2 float8, 3 string */
	BlockTable *T;
	uint64_t k0, k1, k2, k3;
	uint32_t knull;
	int nkeys, gcap, lane, gid;
	uint32_t *err;
	unsigned long long npassed;
	bool nonfinite;
	/* MODE_PRIV */
	uint32_t acc_thread;         /* shared address of this thread's slot-0/group-0 accumulator */
	uint32_t cnt_thread;
	uint32_t gstride, sstride, cstride;
	/* MODE_PRIV, plan-specialised kernels with at most GG_REG_GROUPS groups: the last `nreg` value slots are not kept in
	 * shared memory but in registers (rq[group][slot - nsl]) — predicated adds with compile-time indices.  Frees
	 * shared memory for more warps / ring stages; folded through the ring's memory in the epilogue. */
	int nsl, nreg;
	RegAcc rq;
	/* MODE_TR */
	uint32_t sv;                 /* shared address of the warp's transposed values [slot][33] f64 */
	uint32_t vnull;
	/* joins: per-match segment */
	bool jq;                     /* did the join qual pass for this match */
	bool nullext;                /* this lane emits its null-extended row (LEFT / ANTI): the join qual does not apply */
	bool suppress;               /* ANTI probing a match: evaluate the join qual, emit nothing */

	__device__ __forceinline__ void begin_row()
	{
		k0 = k1 = k2 = k3 = 0; knull = 0; gid = -1; vnull = 0;
	}
	__device__ __forceinline__ bool filter(bool pass) { return pass; }
	/* the join qual, in the per-match segment of a join pipeline (ExecHashJoin_guts, nodeHashjoin.c:330-420) */
	__device__ __forceinline__ bool filter_match(bool pass)
	{
		if (nullext) return true;
		jq = pass;
		return pass && !suppress;
	}
	__device__ __forceinline__ void key(int kc, uint64_t v, bool isnull)
	{
		if (isnull) { knull |= 1u << kc; return; }
		v = group_key(v, (int) ((keytypes >> (2 * kc)) & 3));
		if (kc == 0) k0 = v; else if (kc == 1) k1 = v; else if (kc == 2) k2 = v; else k3 = v;
	}
	__device__ __forceinline__ bool same2(uint64_t a0, uint64_t a1) const
	{
		return key_same(k0, a0, f8_keys(keytypes) & 1) && key_same(k1, a1, (f8_keys(keytypes) >> 2) & 1);
	}
	/* the first groups of the block's table, cached in registers: with a handful of groups (Q1 has four) a row finds its group
	 * by comparing against registers, and the shared-memory table (and its lock) is only visited for a key no lane of the warp
	 * has cached yet.  Entries mirror table slots 0 .. cn-1 exactly (slot = group id); a slot with a NULL key ends the cache. */
	int cn;
	bool usecache;
	uint32_t intmask;            /* MODE_PRIV: bit j = value slot j is an int64 sum (int4_sum): added as integers, bit for bit */
	uint64_t c00, c01, c10, c11, c20, c21, c30, c31;
	__device__ __forceinline__ void cache_refresh()
	{
		const volatile BlockTable *V = T;          /* keys of slots below n are final (written before n moved, fenced) */
		const int n = V->n;
		cn = 0;
		if (n > 0 && V->keynull[0] == 0) { c00 = V->key[0][0]; c01 = V->key[0][1]; cn = 1; }
		if (cn == 1 && n > 1 && V->keynull[1] == 0) { c10 = V->key[1][0]; c11 = V->key[1][1]; cn = 2; }
		if (cn == 2 && n > 2 && V->keynull[2] == 0) { c20 = V->key[2][0]; c21 = V->key[2][1]; cn = 3; }
		if (cn == 3 && n > 3 && V->keynull[3] == 0) { c30 = V->key[3][0]; c31 = V->key[3][1]; cn = 4; }
	}
	__device__ __forceinline__ bool group(bool live)
	{
		if (JOIN && suppress) live = false;
		if (nkeys == 0) gid = live ? 0 : -1;
		else if (nkeys <= 2 && usecache)
		{
			int g = -1;
			if (knull == 0)
			{
				if (f8_keys(keytypes) == 0)     /* no float8 key: equal bits are equal keys (a constant in a specialised kernel) */
				{
					if (cn > 0 && k0 == c00 && k1 == c01) g = 0;
					else if (cn > 1 && k0 == c10 && k1 == c11) g = 1;
					else if (cn > 2 && k0 == c20 && k1 == c21) g = 2;
					else if (cn > 3 && k0 == c30 && k1 == c31) g = 3;
				}
				else if (cn > 0 && same2(c00, c01)) g = 0;
				else if (cn > 1 && same2(c10, c11)) g = 1;
				else if (cn > 2 && same2(c20, c21)) g = 2;
				else if (cn > 3 && same2(c30, c31)) g = 3;
			}
			const bool need = live && g < 0;
			if (__any_sync(GG_FULL_MASK, need))
			{
				uint64_t k[GG_MAX_KEYS] = { k0, k1, k2, k3 };
				const int g2 = find_or_insert(T, k, knull, nkeys, keytypes, gcap, need, lane, *err);
				if (need) g = g2;
				cache_refresh();
			}
			gid = live ? g : -1;
		}
		else
		{
			uint64_t k[GG_MAX_KEYS] = { k0, k1, k2, k3 };
			gid = find_or_insert(T, k, knull, nkeys, keytypes, gcap, live, lane, *err);
		}
		if (live) npassed++;
		if (MODE == MODE_PRIV && gid >= 0)
		{
			uint32_t a = cnt_thread + (uint32_t) gid * cstride;
			sts32(a, lds32(a) + 1);
		}
		return gid >= 0;
	}
	__device__ __forceinline__ void out(int slot, double v, bool isnull)
	{
		if (MODE == MODE_PRIV)
		{
			if (slot >= nsl)
			{
				rq.add(gid, slot - nsl, v);
			}
			else if (gid >= 0)
			{
				uint32_t a = acc_thread + (uint32_t) gid * gstride + (uint32_t) slot * sstride;
				if ((intmask >> slot) & 1) sts64(a, lds64(a) + (uint64_t) __double_as_longlong(v));
				else stsf64(a, __dadd_rn(ldsf64(a), v));
			}
		}
		else
		{
			stsf64(sv + (uint32_t) (slot * 33 + lane) * 8, v);
			if (isnull) vnull |= 1u << slot;
			else if (gid >= 0) nonfinite |= !f8_finite(v);
		}
	}
};

/* the per-match segment of a join pipeline: FILTER there is the join qual */
template <class S>
struct MatchSink {
	S &s;
	__device__ __forceinline__ bool filter(bool pass) { return s.filter_match(pass); }
	__device__ __forceinline__ void key(int kc, uint64_t v, bool isnull) { s.key(kc, v, isnull); }
	__device__ __forceinline__ bool group(bool live) { return s.group(live); }
	__device__ __forceinline__ void out(int slot, double v, bool isnull) { s.out(slot, v, isnull); }
};

/* Hash node (MultiExecHash -> ExecHashTableInsert, nodeHash.c:88-176,906): KEY = join key, GROUP = claim a slot
 * once the keys are known, OUT = payload column.  A row with a NULL join key is never inserted: it cannot
 * match a strict equality operator (nodeHash.c:1070-1077). */
struct BuildSink {
	JoinTable jt;
	uint64_t k0, k1;
	uint32_t knull;
	unsigned long long *e;
	unsigned long long npassed;
	uint32_t *err;
	bool nonfinite;
	int gid;
	uint32_t vnull;
	__device__ __forceinline__ void begin_row() { k0 = k1 = 0; knull = 0; e = nullptr; }
	__device__ __forceinline__ bool filter(bool pass) { return pass; }
	__device__ __forceinline__ void key(int kc, uint64_t v, bool isnull)
	{
		if (isnull) { knull |= 1u << kc; return; }
		v = normalize_key(v, (int) ((jt.keytypes >> (2 * kc)) & 3));
		if (kc == 0) k0 = v; else k1 = v;
	}
	__device__ __forceinline__ bool group(bool live)
	{
		if (!live) return false;
		if (knull)
		{
			atomicAdd(jt.nbuilt + 1, 1ull);
			if (!jt.keepnull) return false;
		}
		const uint64_t h = join_hash(k0, k1);
		const unsigned long long hdr = GG_HT_OCCUPIED | (knull ? GG_HT_NULLKEY : 0ull) | (uint32_t) h;
		uint32_t slot = (uint32_t) (h >> 32) & jt.mask & ~1u;       /* chains start on even slots: see the probe loop */
		bool maybe_dup = false;
		for (uint32_t tries = 0; tries <= jt.mask; tries++)
		{
			unsigned long long *c = jt.ent + (size_t) slot * jt.stride;
			const unsigned long long seen = atomicCAS(c, 0ull, hdr);
			if (seen == 0ull) { e = c; break; }
			/* rows with equal keys hash alike, start at the same slot and so pass each other's entries: an equal tag on the way
			 * is the only way two equal keys can get in (the keys themselves may not be written yet, so the tag decides) */
			if ((uint32_t) seen == (uint32_t) h && !knull && !(seen & GG_HT_NULLKEY)) maybe_dup = true;
			slot = (slot + 1) & jt.mask;
		}
		if (maybe_dup) *(volatile unsigned long long *) (jt.nbuilt + 2) = 1ull;
		if (!e) { *err |= GGP_EF_TABLE_FULL; return false; }
		e[1] = k0;
		if (jt.nkeys > 1) e[2] = k1;
		npassed++;
		return true;
	}
	__device__ __forceinline__ void out(int slot, double v, bool isnull)
	{
		if (!e) return;
		if (isnull) atomicOr(e, 1ull << (32 + slot));
		else e[1 + jt.nkeys + slot] = (unsigned long long) __double_as_longlong(v);
	}
};
/* sending Motion: KEY = distribution key (cdbhash), GROUP = route (cdbhashreduce: jump consistent hash) and claim
 * a row of the destination's region, OUT = column that travels */
struct PartSink {
	MotionOut mo;
	uint32_t h;
	unsigned long long *row;
	unsigned long long nullmask;
	unsigned long long npassed;
	uint32_t *err;
	bool nonfinite;
	int gid, lane;
	uint32_t vnull;
	uint32_t win;                /* shared address of this warp's claim windows: [32] x { next free row, end } u64 */
	__device__ __forceinline__ void begin_row() { h = 0; row = nullptr; nullmask = 0; }
	__device__ __forceinline__ bool filter(bool pass) { return pass; }
	__device__ __forceinline__ void key(int kc, uint64_t v, bool isnull)
	{
		const uint32_t hk = isnull ? 0 : key_hash((int) ((mo.hashtypes >> (4 * kc)) & 15), v);
		h = cdbhash_add(h, hk, isnull);
	}
	__device__ __forceinline__ bool group(bool live)
	{
		const int dest = mo.route ? (int) ((h >> mo.shift) & (uint32_t) (mo.nsegs - 1)) : jump_consistent_hash((uint64_t) h, mo.nsegs);
		/* one atomic per destination present in the warp */
		const uint32_t peers = __match_any_sync(GG_FULL_MASK, live ? (uint32_t) dest : 0x80000000u + (uint32_t) lane);
		const int leader = __ffs(peers) - 1;
		const int cnt = __popc(peers);
		unsigned long long base = 0, base2 = 0;
		int split = cnt;                      /* rows [0, split) of the group go to base, the rest to base2 (a fresh window) */
		if (live && lane == leader)
		{
			if (mo.window == 0) base = atomicAdd(&mo.cursor[dest], (unsigned long long) cnt);
			else
			{
				const uint32_t wa = win + (uint32_t) dest * 16;
				const unsigned long long b = lds64(wa), e = lds64(wa + 8);
				base = b;
				if (b + (unsigned long long) cnt <= e) sts64(wa, b + (unsigned long long) cnt);
				else
				{
					split = (int) (e - b);
					base2 = atomicAdd(&mo.cursor[dest], (unsigned long long) mo.window);
					sts64(wa, base2 + (unsigned long long) (cnt - split));
					sts64(wa + 8, base2 + mo.window);
				}
			}
		}
		base = __shfl_sync(GG_FULL_MASK, base, leader);
		base2 = __shfl_sync(GG_FULL_MASK, base2, leader);
		split = __shfl_sync(GG_FULL_MASK, split, leader);
		if (!live) return false;
		const int rank = __popc(peers & ((1u << lane) - 1));
		const unsigned long long pos = rank < split ? base + (unsigned long long) rank : base2 + (unsigned long long) (rank - split);
		if (pos >= mo.cap) { *err |= GGP_EF_TABLE_FULL; return false; }
		row = mo.rows + ((uint64_t) dest * mo.cap + pos) * (uint64_t) mo.rowwords;
		row[0] = 0;
		npassed++;
		return true;
	}
	__device__ __forceinline__ void out(int slot, double v, bool isnull)
	{
		if (!row) return;
		if (isnull) { nullmask |= 1ull << slot; row[0] = nullmask; row[1 + slot] = 0; }
		else row[1 + slot] = (unsigned long long) __double_as_longlong(v);
	}
};
/* the probe of a join with a target list (gg_joinrows_create): PartSink's row claim and output into one destination (claim
 * windows, dead marking at the end), plus what the probe loop asks of a join sink.  KEY = join key (first program piece);
 * in the per-match piece FILTER = the join qual, GROUP = claim a row, OUT = target column.  The row's NULL mask follows the
 * null-extended side: its columns evaluate to NULL. */
struct JoinRowSink : PartSink {
	uint32_t keytypes;
	uint64_t k0, k1;
	uint32_t knull;
	bool jq, nullext, suppress;
	__device__ __forceinline__ void begin_row() { PartSink::begin_row(); k0 = k1 = 0; knull = 0; }
	__device__ __forceinline__ bool filter_match(bool pass)
	{
		if (nullext) return true;
		jq = pass;
		return pass && !suppress;
	}
	__device__ __forceinline__ void key(int kc, uint64_t v, bool isnull)
	{
		if (isnull) { knull |= 1u << kc; return; }
		v = group_key(v, (int) ((keytypes >> (2 * kc)) & 3));
		if (kc == 0) k0 = v; else k1 = v;
	}
	/* ANTI probing a match: the join qual was evaluated, no row is written */
	__device__ __forceinline__ bool group(bool live) { return PartSink::group(live && !suppress); }
};
/* general HashAggregate: KEY = grouping key, GROUP = find or insert the group's slot, OUT = advance one transition value */
struct HashSink {
	HashAggTable ha;
	uint32_t keytypes;
	uint64_t k0, k1, k2, k3;
	uint32_t knull;
	long long e;                 /* slot of this row's group, -1 = none */
	unsigned long long npassed;
	uint32_t *err;
	bool nonfinite, jq, nullext, suppress;
	int gid, lane;
	uint32_t vnull;
	__device__ __forceinline__ void begin_row() { k0 = k1 = k2 = k3 = 0; knull = 0; e = -1; }
	__device__ __forceinline__ bool filter(bool pass) { return pass; }
	__device__ __forceinline__ bool filter_match(bool pass)
	{
		if (nullext) return true;
		jq = pass;
		return pass && !suppress;
	}
	__device__ __forceinline__ void key(int kc, uint64_t v, bool isnull)
	{
		if (isnull) { knull |= 1u << kc; return; }
		v = group_key(v, (int) ((keytypes >> (2 * kc)) & 3));
		if (kc == 0) k0 = v; else if (kc == 1) k1 = v; else if (kc == 2) k2 = v; else k3 = v;
	}
	__device__ __forceinline__ bool group(bool live)
	{
		if (suppress) live = false;
		if (!live) return false;
		npassed++;
		/* hashed normalised (both zeros alike), compared with key_same; the entry keeps the inserting row's key */
		const int t0 = (int) (keytypes & 3), t1 = (int) ((keytypes >> 2) & 3), t2 = (int) ((keytypes >> 4) & 3), t3 = (int) ((keytypes >> 6) & 3);
		uint64_t h = join_hash(normalize_key(k0, t0) ^ (normalize_key(k2, t2) * 0xD6E8FEB86659FD93ull),
		                       normalize_key(k1, t1) ^ (normalize_key(k3, t3) * 0xA0761D6478BD642Full) ^ ((uint64_t) knull << 56));
		const unsigned long long ready = 0x8000000000000000ull | ((unsigned long long) knull << 32) | (uint32_t) h;
		uint64_t slot = (h >> 32) & (ha.cap - 1);
		/* a probe sequence this long means the table is overloaded: report it full so that the host rebuilds it larger */
		const uint64_t maxtries = ha.cap < 256 ? ha.cap : 256;
		for (uint64_t tries = 0; tries < maxtries; )
		{
			unsigned long long *ep = ha.ent + slot * ha.stride;
			volatile unsigned long long *hp = ep;
			unsigned long long cur = *hp;
			if (cur == 0)
			{
				if (atomicCAS(ep, 0ull, GG_HA_LOCKED) == 0ull)
				{
					if (ha.nkeys > 0) ep[1] = k0;                /* plain aggregation has no key words: [1] is the row count */
					if (ha.nkeys > 1) ep[2] = k1;
					if (ha.nkeys > 2) ep[3] = k2;
					if (ha.nkeys > 3) ep[4] = k3;
					__threadfence();
					*hp = ready;
					e = (long long) slot;
					break;
				}
				continue;                           /* somebody else took it: look again */
			}
			if (cur == GG_HA_LOCKED) continue;        /* being written: look again */
			if (cur == ready)
			{
				const volatile unsigned long long *kp = ep + 1;
				if ((ha.nkeys < 1 || key_same(kp[0], k0, t0 == 2)) && (ha.nkeys < 2 || key_same(kp[1], k1, t1 == 2)) &&
				    (ha.nkeys < 3 || key_same(kp[2], k2, t2 == 2)) && (ha.nkeys < 4 || key_same(kp[3], k3, t3 == 2)))
				{ e = (long long) slot; break; }
			}
			slot = (slot + 1) & (ha.cap - 1);
			tries++;
		}
		if (e < 0) { *err |= GGP_EF_TABLE_FULL; return false; }
		atomicAdd(ha.ent + (uint64_t) e * ha.stride + ha.off_cnt, 1ull);
		return true;
	}
	__device__ __forceinline__ void out(int slot, double v, bool isnull)
	{
		if (e < 0 || isnull) return;
		unsigned long long *ep = ha.ent + (uint64_t) e * ha.stride;
		if (slot >= ha.nacc)
		{
			atomicAdd((double *) (ep + ha.off_sq + ha.sqcol[slot]), v);
			return;
		}
		unsigned long long *ap = ep + ha.off_acc + slot;
		const int kind = ha.acckind[slot];
		if (ha.off_accn) atomicAdd(ep + ha.off_accn + slot, 1ull);
		if (kind == GGP_ACC_F8SUM) { if (!f8_finite(v)) nonfinite = true; atomicAdd((double *) ap, v); }
		else if (kind == GGP_ACC_I8SUM) atomicAdd(ap, (unsigned long long) __double_as_longlong(v));
		else if (kind == GGP_ACC_I8MIN) atomicMin((long long *) ap, __double_as_longlong(v));
		else if (kind == GGP_ACC_I8MAX) atomicMax((long long *) ap, __double_as_longlong(v));
		else if (kind == GGP_ACC_F8MIN || kind == GGP_ACC_F8MAX)
		{
			/* float8smaller / float8larger under float8_cmp_internal's order (NaN largest), float.c:964 */
			unsigned long long old = *(volatile unsigned long long *) ap;
			for (;;)
			{
				const int c = f8_cmp(v, __longlong_as_double((long long) old));
				if (kind == GGP_ACC_F8MIN ? c >= 0 : c <= 0) break;
				const unsigned long long seen = atomicCAS(ap, old, (unsigned long long) __double_as_longlong(v));
				if (seen == old) break;
				old = seen;
			}
		}
	}
};
template <int MODE, bool JOIN> struct SinkSel { typedef RowSink<MODE, JOIN> type; };
template <bool JOIN> struct SinkSel<MODE_HASH, JOIN> { typedef HashSink type; };
template <> struct SinkSel<MODE_PART, false> { typedef PartSink type; };
template <> struct SinkSel<MODE_PART, true> { typedef JoinRowSink type; };
template <bool JOIN> struct SinkSel<MODE_BUILD, JOIN> { typedef BuildSink type; };

/* Line pointer -> tuple: ItemId decode, the sanity rules of PageAddItem, the visibility fast path, header checks.
 * Returns whether the lane holds a visible tuple; dead lanes get a harmless view (the page header). */
__device__ __forceinline__ bool heap_tuple_front(uint32_t pg, int idx, int nitems, uint32_t pd_upper, uint32_t pd_special,
                                                 bool all_visible, bool with_mvcc, const uint32_t *snap, uint32_t &tup, uint32_t &tuplen, bool &hasnulls, uint32_t &err)
{
	bool live = false;
	tup = pg; tuplen = 64;
	if (idx < nitems)
	{
		/* ItemIdData: lp_off:15 | lp_flags:2 | lp_len:15 (itemid.h:24-29) */
		const uint32_t lp = lds32(pg + GG_PAGE_HEADER_SIZE + idx * 4);
		const uint32_t lp_off = lp & 0x7FFF, lp_flags = (lp >> 15) & 3, lp_len = lp >> 17;
		if (lp_flags == GG_LP_NORMAL)
		{
			if (lp_off < pd_upper || lp_off + lp_len > pd_special || lp_len < GG_HEAP_HDR_SIZE + 1 || (lp_off & 7))
				err |= GGP_EF_BADPAGE;
			else
			{
				tup = pg + lp_off;
				tuplen = lp_len;
				live = true;
			}
		}
	}
	/* t_infomask2 | t_infomask | t_hoff live in bytes 18..22 of the header (htup_details.h:139-162) */
	const uint32_t hw = lds32(tup + 20);                 /* infomask (lo 16) | t_hoff (byte 2) */
	const uint32_t infomask = hw & 0xFFFF, hoff = (hw >> 16) & 0xFF;
	if (live && !all_visible)
	{
		/* HeapTupleSatisfiesMVCC fast path (tqual.c:1009,1119): frozen xmin + invalid xmax */
		if ((infomask & GG_HEAP_XMIN_FROZEN) == GG_HEAP_XMIN_FROZEN && (infomask & GG_HEAP_XMAX_INVALID)) { }
		else if ((infomask & GG_HEAP_XMIN_INVALID) && !(infomask & GG_HEAP_XMIN_COMMITTED)) live = false;
		/* the full rule, against the scan's snapshot — in the kernels built with it (PL::mvcc: the interpreter kernels, and the
		 * specialised ones of a pipeline whose engine has a snapshot); elsewhere the branch folds away */
		else if (with_mvcc && snap) live = heap_tuple_satisfies_mvcc(tup, infomask, snap, err);
		else { err |= GGP_EF_VISIBILITY; live = false; }
	}
	if (live && (hoff > tuplen || (hoff & 7) || hoff < 24)) { err |= GGP_EF_BADPAGE; live = false; }
	hasnulls = live && (infomask & GG_HEAP_HASNULL);
	return live;
}

/* How the kernel reaches the plan.  DynPlan interprets the program table it receives as a kernel
 * parameter; a plan-specialised translation unit (gg_jit.cpp) defines a StaticPlan whose run()/walk()
 * are the same exec_op()/walk_step() calls with literal arguments, so they fold at compile time. */
struct DynPlan {
	__device__ static __forceinline__ int nkeys(const ggp_program &P) { return P.nkeys; }
	__device__ static __forceinline__ int nslots(const ggp_program &P) { return P.nslots; }
	__device__ static __forceinline__ int nacc(const ggp_program &P) { return P.nacc; }
	__device__ static __forceinline__ int ncols(const ggp_program &P) { return P.outer.ncols; }
	__device__ static __forceinline__ int rowwords(const ggp_program &P) { return P.outer.rowwords; }
	__device__ static __forceinline__ int regslots(const ggp_program &) { return 0; }       /* interpreter: dynamic slot numbers */
	__device__ static __forceinline__ bool mvcc(const ggp_program &) { return true; }        /* interpreter: every rule built in */
	__device__ static __forceinline__ uint32_t intmask(const ggp_program &P)
	{
		uint32_t m = 0;
		for (int j = 0; j < P.nacc; j++) if (P.acckind[j] == GGP_ACC_I8SUM) m |= 1u << j;
		return m;
	}
	__device__ static __forceinline__ uint32_t keytypes(const ggp_program &P)
	{
		return (uint32_t) P.keytype[0] | ((uint32_t) P.keytype[1] << 2) | ((uint32_t) P.keytype[2] << 4) | ((uint32_t) P.keytype[3] << 6);
	}
	template <bool NULLABLE, class Sink>
	__device__ static __forceinline__ void run(const EvalCtx &X, bool live, uint32_t &err, Sink &sink)
	{
		run_prog<NULLABLE, false>(X, live, err, sink);
	}
	template <bool NULLABLE, class Sink>
	__device__ static __forceinline__ void run_range(const EvalCtx &X, MachState &M, int pc0, int pc1, uint32_t &err, Sink &sink)
	{
		ggd::run_range<NULLABLE, true>(X, M, pc0, pc1, err, sink);
	}
	__device__ static __forceinline__ void walk(const ggp_program &P, uint32_t tup, uint32_t tuplen, bool fast,
	                                            uint32_t offs, int lane, TupleView &tv, uint32_t &err)
	{
		walk_tuple(P.outer, tup, tuplen, fast, offs, lane, tv, err);
	}
};

template <int MODE, class PL, bool JOIN = false>
__device__ __forceinline__ void scanagg_body(const ggp_program &P, const ScanAggParams &prm)
{
	constexpr bool NULLABLE = (MODE == MODE_TRN || MODE == MODE_BUILD || MODE == MODE_PART || MODE == MODE_HASH);
	constexpr bool TRMODE = (MODE == MODE_TR || MODE == MODE_TRN);
	extern __shared__ __align__(128) uint8_t smem[];
	const int nstage = prm.nstage;
	const int ncons = (blockDim.x >> 5) - 1;          /* consumer warps; the last warp is the producer */
	const int NT = ncons * 32;                         /* consumer threads */
	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

	const uint32_t smem_base = smem_u32(smem);
	const uint32_t ring = smem_base;
	const uint32_t full_bar = ring + (uint32_t) nstage * GG_BLCKSZ;
	const uint32_t empty_bar = full_bar + (uint32_t) nstage * 8;
	BlockTable *T = (BlockTable *) (smem + (size_t) nstage * GG_BLCKSZ + (size_t) nstage * 16);

	const int nkeys = PL::nkeys(P);
	const int nslots = PL::nslots(P);
	const int nacc = PL::nacc(P);
	const int ncols = PL::ncols(P);
	const int V = nslots > 0 ? nslots : 1;
	const int gcap = prm.gcap;
	const int nreg = (MODE == MODE_PRIV) ? PL::regslots(P) : 0;      /* trailing value slots kept in registers */
	const int nsl = nslots - nreg;                                    /* value slots kept in shared memory */

	if (threadIdx.x == 0)
	{
		for (int s = 0; s < nstage; s++)
		{
			mbar_init(full_bar + s * 8, 1);
			mbar_init(empty_bar + s * 8, prm.team > 0 ? prm.team : ncons);
		}
		if (prm.team > 0)
			for (int i = 0; i < GG_MAX_TEAMS * GG_MAX_STAGES; i++) mbar_init(smem_u32(&T->teamfull[i]), 1);
		T->n = (nkeys == 0) ? 1 : 0;               /* plain aggregation: the single group always exists */
		T->lock = 0;
		if (nkeys == 0) { T->keynull[0] = 0; for (int c = 0; c < GG_MAX_KEYS; c++) T->key[0][c] = 0; }
		mbar_fence_init();
	}
	if (MODE == MODE_PRIV && warp < ncons)
	{
		/* zero this thread's private accumulators: integer sums 0, float8 sums -0 (RegAcc::zero) */
		for (int g = 0; g < gcap; g++)
		{
			sts32(smem_base + prm.cnt_off + (uint32_t) (g * NT + (int) threadIdx.x) * 4, 0);
			for (int s = 0; s < nsl; s++)
				sts64(smem_base + prm.acc_off + (uint32_t) ((g * nsl + s) * NT + (int) threadIdx.x) * 8,
				      ((PL::intmask(P) >> s) & 1) ? 0ull : GG_F8_NEGZERO_BITS);
		}
	}
	__syncthreads();

	/* input format: heap pages, or 32 KB chunks of fixed-width datum rows (what a receiving Motion delivers) */
	/* HJ_FILL_INNER_TUPLES of a right / full join: the input of this launch is the hash table itself, scanned as rows
	 * of `stride` words */
	const bool fill_inner = JOIN && prm.fill_inner != 0;
	const uint32_t rowwords = fill_inner ? prm.jt.stride : (uint32_t) PL::rowwords(P);
	const uint32_t rowbytes = rowwords * 8;
	const uint32_t rows_per_chunk = rowwords ? ((GG_BLCKSZ / rowbytes) & ~1u) : 0;
	const uint32_t chunk_bytes = rowwords ? rows_per_chunk * rowbytes : GG_BLCKSZ;

	/* pages of this block: blockIdx.x, +gridDim.x, ... */
	const uint64_t first = blockIdx.x, stride = gridDim.x;
	/* column files: a block takes the contiguous run of units [aocs_u0, aocs_u0 + npages) — consecutive rows, so the producer
	 * walks each column's block directory forwards instead of looking every unit up */
	const uint64_t aocs_per = (prm.nblocks + stride - 1) / stride;
	const uint64_t aocs_u0 = first * aocs_per;
	/* column files feed SeqScan -> Agg pipelines over a datum-row descriptor: folds away in join kernels and in kernels specialised
	 * for a heap plan */
	const bool aocs_feed = !JOIN && MODE != MODE_BUILD && MODE != MODE_PART && PL::rowwords(P) != 0 && prm.aocs_tile_rows > 0;
	const uint32_t npages = aocs_feed
		? (uint32_t) (aocs_u0 < prm.nblocks ? (prm.nblocks - aocs_u0 < aocs_per ? prm.nblocks - aocs_u0 : aocs_per) : 0)
		: (uint32_t) (first < prm.nblocks ? (prm.nblocks - first + stride - 1) / stride : 0);

	/* MODE_TR accumulators: round r of this lane owns pair p = r*32+lane -> (g = p / V, slot = p % V) */
	double acc_sum[TRMODE ? GG_NROUNDS : 1];
	uint32_t acc_cnt[TRMODE ? GG_NROUNDS : 1], acc_n[TRMODE ? GG_NROUNDS : 1];
	int pair_g[TRMODE ? GG_NROUNDS : 1], pair_j[TRMODE ? GG_NROUNDS : 1], pair_kind[TRMODE ? GG_NROUNDS : 1];
	if (TRMODE)
	{
#pragma unroll
		for (int r = 0; r < GG_NROUNDS; r++)
		{
			int p = r * 32 + lane;
			pair_g[r] = p / V;
			pair_j[r] = p % V;
			pair_kind[r] = nacc == 0 ? GGP_ACC_COUNT : (pair_j[r] < nacc ? P.acckind[pair_j[r]] : GGP_ACC_F8SUM);
			acc_sum[r] = pair_kind[r] == GGP_ACC_F8SUM ? -0.0 : 0.0; acc_cnt[r] = 0; acc_n[r] = 0;
		}
	}
	uint32_t err = 0;
	unsigned long long n_scanned = 0, n_passed = 0;
	RegAcc rq_keep;                                   /* MODE_PRIV: the thread's register-resident accumulators, for the epilogue */
	rq_keep.zero();

	if (warp == ncons)
	{
		/* ===== producer: one elected lane streams pages through the ring ===== */
		if (aocs_feed)
		{
			/* Column files (aocs_getnext, aocsam.c:661): lane sl owns projected column sl.  It keeps its place in the column's
			 * block directory (block b, row j inside it) across the block's consecutive units; per unit it finds the byte range
			 * of the unit's values in the file (values of a block are packed: data_off + row * stride; the range may run over
			 * block ends, the headers in between are copied along), publishes where each run of rows landed (GG_AOCS_META_*
			 * at the head of the slot) and bulk-copies the range.  A column whose unit cannot be staged this way — NULL
			 * bitmaps, values without a common stride, more than four blocks, a misaligned file, no room left in the slot —
			 * is flagged and read by the consumers row by row through gg_aocs_fetch. */
			const int UR = prm.aocs_unit_rows;
			const bool active = lane < ncols;
			const gg_aocs_devcol *cd = prm.aocs + (active ? P.outer.colatt[lane] : 0);
			const int kind = active ? cd->kind : 0;
			const uint32_t valign = kind == GG_AOCS_K_W8 ? 7u : kind == GG_AOCS_K_I4 ? 3u : kind == GG_AOCS_K_I2 ? 1u : 0u;
			const bool misaligned = (((unsigned long long) cd->file) & 15ull) != 0;
			int64_t b = 0, nb = active ? cd->nblocks : 0;
			int32_t j = 0;
			gg_aocs_block blk;
			blk.first_row = 0; blk.data_off = 0; blk.null_off = -1; blk.nrows = 0; blk.data_len = 0; blk.stride = 0; blk.pad = 0;
			if (active && npages > 0)
			{
				const uint64_t row0 = aocs_u0 * (uint64_t) UR;
				const uint64_t tile = row0 / (uint64_t) prm.aocs_tile_rows;
				const gg_aocs_tile t = cd->tiles[tile];
				int64_t jj = (int64_t) t.row_in_block + (int64_t) (row0 - tile * (uint64_t) prm.aocs_tile_rows);
				b = t.block;
				while (b < nb) { blk = cd->dir[b]; if (jj < blk.nrows) break; jj -= blk.nrows; b++; }
				j = (int32_t) jj;
			}
			int s = 0;
			uint32_t ph = 0;
			for (uint32_t it = 0; it < npages; it++)
			{
				if (lane == 0) mbar_wait(empty_bar + s * 8, ph ^ 1, 128);
				__syncwarp();
				const uint32_t slot = ring + (uint32_t) s * GG_BLCKSZ;
				const uint64_t left = prm.nrows - (aocs_u0 + it) * (uint64_t) UR;
				const int nitems = (int) (left < (uint64_t) UR ? left : (uint64_t) UR);
				uint32_t nbytes = 0;
				bool slow = misaligned;
				int64_t a0 = 0;
				if (active)
				{
					const uint32_t meta = slot + (uint32_t) lane * GG_AOCS_META_BYTES;
					int rem = nitems, nseg = 0;
					int64_t end_off = 0;
					while (rem > 0)
					{
						if (b >= nb) { slow = true; break; }
						const int take = rem < blk.nrows - j ? rem : blk.nrows - j;
						const int64_t off = blk.data_off + (int64_t) j * blk.stride;
						if (blk.null_off >= 0 || blk.stride <= 0 || blk.stride > 0xFFFF || ((off | (int64_t) blk.stride) & valign)) slow = true;
						if (nseg == 0) a0 = off & ~(int64_t) 15;
						if (nseg < 4)
						{
							sts32(meta + GG_AOCS_META_CUM + (uint32_t) nseg * 4, (uint32_t) (nitems - rem + take));
							sts32(meta + GG_AOCS_META_REL + (uint32_t) nseg * 4, (uint32_t) (off - a0));
							sts16(meta + GG_AOCS_META_STRIDE + (uint32_t) nseg * 2, (uint32_t) blk.stride);
						}
						else slow = true;
						nseg++;
						end_off = off + (int64_t) take * blk.stride;
						rem -= take; j += take;
						if (j >= blk.nrows) { b++; j = 0; if (b < nb) blk = cd->dir[b]; }
					}
					for (; nseg < 4; nseg++)
					{
						sts32(meta + GG_AOCS_META_CUM + (uint32_t) nseg * 4, 0xFFFFFFFFu);
						sts32(meta + GG_AOCS_META_REL + (uint32_t) nseg * 4, 0);
						sts16(meta + GG_AOCS_META_STRIDE + (uint32_t) nseg * 2, 0);
					}
					if (!slow && end_off - a0 > (int64_t) (GG_BLCKSZ - GG_AOCS_DATA_OFF)) slow = true;
					if (!slow) nbytes = (uint32_t) (((end_off + 15) & ~(int64_t) 15) - a0);
				}
				/* the columns' ranges one after the other in the slot's data area */
				uint32_t at = nbytes;
				for (int o = 1; o < 32; o <<= 1)
				{
					const uint32_t up = __shfl_up_sync(GG_FULL_MASK, at, o);
					if (lane >= o) at += up;
				}
				at -= nbytes;
				if (at + nbytes > (uint32_t) (GG_BLCKSZ - GG_AOCS_DATA_OFF)) { slow = true; nbytes = 0; }
				uint32_t total = nbytes;
				for (int o = 16; o > 0; o >>= 1) total += __shfl_xor_sync(GG_FULL_MASK, total, o);
				if (active)
				{
					const uint32_t meta = slot + (uint32_t) lane * GG_AOCS_META_BYTES;
					sts32(meta + GG_AOCS_META_FLAGS, (slow ? GG_AOCS_META_SLOW : 0u) | ((uint32_t) kind << 8));
					sts32(meta + GG_AOCS_META_BASE, slot + GG_AOCS_DATA_OFF + at);
				}
				__syncwarp();
				if (lane == 0) mbar_arrive_expect_tx(full_bar + s * 8, total);
				__syncwarp();
				if (nbytes) tma_load_1d(slot + GG_AOCS_DATA_OFF + at, cd->file + a0, nbytes, full_bar + s * 8);
				if (++s == nstage) { s = 0; ph ^= 1; }
			}
		}
		else if (lane == 0)
		{
			int s = 0;
			uint32_t ph = 0;
			const uint8_t *src = prm.pages + first * (uint64_t) chunk_bytes;
			/* teams: page `it` is team (it mod nteams)'s; its arrival is signalled on that team's barrier tq = (it / nteams) mod nstage */
			const int pnteams = prm.team > 0 ? ncons / prm.team : 1;
			int tm = 0, tq = 0;
			for (uint32_t it = 0; it < npages; it++)
			{
				mbar_wait(empty_bar + s * 8, ph ^ 1, 128);
				/* datum rows: the last chunk is short; bulk copies move multiples of 16 bytes */
				uint32_t nbytes = chunk_bytes;
				if (rowwords && first + (uint64_t) it * stride == prm.nblocks - 1)
					nbytes = (uint32_t) (((prm.nrows - (prm.nblocks - 1) * (uint64_t) rows_per_chunk) * rowbytes + 15) & ~15ull);
				const uint32_t fb = prm.team > 0 ? smem_u32(&T->teamfull[tm * GG_MAX_STAGES + tq]) : full_bar + s * 8;
				mbar_arrive_expect_tx(fb, nbytes);
				tma_load_1d(ring + (uint32_t) s * GG_BLCKSZ, src, nbytes, fb);
				src += stride * (uint64_t) chunk_bytes;
				if (++s == nstage) { s = 0; ph ^= 1; }
				if (++tm == pnteams) { tm = 0; if (++tq == nstage) tq = 0; }
			}
		}
	}
	else
	{
		/* ===== consumers ===== */
		const uint32_t myscr = smem_base + prm.scratch_off + (uint32_t) warp * prm.scratch_per_warp;
		const uint32_t offs = myscr;                                               /* [ncols][32] u16 */
		const uint32_t sv = myscr + ((ncols * 64 + 15) & ~15);             /* TR: [V][33] f64 */
		const uint32_t sg = sv + (uint32_t) V * 33 * 8;                            /* TR: [32] i32 group of each tuple, -1 = none */
		const uint32_t snull = sg + 128;                                           /* TR: [32] u32 bit s: value slot s is NULL */

		EvalCtx X;
		X.P = &P; X.offs = offs; X.lane = lane;
		X.ipay = (const uint64_t *) prm.jt.ent; X.ipaynull = 0;
		typename SinkSel<MODE, JOIN>::type sink;
		sink.err = &err; sink.npassed = 0; sink.nonfinite = false; sink.gid = -1; sink.vnull = 0;
		if constexpr (MODE == MODE_BUILD)
			sink.jt = prm.jt;
		else if constexpr (MODE == MODE_PART)
		{
			sink.mo = prm.mo; sink.lane = lane;
			sink.win = sv;                       /* the per-warp scratch behind the column offsets */
			sts64(sv + (uint32_t) lane * 16, 0); sts64(sv + (uint32_t) lane * 16 + 8, 0);
			__syncwarp();
			if constexpr (JOIN) { sink.keytypes = PL::keytypes(P); sink.jq = false; sink.nullext = false; sink.suppress = false; }
		}
		else if constexpr (MODE == MODE_HASH)
		{
			sink.ha = prm.ha; sink.keytypes = PL::keytypes(P); sink.lane = lane;
			sink.jq = false; sink.nullext = false; sink.suppress = false;
		}
		else
		{
			sink.keytypes = PL::keytypes(P); sink.T = T; sink.nkeys = nkeys; sink.gcap = gcap; sink.lane = lane;
			sink.acc_thread = smem_base + prm.acc_off + threadIdx.x * 8;
			sink.cnt_thread = smem_base + prm.cnt_off + threadIdx.x * 4;
			sink.sstride = (uint32_t) NT * 8;
			sink.gstride = (uint32_t) nsl * NT * 8;
			sink.nsl = nsl; sink.nreg = nreg;
			sink.rq.zero();
			sink.cstride = (uint32_t) NT * 4;
			sink.cn = 0; sink.c00 = sink.c01 = sink.c10 = sink.c11 = sink.c20 = sink.c21 = sink.c30 = sink.c31 = 0;
			sink.usecache = prm.nokeycache == 0;
			sink.intmask = MODE == MODE_PRIV ? PL::intmask(P) : 0;
			sink.sv = sv;
			sink.jq = false; sink.nullext = false; sink.suppress = false;
		}

		/* Which warp works on which chunk (32 line pointers) of which page:
		 *   teams (prm.team = TS > 0)  the consumer warps form ncons / TS teams; page `it` of this block belongs to team
		 *       it mod nteams, whose warp j takes chunks j, j + TS, ...  A warp visits only its team's pages (header decode,
		 *       barrier wait and release cost nothing on the others), and the teams work on different pages of the ring
		 *       concurrently.  The host picks TS from the page density (6 chunks per page -> teams of 6).
		 *   dealt (prm.team = 0)  every warp visits every page; chunk c of a page goes to warp (dealt + c) mod ncons, dealt =
		 *       chunks of all earlier pages, so consecutive pages land on disjoint warp sets. */
		const int TS = prm.team > 0 ? prm.team : ncons;
		const int nteams = prm.team > 0 ? ncons / TS : 1;
		const int team = prm.team > 0 ? warp / TS : 0;
		const int tw = prm.team > 0 ? warp - team * TS : warp;
		int s = team, dealt = 0;
		uint32_t ph = 0;
		while (s >= nstage) { s -= nstage; ph ^= 1; }
		/* teams: `dealt` counts which of the team's own barriers the next page arrives on and `ph` is that barrier's phase (a team
		 * never waits on the slots' barriers, and it deals nothing: the two modes share the registers) */
		for (uint32_t it = (uint32_t) team; it < npages && team < nteams; it += (uint32_t) nteams)
		{
			const bool aocs = aocs_feed;
			{
				if (lane == 0)
				{
					/* a team waits on its own barrier set (BlockTable::teamfull): exact, it has seen every earlier phase itself */
					if (prm.team > 0) mbar_wait(smem_u32(&T->teamfull[team * GG_MAX_STAGES + dealt]), ph, 20);
					else mbar_wait(full_bar + s * 8, ph, 20);
				}
				__syncwarp();
			}
			const uint32_t pg = ring + (uint32_t) s * GG_BLCKSZ;

			/* page header, bufpage.h:153-166; sanity rules of PageAddItem (bufpage.c:196-204) */
			const uint32_t w2 = aocs ? 0 : lds32(pg + 8), w3 = aocs ? 0 : lds32(pg + 12), w4 = aocs ? 0 : lds32(pg + 16);
			const uint32_t pd_flags = w2 >> 16, pd_lower = w3 & 0xFFFF, pd_upper = w3 >> 16, pd_special = w4 & 0xFFFF;
			int nitems = 0;
			if (aocs)
			{
				const uint64_t left = prm.nrows - (aocs_u0 + it) * (uint64_t) prm.aocs_unit_rows;
				nitems = (int) (left < (uint64_t) prm.aocs_unit_rows ? left : (uint64_t) prm.aocs_unit_rows);
			}
			else if (rowwords)
			{
				const uint64_t chunk = first + (uint64_t) it * stride;
				const uint64_t left = prm.nrows - chunk * rows_per_chunk;
				nitems = (int) (left < rows_per_chunk ? left : rows_per_chunk);
			}
			else if (pd_lower < GG_PAGE_HEADER_SIZE || pd_lower > pd_upper || pd_upper > pd_special || pd_special > GG_BLCKSZ)
			{
				/* an all-zero page is a valid empty page (PageIsNew) */
				if (pd_upper != 0 || pd_lower != 0) err |= GGP_EF_BADPAGE;
			}
			else
				nitems = (int) ((pd_lower - GG_PAGE_HEADER_SIZE) >> 2);
			const bool all_visible = (pd_flags & GG_PD_ALL_VISIBLE) != 0;     /* heapam.c:391 */
			const int nchunks = (nitems + 31) >> 5;

			int c0 = tw;
			if (prm.team == 0)
			{
				c0 = warp - dealt;
				if (c0 < 0) c0 += ncons;
				dealt += nchunks;
				while (dealt >= ncons) dealt -= ncons;          /* nchunks <= 37: a handful of subtractions beats a division */
			}
			for (int c = c0; c < nchunks; c += TS)
			{
				const int idx = c * 32 + lane;
				bool live = false;
				uint32_t tup = pg, tuplen = 64;
				unsigned long long fill_hdr = 0;
				if (JOIN && fill_inner)
				{
					/* a table entry: emitted iff occupied and never matched; the outer side is all NULL */
					live = idx < nitems;
					const uint32_t rp = pg + (live ? (uint32_t) idx * rowbytes : 0);
					fill_hdr = lds64(rp);
					live = live && (fill_hdr & GG_HT_OCCUPIED) && !(fill_hdr & GG_HT_MATCHED);
					X.fast = true;
					X.tv.tp = pg;
					X.tv.colnull = 0xFFFFFFFFu;
				}
				else if (rowwords)
				{
					/* datum row: NULL mask word, then one word per column at constant offsets */
					live = idx < nitems;
					uint32_t rp = pg + (live ? (uint32_t) idx * rowbytes : 0);
					if (aocs)
					{
						/* the row is assembled here, from the column files: an odd word stride keeps the lanes on distinct banks */
						rp = myscr + (uint32_t) prm.scratch_per_warp - (32u - (uint32_t) lane) * ((rowwords | 1u) * 8);      /* the tail of the warp's scratch */
						/* The producer has copied the unit's values of every projected column into this slot and says where each run
						 * of rows landed; a lane picks its row's run and loads the value from shared memory.  A column the producer
						 * could not stage (NULL bitmaps, no common stride, ...) goes through the general per-row walk over the file in
						 * device memory (gg_aocs_fetch, the function the CPU tests run over the reference-written files). */
						uint64_t m = 0;
						uint32_t aerr = 0;
						for (int sl = 0; sl < ncols; sl++)
						{
							const int a = P.outer.colatt[sl];
							const uint32_t meta = pg + (uint32_t) sl * GG_AOCS_META_BYTES;
							const uint32_t flags = lds32(meta + GG_AOCS_META_FLAGS);
							if (!live) continue;
							uint64_t w = 0;
							int isn = 0;
							uint32_t rc;
							if (flags & GG_AOCS_META_SLOW)
							{
								const uint64_t row = (aocs_u0 + it) * (uint64_t) prm.aocs_unit_rows + (uint64_t) idx;
								const uint64_t tile = row / (uint64_t) prm.aocs_tile_rows;
								rc = gg_aocs_fetch(prm.aocs + a, (int64_t) tile, (int32_t) (row - tile * (uint64_t) prm.aocs_tile_rows), &w, &isn);
							}
							else
							{
								const uint4 cum = lds128(meta + GG_AOCS_META_CUM), rel = lds128(meta + GG_AOCS_META_REL);
								const uint64_t st4 = lds64(meta + GG_AOCS_META_STRIDE);
								const uint32_t r = (uint32_t) idx;
								const int k = (r >= cum.x) + (r >= cum.y) + (r >= cum.z);
								const uint32_t prev = k == 0 ? 0u : k == 1 ? cum.x : k == 2 ? cum.y : cum.z;
								const uint32_t relk = k == 0 ? rel.x : k == 1 ? rel.y : k == 2 ? rel.z : rel.w;
								const uint32_t stk = (uint32_t) (st4 >> (16 * k)) & 0xFFFFu;
								rc = aocs_value_smem((int) (flags >> 8) & 0xFF, lds32(meta + GG_AOCS_META_BASE) + relk + (r - prev) * stk, w);
							}
							aerr |= rc;
							if (rc || isn) { w = 0; m |= 1ull << a; }
							sts64(rp + 8 + (uint32_t) a * 8, w);
						}
						if (aerr & GG_AOCS_E_RANGE) err |= GGP_EF_BADPAGE;
						if (aerr & GG_AOCS_E_IRREGULAR) err |= GGP_EF_STRING_TOO_LONG;
						if (aerr) live = false;
						sts64(rp, m);
					}
					X.fast = true;
					X.tv.tp = rp + 8;
					X.tv.colnull = 0;
					const uint64_t mask = live ? lds64(rp) : 0;
					if (mask & GG_ROW_DEAD) live = false;      /* claimed by a sending Motion and never filled */
					if (live)
					{
						n_scanned++;
						uint32_t cn = 0;
						for (int sl = 0; sl < ncols; sl++) cn |= (uint32_t) ((mask >> P.outer.colatt[sl]) & 1) << sl;
						X.tv.colnull = cn;
						if (!NULLABLE && cn) { err |= GGP_EF_NOTNULL_VIOLATED; live = false; }
					}
				}
				else
				{
				bool hasnulls;
				live = heap_tuple_front(pg, idx, nitems, pd_upper, pd_special, all_visible, PL::mvcc(P), prm.snap, tup, tuplen, hasnulls, err);
				const bool fast = !__any_sync(GG_FULL_MASK, hasnulls);
				X.fast = fast;
				X.tv.tp = pg;
				X.tv.colnull = 0;
				if (live)
				{
					n_scanned++;
					const uint32_t e0 = err;
					PL::walk(P, tup, tuplen, fast, offs, lane, X.tv, err);
					if (err != e0 && (err & GGP_EF_BADPAGE)) live = false;
					if (!NULLABLE && X.tv.colnull) { err |= GGP_EF_NOTNULL_VIOLATED; live = false; }
				}
				if (!live)
				{
					/* offsets of walked columns must be readable: point them at offset 0 */
					X.tv.tp = pg;
					for (int sl = 0; sl < ncols; sl++) sts16(offs + (uint32_t) (sl * 32 + lane) * 2, 0);
					X.fast = false;
				}
				/* X.fast must be warp-uniform only in the sense that every lane reads valid memory:
				 * a dead lane with fast=false reads offset 0 of the page, which is always mapped */
				}

				/* ---- lane-owns-(group, slot) accumulate of the 32 rows the warp just evaluated ---- */
				auto tr_accumulate = [&]()
				{

					sts32(sg + lane * 4, (uint32_t) sink.gid);
					if (NULLABLE) sts32(snull + lane * 4, sink.vnull);
					__syncwarp();

					/* ---- lane-owns-(group, slot) accumulate ---- */
					const int G = T->n;
#pragma unroll
					for (int r = 0; r < GG_NROUNDS; r++)
					{
						if (r * 32 < G * V)              /* warp-uniform */
						{
							const int g = pair_g[r], j = pair_j[r], kind = pair_kind[r];
							double s0 = acc_sum[r];
							uint32_t cnt = acc_cnt[r], nn = acc_n[r];
#pragma unroll 8
							for (int i = 0; i < 32; i++)
							{
								if ((int) lds32(sg + i * 4) == g)
								{
									cnt++;
									bool isn = NULLABLE && ((lds32(snull + i * 4) >> j) & 1);
									if (!isn && nacc > 0)
									{
										double v = ldsf64(sv + (uint32_t) (j * 33 + i) * 8);
										if (kind == GGP_ACC_F8SUM) s0 = __dadd_rn(s0, v);
										else if (kind == GGP_ACC_I8SUM)
											s0 = __longlong_as_double(__double_as_longlong(s0) + __double_as_longlong(v));
										else if (kind == GGP_ACC_F8MIN) { if (nn == 0 || f8_cmp(v, s0) < 0) s0 = v; }
										else if (kind == GGP_ACC_F8MAX) { if (nn == 0 || f8_cmp(v, s0) > 0) s0 = v; }
										else if (kind == GGP_ACC_I8MIN) { if (nn == 0 || __double_as_longlong(v) < __double_as_longlong(s0)) s0 = v; }
										else if (kind == GGP_ACC_I8MAX) { if (nn == 0 || __double_as_longlong(v) > __double_as_longlong(s0)) s0 = v; }
										nn++;
									}
								}
							}
							acc_sum[r] = s0; acc_cnt[r] = cnt; acc_n[r] = nn;
						}
					}
					__syncwarp();
				
				};

				sink.begin_row();
				if constexpr (!JOIN)
				{
					PL::template run<NULLABLE>(X, live, err, sink);
					if constexpr (TRMODE) tr_accumulate();
				}
				else if (fill_inner)
				{
					/* ExecScanHashTableForUnmatched (nodeHashjoin.c:460-490): the per-match piece runs once for the entry,
					 * outer columns NULL, the join qual not applied */
					const JoinTable &jt = prm.jt;
					const uint64_t entry = (first + (uint64_t) it * stride) * rows_per_chunk + (uint64_t) (live ? idx : 0);
					MachState M2;
					M2.reset(live);
					M2.tnull = 0xF;                           /* whatever the first piece would have kept in temporaries is NULL */
					X.ipay = (const uint64_t *) (jt.ent + entry * jt.stride + 1 + jt.nkeys);
					X.ipaynull = (uint32_t) (fill_hdr >> 32) & 0xFFu;
					sink.begin_row();
					sink.jq = false; sink.nullext = live;      /* only the lanes that hold an unmatched entry skip the join qual */
					sink.suppress = false;
					MatchSink<decltype(sink)> ms = { sink };
					PL::template run_range<NULLABLE>(X, M2, jt.probe_pc, GGP_MAX_CODE, err, ms);
					if constexpr (TRMODE) tr_accumulate();
				}
				else
				{
					/* ExecHashJoin_guts (nodeHashjoin.c:78-509): HJ_NEED_NEW_OUTER = the first program piece (outer
					 * qual + join keys); HJ_SCAN_BUCKET = the probe loop; every match runs the second piece (join
					 * qual, grouping keys, aggregate arguments) with the matched entry's payload as inner columns;
					 * HJ_FILL_OUTER_TUPLE = the null-extended run for LEFT / ANTI */
					const JoinTable &jt = prm.jt;
					const bool lasj = jt.jointype == GG_JOIN_LASJ_NOTIN;
					const bool anti = jt.jointype == GG_JOIN_ANTI || lasj;
					const bool fill_outer = jt.jointype == GG_JOIN_LEFT || jt.jointype == GG_JOIN_FULL || anti;
					const bool single = jt.jointype == GG_JOIN_SEMI || anti;
					MachState M1;
					M1.reset(live);
					const uint32_t gkt = sink.keytypes;
					sink.keytypes = jt.keytypes;
					PL::template run_range<NULLABLE>(X, M1, 0, jt.probe_pc, err, sink);
					sink.keytypes = gkt;
					/* the sink keeps a zero's sign (group_key); the hash table holds join keys normalised */
					const uint64_t jk0 = normalize_key(sink.k0, (int) (jt.keytypes & 3)), jk1 = normalize_key(sink.k1, (int) ((jt.keytypes >> 2) & 3));
					const bool jknull = sink.knull != 0;
					bool pending = M1.live && (fill_outer || !jknull);     /* a NULL key matches nothing (nodeHash.c:1070) */
					if (lasj && jknull && !jt.inner_empty) pending = false;     /* NULL NOT IN (non-empty set): dropped (nodeHashjoin.c:361) */
					bool probing = pending && !jknull;
					bool matched = false;
					const uint64_t h = join_hash(jk0, jk1);
					/* a chain starts on an even slot and the probe takes slots in pairs: with entries of 32 bytes a pair is one
					 * aligned 64-byte piece of memory, which is what HBM delivers per access anyway */
					uint32_t slot = (uint32_t) (h >> 32) & jt.mask & ~1u;
					for (;;)
					{
						bool have = false;
						unsigned long long hdr = 0;
						const unsigned long long *e = jt.ent;
						if (probing)
						{
							/* One round trip to HBM covers two probe steps: the entry at `slot` and its successor are requested
							 * together (header and first key of an entry in one 16-byte load where entries are 16-byte aligned).
							 * The 32 lanes of a warp wait for the slowest of them, so what counts is the longest chain in the warp,
							 * and with the table at most half full few chains are longer than two. */
							for (;;)
							{
								const unsigned long long *ea = jt.ent + (size_t) slot * jt.stride;
								const uint32_t slot_b = (slot + 1) & jt.mask;
								const unsigned long long *eb = jt.ent + (size_t) slot_b * jt.stride;
								unsigned long long hdr_a, ka0, hdr_b, kb0;
								if ((jt.stride & 1) == 0)
								{
									const ulonglong2 ha = __ldg((const ulonglong2 *) ea), hb = __ldg((const ulonglong2 *) eb);
									hdr_a = ha.x; ka0 = ha.y; hdr_b = hb.x; kb0 = hb.y;
								}
								else { hdr_a = __ldg(ea); ka0 = __ldg(ea + 1); hdr_b = __ldg(eb); kb0 = __ldg(eb + 1); }
								const unsigned long long ka1 = jt.nkeys > 1 ? __ldg(ea + 2) : 0ull, kb1 = jt.nkeys > 1 ? __ldg(eb + 2) : 0ull;
								e = ea; hdr = hdr_a;
								slot = slot_b;
								if (hdr_a == 0) { probing = false; break; }
								if ((uint32_t) hdr_a == (uint32_t) h && !(hdr_a & GG_HT_NULLKEY) && ka0 == jk0 && (jt.nkeys < 2 || ka1 == jk1)) { have = true; break; }
								e = eb; hdr = hdr_b;
								slot = (slot_b + 1) & jt.mask;
								if (hdr_b == 0) { probing = false; break; }
								if ((uint32_t) hdr_b == (uint32_t) h && !(hdr_b & GG_HT_NULLKEY) && kb0 == jk0 && (jt.nkeys < 2 || kb1 == jk1)) { have = true; break; }
							}
						}
						bool nullext = false;
						if (pending && !probing && !have) { nullext = fill_outer && !matched; pending = false; }
						if (!__any_sync(GG_FULL_MASK, have || nullext)) break;

						MachState M2 = M1;
						M2.live = have || nullext;
						X.ipay = (const uint64_t *) (e + 1 + jt.nkeys);
						X.ipaynull = nullext ? 0xFFFFFFFFu : (uint32_t) (hdr >> 32) & 0xFFu;
						sink.begin_row();
						sink.jq = have; sink.nullext = nullext; sink.suppress = have && anti;
						MatchSink<decltype(sink)> ms = { sink };
						PL::template run_range<NULLABLE>(X, M2, jt.probe_pc, GGP_MAX_CODE, err, ms);
						if (have && sink.jq)
						{
							matched = true;
							if (jt.mark_matched && !(hdr & GG_HT_MATCHED)) atomicOr((unsigned long long *) e, GG_HT_MATCHED);
							if (single) { probing = false; pending = false; }
						}
						/* distinct inner keys: this key match was the row's only one, whatever the join qual said of it */
						if (have && jt.unique) probing = false;
						if constexpr (TRMODE) tr_accumulate();
					}
				}
			}
			__syncwarp();
			if (lane == 0) mbar_arrive(empty_bar + s * 8);
			s += nteams;
			if (prm.team > 0)
			{
				while (s >= nstage) s -= nstage;
				if (++dealt == nstage) { dealt = 0; ph ^= 1; }
			}
			else
				while (s >= nstage) { s -= nstage; ph ^= 1; }
		}
		if constexpr (MODE == MODE_PART)
		{
			/* what this warp claimed of each region and did not fill is marked dead */
			__syncwarp();
			if (prm.mo.window > 0 && lane < prm.mo.nsegs)
			{
				const unsigned long long b = lds64(sink.win + (uint32_t) lane * 16);
				unsigned long long e = lds64(sink.win + (uint32_t) lane * 16 + 8);
				if (e > prm.mo.cap) e = prm.mo.cap;
				for (unsigned long long r = b; r < e; r++)
					prm.mo.rows[((uint64_t) lane * prm.mo.cap + r) * (uint64_t) prm.mo.rowwords] = GG_ROW_DEAD;
			}
		}
		n_passed = sink.npassed;
		if (sink.nonfinite) err |= GGP_EF_SAW_INF;     /* an infinite/NaN input legitimises an infinite sum */
		if constexpr (MODE == MODE_PRIV) rq_keep = sink.rq;
	}

	/* ===== epilogue: threads -> block records, all in fixed order ===== */
	__syncthreads();
	if (warp < ncons)
	{
		/* per-warp counters and error bits */
		for (int o = 16; o > 0; o >>= 1)
		{
			n_scanned += __shfl_xor_sync(GG_FULL_MASK, n_scanned, o);
			n_passed += __shfl_xor_sync(GG_FULL_MASK, n_passed, o);
			err |= __shfl_xor_sync(GG_FULL_MASK, err, o);
		}
		if (lane == 0)
		{
			if (n_scanned) atomicAdd(&prm.counters[0], n_scanned);
			if (n_passed) atomicAdd(&prm.counters[1], n_passed);
			if (err) atomicOr(prm.errflags, err);
		}
	}
	if constexpr (MODE == MODE_PART || MODE == MODE_HASH) return;
	if constexpr (MODE == MODE_BUILD)
	{
		/* n_passed was folded across the warp above */
		if (warp < ncons && lane == 0 && n_passed) atomicAdd(prm.jt.nbuilt, n_passed);
		return;
	}
	const int G = T->n;
	ggp_grec *out = prm.block_recs + (size_t) blockIdx.x * GGP_FAST_GROUPS;
	for (int g = G + (int) threadIdx.x; g < GGP_FAST_GROUPS; g += blockDim.x) out[g].valid = 0;

	if (MODE == MODE_PRIV)
	{
		/* register-resident accumulators -> the ring's memory, now that no page in it is in use any more */
		double *reg_stage = (double *) smem;          /* [GG_REG_GROUPS][GG_REG_SLOTS][NT] <= 48 KB, inside the ring */
		if (nreg > 0)
		{
			if (warp < ncons)
			{
#define GG_RQ_STAGE(G, J) if (J < nreg) reg_stage[(G * GG_REG_SLOTS + J) * NT + (int) threadIdx.x] = rq_keep.r##G##J;
				GG_RQ_FOREACH(GG_RQ_STAGE)
#undef GG_RQ_STAGE
			}
			__syncthreads();
		}
		/* one warp per (group, slot): lane l folds threads l, l+32, ... in order, then a fixed butterfly */
		for (int e = warp; e < G * V; e += (int) (blockDim.x >> 5))
		{
			const int g = e / V, sl = e % V;
			const bool isint = ((PL::intmask(P) >> sl) & 1) != 0;
			double s0 = isint ? 0.0 : -0.0;
			unsigned long long cnt = 0;
			for (int t = lane; t < NT; t += 32)
			{
				if (nslots > 0)
				{
					const double pv = sl < nsl ? ldsf64(smem_base + prm.acc_off + (uint32_t) ((g * nsl + sl) * NT + t) * 8)
					                           : reg_stage[(g * GG_REG_SLOTS + (sl - nsl)) * NT + t];
					if (isint) s0 = __longlong_as_double(__double_as_longlong(s0) + __double_as_longlong(pv));
					else
					{
						/* a non-finite private sum is either a legitimate +-Inf/NaN input or a float8pl overflow
						 * (ERROR in the reference, float.c:782): this variant does not track which, so it asks the host
						 * to decide by replaying the input on the fully checked interpreter kernel */
						if (!f8_finite(pv)) atomicOr(prm.errflags, GGP_EF_RECHECK);
						s0 = __dadd_rn(s0, pv);
					}
				}
				if (sl == 0) cnt += lds32(smem_base + prm.cnt_off + (uint32_t) (g * NT + t) * 4);
			}
			for (int o = 16; o > 0; o >>= 1)
			{
				const double other = __shfl_xor_sync(GG_FULL_MASK, s0, o);
				s0 = isint ? __longlong_as_double(__double_as_longlong(s0) + __double_as_longlong(other)) : __dadd_rn(s0, other);
				cnt += __shfl_xor_sync(GG_FULL_MASK, cnt, o);
			}
			if (lane == 0)
			{
				if (nslots > 0)
				{
					if (sl < nacc) { out[g].sum[sl] = s0; if (P.accsq[sl] < 0) out[g].sumsq[sl] = 0.0; }
					else
						for (int j = 0; j < nacc; j++)
							if (P.accsq[j] == sl) out[g].sumsq[j] = s0;
				}
				if (sl == 0)
				{
					out[g].count = cnt;
					for (int j = 0; j < nacc; j++) out[g].n[j] = cnt;     /* NOT NULL inputs: every row counts */
					out[g].keynull = T->keynull[g];
					for (int c = 0; c < GG_MAX_KEYS; c++) out[g].key[c] = T->key[g][c];
					out[g].valid = 1;
				}
			}
		}
		return;
	}

	struct Red { double sum; unsigned long long cnt, n; };
	Red *red = (Red *) smem;                       /* [ncons][GGP_MAX_PAIRS]: 21 KB for 7 warps, inside the ring */
	if (warp < ncons)
	{
#pragma unroll
		for (int r = 0; r < GG_NROUNDS; r++)
		{
			Red x;
			x.sum = acc_sum[r]; x.cnt = acc_cnt[r]; x.n = acc_n[r];
			red[warp * GGP_MAX_PAIRS + r * 32 + lane] = x;
		}
	}
	__syncthreads();
	for (int p = threadIdx.x; p < GGP_MAX_PAIRS; p += blockDim.x)
	{
		int g = p / V, sl = p % V;
		if (g >= G || g >= GGP_FAST_GROUPS) continue;
		int kind = nacc == 0 ? GGP_ACC_COUNT : (sl < nacc ? P.acckind[sl] : GGP_ACC_F8SUM);
		double s0 = kind == GGP_ACC_F8SUM ? -0.0 : 0.0;
		unsigned long long cnt = 0, nn = 0;
		for (int w = 0; w < ncons; w++)
		{
			Red x = red[w * GGP_MAX_PAIRS + p];
			cnt += x.cnt;
			if (x.n)
			{
				if (kind == GGP_ACC_F8SUM) s0 = __dadd_rn(s0, x.sum);
				else if (kind == GGP_ACC_I8SUM) s0 = __longlong_as_double(__double_as_longlong(s0) + __double_as_longlong(x.sum));
				else if (kind == GGP_ACC_F8MIN) { if (nn == 0 || f8_cmp(x.sum, s0) < 0) s0 = x.sum; }
				else if (kind == GGP_ACC_F8MAX) { if (nn == 0 || f8_cmp(x.sum, s0) > 0) s0 = x.sum; }
				else if (kind == GGP_ACC_I8MIN) { if (nn == 0 || __double_as_longlong(x.sum) < __double_as_longlong(s0)) s0 = x.sum; }
				else if (kind == GGP_ACC_I8MAX) { if (nn == 0 || __double_as_longlong(x.sum) > __double_as_longlong(s0)) s0 = x.sum; }
				nn += x.n;
			}
		}
		if (nacc > 0)
		{
			if (sl < nacc) { out[g].sum[sl] = s0; out[g].n[sl] = nn; if (P.accsq[sl] < 0) out[g].sumsq[sl] = 0.0; }
			else
				for (int j = 0; j < nacc; j++)
					if (P.accsq[j] == sl) out[g].sumsq[j] = s0;
		}
		if (sl == 0)
		{
			out[g].count = cnt;
			out[g].keynull = T->keynull[g];
			for (int c = 0; c < GG_MAX_KEYS; c++) out[g].key[c] = T->key[g][c];
			out[g].valid = 1;
		}
	}
}

}  // namespace ggd
