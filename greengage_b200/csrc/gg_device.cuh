/*
 * gg_device.cuh — device-side building blocks shared by the kernels:
 *   - mbarrier / TMA bulk-copy PTX wrappers (sm_90a: Hopper and later)
 *   - shared-memory accessors on 32-bit shared addresses (pages are staged in shared memory;
 *     explicit ld.shared keeps address arithmetic 32-bit and off the generic path)
 *   - heap page / tuple decoding (bufpage.h:153, itemid.h:24, htup_details.h:139,
 *     tupmacs.h:23-175, postgres.h:158-300 big-endian varlena headers)
 *   - the accumulator-machine interpreter for compiled plans (gg_program.h)
 *   - bit-exact Jenkins hash / cdbhash / jump-consistent-hash (hashfunc.c:241-552,
 *     cdbhash.c:191-287,549-560)
 */
#pragma once
#ifdef GG_HOST_EMU
/* tests/emu/gg_host_emu.h: host stand-ins for the shared-memory accessors and the few intrinsics used below, so that the
 * tuple walk and the interpreter of THIS file can be compiled by g++ and run on a CPU against the oracle
 * (tests/test_device_emu.py).  Never defined in a product build. */
#include "gg_host_emu.h"
#else
#include <cuda_runtime.h>
#endif
#include <stdint.h>
#include "gg_program.h"

#define GG_FULL_MASK 0xffffffffu
#define GG_F8_NEGZERO_BITS 0x8000000000000000ull    /* -0.0: where float8 sums start */

namespace ggd {

#ifndef GG_HOST_EMU
/* ---------------- PTX wrappers ---------------- */
__device__ __forceinline__ uint32_t smem_u32(const void *p)
{
	return (uint32_t) __cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count)
{
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init()
{
	asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes)
{
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar)
{
	asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity)
{
	uint32_t done;
	asm volatile(
		"{\n\t.reg .pred p;\n\t"
		"mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
		"selp.u32 %0, 1, 0, p;\n\t}"
		: "=r"(done) : "r"(bar), "r"(parity) : "memory");
	return done != 0;
}
/* wait with back-off: a waiting warp must not steal issue slots from the working ones */
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, unsigned sleep_ns)
{
	while (!mbar_try_wait(bar, parity))
		__nanosleep(sleep_ns);
}
/* TMA 1-D bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP) */
__device__ __forceinline__ void tma_load_1d(uint32_t dst_smem, const void *src_gmem, uint32_t bytes, uint32_t bar)
{
	asm volatile(
		"cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
		::"r"(dst_smem), "l"(src_gmem), "r"(bytes), "r"(bar) : "memory");
}

/* shared-memory accessors on 32-bit shared addresses */
__device__ __forceinline__ uint32_t lds8(uint32_t a) { uint32_t v; asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ uint32_t lds16(uint32_t a) { uint32_t v; asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ uint32_t lds32(uint32_t a) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ uint64_t lds64(uint32_t a) { uint64_t v; asm volatile("ld.shared.u64 %0, [%1];" : "=l"(v) : "r"(a)); return v; }
__device__ __forceinline__ double ldsf64(uint32_t a) { double v; asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(a)); return v; }
__device__ __forceinline__ void sts16(uint32_t a, uint32_t v) { asm volatile("st.shared.u16 [%0], %1;" ::"r"(a), "r"(v)); }
__device__ __forceinline__ void sts32(uint32_t a, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(a), "r"(v)); }
__device__ __forceinline__ void sts64(uint32_t a, uint64_t v) { asm volatile("st.shared.u64 [%0], %1;" ::"r"(a), "l"(v)); }
__device__ __forceinline__ void stsf64(uint32_t a, double v) { asm volatile("st.shared.f64 [%0], %1;" ::"r"(a), "d"(v)); }
#endif /* !GG_HOST_EMU */

/* ---------------- hashing: bit-exact with hashfunc.c ---------------- */
__device__ __forceinline__ uint32_t rot32(uint32_t x, int k) { return (x << k) | (x >> (32 - k)); }

#define GGD_FINAL(a, b, c) \
	{ c ^= b; c -= rot32(b, 14); a ^= c; a -= rot32(c, 11); b ^= a; b -= rot32(a, 25); \
	  c ^= b; c -= rot32(b, 16); a ^= c; a -= rot32(c, 4);  b ^= a; b -= rot32(a, 14); \
	  c ^= b; c -= rot32(b, 24); }

/* hash_uint32, hashfunc.c:527 */
__device__ __forceinline__ uint32_t hash_uint32(uint32_t k)
{
	uint32_t a, b, c;
	a = b = c = 0x9e3779b9u + 4u + 3923095u;
	a += k;
	GGD_FINAL(a, b, c);
	return c;
}
/* hash_any over <= 8 bytes held LSB-first in a register (hashfunc.c:302; tail switch cases 0..8) */
__device__ __forceinline__ uint32_t hash_any_le8(uint64_t v, int len)
{
	uint32_t a, b, c;
	a = b = c = 0x9e3779b9u + (uint32_t) len + 3923095u;
	uint64_t m = len >= 8 ? ~0ull : ((1ull << (8 * len)) - 1ull);
	v &= m;
	a += (uint32_t) v;
	b += (uint32_t) (v >> 32);
	GGD_FINAL(a, b, c);
	return c;
}
/* hashint8, hashfunc.c:52 */
__device__ __forceinline__ uint32_t hashint8(int64_t val)
{
	uint32_t lo = (uint32_t) val, hi = (uint32_t) ((uint64_t) val >> 32);
	lo ^= (val >= 0) ? hi : ~hi;
	return hash_uint32(lo);
}
/* hashfloat8, hashfunc.c:110 */
__device__ __forceinline__ uint32_t hashfloat8(uint64_t bits)
{
	double d = __longlong_as_double((long long) bits);
	if (d == 0.0) return 0;
	return hash_any_le8(bits, 8);
}
/* the hash of one non-NULL Motion / distribution key value (cdbhash.c:215-287: the type's default hash opclass function), by
 * ggp_hashtype.  A string arrives packed LSB-first (bpchar already blank-stripped): its length is where its first zero byte is.
 * The one copy of this dispatch: the sending Motion (PartSink), the group-record Motion (route_group) and the emulator use it. */
__device__ __forceinline__ uint32_t key_hash(int t, uint64_t v)
{
	if (t == GGP_HT_INT4) return hash_uint32((uint32_t) v);
	if (t == GGP_HT_INT8) return hashint8((int64_t) v);
	if (t == GGP_HT_FLOAT8) return hashfloat8(v);
	if (t == GGP_HT_BOOL) return hash_uint32((uint32_t) (int32_t) (int8_t) v);      /* hashchar */
	int len = 0;
	while (len < 8 && ((v >> (8 * len)) & 0xff)) len++;
	return hash_any_le8(v, len);
}
/* cdbhash.c:197-219: rotate left 1, xor the column hash unless NULL */
__device__ __forceinline__ uint32_t cdbhash_add(uint32_t h, uint32_t hk, bool isnull)
{
	h = (h << 1) | (h >> 31);
	return isnull ? h : (h ^ hk);
}
/* jump_consistent_hash, cdbhash.c:549-560.  Same IEEE operations as the C code:
 * int->double conversions, one double divide (round-to-nearest), one double multiply,
 * truncating conversion; __dmul_rn/__ddiv_rn keep the compiler from contracting them. */
__device__ __forceinline__ int32_t jump_consistent_hash(uint64_t key, int32_t nsegs)
{
	int64_t b = -1, j = 0;
	while (j < nsegs)
	{
		b = j;
		key = key * 2862933555777941757ULL + 1;
		double q = __ddiv_rn((double) (1LL << 31), (double) ((key >> 33) + 1));
		j = (int64_t) __dmul_rn((double) (b + 1), q);
	}
	return (int32_t) b;
}

/* ---------------- tuple decoding (all addresses are 32-bit shared addresses) ---------------- */
__device__ __forceinline__ uint32_t align_nominal(uint32_t off, int attalign)
{
	/* tupmacs.h:121-130 */
	uint32_t m = attalign == 'd' ? 7u : attalign == 'i' ? 3u : attalign == 's' ? 1u : 0u;
	return (off + m) & ~m;
}
/* VARSIZE_ANY for inline datums, postgres.h:276.  0x80 (external TOAST pointer) and
 * compressed 4-byte headers are reported through bad. */
__device__ __forceinline__ uint32_t varsize_any(uint32_t p, bool &bad)
{
	uint32_t h = lds8(p);
	if (h & 0x80)
	{
		if (h == 0x80) { bad = true; return 4; }
		return h & 0x7F;
	}
	if (h & 0x40) bad = true;   /* compressed in line */
	uint32_t l = ((h & 0x3F) << 24) | (lds8(p + 1) << 16) | (lds8(p + 2) << 8) | lds8(p + 3);
	if (l < 4) { bad = true; return 4; }
	return l;
}

/* ---------------- HeapTupleSatisfiesMVCC against a snapshot (tqual.c:997-1238) ----------------
 * The snapshot in device memory (gg_engine_set_snapshot): 8 header words
 *     [0] xmin  [1] xmax  [2] xcnt  [3] curcid  [4] the scanning backend's own xid (0: none)  [5] clog_base  [6] clog_n
 * then xip[xcnt], then the transaction status bits of xids clog_base .. clog_base + clog_n - 1, two per xid as pg_clog keeps
 * them (clog.h:25-28; clog.c TransactionIdToBIndex: byte xid / 4, shift 2 * (xid % 4); clog_base is a multiple of 4).
 * What only the server can answer raises GGP_EF_VISIBILITY and the relation stays on the CPU scan: multixact xmax,
 * combo command ids, sub-committed status (pg_subtrans), HEAP_MOVED_*, an xid outside the status range.  Distributed
 * snapshots (XidInMVCCSnapshot's first half, tqual.c:1547-1583) are the caller's: it passes the local snapshot only when
 * that decides alone (haveDistribSnapshot false, or every tuple carries the *_DISTRIBUTED_SNAPSHOT_IGNORE bits).  Hint bits
 * are not written back (SetHintBits is an optimisation of the next reader). */
#define GG_SNAP_HDR_WORDS 8
__device__ __forceinline__ bool xid_precedes(uint32_t a, uint32_t b)          /* TransactionIdPrecedes, transam.c:300 */
{
	if (a < 3 || b < 3) return a < b;
	return (int32_t) (a - b) < 0;
}
/* TransactionIdDidCommit (transam.c:125 through TransactionLogFetch :52): 1 committed, 0 not (in progress, aborted, crashed), -1 unknown here */
__device__ __forceinline__ int xid_did_commit(uint32_t xid, const uint32_t *snap)
{
	if (xid == 1 || xid == 2) return 1;                 /* BootstrapTransactionId, FrozenTransactionId */
	if (xid == 0) return 0;
	const uint32_t d = xid - snap[5];
	if (d >= snap[6]) return -1;
	const uint8_t *clog = (const uint8_t *) (snap + GG_SNAP_HDR_WORDS + snap[2]);
	const int st = (clog[d >> 2] >> ((d & 3) * 2)) & 3;
	if (st == 3) return -1;                             /* TRANSACTION_STATUS_SUB_COMMITTED: the parent decides */
	return st == 1;
}
/* XidInMVCCSnapshot_Local (tqual.c:1600-1650), snapshots without subtransaction overflow */
__device__ __forceinline__ bool xid_in_snapshot(uint32_t xid, const uint32_t *snap)
{
	if (xid_precedes(xid, snap[0])) return false;
	if (!xid_precedes(xid, snap[1])) return true;
	for (uint32_t i = 0; i < snap[2]; i++)
		if (snap[GG_SNAP_HDR_WORDS + i] == xid) return true;
	return false;
}
/* tup: shared address of the tuple header.  Returns visibility; err gets GGP_EF_VISIBILITY when the rule cannot be decided here. */
__device__ __forceinline__ bool heap_tuple_satisfies_mvcc(uint32_t tup, uint32_t infomask, const uint32_t *snap, uint32_t &err)
{
	const uint32_t xmin = lds32(tup), xmax = lds32(tup + 4), cid = lds32(tup + 8);
	const uint32_t curcid = snap[3], own = snap[4];
	const bool locked_only = (infomask & GG_HEAP_XMAX_LOCK_ONLY) ||
	                         (infomask & (GG_HEAP_XMAX_IS_MULTI | GG_HEAP_XMAX_EXCL_LOCK | GG_HEAP_XMAX_KEYSHR_LOCK)) == GG_HEAP_XMAX_EXCL_LOCK;
	if (!(infomask & GG_HEAP_XMIN_COMMITTED))
	{
		if (infomask & GG_HEAP_XMIN_INVALID) return false;
		if (infomask & GG_HEAP_MOVED) { err |= GGP_EF_VISIBILITY; return false; }
		if (own && xmin == own)
		{
			if (infomask & GG_HEAP_COMBOCID) { err |= GGP_EF_VISIBILITY; return false; }
			if (cid >= curcid) return false;                     /* inserted after the scan started */
			if (infomask & GG_HEAP_XMAX_INVALID) return true;
			if (locked_only) return true;
			if (infomask & GG_HEAP_XMAX_IS_MULTI) { err |= GGP_EF_VISIBILITY; return false; }
			if (xmax != own) return true;                        /* the deleting subtransaction must have aborted */
			return cid >= curcid;                                /* deleted after / before the scan started */
		}
		const int c = xid_did_commit(xmin, snap);
		if (c < 0) { err |= GGP_EF_VISIBILITY; return false; }
		if (!c) return false;                                    /* in progress, aborted or crashed */
	}
	/* the inserting transaction has committed — but when? */
	if ((infomask & GG_HEAP_XMIN_FROZEN) != GG_HEAP_XMIN_FROZEN && xid_in_snapshot(xmin, snap)) return false;
	if (infomask & GG_HEAP_XMAX_INVALID) return true;
	if (locked_only) return true;
	if (infomask & GG_HEAP_XMAX_IS_MULTI) { err |= GGP_EF_VISIBILITY; return false; }
	if (!(infomask & GG_HEAP_XMAX_COMMITTED))
	{
		if (own && xmax == own)
		{
			if (infomask & GG_HEAP_COMBOCID) { err |= GGP_EF_VISIBILITY; return false; }
			return cid >= curcid;
		}
		const int c = xid_did_commit(xmax, snap);
		if (c < 0) { err |= GGP_EF_VISIBILITY; return false; }
		if (!c) return true;                                     /* deleter in progress, aborted or crashed */
	}
	return xid_in_snapshot(xmax, snap);                          /* deleter committed after the snapshot: still visible */
}

/* Per-lane view of one tuple after the attribute walk */
struct TupleView {
	uint32_t tp;            /* shared address of the start of user data (tuple + t_hoff) */
	uint32_t colnull;       /* bit s: column slot s is NULL */
};

/* The attribute walk: slot_deform_tuple (heaptuple.c:1119-1213) restricted to the attributes the
 * program references.  Offsets go to offs + (slot*32 + lane)*2 (shared memory).
 *   fast == true  (no tuple of the warp carries a null bitmap): columns with a constant offset
 *                 (attcacheoff) are addressed by the constant baked into the program; only the
 *                 attributes from the first varlena on are walked and stored.
 *   fast == false every referenced column gets its per-lane offset stored.
 * The walk is split into begin / one step per attribute / end so that a plan-specialised kernel can
 * emit the steps with literal attribute properties (everything then folds at compile time). */
struct WalkState {
	uint32_t tup, tp, bp, datalen, tnatts, off, colnull;
	bool hasnulls, bad;
};

__device__ __forceinline__ void walk_begin(WalkState &W, uint32_t tup, uint32_t tuplen)
{
	const uint32_t infomask = lds16(tup + 20);
	const uint32_t hoff = lds8(tup + 22);
	W.tup = tup;
	W.tnatts = lds16(tup + 18) & GG_HEAP_NATTS_MASK;
	W.hasnulls = (infomask & GG_HEAP_HASNULL) != 0;
	W.bp = tup + GG_HEAP_HDR_SIZE;
	W.tp = tup + hoff;
	W.datalen = tuplen > hoff ? tuplen - hoff : 0;
	W.colnull = 0;
	W.bad = false;
	W.off = 0;
}
/* publish the constant offset of a column in the fixed prefix (only needed when !fast) */
__device__ __forceinline__ void walk_publish_const(WalkState &W, int slot, int att, int cacheoff, uint32_t offs, int lane)
{
	if ((uint32_t) att >= W.tnatts) W.colnull |= 1u << slot;    /* added after the tuple was written: NULL (heaptuple.c:1252) */
	else sts16(offs + (uint32_t) (slot * 32 + lane) * 2, (uint32_t) cacheoff);
}
/* one attribute of the walk */
__device__ __forceinline__ void walk_step(WalkState &W, int a, int attlen, int attalign, int slot, uint32_t offs, int lane)
{
	if (W.bad) return;
	if ((uint32_t) a >= W.tnatts || (W.hasnulls && !(lds8(W.bp + (a >> 3)) & (1u << (a & 7)))))
	{
		if (slot >= 0) W.colnull |= 1u << slot;
		return;
	}
	uint32_t off = W.off;
	if (attlen == -1)
	{
		/* att_align_pointer: a zero byte is padding (or an aligned 4-byte header) */
		if (off < W.datalen && lds8(W.tp + off) == 0) off = align_nominal(off, attalign);
	}
	else
		off = align_nominal(off, attalign);
	if (slot >= 0) sts16(offs + (uint32_t) (slot * 32 + lane) * 2, off);
	if (off >= W.datalen) { W.bad = true; return; }
	off += attlen > 0 ? (uint32_t) attlen : varsize_any(W.tp + off, W.bad);
	if (off > W.datalen) W.bad = true;
	W.off = off;
}

/* table-driven walk (the interpreter path) */
__device__ __forceinline__ void walk_tuple(const ggp_side &S, uint32_t tup, uint32_t tuplen, bool fast,
                                           uint32_t offs, int lane, TupleView &tv, uint32_t &err)
{
	WalkState W;
	walk_begin(W, tup, tuplen);
	int a0 = 0;
	if (!W.hasnulls)
	{
		a0 = S.first_walk > 0 ? S.first_walk - 1 : 0;
		if (a0 > S.natts_walk) a0 = S.natts_walk;
		if (!fast || W.tnatts < (uint32_t) S.natts_walk)
			for (int s = 0; s < S.ncols; s++)
			{
				int a = S.colatt[s];
				if (a < a0) walk_publish_const(W, s, a, S.att[a].cacheoff, offs, lane);
			}
		if (a0 < S.natts_walk) W.off = a0 > 0 ? (uint32_t) S.att[a0].cacheoff : 0;
	}
	for (int a = a0; a < S.natts_walk; a++)
	{
		const ggp_attr at = S.att[a];
		walk_step(W, a, at.attlen, at.attalign, at.slot, offs, lane);
	}
	if (W.bad) err |= GGP_EF_BADPAGE;
	tv.tp = W.tp;
	tv.colnull = W.colnull;
}

/* short string column -> <= 8 bytes packed LSB-first (VARDATA_ANY / VARSIZE_ANY_EXHDR, postgres.h:276-300;
 * bcTruelen for bpchar, varchar.c:653) */
__device__ __forceinline__ uint64_t load_str(uint32_t p, bool strip, uint32_t &err)
{
	uint32_t h = lds8(p), len, d;
	if (h & 0x80)
	{
		if (h == 0x82)                                    /* the common char(1) / 1-byte value */
		{
			uint32_t b = lds8(p + 1);
			return (strip && b == ' ') ? 0 : b;
		}
		if (h == 0x80) { err |= GGP_EF_STRING_TOO_LONG; return 0; }     /* TOAST pointer */
		len = (h & 0x7F) - 1; d = p + 1;
	}
	else
	{
		if (h & 0x40) { err |= GGP_EF_STRING_TOO_LONG; return 0; }      /* compressed in line */
		len = ((((h & 0x3F) << 24) | (lds8(p + 1) << 16) | (lds8(p + 2) << 8) | lds8(p + 3))) - 4;
		d = p + 4;
	}
	if (strip)
		while (len > 0 && lds8(d + len - 1) == ' ') len--;
	if (len > 8) { err |= GGP_EF_STRING_TOO_LONG; return 0; }
	uint64_t v = 0;
	for (uint32_t i = 0; i < len; i++) v |= (uint64_t) lds8(d + i) << (8 * i);
	return v;
}

/* numeric column -> 64-bit integer scaled by 10^scale.  On-disk form (utils/adt/numeric.c:95-190): varlena header, then
 * n_header (short: bit 15 set, sign bit 13, dscale bits 12-7, weight sign bit 6, weight bits 5-0; long: sign bits 15-14,
 * dscale bits 13-0, followed by int16 weight), then base-10000 digits (int16 each), most significant first, leading and
 * trailing zero digits stripped.  value = sum digit[i] * 10000^(weight - i). */
__device__ __forceinline__ int64_t load_numeric(uint32_t p, int scale, uint32_t &err)
{
	const uint32_t h = lds8(p);
	uint32_t len, d;
	if (h & 0x80)
	{
		if (h == 0x80) { err |= GGP_EF_NUMERIC_RANGE; return 0; }           /* TOAST pointer */
		len = (h & 0x7F) - 1; d = p + 1;
	}
	else
	{
		if (h & 0x40) { err |= GGP_EF_NUMERIC_RANGE; return 0; }            /* compressed in line */
		len = ((((h & 0x3F) << 24) | (lds8(p + 1) << 16) | (lds8(p + 2) << 8) | lds8(p + 3))) - 4;
		d = p + 4;
	}
	if (len < 2) { err |= GGP_EF_NUMERIC_RANGE; return 0; }
	const uint32_t nh = lds8(d) | (lds8(d + 1) << 8);
	if ((nh & 0xC000) == 0xC000) { err |= GGP_EF_NUMERIC_RANGE; return 0; }     /* NaN */
	bool neg;
	int weight;
	uint32_t dp;
	if (nh & 0x8000)
	{
		neg = (nh & 0x2000) != 0;
		weight = (int) (nh & 0x3F) | ((nh & 0x40) ? ~0x3F : 0);
		dp = d + 2;
	}
	else
	{
		if (len < 4) { err |= GGP_EF_NUMERIC_RANGE; return 0; }
		neg = (nh & 0xC000) == 0x4000;
		weight = (int) (int16_t) (lds8(d + 2) | (lds8(d + 3) << 8));
		dp = d + 4;
	}
	const int nd = (int) ((d + len - dp) >> 1);
	if (nd > 8) { err |= GGP_EF_NUMERIC_RANGE; return 0; }                      /* more than 32 decimal digits never fit */
	uint64_t v = 0;
	bool bad = false;
	/* value * 10000^(nd - 1 - weight) is v after the loop; wanted: value * 10^scale, so v is then scaled by 10^e.  When the last
	 * digit reaches 1..3 decimals past the column's scale (a scale that is not a multiple of 4), those decimals are zeros:
	 * they are dropped from the digit before it is added, so that v never holds more than the scaled value */
	int e = 4 * (weight - (nd - 1)) + scale;
	if (nd == 0) e = 0;
	for (int i = 0; i < nd; i++)
	{
		uint32_t dig = lds8(dp + 2 * i) | (lds8(dp + 2 * i + 1) << 8);
		uint64_t mul = 10000ull;
		if (i == nd - 1 && e < 0 && e > -4)
		{
			const uint32_t drop = e == -1 ? 10u : e == -2 ? 100u : 1000u;
			if (dig % drop) bad = true;                                         /* digits beyond the column's scale must be zeros */
			dig /= drop; mul /= drop; e = 0;
		}
		const uint64_t m = v * mul;
		if (__umul64hi(v, mul) != 0 || m + dig < m) bad = true;             /* the product, or the digit's carry, past 2^64 */
		v = m + dig;
	}
	for (; e > 0; e--) { if (__umul64hi(v, 10ull) != 0) bad = true; v *= 10ull; }
	for (; e < 0; e++) { if (v % 10ull) bad = true; v /= 10ull; }               /* digits beyond the column's scale must be zeros */
	if (v >> 63) bad = true;
	if (bad) { err |= GGP_EF_NUMERIC_RANGE; return 0; }
	return neg ? -(int64_t) v : (int64_t) v;
}

/* exact 64-bit integer arithmetic for scaled numerics: overflow is reported, never wrapped */
__device__ __forceinline__ int64_t i64_add_chk(int64_t a, int64_t b, bool &ovf)
{
	const int64_t r = (int64_t) ((uint64_t) a + (uint64_t) b);
	if (((a ^ r) & (b ^ r)) < 0) ovf = true;
	return r;
}
__device__ __forceinline__ int64_t i64_mul_chk(int64_t a, int64_t b, bool &ovf)
{
	const int64_t hi = __mul64hi(a, b);
	const int64_t lo = (int64_t) ((uint64_t) a * (uint64_t) b);
	if (hi != (lo >> 63)) ovf = true;
	return lo;
}

__device__ __forceinline__ int f8_cmp(double a, double b)
{
	/* float8_cmp_internal, float.c:964: NaN = NaN, NaN > everything */
	bool na = a != a, nb = b != b;
	if (na) return nb ? 0 : 1;
	if (nb) return -1;
	return (a > b) - (a < b);
}
__device__ __forceinline__ bool test_cc(int c, int cc)
{
	switch (cc)
	{
		case GGP_LT: return c < 0;
		case GGP_LE: return c <= 0;
		case GGP_EQ: return c == 0;
		case GGP_NE: return c != 0;
		case GGP_GT: return c > 0;
		default: return c >= 0;
	}
}
__device__ __forceinline__ bool f8_isinf(double x) { return fabs(x) == __longlong_as_double(0x7ff0000000000000LL); }
__device__ __forceinline__ bool f8_finite(double x) { return fabs(x) < __longlong_as_double(0x7ff0000000000000LL); }

/* CHECKFLOATVAL (float_utils.h:28), evaluated only when the result is not finite or is zero */
static __device__ __noinline__ uint32_t f8_check_slow(int kind /* 0 add/sub, 1 mul, 2 div */, double x, double y, double r)
{
	uint32_t e = 0;
	if (f8_isinf(r) && !(f8_isinf(x) || f8_isinf(y))) e |= GGP_EF_FLOAT_OVERFLOW;
	if (kind == 1 && r == 0.0 && !(x == 0.0 || y == 0.0)) e |= GGP_EF_FLOAT_UNDERFLOW;
	if (kind == 2 && r == 0.0 && x != 0.0) e |= GGP_EF_FLOAT_UNDERFLOW;
	return e;
}

/* normalise a key so that bitwise equality == SQL equality (join keys: the hash table compares bits) */
__device__ __forceinline__ uint64_t normalize_key(uint64_t v, int keytype)
{
	if (keytype == 2)
	{
		double d = __longlong_as_double((long long) v);
		if (d == 0.0) return 0;                               /* -0 = +0 (float8eq) */
		if (d != d) return 0x7ff8000000000000ull;             /* all NaNs are equal (float.c:964) */
	}
	return v;
}
/* A grouping key as its group stores it.  The group's key is the value of the row that created the group
 * (lookup_agg_hash_entry, execHHashagg.c:456 copies the first tuple's), so a float8 zero keeps its sign; every NaN becomes one
 * encoding, because records are routed and merged by their key bits.  Grouping keys are compared with key_same and hashed
 * (HashAggregate) as normalize_key gives them. */
__device__ __forceinline__ uint64_t group_key(uint64_t v, int keytype)
{
	if (keytype == 2 && __longlong_as_double((long long) v) != __longlong_as_double((long long) v)) return 0x7ff8000000000000ull;
	return v;
}
/* two group_key values are one group: equal bits, or (f8: a float8 key) zeros of either sign */
__device__ __forceinline__ bool key_same(uint64_t a, uint64_t b, bool f8)
{
	return a == b || (f8 && ((a | b) << 1) == 0);
}
/* of 2-bit key types (key c at bits 2c): bit 2c set where key c is float8.  A constant with no float8 key folds to 0, so a
 * plan-specialised kernel without one compares its keys as plain bits */
__device__ __forceinline__ uint32_t f8_keys(uint32_t keytypes) { return (keytypes >> 1) & ~keytypes & 0x55u; }

/* Everything a running program needs to reach its operands */
struct EvalCtx {
	const ggp_program *P;   /* interpreter path only */
	TupleView tv;           /* outer / scan tuple */
	uint32_t offs;          /* shared address of its per-lane column offsets [slot*32 + lane] u16 */
	bool fast;              /* constant offsets usable (no tuple of the warp has NULLs) */
	const uint64_t *ipay;   /* joins: the matched hash-table entry's payload = the inner columns, already loaded
	                         * (sign-extended / packed) by the build program; slot i = inner column slot i */
	uint32_t ipaynull;      /* bit i: inner column slot i is NULL (all ones for a null-extended row) */
	int lane;
};

/* registers of the accumulator machine */
struct MachState {
	uint64_t acc, t0, t1, t2, t3;
	uint32_t tnull;
	uint32_t livestk;       /* `live` of the enclosing AND / OR arms (GGP_GUARD_*), innermost in bit 0 */
	bool accnull;
	bool live;              /* this lane carries a row that still counts; dead lanes keep executing (the op
	                         * stream is warp-uniform) but raise no errors and produce no effects */
	__device__ __forceinline__ void reset(bool l) { acc = t0 = t1 = t2 = t3 = 0; tnull = 0; livestk = 0; accnull = false; live = l; }
};

/* One op of the accumulator machine, including its post-actions.  `o` is passed by value: on the
 * interpreter path it comes from the program table; in a plan-specialised kernel it is a literal and
 * the whole function folds down to the few instructions of that one op.  KF(idx) yields constant idx.
 * `Sink` receives the post-actions:
 *     bool filter(bool pass)  /  void key(int k, uint64_t v, bool n)  /  bool group(bool live)
 *     void out(int slot, double v, bool n) */
template <bool NULLABLE, bool HAS_INNER, class Sink, class KF>
__device__ __forceinline__ void exec_op(const ggp_op o, const EvalCtx &X, const KF &KV, uint32_t constnull,
                                        MachState &M, uint32_t &err, Sink &sink)
{
#define GG_COLADDR(O) (X.tv.tp + ((X.fast && (O).off != 0xFFFF) ? (uint32_t) (O).off : lds16(X.offs + (uint32_t) (((O).idx * 32) + X.lane) * 2)))
#define GG_ISINNER(O) (HAS_INNER && ((O).idx & 0x80))
#define GG_INNERVAL(O) (__ldg(X.ipay + ((O).idx & 0x7F)))
#define GG_COL64(O) (GG_ISINNER(O) ? GG_INNERVAL(O) : lds64(GG_COLADDR(O)))
#define GG_COLI4(O) (GG_ISINNER(O) ? GG_INNERVAL(O) : (uint64_t) (int64_t) (int32_t) lds32(GG_COLADDR(O)))
#define GG_COLNULL(O) (NULLABLE && ((GG_ISINNER(O) ? (X.ipaynull >> ((O).idx & 0x7F)) : (X.tv.colnull >> (O).idx)) & 1))
#define GG_TEMP(IDX) ((IDX) == 0 ? M.t0 : (IDX) == 1 ? M.t1 : (IDX) == 2 ? M.t2 : M.t3)
#define GG_TNULL(IDX) (NULLABLE && ((M.tnull >> (IDX)) & 1))
#define GG_KNULL(IDX) (NULLABLE && ((constnull >> (IDX)) & 1))
#define GG_D(V) __longlong_as_double((long long) (V))
#define GG_ACCD GG_D(M.acc)
#define GG_F8(KIND, EXPR, XV, YV, SN) \
	{ const double x = (XV), y = (YV), r = (EXPR); const bool isn = NULLABLE && (M.accnull || (SN)); \
	  if (!f8_finite(r) || ((KIND) != 0 && r == 0.0)) { if (M.live && !isn) err |= f8_check_slow((KIND), x, y, r); } \
	  M.acc = (uint64_t) __double_as_longlong(r); M.accnull = isn; }
#define GG_COLF8(O, SN, V) const bool SN = GG_COLNULL(O); const double V = SN ? 1.0 : GG_D(GG_COL64(O));

	const int op = o.op;
	/* most frequent first; the op stream is uniform across the warp, so these branches never diverge */
	if (op == GGP_LD_C8) { M.accnull = GG_COLNULL(o); M.acc = M.accnull ? 0 : GG_COL64(o); }
	else if (op == GGP_MUL_C) { GG_COLF8(o, sn, v) GG_F8(1, __dmul_rn(x, y), GG_ACCD, v, sn) }
	else if (op == GGP_MUL_T) { GG_F8(1, __dmul_rn(x, y), GG_ACCD, GG_D(GG_TEMP(o.idx)), GG_TNULL(o.idx)) }
	else if (op == GGP_LD_K) { M.acc = (uint64_t) KV(o.idx); M.accnull = GG_KNULL(o.idx); }
	else if (op == GGP_ADD_C) { GG_COLF8(o, sn, v) GG_F8(0, __dadd_rn(x, y), GG_ACCD, v, sn) }
	else if (op == GGP_SUB_C) { GG_COLF8(o, sn, v) GG_F8(0, __dsub_rn(x, y), GG_ACCD, v, sn) }
	else if (op == GGP_LD_C4) { M.accnull = GG_COLNULL(o); M.acc = M.accnull ? 0 : GG_COLI4(o); }
	else if (op == GGP_CMPI_K) { const int64_t y = KV(o.idx), x = (int64_t) M.acc;
		M.acc = test_cc((x > y) - (x < y), o.aux & 7); if (NULLABLE) M.accnull = M.accnull || GG_KNULL(o.idx); }
	else if (op == GGP_LD_BP) { uint32_t e2 = 0; M.accnull = GG_COLNULL(o); M.acc = M.accnull ? 0 : (GG_ISINNER(o) ? GG_INNERVAL(o) : load_str(GG_COLADDR(o), true, e2)); if (M.live) err |= e2; }
	else switch (op)
	{
		case GGP_LD_VS: { uint32_t e2 = 0; M.accnull = GG_COLNULL(o); M.acc = M.accnull ? 0 : (GG_ISINNER(o) ? GG_INNERVAL(o) : load_str(GG_COLADDR(o), false, e2)); if (M.live) err |= e2; } break;
		case GGP_LD_BOOL: M.accnull = GG_COLNULL(o); M.acc = M.accnull ? 0 : (GG_ISINNER(o) ? GG_INNERVAL(o) : (uint64_t) (lds8(GG_COLADDR(o)) != 0)); break;
		case GGP_LD_T: M.acc = GG_TEMP(o.idx); M.accnull = GG_TNULL(o.idx); break;
		case GGP_ADD_K: GG_F8(0, __dadd_rn(x, y), GG_ACCD, GG_D(KV(o.idx)), GG_KNULL(o.idx)) break;
		case GGP_ADD_T: GG_F8(0, __dadd_rn(x, y), GG_ACCD, GG_D(GG_TEMP(o.idx)), GG_TNULL(o.idx)) break;
		case GGP_SUB_K: GG_F8(0, __dsub_rn(x, y), GG_ACCD, GG_D(KV(o.idx)), GG_KNULL(o.idx)) break;
		case GGP_SUB_T: GG_F8(0, __dsub_rn(x, y), GG_ACCD, GG_D(GG_TEMP(o.idx)), GG_TNULL(o.idx)) break;
		case GGP_RSUB_C: { GG_COLF8(o, sn, v) GG_F8(0, __dsub_rn(x, y), v, GG_ACCD, sn) } break;
		case GGP_RSUB_K: GG_F8(0, __dsub_rn(x, y), GG_D(KV(o.idx)), GG_ACCD, GG_KNULL(o.idx)) break;
		case GGP_RSUB_T: GG_F8(0, __dsub_rn(x, y), GG_D(GG_TEMP(o.idx)), GG_ACCD, GG_TNULL(o.idx)) break;
		case GGP_MUL_K: GG_F8(1, __dmul_rn(x, y), GG_ACCD, GG_D(KV(o.idx)), GG_KNULL(o.idx)) break;
		case GGP_DIV_C: case GGP_DIV_K: case GGP_DIV_T: case GGP_RDIV_C: case GGP_RDIV_K: case GGP_RDIV_T:
		{
			/* float8div (float.c:808): division by zero is its own error */
			const int v3 = (op - GGP_DIV_C) % 3;
			const bool rev = op >= GGP_RDIV_C;
			bool sn;
			double v;
			if (v3 == 0) { sn = GG_COLNULL(o); v = sn ? 1.0 : GG_D(GG_COL64(o)); }
			else if (v3 == 1) { sn = GG_KNULL(o.idx); v = GG_D(KV(o.idx)); }
			else { sn = GG_TNULL(o.idx); v = GG_D(GG_TEMP(o.idx)); }
			const double xn = rev ? v : GG_ACCD, yd = rev ? GG_ACCD : v;
			if (yd == 0.0)
			{
				/* ereport(division by zero) comes before the division and its CHECKFLOATVAL (float.c:818) */
				const bool isn = NULLABLE && (M.accnull || sn);
				if (M.live && !isn) err |= GGP_EF_DIV_ZERO;
				M.acc = (uint64_t) __double_as_longlong(__ddiv_rn(xn, yd)); M.accnull = isn;
			}
			else
				GG_F8(2, __ddiv_rn(x, y), xn, yd, sn)
			break;
		}
		case GGP_CMPF_C: { GG_COLF8(o, sn, v) M.acc = test_cc(f8_cmp(GG_ACCD, v), o.aux & 7); if (NULLABLE) M.accnull = M.accnull || sn; } break;
		case GGP_CMPF_K: M.acc = test_cc(f8_cmp(GG_ACCD, GG_D(KV(o.idx))), o.aux & 7); if (NULLABLE) M.accnull = M.accnull || GG_KNULL(o.idx); break;
		case GGP_CMPF_T: M.acc = test_cc(f8_cmp(GG_ACCD, GG_D(GG_TEMP(o.idx))), o.aux & 7); if (NULLABLE) M.accnull = M.accnull || GG_TNULL(o.idx); break;
		case GGP_CMPI_C4: { const bool sn = GG_COLNULL(o); const int64_t y = sn ? 0 : (int64_t) GG_COLI4(o), x = (int64_t) M.acc;
			M.acc = test_cc((x > y) - (x < y), o.aux & 7); if (NULLABLE) M.accnull = M.accnull || sn; } break;
		case GGP_CMPI_C8: { const bool sn = GG_COLNULL(o); const int64_t y = sn ? 0 : (int64_t) GG_COL64(o), x = (int64_t) M.acc;
			M.acc = test_cc((x > y) - (x < y), o.aux & 7); if (NULLABLE) M.accnull = M.accnull || sn; } break;
		case GGP_CMPI_T: { const int64_t y = (int64_t) GG_TEMP(o.idx), x = (int64_t) M.acc;
			M.acc = test_cc((x > y) - (x < y), o.aux & 7); if (NULLABLE) M.accnull = M.accnull || GG_TNULL(o.idx); } break;
		case GGP_CMPS_K: M.acc = ((o.aux & 7) == GGP_EQ) ? (M.acc == (uint64_t) KV(o.idx)) : (M.acc != (uint64_t) KV(o.idx));
			if (NULLABLE) M.accnull = M.accnull || GG_KNULL(o.idx); break;
		case GGP_CMPS_T: M.acc = ((o.aux & 7) == GGP_EQ) ? (M.acc == GG_TEMP(o.idx)) : (M.acc != GG_TEMP(o.idx));
			if (NULLABLE) M.accnull = M.accnull || GG_TNULL(o.idx); break;
		case GGP_DATE2TS:
		{
			/* date2timestamp, date.c:457: +-infinity map to +-infinity; otherwise days * USECS_PER_DAY,
			 * "date out of range for timestamp" when that overflows int64 (|d| > 106751991) */
			const int32_t d = (int32_t) M.acc;
			int64_t r;
			if (d == INT32_MIN) r = INT64_MIN;
			else if (d == INT32_MAX) r = INT64_MAX;
			else
			{
				r = (int64_t) d * 86400000000LL;
				if ((d > 106751991 || d < -106751991) && M.live && !(NULLABLE && M.accnull)) err |= GGP_EF_DATE_RANGE;
			}
			M.acc = (uint64_t) r;
			break;
		}
		case GGP_I2F8: M.acc = (uint64_t) __double_as_longlong((double) (int64_t) M.acc); break;
		case GGP_AND_T:
		case GGP_OR_T:
		{
			const bool a = M.acc != 0, b = GG_TEMP(o.idx) != 0, an = NULLABLE && M.accnull, bn = GG_TNULL(o.idx);
			if (op == GGP_AND_T)
			{
				if ((!an && !a) || (!bn && !b)) { M.acc = 0; M.accnull = false; }
				else if (an || bn) { M.acc = 0; M.accnull = true; }
				else { M.acc = 1; M.accnull = false; }
			}
			else
			{
				if ((!an && a) || (!bn && b)) { M.acc = 1; M.accnull = false; }
				else if (an || bn) { M.acc = 0; M.accnull = true; }
				else { M.acc = 0; M.accnull = false; }
			}
			break;
		}
		case GGP_GUARD_AND:
		case GGP_GUARD_OR:
		{
			/* the arm that follows is reached only if temp[idx] has not decided the result (execQual.c:3385,3455) */
			const bool decided = !GG_TNULL(o.idx) && ((GG_TEMP(o.idx) != 0) == (op == GGP_GUARD_OR));
			M.livestk = (M.livestk << 1) | (M.live ? 1u : 0u);
			M.live = M.live && !decided;
			break;
		}
		case GGP_UNGUARD: M.live = (M.livestk & 1u) != 0; M.livestk >>= 1; break;
		case GGP_LD_NUM:
		{
			uint32_t e2 = 0;
			M.accnull = GG_COLNULL(o);
			/* an inner column above a join: the build program loaded it at its column scale into the payload */
			M.acc = M.accnull ? 0 : GG_ISINNER(o) ? GG_INNERVAL(o) : (uint64_t) load_numeric(GG_COLADDR(o), o.aux & 15, e2);
			if (M.live) err |= e2;
			break;
		}
		case GGP_IADD_K: case GGP_IADD_T: case GGP_ISUB_K: case GGP_ISUB_T: case GGP_IRSUB_K: case GGP_IRSUB_T: case GGP_IMUL_K: case GGP_IMUL_T:
		{
			const bool isk = op == GGP_IADD_K || op == GGP_ISUB_K || op == GGP_IRSUB_K || op == GGP_IMUL_K;
			const int64_t x = isk ? (int64_t) KV(o.idx) : (int64_t) GG_TEMP(o.idx), a = (int64_t) M.acc;
			const bool xn = isk ? GG_KNULL(o.idx) : GG_TNULL(o.idx);
			bool ovf = false;
			int64_t r;
			if (op == GGP_IADD_K || op == GGP_IADD_T) r = i64_add_chk(a, x, ovf);
			else if (op == GGP_ISUB_K || op == GGP_ISUB_T) { if (x == INT64_MIN) ovf = true; r = i64_add_chk(a, -x, ovf); }
			else if (op == GGP_IRSUB_K || op == GGP_IRSUB_T) { if (a == INT64_MIN) ovf = true; r = i64_add_chk(x, -a, ovf); }
			else r = i64_mul_chk(a, x, ovf);
			const bool isn = NULLABLE && (M.accnull || xn);
			if (ovf && M.live && !isn) err |= GGP_EF_NUMERIC_RANGE;
			M.acc = (uint64_t) r; M.accnull = isn;
			break;
		}
		case GGP_LO32: M.acc = M.acc & 0xFFFFFFFFull; break;
		case GGP_SAR32: M.acc = (uint64_t) ((int64_t) M.acc >> 32); break;
		case GGP_NOT: M.acc = (M.acc == 0); break;
		case GGP_ISNULL: M.acc = M.accnull; M.accnull = false; break;
		case GGP_ISNOTNULL: M.acc = !M.accnull; M.accnull = false; break;
		default: break;                         /* GGP_NOP, GGP_END */
	}

	if (o.flags)
	{
		if (o.flags & GGP_F_ST)
		{
			const int t = (o.aux >> 4) & 3;
			if (t == 0) M.t0 = M.acc; else if (t == 1) M.t1 = M.acc; else if (t == 2) M.t2 = M.acc; else M.t3 = M.acc;
			if (NULLABLE) M.tnull = (M.tnull & ~(1u << t)) | ((uint32_t) M.accnull << t);
		}
		if (o.flags & GGP_F_FILTER) M.live = sink.filter(M.live && !M.accnull && M.acc != 0);
		if (o.flags & GGP_F_KEY) sink.key((o.aux >> 6) & 3, M.acc, M.accnull);
		if (o.flags & GGP_F_GROUP) M.live = sink.group(M.live);
		if (o.flags & GGP_F_OUT) sink.out(o.out, GG_ACCD, M.accnull);
		if (o.flags & GGP_F_OUTSQ)
		{
			const double v = GG_ACCD, sq = __dmul_rn(v, v);
			if (o.out2 == GGP_OUTSQ_CHECK_ONLY)
			{
				if (!f8_finite(sq) && f8_finite(v) && M.live && !(NULLABLE && M.accnull)) err |= GGP_EF_FLOAT_OVERFLOW;
			}
			else sink.out(o.out2, sq, M.accnull);
		}
	}
#undef GG_COLADDR
#undef GG_ISINNER
#undef GG_INNERVAL
#undef GG_COL64
#undef GG_COLI4
#undef GG_COLNULL
#undef GG_TEMP
#undef GG_TNULL
#undef GG_KNULL
#undef GG_F8
#undef GG_ACCD
#undef GG_D
#undef GG_COLF8
}

/* the interpreter: walk the program table */
struct DynConsts {
	const ggp_program *P;
	__device__ __forceinline__ int64_t operator()(int i) const { return P->consts[i]; }
};
/* ops [pc0, pc1) — or up to END — on machine state M (joins run the program in two pieces) */
template <bool NULLABLE, bool HAS_INNER, class Sink>
__device__ __forceinline__ void run_range(const EvalCtx &X, MachState &M, int pc0, int pc1, uint32_t &err, Sink &sink)
{
	const ggp_program &P = *X.P;
	DynConsts KV;
	KV.P = &P;
	for (int pc = pc0; pc < pc1; pc++)
	{
		const ggp_op o = P.code[pc];
		if (o.op == GGP_END) break;
		exec_op<NULLABLE, HAS_INNER>(o, X, KV, (uint32_t) P.constnull, M, err, sink);
	}
}
template <bool NULLABLE, bool HAS_INNER, class Sink>
__device__ __forceinline__ void run_prog(const EvalCtx &X, bool live, uint32_t &err, Sink &sink)
{
	MachState M;
	M.reset(live);
	run_range<NULLABLE, HAS_INNER>(X, M, 0, GGP_MAX_CODE, err, sink);
}

/* the sink of a program that only filters (ggp_compile_filter): the row passes when every FILTER saw TRUE */
struct FilterSink {
	bool pass;
	__device__ __forceinline__ bool filter(bool p) { pass = p; return p; }
	__device__ __forceinline__ void key(int, uint64_t, bool) {}
	__device__ __forceinline__ bool group(bool l) { return l; }
	__device__ __forceinline__ void out(int, double, bool) {}
};
/* An Agg's HAVING over one datum row at shared address rp (NULL mask word, then one word per column; the front end of the scan
 * kernels' datum rows): TRUE passes, FALSE and NULL do not (ExecQual), a dead slot never does.  Errors of the rows that are
 * evaluated go to err; an arm the reference skips raises nothing (GGP_GUARD_*). */
__device__ __forceinline__ bool datumrow_passes(const ggp_program &P, uint32_t rp, bool present, int lane, uint32_t &err)
{
	EvalCtx X;
	const uint64_t mask = present ? lds64(rp) : GG_DATUMROW_DEAD;
	const bool live = !(mask & GG_DATUMROW_DEAD);
	uint32_t cn = 0;
	for (int sl = 0; sl < P.outer.ncols; sl++) cn |= (uint32_t) ((mask >> P.outer.colatt[sl]) & 1) << sl;
	X.P = &P;
	X.tv.tp = rp + 8;
	X.tv.colnull = live ? cn : 0;
	X.offs = 0;
	X.fast = true;
	X.ipay = nullptr;
	X.ipaynull = 0;
	X.lane = lane;
	FilterSink sink;
	sink.pass = live;
	run_prog<true, false>(X, live, err, sink);
	return sink.pass;
}

}  // namespace ggd
