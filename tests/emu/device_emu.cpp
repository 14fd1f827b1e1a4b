/*
 * device_emu.cpp — TEST INFRASTRUCTURE.  The product's plan compiler (gg_compile.cpp) and the product's device
 * interpreter (gg_device.cuh: walk_tuple + run_prog, compiled for the host through gg_host_emu.h) driven over heap pages by
 * a plain loop, one tuple at a time; a host sink folds what the program emits the way the kernels' sinks and the merge
 * kernel do (per accumulator kind).  tests/test_device_emu.py compares the result with the oracle for random plans: a
 * differential test of compiler + interpreter semantics that needs no GPU.  What it does NOT cover is everything
 * parallel — warps, the TMA ring, shared-memory accumulators, the merge kernel, atomics: that is the GPU tests' job.
 */
#define GG_HOST_EMU
#include "gg_host_emu.h"
#include "../../greengage_b200/csrc/gg_device.cuh"
#include "../../include/ggb200.h"
#include <map>
#include <vector>
#include <array>

uint8_t gg_emu_smem[GG_EMU_SMEM_BYTES];
void gg_set_error(const char *, ...) {}

using namespace ggd;

struct EmuGroup {
	uint64_t key[GG_MAX_KEYS];
	uint32_t keynull;
	uint32_t pad;
	uint64_t count;
	double   sum[GGP_MAX_ACCS];      /* by accumulator column; I8* kinds keep int64 bits */
	double   sumsq[GGP_MAX_ACCS];
	uint64_t n[GGP_MAX_ACCS];
};

struct HostSink {
	const ggp_program *P;
	std::map<std::array<uint64_t, GG_MAX_KEYS + 1>, EmuGroup> groups;
	uint64_t k[GG_MAX_KEYS];
	uint32_t knull;
	EmuGroup *cur;
	unsigned long long npassed;

	void begin_row() { memset(k, 0, sizeof k); knull = 0; cur = nullptr; }
	bool filter(bool pass) { return pass; }
	void key(int kc, uint64_t v, bool isnull)
	{
		if (isnull) { knull |= 1u << kc; return; }
		k[kc] = group_key(v, P->keytype[kc]);
	}
	bool group(bool live)
	{
		if (!live) { cur = nullptr; return false; }
		std::array<uint64_t, GG_MAX_KEYS + 1> id;
		for (int i = 0; i < GG_MAX_KEYS; i++) id[i] = (i < P->nkeys && !((knull >> i) & 1)) ? normalize_key(k[i], P->keytype[i]) : 0;
		id[GG_MAX_KEYS] = knull;
		auto it = groups.find(id);
		if (it == groups.end())
		{
			EmuGroup g;
			memset(&g, 0, sizeof g);
			for (int j = 0; j < P->nacc; j++)                  /* float8 sums start from -0, as the kernels' accumulators do */
				if (P->acckind[j] == GGP_ACC_F8SUM) g.sum[j] = -0.0;
			for (int i = 0; i < GG_MAX_KEYS; i++) g.key[i] = (i < P->nkeys && !((knull >> i) & 1)) ? k[i] : 0;     /* the first row's key */
			g.keynull = knull;
			it = groups.emplace(id, g).first;
		}
		cur = &it->second;
		cur->count++;
		npassed++;
		return true;
	}
	/* slot j < nacc is accumulator column j; a slot >= nacc is the sum of squares of the column whose accsq names it */
	void out(int slot, double v, bool isnull)
	{
		if (!cur || isnull) return;
		if (slot >= P->nacc)
		{
			for (int j = 0; j < P->nacc; j++)
				if (P->accsq[j] == slot) cur->sumsq[j] = cur->sumsq[j] + v;
			return;
		}
		const int kind = P->acckind[slot];
		double &s = cur->sum[slot];
		uint64_t &nn = cur->n[slot];
		const long long vi = __double_as_longlong(v), si = __double_as_longlong(s);
		switch (kind)
		{
			case GGP_ACC_F8SUM: s = s + v; break;
			case GGP_ACC_I8SUM: s = __longlong_as_double(si + vi); break;
			case GGP_ACC_F8MIN: if (nn == 0 || f8_cmp(v, s) < 0) s = v; break;
			case GGP_ACC_F8MAX: if (nn == 0 || f8_cmp(v, s) > 0) s = v; break;
			case GGP_ACC_I8MIN: if (nn == 0 || vi < si) s = v; break;
			case GGP_ACC_I8MAX: if (nn == 0 || vi > si) s = v; break;
			default: break;                              /* GGP_ACC_COUNT: only n */
		}
		nn++;
	}
};

template <bool NULLABLE>
static void run_pages(const ggp_program &P, const uint8_t *pages, uint64_t nblocks, HostSink &sink, uint32_t &err, uint64_t &scanned)
{
	const uint32_t PG = 0, OFFS = GG_BLCKSZ + 1024;         /* page at 0, the per-lane offset scratch after it */
	for (uint64_t b = 0; b < nblocks; b++)
	{
		memcpy(gg_emu_smem + PG, pages + b * (uint64_t) GG_BLCKSZ, GG_BLCKSZ);
		const uint32_t pd_lower = lds16(PG + 12);
		const int nitems = pd_lower >= GG_PAGE_HEADER_SIZE ? (int) ((pd_lower - GG_PAGE_HEADER_SIZE) >> 2) : 0;
		for (int i = 0; i < nitems; i++)
		{
			const uint32_t lp = lds32(PG + GG_PAGE_HEADER_SIZE + 4 * (uint32_t) i);
			const uint32_t off = lp & 0x7FFF, flags = (lp >> 15) & 3, len = lp >> 17;
			if (flags != 1) continue;                       /* LP_NORMAL */
			const uint32_t tup = PG + off;
			const bool hasnulls = (lds16(tup + 20) & GG_HEAP_HASNULL) != 0;
			EvalCtx X;
			memset(&X, 0, sizeof X);
			X.P = &P; X.offs = OFFS; X.lane = 0; X.fast = !hasnulls;
			uint32_t e0 = err;
			walk_tuple(P.outer, tup, len, X.fast, OFFS, 0, X.tv, err);
			scanned++;
			bool live = !(err != e0 && (err & GGP_EF_BADPAGE));
			if (!NULLABLE && X.tv.colnull) { err |= GGP_EF_NOTNULL_VIOLATED; live = false; }
			sink.begin_row();
			run_prog<NULLABLE, false>(X, live, err, sink);
		}
	}
}

/* GG_FMT_DATUMROWS input (what a receiving Motion delivers and what gg_aocs_decode_rows produces): the datum-row front end of
 * scanagg_body — NULL mask word, then one 64-bit word per column at constant offsets (gg_scanagg_kernel.cuh) */
template <bool NULLABLE>
static void run_rows(const ggp_program &P, const uint64_t *rows, uint64_t nrows, HostSink &sink, uint32_t &err, uint64_t &scanned)
{
	const uint32_t RP = 0, rowwords = (uint32_t) P.outer.rowwords;
	for (uint64_t r = 0; r < nrows; r++)
	{
		memcpy(gg_emu_smem + RP, rows + r * rowwords, (size_t) rowwords * 8);
		EvalCtx X;
		memset(&X, 0, sizeof X);
		X.P = &P; X.offs = 65536; X.lane = 0; X.fast = true;
		X.tv.tp = RP + 8;
		uint32_t cn = 0;
		const uint64_t mask = lds64(RP);
		for (int sl = 0; sl < P.outer.ncols; sl++) cn |= (uint32_t) ((mask >> P.outer.colatt[sl]) & 1) << sl;
		X.tv.colnull = cn;
		bool live = true;
		scanned++;
		if (!NULLABLE && cn) { err |= GGP_EF_NOTNULL_VIOLATED; live = false; }
		sink.begin_row();
		run_prog<NULLABLE, false>(X, live, err, sink);
	}
}

/* compile with the product's compiler, run with the product's interpreter; groups come back as EmuGroup records */
extern "C" int emu_scanagg(const gg_scan *scan, const gg_agg *agg, const gg_exprpool *pool, const uint8_t *pages, uint64_t nblocks,
                           EmuGroup *out, int cap, int *nout, int32_t *aggcol /* [GG_MAX_AGGS] */, int32_t *accsq /* [GGP_MAX_ACCS] */,
                           uint64_t *scanned, uint64_t *passed, uint32_t *errflags, char *msg, int msglen)
{
	static ggp_program P;
	ggp_aggmap aggmap[GG_MAX_AGGS];
	int rc = ggp_compile_scanagg(scan, agg, pool, &P, aggmap, msg, msglen);
	if (rc != GG_OK) return rc;
	HostSink sink;
	sink.P = &P; sink.npassed = 0; sink.cur = nullptr;
	uint32_t err = 0;
	uint64_t nscan = 0;
	if (P.outer.rowwords > 0)
	{
		/* datum rows: `pages` is the row array, `nblocks` the row count */
		if (P.nullable) run_rows<true>(P, (const uint64_t *) pages, nblocks, sink, err, nscan);
		else run_rows<false>(P, (const uint64_t *) pages, nblocks, sink, err, nscan);
	}
	else if (P.nullable) run_pages<true>(P, pages, nblocks, sink, err, nscan);
	else run_pages<false>(P, pages, nblocks, sink, err, nscan);
	if (P.nkeys == 0 && sink.groups.empty())               /* plain aggregate over no rows: the one group exists (count 0) */
	{
		sink.begin_row();
		std::array<uint64_t, GG_MAX_KEYS + 1> id{};
		EmuGroup g; memset(&g, 0, sizeof g);
		sink.groups.emplace(id, g);
	}
	int n = 0;
	for (auto &kv : sink.groups)
	{
		if (n >= cap) return GG_ERR_NOMEM;
		out[n++] = kv.second;
	}
	*nout = n;
	for (int i = 0; i < agg->numAggs; i++) aggcol[i] = aggmap[i].col;
	for (int j = 0; j < GGP_MAX_ACCS; j++) accsq[j] = P.accsq[j];
	*scanned = nscan; *passed = sink.npassed; *errflags = err;
	return GG_OK;
}

/* the device hashing and routing functions (gg_device.cuh), for the golden vectors the reference's own objects produced */
extern "C" uint32_t emu_hash_uint32(uint32_t k) { return hash_uint32(k); }
extern "C" uint32_t emu_hashint8(int64_t v) { return hashint8(v); }
extern "C" uint32_t emu_hashfloat8(uint64_t bits) { return hashfloat8(bits); }
extern "C" uint32_t emu_hash_any_le8(uint64_t v, int len) { return hash_any_le8(v, len); }
extern "C" int32_t emu_route(const int32_t *typids, const int64_t *vals, const int32_t *lens, const int32_t *isnull, int nkeys, int nsegs)
{
	/* the kernels' key_hash; a string's length is where its packed bytes end, so `lens` is not read */
	(void) lens;
	uint32_t h = 0;
	for (int i = 0; i < nkeys; i++)
		h = cdbhash_add(h, isnull[i] ? 0 : key_hash(ggp_hashtype_of(typids[i]), (uint64_t) vals[i]), isnull[i] != 0);
	return jump_consistent_hash((uint64_t) h, nsegs);
}

/* The device's attribute walk over ONE tuple (walk_tuple, slot_deform_tuple's restatement for the GPU): every attribute of
 * the descriptor is referenced through a count(col) plan so that the compiled side description covers them all.
 * values[a]: the Datum of a fixed-width attribute as the interpreter's loads read it (LD_C8 / LD_C4), or for a varlena the
 * offset of its header byte from the tuple start — the convention of tests/golden/heap_kat.json. */
extern "C" int emu_walk(const gg_tupdesc *desc, const uint8_t *tuple, int len, int force_slow, int64_t *values, uint8_t *nulls, uint32_t *errflags)
{
	static gg_scan scan; static gg_agg agg; static gg_exprpool pool; static ggp_program P;
	ggp_aggmap aggmap[GG_MAX_AGGS];
	char msg[256];
	if (desc->natts < 1 || desc->natts > GG_MAX_AGGS) return GG_ERR_ARG;
	memset(&scan, 0, sizeof scan); memset(&agg, 0, sizeof agg); memset(&pool, 0, sizeof pool);
	scan.desc = *desc; scan.qual = -1;
	for (int a = 0; a < desc->natts; a++)
	{
		gg_expr &e = pool.nodes[pool.nnodes];
		e.kind = GG_E_VAR; e.varno = 0; e.varattno = (int16_t) (a + 1); e.rettype = desc->attrs[a].atttypid;
		agg.aggs[a].aggfnoid = GG_AGG_COUNT_ANY; agg.aggs[a].arg = pool.nnodes++;
	}
	agg.numAggs = desc->natts;
	int rc = ggp_compile_scanagg(&scan, &agg, &pool, &P, aggmap, msg, sizeof msg);
	if (rc != GG_OK) return rc;
	const uint32_t TUP = 64, OFFS = 40000;
	memset(gg_emu_smem, 0xEE, 65536);
	memcpy(gg_emu_smem + TUP, tuple, (size_t) len);
	const bool hasnulls = (lds16(TUP + 20) & GG_HEAP_HASNULL) != 0;
	const bool fast = !hasnulls && !force_slow;
	TupleView tv;
	uint32_t err = 0;
	walk_tuple(P.outer, TUP, (uint32_t) len, fast, OFFS, 0, tv, err);
	*errflags = err;
	for (int a = 0; a < desc->natts; a++) { nulls[a] = 2; values[a] = 0; }       /* 2 = not referenced (cannot happen here) */
	for (int s = 0; s < P.outer.ncols; s++)
	{
		const int a = P.outer.colatt[s];
		nulls[a] = (uint8_t) ((tv.colnull >> s) & 1);
		if (nulls[a]) continue;
		const int cacheoff = P.outer.att[a].cacheoff;
		const uint32_t off = (fast && cacheoff >= 0) ? (uint32_t) cacheoff : lds16(OFFS + (uint32_t) (s * 32) * 2);
		const uint32_t addr = tv.tp + off;
		switch (desc->attrs[a].attlen)
		{
			case 8: values[a] = (int64_t) lds64(addr); break;
			case 4: values[a] = (int64_t) (int32_t) lds32(addr); break;
			case 2: values[a] = (int64_t) (int16_t) lds16(addr); break;
			case 1: values[a] = (int64_t) (int8_t) lds8(addr); break;
			default: values[a] = (int64_t) (addr - TUP); break;
		}
	}
	return GG_OK;
}

/* the device's HeapTupleSatisfiesMVCC (gg_device.cuh) over one tuple header and a snapshot in the device layout:
 * 1 visible, 0 not, -1 GGP_EF_VISIBILITY raised */
extern "C" int emu_tuple_satisfies_mvcc(const uint8_t *header, const uint32_t *snap_words)
{
	memcpy(gg_emu_smem, header, 24);
	uint16_t infomask;
	memcpy(&infomask, header + 20, 2);
	uint32_t err = 0;
	const bool vis = heap_tuple_satisfies_mvcc(0, infomask, snap_words, err);
	if (err & GGP_EF_VISIBILITY) return -1;
	return vis ? 1 : 0;
}
