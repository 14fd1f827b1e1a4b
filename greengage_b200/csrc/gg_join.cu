/*
 * gg_join.cu — Hash / HashJoin (+ the Agg above): the build kernel and the probe into the general HashAggregate (interpreter
 * path), and the host pipeline behind gg_joinagg_* (include/ggb200.h).  The probe side IS a gg_scanagg pipeline (gg_pipeline.h)
 * whose row program has a per-match piece; everything after the probe (merge, fetch, escalation to the general HashAggregate)
 * is shared, and gg_scanagg.cu launches its kernels.  A join with a target list (gg_joinrows_create) is the same pipeline whose
 * probe writes every joined row as a datum row instead (MODE_PART with JOIN = true: JoinRowSink).
 */
#include "gg_pipeline.h"
#include "gg_groups.h"

using namespace ggd;

/* Hash node: scan the inner relation into the join hash table */
__global__ void __launch_bounds__(256, 2)
gg_joinbuild_kernel(const __grid_constant__ ggp_program P, const ScanAggParams prm)
{
	scanagg_body<MODE_BUILD, DynPlan>(P, prm);
}

/* probe feeding the general HashAggregate (any number of groups) */
__global__ void __launch_bounds__(256, 2)
gg_joinhash_kernel(const __grid_constant__ ggp_program P, const ScanAggParams prm)
{
	scanagg_body<MODE_HASH, DynPlan, true>(P, prm);
}

/* probe writing the joined rows of a join with a target list */
__global__ void __launch_bounds__(256, 2)
gg_joinrows_kernel(const __grid_constant__ ggp_program P, const ScanAggParams prm)
{
	scanagg_body<MODE_PART, DynPlan, true>(P, prm);
}

/* upper bound on the inner rows = line pointers of the pages (exact for a freshly loaded relation) */
__global__ void gg_count_lp_kernel(const uint8_t *pages, uint64_t nblocks, unsigned long long *out)
{
	unsigned long long n = 0;
	for (uint64_t b = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; b < nblocks; b += (uint64_t) gridDim.x * blockDim.x)
	{
		const uint32_t w3 = *(const uint32_t *) (pages + b * GG_BLCKSZ + 12);
		const uint32_t pd_lower = w3 & 0xFFFF;
		if (pd_lower >= GG_PAGE_HEADER_SIZE && pd_lower <= GG_BLCKSZ) n += (pd_lower - GG_PAGE_HEADER_SIZE) >> 2;
	}
	for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(GG_FULL_MASK, n, o);
	if ((threadIdx.x & 31) == 0 && n) atomicAdd(out, n);
}

/* ExecReScanHashJoin with the table kept: forget which entries matched */
__global__ void gg_clear_matched_kernel(unsigned long long *ent, uint64_t slots, uint32_t stride)
{
	for (uint64_t i = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; i < slots; i += (uint64_t) gridDim.x * blockDim.x)
		ent[i * stride] &= ~GG_HT_MATCHED;
}

extern "C" {

/* how many tuples a relation holds at most: line pointers of its heap pages (exact for a loaded relation without dead
 * items), or the row count of datum rows.  Sizes Motion buffers and hash tables (ExecChooseHashTableSize sizes from the
 * planner's estimate, nodeHash.c:463; the pages give a tight bound for one pass over their headers). */
int gg_relation_count_rows(gg_relation *r, uint64_t *nrows)
{
	if (!r || !nrows) return GG_ERR_ARG;
	if (r->rowwords) { *nrows = r->nrows; return GG_OK; }
	gg_engine *e = r->eng;
	GG_CUDA(cudaSetDevice(e->device));
	unsigned long long *d = nullptr, n = 0;
	GG_CUDA(cudaMalloc((void **) &d, sizeof n));
	cudaError_t ce = cudaMemsetAsync(d, 0, sizeof n, e->stream);
	if (ce == cudaSuccess)
	{
		gg_count_lp_kernel<<<e->sm_count, 256, 0, e->stream>>>(r->pages, r->nblocks, d);
		ce = cudaGetLastError();
		e->launches++;
	}
	if (ce == cudaSuccess) ce = cudaMemcpyAsync(&n, d, sizeof n, cudaMemcpyDeviceToHost, e->stream);
	if (ce == cudaSuccess) ce = cudaStreamSynchronize(e->stream);
	cudaFree(d);
	if (ce != cudaSuccess) return gg_cuda_fail(ce, "gg_relation_count_rows");
	*nrows = n;
	return GG_OK;
}

/* =====================================================================================
 * HashJoin + Agg (include/ggb200.h gg_joinagg_*)
 * ===================================================================================== */
struct gg_joinagg {
	gg_engine *eng = nullptr;
	ggp_joinprog jp;
	gg_scanagg *probe = nullptr;    /* the probe-side pipeline (outer scan -> probe -> Agg) */
	unsigned long long *ent = nullptr, *d_cnt = nullptr;   /* d_cnt[0] line-pointer count, [1] rows inserted */
	uint64_t slots = 0;
	uint32_t stride = 0;            /* 64-bit words per table entry */
	size_t ent_bytes = 0;           /* size of the allocation behind ent (kept across builds of the same size) */
	uint64_t rows_built = 0, null_keys = 0;
	bool filled = false;            /* right / full join: the unmatched inner rows have been emitted */
	bool lasj_empty = false;        /* LASJ_NOTIN met a NULL inner key: the result is empty */
	float build_ms = 0;
	cudaEvent_t ev0 = nullptr, ev1 = nullptr;
	unsigned long long *d_buildcnt = nullptr;   /* rows scanned / passed by the build kernel (kept apart from the probe's counters),
	                                             * then the build kernel's error flags */
	/* hybrid hash join (nodeHash.c:713,1132; gg_joinagg_set_work_mem / gg_joinagg_run): the plan as given, and what a
	 * batched run builds from it */
	gg_scan outer_scan, inner_scan;
	gg_hashjoin hj;
	gg_agg agg;
	gg_exprpool pool;
	uint64_t work_mem = 0;
	int nbatch = 1;                 /* batches of the last run */
	int log2_nbuckets = 0;
	gg_joinagg *bj = nullptr;       /* the join of one batch pair: the same plan over the partitions' datum rows */
	gg_exprpool *ipool = nullptr;   /* `pool` with the inner side's Vars as varno 0: what partitions the inner relation */
	int32_t otargets[GGP_MAX_ACCS], itargets[GGP_MAX_ACCS];   /* expression roots that travel, per side: join keys first */
	int notargets = 0, nitargets = 0;
	gg_relation *obuf = nullptr, *ibuf = nullptr;            /* the partitions: nbatch regions of datum rows each */
	uint64_t ocap = 0, icap = 0;                             /* rows per region */
	std::vector<uint64_t> ocounts, icounts;
	float part_ms = 0;
	/* a join with a target list (gg_joinrows_create): the probe writes its rows here instead of feeding `agg` (all zero) */
	int ntargets = 0;
	int32_t targets[16];
	gg_relation *rows_buf = nullptr;            /* owned: datum rows of 1 + ntargets words, probe->mo.cap of them */
	unsigned long long *d_rowcur = nullptr;     /* probe->mo.cursor: rows claimed, counted on past the capacity */
	gg_relation *rows_view = nullptr;           /* what gg_joinagg_rows handed out (until reset / free) */
	uint64_t rows_n = 0, rows_live = 0;
};

/* agg == nullptr: a join with a target list */
static int joinagg_create(gg_engine *e, const gg_scan *outer, const gg_scan *inner, const gg_hashjoin *hj, const gg_agg *agg,
                          const int32_t *targets, int ntargets, const gg_exprpool *pool, gg_joinagg **out)
{
	*out = nullptr;
	GG_CUDA(cudaSetDevice(e->device));
	gg_joinagg *j = new gg_joinagg();
	j->eng = e;
	gg_scanagg *p = new gg_scanagg();
	p->eng = e;
	p->scan = *outer;
	memset(&p->agg, 0, sizeof p->agg);
	if (agg) p->agg = *agg;
	p->pool = *pool;
	p->is_join = true;
	p->join_rows = agg == nullptr;
	char msg[256];
	int rc = agg ? ggp_compile_join(outer, inner, hj, agg, pool, &j->jp, p->aggmap, msg, sizeof msg)
	             : ggp_compile_joinrows(outer, inner, hj, targets, ntargets, pool, &j->jp, msg, sizeof msg);
	if (rc != GG_OK) { gg_set_error("%s", msg); delete p; delete j; return rc; }
	p->prog = j->jp.probe;
	p->join_probe_pc = j->jp.probe_pc;
	p->prog.nullable = p->prog.nullable || j->jp.build.nullable;     /* a NULL payload column shows up on the probe side */
	if (p->prog.nullable) p->prog.priv_ok = 0;
	rc = scanagg_finish_create(p, &j->probe);
	if (rc) { delete j; return rc; }
	j->outer_scan = *outer; j->inner_scan = *inner; j->hj = *hj; j->agg = p->agg; j->pool = *pool;
	if (!agg)
	{
		j->ntargets = ntargets;
		memcpy(j->targets, targets, sizeof(int32_t) * (size_t) ntargets);
		GG_CUDA(cudaMalloc((void **) &j->d_rowcur, sizeof(unsigned long long)));
		GG_CUDA(cudaMemsetAsync(j->d_rowcur, 0, sizeof(unsigned long long), e->stream));
		j->probe->mo.cursor = j->d_rowcur;
	}
	GG_CUDA(cudaMalloc((void **) &j->d_cnt, 4 * sizeof(unsigned long long)));      /* line pointers | nbuilt[0..2] (JoinTable) */
	GG_CUDA(cudaMalloc((void **) &j->d_buildcnt, 3 * sizeof(unsigned long long)));      /* rows scanned | passed | error flags */
	GG_CUDA(cudaEventCreate(&j->ev0));
	GG_CUDA(cudaEventCreate(&j->ev1));
	*out = j;
	return GG_OK;
}

int gg_joinagg_create(gg_engine *e, const gg_scan *outer, const gg_scan *inner, const gg_hashjoin *hj,
                      const gg_agg *agg, const gg_exprpool *pool, gg_joinagg **out)
{
	if (!e || !outer || !inner || !hj || !agg || !pool || !out) return GG_ERR_ARG;
	return joinagg_create(e, outer, inner, hj, agg, nullptr, 0, pool, out);
}

int gg_joinrows_create(gg_engine *e, const gg_scan *outer, const gg_scan *inner, const gg_hashjoin *hj,
                       const int32_t *targets, int ntargets, const gg_exprpool *pool, gg_joinagg **out)
{
	if (!e || !outer || !inner || !hj || !targets || !pool || !out) return GG_ERR_ARG;
	return joinagg_create(e, outer, inner, hj, nullptr, targets, ntargets, pool, out);
}

/* a right / full join also writes the inner rows no outer row matched (the fill-inner launch after every probe) */
static bool joinrows_fill_inner(const gg_joinagg *j)
{
	return j->jp.jointype == GG_JOIN_RIGHT || j->jp.jointype == GG_JOIN_FULL;
}

/* Room for `rows` joined rows written by `launches` kernel launches, plus the claim windows' slack: the probe's warps claim
 * rows `window` at a time (as a sending Motion does, MotionOut.window), and every launch starts with empty windows and marks
 * what each warp left unused of its last one dead, so each launch leaves at most one window per warp partly unused.  The
 * window is sized from the rows of one launch, which keeps all tails together below 1/8 of the rows.  Keeps a buffer that is
 * large enough already. */
static int joinrows_reserve(gg_joinagg *j, uint64_t rows, uint64_t launches)
{
	gg_scanagg *p = j->probe;
	const uint64_t warps = (uint64_t) p->grid * (uint64_t) (p->cfg.threads / 32 - 1);
	if (launches < 1) launches = 1;
	const uint64_t w = rows / launches / (warps * 8);
	uint32_t window = 0;
	if (w >= 32) { window = 32; while (window * 2 <= w && window < 1024) window *= 2; }
	const uint64_t cap = (rows + launches * warps * window + 1) & ~1ull;
	const uint64_t W = 1 + (uint64_t) j->ntargets;
	const uint64_t nb = ((cap * W + 8) * 8 + GG_BLCKSZ - 1) / GG_BLCKSZ;      /* + 64 bytes: bulk copies read whole 16 bytes */
	if (j->rows_buf && j->rows_buf->nblocks < nb) { GG_CUDA(cudaStreamSynchronize(j->eng->stream)); gg_relation_free(j->rows_buf); j->rows_buf = nullptr; }
	if (!j->rows_buf)
	{
		int rc = gg_relation_create(j->eng, nb, &j->rows_buf);
		if (rc) { j->rows_buf = nullptr; gg_set_error("join output of %llu rows does not fit in device memory", (unsigned long long) cap); return rc; }
	}
	MotionOut &mo = p->mo;
	mo.rows = (unsigned long long *) j->rows_buf->pages;
	mo.cap = cap;
	mo.nsegs = 1;
	mo.rowwords = (int) W;
	mo.hashtypes = 0;
	mo.window = window;
	mo.route = 0; mo.shift = 0;
	return GG_OK;
}

/* MultiExecHash: size the table from the inner relation's line pointers (ExecChooseHashTableSize sizes from the
 * planner's row estimate, nodeHash.c:463; the pages give a tight bound for free), then one scan inserts. */
int gg_joinagg_build(gg_joinagg *j, gg_relation *inner, uint64_t first_block, uint64_t nblocks)
{
	if (!j || !inner || nblocks > inner->nblocks || first_block > inner->nblocks - nblocks) return GG_ERR_ARG;
	if (j->rows_view) { gg_set_error("the joined rows were already handed out: reset before building again"); return GG_ERR_ARG; }
	if (inner->rowwords != j->jp.build.outer.rowwords) { gg_set_error("inner relation format does not match the plan's tuple descriptor"); return GG_ERR_ARG; }
	if (inner->rowwords && (first_block != 0 || nblocks != inner->nblocks)) { gg_set_error("datum-row relations are scanned whole"); return GG_ERR_ARG; }
	gg_engine *e = j->eng;
	cudaStream_t st = e->stream;
	GG_CUDA(cudaSetDevice(e->device));
	const uint8_t *pages = inner->pages + first_block * GG_BLCKSZ;
	GG_CUDA(cudaMemsetAsync(j->d_cnt, 0, 4 * sizeof(unsigned long long), st));
	GG_CUDA(cudaEventRecord(j->ev0, st));
	unsigned long long nlp = inner->nrows;
	if (!inner->rowwords)
	{
		gg_count_lp_kernel<<<e->sm_count, 256, 0, st>>>(pages, nblocks, j->d_cnt);
		GG_CUDA(cudaGetLastError());
		e->launches++;
		GG_CUDA(cudaMemcpyAsync(&nlp, j->d_cnt, sizeof nlp, cudaMemcpyDeviceToHost, st));
		GG_CUDA(cudaStreamSynchronize(st));
	}
	uint64_t slots = 1024;
	while (slots < 2 * (uint64_t) nlp) slots <<= 1;
	if (slots > (1ull << 31)) { gg_set_error("inner relation too large for one hash table (%llu rows)", nlp); return GG_ERR_NOMEM; }
	JoinTable jt;
	memset(&jt, 0, sizeof jt);
	/* header | keys | payload, padded to a whole 32-byte sector when that costs one word: an entry of 3 (7) words becomes 4
	 * (8), so a probe step — header, keys and payload — touches exactly one (two) sectors instead of straddling */
	jt.stride = (uint32_t) (1 + j->jp.nkeys + j->jp.npayload);
	if ((jt.stride & 3) == 3) jt.stride++;
	jt.mask = (uint32_t) (slots - 1);
	jt.nkeys = j->jp.nkeys;
	jt.npayload = j->jp.npayload;
	jt.jointype = j->jp.jointype;
	jt.probe_pc = j->jp.probe_pc;
	jt.keepnull = jt.mark_matched = (j->jp.jointype == GG_JOIN_RIGHT || j->jp.jointype == GG_JOIN_FULL);
	for (int k = 0; k < j->jp.nkeys; k++) jt.keytypes |= (uint32_t) j->jp.keytype[k] << (2 * k);
	const size_t bytes = (size_t) slots * jt.stride * 8;
	if (j->ent && j->ent_bytes != bytes) { cudaFree(j->ent); j->ent = nullptr; }      /* a rescan of the same inner side keeps the allocation */
	if (!j->ent)
	{
		cudaError_t ce = cudaMalloc((void **) &j->ent, bytes + 64);      /* slack: the fill-inner pass reads it in 16-byte multiples */
		if (ce != cudaSuccess) { cudaGetLastError(); j->ent = nullptr; gg_set_error("hash table of %zu bytes does not fit in device memory", bytes); return GG_ERR_NOMEM; }
		j->ent_bytes = bytes;
	}
	GG_CUDA(cudaMemsetAsync(j->ent, 0, bytes, st));
	jt.ent = j->ent;
	jt.nbuilt = j->d_cnt + 1;
	j->slots = slots;
	j->stride = jt.stride;

	ScanAggParams prm;
	memset(&prm, 0, sizeof prm);
	prm.pages = pages;
	prm.nblocks = nblocks;
	uint32_t *d_builderr = (uint32_t *) (j->d_buildcnt + 2);
	GG_CUDA(cudaMemsetAsync(d_builderr, 0, sizeof(uint32_t), st));
	prm.errflags = d_builderr;
	prm.snap = e->d_snapshot;
	prm.counters = j->d_buildcnt;           /* the probe's counters describe the outer side only */
	const gg_launch c = gg_np_launch(2, ((j->jp.build.outer.ncols * 64 + 15) & ~15) + 16);
	prm.nstage = c.nstage;
	prm.team = c.team;
	prm.scratch_per_warp = c.scratch_per_warp;
	prm.scratch_off = c.scratch_off;
	prm.jt = jt;
	prm.nrows = inner->nrows;
	const void *fn = nullptr;
	int rc = gg_scan_kernel(&j->jp.build, MODE_BUILD, -1, c, e->device, e->d_snapshot != nullptr, &fn);
	if (rc) return rc;
	void *args[] = { (void *) &j->jp.build, (void *) &prm };
	GG_CUDA(cudaLaunchKernel(fn, dim3(e->sm_count * c.ctas), dim3(c.threads), args, c.smem, st));
	GG_CUDA(cudaGetLastError());
	e->launches++;
	GG_CUDA(cudaEventRecord(j->ev1, st));
	unsigned long long nb[3] = { 0, 0, 0 };
	GG_CUDA(cudaMemcpyAsync(nb, j->d_cnt + 1, sizeof nb, cudaMemcpyDeviceToHost, st));
	uint32_t builderr = 0;
	GG_CUDA(cudaMemcpyAsync(&builderr, d_builderr, sizeof builderr, cudaMemcpyDeviceToHost, st));
	GG_CUDA(cudaStreamSynchronize(st));
	j->probe->build_err = builderr & ~(uint32_t) GGP_EF_INFO_MASK;
	GG_CUDA(cudaEventElapsedTime(&j->build_ms, j->ev0, j->ev1));
	j->rows_built = nb[0];
	j->null_keys = nb[1];
	jt.inner_empty = nb[0] == 0;
	{
		/* no insert passed an entry with its own hash tag: the inner join keys are pairwise distinct (orders.o_orderkey under
		 * lineitem) and a probing row stops at its first key match.  GGB200_JOIN_UNIQUE=0 keeps the full scan to the empty slot
		 * (experiments). */
		const char *ju = getenv("GGB200_JOIN_UNIQUE");
		jt.unique = nb[2] == 0 && !(ju && atoi(ju) == 0);
	}
	j->lasj_empty = j->jp.jointype == GG_JOIN_LASJ_NOTIN && nb[1] > 0;      /* nodeHashjoin.c:238 */
	j->filled = false;
	j->probe->jt = jt;
	return GG_OK;
}

int gg_joinagg_probe(gg_joinagg *j, gg_relation *outer, uint64_t first_block, uint64_t nblocks)
{
	if (!j || !outer) return GG_ERR_ARG;
	if (j->filled) { gg_set_error("the unmatched inner rows were already emitted: reset before probing again"); return GG_ERR_ARG; }
	if (j->rows_view) { gg_set_error("the joined rows were already handed out: reset before probing again"); return GG_ERR_ARG; }
	if (j->ntargets && !j->rows_buf)
	{
		/* the output is sized once, from the outer rows (+ the inner rows a right / full join may add); gg_joinagg_rows grows
		 * it and probes again if the join turns out to produce more */
		uint64_t nouter = 0;
		int rc = gg_relation_count_rows(outer, &nouter);
		if (rc == GG_OK) rc = joinrows_fill_inner(j) ? joinrows_reserve(j, nouter + j->rows_built, 2) : joinrows_reserve(j, nouter, 1);
		if (rc) return rc;
	}
	if (j->lasj_empty) return GG_OK;          /* x NOT IN (.., NULL, ..): no outer row can qualify */
	return gg_scanagg_run(j->probe, outer, first_block, nblocks);
}

int gg_joinagg_probe_host(gg_joinagg *j, const void *host_pages, uint64_t nblocks)
{
	if (!j) return GG_ERR_ARG;
	if (j->ntargets) { gg_set_error("a join with a target list probes device-resident relations"); return GG_ERR_UNSUPPORTED; }
	if (j->filled) { gg_set_error("the unmatched inner rows were already emitted: reset before probing again"); return GG_ERR_ARG; }
	if (j->lasj_empty) return GG_OK;
	return gg_scanagg_run_host(j->probe, host_pages, nblocks);
}

/* HJ_FILL_INNER_TUPLES of a right / full join, for the table as it stands (nodeHashjoin.c:460-490) */
static int joinagg_fill_inner(gg_joinagg *j)
{
	if (j->probe->jt.mark_matched && !j->filled && j->ent)
	{
		/* HJ_FILL_INNER_TUPLES: every outer row has been through the probe; what is still unmatched in the table comes
		 * out with a null-extended outer side.  The table is scanned by the probe kernel itself, as rows of entries. */
		gg_scanagg *p = j->probe;
		const JoinTable &jt = p->jt;
		const uint64_t per_chunk = (GG_BLCKSZ / (8ull * jt.stride)) & ~1ull;
		const uint64_t chunks = (j->slots + per_chunk - 1) / per_chunk;
		GG_CUDA(cudaSetDevice(j->eng->device));
		int rc = scanagg_launch(p, (const uint8_t *) j->ent, chunks, j->eng->stream, j->slots, true);
		if (rc) return rc;
		p->fed.push_back({ (const uint8_t *) j->ent, nullptr, chunks, j->slots, true, 0 });
		j->filled = true;
	}
	return GG_OK;
}

int gg_joinagg_fetch(gg_joinagg *j, gg_aggrow *out, int outcap, int *nout, uint64_t *rows_joined)
{
	if (!j) return GG_ERR_ARG;
	if (j->ntargets) { gg_set_error("a join with a target list returns rows (gg_joinagg_rows), not aggregate rows"); return GG_ERR_ARG; }
	if (j->bj && j->nbatch > 1) return gg_scanagg_fetch(j->bj->probe, out, outcap, nout, nullptr, rows_joined);   /* every batch was filled as it went */
	int rc = joinagg_fill_inner(j);
	if (rc) return rc;
	return gg_scanagg_fetch(j->probe, out, outcap, nout, nullptr, rows_joined);
}

/* the joined-and-aggregated groups as datum rows: the last pass as gg_joinagg_fetch runs it, then the probe pipeline's rows */
int gg_joinagg_datumrows(gg_joinagg *j, gg_relation **rows, uint64_t *nrows)
{
	if (!j) return GG_ERR_ARG;
	if (j->ntargets) { gg_set_error("a join with a target list returns rows (gg_joinagg_rows), not aggregate rows"); return GG_ERR_ARG; }
	if (j->bj && j->nbatch > 1) return gg_scanagg_datumrows(j->bj->probe, rows, nrows);     /* every batch was filled as it went */
	int rc = joinagg_fill_inner(j);
	if (rc) return rc;
	return gg_scanagg_datumrows(j->probe, rows, nrows);
}

/* ---- hybrid hash join: batches (nodeHash.c:713 ExecHashIncreaseNumBatches, :1132 ExecHashGetBucketAndBatch) ----
 * When the hash table of the whole inner side would not fit the operator's memory, both inputs are split by the batch bits
 * of the join's hash value — the reference's hash function (per key: rotate left one bit, xor the key type's hash function,
 * nodeHash.c:1044-1085) and its bit usage (batchno = (hashvalue >> log2_nbuckets) & (nbatch - 1)) — with the kernel that
 * also sends Motions, into nbatch regions of datum rows each (the columns the join and the aggregate above it need; the
 * scan quals are applied on the way), and the batches are joined pair by pair into ONE aggregate state.  Where the reference
 * writes batch files (nodeHashjoin.c:906,1083), the partitions stay in device memory: the budget bounds the hash table. */
static void collect_vars(const gg_exprpool &pool, int32_t root, int varno, std::vector<int32_t> &nodes)
{
	if (root < 0 || root >= pool.nnodes) return;
	const gg_expr &x = pool.nodes[root];
	if (x.kind == GG_E_VAR)
	{
		if (x.varno != varno) return;
		for (int32_t n : nodes) if (pool.nodes[n].varattno == x.varattno) return;
		nodes.push_back(root);
		return;
	}
	for (int a = 0; a < x.nargs && a < 2; a++) collect_vars(pool, x.args[a], varno, nodes);
}

/* compile the batch-pair join: the plan with every Var above the join renumbered to its column in the partition rows */
static int joinagg_prepare_batches(gg_joinagg *j)
{
	if (j->bj) return GG_OK;
	const gg_exprpool &pool = j->pool;
	std::vector<int32_t> ov, iv;
	const int32_t above[] = { j->hj.joinqual };
	for (int32_t r : above) { collect_vars(pool, r, 0, ov); collect_vars(pool, r, 1, iv); }
	for (int t = 0; t < j->ntargets; t++) { collect_vars(pool, j->targets[t], 0, ov); collect_vars(pool, j->targets[t], 1, iv); }
	for (int c = 0; c < j->agg.numCols; c++) { collect_vars(pool, j->agg.grpCol[c], 0, ov); collect_vars(pool, j->agg.grpCol[c], 1, iv); }
	for (int a = 0; a < j->agg.numAggs; a++) { collect_vars(pool, j->agg.aggs[a].arg, 0, ov); collect_vars(pool, j->agg.aggs[a].arg, 1, iv); }
	const int nk = j->hj.nkeys;
	if (nk + (int) ov.size() > GGP_MAX_ACCS || nk + (int) iv.size() > GGP_MAX_ACCS || pool.nnodes + 2 * nk > GG_MAX_EXPR_NODES)
	{ gg_set_error("batched hash join: too many columns travel (%zu outer, %zu inner)", ov.size() + nk, iv.size() + nk); return GG_ERR_UNSUPPORTED; }
	j->notargets = j->nitargets = 0;
	for (int k = 0; k < nk; k++) { j->otargets[j->notargets++] = j->hj.outerkey[k]; j->itargets[j->nitargets++] = j->hj.innerkey[k]; }
	for (int32_t n : ov) j->otargets[j->notargets++] = n;
	for (int32_t n : iv) j->itargets[j->nitargets++] = n;
	/* the batch join's pool: Vars above the join -> their column of the partition rows; the join keys -> new Vars */
	std::vector<gg_exprpool> pb(1);
	gg_exprpool &bp = pb[0];
	bp = pool;
	for (int n = 0; n < bp.nnodes; n++)
	{
		gg_expr &x = bp.nodes[n];
		if (x.kind != GG_E_VAR) continue;
		const std::vector<int32_t> &side = x.varno == 0 ? ov : iv;
		for (size_t i = 0; i < side.size(); i++)
			if (pool.nodes[side[i]].varattno == x.varattno) { x.varattno = (int16_t) (nk + (int) i + 1); break; }
	}
	gg_hashjoin hj2 = j->hj;
	for (int k = 0; k < nk; k++)
		for (int sidei = 0; sidei < 2; sidei++)
		{
			gg_expr v;
			memset(&v, 0, sizeof v);
			v.kind = GG_E_VAR; v.varno = (int16_t) sidei; v.varattno = (int16_t) (k + 1);
			v.rettype = pool.nodes[sidei == 0 ? j->hj.outerkey[k] : j->hj.innerkey[k]].rettype;
			bp.nodes[bp.nnodes] = v;
			if (sidei == 0) hj2.outerkey[k] = bp.nnodes; else hj2.innerkey[k] = bp.nnodes;
			bp.nnodes++;
		}
	/* the partitions' descriptors: one 8-byte Datum per travelling expression; a plain Var of a NOT NULL column stays so */
	gg_scan os, is;
	memset(&os, 0, sizeof os); memset(&is, 0, sizeof is);
	os.qual = is.qual = -1;
	for (int sidei = 0; sidei < 2; sidei++)
	{
		gg_scan &sc = sidei == 0 ? os : is;
		const gg_scan &base = sidei == 0 ? j->outer_scan : j->inner_scan;
		const int nt = sidei == 0 ? j->notargets : j->nitargets;
		const int32_t *t = sidei == 0 ? j->otargets : j->itargets;
		sc.desc.natts = nt;
		sc.desc.format = GG_FMT_DATUMROWS;
		for (int i = 0; i < nt; i++)
		{
			const gg_expr &x = pool.nodes[t[i]];
			gg_attr &a = sc.desc.attrs[i];
			a.atttypid = x.rettype; a.atttypmod = -1; a.attlen = 8; a.attalign = 'd'; a.attbyval = 1;
			a.attnotnull = (x.kind == GG_E_VAR && x.varattno >= 1 && x.varattno <= base.desc.natts) ? base.desc.attrs[x.varattno - 1].attnotnull : 0;
		}
	}
	/* the targets keep their roots: the Vars under them were renumbered in place */
	int rc = joinagg_create(j->eng, &os, &is, &hj2, j->ntargets ? nullptr : &j->agg, j->targets, j->ntargets, &bp, &j->bj);
	if (rc) return rc;
	/* the inner relation is partitioned by a program that sees it as "the scan": its Vars as varno 0 */
	j->ipool = new gg_exprpool(pool);
	for (int n = 0; n < j->ipool->nnodes; n++)
		if (j->ipool->nodes[n].kind == GG_E_VAR) j->ipool->nodes[n].varno = j->ipool->nodes[n].varno == 1 ? 0 : 1;
	return GG_OK;
}

/* one pass over the batches: build batch b's table, probe with batch b, fill unmatched inner rows; everything accumulates
 * in the batch join's aggregate state */
static int joinagg_run_batches(gg_joinagg *j)
{
	gg_joinagg *b = j->bj;
	const int Wo = 1 + j->notargets, Wi = 1 + j->nitargets;
	j->build_ms = 0; j->rows_built = 0; j->null_keys = 0;
	uint32_t builderr = 0;          /* every batch's build counts, not only the last one's */
	for (int k = 0; k < j->nbatch; k++)
	{
		gg_relation *irel = nullptr, *orel = nullptr;
		int rc = gg_relation_attach_rows(j->eng, j->ibuf->pages + (uint64_t) k * j->icap * Wi * 8, j->icounts[(size_t) k], j->nitargets, &irel);
		if (rc == GG_OK) rc = gg_relation_attach_rows(j->eng, j->obuf->pages + (uint64_t) k * j->ocap * Wo * 8, j->ocounts[(size_t) k], j->notargets, &orel);
		if (rc == GG_OK) rc = gg_joinagg_build(b, irel, 0, irel->nblocks);
		if (rc == GG_OK) { j->build_ms += b->build_ms; j->rows_built += b->rows_built; j->null_keys += b->null_keys; builderr |= b->probe->build_err; b->probe->build_err = builderr; }
		if (rc == GG_OK && !b->lasj_empty) rc = gg_scanagg_run(b->probe, orel, 0, orel->nblocks);
		if (rc == GG_OK) rc = joinagg_fill_inner(b);
		gg_relation_free(irel);
		gg_relation_free(orel);
		if (rc) return rc;
	}
	return GG_OK;
}

int gg_joinagg_set_work_mem(gg_joinagg *j, uint64_t bytes)
{
	if (!j) return GG_ERR_ARG;
	j->work_mem = bytes;
	return GG_OK;
}

int gg_joinagg_nbatch(gg_joinagg *j) { return j ? j->nbatch : 0; }

int gg_joinagg_run(gg_joinagg *j, gg_relation *inner, gg_relation *outer)
{
	if (!j || !inner || !outer) return GG_ERR_ARG;
	/* the rows handed out live in the output buffer this run would rewrite (or reallocate) */
	if (j->rows_view) { gg_set_error("the joined rows were already handed out: reset before running again"); return GG_ERR_ARG; }
	gg_engine *e = j->eng;
	uint64_t nlp = 0;
	int rc = gg_relation_count_rows(inner, &nlp);
	if (rc) return rc;
	uint64_t slots = 1024;
	while (slots < 2 * nlp) slots <<= 1;
	uint32_t stride = (uint32_t) (1 + j->jp.nkeys + j->jp.npayload);
	if ((stride & 3) == 3) stride++;
	const uint64_t bytes = slots * stride * 8;
	j->nbatch = 1;
	/* NOT IN needs to know about a NULL inner key anywhere before any outer row is judged (nodeHashjoin.c:220-239): one batch */
	if (!j->work_mem || bytes <= j->work_mem || j->jp.jointype == GG_JOIN_LASJ_NOTIN)
	{
		rc = gg_joinagg_build(j, inner, 0, inner->nblocks);
		if (rc == GG_OK) rc = gg_joinagg_probe(j, outer, 0, outer->nblocks);
		return rc;
	}
	int nbatch = 2;
	while ((uint64_t) nbatch * j->work_mem < 2 * bytes && nbatch < 1024) nbatch <<= 1;     /* x2: tables are sized in powers of two */
	rc = joinagg_prepare_batches(j);
	if (rc) return rc;
	j->nbatch = nbatch;
	/* ExecChooseHashTableSize (nodeHash.c:450-659): nbuckets = a power of two near tuples per batch / gp_hashjoin_tuples_per_bucket */
	{
		uint64_t per = nlp / (uint64_t) nbatch / 5 + 1, nb = 1024;
		int l2 = 10;
		while (nb < per && l2 < 30) { nb <<= 1; l2++; }
		j->log2_nbuckets = l2;
	}
	uint64_t nouter = 0;
	rc = gg_relation_count_rows(outer, &nouter);
	if (rc) return rc;
	GG_CUDA(cudaEventRecord(j->ev0, e->stream));
	for (int side = 0; side < 2; side++)
	{
		gg_relation *rel = side == 0 ? outer : inner;
		gg_relation *&buf = side == 0 ? j->obuf : j->ibuf;
		uint64_t &cap = side == 0 ? j->ocap : j->icap;
		std::vector<uint64_t> &counts = side == 0 ? j->ocounts : j->icounts;
		const int nt = side == 0 ? j->notargets : j->nitargets;
		const uint64_t rows = side == 0 ? nouter : nlp;
		const int W = 1 + nt;
		uint64_t want = (rows / (uint64_t) nbatch + rows / (uint64_t) (4 * nbatch) + 8192) & ~1ull;
		for (int attempt = 0; ; attempt++)
		{
			if (buf && (cap < want || buf->nblocks * (uint64_t) GG_BLCKSZ < (want * nbatch * W + 8) * 8)) { gg_relation_free(buf); buf = nullptr; }
			if (!buf)
			{
				rc = gg_relation_create(e, ((want * nbatch * W + 8) * 8 + GG_BLCKSZ - 1) / GG_BLCKSZ, &buf);
				if (rc) return rc;
				cap = want;
			}
			counts.assign((size_t) nbatch, 0);
			std::vector<uint64_t> offs((size_t) nbatch);
			rc = gg_partition_rows(e, side == 0 ? &j->outer_scan : &j->inner_scan, side == 0 ? &j->pool : j->ipool,
			                       side == 0 ? j->hj.outerkey : j->hj.innerkey, j->hj.nkeys, side == 0 ? j->otargets : j->itargets, nt,
			                       nbatch, 1, j->log2_nbuckets, rel, 0, rel->nblocks, buf->pages, cap * (uint64_t) nbatch, counts.data(), offs.data());
			if (rc != GG_ERR_NOMEM || attempt >= 3) break;
			want *= 2;                      /* a skewed key: one batch got more than its share */
		}
		if (rc) return rc;
	}
	GG_CUDA(cudaEventRecord(j->ev1, e->stream));
	GG_CUDA(cudaEventSynchronize(j->ev1));
	GG_CUDA(cudaEventElapsedTime(&j->part_ms, j->ev0, j->ev1));
	rc = gg_scanagg_reset(j->bj->probe);
	if (rc) return rc;
	/* every batch appends its rows to the one output of the batch join */
	if (j->ntargets)
		rc = joinrows_fill_inner(j) ? joinrows_reserve(j->bj, nouter + nlp, 2 * (uint64_t) nbatch) : joinrows_reserve(j->bj, nouter, (uint64_t) nbatch);
	if (rc) return rc;
	j->bj->probe->replay_hook = [j]() { return joinagg_run_batches(j); };
	return joinagg_run_batches(j);
}

/* the joined-and-aggregated result as device-resident group records (after gg_joinagg_fetch ran the last pass) */
int gg_scanagg_groups(gg_scanagg *p, gg_groups **out);
int gg_joinagg_groups(gg_joinagg *j, gg_groups **out)
{
	if (!j) return GG_ERR_ARG;
	if (j->ntargets) { gg_set_error("a join with a target list returns rows (gg_joinagg_rows), not group records"); return GG_ERR_ARG; }
	if (!(j->bj && j->nbatch > 1))
	{
		int rc = joinagg_fill_inner(j);          /* right / full joins: the unmatched inner rows belong to the result */
		if (rc) return rc;
	}
	gg_scanagg *p = j->bj && j->nbatch > 1 ? j->bj->probe : j->probe;
	if (p->build_err)
	{
		const int rc = gg_errflags_to_code(p->build_err);         /* the hash table holds a value the device refused */
		if (rc) return rc;
	}
	return gg_scanagg_groups(p, out);
}

/* the probe's status words and row cursor */
static int joinrows_status(gg_scanagg *p, gg_scanagg::Status *st, unsigned long long *cursor)
{
	cudaStream_t s = p->eng->stream;
	GG_CUDA(cudaMemcpyAsync(st, p->d_status, sizeof *st, cudaMemcpyDeviceToHost, s));
	GG_CUDA(cudaMemcpyAsync(cursor, p->mo.cursor, sizeof *cursor, cudaMemcpyDeviceToHost, s));
	GG_CUDA(cudaStreamSynchronize(s));
	return GG_OK;
}

int gg_joinagg_rows(gg_joinagg *j, gg_relation **rows, uint64_t *nrows, uint64_t *nlive)
{
	if (!j || !rows || !nrows || !nlive) return GG_ERR_ARG;
	if (!j->ntargets) { gg_set_error("the join has no target list: its matches feed the aggregate above it"); return GG_ERR_ARG; }
	if (!j->rows_view)
	{
		const bool batched = j->bj && j->nbatch > 1;
		gg_joinagg *r = batched ? j->bj : j;            /* the join whose probe wrote the rows */
		gg_scanagg *p = r->probe;
		GG_CUDA(cudaSetDevice(j->eng->device));
		int rc = batched ? GG_OK : joinagg_fill_inner(j);         /* right / full joins: the unmatched inner rows belong to the result */
		if (rc) return rc;
		if (!r->rows_buf) { gg_set_error("no probe has run"); return GG_ERR_ARG; }
		if (p->build_err)
		{
			rc = gg_errflags_to_code(p->build_err);       /* the hash table holds a value the device refused */
			if (rc) return rc;
		}
		gg_scanagg::Status st;
		unsigned long long cur = 0;
		rc = joinrows_status(p, &st, &cur);
		if (rc) return rc;
		if ((st.err & GGP_EF_TABLE_FULL) && cur > p->mo.cap)
		{
			/* The join produced more rows than the output holds.  The cursor counted every row claimed, so one buffer of that
			 * size, plus the windows' slack of the launches the replay makes (those of the first pass, `fed`), holds them all:
			 * grow it and probe again against the kept table(s), exactly once. */
			rc = joinrows_reserve(r, cur, (uint64_t) p->fed.size());
			if (rc) return rc;
			if (!batched && p->jt.mark_matched)
			{
				/* the replayed fill-inner pass must see only what the replayed probe matches */
				gg_clear_matched_kernel<<<j->eng->sm_count * 4, 256, 0, j->eng->stream>>>(j->ent, j->slots, p->jt.stride);
				GG_CUDA(cudaGetLastError());
				j->eng->launches++;
			}
			rc = scanagg_replay(p, MODE_PART, 0);
			if (rc == GG_OK) rc = joinrows_status(p, &st, &cur);
			if (rc) return rc;
			if ((st.err & GGP_EF_TABLE_FULL) && cur > p->mo.cap)
			{ gg_set_error("join output: %llu rows claimed, capacity %llu after growing", cur, (unsigned long long) p->mo.cap); return GG_ERR_NOMEM; }
		}
		rc = gg_errflags_to_code(st.err);
		if (rc) return rc;
		j->rows_n = cur < p->mo.cap ? cur : p->mo.cap;
		j->rows_live = st.counters[1];
		rc = gg_relation_attach_rows(j->eng, r->rows_buf->pages, j->rows_n, j->ntargets, &j->rows_view);
		if (rc) { j->rows_view = nullptr; return rc; }
	}
	*rows = j->rows_view;
	*nrows = j->rows_n;
	*nlive = j->rows_live;
	return GG_OK;
}

int gg_joinagg_reset(gg_joinagg *j)
{
	if (!j) return GG_ERR_ARG;
	if (j->probe->jt.mark_matched && j->ent)
	{
		GG_CUDA(cudaSetDevice(j->eng->device));
		gg_clear_matched_kernel<<<j->eng->sm_count * 4, 256, 0, j->eng->stream>>>(j->ent, j->slots, j->probe->jt.stride);
		GG_CUDA(cudaGetLastError());
		j->eng->launches++;
	}
	j->filled = false;
	if (j->rows_view) { gg_relation_free(j->rows_view); j->rows_view = nullptr; }
	if (j->bj) { int rc = gg_joinagg_reset(j->bj); if (rc) return rc; }
	return gg_scanagg_reset(j->probe);
}

int gg_joinagg_stats(gg_joinagg *j, uint64_t *rows_built, uint64_t *table_bytes, float *build_ms, float *probe_ms)
{
	if (!j) return GG_ERR_ARG;
	if (rows_built) *rows_built = j->rows_built;
	if (table_bytes) *table_bytes = j->slots * (uint64_t) j->stride * 8;
	if (build_ms) *build_ms = j->build_ms;
	if (probe_ms) return gg_scanagg_scan_kernel_ms(j->bj && j->nbatch > 1 ? j->bj->probe : j->probe, probe_ms, nullptr);
	return GG_OK;
}

int gg_joinagg_variant(gg_joinagg *j) { return j ? gg_scanagg_variant(j->bj && j->nbatch > 1 ? j->bj->probe : j->probe) : -1; }

void gg_joinagg_free(gg_joinagg *j)
{
	if (!j) return;
	cudaSetDevice(j->eng->device);
	cudaStreamSynchronize(j->eng->stream);
	if (j->bj) gg_joinagg_free(j->bj);
	delete j->ipool;
	if (j->obuf) gg_relation_free(j->obuf);
	if (j->ibuf) gg_relation_free(j->ibuf);
	if (j->probe) gg_scanagg_free(j->probe);
	if (j->rows_view) gg_relation_free(j->rows_view);
	if (j->rows_buf) gg_relation_free(j->rows_buf);
	cudaFree(j->ent); cudaFree(j->d_cnt); cudaFree(j->d_buildcnt); cudaFree(j->d_rowcur);
	if (j->ev0) cudaEventDestroy(j->ev0);
	if (j->ev1) cudaEventDestroy(j->ev1);
	delete j;
}

}  /* extern "C" */
