/*
 * gg_scanagg.cu — SeqScan -> qual -> Agg: the ahead-of-time kernels (interpreter path), the merge
 * kernel, and the host pipeline behind gg_scanagg_* / gg_agg_final (include/ggb200.h).  The same pipeline
 * object is the probe side of a join (gg_join.cu).
 * The kernel body lives in gg_scanagg_kernel.cuh so that gg_jit.cpp can instantiate it again,
 * specialised for one plan.
 */
#include <cuda_runtime.h>
#include <stdint.h>
#include "gg_scanagg_kernel.cuh"
#include "gg_engine.h"
#include "gg_jit.h"

using namespace ggd;

template <int MODE>
__global__ void __launch_bounds__(MODE == MODE_PRIV ? 704 : 256, MODE == MODE_PRIV ? 1 : 2)
gg_scanagg_kernel(const __grid_constant__ ggp_program P, const ScanAggParams prm)
{
	scanagg_body<MODE, DynPlan>(P, prm);
}

/* HashJoin probe side: the same scan front end; every outer row probes the join hash table and each
 * match runs the per-match piece of the program (join qual, grouping keys, aggregate arguments) */
template <int MODE>
__global__ void __launch_bounds__(MODE == MODE_PRIV ? 704 : 256, MODE == MODE_PRIV ? 1 : 2)
gg_joinprobe_kernel(const __grid_constant__ ggp_program P, const ScanAggParams prm)
{
	scanagg_body<MODE, DynPlan, true>(P, prm);
}

/* general HashAggregate (any number of groups): scan + probe side variants */
__global__ void __launch_bounds__(256, 2)
gg_hashagg_kernel(const __grid_constant__ ggp_program P, const ScanAggParams prm)
{
	scanagg_body<MODE_HASH, DynPlan>(P, prm);
}

/* MIN/MAX start from the identity of their comparison, float8 sums from -0 (RegAcc::zero); everything else from zero (the
 * table is memset first) */
__global__ void gg_hashagg_init_kernel(HashAggTable ha)
{
	for (int j = 0; j < ha.nacc; j++)
	{
		const int kind = ha.acckind[j];
		unsigned long long init;
		if (kind == GGP_ACC_F8MIN) init = 0x7ff8000000000000ull;              /* NaN sorts above everything */
		else if (kind == GGP_ACC_F8MAX) init = 0xfff0000000000000ull;         /* -Infinity */
		else if (kind == GGP_ACC_I8MIN) init = 0x7fffffffffffffffull;
		else if (kind == GGP_ACC_I8MAX) init = 0x8000000000000000ull;
		else if (kind == GGP_ACC_F8SUM) init = GG_F8_NEGZERO_BITS;
		else continue;
		for (uint64_t i = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; i < ha.cap; i += (uint64_t) gridDim.x * blockDim.x)
			ha.ent[i * ha.stride + ha.off_acc + j] = init;
	}
}

/* table -> group records (order unspecified, like a hash aggregate's output) */
__global__ void gg_hashagg_emit_kernel(HashAggTable ha, ggp_grec *out, unsigned long long outcap, unsigned long long *nout,
                                       uint32_t *errflags)
{
	const bool saw_inf = (*errflags & GGP_EF_SAW_INF) != 0;
	for (uint64_t i = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; i < ha.cap; i += (uint64_t) gridDim.x * blockDim.x)
	{
		const unsigned long long *ep = ha.ent + i * ha.stride;
		const unsigned long long h = ep[0];
		if (!(h >> 63)) continue;
		const unsigned long long at = atomicAdd(nout, 1ull);
		if (at >= outcap) continue;
		ggp_grec r;
		memset(&r, 0, sizeof r);
		for (int c = 0; c < ha.nkeys; c++) r.key[c] = ep[1 + c];
		r.keynull = (uint32_t) (h >> 32) & 0xF;
		r.valid = 1;
		r.count = ep[ha.off_cnt];
		for (int j = 0; j < ha.nacc; j++)
		{
			r.sum[j] = __longlong_as_double((long long) ep[ha.off_acc + j]);
			r.sumsq[j] = ha.off_sq ? __longlong_as_double((long long) ep[ha.off_sq + j]) : 0.0;
			r.n[j] = ha.off_accn ? ep[ha.off_accn + j] : r.count;          /* no NULLs anywhere: every row counted */
			/* float8pl's CHECKFLOATVAL (float.c:782): an infinite sum of finite inputs is an overflow */
			if (ha.acckind[j] == GGP_ACC_F8SUM && !saw_inf && r.n[j] && !f8_finite(r.sum[j])) atomicOr(errflags, GGP_EF_FLOAT_OVERFLOW);
		}
		out[at] = r;
	}
}

/* the key types of a program or group set, 2 bits per key as the kernels take them */
static inline uint32_t keytypes_of(const uint8_t *kt)
{
	return (uint32_t) kt[0] | ((uint32_t) kt[1] << 2) | ((uint32_t) kt[2] << 4) | ((uint32_t) kt[3] << 6);
}

/* ---- merge kernel: fold group records with equal keys (key_same), in record order (deterministic) ----
 * One block.  A: ordered compaction of the valid records.  B: every valid record finds (or, under a
 * lock, creates) its merged group.  C: thread (group, column) folds that group's records in record
 * order.  This is also the combine step of a FINAL-stage Agg (float8pl / float8_combine / int8pl,
 * nodeAgg.c:2123-2148) when the records come from other segments. */
__global__ void __launch_bounds__(1024, 1)
gg_merge_recs_kernel(const ggp_grec *recs, int nrecs, int nkeys, uint32_t keytypes, int nacc, ggp_acckinds kinds,
                     ggp_grec *out, int outcap, int *nout, int *vidx /* [nrecs] */, int *vmap /* [nrecs] */,
                     uint32_t *errflags, int prefix_sets /* 1: the valid records of a set are a prefix of it */)
{
	__shared__ int s_nvalid, s_nout, s_lock;
	__shared__ int s_warpsum[32];
	const int nthreads = (int) blockDim.x, nwarps = nthreads >> 5;
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	if (tid == 0) { s_nvalid = 0; s_nout = 0; s_lock = 0; }
	__syncthreads();

	/* A: ordered compaction (chunks of blockDim.x records, in order) */
	for (int base = 0; base < nrecs; base += nthreads)
	{
		int i = base + tid;
		bool v = i < nrecs && recs[i].valid != 0;
		unsigned b = __ballot_sync(GG_FULL_MASK, v);
		if (lane == 0) s_warpsum[warp] = __popc(b);
		__syncthreads();
		int pre = 0;
		for (int w = 0; w < warp; w++) pre += s_warpsum[w];
		int tot = 0;
		for (int w = 0; w < nwarps; w++) tot += s_warpsum[w];
		int pos = s_nvalid + pre + __popc(b & ((1u << lane) - 1));
		if (v) vidx[pos] = i;
		__syncthreads();
		if (tid == 0) s_nvalid += tot;
		__syncthreads();
	}
	const int nvalid = s_nvalid;

	/* B: group assignment */
	for (int base = 0; base < nvalid; base += nthreads)
	{
		int k = base + tid;
		bool need = k < nvalid;
		const ggp_grec *x = need ? &recs[vidx[k]] : nullptr;
		int f = -1;
		if (need)
		{
			int n = *(volatile int *) &s_nout;
			for (int m = 0; m < n && f < 0; m++)
			{
				bool eq = out[m].keynull == x->keynull;
				for (int c = 0; eq && c < nkeys; c++) eq = key_same(out[m].key[c], x->key[c], (f8_keys(keytypes) >> (2 * c)) & 1);
				if (eq) f = m;
			}
			need = f < 0;
		}
		unsigned mm = __ballot_sync(GG_FULL_MASK, need);
		while (mm)
		{
			int leader = __ffs(mm) - 1;
			if (lane == leader)
			{
				while (atomicCAS(&s_lock, 0, 1) != 0) { }
				__threadfence();
				int n = *(volatile int *) &s_nout;
				for (int m = 0; m < n && f < 0; m++)
				{
					bool eq = ((volatile ggp_grec *) out)[m].keynull == x->keynull;
					for (int c = 0; eq && c < nkeys; c++) eq = key_same(((volatile ggp_grec *) out)[m].key[c], x->key[c], (f8_keys(keytypes) >> (2 * c)) & 1);
					if (eq) f = m;
				}
				if (f < 0)
				{
					if (n < outcap)
					{
						for (int c = 0; c < GG_MAX_KEYS; c++) out[n].key[c] = x->key[c];
						out[n].keynull = x->keynull;
						out[n].valid = 1;
						__threadfence();
						*(volatile int *) &s_nout = n + 1;
						f = n;
					}
					else
						atomicOr(errflags, GGP_EF_GROUP_OVERFLOW);
				}
				__threadfence();
				atomicExch(&s_lock, 0);
				need = false;
			}
			__syncwarp();
			if (need)
			{
				int n = *(volatile int *) &s_nout;
				for (int m = 0; m < n && f < 0; m++)
				{
					bool eq = ((volatile ggp_grec *) out)[m].keynull == x->keynull;
					for (int c = 0; eq && c < nkeys; c++) eq = key_same(((volatile ggp_grec *) out)[m].key[c], x->key[c], (f8_keys(keytypes) >> (2 * c)) & 1);
					if (eq) f = m;
				}
				need = f < 0;
			}
			mm = __ballot_sync(GG_FULL_MASK, need);
		}
		if (k < nvalid) vmap[vidx[k]] = f;          /* merged group of record vidx[k], indexed by RECORD */
	}
	__threadfence();
	__syncthreads();

	/* C: fold.  One warp per (merged group, column).  Records come in sets of GGP_FAST_GROUPS (one set per
	 * producing block; a set holds a group at most once).  Lane l folds sets l, l+32, ... in order and the 32
	 * partials are combined by a fixed butterfly, so the summation tree depends only on WHICH block produced a
	 * record, never on the order in which groups were discovered => bit-identical results run to run. */
	const int n = s_nout;
	if (tid == 0) *nout = n;
	const int V = nacc > 0 ? nacc : 1;
	const bool saw_inf = (*errflags & GGP_EF_SAW_INF) != 0;
	const int nsets = (nrecs + GGP_FAST_GROUPS - 1) / GGP_FAST_GROUPS;
	for (int t = warp; t < n * V; t += (int) (blockDim.x >> 5))
	{
		int mg = t / V, j = t % V;
		int kind = nacc > 0 ? kinds.k[j] : GGP_ACC_COUNT;
		double s0 = kind == GGP_ACC_F8SUM ? -0.0 : 0.0, s1 = 0.0;
		unsigned long long cnt = 0, nn = 0;
		for (int set = lane; set < nsets; set += 32)
		for (int slot = 0; slot < GGP_FAST_GROUPS; slot++)
		{
			const int i = set * GGP_FAST_GROUPS + slot;
			/* within a set the valid records are a prefix (a block fills slots 0..G-1; merged / FINAL-stage input is
			 * dense), so the first invalid slot ends the set */
			if (i >= nrecs) break;
			if (!recs[i].valid) { if (prefix_sets) break; else continue; }
			if (vmap[i] != mg) continue;
			const ggp_grec &x = recs[i];
			cnt += x.count;
			if (nacc > 0 && x.n[j])
			{
				if (kind == GGP_ACC_F8SUM) { s0 = __dadd_rn(s0, x.sum[j]); s1 = __dadd_rn(s1, x.sumsq[j]); }
				else if (kind == GGP_ACC_I8SUM)
				{
					long long a = __double_as_longlong(s0), b = __double_as_longlong(x.sum[j]), r = (long long) ((unsigned long long) a + (unsigned long long) b);
					if (((a ^ r) & (b ^ r)) < 0) atomicOr(errflags, GGP_EF_INT_OVERFLOW);   /* int8pl, int8.c:526 */
					s0 = __longlong_as_double(r);
				}
				else if (kind == GGP_ACC_F8MIN) { if (nn == 0 || f8_cmp(x.sum[j], s0) < 0) s0 = x.sum[j]; }
				else if (kind == GGP_ACC_F8MAX) { if (nn == 0 || f8_cmp(x.sum[j], s0) > 0) s0 = x.sum[j]; }
				else if (kind == GGP_ACC_I8MIN) { if (nn == 0 || __double_as_longlong(x.sum[j]) < __double_as_longlong(s0)) s0 = x.sum[j]; }
				else if (kind == GGP_ACC_I8MAX) { if (nn == 0 || __double_as_longlong(x.sum[j]) > __double_as_longlong(s0)) s0 = x.sum[j]; }
				nn += x.n[j];
			}
		}
		for (int o = 16; o > 0; o >>= 1)
		{
			double os0 = __shfl_xor_sync(GG_FULL_MASK, s0, o), os1 = __shfl_xor_sync(GG_FULL_MASK, s1, o);
			unsigned long long ocnt = __shfl_xor_sync(GG_FULL_MASK, cnt, o), onn = __shfl_xor_sync(GG_FULL_MASK, nn, o);
			/* both partners must compute the identical combined value: order operands by lane */
			bool lo = (lane & o) == 0;
			double a0 = lo ? s0 : os0, b0 = lo ? os0 : s0;
			unsigned long long an = lo ? nn : onn, bn = lo ? onn : nn;
			if (kind == GGP_ACC_F8SUM) { s0 = __dadd_rn(a0, b0); s1 = __dadd_rn(lo ? s1 : os1, lo ? os1 : s1); }
			else if (kind == GGP_ACC_I8SUM)
			{
				long long a = __double_as_longlong(a0), b = __double_as_longlong(b0), r = (long long) ((unsigned long long) a + (unsigned long long) b);
				if (((a ^ r) & (b ^ r)) < 0) atomicOr(errflags, GGP_EF_INT_OVERFLOW);
				s0 = __longlong_as_double(r);
			}
			else if (kind == GGP_ACC_F8MIN) s0 = an == 0 ? b0 : bn == 0 ? a0 : (f8_cmp(b0, a0) < 0 ? b0 : a0);
			else if (kind == GGP_ACC_F8MAX) s0 = an == 0 ? b0 : bn == 0 ? a0 : (f8_cmp(b0, a0) > 0 ? b0 : a0);
			else if (kind == GGP_ACC_I8MIN) s0 = an == 0 ? b0 : bn == 0 ? a0 : (__double_as_longlong(b0) < __double_as_longlong(a0) ? b0 : a0);
			else if (kind == GGP_ACC_I8MAX) s0 = an == 0 ? b0 : bn == 0 ? a0 : (__double_as_longlong(b0) > __double_as_longlong(a0) ? b0 : a0);
			cnt += ocnt;
			nn += onn;
		}
		if (lane == 0)
		{
			if (nacc > 0)
			{
				/* CHECKFLOATVAL of float8pl / float8_accum / float8_combine (float.c:782,1842,1878): a sum that
				 * became infinite although no input was infinite is an overflow ERROR */
				if (kind == GGP_ACC_F8SUM && !saw_inf && (!f8_finite(s0) || !f8_finite(s1)))
					atomicOr(errflags, GGP_EF_FLOAT_OVERFLOW);
				out[mg].sum[j] = s0; out[mg].sumsq[j] = s1; out[mg].n[j] = nn;
			}
			if (j == 0) out[mg].count = cnt;
		}
	}
}

/* =====================================================================================
 * host side: the pipeline object behind gg_scanagg_* (include/ggb200.h)
 * ===================================================================================== */
#include <cstdio>
#include <cstring>
#include <vector>

#include "gg_pipeline.h"
#include "gg_groups.h"

static_assert(sizeof(BlockTable) == GG_BLOCKTABLE_BYTES && GG_REG_GROUPS == 4, "gg_launch.h sizes the shared memory with these");
static_assert((int) GGL_PRIV == MODE_PRIV && (int) GGL_TR == MODE_TR && (int) GGL_TRN == MODE_TRN && (int) GGL_BUILD == MODE_BUILD &&
              (int) GGL_PART == MODE_PART && (int) GGL_HASH == MODE_HASH, "gg_launch.h names the kernel roles");

/* the interpreter instance of every role: [join][mode] */
static const void *const interp_kernels[2][6] = {
	{ (const void *) gg_scanagg_kernel<MODE_PRIV>, (const void *) gg_scanagg_kernel<MODE_TR>, (const void *) gg_scanagg_kernel<MODE_TRN>,
	  (const void *) gg_joinbuild_kernel, (const void *) gg_motion_part_kernel, (const void *) gg_hashagg_kernel },
	{ (const void *) gg_joinprobe_kernel<MODE_PRIV>, (const void *) gg_joinprobe_kernel<MODE_TR>, (const void *) gg_joinprobe_kernel<MODE_TRN>,
	  nullptr, (const void *) gg_joinrows_kernel, (const void *) gg_joinhash_kernel },
};

/* the plan-specialised kernel for a launch shape, or nullptr (why: jmsg) */
static gg_jit_kernel *scan_jit(const ggp_program *prog, int mode, int probe_pc, const gg_launch &c, int device, bool mvcc, char *jmsg, int jlen)
{
	return gg_jit_scanagg(prog, mode, c.threads, device, jmsg, jlen, probe_pc, c.regslots,
	                      c.forced || (mode == MODE_PRIV && c.ctas > 1) ? c.ctas : 0, mvcc);
}

int gg_scan_kernel(const ggp_program *prog, int mode, int probe_pc, const gg_launch &c, int device, bool mvcc, const void **fn, gg_jit_kernel **jit)
{
	char jmsg[512];
	gg_jit_kernel *jk = nullptr;
	if (probe_pc >= 0 && mode == MODE_PART) snprintf(jmsg, sizeof jmsg, "the probe that writes join rows has no specialised kernel");
	else jk = scan_jit(prog, mode, probe_pc, c, device, mvcc, jmsg, sizeof jmsg);
	if (jit) *jit = jk;
	if (!jk && getenv("GGB200_JIT_VERBOSE")) fprintf(stderr, "ggb200: interpreter kernel in use (%s)\n", jmsg);
	if (!jk && mode != MODE_PRIV && c.threads != 256) { gg_set_error("GGB200_NP_CONFIG needs the run-time specialised kernel: %s", jmsg); return GG_ERR_UNSUPPORTED; }
	*fn = jk ? (const void *) jk->kernel : interp_kernels[probe_pc >= 0][mode];
	GG_CUDA(cudaFuncSetAttribute(*fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) c.smem));
	return GG_OK;
}

/* launch configuration (gg_launch.h gg_scan_config) and kernel for the current variant */
static int scanagg_configure(gg_scanagg *p)
{
	gg_engine *e = p->eng;
	const int probe_pc = p->is_join ? p->join_probe_pc : -1;
	if (!gg_scan_config(p->cfg, p->mode, p->is_join, p->prog, p->chunks_per_page, p->items_per_page,
	                    gg_priv_regslots(&p->prog, p->mode, p->agg.numGroups, probe_pc), e->smem_optin))
	{ gg_set_error("plan needs too much shared memory"); return GG_ERR_UNSUPPORTED; }
	p->grid = e->sm_count * p->cfg.ctas;
	p->jit_snap = nullptr;
	int rc = gg_scan_kernel(&p->prog, p->mode, probe_pc, p->cfg, e->device, false, &p->kernel, &p->jit);
	if (rc) return rc;
	if (!p->jit && p->cfg.regslots > 0)
	{
		/* the interpreter kernel addresses value slots dynamically: everything in shared memory */
		p->cfg.regslots = 0;
		return scanagg_configure(p);
	}
	return GG_OK;
}

/* (re)allocate and initialise the HBM group table of the general HashAggregate */
static int hashagg_alloc(gg_scanagg *p, uint64_t cap)
{
	cudaStream_t st = p->eng->stream;
	const ggp_program &P = p->prog;
	bool anysq = false;
	for (int j = 0; j < P.nacc; j++) anysq = anysq || P.accsq[j] >= 0;
	HashAggTable ha;
	memset(&ha, 0, sizeof ha);
	ha.cap = cap;
	ha.nacc = P.nacc; ha.nkeys = P.nkeys;
	uint32_t w = 1 + (uint32_t) P.nkeys;
	ha.off_cnt = w++;
	ha.off_acc = w; w += (uint32_t) P.nacc;
	if (P.nullable && P.nacc) { ha.off_accn = w; w += (uint32_t) P.nacc; }      /* NOT NULL inputs: n == row count */
	if (anysq) { ha.off_sq = w; w += (uint32_t) P.nacc; }
	ha.stride = (w + 3) & ~3u;                                                    /* entries start on 32-byte sectors */
	memcpy(ha.acckind, P.acckind, sizeof ha.acckind);
	for (int j = 0; j < P.nacc; j++) if (P.accsq[j] >= 0 && P.accsq[j] < GGP_MAX_SLOTS) ha.sqcol[P.accsq[j]] = (uint8_t) j;
	const size_t bytes = (size_t) cap * ha.stride * 8;
	if (p->ha_mem && p->ha_cap != cap) { GG_CUDA(cudaStreamSynchronize(st)); cudaFree(p->ha_mem); p->ha_mem = nullptr; }
	if (!p->ha_mem)
	{
		cudaError_t ce = cudaMalloc(&p->ha_mem, bytes);
		if (ce != cudaSuccess) { cudaGetLastError(); gg_set_error("group table of %zu bytes does not fit in device memory", bytes); return GG_ERR_NOMEM; }
	}
	p->ha_cap = cap;
	ha.ent = (unsigned long long *) p->ha_mem;
	p->ha = ha;
	GG_CUDA(cudaMemsetAsync(p->ha_mem, 0, bytes, st));
	gg_hashagg_init_kernel<<<p->eng->sm_count * 4, 256, 0, st>>>(ha);
	GG_CUDA(cudaGetLastError());
	p->eng->launches++;
	return GG_OK;
}

int scanagg_launch(gg_scanagg *p, const uint8_t *dev_pages, uint64_t nblocks, cudaStream_t st, uint64_t nrows, bool fill_inner, int32_t aocs_tile_rows)
{
	gg_engine *e = p->eng;
	ScanAggParams prm;
	prm.pages = dev_pages;
	prm.nblocks = nblocks;
	prm.block_recs = p->recs + GG_MERGE_CAP;
	prm.errflags = p->d_err;
	prm.counters = p->d_counters;
	prm.nstage = p->cfg.nstage;
	prm.gcap = p->cfg.gcap;
	prm.scratch_per_warp = p->cfg.scratch_per_warp;
	prm.scratch_off = p->cfg.scratch_off;
	prm.cnt_off = p->cfg.cnt_off;
	prm.acc_off = p->cfg.acc_off;
	prm.jt = p->jt;
	prm.mo = p->mo;
	prm.nrows = nrows;
	prm.fill_inner = fill_inner ? 1 : 0;
	prm.team = p->cfg.team;
	prm.snap = e->d_snapshot;
	{
		const char *kc = getenv("GGB200_KEYCACHE");
		prm.nokeycache = kc && atoi(kc) == 0;
	}
	prm.aocs = aocs_tile_rows > 0 ? (const gg_aocs_devcol *) dev_pages : nullptr;
	prm.aocs_tile_rows = aocs_tile_rows;
	prm.aocs_unit_rows = 0;
	if (aocs_tile_rows > 0)
	{
		/* the kernel's unit of work is a staging unit, not a tile of the plan (the caller counts tiles) */
		prm.aocs_unit_rows = p->aocs_unit_rows;
		prm.nblocks = (nrows + (uint64_t) p->aocs_unit_rows - 1) / (uint64_t) p->aocs_unit_rows;
	}
	prm.ha = p->ha;
	if (p->kev_used == p->kev.size())
	{
		cudaEvent_t a, b;
		GG_CUDA(cudaEventCreate(&a));
		GG_CUDA(cudaEventCreate(&b));
		p->kev.push_back({ a, b });
	}
	GG_CUDA(cudaEventRecord(p->kev[p->kev_used].first, st));
	if (p->is_join && !p->jt.ent) { gg_set_error("probe before build"); return GG_ERR_ARG; }
	const void *fn = p->kernel;
	if (p->jit && e->d_snapshot)
	{
		/* With a snapshot on the engine the scan needs the specialised kernel that carries the snapshot rule; the plain one raises
		 * GGP_EF_VISIBILITY for every tuple whose hint bits do not decide (the interpreter kernels carry the rule) */
		if (!p->jit_snap)
		{
			char jmsg[512];
			p->jit_snap = scan_jit(&p->prog, p->mode, p->is_join ? p->join_probe_pc : -1, p->cfg, e->device, true, jmsg, sizeof jmsg);
			if (p->jit_snap) GG_CUDA(cudaFuncSetAttribute((const void *) p->jit_snap->kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) p->cfg.smem));
			else
			{
				if (getenv("GGB200_JIT_VERBOSE")) fprintf(stderr, "ggb200: no specialised kernel with the snapshot rule (%s)\n", jmsg);
				p->jit_snap = p->jit;        /* undecided tuples make the scan fail, never pass */
			}
		}
		fn = (const void *) p->jit_snap->kernel;
	}
	void *args[] = { (void *) &p->prog, (void *) &prm };
	GG_CUDA(cudaLaunchKernel(fn, dim3(p->grid), dim3(p->cfg.threads), args, p->cfg.smem, st));
	GG_CUDA(cudaGetLastError());
	GG_CUDA(cudaEventRecord(p->kev[p->kev_used].second, st));
	p->kev_used++;
	e->launches++;
	p->has_state = true;
	if (p->mode == MODE_HASH || p->mode == MODE_PART) return GG_OK;     /* group table in HBM / rows written: nothing to fold */
	/* fold the block records (and the previously merged groups) */
	ggp_acckinds kinds;
	memcpy(kinds.k, p->prog.acckind, sizeof kinds.k);
	gg_merge_recs_kernel<<<1, 1024, 0, st>>>(p->recs, p->nrecs_total, p->prog.nkeys, keytypes_of(p->prog.keytype), p->prog.nacc, kinds,
	                                        p->merged, GG_MERGE_CAP, p->d_nout, p->vidx, p->vmap, p->d_err, 1);
	GG_CUDA(cudaGetLastError());
	e->launches++;
	/* merged -> first GG_MERGE_CAP slots of recs (input of the next fold); slots beyond nout are invalidated
	 * by copying the whole (zero-initialised) merged array */
	GG_CUDA(cudaMemcpyAsync(p->recs, p->merged, sizeof(ggp_grec) * GG_MERGE_CAP, cudaMemcpyDeviceToDevice, st));
	GG_CUDA(cudaMemsetAsync(p->merged, 0, sizeof(ggp_grec) * GG_MERGE_CAP, st));
	return GG_OK;
}

extern "C" int gg_scanagg_reset(gg_scanagg *p);

/* First feed of a private-accumulator pipeline: look at one page header to see how densely the relation's pages
 * are populated and pick the launch configuration for it (see scanagg_configure). */
static int scanagg_adapt_to_pages(gg_scanagg *p, const uint8_t *dev_page, const void *host_page)
{
	if (p->mode != MODE_PRIV || p->has_state || p->chunks_per_page || p->prog.outer.rowwords || getenv("GGB200_PRIV_CONFIG")) return GG_OK;
	uint32_t hdr[6] = { 0 };
	if (host_page) memcpy(hdr, host_page, sizeof hdr);
	else GG_CUDA(cudaMemcpy(hdr, dev_page, sizeof hdr, cudaMemcpyDeviceToHost));
	const uint32_t pd_lower = hdr[3] & 0xFFFF;
	int items = pd_lower >= GG_PAGE_HEADER_SIZE && pd_lower <= GG_BLCKSZ ? (int) ((pd_lower - GG_PAGE_HEADER_SIZE) >> 2) : 0;
	p->chunks_per_page = items > 0 ? (items + 31) / 32 : 1;
	p->items_per_page = items;
	p->cfg.regslots = -1;                      /* decided again for this page density */
	int rc = scanagg_configure(p);
	if (rc) return rc;
	if (p->mode == MODE_PRIV && p->agg.numGroups > p->cfg.gcap)
	{
		/* the denser configuration leaves room for fewer groups than the planner expects: keep the default one */
		p->chunks_per_page = 1;
		rc = scanagg_configure(p);
	}
	return rc;
}

/* the part of pipeline creation that follows plan compilation (p->prog / p->aggmap are set) */
int scanagg_finish_create(gg_scanagg *p, gg_scanagg **out)
{
	gg_engine *e = p->eng;
	const gg_agg *agg = &p->agg;
	int rc;
	/* kernel variant: private accumulators when the plan allows it (NOT NULL float8 sums); the planner's
	 * group estimate decides whether they can hold the groups */
	p->mode = p->prog.nullable ? MODE_TRN : MODE_TR;
	if (p->prog.priv_ok) p->mode = MODE_PRIV;
	const char *force = getenv("GGB200_SCAN_MODE");           /* experiments: 0 PRIV, 1 TR, 2 TRN, 5 HASH */
	if (p->join_rows) p->mode = MODE_PART;
	else if (force && atoi(force) == MODE_HASH) p->mode = MODE_HASH;
	else if (force && !p->is_join)
	{ int m = atoi(force); if (m == MODE_PRIV && !p->prog.priv_ok) m = MODE_TR; if (p->prog.nullable) m = MODE_TRN; p->mode = m; }
	rc = scanagg_configure(p);
	if (rc == GG_OK && p->mode == MODE_PRIV && agg->numGroups > p->cfg.gcap)
	{
		p->mode = p->prog.nullable ? MODE_TRN : MODE_TR;
		rc = scanagg_configure(p);
	}
	if (rc == GG_OK && p->mode != MODE_HASH && agg->numGroups > p->cfg.gcap)
	{
		/* the planner expects more groups than a block holds on chip: the HBM hash table from the start */
		p->mode = MODE_HASH;
		rc = scanagg_configure(p);
	}
	if (rc) { delete p; return rc; }
	/* block records are sized for the largest grid either configuration uses */
	p->nrecs_cap = GG_MERGE_CAP + e->sm_count * 4 * GGP_FAST_GROUPS;
	p->nrecs_total = GG_MERGE_CAP + p->grid * GGP_FAST_GROUPS;
	GG_CUDA(cudaMalloc((void **) &p->recs, sizeof(ggp_grec) * p->nrecs_cap));
	GG_CUDA(cudaMalloc((void **) &p->merged, sizeof(ggp_grec) * GG_MERGE_CAP));
	GG_CUDA(cudaMalloc((void **) &p->vidx, sizeof(int) * p->nrecs_cap));
	GG_CUDA(cudaMalloc((void **) &p->vmap, sizeof(int) * p->nrecs_cap));
	GG_CUDA(cudaMalloc((void **) &p->d_status, sizeof(gg_scanagg::Status)));
	p->d_nout = &p->d_status->nout;
	p->d_err = &p->d_status->err;
	p->d_counters = p->d_status->counters;
	GG_CUDA(cudaHostAlloc((void **) &p->h_mirror, sizeof(gg_scanagg::HostMirror), cudaHostAllocDefault));
	GG_CUDA(cudaMalloc((void **) &p->d_nout64, sizeof(unsigned long long)));
	*out = p;
	return gg_scanagg_reset(p);
}

extern "C" {

int gg_scanagg_create(gg_engine *e, const gg_scan *scan, const gg_agg *agg, const gg_exprpool *pool,
                      gg_scanagg **out)
{
	if (!e || !scan || !agg || !pool || !out) return GG_ERR_ARG;
	*out = nullptr;
	GG_CUDA(cudaSetDevice(e->device));
	gg_scanagg *p = new gg_scanagg();
	p->eng = e;
	p->scan = *scan;
	p->agg = *agg;
	p->pool = *pool;
	char msg[256];
	int rc = ggp_compile_scanagg(scan, agg, pool, &p->prog, p->aggmap, msg, sizeof msg);
	if (rc != GG_OK) { gg_set_error("%s", msg); delete p; return rc; }
	return scanagg_finish_create(p, out);
}

int gg_scanagg_reset(gg_scanagg *p)
{
	if (!p) return GG_ERR_ARG;
	cudaStream_t st = p->eng->stream;
	GG_CUDA(cudaSetDevice(p->eng->device));
	GG_CUDA(cudaMemsetAsync(p->recs, 0, sizeof(ggp_grec) * p->nrecs_cap, st));
	p->fed.clear();
	GG_CUDA(cudaMemsetAsync(p->merged, 0, sizeof(ggp_grec) * GG_MERGE_CAP, st));
	GG_CUDA(cudaMemsetAsync(p->d_status, 0, sizeof(gg_scanagg::Status), st));
	if (p->mo.cursor) GG_CUDA(cudaMemsetAsync(p->mo.cursor, 0, sizeof(unsigned long long), st));
	p->has_state = false;
	p->kev_used = 0;
	if (p->mode == MODE_HASH)
	{
		/* planner's estimate (Agg.numGroups) x 2, at least 64 K slots; a full table is rebuilt larger by fetch */
		uint64_t cap = p->ha_cap ? p->ha_cap : 65536;
		while (cap < 2 * (uint64_t) (p->agg.numGroups > 0 ? p->agg.numGroups : 0)) cap <<= 1;
		return hashagg_alloc(p, cap);
	}
	return GG_OK;
}

int gg_scanagg_run(gg_scanagg *p, gg_relation *r, uint64_t first_block, uint64_t nblocks)
{
	if (!p || !r || nblocks > r->nblocks || first_block > r->nblocks - nblocks) return GG_ERR_ARG;
	if (r->rowwords != p->prog.outer.rowwords) { gg_set_error("relation format does not match the plan's tuple descriptor"); return GG_ERR_ARG; }
	if (r->rowwords && (first_block != 0 || nblocks != r->nblocks)) { gg_set_error("datum-row relations are scanned whole"); return GG_ERR_ARG; }
	gg_engine *e = p->eng;
	GG_CUDA(cudaSetDevice(e->device));
	int rc = nblocks ? scanagg_adapt_to_pages(p, r->pages + first_block * GG_BLCKSZ, nullptr) : GG_OK;
	if (rc) return rc;
	GG_CUDA(cudaEventRecord(e->ev_start, e->stream));
	rc = scanagg_launch(p, r->pages + first_block * GG_BLCKSZ, nblocks, e->stream, r->nrows);
	if (rc) return rc;
	p->fed.push_back({ r->pages + first_block * GG_BLCKSZ, nullptr, nblocks, r->nrows, false, 0 });
	GG_CUDA(cudaEventRecord(e->ev_stop, e->stream));
	e->timed = true;
	return GG_OK;
}

/* SeqScan over an append-only column-oriented relation, fused with the Agg above it (aocsam.c:661 aocs_getnext + the same
 * qual / aggregate path as heap pages): the projected column files are resident in device memory with their block directories
 * and tile plans (include/gg_aocs.h); the plan's scan descriptor is the GG_FMT_DATUMROWS descriptor of those columns. */
int gg_scanagg_run_aocs(gg_scanagg *p, const struct gg_aocs_devcol *cols, int ncols, uint64_t nrows, int32_t tile_rows)
{
	if (!p || !cols || ncols < 1 || ncols > GG_MAX_ATTS || tile_rows < 32 || (tile_rows & 31)) return GG_ERR_ARG;
	if (!p->prog.outer.rowwords || p->prog.outer.rowwords != 1 + ncols)
	{ gg_set_error("the plan's scan descriptor must be the datum-row descriptor of the %d projected columns", ncols); return GG_ERR_ARG; }
	if (p->is_join || p->mode == MODE_BUILD || p->mode == MODE_PART) { gg_set_error("column files feed SeqScan -> Agg pipelines"); return GG_ERR_UNSUPPORTED; }
	gg_engine *e = p->eng;
	GG_CUDA(cudaSetDevice(e->device));
	for (int c = 0; c < ncols; c++)
		if (!cols[c].file || !cols[c].dir || !cols[c].tiles || cols[c].nblocks < 1 || cols[c].kind < GG_AOCS_K_W8 || cols[c].kind > GG_AOCS_K_TEXT)
		{ gg_set_error("AOCS column %d: incomplete descriptor", c); return GG_ERR_ARG; }
	{
		/* Rows per staging unit: the unit's values of every projected column share one 32 KB ring slot behind the 1.5 KB of run
		 * records (GG_AOCS_DATA_OFF), each column's range rounded out to 16 bytes and, where it crosses storage blocks, with the
		 * block headers in between (a block of the default 32 KB holds >= 1 800 values of these widths, so a unit crosses few).
		 * Strings are counted at the 9 bytes of the longest value the scan packs; a column that does not fit after all is read
		 * row by row, so this is a matter of speed only. */
		int rowbytes = 0;
		for (int c = 0; c < ncols; c++)
			rowbytes += cols[c].kind == GG_AOCS_K_W8 ? 8 : cols[c].kind == GG_AOCS_K_I4 ? 4 : cols[c].kind == GG_AOCS_K_I2 ? 2 : cols[c].kind == GG_AOCS_K_B1 ? 1 : 9;
		int ur = (GG_BLCKSZ - 32 * 48 - ncols * (32 + 3 * 64)) / rowbytes;
		ur &= ~31;
		if (ur > 1024) ur = 1024;
		if (ur < 32) ur = 32;
		p->aocs_unit_rows = ur;
	}
	if (!p->d_aocs) GG_CUDA(cudaMalloc((void **) &p->d_aocs, sizeof(gg_aocs_devcol) * GG_MAX_ATTS));
	GG_CUDA(cudaMemcpyAsync(p->d_aocs, cols, sizeof(gg_aocs_devcol) * (size_t) ncols, cudaMemcpyHostToDevice, e->stream));
	if (nrows == 0) return GG_OK;
	const uint64_t ntiles = (nrows + (uint64_t) tile_rows - 1) / (uint64_t) tile_rows;
	GG_CUDA(cudaEventRecord(e->ev_start, e->stream));
	int rc = scanagg_launch(p, (const uint8_t *) p->d_aocs, ntiles, e->stream, nrows, false, tile_rows);
	if (rc) return rc;
	p->fed.push_back({ (const uint8_t *) p->d_aocs, nullptr, ntiles, nrows, false, tile_rows });
	GG_CUDA(cudaEventRecord(e->ev_stop, e->stream));
	e->timed = true;
	return GG_OK;
}

/* Streamed end-to-end path: pages live in HOST memory (the segment's shared buffers / file cache).
 * Double-buffered 256 MB chunks: H2D on the copy stream overlaps the scan kernel of the previous
 * chunk on the compute stream. */
static int scanagg_stream_host(gg_scanagg *p, const void *host_pages, uint64_t nblocks);

int gg_scanagg_run_host(gg_scanagg *p, const void *host_pages, uint64_t nblocks)
{
	if (!p || (!host_pages && nblocks)) return GG_ERR_ARG;
	if (p->prog.outer.rowwords) { gg_set_error("datum rows are device-resident; the streamed path takes heap pages"); return GG_ERR_ARG; }
	int rc = nblocks ? scanagg_adapt_to_pages(p, nullptr, host_pages) : GG_OK;
	if (rc) return rc;
	rc = scanagg_stream_host(p, host_pages, nblocks);
	if (rc == GG_OK) p->fed.push_back({ nullptr, host_pages, nblocks, 0, false, 0 });
	return rc;
}

static int scanagg_stream_host(gg_scanagg *p, const void *host_pages, uint64_t nblocks)
{
	gg_engine *e = p->eng;
	GG_CUDA(cudaSetDevice(e->device));
	const uint64_t chunk = GG_STREAM_CHUNK_BLOCKS;
	for (int b = 0; b < 2; b++)
	{
		if (!p->stage[b])
		{
			GG_CUDA(cudaMalloc((void **) &p->stage[b], (size_t) chunk * GG_BLCKSZ));
			GG_CUDA(cudaEventCreateWithFlags(&p->ev_copied[b], cudaEventDisableTiming));
			GG_CUDA(cudaEventCreateWithFlags(&p->ev_consumed[b], cudaEventDisableTiming));
		}
	}
	GG_CUDA(cudaEventRecord(e->ev_start, e->stream));
	/* the copy stream must not overtake earlier work on the compute stream that used the staging buffers */
	GG_CUDA(cudaEventRecord(p->ev_consumed[0], e->stream));
	GG_CUDA(cudaEventRecord(p->ev_consumed[1], e->stream));
	uint64_t done = 0;
	int i = 0;
	while (done < nblocks)
	{
		uint64_t n = nblocks - done < chunk ? nblocks - done : chunk;
		int b = i & 1;
		GG_CUDA(cudaStreamWaitEvent(e->copy_stream, p->ev_consumed[b], 0));
		GG_CUDA(cudaMemcpyAsync(p->stage[b], (const uint8_t *) host_pages + done * GG_BLCKSZ, (size_t) n * GG_BLCKSZ,
		                        cudaMemcpyHostToDevice, e->copy_stream));
		GG_CUDA(cudaEventRecord(p->ev_copied[b], e->copy_stream));
		GG_CUDA(cudaStreamWaitEvent(e->stream, p->ev_copied[b], 0));
		int rc = scanagg_launch(p, p->stage[b], n, e->stream);
		if (rc) return rc;
		GG_CUDA(cudaEventRecord(p->ev_consumed[b], e->stream));
		done += n;
		i++;
	}
	GG_CUDA(cudaEventRecord(e->ev_stop, e->stream));
	e->timed = true;
	return GG_OK;
}

/* finalize_aggregate (nodeAgg.c:871-999) over the merged group records: O(groups) scalar work */
/* ---- numeric results (gg_plan.h "numeric") ----
 * The accumulated 128-bit integer (two int64 sums of the inputs' halves) is the exact sum at the argument's scale.
 * numeric_sum returns it as is; numeric_avg is numeric_div(sum, N::numeric) (numeric.c:3173): the result scale comes from
 * select_div_scale — NUMERIC_MIN_SIG_DIGITS (16) significant digits judged from the operands' base-10000 weights and first
 * digits, at least the operands' display scales (numeric.c select_div_scale) — and div_var rounds the quotient half away from
 * zero at that scale. */
typedef __int128 gg_i128;
typedef unsigned __int128 gg_u128;

/* base-10000 weight and first digit of |v| / 10^scale, as a NumericVar would hold them (leading zero digits stripped;
 * zero has no digits: weight 0, first digit 0) */
static void nbase_weight_first(gg_u128 mag, int scale, int *weight, int *first)
{
	*weight = 0; *first = 0;
	if (mag == 0) return;
	gg_u128 p = 1;
	for (int i = 0; i < scale; i++) p *= 10;
	gg_u128 ip = mag / p, fp = mag % p;
	if (ip > 0)
	{
		int w = 0;
		while (ip >= 10000) { ip /= 10000; w++; }
		*weight = w; *first = (int) ip;
		return;
	}
	/* purely fractional: digit groups of four decimals behind the point */
	int padded = (scale + 3) / 4 * 4;
	for (int i = scale; i < padded; i++) fp *= 10;
	int groups = padded / 4;
	for (int gi = 0; gi < groups; gi++)
	{
		gg_u128 q = 1;
		for (int k = 0; k < (groups - 1 - gi) * 4; k++) q *= 10;
		const int d = (int) ((fp / q) % 10000);
		if (d) { *weight = -(gi + 1); *first = d; return; }
	}
}

static void numeric_store(gg_aggval &v, gg_i128 val, int dscale)
{
	const uint64_t lo = (uint64_t) (gg_u128) val, hi = (uint64_t) ((gg_u128) val >> 64);
	v.i = (int64_t) lo;
	memcpy(&v.f[0], &hi, 8);
	v.f[1] = (double) dscale;
}

/* avg = round(sum / n) at select_div_scale's scale; false if the quotient does not fit 128 bits */
static bool numeric_avg128(gg_i128 sum, int sscale, uint64_t n, gg_i128 *out, int *rscale)
{
	const bool neg = sum < 0;
	const gg_u128 mag = neg ? (gg_u128) (-sum) : (gg_u128) sum;
	int w1, f1, w2, f2;
	nbase_weight_first(mag, sscale, &w1, &f1);
	nbase_weight_first((gg_u128) n, 0, &w2, &f2);
	int qweight = w1 - w2;
	if (f1 <= f2) qweight--;
	int rs = 16 - qweight * 4;                     /* NUMERIC_MIN_SIG_DIGITS - qweight * DEC_DIGITS */
	if (rs < sscale) rs = sscale;
	if (rs < 0) rs = 0;
	if (rs > 1000) rs = 1000;
	gg_u128 num = mag;
	for (int i = sscale; i < rs; i++)
	{
		if (num > ((gg_u128) ~(gg_u128) 0) / 10) return false;
		num *= 10;
	}
	gg_u128 q = num / n, r = num % n;
	if (2 * r >= (gg_u128) n) q++;                 /* round_var: half away from zero */
	if (q >> 127) return false;
	*out = neg ? -(gg_i128) q : (gg_i128) q;
	*rscale = rs;
	return true;
}

/* finalisation of a numeric sum / avg from the two accumulated halves, callable without a device (tests hold it to the
 * reference's numeric.o through tests/golden/numeric_kat.json): which = 0 sum, 1 avg.  Returns 0, or 1 when avg does not fit */
extern "C" int gg_debug_numeric_final(int which, int64_t lo, int64_t hi, int scale, uint64_t n, gg_aggval *out)
{
	const gg_i128 sum = (gg_i128) hi * ((gg_i128) 1 << 32) + (gg_i128) lo;
	memset(out, 0, sizeof *out);
	if (n == 0) { out->isnull = 1; return 0; }
	if (which == 0) { numeric_store(*out, sum, scale); return 0; }
	gg_i128 a = 0;
	int rs = 0;
	if (!numeric_avg128(sum, scale, n, &a, &rs)) { out->isnull = 1; return 1; }
	numeric_store(*out, a, rs);
	return 0;
}

static int finalize_rows(const gg_agg *agg, const ggp_aggmap *aggmap, const uint8_t *keytype, const ggp_grec *recs, int n, gg_aggrow *out)
{
	for (int g = 0; g < n; g++)
	{
		const ggp_grec &x = recs[g];
		gg_aggrow &row = out[g];
		memset(&row, 0, sizeof row);
		for (int c = 0; c < agg->numCols; c++)
		{
			row.keyisnull[c] = (x.keynull >> c) & 1;
			row.key[c] = (int64_t) x.key[c];
			if (keytype[c] == 3 && !row.keyisnull[c])
			{
				int len = 0;
				while (len < 8 && ((x.key[c] >> (8 * len)) & 0xff)) len++;
				row.keylen[c] = len;
			}
		}
		for (int i = 0; i < agg->numAggs; i++)
		{
			gg_aggval &v = row.agg[i];
			int col = aggmap[i].col;
			int fn = agg->aggs[i].aggfnoid;
			bool partial = agg->aggstage == GG_AGGSTAGE_PARTIAL;
			if (col < 0)                      /* count(*) */
			{
				v.i = (int64_t) x.count;
				continue;
			}
			uint64_t nn = x.n[col];
			int64_t ibits;
			memcpy(&ibits, &x.sum[col], 8);
			switch (fn)
			{
				case GG_AGG_COUNT_ANY:
					v.i = (int64_t) nn;
					break;
				case GG_AGG_SUM_FLOAT8:
				case GG_AGG_MIN_FLOAT8:
				case GG_AGG_MAX_FLOAT8:
					v.isnull = nn == 0;
					v.f[0] = nn ? x.sum[col] : 0.0;
					break;
				case GG_AGG_SUM_NUMERIC:
				case GG_AGG_AVG_NUMERIC:
				{
					int64_t lo, hi;
					memcpy(&lo, &x.sum[col], 8); memcpy(&hi, &x.sum[col + 1], 8);
					const gg_i128 sum = (gg_i128) hi * ((gg_i128) 1 << 32) + (gg_i128) lo;
					v.isnull = nn == 0;              /* numeric_sum / numeric_avg over no input: NULL (numeric.c:3181,3213) */
					if (nn == 0) break;
					if (fn == GG_AGG_SUM_NUMERIC) numeric_store(v, sum, aggmap[i].scale);
					else
					{
						gg_i128 a = 0;
						int rs = 0;
						if (!numeric_avg128(sum, aggmap[i].scale, nn, &a, &rs))
						{
							gg_set_error("numeric avg whose quotient does not fit 128 bits at its scale");
							return GG_ERR_UNSUPPORTED;
						}
						numeric_store(v, a, rs);
					}
					break;
				}
				case GG_AGG_AVG_FLOAT8:
					if (partial)
					{
						/* float8_accum's state starts from "{0,0,0}": + 0.0 turns the -0 the sums start from into +0 */
						v.f[0] = (double) nn; v.f[1] = x.sum[col] + 0.0; v.f[2] = x.sumsq[col] + 0.0;
					}
					else if (nn == 0)
						v.isnull = 1;            /* float8_avg: N == 0 => NULL (float.c:1995) */
					else
						v.f[0] = (x.sum[col] + 0.0) / (double) nn;
					break;
				default:                      /* int sum/min/max */
					v.isnull = nn == 0;
					v.i = nn ? ibits : 0;
					break;
			}
		}
	}
	return GG_OK;
}

/* merged group records -> rows (finalize_aggregate, nodeAgg.c:871-999).  Plain aggregation over zero rows still yields one row
 * (nodeAgg.c:1247-1400), unless `empty_is_empty` (a segment that does not own the result). */
static int records_to_rows(const gg_agg *agg, const ggp_aggmap *aggmap, const uint8_t *keytype, std::vector<ggp_grec> &recs,
                           long long n, bool empty_is_empty, gg_aggrow *out, int outcap, int *nout)
{
	if (n == 0 && agg->numCols == 0 && !empty_is_empty) { recs.resize(1); memset(&recs[0], 0, sizeof(ggp_grec)); n = 1; }
	if (n > outcap) { gg_set_error("output capacity %d < %lld groups", outcap, n); return GG_ERR_NOMEM; }
	const int rc = finalize_rows(agg, aggmap, keytype, recs.data(), (int) n, out);
	if (rc) return rc;
	*nout = (int) n;
	return GG_OK;
}

/* Run the fed inputs again on kernel variant `mode` (MODE_HASH: into a group table of `ha_cap` slots): reconfigure, reset, and
 * feed everything again — through the batched join's replay_hook when there is one — like the reference's hybrid hash
 * aggregate re-reading spilled input (execHHashagg.c:1093). */
int scanagg_replay(gg_scanagg *p, int mode, uint64_t ha_cap)
{
	gg_engine *e = p->eng;
	std::vector<gg_scanagg::Fed> replay = p->fed;
	p->mode = mode;
	int rc = scanagg_configure(p);
	if (rc) return rc;
	p->nrecs_total = GG_MERGE_CAP + p->grid * GGP_FAST_GROUPS;
	if (mode == MODE_HASH)
	{
		p->ha_cap = ha_cap;
		if (p->ha_mem) { GG_CUDA(cudaStreamSynchronize(e->stream)); cudaFree(p->ha_mem); p->ha_mem = nullptr; }
	}
	rc = gg_scanagg_reset(p);
	if (rc) return rc;
	if (p->replay_hook) return p->replay_hook();
	for (const auto &f : replay)
	{
		rc = f.dev ? scanagg_launch(p, f.dev, f.nblocks, e->stream, f.nrows, f.fill, f.tile_rows) : scanagg_stream_host(p, f.host, f.nblocks);
		if (rc) return rc;
	}
	p->fed = replay;
	return GG_OK;
}

int gg_scanagg_fetch(gg_scanagg *p, gg_aggrow *out, int outcap, int *nout,
                     uint64_t *rows_scanned, uint64_t *rows_passed)
{
	if (!p || !nout) return GG_ERR_ARG;
	gg_engine *e = p->eng;
	GG_CUDA(cudaSetDevice(e->device));
	GG_CUDA(cudaStreamSynchronize(e->copy_stream));
	/* one round trip: status words and (speculatively) the first merged group records, behind everything queued */
	GG_CUDA(cudaMemcpyAsync(&p->h_mirror->st, p->d_status, sizeof(gg_scanagg::Status), cudaMemcpyDeviceToHost, e->stream));
	GG_CUDA(cudaMemcpyAsync(p->h_mirror->recs, p->recs, sizeof p->h_mirror->recs, cudaMemcpyDeviceToHost, e->stream));
	GG_CUDA(cudaStreamSynchronize(e->stream));
	uint32_t flags = p->h_mirror->st.err;
	unsigned long long counters[2] = { p->h_mirror->st.counters[0], p->h_mirror->st.counters[1] };
	int n = p->h_mirror->st.nout;
	if (p->build_err)
	{
		const int brc = gg_errflags_to_code(p->build_err);        /* the join's hash table holds a value the device refused */
		if (brc) return brc;
	}
	/* Escalation, then the inputs are replayed and fetched again.  Private accumulators: more groups than they hold (the
	 * planner's numGroups was low or absent), or a non-finite private sum, which only the value-tracking transposed variant can
	 * attribute to an infinite input or to a float8pl overflow.  A block-table variant with more groups than a block holds:
	 * the general HashAggregate.  Its table full: one 8 times larger. */
	int next = -1;
	uint64_t cap = 0;
	if (p->mode == MODE_PRIV && (flags & (GGP_EF_GROUP_OVERFLOW | GGP_EF_RECHECK))) next = p->prog.nullable ? MODE_TRN : MODE_TR;
	else if (p->mode != MODE_HASH && (flags & GGP_EF_GROUP_OVERFLOW)) { next = MODE_HASH; cap = p->ha_cap ? p->ha_cap : 1u << 20; }
	else if (p->mode == MODE_HASH && (flags & GGP_EF_TABLE_FULL)) { next = MODE_HASH; cap = p->ha_cap * 8; }
	if (next >= 0)
	{
		if (cap > (1ull << 31)) { gg_set_error("more groups than the device hash aggregate can hold"); return GG_ERR_NOMEM; }
		int rc = scanagg_replay(p, next, cap);
		return rc ? rc : gg_scanagg_fetch(p, out, outcap, nout, rows_scanned, rows_passed);
	}
	if (rows_scanned) *rows_scanned = counters[0];
	if (rows_passed) *rows_passed = counters[1];
	std::vector<ggp_grec> recs;
	if (p->mode == MODE_HASH)
	{
		/* the general HashAggregate: the groups come out of its table */
		unsigned long long n64 = 0;
		const unsigned long long ecap = (unsigned long long) (outcap > 0 ? outcap : 1);
		ggp_grec *d_recs = nullptr;
		if (p->has_state)
		{
			GG_CUDA(cudaMalloc((void **) &d_recs, sizeof(ggp_grec) * ecap));
			cudaError_t ce = cudaMemsetAsync(p->d_nout64, 0, sizeof n64, e->stream);
			if (ce == cudaSuccess)
			{
				gg_hashagg_emit_kernel<<<e->sm_count * 8, 256, 0, e->stream>>>(p->ha, d_recs, ecap, p->d_nout64, p->d_err);
				ce = cudaGetLastError();
				e->launches++;
			}
			if (ce == cudaSuccess) ce = cudaMemcpyAsync(&n64, p->d_nout64, sizeof n64, cudaMemcpyDeviceToHost, e->stream);
			if (ce == cudaSuccess) ce = cudaMemcpyAsync(&flags, p->d_err, sizeof flags, cudaMemcpyDeviceToHost, e->stream);
			if (ce == cudaSuccess) ce = cudaStreamSynchronize(e->stream);
			if (ce == cudaSuccess && n64 <= ecap && n64 > 0)
			{
				recs.resize((size_t) n64);
				ce = cudaMemcpy(recs.data(), d_recs, sizeof(ggp_grec) * (size_t) n64, cudaMemcpyDeviceToHost);
			}
			cudaFree(d_recs);
			if (ce != cudaSuccess) return gg_cuda_fail(ce, "gg_scanagg_fetch(hash)");
		}
		int rc = gg_errflags_to_code(flags & ~(uint32_t) GGP_EF_GROUP_OVERFLOW);
		if (rc) return rc;
		return records_to_rows(&p->agg, p->aggmap, p->prog.keytype, recs, (long long) n64, false, out, outcap, nout);
	}
	int rc = gg_errflags_to_code(flags);
	if (rc) return rc;
	if (!p->has_state) n = 0;
	recs.resize((size_t) (n > 0 ? n : 0));
	if (n > 0 && n <= GGP_FAST_GROUPS) memcpy(recs.data(), p->h_mirror->recs, sizeof(ggp_grec) * (size_t) n);     /* already here */
	else if (n > 0) GG_CUDA(cudaMemcpy(recs.data(), p->recs, sizeof(ggp_grec) * n, cudaMemcpyDeviceToHost));
	return records_to_rows(&p->agg, p->aggmap, p->prog.keytype, recs, n, false, out, outcap, nout);
}

int gg_scanagg_scan_kernel_ms(gg_scanagg *p, float *ms, int *launches)
{
	if (!p || !ms) return GG_ERR_ARG;
	GG_CUDA(cudaSetDevice(p->eng->device));
	float tot = 0;
	for (size_t i = 0; i < p->kev_used; i++)
	{
		float t = 0;
		GG_CUDA(cudaEventSynchronize(p->kev[i].second));
		GG_CUDA(cudaEventElapsedTime(&t, p->kev[i].first, p->kev[i].second));
		tot += t;
	}
	*ms = tot;
	if (launches) *launches = (int) p->kev_used;
	return GG_OK;
}

int gg_scanagg_variant(gg_scanagg *p)
{
	if (!p) return -1;
	return p->mode + (p->jit ? (p->jit->precompiled ? 16 : 32) : 0);
}

void gg_scanagg_free(gg_scanagg *p)
{
	if (!p) return;
	for (auto &ev : p->kev) { cudaEventDestroy(ev.first); cudaEventDestroy(ev.second); }
	cudaSetDevice(p->eng->device);
	cudaStreamSynchronize(p->eng->stream);
	cudaFree(p->recs); cudaFree(p->merged); cudaFree(p->vidx); cudaFree(p->vmap);
	cudaFree(p->d_status); cudaFreeHost(p->h_mirror); cudaFree(p->d_nout64); cudaFree(p->ha_mem); cudaFree(p->d_aocs);
	for (int b = 0; b < 2; b++)
	{
		if (p->stage[b]) cudaFree(p->stage[b]);
		if (p->ev_copied[b]) cudaEventDestroy(p->ev_copied[b]);
		if (p->ev_consumed[b]) cudaEventDestroy(p->ev_consumed[b]);
	}
	delete p;
}

/* FINAL-stage Agg over partial rows on the host: the rows become group records laid out as a PARTIAL pipeline leaves them on
 * the device, and gg_groups_final combines them (float8pl / float8_combine / int8pl, nodeAgg.c:2123-2148, float.c:1842,
 * int8.c:513). */
int gg_agg_final(gg_engine *e, const gg_agg *agg, const gg_aggrow *in, int nin,
                 gg_aggrow *out, int outcap, int *nout)
{
	if (!e || !agg || !nout || (nin && !in)) return GG_ERR_ARG;
	if (agg->numCols < 0 || agg->numCols > GG_MAX_KEYS || agg->numAggs < 0 || nin < 0 || outcap < 0 || (outcap && !out))
	{ gg_set_error("gg_agg_final: %d grouping columns, %d aggregates, %d rows in, room for %d", agg->numCols, agg->numAggs, nin, outcap); return GG_ERR_ARG; }
	if (agg->numAggs > GGP_MAX_ACCS) { gg_set_error("too many aggregates"); return GG_ERR_UNSUPPORTED; }
	GG_CUDA(cudaSetDevice(e->device));
	gg_groups like = gg_groups();
	like.agg = *agg;
	like.nkeys = agg->numCols;
	for (int c = 0; c < agg->numCols; c++)
	{
		int32_t t = agg->grpCol[c];                    /* a FINAL Agg's grpCol carries the key type OIDs */
		like.keytype[c] = (t == GG_FLOAT8OID) ? 2 : (t == GG_BPCHAROID || t == GG_VARCHAROID || t == GG_TEXTOID) ? 3 : 1;
	}
	for (int i = 0; i < agg->numAggs; i++)
	{
		const int fn = agg->aggs[i].aggfnoid, kind = ggp_acckind_of(fn);
		if (kind < 0 || fn == GG_AGG_SUM_NUMERIC || fn == GG_AGG_AVG_NUMERIC) { gg_set_error("aggregate %d not supported", fn); return GG_ERR_UNSUPPORTED; }
		like.aggmap[i].col = kind ? like.nacc : -1;
		if (kind) like.acckind[like.nacc++] = (uint8_t) kind;
	}
	std::vector<ggp_grec> recs((size_t) nin);
	uint32_t hostflags = 0;
	for (int r = 0; r < nin; r++)
	{
		ggp_grec &x = recs[r];
		x.valid = 1;
		for (int c = 0; c < agg->numCols; c++)
		{
			if (in[r].keyisnull[c]) x.keynull |= 1u << c;
			else
			{
				uint64_t k = (uint64_t) in[r].key[c];
				if (like.keytype[c] == 2)
				{
					/* group_key: a zero keeps its sign, the merge compares ±0 alike; NaNs are one key */
					double d; memcpy(&d, &k, 8);
					if (d != d) k = 0x7ff8000000000000ull;
				}
				else if (agg->grpCol[c] == GG_INT4OID || agg->grpCol[c] == GG_DATEOID)
					k = (uint64_t) (int64_t) (int32_t) k;
				x.key[c] = k;
			}
		}
		for (int i = 0; i < agg->numAggs; i++)
		{
			const gg_aggval &v = in[r].agg[i];
			const int j = like.aggmap[i].col;
			switch (agg->aggs[i].aggfnoid)
			{
				case GG_AGG_COUNT_STAR:
					x.count = v.isnull ? 0 : (uint64_t) v.i;
					break;
				case GG_AGG_COUNT_ANY:
					x.n[j] = v.isnull ? 0 : (uint64_t) v.i;
					break;
				case GG_AGG_AVG_FLOAT8:
					x.n[j] = (uint64_t) v.f[0]; x.sum[j] = v.f[1]; x.sumsq[j] = v.f[2];
					if (!(fabs(v.f[1]) < INFINITY) || !(fabs(v.f[2]) < INFINITY)) hostflags |= GGP_EF_SAW_INF;
					/* float8_combine adds N even when it is 0; a zero-N state contributes nothing */
					break;
				case GG_AGG_SUM_FLOAT8: case GG_AGG_MIN_FLOAT8: case GG_AGG_MAX_FLOAT8:
					x.n[j] = v.isnull ? 0 : 1; x.sum[j] = v.f[0];
					if (!v.isnull && !(fabs(v.f[0]) < INFINITY)) hostflags |= GGP_EF_SAW_INF;
					break;
				default:
					x.n[j] = v.isnull ? 0 : 1; memcpy(&x.sum[j], &v.i, 8);
					break;
			}
		}
	}
	gg_groups *g = gg_groups_alloc(e, &like, nin, false);
	if (!g) return GG_ERR_NOMEM;
	/* GGP_EF_SAW_INF lets the merge tell an infinite partial sum from a float8pl overflow */
	const gg_groupstatus st = { hostflags, nin, { 0, 0 } };
	cudaError_t ce = nin ? cudaMemcpyAsync(g->recs, recs.data(), sizeof(ggp_grec) * (size_t) nin, cudaMemcpyHostToDevice, e->stream) : cudaSuccess;
	if (ce == cudaSuccess) ce = cudaMemcpyAsync(g->d_status, &st, sizeof st, cudaMemcpyHostToDevice, e->stream);
	gg_groups *fin = nullptr;
	int rc = ce != cudaSuccess ? gg_cuda_fail(ce, "gg_agg_final") : gg_groups_final(e, g, &fin);
	if (rc == GG_OK) rc = gg_groups_fetch(fin, out, outcap, nout, nullptr, nullptr);
	gg_groups_free(fin);
	gg_groups_free(g);
	return rc;
}


/* ---------------- device-resident group records (gg_groups.h) ---------------- */

}  /* extern "C" */

/* buffers of the common size are recycled through the engine: a Motion per step must not cost a cudaMalloc */
#define GG_GROUPS_POOL_CAP 256
static size_t groups_bytes(int cap) { return sizeof(ggp_grec) * (size_t) cap + sizeof(gg_groupstatus) + 16 + 2 * sizeof(int) * (size_t) cap; }

gg_groups *gg_groups_alloc(gg_engine *e, const gg_groups *like, int cap, bool sparse)
{
	gg_groups *g = new gg_groups();
	if (like) *g = *like;
	g->eng = e; g->cap = cap; g->sparse = sparse; g->owned = true;
	const int alloc_cap = cap <= GG_GROUPS_POOL_CAP ? GG_GROUPS_POOL_CAP : cap;
	void *mem = nullptr;
	if (alloc_cap == GG_GROUPS_POOL_CAP && !e->groups_pool.empty()) { mem = e->groups_pool.back(); e->groups_pool.pop_back(); }
	else if (cudaMalloc(&mem, groups_bytes(alloc_cap)) != cudaSuccess) { cudaGetLastError(); gg_set_error("out of device memory for %d group records", cap); delete g; return nullptr; }
	g->recs = (ggp_grec *) mem;
	g->d_status = (gg_groupstatus *) (g->recs + alloc_cap);
	g->d_n = &g->d_status->n;
	g->scratch = (int *) ((uint8_t *) g->d_status + sizeof(gg_groupstatus) + 8);
	g->alloc_cap = alloc_cap;
	return g;
}

extern "C" {

void gg_groups_free(gg_groups *g)
{
	if (!g) return;
	if (g->owned && g->recs)
	{
		/* stream-ordered reuse: whoever takes the buffer next works on the same stream */
		if (g->alloc_cap == GG_GROUPS_POOL_CAP && g->eng->groups_pool.size() < 16) g->eng->groups_pool.push_back(g->recs);
		else { cudaStreamSynchronize(g->eng->stream); cudaFree(g->recs); }
	}
	delete g;
}

static void groups_meta_from_pipeline(gg_groups *g, const gg_scanagg *p)
{
	g->agg = p->agg;
	memcpy(g->aggmap, p->aggmap, sizeof g->aggmap);
	g->nkeys = p->prog.nkeys; g->nacc = p->prog.nacc;
	memcpy(g->keytype, p->prog.keytype, sizeof g->keytype);
	memcpy(g->acckind, p->prog.acckind, sizeof g->acckind);
	for (int c = 0; c < GG_MAX_KEYS; c++)
		g->keytypid[c] = (c < p->agg.numCols && p->agg.grpCol[c] >= 0 && p->agg.grpCol[c] < p->pool.nnodes) ? p->pool.nodes[p->agg.grpCol[c]].rettype : 0;
}

/* the result of a pipeline, left where it is: a view into the pipeline's merged records (valid until its next reset).
 * The general HashAggregate keeps its groups in the HBM table: GG_ERR_UNSUPPORTED, the caller fetches rows instead. */
int gg_scanagg_groups(gg_scanagg *p, gg_groups **out)
{
	if (!p || !out) return GG_ERR_ARG;
	*out = nullptr;
	if (p->mode == MODE_HASH) { gg_set_error("the general HashAggregate's groups live in its hash table"); return GG_ERR_UNSUPPORTED; }
	gg_groups *g = new gg_groups();
	g->eng = p->eng;
	g->recs = p->recs; g->cap = GG_MERGE_CAP; g->sparse = false;
	g->d_status = (gg_groupstatus *) p->d_status;
	g->d_n = &g->d_status->n;
	g->owned = false;
	groups_meta_from_pipeline(g, p);
	*out = g;
	return GG_OK;
}

/* FINAL-stage Agg on the device: combine partial group records — what a Motion delivered, a pipeline's result or the rows
 * gg_agg_final was given (float8pl / float8_combine / int8pl, nodeAgg.c:2123-2148) — with the deterministic merge kernel; the
 * result reads like a one-stage aggregate's. */
int gg_groups_final(gg_engine *e, gg_groups *in, gg_groups **out)
{
	if (!e || !in || !out) return GG_ERR_ARG;
	*out = nullptr;
	GG_CUDA(cudaSetDevice(e->device));
	/* every valid record of the input may be a group of its own, so the output has the input's size */
	const int cap = in->cap;
	gg_groups *g = gg_groups_alloc(e, in, cap, false);
	if (!g) return GG_ERR_NOMEM;
	g->agg.aggstage = GG_AGGSTAGE_NORMAL;          /* combined states finalise like a one-stage aggregate's (float8_avg = sumX / N) */
	cudaStream_t st = e->stream;
	ggp_acckinds kinds;
	memcpy(kinds.k, in->acckind, sizeof kinds.k);
	cudaError_t ce = cudaMemcpyAsync(g->d_status, in->d_status, sizeof(gg_groupstatus), cudaMemcpyDeviceToDevice, st);
	if (ce == cudaSuccess) ce = cudaMemsetAsync(g->recs, 0, sizeof(ggp_grec) * (size_t) cap, st);
	if (ce == cudaSuccess)
	{
		gg_merge_recs_kernel<<<1, 1024, 0, st>>>(in->recs, cap, in->nkeys, keytypes_of(in->keytype), in->nacc, kinds, g->recs, cap, g->d_n,
		                                        g->scratch, g->scratch + g->alloc_cap, &g->d_status->err, in->sparse ? 0 : 1);
		ce = cudaGetLastError();
		e->launches++;
	}
	if (ce != cudaSuccess) { gg_groups_free(g); return gg_cuda_fail(ce, "gg_groups_final"); }
	*out = g;
	return GG_OK;
}

/* the one host synchronisation of a device-resident slice: records + status -> rows (finalize_aggregate, nodeAgg.c:871) */
int gg_groups_fetch(gg_groups *g, gg_aggrow *out, int outcap, int *nout, uint64_t *rows_scanned, uint64_t *rows_passed)
{
	if (!g || !nout || outcap < 0 || (outcap && !out)) return GG_ERR_ARG;
	gg_engine *e = g->eng;
	GG_CUDA(cudaSetDevice(e->device));
	cudaStream_t st = e->stream;
	if (!e->groups_mirror) GG_CUDA(cudaHostAlloc(&e->groups_mirror, groups_bytes(GG_GROUPS_POOL_CAP), cudaHostAllocDefault));
	gg_groupstatus *hs = (gg_groupstatus *) e->groups_mirror;
	ggp_grec *hr = (ggp_grec *) ((uint8_t *) e->groups_mirror + 64);
	const int first = g->sparse ? (g->cap < GG_GROUPS_POOL_CAP ? g->cap : GG_GROUPS_POOL_CAP) : GGP_FAST_GROUPS;
	GG_CUDA(cudaMemcpyAsync(hs, g->d_status, sizeof *hs, cudaMemcpyDeviceToHost, st));
	GG_CUDA(cudaMemcpyAsync(hr, g->recs, sizeof(ggp_grec) * (size_t) first, cudaMemcpyDeviceToHost, st));
	GG_CUDA(cudaStreamSynchronize(st));
	if (rows_scanned) *rows_scanned = hs->counters[0];
	if (rows_passed) *rows_passed = hs->counters[1];
	const uint32_t flags = hs->err;
	int rc = gg_errflags_to_code(flags);
	if (rc) return rc;
	std::vector<ggp_grec> recs;
	if (g->sparse)
	{
		std::vector<ggp_grec> all;
		const ggp_grec *src = hr;
		if (g->cap > first)
		{
			all.resize((size_t) g->cap);
			GG_CUDA(cudaMemcpy(all.data(), g->recs, sizeof(ggp_grec) * (size_t) g->cap, cudaMemcpyDeviceToHost));
			src = all.data();
		}
		for (int i = 0; i < g->cap; i++) if (src[i].valid) recs.push_back(src[i]);
	}
	else
	{
		const int n = hs->n;
		if (n < 0 || n > g->cap) { gg_set_error("group record count %d out of range", n); return GG_ERR_CUDA; }
		recs.resize((size_t) n);
		if (n > 0 && n <= first) memcpy(recs.data(), hr, sizeof(ggp_grec) * (size_t) n);
		else if (n > 0) GG_CUDA(cudaMemcpy(recs.data(), g->recs, sizeof(ggp_grec) * (size_t) n, cudaMemcpyDeviceToHost));
	}
	return records_to_rows(&g->agg, g->aggmap, g->keytype, recs, (long long) recs.size(), g->empty_is_empty, out, outcap, nout);
}

int gg_groups_info(gg_groups *g, int *sparse, int *cap)
{
	if (!g) return GG_ERR_ARG;
	if (sparse) *sparse = g->sparse ? 1 : 0;
	if (cap) *cap = g->cap;
	return GG_OK;
}

/* a non-receiving segment of a Gather holds no rows: not even the empty-input row of a plain aggregate */
void gg_groups_set_nonreceiver(gg_groups *g) { if (g) g->empty_is_empty = true; }
}  /* extern "C" */
