/*
 * gg_motion.cu — the sending side of a Redistribute Motion on the device (include/ggb200.h gg_motion_partition):
 * the scan kernel body in its MODE_PART role (interpreter path) and the host call around it.
 */
#include <cstdlib>
#include <vector>
#include "gg_pipeline.h"

using namespace ggd;

/* sending Motion: route every qualifying row and write it into its destination's region */
__global__ void __launch_bounds__(256, 2)
gg_motion_part_kernel(const __grid_constant__ ggp_program P, const ScanAggParams prm)
{
	scanagg_body<MODE_PART, DynPlan>(P, prm);
}

extern "C" {

/* Redistribute Motion, sending side.  out region d = rows [d * cap, d * cap + counts[d]) with cap = out_cap_rows / nsegs. */
int gg_motion_partition(gg_engine *e, const gg_scan *scan, const gg_exprpool *pool,
                        const int32_t *hashkeys, int nkeys, const int32_t *payload, int npayload,
                        int nsegs, gg_relation *r, uint64_t first_block, uint64_t nblocks,
                        void *device_out_rows, uint64_t out_cap_rows,
                        uint64_t *host_counts, uint64_t *host_offsets)
{
	return gg_partition_rows(e, scan, pool, hashkeys, nkeys, payload, npayload, nsegs, 0, 0, r, first_block, nblocks,
	                         device_out_rows, out_cap_rows, host_counts, host_offsets);
}

}  /* extern "C" */

/* the same kernel with either routing rule (MotionOut.route): segments of a Motion, or batches of a hybrid hash join */
int gg_partition_rows(gg_engine *e, const gg_scan *scan, const gg_exprpool *pool,
                      const int32_t *hashkeys, int nkeys, const int32_t *payload, int npayload,
                      int nsegs, int route, int shift, gg_relation *r, uint64_t first_block, uint64_t nblocks,
                      void *device_out_rows, uint64_t out_cap_rows,
                      uint64_t *host_counts, uint64_t *host_offsets)
{
	if (!e || !scan || !pool || !hashkeys || !payload || !r || !host_counts || nsegs < 1 || nsegs > 1024 ||
	    nblocks > r->nblocks || first_block > r->nblocks - nblocks || (!device_out_rows && out_cap_rows))
		return GG_ERR_ARG;
	GG_CUDA(cudaSetDevice(e->device));
	std::vector<ggp_program> progbuf(1);   /* 3 KB: kept off the stack */
	ggp_program &prog = progbuf[0];
	uint8_t hashtype[GG_MAX_KEYS] = { 0 };
	char msg[256];
	int rc = ggp_compile_motion(scan, pool, hashkeys, nkeys, payload, npayload, &prog, hashtype, msg, sizeof msg);
	if (rc != GG_OK) { gg_set_error("%s", msg); return rc; }
	if (r->rowwords != prog.outer.rowwords) { gg_set_error("relation format does not match the plan's tuple descriptor"); return GG_ERR_ARG; }
	if (r->rowwords && (first_block != 0 || nblocks != r->nblocks)) { gg_set_error("datum-row relations are scanned whole"); return GG_ERR_ARG; }
	cudaStream_t st = e->stream;
	/* [nsegs] cursors, [1] error flags, [2] counters: one small block per engine, kept across calls */
	if (!e->motion_state) GG_CUDA(cudaMalloc(&e->motion_state, (size_t) (1024 + 4) * 8));
	unsigned long long *d_state = (unsigned long long *) e->motion_state;
	cudaError_t ce = cudaMemsetAsync(d_state, 0, (size_t) (nsegs + 4) * 8, st);
	ScanAggParams prm;
	memset(&prm, 0, sizeof prm);
	prm.pages = r->pages + first_block * GG_BLCKSZ;
	prm.nblocks = nblocks;
	prm.nrows = r->nrows;
	prm.snap = e->d_snapshot;
	prm.errflags = (uint32_t *) (d_state + nsegs);
	prm.counters = d_state + nsegs + 1;
	const gg_launch c = gg_np_launch(2, ((prog.outer.ncols * 64 + 15) & ~15) + 512 + 16);     /* column offsets + the warp's claim windows */
	prm.nstage = c.nstage;
	prm.team = c.team;
	prm.scratch_per_warp = c.scratch_per_warp;
	prm.scratch_off = c.scratch_off;
	prm.mo.rows = (unsigned long long *) device_out_rows;
	prm.mo.cursor = d_state;
	prm.mo.cap = (out_cap_rows / (uint64_t) nsegs) & ~1ull;      /* even: every region starts 16-byte aligned */
	prm.mo.nsegs = nsegs;
	prm.mo.rowwords = 1 + npayload;
	prm.mo.route = (uint32_t) route;
	prm.mo.shift = (uint32_t) shift;
	if (route && (nsegs & (nsegs - 1))) { gg_set_error("batch routing needs a power-of-two batch count"); return GG_ERR_ARG; }
	for (int k = 0; k < nkeys; k++) prm.mo.hashtypes |= (uint32_t) hashtype[k] << (4 * k);
	{
		/* claim windows (MotionOut.window): as large as keeps the unused tails of all warps below 1/8 of a region */
		const uint64_t warps = (uint64_t) e->sm_count * c.ctas * (c.threads / 32 - 1);
		const uint64_t w = prm.mo.cap / (warps * 8);
		uint32_t window = 0;
		if (nsegs <= 32 && w >= 32) { window = 32; while (window * 2 <= w && window < 1024) window *= 2; }
		const char *env = getenv("GGB200_MOTION_WINDOW");            /* experiments: 0 = exact claims */
		if (env && nsegs <= 32) { int v = atoi(env); if (v == 0 || (v >= 32 && v <= 4096)) window = (uint32_t) v; }
		prm.mo.window = window;
	}
	if (ce == cudaSuccess) ce = cudaEventRecord(e->ev_start, st);
	if (ce == cudaSuccess)
	{
		const void *fn = nullptr;
		int rc2 = gg_scan_kernel(&prog, MODE_PART, -1, c, e->device, e->d_snapshot != nullptr, &fn);
		if (rc2) return rc2;
		void *args[] = { (void *) &prog, (void *) &prm };
		ce = cudaLaunchKernel(fn, dim3(e->sm_count * c.ctas), dim3(c.threads), args, c.smem, st);
		e->launches++;
	}
	if (ce == cudaSuccess) ce = cudaEventRecord(e->ev_stop, st);
	e->timed = true;
	std::vector<unsigned long long> host((size_t) nsegs + 4);
	if (ce == cudaSuccess) ce = cudaMemcpyAsync(host.data(), d_state, (size_t) (nsegs + 4) * 8, cudaMemcpyDeviceToHost, st);
	if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
	if (ce != cudaSuccess) return gg_cuda_fail(ce, "gg_motion_partition");
	uint32_t flags = (uint32_t) host[(size_t) nsegs];
	for (int d = 0; d < nsegs; d++)
	{
		host_counts[d] = host[(size_t) d] < prm.mo.cap ? host[(size_t) d] : prm.mo.cap;
		if (host_offsets) host_offsets[d] = (uint64_t) d * prm.mo.cap;
	}
	if (flags & GGP_EF_TABLE_FULL)
	{
		unsigned long long need = 0;
		for (int d = 0; d < nsegs; d++) if (host[(size_t) d] > need) need = host[(size_t) d];
		gg_set_error("motion output region too small: a destination receives %llu rows, capacity %llu", need, (unsigned long long) prm.mo.cap);
		return GG_ERR_NOMEM;
	}
	return gg_errflags_to_code(flags);
}
