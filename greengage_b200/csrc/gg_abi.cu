/*
 * gg_abi.cu — engine, relation and host-staging entry points of include/ggb200.h.
 * The operator entry points live next to their kernels (gg_scanagg.cu, gg_join.cu, ...).
 */
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <vector>
#include "gg_engine.h"

static thread_local char g_err[512] = "";

void gg_set_error(const char *fmt, ...)
{
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(g_err, sizeof g_err, fmt, ap);
	va_end(ap);
}

int gg_cuda_fail(cudaError_t e, const char *what)
{
	gg_set_error("CUDA error %d (%s) in %s", (int) e, cudaGetErrorString(e), what);
	cudaGetLastError();
	return GG_ERR_CUDA;
}

int gg_errflags_to_code(uint32_t f)
{
	f &= ~(uint32_t) GGP_EF_INFO_MASK;
	if (!f) return GG_OK;
	if (f & GGP_EF_BADPAGE) { gg_set_error("corrupted page or tuple pointers"); return GG_ERR_BADPAGE; }
	if (f & GGP_EF_VISIBILITY) { gg_set_error("tuple visibility needs clog/snapshot (not frozen)"); return GG_ERR_VISIBILITY; }
	if (f & GGP_EF_NOTNULL_VIOLATED) { gg_set_error("NULL found in a column declared NOT NULL"); return GG_ERR_BADPAGE; }
	if (f & GGP_EF_FLOAT_OVERFLOW) { gg_set_error("value out of range: overflow"); return GG_ERR_FLOAT_OVERFLOW; }
	if (f & GGP_EF_FLOAT_UNDERFLOW) { gg_set_error("value out of range: underflow"); return GG_ERR_FLOAT_UNDERFLOW; }
	if (f & GGP_EF_DIV_ZERO) { gg_set_error("division by zero"); return GG_ERR_DIV_ZERO; }
	if (f & GGP_EF_INT_OVERFLOW) { gg_set_error("bigint out of range"); return GG_ERR_INT_OVERFLOW; }
	if (f & GGP_EF_DATE_RANGE) { gg_set_error("date out of range for timestamp"); return GG_ERR_DATE_RANGE; }
	if (f & GGP_EF_NUMERIC_RANGE) { gg_set_error("numeric value outside the scaled 64-bit range of the GPU path (or NaN, or more fractional digits than the column's scale)"); return GG_ERR_UNSUPPORTED; }
	if (f & GGP_EF_STRING_TOO_LONG) { gg_set_error("string value longer than 8 bytes (or toasted) in a GPU expression"); return GG_ERR_UNSUPPORTED; }
	if (f & GGP_EF_PEER_FAILED) { gg_set_error("another segment reported an error in its slice below the Motion"); return GG_ERR_PEER; }
	if (f & GGP_EF_HOSTPATH) { gg_set_error("a segment could not keep its aggregate rows on the device: run the slice with host-row Motions"); return GG_ERR_RETRY_HOST; }
	if (f & GGP_EF_GROUP_OVERFLOW) { gg_set_error("more groups than the GPU aggregate holds"); return GG_ERR_UNSUPPORTED; }
	if (f & GGP_EF_TABLE_FULL) { gg_set_error("hash table full"); return GG_ERR_NOMEM; }
	gg_set_error("device error flags 0x%x", f);
	return GG_ERR_CUDA;
}

extern "C" {

const char *gg_last_error(void) { return g_err; }

const char *gg_strerror(int code)
{
	switch (code)
	{
		case GG_OK: return "ok";
		case GG_ERR_CUDA: return "CUDA error";
		case GG_ERR_FLOAT_OVERFLOW: return "value out of range: overflow";
		case GG_ERR_FLOAT_UNDERFLOW: return "value out of range: underflow";
		case GG_ERR_DIV_ZERO: return "division by zero";
		case GG_ERR_INT_OVERFLOW: return "bigint out of range";
		case GG_ERR_UNSUPPORTED: return "plan not supported on the GPU path";
		case GG_ERR_VISIBILITY: return "tuple visibility needs clog/snapshot";
		case GG_ERR_NOMEM: return "out of memory";
		case GG_ERR_BADPAGE: return "corrupted page";
		case GG_ERR_ARG: return "bad argument";
		case GG_ERR_DATE_RANGE: return "date out of range for timestamp";
		case GG_ERR_PEER: return "another segment reported an error";
		case GG_ERR_RETRY_HOST: return "run the slice again with host-row Motions";
		case GG_ERR_WINDOW_ARG: return "invalid argument for a window function";
	}
	return "unknown error";
}

int gg_engine_create(int device, gg_engine **out)
{
	int ndev = 0;
	if (!out) return GG_ERR_ARG;
	*out = nullptr;
	cudaError_t e = cudaGetDeviceCount(&ndev);
	if (e != cudaSuccess || ndev == 0)
	{
		/* no CPU fallback: the product path fails loudly without a GPU */
		gg_set_error("no CUDA device available (%s): the GPU engine has no CPU fallback",
		             e != cudaSuccess ? cudaGetErrorString(e) : "device count 0");
		cudaGetLastError();
		return GG_ERR_CUDA;
	}
	if (device < 0 || device >= ndev) { gg_set_error("device %d out of range (%d devices)", device, ndev); return GG_ERR_ARG; }
	GG_CUDA(cudaSetDevice(device));
	gg_engine *eng = new gg_engine();
	eng->device = device;
	cudaDeviceProp prop;
	GG_CUDA(cudaGetDeviceProperties(&prop, device));
	eng->sm_count = prop.multiProcessorCount;
	eng->smem_optin = prop.sharedMemPerBlockOptin;
	GG_CUDA(cudaStreamCreateWithFlags(&eng->stream, cudaStreamNonBlocking));
	GG_CUDA(cudaStreamCreateWithFlags(&eng->copy_stream, cudaStreamNonBlocking));
	GG_CUDA(cudaEventCreate(&eng->ev_start));
	GG_CUDA(cudaEventCreate(&eng->ev_stop));
	*out = eng;
	return GG_OK;
}

void gg_engine_free(gg_engine *e)
{
	if (!e) return;
	cudaSetDevice(e->device);
	cudaStreamSynchronize(e->stream);
	cudaStreamSynchronize(e->copy_stream);
	cudaFree(e->sort_scratch);
	cudaFree(e->motion_state);
	cudaFree(e->snapshot_buf);
	for (void *m : e->groups_pool) cudaFree(m);
	cudaFreeHost(e->groups_mirror);
	cudaEventDestroy(e->ev_start);
	cudaEventDestroy(e->ev_stop);
	cudaStreamDestroy(e->stream);
	cudaStreamDestroy(e->copy_stream);
	delete e;
}

/* heap_beginscan's snapshot argument (heapam.c:1573) for every scan this engine launches from now on */
int gg_engine_set_snapshot(gg_engine *e, const gg_snapshot *snap)
{
	if (!e) return GG_ERR_ARG;
	if (!snap) { e->d_snapshot = nullptr; return GG_OK; }
	if (snap->xcnt > GG_SNAPSHOT_MAX_XIP || (snap->xcnt && !snap->xip) || (snap->clog_n && !snap->clog) || (snap->clog_base & 3))
	{ gg_set_error("snapshot: %u xids in progress (at most %d), status range must start at a multiple of 4", snap->xcnt, GG_SNAPSHOT_MAX_XIP); return GG_ERR_ARG; }
	if (snap->suboverflowed || snap->takenDuringRecovery || snap->haveDistribSnapshot)
	{ gg_set_error("snapshot: subtransaction overflow, recovery and distributed snapshots are decided by the CPU scan"); return GG_ERR_UNSUPPORTED; }
	const size_t clog_bytes = ((size_t) snap->clog_n + 3) / 4;
	const size_t bytes = (8 + (size_t) snap->xcnt) * 4 + clog_bytes;
	GG_CUDA(cudaSetDevice(e->device));
	if (e->snapshot_cap < bytes)
	{
		GG_CUDA(cudaStreamSynchronize(e->stream));
		cudaFree(e->snapshot_buf);
		e->snapshot_buf = nullptr; e->snapshot_cap = 0;
		GG_CUDA(cudaMalloc((void **) &e->snapshot_buf, (bytes + 4095) & ~(size_t) 4095));
		e->snapshot_cap = (bytes + 4095) & ~(size_t) 4095;
	}
	std::vector<uint8_t> h(bytes);
	uint32_t *w = (uint32_t *) h.data();
	w[0] = snap->xmin; w[1] = snap->xmax; w[2] = snap->xcnt; w[3] = snap->curcid; w[4] = snap->own_xid;
	w[5] = snap->clog_base; w[6] = snap->clog_n; w[7] = 0;
	if (snap->xcnt) memcpy(w + 8, snap->xip, (size_t) snap->xcnt * 4);
	if (clog_bytes) memcpy(h.data() + (8 + (size_t) snap->xcnt) * 4, snap->clog, clog_bytes);
	GG_CUDA(cudaMemcpyAsync(e->snapshot_buf, h.data(), bytes, cudaMemcpyHostToDevice, e->stream));
	GG_CUDA(cudaStreamSynchronize(e->stream));        /* h is pageable and goes out of scope */
	e->d_snapshot = e->snapshot_buf;
	return GG_OK;
}

int gg_engine_sm_count(gg_engine *e) { return e ? e->sm_count : 0; }

int gg_engine_sync(gg_engine *e)
{
	if (!e) return GG_ERR_ARG;
	GG_CUDA(cudaSetDevice(e->device));
	GG_CUDA(cudaStreamSynchronize(e->copy_stream));
	GG_CUDA(cudaStreamSynchronize(e->stream));
	return GG_OK;
}

int gg_engine_last_kernel_ms(gg_engine *e, float *ms)
{
	if (!e || !ms) return GG_ERR_ARG;
	if (!e->timed) { *ms = 0; return GG_OK; }
	GG_CUDA(cudaEventSynchronize(e->ev_stop));
	GG_CUDA(cudaEventElapsedTime(ms, e->ev_start, e->ev_stop));
	return GG_OK;
}

uint64_t gg_engine_launch_count(gg_engine *e) { return e ? e->launches : 0; }

int gg_engine_timer_start(gg_engine *e)
{
	if (!e) return GG_ERR_ARG;
	GG_CUDA(cudaSetDevice(e->device));
	if (!e->ev_t0) { GG_CUDA(cudaEventCreate(&e->ev_t0)); GG_CUDA(cudaEventCreate(&e->ev_t1)); }
	/* the copy stream may hold the first work of the timed region: make the start event cover it */
	GG_CUDA(cudaEventRecord(e->ev_t0, e->stream));
	GG_CUDA(cudaStreamWaitEvent(e->copy_stream, e->ev_t0, 0));
	return GG_OK;
}

int gg_engine_timer_stop(gg_engine *e, float *ms)
{
	if (!e || !ms || !e->ev_t0) return GG_ERR_ARG;
	GG_CUDA(cudaSetDevice(e->device));
	GG_CUDA(cudaEventRecord(e->ev_t1, e->stream));
	GG_CUDA(cudaEventSynchronize(e->ev_t1));
	GG_CUDA(cudaEventElapsedTime(ms, e->ev_t0, e->ev_t1));
	return GG_OK;
}

void *gg_engine_stream(gg_engine *e) { return e ? (void *) e->stream : nullptr; }

int gg_relation_create(gg_engine *e, uint64_t nblocks, gg_relation **out)
{
	if (!e || !out) return GG_ERR_ARG;
	GG_CUDA(cudaSetDevice(e->device));
	gg_relation *r = new gg_relation();
	r->eng = e;
	r->nblocks = nblocks;
	r->owned = true;
	cudaError_t err = cudaMalloc((void **) &r->pages, (size_t) (nblocks ? nblocks : 1) * GG_BLCKSZ);
	if (err != cudaSuccess) { delete r; return gg_cuda_fail(err, "cudaMalloc(relation)"); }
	*out = r;
	return GG_OK;
}

int gg_relation_attach(gg_engine *e, void *device_pages, uint64_t nblocks, gg_relation **out)
{
	if (!e || !out || (!device_pages && nblocks)) return GG_ERR_ARG;
	if (((uintptr_t) device_pages) & 15) { gg_set_error("relation base must be 16-byte aligned for TMA"); return GG_ERR_ARG; }
	gg_relation *r = new gg_relation();
	r->eng = e;
	r->pages = (uint8_t *) device_pages;
	r->nblocks = nblocks;
	r->owned = false;
	*out = r;
	return GG_OK;
}

/* rows a receiving Motion delivered (GG_FMT_DATUMROWS, gg_plan.h): scanned in 32 KB chunks of whole rows.
 * The buffer must extend at least 16 bytes past the last row (bulk copies move multiples of 16 bytes). */
int gg_relation_attach_rows(gg_engine *e, void *device_rows, uint64_t nrows, int ncols, gg_relation **out)
{
	if (!e || !out || (!device_rows && nrows) || ncols < 1 || ncols > GG_MAX_ATTS) return GG_ERR_ARG;
	if (((uintptr_t) device_rows) & 15) { gg_set_error("row buffer must be 16-byte aligned for TMA"); return GG_ERR_ARG; }
	gg_relation *r = new gg_relation();
	const uint64_t per_chunk = (GG_BLCKSZ / (8ull * (1 + ncols))) & ~1ull;
	r->eng = e;
	r->pages = (uint8_t *) device_rows;
	r->rowwords = 1 + ncols;
	r->nrows = nrows;
	r->nblocks = (nrows + per_chunk - 1) / per_chunk;
	r->owned = false;
	*out = r;
	return GG_OK;
}

int gg_relation_load(gg_relation *r, uint64_t first_block, const void *host_pages, uint64_t nblocks)
{
	if (!r || nblocks > r->nblocks || first_block > r->nblocks - nblocks) return GG_ERR_ARG;
	GG_CUDA(cudaSetDevice(r->eng->device));
	GG_CUDA(cudaMemcpyAsync(r->pages + first_block * GG_BLCKSZ, host_pages, (size_t) nblocks * GG_BLCKSZ,
	                        cudaMemcpyHostToDevice, r->eng->stream));
	return GG_OK;
}

int gg_relation_read(gg_relation *r, uint64_t first_block, void *host_pages, uint64_t nblocks)
{
	if (!r || nblocks > r->nblocks || first_block > r->nblocks - nblocks) return GG_ERR_ARG;
	GG_CUDA(cudaSetDevice(r->eng->device));
	GG_CUDA(cudaMemcpyAsync(host_pages, r->pages + first_block * GG_BLCKSZ, (size_t) nblocks * GG_BLCKSZ,
	                        cudaMemcpyDeviceToHost, r->eng->stream));
	GG_CUDA(cudaStreamSynchronize(r->eng->stream));
	return GG_OK;
}

int gg_relation_copy(gg_relation *dst, uint64_t dst_first, gg_relation *src, uint64_t src_first, uint64_t nblocks)
{
	if (!dst || !src || nblocks > dst->nblocks || dst_first > dst->nblocks - nblocks || nblocks > src->nblocks || src_first > src->nblocks - nblocks)
		return GG_ERR_ARG;
	GG_CUDA(cudaSetDevice(dst->eng->device));
	GG_CUDA(cudaMemcpyAsync(dst->pages + dst_first * GG_BLCKSZ, src->pages + src_first * GG_BLCKSZ, (size_t) nblocks * GG_BLCKSZ,
	                        cudaMemcpyDeviceToDevice, dst->eng->stream));
	return GG_OK;
}

uint64_t gg_relation_nblocks(gg_relation *r) { return r ? r->nblocks : 0; }
void *gg_relation_device_ptr(gg_relation *r) { return r ? r->pages : nullptr; }

void gg_relation_free(gg_relation *r)
{
	if (!r) return;
	if (r->owned && r->pages) { cudaSetDevice(r->eng->device); cudaFree(r->pages); }
	delete r;
}

int gg_host_alloc(uint64_t bytes, void **out)
{
	if (!out) return GG_ERR_ARG;
	GG_CUDA(cudaHostAlloc(out, (size_t) bytes, cudaHostAllocDefault));
	return GG_OK;
}

void gg_host_free(void *p) { if (p) cudaFreeHost(p); }

}  /* extern "C" */

/* debugging aid: compile a SeqScan->Agg plan and list the accumulator-machine program (no GPU needed) */
extern "C" int gg_debug_disasm_scanagg(const gg_scan *scan, const gg_agg *agg, const gg_exprpool *pool, char *buf, int cap)
{
	ggp_program prog;
	ggp_aggmap aggmap[GG_MAX_AGGS];
	char msg[256];
	int rc = ggp_compile_scanagg(scan, agg, pool, &prog, aggmap, msg, sizeof msg);
	if (rc != GG_OK) { gg_set_error("%s", msg); return rc; }
	return ggp_disasm(&prog, buf, cap);
}

/* the compiled device program of a SeqScan->Agg plan, byte for byte (scripts/gen_plan_cache.py stores it next to each
 * build-time specialised kernel so that a lookup compares programs, not just their hashes) */
extern "C" int gg_debug_program_bytes(const gg_scan *scan, const gg_agg *agg, const gg_exprpool *pool, unsigned char *buf, int cap)
{
	ggp_program prog;
	ggp_aggmap aggmap[GG_MAX_AGGS];
	char msg[256];
	int rc = ggp_compile_scanagg(scan, agg, pool, &prog, aggmap, msg, sizeof msg);
	if (rc != GG_OK) { gg_set_error("%s", msg); return rc; }
	if (cap < (int) sizeof prog) return GG_ERR_NOMEM;
	memcpy(buf, &prog, sizeof prog);
	return (int) sizeof prog;
}

/* debugging aid: the build and probe programs of a HashJoin -> Agg plan */
extern "C" int gg_debug_disasm_join(const gg_scan *outer, const gg_scan *inner, const gg_hashjoin *hj, const gg_agg *agg,
                                    const gg_exprpool *pool, char *buf, int cap)
{
	std::vector<ggp_joinprog> jpbuf(1);     /* ~7 KB: kept off the stack */
	ggp_joinprog &jp = jpbuf[0];
	ggp_aggmap aggmap[GG_MAX_AGGS];
	char msg[256];
	int rc = ggp_compile_join(outer, inner, hj, agg, pool, &jp, aggmap, msg, sizeof msg);
	if (rc != GG_OK) { gg_set_error("%s", msg); return rc; }
	int n = snprintf(buf, (size_t) cap, "-- build (payload %d)\n", jp.npayload);
	n += ggp_disasm(&jp.build, buf + n, cap - n);
	n += snprintf(buf + n, (size_t) (cap - n), "-- probe (per-match segment from pc %d)\n", jp.probe_pc);
	n += ggp_disasm(&jp.probe, buf + n, cap - n);
	return n;
}

/* debugging aid: the build and probe programs of a HashJoin with a target list */
extern "C" int gg_debug_disasm_joinrows(const gg_scan *outer, const gg_scan *inner, const gg_hashjoin *hj, const int32_t *targets,
                                        int ntargets, const gg_exprpool *pool, char *buf, int cap)
{
	std::vector<ggp_joinprog> jpbuf(1);
	ggp_joinprog &jp = jpbuf[0];
	char msg[256];
	int rc = ggp_compile_joinrows(outer, inner, hj, targets, ntargets, pool, &jp, msg, sizeof msg);
	if (rc != GG_OK) { gg_set_error("%s", msg); return rc; }
	int n = snprintf(buf, (size_t) cap, "-- build (payload %d)\n", jp.npayload);
	n += ggp_disasm(&jp.build, buf + n, cap - n);
	n += snprintf(buf + n, (size_t) (cap - n), "-- probe (per-match segment from pc %d)\n", jp.probe_pc);
	n += ggp_disasm(&jp.probe, buf + n, cap - n);
	return n;
}

/* debugging aid: the plan-specialised source gg_jit.cpp would compile for this plan and kernel variant */
#include "gg_jit.h"
extern "C" int gg_debug_jit_source(const gg_scan *scan, const gg_agg *agg, const gg_exprpool *pool, int mode, int threads,
                                   const char *suffix, unsigned long long *hash, char *buf, int cap, int regslots_or_rule)
{
	ggp_program prog;
	ggp_aggmap aggmap[GG_MAX_AGGS];
	char msg[256];
	int rc = ggp_compile_scanagg(scan, agg, pool, &prog, aggmap, msg, sizeof msg);
	if (rc != GG_OK) { gg_set_error("%s", msg); return rc; }
	const int regslots = regslots_or_rule >= 0 ? regslots_or_rule : gg_priv_regslots(&prog, mode, agg->numGroups, -1);
	std::string s = gg_jit_scanagg_source(&prog, mode, threads, suffix, -1, regslots);
	if (hash) *hash = gg_plan_hash(&prog, mode) ^ (0x9E3779B97F4A7C15ULL * (uint64_t) regslots);
	snprintf(buf, (size_t) cap, "%s", s.c_str());
	return (int) s.size();
}

/* debugging aid: the plan-specialised sources of a join pipeline (which: 0 build kernel, 1 probe kernel) */
extern "C" int gg_debug_jit_source_join(const gg_scan *outer, const gg_scan *inner, const gg_hashjoin *hj, const gg_agg *agg,
                                        const gg_exprpool *pool, int which, int mode, char *buf, int cap)
{
	std::vector<ggp_joinprog> jpbuf(1);     /* ~7 KB: kept off the stack */
	ggp_joinprog &jp = jpbuf[0];
	ggp_aggmap aggmap[GG_MAX_AGGS];
	char msg[256];
	int rc = ggp_compile_join(outer, inner, hj, agg, pool, &jp, aggmap, msg, sizeof msg);
	if (rc != GG_OK) { gg_set_error("%s", msg); return rc; }
	std::string s = which == 0 ? gg_jit_scanagg_source(&jp.build, 3 /* MODE_BUILD */, 256, "_dbg")
	                           : gg_jit_scanagg_source(&jp.probe, mode, 256, "_dbg", jp.probe_pc);
	snprintf(buf, (size_t) cap, "%s", s.c_str());
	return (int) s.size();
}

