/*
 * gg_pipeline.h — the host object behind gg_scanagg (and, as its probe side, gg_joinagg): shared by gg_scanagg.cu and
 * gg_join.cu.
 */
#pragma once
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <vector>
#include "gg_scanagg_kernel.cuh"
#include "gg_engine.h"
#include "gg_jit.h"
#include "gg_launch.h"

#define GG_MERGE_CAP 1024          /* merged groups the fast path holds per segment */
#define GG_STREAM_CHUNK_BLOCKS 8192 /* 256 MB staging chunks for gg_scanagg_run_host */

struct gg_scanagg {
	gg_engine *eng = nullptr;
	gg_scan scan;
	gg_agg agg;
	gg_exprpool pool;
	ggp_program prog;
	ggp_aggmap aggmap[GG_MAX_AGGS];
	int mode = ggd::MODE_PRIV;           /* kernel variant; escalates PRIV -> TR when a run overflows its group capacity */
	gg_launch cfg;                       /* launch shape of the current variant */
	int grid = 0;
	std::vector<std::pair<cudaEvent_t, cudaEvent_t>> kev;   /* events around every scan kernel launch since reset */
	size_t kev_used = 0;
	const void *kernel = nullptr;   /* the kernel of the current variant: jit's, or the interpreter instance of the role */
	gg_jit_kernel *jit = nullptr;   /* plan-specialised kernel for the current variant, or nullptr: interpreter */
	gg_jit_kernel *jit_snap = nullptr;  /* the same with the snapshot rule built in (gg_jit.h mvcc), or `jit` when there is none;
	                                     * chosen when a launch first finds the engine holding a snapshot, reset by every
	                                     * reconfiguration */
	int chunks_per_page = 0;        /* 32-row chunks per page of the relation being scanned (0: not sampled yet) */
	int items_per_page = 0;         /* line pointers of the sampled page */
	bool is_join = false;           /* probe side of a gg_joinagg: prog = the probe program, jt = the built table */
	bool join_rows = false;         /* probe of a join with a target list: MODE_PART, every joined row written through `mo` */
	ggd::MotionOut mo = {};         /* join_rows: the output rows (one destination) and their cursor */
	ggd::HashAggTable ha = {};           /* MODE_HASH: the group table in HBM */
	void *ha_mem = nullptr;
	uint64_t ha_cap = 0;
	unsigned long long *d_nout64 = nullptr;
	ggd::JoinTable jt = {};
	int join_probe_pc = -1;
	uint32_t build_err = 0;         /* error flags the join's build kernel raised for the table `jt`: fetch reports them, and
	                                 * neither a replay nor a reset of the probe side clears them (the table stays as built) */
	/* device state */
	ggp_grec *recs = nullptr;       /* [GG_MERGE_CAP (previous merged)] ++ [grid * GGP_FAST_GROUPS (block records)] */
	ggp_grec *merged = nullptr;     /* [GG_MERGE_CAP] output of the merge kernel */
	int *vidx = nullptr, *vmap = nullptr;
	/* status words of the pipeline: one device block, mirrored into pinned host memory by ONE copy per fetch
	 * (together with the first merged group records) */
	struct Status { uint32_t err; int nout; unsigned long long counters[2]; };
	Status *d_status = nullptr;
	int *d_nout = nullptr;                  /* = &d_status->nout */
	uint32_t *d_err = nullptr;              /* = &d_status->err */
	unsigned long long *d_counters = nullptr;   /* = d_status->counters */
	struct HostMirror { Status st; ggp_grec recs[GGP_FAST_GROUPS]; };
	HostMirror *h_mirror = nullptr;         /* pinned */
	int nrecs_total = 0, nrecs_cap = 0;
	/* inputs of the current accumulation, kept so that a group-capacity overflow can be replayed on a wider variant */
	struct Fed { const uint8_t *dev; const void *host; uint64_t nblocks; uint64_t nrows; bool fill; int32_t tile_rows; };   /* tile_rows > 0: dev = the column descriptors of an AOCS feed */
	gg_aocs_devcol *d_aocs = nullptr;       /* device copy of the column descriptors of gg_scanagg_run_aocs */
	int32_t aocs_unit_rows = 0;             /* rows of every projected column staged per ring slot (set by gg_scanagg_run_aocs) */
	std::vector<Fed> fed;
	bool has_state = false;
	/* set by a batched join: how to feed the inputs again (its batches, each with its own hash table) when fetch has to
	 * replay them on a wider kernel variant; empty: replay `fed` */
	std::function<int()> replay_hook;
	/* host staging for the streamed path */
	uint8_t *stage[2] = { nullptr, nullptr };
	cudaEvent_t ev_copied[2] = { nullptr, nullptr }, ev_consumed[2] = { nullptr, nullptr };
};

/* gg_scanagg.cu */
int scanagg_finish_create(gg_scanagg *p, gg_scanagg **out);      /* after p->prog / p->aggmap are compiled */
/* one launch of the pipeline's kernel over device pages (fill_inner: the HJ_FILL_INNER_TUPLES pass of a right/full join) */
int scanagg_launch(gg_scanagg *p, const uint8_t *dev_pages, uint64_t nblocks, cudaStream_t st, uint64_t nrows = 0, bool fill_inner = false, int32_t aocs_tile_rows = 0);
/* reset the pipeline and feed its inputs again (through replay_hook when set) on kernel variant `mode` (MODE_HASH: a group
 * table of ha_cap slots) */
extern "C" int scanagg_replay(gg_scanagg *p, int mode, uint64_t ha_cap);
/* gg_motion.cu: the partitioning kernel behind gg_motion_partition, with the routing rule as a parameter (route 0: segments by
 * cdbhash + jump consistent hash; route 1: hash-join batches by the batch bits above `shift`) */
int gg_partition_rows(gg_engine *e, const gg_scan *scan, const gg_exprpool *pool,
                      const int32_t *hashkeys, int nkeys, const int32_t *payload, int npayload,
                      int nsegs, int route, int shift, gg_relation *r, uint64_t first_block, uint64_t nblocks,
                      void *device_out_rows, uint64_t out_cap_rows,
                      uint64_t *host_counts, uint64_t *host_offsets);
/* The kernel that runs the scan kernel body in role `mode` (probe_pc >= 0: the probe side of a join) with launch shape `c`: the
 * plan-specialised kernel (gg_jit_scanagg: build-time plan cache or NVRTC; mvcc: with the snapshot rule) when there is one, else
 * the interpreter instance of the role, made ready for c.smem bytes of dynamic shared memory.  Launch it with
 * cudaLaunchKernel(*fn, grid, c.threads, { &prog, &params }, c.smem).  *jit (optional): the specialised kernel, or nullptr. */
int gg_scan_kernel(const ggp_program *prog, int mode, int probe_pc, const gg_launch &c, int device, bool mvcc, const void **fn, gg_jit_kernel **jit = nullptr);

/* the interpreter instances of the join and Motion roles (gg_join.cu, gg_motion.cu), for gg_scan_kernel's table */
__global__ void gg_joinhash_kernel(const __grid_constant__ ggp_program P, const ggd::ScanAggParams prm);
__global__ void gg_joinbuild_kernel(const __grid_constant__ ggp_program P, const ggd::ScanAggParams prm);
__global__ void gg_motion_part_kernel(const __grid_constant__ ggp_program P, const ggd::ScanAggParams prm);
__global__ void gg_joinrows_kernel(const __grid_constant__ ggp_program P, const ggd::ScanAggParams prm);
