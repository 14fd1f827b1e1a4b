/*
 * gg_engine.h — host-side objects behind the opaque handles of include/ggb200.h.
 */
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>
#include <vector>
#include "gg_program.h"
#include "../../include/ggb200.h"

struct gg_engine {
	int device = 0;
	int sm_count = 0;
	size_t smem_optin = 0;
	cudaStream_t stream = nullptr;       /* compute */
	cudaStream_t copy_stream = nullptr;  /* H2D staging */
	cudaEvent_t ev_start = nullptr, ev_stop = nullptr;
	cudaEvent_t ev_t0 = nullptr, ev_t1 = nullptr;      /* gg_engine_timer_start/stop */
	bool timed = false;
	uint64_t launches = 0;
	void *sort_scratch = nullptr;        /* gg_sort_*: key/value ping-pong buffers, histograms; kept across calls */
	size_t sort_scratch_bytes = 0;
	std::vector<void *> groups_pool;     /* gg_groups buffers of the common size, recycled (gg_scanagg.cu) */
	void *groups_mirror = nullptr;       /* pinned: status + records of one gg_groups_fetch */
	uint32_t *d_snapshot = nullptr;      /* gg_engine_set_snapshot: the snapshot every scan launched from now on decides visibility with */
	uint32_t *snapshot_buf = nullptr;    /* the allocation d_snapshot points into when a snapshot is set */
	size_t snapshot_cap = 0;             /* its size in bytes */
	void *motion_state = nullptr;        /* gg_motion_partition: region cursors, error flags, counters (device) */
};

struct gg_relation {
	gg_engine *eng = nullptr;
	uint8_t *pages = nullptr;
	uint64_t nblocks = 0;            /* heap: pages; datum rows: 32 KB chunks of whole rows */
	int rowwords = 0;                /* 0: heap pages; else GG_FMT_DATUMROWS with this many 64-bit words per row */
	uint64_t nrows = 0;              /* datum rows only */
	bool owned = false;
};

void gg_set_error(const char *fmt, ...);
int  gg_cuda_fail(cudaError_t e, const char *what);
int  gg_errflags_to_code(uint32_t flags);

#define GG_CUDA(call) do { cudaError_t _e = (call); if (_e != cudaSuccess) return gg_cuda_fail(_e, #call); } while (0)
