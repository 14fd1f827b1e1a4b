/*
 * gg_interconnect.cu — the Motion layer of the GPU segment engine in C over NCCL (include/ggb200.h gg_ic_*).
 *
 * Replaces, for GPU segments, the UDP interconnect under ExecMotion:
 *     SetupInterconnect / TeardownInterconnect            cdb/motion/ic_common.c:522,560
 *     ChunkTransportState vtable (SendChunk, RecvTupleChunkFrom[Any], doSendStopMessage, SendEos)
 *                                                          cdb/cdbinterconnect.h:500-533
 *     SendTuple / RecvTupleFrom / SendEndOfStream          cdb/motion/cdbmotion.c:434,559,532
 *     ic_udpifc.c (reliable datagram streams, acks, retransmission)   — nothing of it remains
 * One communicator per query, NCCL rank = contentid (segment), peers over NVLink / NVSwitch.  What moves is not tuple
 * chunks but whole device-resident batches:
 *     group records   the handful of partial-aggregate states a slice emits (ggp_grec): ONE all-gather of fixed-size
 *                     blocks; every receiver keeps the records cdbhash routes to it (Redistribute), the root keeps all
 *                     (Gather), everybody keeps all (Broadcast).  Every block carries its sender's status word, so an
 *                     ERROR on one segment reaches all of them with the data — the reference's error / stop propagation
 *                     (cdbmotion.c:342 SendStopMessage, ic_udpifc.c:5798) — and no rank can be left waiting in a
 *                     collective another rank never enters.
 *     datum rows      what gg_motion_partition wrote per destination: a count exchange (all-gather of the counts) and
 *                     grouped ncclSend / ncclRecv straight out of the sender's regions into the receiver's row buffer.
 *     host rows       the executor's generic row batches (GgRowBatch), staged through device buffers.
 * End of stream is the completion of the collective.  NCCL is dlopen'ed (libnccl.so.2): no link-time dependency.
 */
#include <dlfcn.h>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <chrono>
#include <condition_variable>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>
#include "gg_pipeline.h"
#include "gg_groups.h"

using namespace ggd;

/* ---------------- NCCL through dlopen ---------------- */
namespace {

typedef struct ncclComm *ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
enum { ncclSuccess_ = 0, ncclInProgress_ = 7 };
enum { ncclUint8_ = 1, ncclUint64_ = 5 };

struct Nccl {
	void *h = nullptr;
	int (*GetVersion)(int *) = nullptr;
	int (*GetUniqueId)(ncclUniqueId *) = nullptr;
	int (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
	int (*CommDestroy)(ncclComm_t) = nullptr;
	int (*CommAbort)(ncclComm_t) = nullptr;
	const char *(*GetErrorString)(int) = nullptr;
	int (*AllGather)(const void *, void *, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
	int (*Send)(const void *, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
	int (*Recv)(void *, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
	int (*GroupStart)(void) = nullptr;
	int (*GroupEnd)(void) = nullptr;
	bool ok = false;
	char why[256] = "";
};

Nccl &nccl()
{
	static Nccl n;
	static std::once_flag once;
	std::call_once(once, [] {
		const char *env = getenv("GGB200_NCCL_LIB");
		const char *names[] = { env, "libnccl.so.2", "libnccl.so", "/usr/lib/x86_64-linux-gnu/libnccl.so.2" };
		for (const char *nm : names)
			if (nm && nm[0] && (n.h = dlopen(nm, RTLD_NOW | RTLD_GLOBAL)) != nullptr) break;
		if (!n.h) { snprintf(n.why, sizeof n.why, "libnccl.so.2 not found (%s)", dlerror()); return; }
#define LOADSYM(F) *(void **) (&n.F) = dlsym(n.h, "nccl" #F); if (!n.F) { snprintf(n.why, sizeof n.why, "nccl" #F " missing"); return; }
		LOADSYM(GetVersion) LOADSYM(GetUniqueId) LOADSYM(CommInitRank) LOADSYM(CommDestroy) LOADSYM(CommAbort)
		LOADSYM(GetErrorString) LOADSYM(AllGather) LOADSYM(Send) LOADSYM(Recv) LOADSYM(GroupStart) LOADSYM(GroupEnd)
#undef LOADSYM
		n.ok = true;
	});
	return n;
}

int nccl_fail(int rc, const char *what)
{
	gg_set_error("NCCL error %d (%s) in %s", rc, nccl().GetErrorString ? nccl().GetErrorString(rc) : "?", what);
	return GG_ERR_CUDA;
}
#define GG_NCCL(call) do { int _r = (call); if (_r != ncclSuccess_) return nccl_fail(_r, #call); } while (0)

}  // namespace

/* what one segment contributes to a Motion of group records */
struct GroupBlock {
	uint32_t n;                 /* records this segment sends (may exceed GG_IC_GROUP_CAP: then none travel and every receiver sees it) */
	uint32_t err;               /* GGP_EF_* of the sending pipeline */
	unsigned long long counters[2];
	ggp_grec recs[GG_IC_GROUP_CAP];
};

struct gg_interconnect {
	gg_engine *eng = nullptr;
	ncclComm_t comm = nullptr;       /* nullptr: one segment, loopback */
	int nsegs = 1, seg = 0;
	GroupBlock *d_send = nullptr;    /* [1] */
	GroupBlock *d_all = nullptr;     /* [nsegs] */
	unsigned long long *d_counts = nullptr;   /* [nsegs] mine, [nsegs * nsegs] everybody's; then the words of gg_ic_allgather_u64: [1] mine, [nsegs] everybody's */
	unsigned long long *h_counts = nullptr;   /* pinned mirror of the matrix [nsegs * nsegs], then of gg_ic_allgather_u64's words [nsegs] */
	void *stage = nullptr;           /* host-row exchange: device staging, grown on demand */
	size_t stage_bytes = 0;
	uint64_t ncollectives = 0;
	/* Row exchanges (Redistribute Motion) are personalised: every segment sends a different run of rows to every other.
	 * Grouped ncclSend / ncclRecv do that (`p2p` = the communicator they run on: `comm`, or with GGB200_IC_ROWS=auto one of
	 * their own, proven by a tiny all-pairs exchange when rows first travel — point-to-point connections are set up on first use,
	 * and a segment where that fails leaves the others waiting); p2p_ok == false: rows move with ncclAllGather over `comm`
	 * instead, N times the traffic, the collective every Motion of group records already uses (ic_decide_row_transport). */
	ncclComm_t p2p = nullptr;
	bool p2p_ok = false;
	bool rows_decided = false;       /* the proof has run (it runs when rows first travel: a Motion of rows is collective, so every
	                                  * segment is at the same point; plans that only move group records never pay for it) */
	uint8_t *ag_buf = nullptr;       /* all-gather path: [nsegs] packed regions to send ++ [nsegs * nsegs] regions received */
	size_t ag_bytes = 0;
};

/* ---------------- kernels ---------------- */

/* pipeline result -> the block that travels */
__global__ void gg_ic_pack_groups_kernel(const ggp_grec *recs, const int *d_n, const gg_groupstatus *st, int sparse, int cap,
                                         uint32_t local_flags, GroupBlock *dst)
{
	__shared__ int s_n;
	if (threadIdx.x == 0)
	{
		int n = 0;
		if (!recs) n = 0;                                   /* nothing to send: the status is the message */
		else if (sparse) { for (int i = 0; i < cap; i++) n += recs[i].valid ? 1 : 0; }
		else n = *d_n;
		/* more records than a block carries: none travel, and everybody learns that this Motion has to take the host path */
		const bool over = n > GG_IC_GROUP_CAP;
		s_n = over ? GG_IC_GROUP_CAP + 1 : n;
		dst->n = over ? 0u : (uint32_t) n;
		/* a pipeline whose result was not fetched before it travelled (the executor leaves that to the top of the slice) may
		 * carry "replay me on a wider kernel variant": only a fetch on the producing segment can do that, so it becomes
		 * "this Motion takes the host path" for everybody */
		uint32_t perr = st ? st->err : 0u;
		const bool replay = (perr & (GGP_EF_GROUP_OVERFLOW | GGP_EF_RECHECK)) != 0;
		perr &= ~(uint32_t) (GGP_EF_GROUP_OVERFLOW | GGP_EF_RECHECK);
		dst->err = perr | local_flags | ((over || replay) ? GGP_EF_HOSTPATH : 0u);
		dst->counters[0] = st ? st->counters[0] : 0ull;
		dst->counters[1] = st ? st->counters[1] : 0ull;
	}
	__syncthreads();
	if (!recs || s_n > GG_IC_GROUP_CAP) return;
	/* copy word-wise; a sparse source is compacted in slot order (deterministic) */
	const int W = (int) (sizeof(ggp_grec) / 8);
	if (!sparse)
	{
		for (int i = threadIdx.x; i < s_n * W; i += blockDim.x)
			((unsigned long long *) dst->recs)[i] = ((const unsigned long long *) recs)[i];
	}
	else if (threadIdx.x < 32)
	{
		int at = 0;
		for (int i = 0; i < cap; i++)
		{
			if (!recs[i].valid) continue;
			for (int w = threadIdx.x; w < W; w += 32)
				((unsigned long long *) &dst->recs[at])[w] = ((const unsigned long long *) &recs[i])[w];
			at++;
		}
	}
}

/* evalHashKey + cdbhash + cdbhashreduce over a group record's keys (nodeMotion.c:1481, cdbhash.c:191-287) */
__device__ __forceinline__ int route_group(const ggp_grec &r, int nhash, const int *hashcol, const int *hashtype, int nsegs)
{
	uint32_t h = 0;
	for (int k = 0; k < nhash; k++)
	{
		const int c = hashcol[k];
		const bool isnull = (r.keynull >> c) & 1;
		const uint64_t v = r.key[c];
		h = cdbhash_add(h, isnull ? 0 : key_hash(hashtype[k], v), isnull);
	}
	return jump_consistent_hash((uint64_t) h, nsegs);
}

struct RouteSpec { int nhash; int hashcol[GG_MAX_KEYS]; int hashtype[GG_MAX_KEYS]; };

/* receiving side: out = [nsegs][GG_IC_GROUP_CAP] records, valid where this segment keeps the record */
__global__ void gg_ic_route_groups_kernel(const GroupBlock *all, int nsegs, int myseg, int motion, int root, RouteSpec spec,
                                          ggp_grec *out, gg_groupstatus *st)
{
	const int W = (int) (sizeof(ggp_grec) / 8);
	if (threadIdx.x == 0)
	{
		/* every sender's ERROR flags reach every receiver; the row counters travel once: a Gather adds them up at the root,
		 * any other Motion passes this segment's own through */
		uint32_t e = 0;
		unsigned long long c0 = 0, c1 = 0;
		for (int r = 0; r < nsegs; r++)
		{
			e |= all[r].err;
			if (motion == GG_IC_MOTION_GATHER ? myseg == root : r == myseg) { c0 += all[r].counters[0]; c1 += all[r].counters[1]; }
		}
		st->err = e; st->counters[0] = c0; st->counters[1] = c1; st->n = 0;
	}
	for (int i = threadIdx.x; i < nsegs * GG_IC_GROUP_CAP; i += blockDim.x)
	{
		const int r = i / GG_IC_GROUP_CAP, j = i % GG_IC_GROUP_CAP;
		bool keep = (uint32_t) j < all[r].n && all[r].n <= GG_IC_GROUP_CAP;
		if (keep)
		{
			if (motion == GG_IC_MOTION_HASH) keep = route_group(all[r].recs[j], spec.nhash, spec.hashcol, spec.hashtype, nsegs) == myseg;
			else if (motion == GG_IC_MOTION_GATHER) keep = myseg == root;
		}
		if (keep)
		{
			for (int w = 0; w < W; w++) ((unsigned long long *) &out[i])[w] = ((const unsigned long long *) &all[r].recs[j])[w];
			out[i].valid = 1;
		}
		else
			out[i].valid = 0;
	}
}

/* host rows <-> packed records: [ncols datums][null bytes padded to 8] per row, grouped by destination */
static inline size_t hostrow_words(int ncols) { return (size_t) ncols + (size_t) ((ncols + 7) / 8); }

extern "C" {

int gg_ic_available(void)
{
	return nccl().ok ? 1 : 0;
}

int gg_ic_unique_id(void *out, int len)
{
	if (!out || len < GG_IC_UNIQUE_ID_BYTES) return GG_ERR_ARG;
	Nccl &n = nccl();
	if (!n.ok) { gg_set_error("NCCL not available: %s", n.why); return GG_ERR_UNSUPPORTED; }
	ncclUniqueId id;
	GG_NCCL(n.GetUniqueId(&id));
	memcpy(out, &id, sizeof id);
	return GG_OK;
}

/* GGB200_IC_TRACE=1: one line on stderr per collective entered / left, with the segment — what a stuck exchange looks like
 * from each side (debugging only; the lines are flushed at once) */
static bool ic_trace_on()
{
	static int on = -1;
	if (on < 0) { const char *t = getenv("GGB200_IC_TRACE"); on = t && atoi(t) != 0; }
	return on != 0;
}
#define IC_TRACE(ic, ...) do { if (ic_trace_on()) { fprintf(stderr, "[ic seg %d] ", (ic)->seg); fprintf(stderr, __VA_ARGS__); fputc('\n', stderr); fflush(stderr); } } while (0)

static int ic_allgather(gg_interconnect *ic, const void *send, void *recv, size_t bytes);

/* The proof that ncclSend / ncclRecv work among these segments, on a communicator of its own and in a thread of its own, so that
 * a segment where it never returns can give up on it (gg_interconnect::p2p). */
struct P2pPreflight {
	std::mutex mu;
	std::condition_variable cv;
	bool done = false;
	int rc = -1;
	ncclComm_t comm = nullptr;
	int device = 0, nsegs = 0, seg = 0;
	ncclUniqueId id;
};

static void ic_p2p_preflight(std::shared_ptr<P2pPreflight> pf)
{
	Nccl &n = nccl();
	int rc = cudaSetDevice(pf->device) == cudaSuccess ? 0 : 1000;
	ncclComm_t comm = nullptr;
	cudaStream_t st = nullptr;
	unsigned char *buf = nullptr;
	if (!rc) rc = n.CommInitRank(&comm, pf->nsegs, pf->id, pf->seg);
	{
		std::lock_guard<std::mutex> lk(pf->mu);
		pf->comm = comm;
	}
	if (!rc && cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) != cudaSuccess) rc = 1001;
	if (!rc && cudaMalloc((void **) &buf, (size_t) 2 * 64 * (size_t) pf->nsegs) != cudaSuccess) rc = 1002;
	if (!rc)
	{
		/* the shape of a row exchange: every segment to every segment, itself included, in one group */
		rc = n.GroupStart();
		for (int p = 0; p < pf->nsegs && !rc; p++)
		{
			rc = n.Send(buf + 64 * (size_t) p, 64, ncclUint8_, p, comm, st);
			if (!rc) rc = n.Recv(buf + 64 * (size_t) (pf->nsegs + p), 64, ncclUint8_, p, comm, st);
		}
		const int rc2 = n.GroupEnd();            /* always: an open group would swallow every later call of this thread */
		if (!rc) rc = rc2;
	}
	if (!rc && cudaStreamSynchronize(st) != cudaSuccess) rc = 1003;
	cudaFree(buf);
	if (st) cudaStreamDestroy(st);
	cudaGetLastError();
	std::lock_guard<std::mutex> lk(pf->mu);
	pf->rc = rc;
	pf->done = true;
	pf->cv.notify_all();
}

/* SetupInterconnect (ic_common.c:522): join the query's communicator as segment `segindex` of `nsegs` */
int gg_ic_create(gg_engine *e, const void *unique_id, int nsegs, int segindex, gg_interconnect **out)
{
	if (!e || !out || nsegs < 1 || segindex < 0 || segindex >= nsegs || (nsegs > 1 && !unique_id)) return GG_ERR_ARG;
	*out = nullptr;
	GG_CUDA(cudaSetDevice(e->device));
	gg_interconnect *ic = new gg_interconnect();
	ic->eng = e; ic->nsegs = nsegs; ic->seg = segindex;
	if (nsegs > 1)
	{
		Nccl &n = nccl();
		if (!n.ok) { gg_set_error("NCCL not available: %s", n.why); delete ic; return GG_ERR_UNSUPPORTED; }
		ncclUniqueId id;
		memcpy(&id, unique_id, sizeof id);
		int rc = n.CommInitRank(&ic->comm, nsegs, id, segindex);
		if (rc != ncclSuccess_) { delete ic; return nccl_fail(rc, "ncclCommInitRank"); }
	}
	cudaError_t ce = cudaMalloc((void **) &ic->d_send, sizeof(GroupBlock));
	if (ce == cudaSuccess) ce = cudaMalloc((void **) &ic->d_all, sizeof(GroupBlock) * (size_t) nsegs);
	if (ce == cudaSuccess) ce = cudaMalloc((void **) &ic->d_counts, 8 * (size_t) (nsegs + nsegs * nsegs + 2 + nsegs));
	if (ce == cudaSuccess) ce = cudaHostAlloc((void **) &ic->h_counts, 8 * (size_t) (nsegs * nsegs + nsegs), cudaHostAllocDefault);
	if (ce != cudaSuccess) { gg_ic_free(ic); return gg_cuda_fail(ce, "gg_ic_create"); }
	*out = ic;
	return GG_OK;
}

/* TeardownInterconnect (ic_common.c:560).  has_errors: the query is being aborted — do not wait for peers */
void gg_ic_teardown(gg_interconnect *ic, int has_errors)
{
	if (!ic) return;
	cudaSetDevice(ic->eng->device);
	if (ic->p2p && ic->p2p != ic->comm)
	{
		if (has_errors) nccl().CommAbort(ic->p2p);
		else { cudaStreamSynchronize(ic->eng->stream); nccl().CommDestroy(ic->p2p); }
	}
	ic->p2p = nullptr;
	if (ic->comm)
	{
		if (has_errors) nccl().CommAbort(ic->comm);
		else { cudaStreamSynchronize(ic->eng->stream); nccl().CommDestroy(ic->comm); }
		ic->comm = nullptr;
	}
	cudaFree(ic->d_send); cudaFree(ic->d_all); cudaFree(ic->d_counts); cudaFreeHost(ic->h_counts); cudaFree(ic->stage); cudaFree(ic->ag_buf);
	delete ic;
}

void gg_ic_free(gg_interconnect *ic) { gg_ic_teardown(ic, 0); }

int gg_ic_nsegs(gg_interconnect *ic) { return ic ? ic->nsegs : 0; }
int gg_ic_segindex(gg_interconnect *ic) { return ic ? ic->seg : -1; }
uint64_t gg_ic_collective_count(gg_interconnect *ic) { return ic ? ic->ncollectives : 0; }

/* all-gather of `bytes` per segment on the engine's stream (loopback: a copy) */
static int ic_allgather(gg_interconnect *ic, const void *send, void *recv, size_t bytes)
{
	cudaStream_t st = ic->eng->stream;
	if (!ic->comm)
	{
		GG_CUDA(cudaMemcpyAsync(recv, send, bytes, cudaMemcpyDeviceToDevice, st));
		return GG_OK;
	}
	IC_TRACE(ic, "allgather #%llu of %zu bytes", (unsigned long long) ic->ncollectives, bytes);
	GG_NCCL(nccl().AllGather(send, recv, bytes, ncclUint8_, ic->comm, st));
	ic->ncollectives++;
	return GG_OK;
}

/* A barrier that is also useful: every segment learns every segment's 64-bit word (bench: max-over-ranks timing) */
int gg_ic_allgather_u64(gg_interconnect *ic, uint64_t mine, uint64_t *all /* [nsegs] */)
{
	if (!ic || !all) return GG_ERR_ARG;
	GG_CUDA(cudaSetDevice(ic->eng->device));
	cudaStream_t st = ic->eng->stream;
	/* its own words behind the count matrix, on the device and in the pinned mirror: a row exchange calls this between building
	 * the matrix and using it (the overflow agreement).  It used to share the matrix's first row — and zeroed what segment 0
	 * sends to everybody, which left one segment's group invalid and the others waiting for it (profiles/r2j_p2p_stuck_trace.log) */
	const size_t N = (size_t) ic->nsegs;
	unsigned long long *d_mine = ic->d_counts + N + N * N, *d_all = d_mine + 2, *h_all = ic->h_counts + N * N;
	GG_CUDA(cudaMemcpyAsync(d_mine, &mine, 8, cudaMemcpyHostToDevice, st));
	int rc = ic_allgather(ic, d_mine, d_all, 8);
	if (rc) return rc;
	GG_CUDA(cudaMemcpyAsync(h_all, d_all, 8 * N, cudaMemcpyDeviceToHost, st));
	GG_CUDA(cudaStreamSynchronize(st));
	memcpy(all, h_all, 8 * N);
	IC_TRACE(ic, "allgather_u64 done (mine %llu)", (unsigned long long) mine);
	return GG_OK;
}

/* Decide, once and together, how rows travel (gg_interconnect::p2p).  GGB200_IC_ROWS (every segment must be given the same value):
 *   p2p (default)  grouped ncclSend / ncclRecv on `comm`
 *   auto           prove point-to-point first, on a communicator of its own (ic_p2p_preflight), agree on the outcome, and fall
 *                  back to all-gather where the proof failed or timed out on any segment — for installations where setting up
 *                  point-to-point connections is known to be fragile
 *   allgather      ncclAllGather of equal-stride parts, N times the traffic */
static int ic_decide_row_transport(gg_interconnect *ic)
{
	if (ic->rows_decided) return GG_OK;
	ic->rows_decided = true;
	gg_engine *e = ic->eng;
	const int nsegs = ic->nsegs, segindex = ic->seg;
	cudaError_t ce;
	const char *mode = getenv("GGB200_IC_ROWS");
	if (!mode || !mode[0] || !strcmp(mode, "p2p")) { ic->p2p = ic->comm; ic->p2p_ok = true; return GG_OK; }
	if (!strcmp(mode, "allgather")) { ic->p2p_ok = false; return GG_OK; }
	if (strcmp(mode, "auto")) { gg_set_error("GGB200_IC_ROWS must be p2p, auto or allgather"); return GG_ERR_ARG; }
	Nccl &n = nccl();
	cudaStream_t st = e->stream;
	auto pf = std::make_shared<P2pPreflight>();
	pf->device = e->device; pf->nsegs = nsegs; pf->seg = segindex;
	/* segment 0 makes the second communicator's id; it travels over the first */
	ncclUniqueId id2;
	memset(&id2, 0, sizeof id2);
	int rc = segindex == 0 ? n.GetUniqueId(&id2) : 0;
	if (rc != ncclSuccess_) return nccl_fail(rc, "ncclGetUniqueId");
	ce = cudaMemcpyAsync(ic->d_send, &id2, sizeof id2, cudaMemcpyHostToDevice, st);
	if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
	if (ce != cudaSuccess) return gg_cuda_fail(ce, "row transport proof");
	rc = ic_allgather(ic, ic->d_send, ic->d_all, sizeof(GroupBlock));
	if (rc) return rc;
	ce = cudaMemcpyAsync(&pf->id, ic->d_all, sizeof pf->id, cudaMemcpyDeviceToHost, st);      /* segment 0's block */
	if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
	if (ce != cudaSuccess) return gg_cuda_fail(ce, "row transport proof");
	int wait_s = 20;
	{ const char *t = getenv("GGB200_IC_P2P_TIMEOUT"); if (t && atoi(t) > 0) wait_s = atoi(t); }
	std::thread th(ic_p2p_preflight, pf);
	bool finished;
	{
		std::unique_lock<std::mutex> lk(pf->mu);
		finished = pf->cv.wait_for(lk, std::chrono::seconds(wait_s), [&] { return pf->done; });
	}
	const int mine = finished && pf->rc == 0;
	if (finished) th.join(); else th.detach();          /* a stuck proof is left behind; nothing else uses its communicator */
	IC_TRACE(ic, "point-to-point proof: %s (rc %d)", finished ? "finished" : "timed out", finished ? pf->rc : -1);
	uint64_t all[1024];
	if (nsegs > 1024) return GG_ERR_UNSUPPORTED;
	rc = gg_ic_allgather_u64(ic, (uint64_t) mine, all);
	if (rc) return rc;
	bool ok = true;
	for (int sidx = 0; sidx < nsegs; sidx++) ok = ok && all[sidx] != 0;
	if (ok) { ic->p2p = pf->comm; ic->p2p_ok = true; }
	else if (finished && pf->comm) n.CommAbort(pf->comm);       /* proven here, not everywhere: of no use */
	IC_TRACE(ic, "rows travel by %s", ok ? "ncclSend/ncclRecv" : "ncclAllGather");
	return GG_OK;
}

/* The personalised exchange behind every Motion of rows, on the engine's stream.  ic->h_counts holds the count matrix
 * (h_counts[s * N + d] = units segment s sends to segment d, already exchanged); this segment's part for d starts at
 * send_base + send_off[d] (bytes); what arrives is laid out at recv_base in sender order.  unit = bytes per counted unit.
 *   p2p_ok       grouped ncclSend / ncclRecv on the proven communicator: every byte travels once
 *   otherwise    ncclAllGather: every segment packs its N parts at a common stride (the largest entry of the matrix), all
 *                segments receive all parts and keep theirs — N times the traffic of the above, the price of not depending
 *                on point-to-point connections */
static int ic_alltoallv(gg_interconnect *ic, const uint8_t *send_base, const size_t *send_off, uint8_t *recv_base, size_t unit)
{
	gg_engine *e = ic->eng;
	cudaStream_t st = e->stream;
	const int N = ic->nsegs;
	Nccl &n = nccl();
	if (ic->p2p_ok)
	{
		int rc = n.GroupStart();
		size_t at = 0;
		for (int s = 0; s < N && rc == ncclSuccess_; s++)
		{
			const size_t sendb = (size_t) ic->h_counts[(size_t) ic->seg * N + s] * unit, recvb = (size_t) ic->h_counts[(size_t) s * N + ic->seg] * unit;
			if (sendb) rc = n.Send(send_base + send_off[s], sendb, ncclUint8_, s, ic->p2p, st);
			if (recvb && rc == ncclSuccess_) rc = n.Recv(recv_base + at, recvb, ncclUint8_, s, ic->p2p, st);
			at += recvb;
		}
		const int rc2 = n.GroupEnd();                /* always: a group left open would swallow every later collective */
		if (rc == ncclSuccess_) rc = rc2;
		if (rc != ncclSuccess_) return nccl_fail(rc, "ncclSend / ncclRecv (row exchange)");
		ic->ncollectives++;
		return GG_OK;
	}
	uint64_t maxc = 0;
	for (int i = 0; i < N * N; i++) if (ic->h_counts[i] > maxc) maxc = ic->h_counts[i];
	if (maxc == 0) return GG_OK;
	const size_t part = (size_t) maxc * unit;
	const size_t need = part * (size_t) N * (size_t) (N + 1);
	if (ic->ag_bytes < need)
	{
		GG_CUDA(cudaStreamSynchronize(st));
		cudaFree(ic->ag_buf);
		ic->ag_buf = nullptr; ic->ag_bytes = 0;
		cudaError_t ce = cudaMalloc((void **) &ic->ag_buf, need);
		if (ce != cudaSuccess) { cudaGetLastError(); gg_set_error("row exchange by all-gather: %zu bytes of staging do not fit in device memory", need); return GG_ERR_NOMEM; }
		ic->ag_bytes = need;
	}
	uint8_t *mine = ic->ag_buf, *all = ic->ag_buf + part * (size_t) N;
	for (int d = 0; d < N; d++)
	{
		const size_t b = (size_t) ic->h_counts[(size_t) ic->seg * N + d] * unit;
		if (b) GG_CUDA(cudaMemcpyAsync(mine + part * (size_t) d, send_base + send_off[d], b, cudaMemcpyDeviceToDevice, st));
	}
	int rc = ic_allgather(ic, mine, all, part * (size_t) N);
	if (rc) return rc;
	size_t at = 0;
	for (int s = 0; s < N; s++)
	{
		const size_t b = (size_t) ic->h_counts[(size_t) s * N + ic->seg] * unit;
		if (b) GG_CUDA(cudaMemcpyAsync(recv_base + at, all + part * ((size_t) s * N + (size_t) ic->seg), b, cudaMemcpyDeviceToDevice, st));
		at += b;
	}
	return GG_OK;
}

/* Motion of group records, device to device: the sending half (execMotionSender, nodeMotion.c:270-374) packs the
 * pipeline's result into this segment's block, the all-gather is the interconnect, the receiving half
 * (execMotionUnsortedReceiver, :378) keeps what is routed here. */
static uint32_t errflag_of_code(int code)
{
	switch (code)
	{
		case GG_OK: return 0;
		case GG_ERR_FLOAT_OVERFLOW: return GGP_EF_FLOAT_OVERFLOW;
		case GG_ERR_FLOAT_UNDERFLOW: return GGP_EF_FLOAT_UNDERFLOW;
		case GG_ERR_DIV_ZERO: return GGP_EF_DIV_ZERO;
		case GG_ERR_INT_OVERFLOW: return GGP_EF_INT_OVERFLOW;
		case GG_ERR_VISIBILITY: return GGP_EF_VISIBILITY;
		case GG_ERR_BADPAGE: return GGP_EF_BADPAGE;
		case GG_ERR_DATE_RANGE: return GGP_EF_DATE_RANGE;
		case GG_ERR_RETRY_HOST: return GGP_EF_HOSTPATH;
	}
	return GGP_EF_PEER_FAILED;
}

int gg_ic_motion_groups(gg_interconnect *ic, int motion_type, int root, int nhash, const int32_t *hashcol,
                        const int32_t *hashtypid, gg_groups *in, int local_error, gg_groups **out)
{
	if (!ic || !out || nhash < 0 || nhash > GG_MAX_KEYS || (nhash && (!hashcol || !hashtypid))) return GG_ERR_ARG;
	if (motion_type != GG_IC_MOTION_HASH && motion_type != GG_IC_MOTION_GATHER && motion_type != GG_IC_MOTION_BROADCAST) return GG_ERR_ARG;
	if (motion_type == GG_IC_MOTION_HASH && nhash < 1) return GG_ERR_ARG;
	if (root < 0 || root >= ic->nsegs) return GG_ERR_ARG;
	*out = nullptr;
	gg_engine *e = ic->eng;
	GG_CUDA(cudaSetDevice(e->device));
	cudaStream_t st = e->stream;
	IC_TRACE(ic, "motion_groups type %d root %d in %p local_error %d", motion_type, root, (void *) in, local_error);
	RouteSpec spec;
	memset(&spec, 0, sizeof spec);
	spec.nhash = nhash;
	for (int k = 0; k < nhash; k++)
	{
		if (hashcol[k] < 0 || (in && hashcol[k] >= in->nkeys))
		{ gg_set_error("Motion hash column %d is not a grouping column of the rows below", hashcol[k]); return GG_ERR_UNSUPPORTED; }
		spec.hashcol[k] = hashcol[k];
		spec.hashtype[k] = ggp_hashtype_of(hashtypid[k]);
		if (!spec.hashtype[k]) { gg_set_error("hash column type %d has no device hash function", hashtypid[k]); return GG_ERR_UNSUPPORTED; }
	}
	gg_groups *g = gg_groups_alloc(e, in, ic->nsegs * GG_IC_GROUP_CAP, /*sparse*/ true);
	if (!g) return GG_ERR_NOMEM;
	const uint32_t local_flags = in ? errflag_of_code(local_error) : (local_error != GG_OK ? errflag_of_code(local_error) : GGP_EF_HOSTPATH);
	if (in) gg_ic_pack_groups_kernel<<<1, 256, 0, st>>>(in->recs, in->d_n, in->d_status, in->sparse ? 1 : 0, in->cap, local_flags, ic->d_send);
	else gg_ic_pack_groups_kernel<<<1, 256, 0, st>>>(nullptr, nullptr, nullptr, 0, 0, local_flags, ic->d_send);
	cudaError_t ce = cudaGetLastError();
	e->launches++;
	int rc = ce == cudaSuccess ? ic_allgather(ic, ic->d_send, ic->d_all, sizeof(GroupBlock)) : gg_cuda_fail(ce, "gg_ic_motion_groups");
	if (rc) { gg_groups_free(g); return rc; }
	gg_ic_route_groups_kernel<<<1, 256, 0, st>>>(ic->d_all, ic->nsegs, ic->seg, motion_type, root, spec, g->recs, g->d_status);
	ce = cudaGetLastError();
	e->launches++;
	if (ce != cudaSuccess) { gg_groups_free(g); return gg_cuda_fail(ce, "gg_ic_motion_groups"); }
	*out = g;
	return GG_OK;
}

/* Redistribute Motion of datum rows: send_rows = nsegs regions of region_cap rows of `rowwords` words (what
 * gg_motion_partition wrote), counts[d] rows valid in region d.  Receives into recv_rows (capacity recv_cap rows),
 * senders in segment order; *nrecv = rows received.  The count exchange is the only host synchronisation. */
int gg_ic_exchange_rows(gg_interconnect *ic, const void *send_rows, const uint64_t *counts, uint64_t region_cap, int rowwords,
                        void *recv_rows, uint64_t recv_cap, uint64_t *nrecv)
{
	if (!ic || !send_rows || !counts || !recv_rows || !nrecv || rowwords < 1) return GG_ERR_ARG;
	gg_engine *e = ic->eng;
	GG_CUDA(cudaSetDevice(e->device));
	cudaStream_t st = e->stream;
	const int N = ic->nsegs;
	const size_t rb = (size_t) rowwords * 8;
	if (!ic->comm)
	{
		if (counts[0] > recv_cap) { gg_set_error("Motion receive buffer too small: %llu rows, capacity %llu", (unsigned long long) counts[0], (unsigned long long) recv_cap); return GG_ERR_NOMEM; }
		GG_CUDA(cudaMemcpyAsync(recv_rows, send_rows, counts[0] * rb, cudaMemcpyDeviceToDevice, st));
		*nrecv = counts[0];
		return GG_OK;
	}
	{
		int rcd = ic_decide_row_transport(ic);
		if (rcd) return rcd;
	}
	/* count exchange: row d of the matrix = what segment d sends to everybody */
	IC_TRACE(ic, "exchange_rows: rowwords %d region_cap %llu recv_cap %llu counts[0] %llu", rowwords, (unsigned long long) region_cap,
	         (unsigned long long) recv_cap, (unsigned long long) counts[0]);
	GG_CUDA(cudaMemcpyAsync(ic->d_counts, counts, 8 * (size_t) N, cudaMemcpyHostToDevice, st));
	int rc = ic_allgather(ic, ic->d_counts, ic->d_counts + N, 8 * (size_t) N);
	if (rc) return rc;
	GG_CUDA(cudaMemcpyAsync(ic->h_counts, ic->d_counts + N, 8 * (size_t) N * N, cudaMemcpyDeviceToHost, st));
	GG_CUDA(cudaStreamSynchronize(st));
	uint64_t total = 0;
	for (int s = 0; s < N; s++) total += ic->h_counts[(size_t) s * N + ic->seg];
	*nrecv = total;
	/* every segment computes every segment's total, so an overflow anywhere makes everybody skip the exchange */
	int overflow = 0;
	for (int d = 0; d < N; d++)
	{
		uint64_t t = 0;
		for (int s = 0; s < N; s++) t += ic->h_counts[(size_t) s * N + d];
		if (d == ic->seg ? t > recv_cap : false) overflow = 1;
	}
	/* capacities are local knowledge: agree on the outcome with one more (tiny) exchange */
	{
		uint64_t all[1024];
		if (N > 1024) return GG_ERR_UNSUPPORTED;
		rc = gg_ic_allgather_u64(ic, (uint64_t) overflow, all);
		if (rc) return rc;
		for (int s = 0; s < N; s++) if (all[s]) overflow = 2;
	}
	if (overflow)
	{
		gg_set_error("Motion receive buffer too small on some segment (this one receives %llu rows, capacity %llu)",
		             (unsigned long long) total, (unsigned long long) recv_cap);
		return GG_ERR_NOMEM;
	}
	{
		size_t send_off[1024];
		for (int s = 0; s < N; s++) send_off[s] = (size_t) s * region_cap * rb;
		rc = ic_alltoallv(ic, (const uint8_t *) send_rows, send_off, (uint8_t *) recv_rows, rb);
		if (rc) return rc;
	}
	IC_TRACE(ic, "exchange_rows: issued (%s), %llu rows arrive here", ic->p2p_ok ? "send/recv" : "all-gather", (unsigned long long) total);
	return GG_OK;
}

/* The executor's generic Motion of host rows (GgRowBatch): values [nrows][ncols] Datums, isnull [nrows][ncols], dest[i] =
 * receiving segment or -1 for all.  Staged through device memory; out arrays are malloc'd, the caller frees them. */
int gg_ic_exchange_host(gg_interconnect *ic, int ncols, int64_t nrows, const int64_t *values, const uint8_t *isnull,
                        const int32_t *dest, int my_error, int64_t *out_nrows, int64_t **out_values, uint8_t **out_isnull)
{
	if (my_error) nrows = 0;
	if (ic) IC_TRACE(ic, "exchange_host: ncols %d nrows %lld my_error %d", ncols, (long long) nrows, my_error);
	if (!ic || ncols < 1 || nrows < 0 || (nrows && (!values || !isnull || !dest)) || !out_nrows || !out_values || !out_isnull) return GG_ERR_ARG;
	gg_engine *e = ic->eng;
	GG_CUDA(cudaSetDevice(e->device));
	const int N = ic->nsegs;
	const size_t W = hostrow_words(ncols);
	if (N + 1 > 1024) return GG_ERR_UNSUPPORTED;
	std::vector<uint64_t> counts((size_t) N, 0), offs((size_t) N + 1, 0), fill((size_t) N, 0);
	{
		/* the sender's status travels ahead of the rows: a segment whose slice failed still enters the exchange, with no
		 * rows, and every segment learns of it here (the reference: SendStopMessage / error propagation, cdbmotion.c:342) */
		uint64_t all[1024];
		int rcs = gg_ic_allgather_u64(ic, (uint64_t) (my_error != 0), all);
		if (rcs) return rcs;
		for (int s = 0; s < N; s++)
			if (all[s]) { gg_set_error("segment %d reported an error in its slice below the Motion", s); return GG_ERR_PEER; }
	}
	if (ic->comm)
	{
		int rcd = ic_decide_row_transport(ic);
		if (rcd) return rcd;
	}
	for (int64_t r = 0; r < nrows; r++)
	{
		if (dest[r] < -1 || dest[r] >= N) { gg_set_error("Motion destination %d out of range", dest[r]); return GG_ERR_ARG; }
		if (dest[r] < 0) for (int d = 0; d < N; d++) counts[(size_t) d]++;
		else counts[(size_t) dest[r]]++;
	}
	for (int d = 0; d < N; d++) offs[(size_t) d + 1] = offs[(size_t) d] + counts[(size_t) d];
	const uint64_t nsend = offs[(size_t) N];
	std::vector<uint64_t> packed((size_t) (nsend ? nsend : 1) * W, 0);
	auto put = [&](int d, int64_t r) {
		uint64_t *p = packed.data() + (offs[(size_t) d] + fill[(size_t) d]++) * W;
		memcpy(p, values + (size_t) r * ncols, 8 * (size_t) ncols);
		memcpy(p + ncols, isnull + (size_t) r * ncols, (size_t) ncols);
	};
	for (int64_t r = 0; r < nrows; r++)
	{
		if (dest[r] < 0) for (int d = 0; d < N; d++) put(d, r);
		else put(dest[r], r);
	}
	/* count exchange first: it sizes the staging */
	cudaStream_t st = e->stream;
	GG_CUDA(cudaMemcpyAsync(ic->d_counts, counts.data(), 8 * (size_t) N, cudaMemcpyHostToDevice, st));
	int rc = ic_allgather(ic, ic->d_counts, ic->d_counts + N, 8 * (size_t) N);
	if (rc) return rc;
	GG_CUDA(cudaMemcpyAsync(ic->h_counts, ic->d_counts + N, 8 * (size_t) N * N, cudaMemcpyDeviceToHost, st));
	GG_CUDA(cudaStreamSynchronize(st));
	uint64_t nrecv = 0;
	for (int s = 0; s < N; s++) nrecv += ic->h_counts[(size_t) s * N + ic->seg];
	const size_t need = (size_t) (nsend + nrecv + 2) * W * 8;
	if (ic->stage_bytes < need)
	{
		cudaFree(ic->stage);
		ic->stage = nullptr; ic->stage_bytes = 0;
		GG_CUDA(cudaMalloc(&ic->stage, need));
		ic->stage_bytes = need;
	}
	uint64_t *d_send = (uint64_t *) ic->stage, *d_recv = d_send + (size_t) (nsend + 1) * W;
	if (nsend) GG_CUDA(cudaMemcpyAsync(d_send, packed.data(), (size_t) nsend * W * 8, cudaMemcpyHostToDevice, st));
	if (!ic->comm)
	{
		if (nsend) GG_CUDA(cudaMemcpyAsync(d_recv, d_send, (size_t) nsend * W * 8, cudaMemcpyDeviceToDevice, st));
	}
	else
	{
		size_t send_off[1024];
		for (int s = 0; s < N; s++) send_off[s] = (size_t) offs[(size_t) s] * W * 8;
		rc = ic_alltoallv(ic, (const uint8_t *) d_send, send_off, (uint8_t *) d_recv, W * 8);
		if (rc) return rc;
	}
	std::vector<uint64_t> got((size_t) (nrecv ? nrecv : 1) * W);
	if (nrecv) GG_CUDA(cudaMemcpyAsync(got.data(), d_recv, (size_t) nrecv * W * 8, cudaMemcpyDeviceToHost, st));
	GG_CUDA(cudaStreamSynchronize(st));
	int64_t *ov = (int64_t *) malloc(8 * (size_t) (nrecv ? nrecv : 1) * ncols);
	uint8_t *on = (uint8_t *) malloc((size_t) (nrecv ? nrecv : 1) * ncols);
	if (!ov || !on) { free(ov); free(on); gg_set_error("out of memory"); return GG_ERR_NOMEM; }
	for (uint64_t r = 0; r < nrecv; r++)
	{
		memcpy(ov + r * ncols, got.data() + r * W, 8 * (size_t) ncols);
		memcpy(on + r * ncols, got.data() + r * W + ncols, (size_t) ncols);
	}
	*out_nrows = (int64_t) nrecv; *out_values = ov; *out_isnull = on;
	return GG_OK;
}

}  /* extern "C" */
