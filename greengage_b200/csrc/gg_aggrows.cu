/*
 * gg_aggrows.cu — the groups of an Agg, finalised on the device into GG_FMT_DATUMROWS rows (include/ggb200.h
 * gg_scanagg_datumrows / gg_joinagg_datumrows / gg_groups_datumrows), so that a Sort or a Limit above the Agg takes them where
 * they are (nodeAgg.c:871-999 finalize_aggregate + the slot the Agg hands up, as one kernel).
 *
 * A row is word 0 = NULL mask (bit c: grouping column c, bit numCols + i: aggregate i), then the grouping keys, then one word
 * per aggregate: exactly the bits finalize_rows (gg_scanagg.cu) puts into a gg_aggrow's key[c], f[0] or i, by the one rule
 * both apply (gg_aggfinal.h).
 *
 * Two sources:
 *   group records (ggp_grec)   the merged records of a block-table variant, or a gg_groups set: one row per valid record,
 *                              in record order (the order gg_*_fetch returns them in)
 *   the HBM hash table         of the general HashAggregate, read in place: an order-preserving compaction over the table's
 *                              slots — per-tile counts, the exclusive scan of gg_sort.cu, per-tile writes — so the row order
 *                              is a function of the table's contents, with no atomics deciding it
 *
 * And the row filter of an Agg's HAVING (gg_rowfilter_*): the same order-preserving compaction over datum rows, with the
 * interpreter deciding which rows pass.
 */
#include <cuda_runtime.h>
#include <stdint.h>
#include <cstring>
#include "gg_pipeline.h"
#include "gg_groups.h"
#include "gg_aggfinal.h"

using namespace ggd;

#define AGGROWS_THREADS 256
#define AGGROWS_ITEMS   16
#define AGGROWS_TILE    (AGGROWS_THREADS * AGGROWS_ITEMS)      /* table slots / records per tile of the compaction */

/* how a group becomes a row: the Agg's grouping columns and aggregates, and the accumulator column each aggregate reads */
struct AggRowSpec {
	int nkeys, naggs;
	int32_t fn[GG_MAX_AGGS];
	int32_t col[GG_MAX_AGGS];                 /* ggp_aggmap::col: -1 for count(*) */
};

/* one row: keys, then every aggregate finalised from count, N(col) (non-NULL inputs of accumulator column col) and A(col)
 * (that column's accumulator bits), read straight from the source */
template <class N, class A>
__device__ __forceinline__ void put_row(const AggRowSpec &S, uint64_t keynull, const uint64_t *key, uint64_t count, N nn, A acc,
                                        unsigned long long *row)
{
	uint64_t mask = keynull;
	for (int c = 0; c < S.nkeys; c++) row[1 + c] = key[c];
	for (int i = 0; i < S.naggs; i++)
	{
		const int col = S.col[i];
		int isnull = 0;
		row[1 + S.nkeys + i] = gg_aggfinal(S.fn[i], count, col < 0 ? 0 : nn(col), col < 0 ? 0 : acc(col), &isnull);
		if (isnull) mask |= 1ull << (S.nkeys + i);
	}
	row[0] = mask;
}

/* record -> row (r == nullptr: the all-zero record of a plain aggregate over no input) */
__device__ __forceinline__ void grec_row(const AggRowSpec &S, const ggp_grec *r, unsigned long long *row)
{
	uint64_t key[GG_MAX_KEYS] = { 0, 0, 0, 0 };
	if (!r)
	{
		put_row(S, 0, key, 0, [](int) { return (uint64_t) 0; }, [](int) { return (uint64_t) 0; }, row);
		return;
	}
	for (int c = 0; c < S.nkeys; c++) key[c] = r->key[c];
	put_row(S, r->keynull & ((1u << S.nkeys) - 1), key, r->count, [r](int j) { return (uint64_t) r->n[j]; },
	        [r](int j) { return (uint64_t) __double_as_longlong(r->sum[j]); }, row);
}

/* table entry -> row; float8pl's CHECKFLOATVAL (float.c:782) as gg_hashagg_emit_kernel applies it: an infinite sum of finite
 * inputs is an overflow */
__device__ __forceinline__ void hash_row(const AggRowSpec &S, const HashAggTable &ha, uint64_t slot, bool saw_inf, uint32_t *errflags,
                                         unsigned long long *row)
{
	const unsigned long long *ep = ha.ent + slot * ha.stride;
	uint64_t key[GG_MAX_KEYS] = { 0, 0, 0, 0 };
	const uint64_t count = ep[ha.off_cnt];
	const uint32_t off_accn = ha.off_accn, off_acc = ha.off_acc;
	auto nn = [=](int j) { return off_accn ? (uint64_t) ep[off_accn + j] : count; };      /* no NULLs anywhere: every row counted */
	auto acc = [=](int j) { return (uint64_t) ep[off_acc + j]; };
	for (int c = 0; c < ha.nkeys; c++) key[c] = ep[1 + c];
	for (int j = 0; j < ha.nacc; j++)
		if (ha.acckind[j] == GGP_ACC_F8SUM && !saw_inf && nn(j) && !f8_finite(__longlong_as_double((long long) acc(j))))
			atomicOr(errflags, GGP_EF_FLOAT_OVERFLOW);
	put_row(S, (uint32_t) (ep[0] >> 32) & 0xF & ((1u << S.nkeys) - 1), key, count, nn, acc, row);
}

/* the two sources of the compaction: which slots hold a group, and how a slot becomes a row */
struct GrecSrc {
	const ggp_grec *recs;
	__device__ bool valid(uint64_t i) const { return recs[i].valid != 0; }
	__device__ void row(const AggRowSpec &S, uint64_t i, bool, uint32_t *, unsigned long long *out) const { grec_row(S, recs + i, out); }
};

struct HashSrc {
	HashAggTable ha;
	__device__ bool valid(uint64_t i) const { return (ha.ent[i * ha.stride] >> 63) != 0; }
	__device__ void row(const AggRowSpec &S, uint64_t i, bool saw_inf, uint32_t *errflags, unsigned long long *out) const
	{
		hash_row(S, ha, i, saw_inf, errflags, out);
	}
};

/* dense records [0, n): row i = record i; n == 1 with recs == nullptr: the empty-input row of a plain aggregate */
__global__ void __launch_bounds__(AGGROWS_THREADS)
gg_aggrows_dense_kernel(const ggp_grec *recs, uint64_t n, const AggRowSpec S, unsigned long long *out)
{
	const uint64_t W = 1 + (uint64_t) S.nkeys + (uint64_t) S.naggs;
	for (uint64_t i = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; i < n; i += (uint64_t) gridDim.x * blockDim.x)
		grec_row(S, recs ? recs + i : nullptr, out + i * W);
}

/* compaction, step 1: valid slots per tile -> cnt[tile] */
template <class Src>
__global__ void __launch_bounds__(AGGROWS_THREADS)
gg_aggrows_count_kernel(const Src src, uint64_t nslots, uint32_t *cnt)
{
	__shared__ uint32_t s_warp[AGGROWS_THREADS / 32];
	const uint64_t base = (uint64_t) blockIdx.x * AGGROWS_TILE;
	uint32_t c = 0;
	for (int k = 0; k < AGGROWS_ITEMS; k++)
	{
		const uint64_t i = base + (uint64_t) k * AGGROWS_THREADS + threadIdx.x;
		c += (i < nslots && src.valid(i)) ? 1u : 0u;
	}
	for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(GG_FULL_MASK, c, o);
	if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = c;
	__syncthreads();
	if (threadIdx.x == 0)
	{
		uint32_t t = 0;
		for (int w = 0; w < AGGROWS_THREADS / 32; w++) t += s_warp[w];
		cnt[blockIdx.x] = t;
	}
}

/* compaction, step 3: every tile writes its valid slots, in slot order, from the tile's exclusive prefix cnt[tile] on */
template <class Src>
__global__ void __launch_bounds__(AGGROWS_THREADS)
gg_aggrows_write_kernel(const Src src, uint64_t nslots, const uint32_t *cnt, const AggRowSpec S, uint32_t *errflags,
                        unsigned long long *out)
{
	__shared__ uint32_t s_warp[AGGROWS_THREADS / 32];
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const uint64_t W = 1 + (uint64_t) S.nkeys + (uint64_t) S.naggs;
	const uint64_t base = (uint64_t) blockIdx.x * AGGROWS_TILE;
	const bool saw_inf = (*errflags & GGP_EF_SAW_INF) != 0;
	uint64_t at = cnt[blockIdx.x];
	for (int k = 0; k < AGGROWS_ITEMS; k++)
	{
		const uint64_t i = base + (uint64_t) k * AGGROWS_THREADS + threadIdx.x;
		const bool v = i < nslots && src.valid(i);
		const unsigned b = __ballot_sync(GG_FULL_MASK, v);
		if (lane == 0) s_warp[warp] = __popc(b);
		__syncthreads();
		uint32_t pre = 0, tot = 0;
		for (int w = 0; w < AGGROWS_THREADS / 32; w++) { const uint32_t s = s_warp[w]; pre += w < warp ? s : 0; tot += s; }
		__syncthreads();
		if (v)
		{
			unsigned long long *row = out + (at + pre + __popc(b & ((1u << lane) - 1))) * W;
			src.row(S, i, saw_inf, errflags, row);
		}
		at += tot;
	}
}

/* ---- the row filter (gg_rowfilter_*): an Agg's HAVING over its datum rows, order-preserving ----
 * pass 1  a tile of RF_TILE rows, RF_THREADS at a time, is copied coalesced into shared memory (odd word stride: the lanes read
 *         their own rows from distinct banks); every thread runs the interpreter over its row (datumrow_passes); one pass bit per
 *         row, one count per tile
 * pass 2  the exclusive scan of the counts (gg_scan_*)
 * pass 3  every tile copies its passing rows, in row order, from its exclusive prefix on: placement is a function of the input */
#define RF_THREADS 256
#define RF_ITEMS   8
#define RF_TILE    (RF_THREADS * RF_ITEMS)

__global__ void __launch_bounds__(RF_THREADS)
gg_rowfilter_count_kernel(const __grid_constant__ ggp_program P, const unsigned long long *rows, uint64_t n, uint32_t W, uint32_t *bits,
                          uint32_t *cnt, uint32_t *errflags)
{
	extern __shared__ __align__(16) unsigned long long s_rows[];
	__shared__ uint32_t s_warp[RF_THREADS / 32];
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const uint32_t S = W | 1u;
	uint32_t c = 0, err = 0;
	for (int k = 0; k < RF_ITEMS; k++)
	{
		const uint64_t base = (uint64_t) blockIdx.x * RF_TILE + (uint64_t) k * RF_THREADS;
		if (base >= n) break;                                              /* the same for the whole block */
		const uint32_t m = n - base < RF_THREADS ? (uint32_t) (n - base) : RF_THREADS;
		const unsigned long long *src = rows + base * W;
		__syncthreads();
		for (uint32_t j = threadIdx.x; j < m * W; j += RF_THREADS)
		{
			const uint32_t r = j / W;
			s_rows[r * S + (j - r * W)] = src[j];
		}
		__syncthreads();
		const bool present = threadIdx.x < m;
		const bool pass = datumrow_passes(P, smem_u32(s_rows + (present ? threadIdx.x : 0) * S), present, lane, err);
		const unsigned b = __ballot_sync(GG_FULL_MASK, pass);
		if (lane == 0) bits[(base >> 5) + warp] = b;
		c += pass ? 1u : 0u;
	}
	if (err) atomicOr(errflags, err);
	for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(GG_FULL_MASK, c, o);
	if (lane == 0) s_warp[warp] = c;
	__syncthreads();
	if (threadIdx.x == 0)
	{
		uint32_t t = 0;
		for (int w = 0; w < RF_THREADS / 32; w++) t += s_warp[w];
		cnt[blockIdx.x] = t;
	}
}

__global__ void __launch_bounds__(RF_THREADS)
gg_rowfilter_write_kernel(const unsigned long long *rows, uint64_t n, uint32_t W, const uint32_t *bits, const uint32_t *cnt,
                          unsigned long long *out)
{
	__shared__ uint32_t s_warp[RF_THREADS / 32];
	__shared__ uint16_t s_idx[RF_THREADS];
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	uint64_t at = cnt[blockIdx.x];
	for (int k = 0; k < RF_ITEMS; k++)
	{
		const uint64_t base = (uint64_t) blockIdx.x * RF_TILE + (uint64_t) k * RF_THREADS;
		if (base >= n) break;
		const unsigned b = bits[(base >> 5) + warp];
		if (lane == 0) s_warp[warp] = __popc(b);
		__syncthreads();
		uint32_t pre = 0, tot = 0;
		for (int w = 0; w < RF_THREADS / 32; w++) { const uint32_t s = s_warp[w]; pre += w < warp ? s : 0; tot += s; }
		if ((b >> lane) & 1u) s_idx[pre + __popc(b & ((1u << lane) - 1u))] = (uint16_t) threadIdx.x;
		__syncthreads();
		/* the survivors' words, written contiguously */
		unsigned long long *dst = out + at * W;
		for (uint32_t j = threadIdx.x; j < tot * W; j += RF_THREADS)
		{
			const uint32_t r = j / W;
			dst[j] = rows[(base + s_idx[r]) * W + (j - r * W)];
		}
		at += tot;
		__syncthreads();                                                   /* s_warp / s_idx are reused */
	}
}

/* the exclusive scan of gg_sort.cu over m counters (three phases over chunks of 4096) */
__global__ void gg_scan_sums_kernel(const uint32_t *x, uint64_t m, uint32_t *sums);
__global__ void gg_scan_top_kernel(uint32_t *sums, uint32_t nblk);
__global__ void gg_scan_apply_kernel(uint32_t *x, uint64_t m, const uint32_t *sums);

struct gg_rowfilter {
	gg_engine *eng = nullptr;
	ggp_program prog;                    /* ggp_compile_filter */
	int ncols = 0;                       /* columns of the rows filtered (a row is 1 + ncols words) */
	uint32_t *scratch = nullptr;         /* error word, tile counts, scan sums, pass bits; grown as needed */
	uint64_t scratch_words = 0;
	gg_relation *rows_buf = nullptr;     /* the survivors (owned) */
	gg_relation *rows_view = nullptr;    /* the view handed out */
};

/* =====================================================================================
 * host side
 * ===================================================================================== */

/* the row layout of an Agg's groups; GG_ERR_UNSUPPORTED for what only the host finalises */
static int aggrow_spec(const gg_agg *agg, const ggp_aggmap *aggmap, AggRowSpec *S)
{
	if (agg->aggstage == GG_AGGSTAGE_PARTIAL)
	{ gg_set_error("a PARTIAL-stage Agg hands up transition states: its consumers read group records"); return GG_ERR_UNSUPPORTED; }
	if (agg->numCols < 0 || agg->numCols > GG_MAX_KEYS || agg->numAggs < 0 || agg->numAggs > GG_MAX_AGGS) return GG_ERR_ARG;
	memset(S, 0, sizeof *S);
	S->nkeys = agg->numCols;
	S->naggs = agg->numAggs;
	for (int i = 0; i < agg->numAggs; i++)
	{
		const int32_t fn = agg->aggs[i].aggfnoid;
		if (!gg_aggfinal_covers(fn)) { gg_set_error("aggregate %d is finalised on the host only (numeric sum / avg)", fn); return GG_ERR_UNSUPPORTED; }
		S->fn[i] = fn;
		S->col[i] = aggmap[i].col;
		if (S->col[i] >= GGP_MAX_ACCS || (S->col[i] < 0 && fn != GG_AGG_COUNT_STAR)) { gg_set_error("aggregate %d: accumulator column %d", i, S->col[i]); return GG_ERR_ARG; }
	}
	return GG_OK;
}

/* an owned buffer of at least `n` rows of W words plus 16 bytes of slack, in whole 32 KB blocks (readers copy whole blocks) */
static int reserve_rows(gg_engine *e, gg_relation **buf, uint64_t n, uint64_t W)
{
	const uint64_t nb = (n * W * 8 + 16 + GG_BLCKSZ - 1) / GG_BLCKSZ;
	if (*buf && (*buf)->nblocks >= nb) return GG_OK;
	if (*buf) { gg_relation_free(*buf); *buf = nullptr; }
	return gg_relation_create(e, nb, buf);
}

/* rows of the valid entries among nslots of `src`, in slot order, into *buf (grown as needed); *nrows = their number */
template <class Src>
static int compact_rows(gg_engine *e, const Src &src, uint64_t nslots, const AggRowSpec &S, uint32_t *d_err, gg_relation **buf, uint64_t *nrows)
{
	cudaStream_t st = e->stream;
	const uint64_t W = 1 + (uint64_t) S.nkeys + (uint64_t) S.naggs;
	const uint64_t ntiles = (nslots + AGGROWS_TILE - 1) / AGGROWS_TILE;
	const uint64_t m = ntiles + 1;                              /* per-tile counts, then the total */
	const uint32_t nblk = (uint32_t) ((m + 4095) / 4096);
	uint32_t *cnt = nullptr, total = 0;
	*nrows = 0;
	if (ntiles == 0) return reserve_rows(e, buf, 0, W);
	cudaError_t ce = cudaMalloc((void **) &cnt, (size_t) (m + nblk) * 4);
	if (ce != cudaSuccess) { cudaGetLastError(); gg_set_error("aggregate rows: scratch of %llu counters does not fit in device memory", (unsigned long long) m); return GG_ERR_NOMEM; }
	uint32_t *sums = cnt + m;
	int rc = GG_OK;
	if ((ce = cudaMemsetAsync(cnt, 0, (size_t) m * 4, st)) != cudaSuccess) goto fail;
	gg_aggrows_count_kernel<Src><<<(unsigned) ntiles, AGGROWS_THREADS, 0, st>>>(src, nslots, cnt);
	gg_scan_sums_kernel<<<nblk, 256, 0, st>>>(cnt, m, sums);
	gg_scan_top_kernel<<<1, 256, 0, st>>>(sums, nblk);
	gg_scan_apply_kernel<<<nblk, 256, 0, st>>>(cnt, m, sums);
	e->launches += 4;
	if ((ce = cudaGetLastError()) != cudaSuccess) goto fail;
	if ((ce = cudaMemcpyAsync(&total, cnt + ntiles, 4, cudaMemcpyDeviceToHost, st)) != cudaSuccess) goto fail;
	if ((ce = cudaStreamSynchronize(st)) != cudaSuccess) goto fail;
	rc = reserve_rows(e, buf, total, W);
	if (rc == GG_OK && total)
	{
		gg_aggrows_write_kernel<Src><<<(unsigned) ntiles, AGGROWS_THREADS, 0, st>>>(src, nslots, cnt, S, d_err, (unsigned long long *) (*buf)->pages);
		e->launches++;
		if ((ce = cudaGetLastError()) != cudaSuccess) goto fail;
	}
	cudaFree(cnt);
	*nrows = total;
	return rc;
fail:
	cudaFree(cnt);
	return gg_cuda_fail(ce, "aggregate rows");
}

/* dense records [0, n) -> rows; n == 0 with `empty_row`: the one row of a plain aggregate over no input (nodeAgg.c:1247-1400) */
static int dense_rows(gg_engine *e, const ggp_grec *recs, uint64_t n, bool empty_row, const AggRowSpec &S, gg_relation **buf, uint64_t *nrows)
{
	const uint64_t W = 1 + (uint64_t) S.nkeys + (uint64_t) S.naggs;
	const bool zero = n == 0 && empty_row;
	const uint64_t rows = zero ? 1 : n;
	int rc = reserve_rows(e, buf, rows, W);
	if (rc) return rc;
	if (rows)
	{
		const uint64_t blocks = (rows + AGGROWS_THREADS - 1) / AGGROWS_THREADS;
		gg_aggrows_dense_kernel<<<(unsigned) (blocks < 65535 ? blocks : 65535), AGGROWS_THREADS, 0, e->stream>>>(zero ? nullptr : recs, rows, S,
		                                                                                                      (unsigned long long *) (*buf)->pages);
		GG_CUDA(cudaGetLastError());
		e->launches++;
	}
	*nrows = rows;
	return GG_OK;
}

/* the view handed out: valid until the owner's reset or free */
static int rows_view(gg_engine *e, gg_relation *buf, uint64_t n, int ncols, gg_relation **view)
{
	if (*view) { gg_relation_free(*view); *view = nullptr; }
	const int rc = gg_relation_attach_rows(e, buf->pages, n, ncols, view);
	if (rc) *view = nullptr;
	return rc;
}

extern "C" {

int gg_scanagg_datumrows(gg_scanagg *p, gg_relation **rows, uint64_t *nrows)
{
	if (!p || !rows || !nrows) return GG_ERR_ARG;
	if (p->join_rows) { gg_set_error("a join with a target list returns its rows through gg_joinagg_rows"); return GG_ERR_ARG; }
	if (!p->rows_view)
	{
		AggRowSpec S;
		int rc = aggrow_spec(&p->agg, p->aggmap, &S);
		if (rc) return rc;
		if (S.nkeys + S.naggs < 1) { gg_set_error("an Agg without columns has no datum rows"); return GG_ERR_UNSUPPORTED; }
		gg_engine *e = p->eng;
		uint32_t flags = 0;
		unsigned long long counters[2];
		int nmerged = 0;
		rc = scanagg_settle(p, &flags, &nmerged, counters);
		if (rc) return rc;
		uint64_t n = 0;
		if (p->mode == MODE_HASH)
		{
			/* the general HashAggregate: the groups come out of its table; the float8pl overflow rule raises into the status */
			if (p->has_state)
			{
				HashSrc src;
				src.ha = p->ha;
				rc = compact_rows(e, src, p->ha.cap, S, p->d_err, &p->rows_buf, &n);
				if (rc) return rc;
				GG_CUDA(cudaMemcpyAsync(&flags, p->d_err, sizeof flags, cudaMemcpyDeviceToHost, e->stream));
				GG_CUDA(cudaStreamSynchronize(e->stream));
			}
			rc = gg_errflags_to_code(flags & ~(uint32_t) GGP_EF_GROUP_OVERFLOW);
		}
		else
		{
			rc = gg_errflags_to_code(flags);
			n = p->has_state && nmerged > 0 ? (uint64_t) nmerged : 0;
		}
		if (rc) return rc;
		if (p->mode != MODE_HASH || n == 0) rc = dense_rows(e, p->recs, n, p->agg.numCols == 0, S, &p->rows_buf, &n);
		if (rc == GG_OK) rc = rows_view(e, p->rows_buf, n, S.nkeys + S.naggs, &p->rows_view);
		if (rc) return rc;
		p->rows_n = n;
	}
	*rows = p->rows_view;
	*nrows = p->rows_n;
	return GG_OK;
}

int gg_groups_datumrows(gg_groups *g, gg_relation **rows, uint64_t *nrows)
{
	if (!g || !rows || !nrows) return GG_ERR_ARG;
	if (!g->rows_view)
	{
		AggRowSpec S;
		int rc = aggrow_spec(&g->agg, g->aggmap, &S);
		if (rc) return rc;
		if (S.nkeys + S.naggs < 1) { gg_set_error("an Agg without columns has no datum rows"); return GG_ERR_UNSUPPORTED; }
		gg_engine *e = g->eng;
		GG_CUDA(cudaSetDevice(e->device));
		gg_groupstatus hs;
		GG_CUDA(cudaMemcpyAsync(&hs, g->d_status, sizeof hs, cudaMemcpyDeviceToHost, e->stream));
		GG_CUDA(cudaStreamSynchronize(e->stream));
		rc = gg_errflags_to_code(hs.err);
		if (rc) return rc;
		uint64_t n = 0;
		const bool empty_row = g->agg.numCols == 0 && !g->empty_is_empty;
		if (g->sparse)
		{
			GrecSrc src;
			src.recs = g->recs;
			rc = compact_rows(e, src, (uint64_t) g->cap, S, &g->d_status->err, &g->rows_buf, &n);
			if (rc == GG_OK && n == 0) rc = dense_rows(e, g->recs, 0, empty_row, S, &g->rows_buf, &n);
		}
		else
		{
			if (hs.n < 0 || hs.n > g->cap) { gg_set_error("group record count %d out of range", hs.n); return GG_ERR_CUDA; }
			rc = dense_rows(e, g->recs, (uint64_t) hs.n, empty_row, S, &g->rows_buf, &n);
		}
		if (rc == GG_OK) rc = rows_view(e, g->rows_buf, n, S.nkeys + S.naggs, &g->rows_view);
		if (rc) return rc;
		g->rows_n = n;
	}
	*rows = g->rows_view;
	*nrows = g->rows_n;
	return GG_OK;
}

int gg_rowfilter_create(gg_engine *e, const gg_tupdesc *rows_desc, int32_t qual, const gg_exprpool *pool, gg_rowfilter **out)
{
	if (!e || !rows_desc || !pool || !out) return GG_ERR_ARG;
	*out = nullptr;
	gg_scan scan;
	memset(&scan, 0, sizeof scan);
	scan.desc = *rows_desc;
	scan.qual = qual;
	gg_rowfilter *f = new gg_rowfilter();
	char msg[256];
	const int rc = ggp_compile_filter(&scan, pool, &f->prog, msg, sizeof msg);
	if (rc != GG_OK) { gg_set_error("HAVING: %s", msg); delete f; return rc; }
	f->eng = e;
	f->ncols = rows_desc->natts;
	*out = f;
	return GG_OK;
}

int gg_rowfilter_run(gg_rowfilter *f, gg_relation *rows, uint64_t nrows, gg_relation **out_view, uint64_t *nout)
{
	if (!f || !rows || !out_view || !nout) return GG_ERR_ARG;
	const uint64_t W = 1 + (uint64_t) f->ncols;
	if ((uint64_t) rows->rowwords != W) { gg_set_error("row filter over %d columns: the relation has rows of %d words", f->ncols, rows->rowwords); return GG_ERR_ARG; }
	if (nrows > rows->nrows) { gg_set_error("row filter: %llu rows of a relation of %llu", (unsigned long long) nrows, (unsigned long long) rows->nrows); return GG_ERR_ARG; }
	gg_engine *e = f->eng;
	cudaStream_t st = e->stream;
	GG_CUDA(cudaSetDevice(e->device));
	uint32_t total = 0;
	if (nrows)
	{
		/* scratch: the error word, ntiles + 1 counters (the last one becomes the total), the scan's block sums, the pass bits */
		const uint64_t ntiles = (nrows + RF_TILE - 1) / RF_TILE;
		const uint64_t m = ntiles + 1;
		const uint32_t nblk = (uint32_t) ((m + 4095) / 4096);
		const uint64_t words = 1 + m + nblk + ntiles * (RF_TILE / 32);
		if (f->scratch_words < words)
		{
			cudaFree(f->scratch);
			f->scratch = nullptr;
			f->scratch_words = 0;
			const cudaError_t ce = cudaMalloc((void **) &f->scratch, (size_t) words * 4);
			if (ce != cudaSuccess) { cudaGetLastError(); gg_set_error("row filter: scratch of %llu words does not fit in device memory", (unsigned long long) words); return GG_ERR_NOMEM; }
			f->scratch_words = words;
		}
		uint32_t *d_err = f->scratch, *cnt = f->scratch + 1, *sums = cnt + m, *bits = sums + nblk;
		const unsigned long long *in = (const unsigned long long *) rows->pages;
		const int smem = RF_THREADS * (int) (W | 1) * 8;
		GG_CUDA(cudaFuncSetAttribute(gg_rowfilter_count_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
		GG_CUDA(cudaMemsetAsync(f->scratch, 0, (size_t) (1 + m) * 4, st));
		gg_rowfilter_count_kernel<<<(unsigned) ntiles, RF_THREADS, smem, st>>>(f->prog, in, nrows, (uint32_t) W, bits, cnt, d_err);
		gg_scan_sums_kernel<<<nblk, 256, 0, st>>>(cnt, m, sums);
		gg_scan_top_kernel<<<1, 256, 0, st>>>(sums, nblk);
		gg_scan_apply_kernel<<<nblk, 256, 0, st>>>(cnt, m, sums);
		e->launches += 4;
		GG_CUDA(cudaGetLastError());
		uint32_t flags = 0;
		GG_CUDA(cudaMemcpyAsync(&flags, d_err, 4, cudaMemcpyDeviceToHost, st));
		GG_CUDA(cudaMemcpyAsync(&total, cnt + ntiles, 4, cudaMemcpyDeviceToHost, st));
		GG_CUDA(cudaStreamSynchronize(st));
		const int rc = gg_errflags_to_code(flags);
		if (rc != GG_OK) return rc;
		int r2 = reserve_rows(e, &f->rows_buf, total, W);
		if (r2) return r2;
		if (total)
		{
			gg_rowfilter_write_kernel<<<(unsigned) ntiles, RF_THREADS, 0, st>>>(in, nrows, (uint32_t) W, bits, cnt, (unsigned long long *) f->rows_buf->pages);
			e->launches++;
			GG_CUDA(cudaGetLastError());
		}
	}
	else
	{
		const int rc = reserve_rows(e, &f->rows_buf, 0, W);
		if (rc) return rc;
	}
	const int rc = rows_view(e, f->rows_buf, total, f->ncols, &f->rows_view);
	if (rc) return rc;
	*out_view = f->rows_view;
	*nout = total;
	return GG_OK;
}

void gg_rowfilter_free(gg_rowfilter *f)
{
	if (!f) return;
	if (f->eng) cudaSetDevice(f->eng->device);
	if (f->rows_view) gg_relation_free(f->rows_view);
	if (f->rows_buf) gg_relation_free(f->rows_buf);
	cudaFree(f->scratch);
	delete f;
}

}  /* extern "C" */
