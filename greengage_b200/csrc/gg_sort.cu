/*
 * gg_sort.cu — Sort: device LSD radix sort of fixed-width rows.
 *
 * Replaces tuplesort_begin_heap_mk / puttupleslot / performsort / gettupleslot
 * (tuplesort_mk.c:771,1154,1378,1668) and the comparator inlineApplySortFunction
 * (tuplesort_mk.c:2816-2850) for rows of int64 Datum columns.
 *
 * The comparator is turned into bits: every sort column becomes an order-preserving 64-bit radix key
 *     int4/int8/date/timestamp   x ^ sign bit                       (btint4cmp / btint8cmp / date_cmp)
 *     float8                     -0 -> +0, every NaN -> all ones,   (float8_cmp_internal, float.c:964:
 *                                negatives inverted, else ^ sign     NaN = NaN, NaN > everything)
 *     packed strings             byte swap: first character most significant, zero padding sorts
 *                                shorter-first (bpcharcmp on stripped bytes, varstr_cmp C locale)
 *     DESC                       ~key
 * plus one more 1-bit "digit" for NULLS FIRST/LAST.  mk_qsort is unstable, so only the comparator is
 * the contract; an LSD radix sort (stable passes, last sort column first) satisfies it.
 *
 * One pass = histogram kernel (per-tile digit counts) + scan + scatter kernel (stable ranking of a
 * 4096-key tile by warp match, reorder in shared memory, coalesced runs out).  Passes whose digit
 * does not vary over the input are skipped (one OR/AND reduction decides), so int64 keys below 2^32
 * cost 4 passes, not 8.  Algorithmic traffic per executed pass: 8 (histogram) + 12 + 12 bytes/row.
 */
#include <cuda_runtime.h>
#include <stdint.h>
#include <cstring>
#include <vector>
#include "gg_engine.h"

#define SORT_THREADS 256
#define SORT_ITEMS   16
#define SORT_TILE    (SORT_THREADS * SORT_ITEMS)
#define SORT_WARPS   (SORT_THREADS / 32)
#define FULL 0xffffffffu

enum { KEYMODE_VALUE = 0, KEYMODE_NULLBIT = 1, KEYMODE_DEADBIT = 2 };

__device__ __forceinline__ uint64_t bswap64(uint64_t v)
{
	uint32_t lo = (uint32_t) v, hi = (uint32_t) (v >> 32);
	return ((uint64_t) __byte_perm(lo, 0, 0x0123) << 32) | __byte_perm(hi, 0, 0x0123);
}

/* order-preserving radix key of one Datum */
__device__ __forceinline__ uint64_t radix_key(int64_t v, int typid, int desc)
{
	uint64_t k;
	switch (typid)
	{
		case GG_INT4OID: case GG_DATEOID:
			k = (uint64_t) (int64_t) (int32_t) v ^ 0x8000000000000000ull;
			break;
		case GG_FLOAT8OID:
		{
			double d = __longlong_as_double(v);
			if (d != d) k = ~0ull;
			else
			{
				if (d == 0.0) v = 0;
				k = (uint64_t) v;
				k = (k >> 63) ? ~k : (k ^ 0x8000000000000000ull);
			}
			break;
		}
		case GG_BPCHAROID: case GG_VARCHAROID: case GG_TEXTOID:
			k = bswap64((uint64_t) v);
			break;
		default:
			k = (uint64_t) v ^ 0x8000000000000000ull;
			break;
	}
	return desc ? ~k : k;
}

/* keys of the current order: kout[i] = key(rows[perm[i]][col]); also OR / AND over all keys (which bits vary).
 * datumrows: the rows are GG_FMT_DATUMROWS (ncols + 1 words: NULL mask, columns), as a row-producing scan or a receiving
 * Motion leaves them on the device; KEYMODE_DEADBIT keys the slots a sending kernel claimed and did not fill (bit 63 of the
 * mask word) behind everything else and counts them into orand[2]. */
__global__ void __launch_bounds__(256)
gg_sort_keys_kernel(const int64_t *rows, const uint8_t *nulls, int ncols, int col, int typid, int desc, int nulls_first,
                    int mode, const uint32_t *perm, uint64_t n, uint64_t *kout, unsigned long long *orand, int datumrows)
{
	uint64_t vor = 0, vand = ~0ull;
	unsigned long long ndead = 0;
	for (uint64_t i = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; i < n; i += (uint64_t) gridDim.x * blockDim.x)
	{
		const uint64_t r = perm ? perm[i] : i;
		uint64_t k;
		if (datumrows)
		{
			const uint64_t mask = (uint64_t) rows[r * (uint64_t) (ncols + 1)];
			if (mode == KEYMODE_DEADBIT) { k = mask >> 63; ndead += k; }
			else
			{
				const bool isnull = (mask >> col) & 1;
				if (mode == KEYMODE_VALUE) k = isnull ? 0 : radix_key(rows[r * (uint64_t) (ncols + 1) + 1 + col], typid, desc);
				else k = isnull ? (nulls_first ? 0 : 1) : (nulls_first ? 1 : 0);
			}
		}
		else
		{
			const bool isnull = nulls && nulls[r * ncols + col];
			if (mode == KEYMODE_VALUE) k = isnull ? 0 : radix_key(rows[r * ncols + col], typid, desc);
			else k = isnull ? (nulls_first ? 0 : 1) : (nulls_first ? 1 : 0);
		}
		kout[i] = k;
		vor |= k; vand &= k;
	}
	if (mode == KEYMODE_DEADBIT)
	{
		for (int o = 16; o > 0; o >>= 1) ndead += __shfl_xor_sync(FULL, ndead, o);
		if ((threadIdx.x & 31) == 0 && ndead) atomicAdd(&orand[2], ndead);
	}
	for (int o = 16; o > 0; o >>= 1)
	{
		vor |= __shfl_xor_sync(FULL, vor, o);
		vand &= __shfl_xor_sync(FULL, vand, o);
	}
	if ((threadIdx.x & 31) == 0)
	{
		atomicOr(&orand[0], (unsigned long long) vor);
		atomicAnd(&orand[1], (unsigned long long) vand);
	}
}

__global__ void __launch_bounds__(256)
gg_sort_iota_kernel(uint32_t *perm, uint64_t n)
{
	for (uint64_t i = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; i < n; i += (uint64_t) gridDim.x * blockDim.x)
		perm[i] = (uint32_t) i;
}

/* per-tile digit counts, digit-major: hist[d * ntiles + tile] */
__global__ void __launch_bounds__(SORT_THREADS)
gg_sort_hist_kernel(const uint64_t *keys, uint64_t n, int shift, uint32_t *hist, uint32_t ntiles)
{
	__shared__ uint32_t cnt[256];
	const uint32_t tile = blockIdx.x;
	cnt[threadIdx.x] = 0;
	__syncthreads();
	const uint64_t base = (uint64_t) tile * SORT_TILE;
#pragma unroll 4
	for (int i = 0; i < SORT_ITEMS; i++)
	{
		const uint64_t e = base + (uint64_t) i * SORT_THREADS + threadIdx.x;
		if (e < n) atomicAdd(&cnt[(keys[e] >> shift) & 0xFF], 1u);
	}
	__syncthreads();
	hist[(uint64_t) threadIdx.x * ntiles + tile] = cnt[threadIdx.x];
}

/* exclusive scan of m counters, three phases over chunks of 4096 */
__device__ __forceinline__ uint32_t block_exclusive_scan_256(uint32_t v, uint32_t *warpsums /* [8] shared */, uint32_t &total)
{
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	uint32_t inc = v;
	for (int o = 1; o < 32; o <<= 1)
	{
		uint32_t t = __shfl_up_sync(FULL, inc, o);
		if (lane >= o) inc += t;
	}
	if (lane == 31) warpsums[warp] = inc;
	__syncthreads();
	uint32_t pre = 0, tot = 0;
	for (int w = 0; w < SORT_WARPS; w++)
	{
		uint32_t s = warpsums[w];
		if (w < warp) pre += s;
		tot += s;
	}
	__syncthreads();
	total = tot;
	return pre + inc - v;
}

__global__ void __launch_bounds__(256)
gg_scan_sums_kernel(const uint32_t *x, uint64_t m, uint32_t *sums)
{
	__shared__ uint32_t ws[8];
	const uint64_t base = (uint64_t) blockIdx.x * 4096 + (uint64_t) threadIdx.x * 16;
	uint32_t s = 0;
	for (int i = 0; i < 16; i++) if (base + i < m) s += x[base + i];
	uint32_t tot;
	block_exclusive_scan_256(s, ws, tot);
	if (threadIdx.x == 0) sums[blockIdx.x] = tot;
}

__global__ void __launch_bounds__(256)
gg_scan_top_kernel(uint32_t *sums, uint32_t nblk)
{
	__shared__ uint32_t ws[8];
	__shared__ uint32_t carry;
	if (threadIdx.x == 0) carry = 0;
	__syncthreads();
	for (uint32_t b = 0; b < nblk; b += 256)
	{
		const uint32_t i = b + threadIdx.x;
		const uint32_t v = i < nblk ? sums[i] : 0;
		uint32_t tot;
		const uint32_t ex = block_exclusive_scan_256(v, ws, tot);
		if (i < nblk) sums[i] = carry + ex;
		__syncthreads();
		if (threadIdx.x == 0) carry += tot;
		__syncthreads();
	}
}

__global__ void __launch_bounds__(256)
gg_scan_apply_kernel(uint32_t *x, uint64_t m, const uint32_t *sums)
{
	__shared__ uint32_t ws[8];
	const uint64_t base = (uint64_t) blockIdx.x * 4096 + (uint64_t) threadIdx.x * 16;
	uint32_t v[16], s = 0;
	for (int i = 0; i < 16; i++) { v[i] = base + i < m ? x[base + i] : 0; s += v[i]; }
	uint32_t tot;
	uint32_t run = sums[blockIdx.x] + block_exclusive_scan_256(s, ws, tot);
	for (int i = 0; i < 16; i++)
	{
		if (base + i < m) x[base + i] = run;
		run += v[i];
	}
}

/* stable scatter of one tile by the digit at `shift` */
__global__ void __launch_bounds__(SORT_THREADS)
gg_sort_scatter_kernel(const uint64_t *kin, const uint32_t *vin, uint64_t *kout, uint32_t *vout, uint64_t n, int shift,
                       const uint32_t *offsets /* scanned hist */, uint32_t ntiles)
{
	extern __shared__ __align__(16) uint8_t sm[];
	uint64_t *skey = (uint64_t *) sm;                                   /* [SORT_TILE] */
	uint32_t *sval = (uint32_t *) (sm + (size_t) SORT_TILE * 8);         /* [SORT_TILE] */
	uint32_t *cnt = sval + SORT_TILE;                                   /* [SORT_WARPS][256] */
	uint32_t *dstart = cnt + SORT_WARPS * 256;                          /* [256] */
	uint32_t *goff = dstart + 256;                                      /* [256] */
	__shared__ uint32_t ws[8];

	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const uint32_t tile = blockIdx.x;
	const uint64_t base = (uint64_t) tile * SORT_TILE;
	const uint32_t count = (uint32_t) (n - base < SORT_TILE ? n - base : SORT_TILE);

	for (int w = 0; w < SORT_WARPS; w++) cnt[w * 256 + threadIdx.x] = 0;
	goff[threadIdx.x] = offsets[(uint64_t) threadIdx.x * ntiles + tile];
	__syncthreads();

	/* element order inside the tile: (warp, item, lane) — every warp ranks its own 512 consecutive keys */
	uint64_t key[SORT_ITEMS];
	uint32_t val[SORT_ITEMS];
	uint32_t local[SORT_ITEMS];
	const uint32_t lt = (1u << lane) - 1;
	uint32_t *mycnt = cnt + warp * 256;
#pragma unroll
	for (int i = 0; i < SORT_ITEMS; i++)
	{
		const uint32_t j = (uint32_t) warp * (32 * SORT_ITEMS) + (uint32_t) i * 32 + lane;
		const bool valid = j < count;
		key[i] = valid ? kin[base + j] : 0;
		val[i] = valid ? vin[base + j] : 0;
	}
#pragma unroll
	for (int i = 0; i < SORT_ITEMS; i++)
	{
		const uint32_t j = (uint32_t) warp * (32 * SORT_ITEMS) + (uint32_t) i * 32 + lane;
		const bool valid = j < count;
		const uint32_t d = valid ? (uint32_t) ((key[i] >> shift) & 0xFF) : 0x100u + lane;
		const uint32_t peers = __match_any_sync(FULL, d);
		const int leader = __ffs(peers) - 1;
		uint32_t old = 0;
		if (lane == leader && valid)
		{
			old = mycnt[d];
			mycnt[d] = old + __popc(peers);
		}
		old = __shfl_sync(FULL, old, leader);
		local[i] = old + __popc(peers & lt);
		__syncwarp();
	}
	__syncthreads();

	/* digit t: exclusive prefix over warps, then over digits */
	{
		uint32_t run = 0;
		for (int w = 0; w < SORT_WARPS; w++)
		{
			uint32_t c = cnt[w * 256 + threadIdx.x];
			cnt[w * 256 + threadIdx.x] = run;
			run += c;
		}
		uint32_t tot;
		const uint32_t ex = block_exclusive_scan_256(run, ws, tot);
		dstart[threadIdx.x] = ex;
	}
	__syncthreads();

#pragma unroll
	for (int i = 0; i < SORT_ITEMS; i++)
	{
		const uint32_t j = (uint32_t) warp * (32 * SORT_ITEMS) + (uint32_t) i * 32 + lane;
		if (j < count)
		{
			const uint32_t d = (uint32_t) ((key[i] >> shift) & 0xFF);
			const uint32_t pos = dstart[d] + mycnt[d] + local[i];
			skey[pos] = key[i];
			sval[pos] = val[i];
		}
	}
	__syncthreads();

	for (uint32_t j = threadIdx.x; j < count; j += SORT_THREADS)
	{
		const uint64_t k = skey[j];
		const uint32_t d = (uint32_t) ((k >> shift) & 0xFF);
		const uint64_t dst = (uint64_t) goff[d] + (j - dstart[d]);
		kout[dst] = k;
		vout[dst] = sval[j];
	}
}

__global__ void __launch_bounds__(256)
gg_sort_widen_kernel(const uint32_t *perm, uint64_t *out, uint64_t n)
{
	for (uint64_t i = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; i < n; i += (uint64_t) gridDim.x * blockDim.x)
		out[i] = perm[i];
}

/* rows in sorted order: out row i = in row perm[i], W words each; a warp moves a row's words with consecutive lanes */
__global__ void __launch_bounds__(256)
gg_sort_gather_rows_kernel(const uint64_t *rows, const uint32_t *perm, uint64_t n, int W, uint64_t *out)
{
	const uint64_t total = n * (uint64_t) W;
	for (uint64_t i = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; i < total; i += (uint64_t) gridDim.x * blockDim.x)
	{
		const uint64_t r = i / (uint64_t) W;
		const uint32_t w = (uint32_t) (i - r * (uint64_t) W);
		out[i] = rows[(uint64_t) perm[r] * (uint64_t) W + w];
	}
}

/* ---- bounded Sort (tuplesort_set_bound, tuplesort_mk.c:1000): MSB-first radix select on the comparator's leading part ----
 * The prefix of a row is (dead digit, first key's NULL digit) in hi and the first key's radix key in key: the most significant
 * digits of exactly the order sort_device produces.  A row whose prefix is above the threshold has at least `bound` rows strictly
 * before it in that order, so it is not among the first `bound`. */
__global__ void __launch_bounds__(256)
gg_topn_prefix_kernel(const int64_t *rows, const uint8_t *nulls, int ncols, int col, int typid, int desc, int nulls_first,
                      uint64_t n, uint64_t *kout, uint8_t *hout, unsigned long long *orand /* key or, key and, ndead, hi or, hi and */,
                      int datumrows)
{
	uint64_t vor = 0, vand = ~0ull;
	uint32_t hor = 0, hand = 0xFF;
	unsigned long long ndead = 0;
	for (uint64_t i = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; i < n; i += (uint64_t) gridDim.x * blockDim.x)
	{
		bool isnull, dead = false;
		int64_t v;
		if (datumrows)
		{
			const uint64_t mask = (uint64_t) rows[i * (uint64_t) (ncols + 1)];
			dead = mask >> 63;
			isnull = (mask >> col) & 1;
			v = rows[i * (uint64_t) (ncols + 1) + 1 + col];
		}
		else
		{
			isnull = nulls && nulls[i * ncols + col];
			v = rows[i * ncols + col];
		}
		const uint64_t k = isnull ? 0 : radix_key(v, typid, desc);
		const uint32_t nd = (datumrows || nulls) ? (isnull ? (nulls_first ? 0 : 1) : (nulls_first ? 1 : 0)) : 0;
		const uint32_t h = ((uint32_t) dead << 1) | nd;
		kout[i] = k; hout[i] = (uint8_t) h;
		vor |= k; vand &= k; hor |= h; hand &= h;
		ndead += dead;
	}
	for (int o = 16; o > 0; o >>= 1)
	{
		vor |= __shfl_xor_sync(FULL, vor, o);
		vand &= __shfl_xor_sync(FULL, vand, o);
		hor |= __shfl_xor_sync(FULL, hor, o);
		hand &= __shfl_xor_sync(FULL, hand, o);
		ndead += __shfl_xor_sync(FULL, ndead, o);
	}
	if ((threadIdx.x & 31) == 0)
	{
		atomicOr(&orand[0], (unsigned long long) vor);
		atomicAnd(&orand[1], (unsigned long long) vand);
		if (ndead) atomicAdd(&orand[2], ndead);
		atomicOr(&orand[3], (unsigned long long) hor);
		atomicAnd(&orand[4], (unsigned long long) hand);
	}
}

/* the digit of a prefix: 8 = hi, 7..0 = a byte of key */
__device__ __forceinline__ uint32_t topn_digit(uint8_t h, uint64_t k, int digit)
{
	return digit == 8 ? h : (uint32_t) ((k >> (8 * digit)) & 0xFF);
}

/* histogram of one digit over the rows whose already-chosen digits equal the threshold's; shared bins, one global add per bin */
__global__ void __launch_bounds__(256)
gg_topn_hist_kernel(const uint64_t *key, const uint8_t *hi, uint64_t n, int digit, uint32_t hmask, uint32_t th_hi,
                    uint64_t kmask, uint64_t th_key, uint32_t *hist)
{
	__shared__ uint32_t cnt[256];
	cnt[threadIdx.x] = 0;
	__syncthreads();
	for (uint64_t i = blockIdx.x * (uint64_t) blockDim.x + threadIdx.x; i < n; i += (uint64_t) gridDim.x * blockDim.x)
	{
		const uint8_t h = hi[i];
		const uint64_t k = key[i];
		if (((h ^ th_hi) & hmask) == 0 && ((k ^ th_key) & kmask) == 0) atomicAdd(&cnt[topn_digit(h, k, digit)], 1u);
	}
	__syncthreads();
	if (cnt[threadIdx.x]) atomicAdd(&hist[threadIdx.x], cnt[threadIdx.x]);
}

__device__ __forceinline__ bool topn_survives(uint8_t h, uint64_t k, uint32_t hmask, uint32_t th_hi, uint64_t kmask, uint64_t th_key)
{
	const uint32_t hh = h & hmask;
	return hh < th_hi || (hh == th_hi && (k & kmask) <= th_key);
}

/* survivors per tile of SORT_TILE rows (thread t owns rows t*16 .. t*16+15 of its tile); cnt[ntiles] stays 0 for the total */
__global__ void __launch_bounds__(SORT_THREADS)
gg_topn_count_kernel(const uint64_t *key, const uint8_t *hi, uint64_t n, uint32_t hmask, uint32_t th_hi, uint64_t kmask,
                     uint64_t th_key, uint32_t *cnt)
{
	__shared__ uint32_t ws[8];
	const uint64_t base = (uint64_t) blockIdx.x * SORT_TILE + (uint64_t) threadIdx.x * SORT_ITEMS;
	uint32_t s = 0;
	for (int i = 0; i < SORT_ITEMS; i++)
		if (base + i < n) s += topn_survives(hi[base + i], key[base + i], hmask, th_hi, kmask, th_key);
	uint32_t tot;
	block_exclusive_scan_256(s, ws, tot);
	if (threadIdx.x == 0) cnt[blockIdx.x] = tot;
}

/* the survivors' row numbers in input order: out[off[tile] + rank within the tile] */
__global__ void __launch_bounds__(SORT_THREADS)
gg_topn_compact_kernel(const uint64_t *key, const uint8_t *hi, uint64_t n, uint32_t hmask, uint32_t th_hi, uint64_t kmask,
                       uint64_t th_key, const uint32_t *off, uint32_t *out)
{
	__shared__ uint32_t ws[8];
	const uint64_t base = (uint64_t) blockIdx.x * SORT_TILE + (uint64_t) threadIdx.x * SORT_ITEMS;
	uint32_t flags = 0, s = 0;
	for (int i = 0; i < SORT_ITEMS; i++)
		if (base + i < n && topn_survives(hi[base + i], key[base + i], hmask, th_hi, kmask, th_key)) { flags |= 1u << i; s++; }
	uint32_t tot;
	uint32_t pos = off[blockIdx.x] + block_exclusive_scan_256(s, ws, tot);
	for (int i = 0; i < SORT_ITEMS; i++)
		if ((flags >> i) & 1) out[pos++] = (uint32_t) (base + i);
}

/* ===================================================================================== */

static bool sort_type_ok(int32_t t)
{
	switch (t)
	{
		case GG_INT4OID: case GG_INT8OID: case GG_DATEOID: case GG_TIMESTAMPOID: case GG_FLOAT8OID:
		case GG_BPCHAROID: case GG_VARCHAROID: case GG_TEXTOID: case GG_BOOLOID:
			return true;
	}
	return false;
}

struct SortScratch {                      /* carved out of one allocation the engine keeps (grown on demand) */
	uint64_t *k[2] = { nullptr, nullptr };
	uint32_t *v[2] = { nullptr, nullptr };
	uint32_t *hist = nullptr, *sums = nullptr;
	unsigned long long *orand = nullptr;
};

/* sort rows resident on the device; dev_perm receives n uint32 row numbers in sorted order.
 * passes_out (optional): radix passes executed (for the traffic model).
 * perm_given: dev_perm already holds the n row numbers to sort (ascending: a subset of the rows, in input order), not 0..n-1. */
static int sort_device(gg_engine *e, const gg_sortkey *keys, int nkeys, int ncols, const int64_t *d_rows,
                       const uint8_t *d_nulls, uint64_t n, uint32_t *dev_perm, int *passes_out,
                       bool datumrows = false, uint64_t *ndead_out = nullptr, bool perm_given = false)
{
	if (n >= (1ull << 32)) { gg_set_error("sort of %llu rows: row numbers are 32-bit", (unsigned long long) n); return GG_ERR_UNSUPPORTED; }
	for (int k = 0; k < nkeys; k++)
	{
		if (keys[k].col < 0 || keys[k].col >= ncols) { gg_set_error("sort key %d: column %d out of range", k, keys[k].col); return GG_ERR_ARG; }
		if (!sort_type_ok(keys[k].typid)) { gg_set_error("sort key %d: type %d not supported on the GPU path", k, keys[k].typid); return GG_ERR_UNSUPPORTED; }
	}
	cudaStream_t st = e->stream;
	int passes = 0;
	if (passes_out) *passes_out = 0;
	if (n == 0) return GG_OK;
	const uint32_t ntiles = (uint32_t) ((n + SORT_TILE - 1) / SORT_TILE);
	const uint64_t m = (uint64_t) ntiles * 256;
	const uint32_t nblk = (uint32_t) ((m + 4095) / 4096);
	const int grid1d = e->sm_count * 8;
	SortScratch s;
	{
		auto up = [](size_t x) { return (x + 255) & ~(size_t) 255; };
		const size_t need = 2 * up(n * 8) + up(n * 4) + up(m * 4) + up((size_t) nblk * 4) + 256;
		if (e->sort_scratch_bytes < need)
		{
			GG_CUDA(cudaStreamSynchronize(st));
			cudaFree(e->sort_scratch);
			e->sort_scratch = nullptr; e->sort_scratch_bytes = 0;
			cudaError_t ce = cudaMalloc(&e->sort_scratch, need);
			if (ce != cudaSuccess) { cudaGetLastError(); gg_set_error("sort scratch of %zu bytes does not fit in device memory", need); return GG_ERR_NOMEM; }
			e->sort_scratch_bytes = need;
		}
		uint8_t *b = (uint8_t *) e->sort_scratch;
		s.k[0] = (uint64_t *) b; b += up(n * 8);
		s.k[1] = (uint64_t *) b; b += up(n * 8);
		s.v[1] = (uint32_t *) b; b += up(n * 4);
		s.hist = (uint32_t *) b; b += up(m * 4);
		s.sums = (uint32_t *) b; b += up((size_t) nblk * 4);
		s.orand = (unsigned long long *) b;
	}
	const size_t smem = (size_t) SORT_TILE * 12 + (SORT_WARPS * 256 + 512) * 4;
	GG_CUDA(cudaFuncSetAttribute(gg_sort_scatter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem));

	/* the permutation ping-pongs between dev_perm and s.v[1]; `cur` says where the current order lives */
	uint32_t *vbuf[2] = { dev_perm, s.v[1] };
	int cur = 0, kcur = 0;
	if (!perm_given)
	{
		gg_sort_iota_kernel<<<grid1d, 256, 0, st>>>(vbuf[0], n);
		e->launches++;
	}
	bool first = !perm_given;
	/* least significant first: the last sort column's value, its NULL digit, ..., the first column's; for datum rows one
	 * more digit on top puts the dead slots behind every row */
	for (int kc = nkeys - 1; kc >= (datumrows ? -1 : 0); kc--)
	{
		for (int mode = kc < 0 ? KEYMODE_DEADBIT : KEYMODE_VALUE; mode <= (kc < 0 ? KEYMODE_DEADBIT : KEYMODE_NULLBIT); mode++)
		{
			if (mode == KEYMODE_NULLBIT && !d_nulls && !datumrows) break;
			const gg_sortkey &K = keys[kc < 0 ? 0 : kc];
			const unsigned long long init[3] = { 0ull, ~0ull, 0ull };
			GG_CUDA(cudaMemcpyAsync(s.orand, init, 24, cudaMemcpyHostToDevice, st));
			gg_sort_keys_kernel<<<grid1d, 256, 0, st>>>(d_rows, d_nulls, ncols, K.col, K.typid, K.desc,
			                                            K.nulls_first, mode, first ? nullptr : vbuf[cur], n, s.k[kcur], s.orand, datumrows ? 1 : 0);
			GG_CUDA(cudaGetLastError());
			e->launches++;
			unsigned long long oa[3];
			GG_CUDA(cudaMemcpyAsync(oa, s.orand, 24, cudaMemcpyDeviceToHost, st));
			GG_CUDA(cudaStreamSynchronize(st));
			if (mode == KEYMODE_DEADBIT && ndead_out) *ndead_out = oa[2];
			const uint64_t varying = oa[0] ^ oa[1];          /* bits that are not the same in every key */
			for (int byte = 0; byte < 8; byte++)
			{
				if (!((varying >> (8 * byte)) & 0xFF)) continue;
				const int shift = 8 * byte;
				gg_sort_hist_kernel<<<ntiles, SORT_THREADS, 0, st>>>(s.k[kcur], n, shift, s.hist, ntiles);
				gg_scan_sums_kernel<<<nblk, 256, 0, st>>>(s.hist, m, s.sums);
				gg_scan_top_kernel<<<1, 256, 0, st>>>(s.sums, nblk);
				gg_scan_apply_kernel<<<nblk, 256, 0, st>>>(s.hist, m, s.sums);
				gg_sort_scatter_kernel<<<ntiles, SORT_THREADS, smem, st>>>(s.k[kcur], vbuf[cur], s.k[kcur ^ 1], vbuf[cur ^ 1], n, shift,
				                                                          s.hist, ntiles);
				GG_CUDA(cudaGetLastError());
				e->launches += 5;
				kcur ^= 1; cur ^= 1;
				passes++;
				first = false;
			}
		}
	}
	if (cur != 0)
		GG_CUDA(cudaMemcpyAsync(dev_perm, vbuf[1], n * 4, cudaMemcpyDeviceToDevice, st));
	GG_CUDA(cudaStreamSynchronize(st));
	if (passes_out) *passes_out = passes;
	return GG_OK;
}

/* Whether a bound pays for the selection: the prefix, histogram and compaction passes cost about two radix passes over all
 * rows, and the survivors (up to twice the bound, more under a coarse first digit) are sorted through their row numbers.  On an
 * H100 at 10^8 rows a bound of n/2 was faster than the full sort for an int8 key and slower for a float8 key, while 1 % of n was
 * 4.7x faster for both (DESIGN §4.4), so a bound above n/4 sorts everything. */
static bool topn_worth_selecting(uint64_t bound, uint64_t n) { return bound <= n / 4; }

/* Radix select for the first `bound` rows of the order sort_device gives (bound < n): *d_surv (cudaMalloc'd, the caller frees)
 * receives the *nsurv rows whose comparator prefix is at or below the threshold, in input order — every row among the first
 * `bound` is one of them.  *d_surv == nullptr: bound >= live rows, nothing was selected.  *ndead: dead slots of datum rows;
 * *passes: histogram passes run. */
static int topn_select(gg_engine *e, const gg_sortkey &K, int ncols, const int64_t *d_rows, const uint8_t *d_nulls, uint64_t n,
                       uint64_t bound, bool datumrows, uint32_t **d_surv, uint64_t *nsurv, uint64_t *ndead, int *passes)
{
	cudaStream_t st = e->stream;
	const uint32_t ntiles = (uint32_t) ((n + SORT_TILE - 1) / SORT_TILE);
	const uint64_t m = (uint64_t) ntiles + 1;                     /* per-tile counts, then the total */
	const uint32_t nblk = (uint32_t) ((m + 4095) / 4096);
	const uint64_t want_blocks = (n + 255) / 256;
	const int grid = (int) (want_blocks < (uint64_t) e->sm_count * 8 ? want_blocks : (uint64_t) e->sm_count * 8);
	auto up = [](size_t x) { return (x + 255) & ~(size_t) 255; };
	const size_t bytes = up(n * 8) + up(n) + up(m * 4) + up((size_t) nblk * 4) + up(256 * 4) + 64;
	*d_surv = nullptr; *nsurv = 0; *ndead = 0; *passes = 0;
	uint8_t *buf = nullptr;
	cudaError_t ce = cudaMalloc((void **) &buf, bytes);
	if (ce != cudaSuccess) { cudaGetLastError(); gg_set_error("bounded sort: scratch of %zu bytes does not fit in device memory", bytes); return GG_ERR_NOMEM; }
	uint8_t *b = buf;
	uint64_t *key = (uint64_t *) b; b += up(n * 8);
	uint8_t *hi = b; b += up(n);
	uint32_t *cnt = (uint32_t *) b; b += up(m * 4);
	uint32_t *sums = (uint32_t *) b; b += up((size_t) nblk * 4);
	uint32_t *hist = (uint32_t *) b; b += up(256 * 4);
	unsigned long long *orand = (unsigned long long *) b;
	int rc = GG_OK;
	uint32_t hmask = 0, th_hi = 0, total = 0;
	uint64_t kmask = 0, th_key = 0, want = bound, below = 0;
	{
		const unsigned long long init[5] = { 0ull, ~0ull, 0ull, 0ull, 0xFFull };
		unsigned long long oa[5];
		if ((ce = cudaMemcpyAsync(orand, init, sizeof init, cudaMemcpyHostToDevice, st)) != cudaSuccess) goto cuda_fail;
		gg_topn_prefix_kernel<<<grid, 256, 0, st>>>(d_rows, d_nulls, ncols, K.col, K.typid, K.desc, K.nulls_first, n, key, hi, orand,
		                                            datumrows ? 1 : 0);
		e->launches++;
		if ((ce = cudaGetLastError()) != cudaSuccess) goto cuda_fail;
		if ((ce = cudaMemcpyAsync(oa, orand, sizeof oa, cudaMemcpyDeviceToHost, st)) != cudaSuccess) goto cuda_fail;
		if ((ce = cudaStreamSynchronize(st)) != cudaSuccess) goto cuda_fail;
		*ndead = oa[2];
		if (bound >= n - oa[2]) { cudaFree(buf); return GG_OK; }   /* every live row is wanted */
		const uint64_t kvary = oa[0] ^ oa[1];
		const uint32_t hvary = (uint32_t) (oa[3] ^ oa[4]);
		if (!hvary) { hmask = 0xFF; th_hi = (uint32_t) oa[3]; }
		/* most significant digit first: hi, then the key's bytes from the top; digits that never vary are skipped */
		for (int digit = hvary ? 8 : 7; digit >= 0; digit--)
		{
			if (digit < 8 && !((kvary >> (8 * digit)) & 0xFF)) continue;
			uint32_t h[256];
			if ((ce = cudaMemsetAsync(hist, 0, 256 * 4, st)) != cudaSuccess) goto cuda_fail;
			gg_topn_hist_kernel<<<grid, 256, 0, st>>>(key, hi, n, digit, hmask, th_hi, kmask, th_key, hist);
			e->launches++;
			if ((ce = cudaGetLastError()) != cudaSuccess) goto cuda_fail;
			if ((ce = cudaMemcpyAsync(h, hist, sizeof h, cudaMemcpyDeviceToHost, st)) != cudaSuccess) goto cuda_fail;
			if ((ce = cudaStreamSynchronize(st)) != cudaSuccess) goto cuda_fail;
			(*passes)++;
			/* the bucket where the running count reaches the rank still wanted */
			uint64_t cum = 0;
			uint32_t bk = 0;
			for (; bk < 255 && cum + h[bk] < want; bk++) cum += h[bk];
			below += cum; want -= cum;
			if (digit == 8) { hmask = 0xFF; th_hi = bk; }
			else { kmask |= 0xFFull << (8 * digit); th_key |= (uint64_t) bk << (8 * digit); }
			if (below + h[bk] <= 2 * bound) break;                    /* few enough to sort */
		}
	}
	/* order-preserving compaction: survivors per tile, exclusive scan, then every tile writes its survivors in input order */
	if ((ce = cudaMemsetAsync(cnt, 0, m * 4, st)) != cudaSuccess) goto cuda_fail;
	gg_topn_count_kernel<<<ntiles, SORT_THREADS, 0, st>>>(key, hi, n, hmask, th_hi, kmask, th_key, cnt);
	gg_scan_sums_kernel<<<nblk, 256, 0, st>>>(cnt, m, sums);
	gg_scan_top_kernel<<<1, 256, 0, st>>>(sums, nblk);
	gg_scan_apply_kernel<<<nblk, 256, 0, st>>>(cnt, m, sums);
	e->launches += 4;
	if ((ce = cudaGetLastError()) != cudaSuccess) goto cuda_fail;
	if ((ce = cudaMemcpyAsync(&total, cnt + ntiles, 4, cudaMemcpyDeviceToHost, st)) != cudaSuccess) goto cuda_fail;
	if ((ce = cudaStreamSynchronize(st)) != cudaSuccess) goto cuda_fail;
	if ((ce = cudaMalloc((void **) d_surv, (size_t) (total ? total : 1) * 4)) != cudaSuccess)
	{
		cudaGetLastError(); *d_surv = nullptr; cudaFree(buf);
		gg_set_error("bounded sort: %u row numbers do not fit in device memory", total);
		return GG_ERR_NOMEM;
	}
	gg_topn_compact_kernel<<<ntiles, SORT_THREADS, 0, st>>>(key, hi, n, hmask, th_hi, kmask, th_key, cnt, *d_surv);
	e->launches++;
	if ((ce = cudaGetLastError()) != cudaSuccess) goto cuda_fail;
	if ((ce = cudaStreamSynchronize(st)) != cudaSuccess) goto cuda_fail;
	*nsurv = total;
	cudaFree(buf);
	return rc;
cuda_fail:
	cudaFree(buf); cudaFree(*d_surv); *d_surv = nullptr;
	return gg_cuda_fail(ce, "bounded sort");
}

/* dev_perm_out (cudaMalloc'd, the caller frees) = the first min(bound, live) row numbers of sort_device's order, *nout = that
 * count.  bound >= n, or one not worth a selection: the whole sort. */
static int sort_bounded(gg_engine *e, const gg_sortkey *keys, int nkeys, int ncols, const int64_t *d_rows, const uint8_t *d_nulls,
                        uint64_t n, uint64_t bound, bool datumrows, uint32_t **dev_perm_out, uint64_t *nout, int *passes_out)
{
	uint32_t *perm = nullptr;
	uint64_t nsort = n, ndead = 0;
	int sel_passes = 0, sort_passes = 0, rc;
	*dev_perm_out = nullptr; *nout = 0;
	if (passes_out) *passes_out = 0;
	if (n >= (1ull << 32)) { gg_set_error("sort of %llu rows: row numbers are 32-bit", (unsigned long long) n); return GG_ERR_UNSUPPORTED; }
	for (int k = 0; k < nkeys; k++)
	{
		if (keys[k].col < 0 || keys[k].col >= ncols) { gg_set_error("sort key %d: column %d out of range", k, keys[k].col); return GG_ERR_ARG; }
		if (!sort_type_ok(keys[k].typid)) { gg_set_error("sort key %d: type %d not supported on the GPU path", k, keys[k].typid); return GG_ERR_UNSUPPORTED; }
	}
	if (bound < n && topn_worth_selecting(bound, n))
	{
		rc = topn_select(e, keys[0], ncols, d_rows, d_nulls, n, bound, datumrows, &perm, &nsort, &ndead, &sel_passes);
		if (rc != GG_OK) return rc;
	}
	const bool selected = perm != nullptr;
	if (!selected)
	{
		cudaError_t ce = cudaMalloc((void **) &perm, n * 4);
		if (ce != cudaSuccess) { cudaGetLastError(); gg_set_error("sort: %llu row numbers do not fit in device memory", (unsigned long long) n); return GG_ERR_NOMEM; }
		nsort = n;
	}
	rc = sort_device(e, keys, nkeys, ncols, d_rows, d_nulls, nsort, perm, &sort_passes, datumrows, selected ? nullptr : &ndead, selected);
	if (rc != GG_OK) { cudaFree(perm); return rc; }
	const uint64_t live = n - ndead;
	*dev_perm_out = perm;
	*nout = bound < live ? bound : live;
	if (passes_out) *passes_out = sel_passes + sort_passes;
	return GG_OK;
}

/* datum rows: dev_out_rows = the first min(bound, live) rows of the sorted order */
static int sort_datumrows_bounded(gg_engine *e, const gg_sortkey *keys, int nkeys, int ncols, const void *dev_rows, uint64_t n,
                                  uint64_t bound, void *dev_out_rows, uint64_t *nout, int *passes)
{
	if (!e || !keys || nkeys < 1 || ncols < 1 || ncols > 63 || !nout || (n && bound && (!dev_rows || !dev_out_rows))) return GG_ERR_ARG;
	*nout = 0;
	if (passes) *passes = 0;
	if (n == 0 || bound == 0) return GG_OK;
	GG_CUDA(cudaSetDevice(e->device));
	GG_CUDA(cudaEventRecord(e->ev_start, e->stream));
	uint32_t *d_perm = nullptr;
	uint64_t cnt = 0;
	int rc = sort_bounded(e, keys, nkeys, ncols, (const int64_t *) dev_rows, nullptr, n, bound, true, &d_perm, &cnt, passes);
	if (rc != GG_OK) return rc;
	if (cnt)
	{
		gg_sort_gather_rows_kernel<<<e->sm_count * 8, 256, 0, e->stream>>>((const uint64_t *) dev_rows, d_perm, cnt, ncols + 1, (uint64_t *) dev_out_rows);
		e->launches++;
	}
	cudaError_t ce = cudaGetLastError();
	if (ce == cudaSuccess) ce = cudaEventRecord(e->ev_stop, e->stream);
	if (ce == cudaSuccess) ce = cudaStreamSynchronize(e->stream);
	cudaFree(d_perm);
	if (ce != cudaSuccess) return gg_cuda_fail(ce, "gg_sort_datumrows");
	e->timed = true;
	*nout = cnt;
	return GG_OK;
}

/* host rows: host_perm = the first min(bound, n) entries of the sorted order */
static int sort_rows_bounded(gg_engine *e, const gg_sortkey *keys, int nkeys, int ncols, const int64_t *host_rows,
                             const uint8_t *host_nulls, uint64_t n, uint64_t bound, uint64_t *host_perm, uint64_t *nperm)
{
	if (!e || !keys || nkeys < 1 || ncols < 1 || (n && bound && (!host_rows || !host_perm))) return GG_ERR_ARG;
	if (nperm) *nperm = 0;
	if (n == 0 || bound == 0) return GG_OK;
	GG_CUDA(cudaSetDevice(e->device));
	int64_t *d_rows = nullptr;
	uint8_t *d_nulls = nullptr;
	uint32_t *d_perm = nullptr;
	uint64_t *d_wide = nullptr;
	uint64_t cnt = 0;
	int rc = GG_OK;
	cudaError_t ce;
	bool anynull = false;
	if (host_nulls)
		for (uint64_t i = 0; i < n * (uint64_t) ncols && !anynull; i++) anynull = host_nulls[i] != 0;
	if ((ce = cudaMalloc((void **) &d_rows, n * ncols * 8)) != cudaSuccess) goto fail;
	if (anynull && (ce = cudaMalloc((void **) &d_nulls, n * ncols)) != cudaSuccess) goto fail;
	if ((ce = cudaMemcpyAsync(d_rows, host_rows, n * ncols * 8, cudaMemcpyHostToDevice, e->stream)) != cudaSuccess) goto fail;
	if (anynull && (ce = cudaMemcpyAsync(d_nulls, host_nulls, n * ncols, cudaMemcpyHostToDevice, e->stream)) != cudaSuccess) goto fail;
	rc = sort_bounded(e, keys, nkeys, ncols, d_rows, d_nulls, n, bound, false, &d_perm, &cnt, nullptr);
	if (rc == GG_OK)
	{
		if ((ce = cudaMalloc((void **) &d_wide, cnt * 8)) != cudaSuccess) goto fail;
		gg_sort_widen_kernel<<<e->sm_count * 4, 256, 0, e->stream>>>(d_perm, d_wide, cnt);
		e->launches++;
		if ((ce = cudaMemcpyAsync(host_perm, d_wide, cnt * 8, cudaMemcpyDeviceToHost, e->stream)) != cudaSuccess) goto fail;
		if ((ce = cudaStreamSynchronize(e->stream)) != cudaSuccess) goto fail;
		if (nperm) *nperm = cnt;
	}
	cudaFree(d_rows); cudaFree(d_nulls); cudaFree(d_perm); cudaFree(d_wide);
	return rc;
fail:
	cudaGetLastError();
	cudaFree(d_rows); cudaFree(d_nulls); cudaFree(d_perm); cudaFree(d_wide);
	return gg_cuda_fail(ce, "gg_sort_rows");
}

extern "C" {

int gg_sort_device(gg_engine *e, const gg_sortkey *keys, int nkeys, int ncols, const int64_t *dev_rows,
                   const uint8_t *dev_nulls, uint64_t n, uint32_t *dev_perm, int *passes)
{
	if (!e || !keys || nkeys < 1 || ncols < 1 || (n && (!dev_rows || !dev_perm))) return GG_ERR_ARG;
	GG_CUDA(cudaSetDevice(e->device));
	GG_CUDA(cudaEventRecord(e->ev_start, e->stream));
	int rc = sort_device(e, keys, nkeys, ncols, dev_rows, dev_nulls, n, dev_perm, passes);
	if (rc) return rc;
	GG_CUDA(cudaEventRecord(e->ev_stop, e->stream));
	e->timed = true;
	return GG_OK;
}

int gg_sort_datumrows(gg_engine *e, const gg_sortkey *keys, int nkeys, int ncols, const void *dev_rows, uint64_t n,
                      void *dev_out_rows, uint64_t *nlive, int *passes)
{
	return sort_datumrows_bounded(e, keys, nkeys, ncols, dev_rows, n, UINT64_MAX, dev_out_rows, nlive, passes);
}

int gg_sort_datumrows_bounded(gg_engine *e, const gg_sortkey *keys, int nkeys, int ncols, const void *dev_rows, uint64_t n,
                              uint64_t bound, void *dev_out_rows, uint64_t *nout, int *passes)
{
	return sort_datumrows_bounded(e, keys, nkeys, ncols, dev_rows, n, bound, dev_out_rows, nout, passes);
}

int gg_sort_rows(gg_engine *e, const gg_sortkey *keys, int nkeys, int ncols,
                 const int64_t *host_rows, const uint8_t *host_nulls, uint64_t n, uint64_t *host_perm)
{
	return sort_rows_bounded(e, keys, nkeys, ncols, host_rows, host_nulls, n, UINT64_MAX, host_perm, nullptr);
}

int gg_sort_rows_bounded(gg_engine *e, const gg_sortkey *keys, int nkeys, int ncols, const int64_t *host_rows,
                         const uint8_t *host_nulls, uint64_t n, uint64_t bound, uint64_t *host_perm, uint64_t *nperm)
{
	if (!nperm) return GG_ERR_ARG;
	return sort_rows_bounded(e, keys, nkeys, ncols, host_rows, host_nulls, n, bound, host_perm, nperm);
}

}  /* extern "C" */
