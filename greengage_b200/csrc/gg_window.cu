/*
 * gg_window.cu — WindowAgg over datum rows on the device (include/ggb200.h gg_window_*; nodeWindowAgg.c, windowfuncs.c).
 *
 * The input arrives sorted (partitions, then peer groups, are runs of rows).  Every supported frame is a contiguous range of
 * rows [head, tail] of the row's partition that contains the row (gg_window.h), so every result is a function of a few scans:
 *
 *   1. live    the live slots counted per tile; only when some slot is dead, the inclusive scan of the live flags and a
 *              compaction: idx[j] = the slot of the j-th live row (input order); else row j is slot j
 *   2. heads   for each live row, whether it starts a partition / a peer group (execTuplesMatch against its predecessor on
 *              normalised keys), packed into one word; its inclusive scan numbers the partitions (high half) and the peer groups
 *              (low half); the starts of both are scattered by number, so each row finds [ps, pe) and [gs, ge) by two loads
 *   3. aggs    count(x) and the int sums: global inclusive prefix sums, read as P[tail] - P[head - 1] (exact: int64 arithmetic
 *              wraps and the true result fits); float8 sum / avg and min / max: a segmented scan (restarting at each partition,
 *              or at each peer group for RANGE CURRENT ROW .. CURRENT ROW), forward when the frame starts at the partition and
 *              read at the tail, backward when it ends at the partition's end and read at the head
 *   4. write   one output row per live row: the input's words, then one word per function; ranks and ntile from the bounds,
 *              lag / lead / first / last / nth_value as one gather each
 *
 * Each scan is tile reduce -> carry scan in one block -> tile apply, over tiles of WIN_TILE elements with a fixed reduction tree:
 * float8 sums are bit-identical run to run, and a result that is infinite (or NaN) with no non-finite input in its frame raises
 * GG_ERR_FLOAT_OVERFLOW, as float8pl's CHECKFLOATVAL does for the reference's left-to-right sum (DESIGN §4.10).  No atomics
 * decide where anything goes; one atomicOr reports an overflow.
 */
#include <cuda_runtime.h>
#include <stdint.h>
#include <cstring>
#include "gg_pipeline.h"
#include "gg_aggfinal.h"
#include "gg_window.h"

#define WIN_THREADS 256
#define WIN_ITEMS   8
#define WIN_TILE    (WIN_THREADS * WIN_ITEMS)
#define WIN_CARRY_THREADS 1024

/* one scan element: a 64-bit value, and for the segmented scans the flags HAS (a non-NULL value) and HEAD (a segment starts) */
struct WE {
	unsigned long long v;
	uint32_t f;
};
#define WE_HAS  1u
#define WE_HEAD 2u

enum { WOP_ADD = 0, WOP_SUM_F8, WOP_MIN_I, WOP_MAX_I, WOP_MIN_F8, WOP_MAX_F8 };
enum { LD_LIVE = 0, LD_ARRAY, LD_COUNT, LD_ISUM, LD_SEG };

/* where a scan reads its elements: scan position k is row r = k (forward) or m - 1 - k (backward), and the result of position
 * k is stored at row r */
struct WLoad {
	int kind, col, isf8, seg, rev;
	uint32_t W;
	uint64_t m;
	const unsigned long long *rows;
	const uint32_t *idx;
	const unsigned long long *arr;      /* LD_ARRAY: the words; LD_SEG: the packed partition / peer numbers */
};

__device__ __forceinline__ double u2d(unsigned long long u) { return __longlong_as_double((long long) u); }
__device__ __forceinline__ unsigned long long d2u(double d) { return (unsigned long long) __double_as_longlong(d); }

/* float8_cmp_internal (float.c:964): NaN equals NaN and sorts above everything else; -0 = +0 */
__device__ __forceinline__ int f8cmp(double a, double b)
{
	if (isnan(a)) return isnan(b) ? 0 : 1;
	if (isnan(b)) return -1;
	return a > b ? 1 : (a < b ? -1 : 0);
}

/* a then b in scan order.  float8larger / float8smaller keep the later row of a tie (float.c:680-700): forward that is b,
 * backward a */
__device__ __forceinline__ unsigned long long agg2(int op, int rev, unsigned long long a, unsigned long long b)
{
	switch (op)
	{
		case WOP_SUM_F8: return d2u(u2d(a) + u2d(b));
		case WOP_MIN_I: return (long long) a < (long long) b ? a : b;
		case WOP_MAX_I: return (long long) a > (long long) b ? a : b;
		case WOP_MIN_F8: return rev ? (f8cmp(u2d(b), u2d(a)) < 0 ? b : a) : (f8cmp(u2d(a), u2d(b)) < 0 ? a : b);
		default: return rev ? (f8cmp(u2d(b), u2d(a)) > 0 ? b : a) : (f8cmp(u2d(a), u2d(b)) > 0 ? a : b);
	}
}

/* the scan operator: a plain sum, or the segmented form of a strict aggregate (a segment head restarts it) */
__device__ __forceinline__ WE wcombine(int op, int rev, WE a, WE b)
{
	WE r;
	if (op == WOP_ADD) { r.v = a.v + b.v; r.f = 0; return r; }
	if (b.f & WE_HEAD) return b;
	r.f = (a.f & WE_HEAD) | ((a.f | b.f) & WE_HAS);
	r.v = !(a.f & WE_HAS) ? b.v : (!(b.f & WE_HAS) ? a.v : agg2(op, rev, a.v, b.v));
	return r;
}

__device__ __forceinline__ uint32_t seg_no(unsigned long long hp, int seg) { return seg == 0 ? (uint32_t) (hp >> 32) : (uint32_t) hp; }

/* the slot of live row j: idx == nullptr when every slot is live */
__device__ __forceinline__ uint64_t slot_of(const uint32_t *idx, uint64_t j) { return idx ? (uint64_t) idx[j] : j; }

__device__ __forceinline__ WE wload(const WLoad &L, uint64_t r)
{
	WE e;
	e.v = 0; e.f = 0;
	if (L.kind == LD_LIVE) { e.v = (L.rows[r * L.W] & GG_DATUMROW_DEAD) ? 0ull : 1ull; return e; }
	if (L.kind == LD_ARRAY) { e.v = L.arr[r]; return e; }
	const unsigned long long *row = L.rows + slot_of(L.idx, r) * L.W;
	const bool nn = !((row[0] >> L.col) & 1ull);
	const unsigned long long x = row[1 + L.col];
	if (L.kind == LD_COUNT) { e.v = nn ? (1ull | ((L.isf8 && !isfinite(u2d(x))) ? (1ull << 32) : 0ull)) : 0ull; return e; }
	if (L.kind == LD_ISUM) { e.v = nn ? x : 0ull; return e; }
	e.v = x;
	e.f = nn ? WE_HAS : 0u;
	const bool head = L.rev ? (r == L.m - 1 || seg_no(L.arr[r + 1], L.seg) != seg_no(L.arr[r], L.seg))
	                        : (r == 0 || seg_no(L.arr[r], L.seg) != seg_no(L.arr[r - 1], L.seg));
	if (head) e.f |= WE_HEAD;
	return e;
}

__device__ __forceinline__ WE shfl_up_we(WE x, int d)
{
	WE r;
	r.v = __shfl_up_sync(0xffffffffu, x.v, d);
	r.f = __shfl_up_sync(0xffffffffu, x.f, d);
	return r;
}

/* exclusive scan of one value per thread over the block (blockDim.x a multiple of 32, at most 1024); *total = the block's sum */
__device__ WE block_exscan(int op, int rev, WE x, WE *warp_tot, WE *total)
{
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
	const WE id = { 0ull, 0u };
	WE inc = x;
	for (int d = 1; d < 32; d <<= 1)
	{
		const WE o = shfl_up_we(inc, d);
		if (lane >= d) inc = wcombine(op, rev, o, inc);
	}
	if (lane == 31) warp_tot[warp] = inc;
	__syncthreads();
	if (warp == 0)
	{
		WE t = lane < nwarps ? warp_tot[lane] : id;
		for (int d = 1; d < 32; d <<= 1)
		{
			const WE o = shfl_up_we(t, d);
			if (lane >= d) t = wcombine(op, rev, o, t);
		}
		warp_tot[lane] = t;                       /* inclusive over the warps */
	}
	__syncthreads();
	const WE wpre = warp == 0 ? id : warp_tot[warp - 1];
	WE ex = shfl_up_we(inc, 1);
	ex = lane == 0 ? wpre : wcombine(op, rev, wpre, ex);
	*total = warp_tot[nwarps - 1];
	__syncthreads();
	return ex;
}

/* one tile of a scan: APPLY = 0 writes the tile's total, APPLY = 1 the inclusive results after the tile's carry */
template <int APPLY>
__global__ void __launch_bounds__(WIN_THREADS)
gg_window_scan_kernel(WLoad L, int op, WE *tile_tot, unsigned long long *outv)
{
	__shared__ WE sh[WIN_TILE];
	__shared__ WE warp_tot[32];
	const uint64_t base = (uint64_t) blockIdx.x * WIN_TILE;
	const WE id = { 0ull, 0u };
	for (int i = 0; i < WIN_ITEMS; i++)
	{
		const uint64_t k = base + (uint64_t) i * WIN_THREADS + threadIdx.x;
		sh[i * WIN_THREADS + threadIdx.x] = k < L.m ? wload(L, L.rev ? L.m - 1 - k : k) : id;
	}
	__syncthreads();
	WE x[WIN_ITEMS], agg = id;
	for (int i = 0; i < WIN_ITEMS; i++) { x[i] = sh[threadIdx.x * WIN_ITEMS + i]; agg = wcombine(op, L.rev, agg, x[i]); }
	WE total;
	WE run = block_exscan(op, L.rev, agg, warp_tot, &total);
	if (!APPLY)
	{
		if (threadIdx.x == 0) tile_tot[blockIdx.x] = total;
		return;
	}
	run = wcombine(op, L.rev, tile_tot[blockIdx.x], run);
	for (int i = 0; i < WIN_ITEMS; i++) { run = wcombine(op, L.rev, run, x[i]); sh[threadIdx.x * WIN_ITEMS + i] = run; }
	__syncthreads();
	for (int i = 0; i < WIN_ITEMS; i++)
	{
		const uint64_t k = base + (uint64_t) i * WIN_THREADS + threadIdx.x;
		if (k >= L.m) break;
		const uint64_t r = L.rev ? L.m - 1 - k : k;
		outv[r] = sh[i * WIN_THREADS + threadIdx.x].v;
	}
}

/* the carry scan: exclusive, in place, over the tiles' totals, one block (each thread a contiguous run of tiles) */
__global__ void __launch_bounds__(WIN_CARRY_THREADS)
gg_window_carry_kernel(int op, int rev, WE *tile_tot, uint32_t ntiles)
{
	__shared__ WE warp_tot[32];
	const uint32_t per = (ntiles + WIN_CARRY_THREADS - 1) / WIN_CARRY_THREADS;
	const uint32_t lo = threadIdx.x * per, hi = min(lo + per, ntiles);
	WE agg = { 0ull, 0u }, total;
	for (uint32_t t = lo; t < hi; t++) agg = wcombine(op, rev, agg, tile_tot[t]);
	WE run = block_exscan(op, rev, agg, warp_tot, &total);
	for (uint32_t t = lo; t < hi; t++) { const WE x = tile_tot[t]; tile_tot[t] = run; run = wcombine(op, rev, run, x); }
}

/* idx[j] = slot of the j-th live row: pos = inclusive scan of the live flags */
__global__ void gg_window_compact_kernel(const unsigned long long *rows, uint32_t W, uint64_t n, const unsigned long long *pos, uint32_t *idx)
{
	const uint64_t s = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x;
	if (s < n && !(rows[s * W] & GG_DATUMROW_DEAD)) idx[pos[s] - 1] = (uint32_t) s;
}

struct WinKeys {
	int npart, nord;
	int col[2 * GG_MAX_KEYS];               /* partition columns, then order columns */
	uint32_t f8mask;                        /* columns that are float8: compared normalised */
};

/* execTuplesMatch (execGrouping.c) of one column: two NULLs match; float8 -0 = +0, NaN = NaN; everything else by bits */
__device__ __forceinline__ bool col_differs(const unsigned long long *a, const unsigned long long *b, int c, uint32_t f8mask)
{
	const unsigned long long na = (a[0] >> c) & 1ull, nb = (b[0] >> c) & 1ull;
	if (na != nb) return true;
	if (na) return false;
	unsigned long long x = a[1 + c], y = b[1 + c];
	if ((f8mask >> c) & 1u)
	{
		const double dx = u2d(x), dy = u2d(y);
		if (isnan(dx) || isnan(dy)) return isnan(dx) != isnan(dy);
		return dx != dy;
	}
	return x != y;
}

/* hp[j] = (starts a partition) << 32 | (starts a peer group) */
__global__ void gg_window_heads_kernel(const unsigned long long *rows, uint32_t W, const uint32_t *idx, uint64_t m, WinKeys K,
                                       unsigned long long *hp)
{
	const uint64_t j = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x;
	if (j >= m) return;
	bool ph = j == 0, gh;
	if (!ph)
	{
		const unsigned long long *a = rows + slot_of(idx, j) * W, *b = rows + slot_of(idx, j - 1) * W;
		for (int k = 0; k < K.npart && !ph; k++) ph = col_differs(a, b, K.col[k], K.f8mask);
		gh = ph;
		for (int k = 0; k < K.nord && !gh; k++) gh = col_differs(a, b, K.col[K.npart + k], K.f8mask);
	}
	else
		gh = true;
	hp[j] = ((unsigned long long) ph << 32) | (unsigned long long) gh;
}

/* after the scan of hp: pstart[p] = first row of partition p, gstart[g] = first row of peer group g, each closed by m */
__global__ void gg_window_starts_kernel(const unsigned long long *hp, uint64_t m, uint32_t *pstart, uint32_t *gstart)
{
	const uint64_t j = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x;
	if (j >= m) return;
	const uint32_t p = (uint32_t) (hp[j] >> 32), g = (uint32_t) hp[j];
	if (j == 0 || (uint32_t) (hp[j - 1] >> 32) != p) pstart[p - 1] = (uint32_t) j;
	if (j == 0 || (uint32_t) hp[j - 1] != g) gstart[g - 1] = (uint32_t) j;
	if (j == m - 1) { pstart[p] = (uint32_t) m; gstart[g] = (uint32_t) m; }
}

/* an argument: a column of a row (col >= 0) or a Const */
struct WinArg {
	int col, isnull;
	unsigned long long v;
};

enum { SEG_NONE = 0, SEG_ROW, SEG_FWD_PART, SEG_REV_PART, SEG_FWD_PEER };

struct WinFn {
	int32_t fn, seg;
	WinArg a[3];
	const unsigned long long *cnt;          /* count(x), sum, avg, min, max: prefix of (non-NULL) | (non-finite) << 32 */
	const unsigned long long *sum;          /* sum(int4): prefix of the values */
	const unsigned long long *segv;         /* float8 sum / avg, min / max: segmented scan (NULL when the count prefix says so) */
};

struct WinFns {
	int n, frame;
	WinFn f[GG_MAX_WINFUNCS];
};

__device__ __forceinline__ unsigned long long arg_at(const WinArg &a, const unsigned long long *row, bool *isnull)
{
	if (a.col < 0) { *isnull = a.isnull != 0; return a.isnull ? 0ull : a.v; }
	*isnull = (row[0] >> a.col) & 1ull;
	return *isnull ? 0ull : row[1 + a.col];
}

__device__ __forceinline__ unsigned long long pref(const unsigned long long *p, int64_t head, int64_t tail)
{
	return p[tail] - (head > 0 ? p[head - 1] : 0ull);
}

__global__ void __launch_bounds__(256)
gg_window_write_kernel(const unsigned long long *rows, uint32_t W, const uint32_t *idx, uint64_t m, const unsigned long long *hp,
                       const uint32_t *pstart, const uint32_t *gstart, WinFns F, unsigned long long *out, uint32_t *d_err)
{
	const uint64_t j = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x;
	if (j >= m) return;
	const uint32_t W2 = W + (uint32_t) F.n;
	const unsigned long long *in = rows + slot_of(idx, j) * W;
	unsigned long long *o = out + j * W2;
	const uint32_t p = (uint32_t) (hp[j] >> 32) - 1, g = (uint32_t) hp[j] - 1;
	ggw_bounds b;
	b.ps = pstart[p]; b.pe = pstart[p + 1]; b.gs = gstart[g]; b.ge = gstart[g + 1];
	int64_t head, tail;
	ggw_frame(F.frame, (int64_t) j, b, &head, &tail);
	unsigned long long mask = in[0];
	for (uint32_t c = 1; c < W; c++) o[c] = in[c];
	for (int i = 0; i < F.n; i++)
	{
		const WinFn &f = F.f[i];
		unsigned long long v = 0;
		bool isnull = false;
		switch (f.fn)
		{
			case GG_WF_ROW_NUMBER: v = (unsigned long long) ggw_row_number((int64_t) j, b); break;
			case GG_WF_RANK: v = (unsigned long long) ggw_rank(b); break;
			case GG_WF_DENSE_RANK: v = (unsigned long long) ((uint32_t) hp[j] - (uint32_t) hp[b.ps] + 1u); break;
			case GG_WF_PERCENT_RANK: v = d2u(ggw_percent_rank(b)); break;
			case GG_WF_CUME_DIST: v = d2u(ggw_cume_dist(b)); break;
			case GG_WF_NTILE:
				/* a NULL bucket count gives NULL; one <= 0 was refused before the launch */
				if (f.a[0].isnull) isnull = true;
				else v = (unsigned long long) (long long) ggw_ntile(b.pe - b.ps, (int32_t) f.a[0].v, (int64_t) j - b.ps);
				break;
			case GG_WF_LAG: case GG_WF_LAG_OFFSET: case GG_WF_LAG_DEFAULT:
			case GG_WF_LEAD: case GG_WF_LEAD_OFFSET: case GG_WF_LEAD_DEFAULT:
			{
				const bool fwd = f.fn >= GG_WF_LEAD;
				int64_t off = 1, t;
				if (f.a[1].col >= 0 || f.a[1].isnull >= 0)
				{
					bool onull;
					off = (int64_t) (int32_t) arg_at(f.a[1], in, &onull);
					if (onull) { isnull = true; break; }
				}
				if (ggw_leadlag((int64_t) j, off, fwd, b, &t)) v = arg_at(f.a[0], rows + slot_of(idx, (uint64_t) t) * W, &isnull);
				else if (f.a[2].col >= 0 || f.a[2].isnull >= 0) v = arg_at(f.a[2], in, &isnull);
				else isnull = true;
				break;
			}
			case GG_WF_FIRST_VALUE: v = arg_at(f.a[0], rows + slot_of(idx, (uint64_t) head) * W, &isnull); break;
			case GG_WF_LAST_VALUE: v = arg_at(f.a[0], rows + slot_of(idx, (uint64_t) tail) * W, &isnull); break;
			case GG_WF_NTH_VALUE:
			{
				if (f.a[1].isnull) { isnull = true; break; }
				const int64_t t = head + (int64_t) (int32_t) f.a[1].v - 1;
				if (t > tail) isnull = true;
				else v = arg_at(f.a[0], rows + slot_of(idx, (uint64_t) t) * W, &isnull);
				break;
			}
			default:
			{
				/* an aggregate over the frame [head, tail] */
				const uint64_t count = (uint64_t) (tail - head + 1);
				uint64_t nn = 0, nonfinite = 0;
				unsigned long long acc = 0;
				int nul = 0;
				if (f.cnt)
				{
					const unsigned long long c = pref(f.cnt, head, tail);
					nn = (uint32_t) c; nonfinite = c >> 32;
				}
				else if (f.fn == GG_AGG_COUNT_ANY)
					nn = f.a[0].isnull ? 0 : count;                      /* count(Const) */
				if (f.sum) acc = pref(f.sum, head, tail);
				else if (f.segv)
				{
					const int64_t at = f.seg == SEG_REV_PART ? head : tail;
					acc = f.segv[at];
				}
				else if (f.seg == SEG_ROW) acc = in[1 + f.a[0].col];
				v = gg_aggfinal(f.fn, count, nn, acc, &nul);
				isnull = nul != 0;
				if (!isnull && (f.fn == GG_AGG_SUM_FLOAT8 || f.fn == GG_AGG_AVG_FLOAT8) && nonfinite == 0 && !isfinite(u2d(v)))
					atomicOr(d_err, (uint32_t) GGP_EF_FLOAT_OVERFLOW);
				break;
			}
		}
		if (isnull) { mask |= 1ull << (W - 1 + i); v = 0; }
		o[W + i] = v;
	}
	o[0] = mask;
}

struct gg_window_obj {
	gg_engine *eng = nullptr;
	gg_window win;
	int ncols = 0;
	WinKeys keys;
	WinFns fns;
	void *scratch = nullptr;
	size_t scratch_bytes = 0;
	gg_relation *rows_buf = nullptr, *rows_view = nullptr;
};

static const char *wf_name(int32_t fn)
{
	switch (fn)
	{
		case GG_WF_NTILE: return "ntile";
		case GG_WF_NTH_VALUE: return "nth_value";
		default: return "window function";
	}
}

/* the result type of a function, given its first argument's type; 0 for a function the device does not run */
static int32_t wf_result_type(int32_t fn, int32_t argtype)
{
	switch (fn)
	{
		case GG_WF_ROW_NUMBER: case GG_WF_RANK: case GG_WF_DENSE_RANK: return GG_INT8OID;
		case GG_WF_PERCENT_RANK: case GG_WF_CUME_DIST: return GG_FLOAT8OID;
		case GG_WF_NTILE: return GG_INT4OID;
		case GG_WF_LAG: case GG_WF_LAG_OFFSET: case GG_WF_LAG_DEFAULT: case GG_WF_LEAD: case GG_WF_LEAD_OFFSET: case GG_WF_LEAD_DEFAULT:
		case GG_WF_FIRST_VALUE: case GG_WF_LAST_VALUE: case GG_WF_NTH_VALUE:
			return argtype;
		case GG_AGG_COUNT_ANY: case GG_AGG_COUNT_STAR: case GG_AGG_SUM_INT4: case GG_AGG_MAX_INT8: case GG_AGG_MIN_INT8: return GG_INT8OID;
		case GG_AGG_MAX_INT4: case GG_AGG_MIN_INT4: return GG_INT4OID;
		case GG_AGG_MAX_DATE: case GG_AGG_MIN_DATE: return GG_DATEOID;
		case GG_AGG_SUM_FLOAT8: case GG_AGG_AVG_FLOAT8: case GG_AGG_MAX_FLOAT8: case GG_AGG_MIN_FLOAT8: return GG_FLOAT8OID;
	}
	return 0;
}

/* how many arguments a function takes (minimum, maximum) */
static void wf_nargs(int32_t fn, int *lo, int *hi)
{
	*lo = *hi = 1;
	switch (fn)
	{
		case GG_WF_ROW_NUMBER: case GG_WF_RANK: case GG_WF_DENSE_RANK: case GG_WF_PERCENT_RANK: case GG_WF_CUME_DIST: case GG_AGG_COUNT_STAR:
			*lo = *hi = 0; break;
		case GG_WF_LAG_OFFSET: case GG_WF_LEAD_OFFSET: case GG_WF_NTH_VALUE: *lo = *hi = 2; break;
		case GG_WF_LAG_DEFAULT: case GG_WF_LEAD_DEFAULT: *lo = *hi = 3; break;
	}
}

extern "C" {

int gg_window_create(gg_engine *e, const gg_tupdesc *rows_desc, const gg_window *win, const gg_exprpool *pool, gg_window_obj **out)
{
	if (!e || !rows_desc || !win || !pool || !out) return GG_ERR_ARG;
	*out = nullptr;
	const int ncols = rows_desc->natts;
	if (ncols < 1 || ncols > GG_MAX_ATTS || rows_desc->format != GG_FMT_DATUMROWS)
	{ gg_set_error("WindowAgg: the input must be datum rows of 1..%d columns", GG_MAX_ATTS); return GG_ERR_ARG; }
	if (win->partNumCols < 0 || win->partNumCols > GG_MAX_KEYS || win->ordNumCols < 0 || win->ordNumCols > GG_MAX_KEYS)
	{ gg_set_error("WindowAgg with %d partition and %d order columns (at most %d each)", win->partNumCols, win->ordNumCols, GG_MAX_KEYS); return GG_ERR_UNSUPPORTED; }
	if (win->numFuncs < 1 || win->numFuncs > GG_MAX_WINFUNCS)
	{ gg_set_error("WindowAgg with %d functions (1..%d)", win->numFuncs, GG_MAX_WINFUNCS); return GG_ERR_UNSUPPORTED; }
	if (ncols + win->numFuncs > GG_MAX_ATTS)
	{ gg_set_error("WindowAgg with %d output columns (datum rows carry up to %d)", ncols + win->numFuncs, GG_MAX_ATTS); return GG_ERR_UNSUPPORTED; }
	if (!ggw_frame_supported(win->frameOptions))
	{ gg_set_error("WindowAgg: frame options 0x%x (only ROWS / RANGE from UNBOUNDED PRECEDING or CURRENT ROW to CURRENT ROW or UNBOUNDED FOLLOWING)", win->frameOptions); return GG_ERR_UNSUPPORTED; }
	gg_window_obj *w = new gg_window_obj();
	w->eng = e; w->win = *win; w->ncols = ncols;
	memset(&w->keys, 0, sizeof w->keys);
	memset(&w->fns, 0, sizeof w->fns);
	w->keys.npart = win->partNumCols; w->keys.nord = win->ordNumCols;
	for (int k = 0; k < win->partNumCols + win->ordNumCols; k++)
	{
		const int c = k < win->partNumCols ? win->partColIdx[k] : win->ordColIdx[k - win->partNumCols];
		if (c < 0 || c >= ncols) { gg_set_error("WindowAgg key column %d out of range (%d columns)", c, ncols); delete w; return GG_ERR_ARG; }
		w->keys.col[k] = c;
	}
	for (int c = 0; c < ncols; c++) if (rows_desc->attrs[c].atttypid == GG_FLOAT8OID) w->keys.f8mask |= 1u << c;
	w->fns.n = win->numFuncs;
	w->fns.frame = win->frameOptions;
	const bool rows_mode = (win->frameOptions & GG_FRAMEOPTION_ROWS) != 0;
	for (int i = 0; i < win->numFuncs; i++)
	{
		const gg_winfunc &wf = win->funcs[i];
		WinFn &f = w->fns.f[i];
		int lo, hi, nargs = 0;
		int32_t argtype[3] = { 0, 0, 0 };
		f.fn = wf.winfnoid;
		wf_nargs(wf.winfnoid, &lo, &hi);
		for (int a = 0; a < 3; a++)
		{
			f.a[a].col = -1; f.a[a].isnull = -1; f.a[a].v = 0;       /* isnull = -1 with col = -1: absent */
			const int32_t root = wf.arg[a];
			if (root < 0) continue;
			if (a >= hi) { gg_set_error("window function %d: argument %d is one too many", wf.winfnoid, a + 1); delete w; return GG_ERR_ARG; }
			if (root >= pool->nnodes) { gg_set_error("window function %d: argument node %d is not in the pool", wf.winfnoid, root); delete w; return GG_ERR_ARG; }
			const gg_expr &x = pool->nodes[root];
			nargs = a + 1;
			argtype[a] = x.rettype;
			if (x.kind == GG_E_VAR)
			{
				if (x.varno != 0 || x.varattno < 1 || x.varattno > ncols)
				{ gg_set_error("window function %d: Var %d.%d is not a column of the input rows", wf.winfnoid, x.varno, x.varattno); delete w; return GG_ERR_ARG; }
				f.a[a].col = x.varattno - 1;
				argtype[a] = rows_desc->attrs[x.varattno - 1].atttypid;
			}
			else if (x.kind == GG_E_CONST) { f.a[a].isnull = x.constisnull ? 1 : 0; f.a[a].v = (unsigned long long) x.constvalue; }
			else { gg_set_error("window function %d: argument %d is neither a Var nor a Const", wf.winfnoid, a + 1); delete w; return GG_ERR_UNSUPPORTED; }
		}
		const int32_t rt = wf_result_type(wf.winfnoid, argtype[0]);
		if (!rt)
		{
			gg_set_error("window function %d is not on the device path%s", wf.winfnoid,
			             (wf.winfnoid == GG_AGG_SUM_NUMERIC || wf.winfnoid == GG_AGG_AVG_NUMERIC) ? " (numeric aggregates)" : "");
			delete w; return GG_ERR_UNSUPPORTED;
		}
		if (argtype[0] == GG_NUMERICOID) { gg_set_error("window function %d over a numeric argument", wf.winfnoid); delete w; return GG_ERR_UNSUPPORTED; }
		if (gg_aggfinal_covers(wf.winfnoid) && wf.winfnoid != GG_AGG_COUNT_ANY && wf.winfnoid != GG_AGG_COUNT_STAR &&
		    (argtype[0] == GG_BPCHAROID || argtype[0] == GG_VARCHAROID || argtype[0] == GG_TEXTOID))
		{ gg_set_error("window aggregate %d over a string argument", wf.winfnoid); delete w; return GG_ERR_UNSUPPORTED; }
		if (nargs < lo) { gg_set_error("window function %d takes %d arguments, %d given", wf.winfnoid, lo, nargs); delete w; return GG_ERR_ARG; }
		if (wf.wintype != rt) { gg_set_error("window function %d returns type %d, the plan says %d", wf.winfnoid, rt, wf.wintype); delete w; return GG_ERR_ARG; }
		if ((wf.winfnoid == GG_WF_NTILE && f.a[0].col >= 0) || (wf.winfnoid == GG_WF_NTH_VALUE && f.a[1].col >= 0))
		{ gg_set_error("%s: the argument must be a Const", wf_name(wf.winfnoid)); delete w; return GG_ERR_UNSUPPORTED; }
		if ((wf.winfnoid == GG_WF_LAG_OFFSET || wf.winfnoid == GG_WF_LAG_DEFAULT || wf.winfnoid == GG_WF_LEAD_OFFSET || wf.winfnoid == GG_WF_LEAD_DEFAULT) &&
		    argtype[1] != GG_INT4OID)
		{ gg_set_error("lag / lead: the offset must be int4"); delete w; return GG_ERR_ARG; }
		if (gg_aggfinal_covers(wf.winfnoid) && wf.winfnoid != GG_AGG_COUNT_STAR && wf.winfnoid != GG_AGG_COUNT_ANY && f.a[0].col < 0)
		{ gg_set_error("window aggregate %d over a constant", wf.winfnoid); delete w; return GG_ERR_UNSUPPORTED; }
		/* the segmented scan a float8 sum / avg or a min / max reads (the int sums and counts read prefix differences) */
		if (gg_aggfinal_covers(wf.winfnoid) && wf.winfnoid != GG_AGG_COUNT_STAR && wf.winfnoid != GG_AGG_COUNT_ANY && wf.winfnoid != GG_AGG_SUM_INT4)
		{
			if (win->frameOptions & GG_FRAMEOPTION_START_UNBOUNDED_PRECEDING) f.seg = SEG_FWD_PART;
			else if (win->frameOptions & GG_FRAMEOPTION_END_UNBOUNDED_FOLLOWING) f.seg = SEG_REV_PART;
			else f.seg = rows_mode ? SEG_ROW : SEG_FWD_PEER;
		}
	}
	*out = w;
	return GG_OK;
}

static int win_scan(gg_engine *e, const WLoad &L, int op, WE *tile_tot, unsigned long long *outv)
{
	cudaStream_t st = e->stream;
	const uint64_t ntiles = (L.m + WIN_TILE - 1) / WIN_TILE;
	if (!ntiles) return GG_OK;
	gg_window_scan_kernel<0><<<(unsigned) ntiles, WIN_THREADS, 0, st>>>(L, op, tile_tot, outv);
	gg_window_carry_kernel<<<1, WIN_CARRY_THREADS, 0, st>>>(op, L.rev, tile_tot, (uint32_t) ntiles);
	gg_window_scan_kernel<1><<<(unsigned) ntiles, WIN_THREADS, 0, st>>>(L, op, tile_tot, outv);
	e->launches += 3;
	GG_CUDA(cudaGetLastError());
	return GG_OK;
}

int gg_window_run(gg_window_obj *w, gg_relation *rows, uint64_t nrows, gg_relation **out_view, uint64_t *nout)
{
	if (!w || !rows || !out_view || !nout) return GG_ERR_ARG;
	const uint32_t W = 1 + (uint32_t) w->ncols, W2 = W + (uint32_t) w->fns.n;
	if ((uint32_t) rows->rowwords != W) { gg_set_error("WindowAgg over %d columns: the relation has rows of %d words", w->ncols, rows->rowwords); return GG_ERR_ARG; }
	if (nrows > rows->nrows) { gg_set_error("WindowAgg: %llu rows of a relation of %llu", (unsigned long long) nrows, (unsigned long long) rows->nrows); return GG_ERR_ARG; }
	if (nrows >= 0xFFFFFFFFull) { gg_set_error("WindowAgg over %llu rows (row numbers are 32-bit)", (unsigned long long) nrows); return GG_ERR_UNSUPPORTED; }
	gg_engine *e = w->eng;
	cudaStream_t st = e->stream;
	GG_CUDA(cudaSetDevice(e->device));
	GG_CUDA(cudaEventRecord(e->ev_start, st));
	uint64_t m = 0;
	if (nrows)
	{
		/* scratch, sized by the slots: the error word, the tiles' totals, the live positions (then the packed partition / peer
		 * numbers), idx, the two start arrays, and per function its prefix / scan arrays */
		const uint64_t n = nrows, ntiles = (n + WIN_TILE - 1) / WIN_TILE;
		int nper = 0;
		for (int i = 0; i < w->fns.n; i++)
		{
			const WinFn &f = w->fns.f[i];
			if (!gg_aggfinal_covers(f.fn) || f.fn == GG_AGG_COUNT_STAR || (f.fn == GG_AGG_COUNT_ANY && f.a[0].col < 0)) continue;
			nper += 8 + (f.fn == GG_AGG_SUM_INT4 ? 8 : 0) + (f.seg == SEG_FWD_PART || f.seg == SEG_REV_PART || f.seg == SEG_FWD_PEER ? 8 : 0);
		}
		const size_t bytes = 256 + (size_t) ntiles * sizeof(WE) + (size_t) n * (8 + 4 + 4 + 4 + (size_t) nper) + 64 * 16;
		if (w->scratch_bytes < bytes)
		{
			cudaFree(w->scratch);
			w->scratch = nullptr; w->scratch_bytes = 0;
			const cudaError_t ce = cudaMalloc(&w->scratch, bytes);
			if (ce != cudaSuccess) { cudaGetLastError(); gg_set_error("WindowAgg: scratch of %llu bytes does not fit in device memory", (unsigned long long) bytes); return GG_ERR_NOMEM; }
			w->scratch_bytes = bytes;
		}
		uint8_t *p = (uint8_t *) w->scratch;
		auto take = [&](size_t b) { uint8_t *r = p; p += (b + 15) & ~(size_t) 15; return r; };
		uint32_t *d_err = (uint32_t *) take(16);
		WE *tile_tot = (WE *) take((size_t) ntiles * sizeof(WE));
		unsigned long long *hp = (unsigned long long *) take((size_t) n * 8);
		uint32_t *idx = (uint32_t *) take((size_t) n * 4);
		uint32_t *pstart = (uint32_t *) take((size_t) (n + 1) * 4);
		uint32_t *gstart = (uint32_t *) take((size_t) (n + 1) * 4);
		const unsigned long long *in = (const unsigned long long *) rows->pages;
		GG_CUDA(cudaMemsetAsync(d_err, 0, 4, st));

		/* 1. live rows, in input order: counted per tile (the scan's reduce and carry); only when some slot is dead, the apply
		 * pass and the compaction into idx */
		WLoad L;
		memset(&L, 0, sizeof L);
		L.kind = LD_LIVE; L.rows = in; L.W = W; L.m = n;
		WE last_tot, last_ex;
		gg_window_scan_kernel<0><<<(unsigned) ntiles, WIN_THREADS, 0, st>>>(L, WOP_ADD, tile_tot, hp);
		GG_CUDA(cudaMemcpyAsync(&last_tot, tile_tot + ntiles - 1, sizeof(WE), cudaMemcpyDeviceToHost, st));
		gg_window_carry_kernel<<<1, WIN_CARRY_THREADS, 0, st>>>(WOP_ADD, 0, tile_tot, (uint32_t) ntiles);
		e->launches += 2;
		GG_CUDA(cudaGetLastError());
		GG_CUDA(cudaMemcpyAsync(&last_ex, tile_tot + ntiles - 1, sizeof(WE), cudaMemcpyDeviceToHost, st));
		GG_CUDA(cudaStreamSynchronize(st));
		m = last_ex.v + last_tot.v;
		int rc = GG_OK;
		for (int i = 0; m && i < w->fns.n; i++)
		{
			/* ntile / nth_value raise at their first row (windowfuncs.c:240, :462) */
			const WinFn &f = w->fns.f[i];
			const WinArg &a = f.fn == GG_WF_NTILE ? f.a[0] : f.a[1];
			if ((f.fn == GG_WF_NTILE || f.fn == GG_WF_NTH_VALUE) && !a.isnull && (int32_t) a.v <= 0)
			{ gg_set_error("argument of %s must be greater than zero", wf_name(f.fn)); return GG_ERR_WINDOW_ARG; }
		}
		if (m)
		{
			const unsigned nb = (unsigned) ((n + 255) / 256), mb = (unsigned) ((m + 255) / 256);
			if (m < n)
			{
				gg_window_scan_kernel<1><<<(unsigned) ntiles, WIN_THREADS, 0, st>>>(L, WOP_ADD, tile_tot, hp);
				gg_window_compact_kernel<<<nb, 256, 0, st>>>(in, W, n, hp, idx);
				e->launches += 2;
			}
			else
				idx = nullptr;
			/* 2. partitions and peer groups */
			gg_window_heads_kernel<<<mb, 256, 0, st>>>(in, W, idx, m, w->keys, hp);
			e->launches++;
			GG_CUDA(cudaGetLastError());
			L.kind = LD_ARRAY; L.arr = hp; L.m = m;
			if ((rc = win_scan(e, L, WOP_ADD, tile_tot, hp))) return rc;
			gg_window_starts_kernel<<<mb, 256, 0, st>>>(hp, m, pstart, gstart);
			e->launches++;
			/* 3. the aggregates' scans */
			WinFns F = w->fns;
			for (int i = 0; i < F.n; i++)
			{
				WinFn &f = F.f[i];
				if (!gg_aggfinal_covers(f.fn) || f.fn == GG_AGG_COUNT_STAR || (f.fn == GG_AGG_COUNT_ANY && f.a[0].col < 0)) continue;
				const int isf8 = gg_aggfinal_is_float8(f.fn);
				WLoad A;
				memset(&A, 0, sizeof A);
				A.rows = in; A.W = W; A.idx = idx; A.m = m; A.col = f.a[0].col; A.isf8 = isf8; A.arr = hp;
				unsigned long long *cnt = (unsigned long long *) take((size_t) m * 8);
				A.kind = LD_COUNT;
				if ((rc = win_scan(e, A, WOP_ADD, tile_tot, cnt))) return rc;
				f.cnt = cnt;
				if (f.fn == GG_AGG_SUM_INT4)
				{
					unsigned long long *s = (unsigned long long *) take((size_t) m * 8);
					A.kind = LD_ISUM;
					if ((rc = win_scan(e, A, WOP_ADD, tile_tot, s))) return rc;
					f.sum = s;
				}
				else if (f.seg == SEG_FWD_PART || f.seg == SEG_REV_PART || f.seg == SEG_FWD_PEER)
				{
					unsigned long long *sv = (unsigned long long *) take((size_t) m * 8);
					const int32_t fn = f.fn;
					const bool isint = fn == GG_AGG_MIN_INT4 || fn == GG_AGG_MIN_INT8 || fn == GG_AGG_MIN_DATE || fn == GG_AGG_MAX_INT4 ||
					                   fn == GG_AGG_MAX_INT8 || fn == GG_AGG_MAX_DATE;
					const bool ismin = fn == GG_AGG_MIN_INT4 || fn == GG_AGG_MIN_INT8 || fn == GG_AGG_MIN_DATE || fn == GG_AGG_MIN_FLOAT8;
					const int op = (fn == GG_AGG_SUM_FLOAT8 || fn == GG_AGG_AVG_FLOAT8) ? WOP_SUM_F8
					             : isint ? (ismin ? WOP_MIN_I : WOP_MAX_I) : (ismin ? WOP_MIN_F8 : WOP_MAX_F8);
					A.kind = LD_SEG;
					A.seg = f.seg == SEG_FWD_PEER ? 1 : 0;
					A.rev = f.seg == SEG_REV_PART;
					if ((rc = win_scan(e, A, op, tile_tot, sv))) return rc;
					f.segv = sv;
				}
			}
			/* 4. the output rows */
			rc = GG_OK;
			{
				const uint64_t nb2 = (m * W2 * 8 + 16 + GG_BLCKSZ - 1) / GG_BLCKSZ;
				if (w->rows_buf && w->rows_buf->nblocks < nb2) { gg_relation_free(w->rows_buf); w->rows_buf = nullptr; }
				if (!w->rows_buf && (rc = gg_relation_create(e, nb2, &w->rows_buf)) != GG_OK) { w->rows_buf = nullptr; return rc; }
			}
			gg_window_write_kernel<<<mb, 256, 0, st>>>(in, W, idx, m, hp, pstart, gstart, F, (unsigned long long *) w->rows_buf->pages, d_err);
			e->launches++;
			GG_CUDA(cudaGetLastError());
			uint32_t flags = 0;
			GG_CUDA(cudaMemcpyAsync(&flags, d_err, 4, cudaMemcpyDeviceToHost, st));
			GG_CUDA(cudaStreamSynchronize(st));
			if ((rc = gg_errflags_to_code(flags)) != GG_OK) return rc;
		}
	}
	if (!w->rows_buf)
	{
		const int rc = gg_relation_create(e, 1, &w->rows_buf);
		if (rc) { w->rows_buf = nullptr; return rc; }
	}
	GG_CUDA(cudaEventRecord(e->ev_stop, st));
	if (w->rows_view) { gg_relation_free(w->rows_view); w->rows_view = nullptr; }
	const int rc = gg_relation_attach_rows(e, w->rows_buf->pages, m, w->ncols + w->fns.n, &w->rows_view);
	if (rc) { w->rows_view = nullptr; return rc; }
	*out_view = w->rows_view;
	*nout = m;
	return GG_OK;
}

void gg_window_free(gg_window_obj *w)
{
	if (!w) return;
	if (w->eng) cudaSetDevice(w->eng->device);
	if (w->rows_view) gg_relation_free(w->rows_view);
	if (w->rows_buf) gg_relation_free(w->rows_buf);
	cudaFree(w->scratch);
	delete w;
}

}  /* extern "C" */
