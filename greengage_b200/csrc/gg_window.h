/*
 * gg_window.h — the per-row rules of WindowAgg (nodeWindowAgg.c, utils/adt/windowfuncs.c) over rows already numbered into
 * partitions and peer groups: the frame of a row, the ranking functions, ntile's bucket and the row lag / lead read.  Plain C,
 * compiled by nvcc for the kernels of gg_window.cu and by gcc in tests/test_window_rules.py, so there is one statement of them.
 *
 * Row positions count the live rows of the window's input from 0.  For a row j:
 *   ps, pe   its partition: rows [ps, pe)
 *   gs, ge   its peer group (rows equal on the ORDER BY columns; the whole partition without ORDER BY): rows [gs, ge)
 */
#ifndef GG_WINDOW_H
#define GG_WINDOW_H

#include <stdint.h>
#include "../../include/gg_plan.h"

#if defined(__CUDACC__)
#define GGW_FN __host__ __device__ __forceinline__
#else
#define GGW_FN static inline
#endif

typedef struct ggw_bounds {
	int64_t ps, pe, gs, ge;
} ggw_bounds;

/* whether the device evaluates a frame: ROWS or RANGE, start UNBOUNDED PRECEDING or CURRENT ROW, end CURRENT ROW or UNBOUNDED
 * FOLLOWING (parsenodes.h:495-517); value offsets and the disallowed bounds are not */
GGW_FN int ggw_frame_supported(int32_t opt)
{
	const int32_t mode = opt & (GG_FRAMEOPTION_RANGE | GG_FRAMEOPTION_ROWS);
	const int32_t start = opt & (GG_FRAMEOPTION_START_UNBOUNDED_PRECEDING | GG_FRAMEOPTION_START_CURRENT_ROW);
	const int32_t end = opt & (GG_FRAMEOPTION_END_CURRENT_ROW | GG_FRAMEOPTION_END_UNBOUNDED_FOLLOWING);
	const int32_t other = GG_FRAMEOPTION_END_UNBOUNDED_PRECEDING | GG_FRAMEOPTION_START_UNBOUNDED_FOLLOWING | GG_FRAMEOPTION_START_VALUE_PRECEDING |
	                      GG_FRAMEOPTION_END_VALUE_PRECEDING | GG_FRAMEOPTION_START_VALUE_FOLLOWING | GG_FRAMEOPTION_END_VALUE_FOLLOWING;
	if (opt & other) return 0;
	if (mode != GG_FRAMEOPTION_RANGE && mode != GG_FRAMEOPTION_ROWS) return 0;
	if (start != GG_FRAMEOPTION_START_UNBOUNDED_PRECEDING && start != GG_FRAMEOPTION_START_CURRENT_ROW) return 0;
	return end == GG_FRAMEOPTION_END_CURRENT_ROW || end == GG_FRAMEOPTION_END_UNBOUNDED_FOLLOWING;
}

/* the frame of row j, rows [*head, *tail] (update_frameheadpos / update_frametailpos, nodeWindowAgg.c): CURRENT ROW is the row
 * itself in ROWS mode and its first / last peer in RANGE mode.  Every supported frame holds the current row. */
GGW_FN void ggw_frame(int32_t opt, int64_t j, ggw_bounds b, int64_t *head, int64_t *tail)
{
	const int rows = (opt & GG_FRAMEOPTION_ROWS) != 0;
	*head = (opt & GG_FRAMEOPTION_START_UNBOUNDED_PRECEDING) ? b.ps : rows ? j : b.gs;
	*tail = (opt & GG_FRAMEOPTION_END_UNBOUNDED_FOLLOWING) ? b.pe - 1 : rows ? j : b.ge - 1;
}

/* window_row_number / window_rank / window_percent_rank / window_cume_dist (windowfuncs.c:81-200) */
GGW_FN int64_t ggw_row_number(int64_t j, ggw_bounds b) { return j - b.ps + 1; }
GGW_FN int64_t ggw_rank(ggw_bounds b) { return b.gs - b.ps + 1; }
GGW_FN double ggw_percent_rank(ggw_bounds b)
{
	const int64_t total = b.pe - b.ps;
	return total <= 1 ? 0.0 : (double) (ggw_rank(b) - 1) / (double) (total - 1);
}
GGW_FN double ggw_cume_dist(ggw_bounds b) { return (double) (b.ge - b.ps) / (double) (b.pe - b.ps); }

/* window_ntile (windowfuncs.c:211-276) in closed form: of `total` rows in n > 0 buckets, the first total % n buckets hold one
 * row more than the others (every row its own bucket when total < n); k = the row's position in its partition */
GGW_FN int32_t ggw_ntile(int64_t total, int32_t n, int64_t k)
{
	const int64_t q = total / n, r = total % n;
	if (k < r * (q + 1)) return (int32_t) (k / (q + 1) + 1);
	return (int32_t) (r + (k - r * (q + 1)) / q + 1);
}

/* leadlag_common (windowfuncs.c:286-329): the row lag (forward = 0) or lead (forward = 1) reads `offset` rows away from j, a
 * negative offset seeking the other way; 1 and *target = that row when it lies in the partition, else 0 (the default, or NULL) */
GGW_FN int ggw_leadlag(int64_t j, int64_t offset, int forward, ggw_bounds b, int64_t *target)
{
	const int64_t t = forward ? j + offset : j - offset;
	*target = t;
	return t >= b.ps && t < b.pe;
}

#endif /* GG_WINDOW_H */
