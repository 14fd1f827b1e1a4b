/*
 * gg_aggfinal.h — finalize_aggregate (nodeAgg.c:871-999) of ONE aggregate of ONE group at the NORMAL / FINAL stage, from the
 * group's accumulated state: the rule the host's finalize_rows (gg_scanagg.cu) applies when it fills a gg_aggrow, and the rule
 * the kernels of gg_aggrows.cu apply when they write a group as a datum row.  Plain C, compiled by nvcc for both and by gcc in
 * tests/test_aggfinal.py, so that there is one statement of it.
 *
 * Covered: count(*), count(expr), the int sums, min/max of int4 / int8 / date / float8, the float8 sum and avg(float8).
 * Not covered: numeric sum / avg and the PARTIAL stage's transition states, which only the host finalises.
 */
#ifndef GG_AGGFINAL_H
#define GG_AGGFINAL_H

#include <stdint.h>
#include "../../include/gg_plan.h"

#if defined(__CUDACC__)
#define GG_AGGFINAL_FN __host__ __device__ __forceinline__
#else
#define GG_AGGFINAL_FN static inline
#endif

/* whether gg_aggfinal covers the aggregate */
GG_AGGFINAL_FN int gg_aggfinal_covers(int32_t aggfnoid)
{
	switch (aggfnoid)
	{
		case GG_AGG_COUNT_STAR: case GG_AGG_COUNT_ANY: case GG_AGG_SUM_INT4: case GG_AGG_SUM_FLOAT8: case GG_AGG_AVG_FLOAT8:
		case GG_AGG_MIN_INT4: case GG_AGG_MIN_INT8: case GG_AGG_MIN_DATE: case GG_AGG_MIN_FLOAT8:
		case GG_AGG_MAX_INT4: case GG_AGG_MAX_INT8: case GG_AGG_MAX_DATE: case GG_AGG_MAX_FLOAT8:
			return 1;
		default:
			return 0;
	}
}

/* whether the result is a float8 (the word holds the double's bits; else the integer itself) */
GG_AGGFINAL_FN int gg_aggfinal_is_float8(int32_t aggfnoid)
{
	return aggfnoid == GG_AGG_SUM_FLOAT8 || aggfnoid == GG_AGG_AVG_FLOAT8 || aggfnoid == GG_AGG_MIN_FLOAT8 || aggfnoid == GG_AGG_MAX_FLOAT8;
}

/* The result of a covered aggregate as a 64-bit word, *isnull = whether it is NULL (then the word is 0).
 *   count  rows of the group (count(*))
 *   n      non-NULL inputs of the aggregate's accumulator column (ggp_grec::n)
 *   acc    that column's accumulator, its bits (ggp_grec::sum: the float8 sum / extreme, or the int64)
 * Strict aggregates over no input are NULL (int4_sum, float8pl, the min/max functions: state init NULL); avg(float8) is
 * float8_avg's sumX / N, where "+ 0.0" turns the -0 float8 sums start from into the +0 of float8_accum's "{0,0,0}"
 * (float.c:1995). */
GG_AGGFINAL_FN uint64_t gg_aggfinal(int32_t aggfnoid, uint64_t count, uint64_t n, uint64_t acc, int *isnull)
{
	union { uint64_t u; double d; } v;
	*isnull = 0;
	if (aggfnoid == GG_AGG_COUNT_STAR) return count;
	if (aggfnoid == GG_AGG_COUNT_ANY) return n;
	if (n == 0) { *isnull = 1; return 0; }
	if (aggfnoid != GG_AGG_AVG_FLOAT8) return acc;
	v.u = acc;
	v.d = (v.d + 0.0) / (double) n;
	return v.u;
}

#endif /* GG_AGGFINAL_H */
