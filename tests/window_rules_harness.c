/*
 * window_rules_harness.c — TEST INFRASTRUCTURE: the per-row rules of greengage_b200/csrc/gg_window.h compiled with gcc, so that
 * tests/test_window_rules.py holds them to the row-at-a-time reference (tests/window_ref.c) and to windowfuncs.c's ntile loop.
 */
#include <stdint.h>
#include "../greengage_b200/csrc/gg_window.h"

/* window_ntile's loop (windowfuncs.c:211-276) against the closed form, for every total <= maxtotal and n <= maxn: mismatches */
int64_t ntile_mismatches(int64_t maxtotal, int32_t maxn)
{
	int64_t bad = 0;
	for (int64_t total = 1; total <= maxtotal; total++)
		for (int32_t n = 1; n <= maxn; n++)
		{
			int32_t ntile = 1;
			int64_t rows_per_bucket = 0, boundary = total / n, remainder = 0;
			if (boundary <= 0) boundary = 1;
			else { remainder = total % n; if (remainder != 0) boundary++; }
			for (int64_t k = 0; k < total; k++)
			{
				rows_per_bucket++;
				if (boundary < rows_per_bucket)
				{
					if (remainder != 0 && ntile == remainder) { remainder = 0; boundary -= 1; }
					ntile += 1;
					rows_per_bucket = 1;
				}
				if (ggw_ntile(total, n, k) != ntile) bad++;
			}
		}
	return bad;
}

/* the rules over rows whose partition [ps, pe) and peer group [gs, ge) are given */
void rules_rows(int32_t opt, int64_t m, const int64_t *ps, const int64_t *pe, const int64_t *gs, const int64_t *ge, int64_t *rownum,
                int64_t *rank, double *prank, double *cdist, int64_t *head, int64_t *tail, int32_t nt, int32_t *ntile, int64_t lagoff,
                int64_t *lagrow)
{
	for (int64_t j = 0; j < m; j++)
	{
		ggw_bounds b;
		int64_t t;
		b.ps = ps[j]; b.pe = pe[j]; b.gs = gs[j]; b.ge = ge[j];
		rownum[j] = ggw_row_number(j, b);
		rank[j] = ggw_rank(b);
		prank[j] = ggw_percent_rank(b);
		cdist[j] = ggw_cume_dist(b);
		ggw_frame(opt, j, b, &head[j], &tail[j]);
		ntile[j] = ggw_ntile(b.pe - b.ps, nt, j - b.ps);
		lagrow[j] = ggw_leadlag(j, lagoff, 0, b, &t) ? t : -1;
	}
}
