/*
 * ggb200_mock_topn.c — TEST INFRASTRUCTURE: the bounded sorts of the C-ABI for the oracle-backed stand-in of libggb200.so
 * (tests/mock/ggb200_mock.c).  Linked next to it by tests/test_executor_limit.py, so that a Limit over a Sort runs through the
 * product's gg_executor.c on a CPU-only box.  Never shipped, never loaded by the product.
 */
#include <stdlib.h>
#include <string.h>
#include "../../include/ggb200.h"
#include "../../oracle/gg_oracle.h"

void gg_set_error(const char *fmt, ...);          /* ggb200_mock.c */

/* the bounded sort's contract: the first min(bound, n) entries of the whole sort's permutation */
int gg_sort_rows_bounded(gg_engine *e, const gg_sortkey *keys, int nkeys, int ncols, const int64_t *host_rows, const uint8_t *host_nulls,
                         uint64_t n, uint64_t bound, uint64_t *host_perm, uint64_t *nperm)
{
	uint64_t *all = malloc(8 * (size_t) (n ? n : 1));
	const uint64_t cnt = bound < n ? bound : n;
	int rc;
	(void) e;
	if (!all) { gg_set_error("mock: out of memory"); return GG_ERR_NOMEM; }
	rc = or_sort_perm(keys, nkeys, ncols, host_rows, host_nulls, n, all);
	if (rc == 0) { memcpy(host_perm, all, 8 * (size_t) cnt); *nperm = cnt; }
	else gg_set_error("mock: or_sort_perm failed");
	free(all);
	return rc == 0 ? GG_OK : (rc == OR_ERR_NOMEM ? GG_ERR_NOMEM : rc);
}

/* device-resident rows have no stand-in (as gg_sort_datumrows in ggb200_mock.c) */
int gg_sort_datumrows_bounded(gg_engine *e, const gg_sortkey *keys, int nkeys, int ncols, const void *rows, uint64_t n, uint64_t bound, void *out,
                              uint64_t *nout, int *passes)
{
	(void) e; (void) keys; (void) nkeys; (void) ncols; (void) rows; (void) n; (void) bound; (void) out; (void) nout; (void) passes;
	gg_set_error("mock: no device-resident results");
	return GG_ERR_UNSUPPORTED;
}
