/*
 * ggb200_mock_window.c — TEST INFRASTRUCTURE: gg_window_* for the oracle-backed stand-in of libggb200.so (tests/mock/ggb200_mock.c),
 * answered by the row-at-a-time reference (tests/window_ref.c), plus the datum-row relations a WindowAgg node uploads its input to
 * and hands its output up in, kept in host memory, and a Sort of such rows (the oracle's sort), so that a Sort above a WindowAgg
 * runs.  Linked by tests/test_executor_window.py, with ggb200_mock.c compiled so that its refusing gg_relation_create /
 * _attach_rows / _read / _device_ptr / _free and gg_sort_datumrows step aside for the ones below.  Never shipped.
 */
#include <stdlib.h>
#include <string.h>
#include "../../include/ggb200.h"
#include "../../greengage_b200/csrc/gg_window.h"
#include "../../oracle/gg_oracle.h"

void gg_set_error(const char *fmt, ...);          /* ggb200_mock.c */
int ref_window(const gg_window *win, const int32_t *types, int ncols, const gg_exprpool *pool, const uint64_t *rows, uint64_t n,
               uint64_t *out, uint64_t *nout, char *err, int errlen);      /* tests/window_ref.c */

/* the layout of ggb200_mock.c's relation, and the buffer a relation created here owns */
struct gg_relation { const uint8_t *pages; uint64_t nblocks; uint8_t *owned; };

int gg_relation_create(gg_engine *e, uint64_t nblocks, gg_relation **out)
{
	gg_relation *r = calloc(1, sizeof *r);
	(void) e;
	if (!r || !(r->owned = calloc((size_t) (nblocks ? nblocks : 1), GG_BLCKSZ))) { free(r); gg_set_error("mock: out of memory"); return GG_ERR_NOMEM; }
	r->pages = r->owned; r->nblocks = nblocks;
	*out = r;
	return GG_OK;
}

int gg_relation_load(gg_relation *r, uint64_t first_block, const void *host_pages, uint64_t nblocks)
{
	if (!r->owned || nblocks > r->nblocks || first_block > r->nblocks - nblocks) { gg_set_error("mock: load outside the relation"); return GG_ERR_ARG; }
	memcpy(r->owned + first_block * GG_BLCKSZ, host_pages, (size_t) nblocks * GG_BLCKSZ);
	return GG_OK;
}

int gg_relation_attach_rows(gg_engine *e, void *rows, uint64_t nrows, int ncols, gg_relation **out)
{
	gg_relation *r = calloc(1, sizeof *r);
	(void) e;
	if (!r) { gg_set_error("mock: out of memory"); return GG_ERR_NOMEM; }
	r->pages = rows;
	{
		/* the device's view (gg_abi.cu): 32 KB chunks of whole rows, an even number of them each */
		const uint64_t per_chunk = (GG_BLCKSZ / (8ull * (1 + ncols))) & ~1ull;
		r->nblocks = (nrows + per_chunk - 1) / per_chunk;
	}
	*out = r;
	return GG_OK;
}

int gg_relation_read(gg_relation *r, uint64_t first_block, void *host_pages, uint64_t nblocks)
{
	if (nblocks > r->nblocks || first_block > r->nblocks - nblocks) { gg_set_error("mock: read outside the relation"); return GG_ERR_ARG; }
	memcpy(host_pages, r->pages + first_block * GG_BLCKSZ, (size_t) nblocks * GG_BLCKSZ);
	return GG_OK;
}

void *gg_relation_device_ptr(gg_relation *r) { return (void *) r->pages; }
void gg_relation_free(gg_relation *r) { if (r) { free(r->owned); free(r); } }

/* gg_sort_datumrows' contract: the live rows in the sorted order of or_sort_perm (stable) */
int gg_sort_datumrows(gg_engine *e, const gg_sortkey *keys, int nkeys, int ncols, const void *rows, uint64_t n, void *out, uint64_t *nlive,
                      int *passes)
{
	const uint64_t W = 1 + (uint64_t) ncols, *in = rows;
	int64_t *vals = calloc((size_t) (n ? n : 1) * (size_t) ncols, 8);
	uint8_t *nulls = calloc((size_t) (n ? n : 1) * (size_t) ncols, 1);
	uint64_t *live = calloc((size_t) (n ? n : 1), 8), *perm = calloc((size_t) (n ? n : 1), 8), m = 0;
	int rc = GG_ERR_NOMEM;
	(void) e;
	if (passes) *passes = 0;
	if (vals && nulls && live && perm)
	{
		for (uint64_t r = 0; r < n; r++)
		{
			if (in[r * W] & GG_DATUMROW_DEAD) continue;
			for (int c = 0; c < ncols; c++) { vals[m * ncols + c] = (int64_t) in[r * W + 1 + c]; nulls[m * ncols + c] = (in[r * W] >> c) & 1; }
			live[m++] = r;
		}
		rc = or_sort_perm(keys, nkeys, ncols, vals, nulls, m, perm);
		for (uint64_t i = 0; rc == 0 && i < m; i++) memcpy((uint64_t *) out + i * W, in + live[perm[i]] * W, 8 * W);
		*nlive = m;
	}
	free(vals); free(nulls); free(live); free(perm);
	if (rc) gg_set_error("mock: sort failed");
	return rc == 0 ? GG_OK : (rc == OR_ERR_NOMEM ? GG_ERR_NOMEM : rc);
}

struct gg_window_obj {
	gg_window win;
	gg_exprpool pool;
	int32_t types[GG_MAX_ATTS];
	int ncols;
	gg_relation *out, *view;
};

int gg_window_create(gg_engine *e, const gg_tupdesc *rows_desc, const gg_window *win, const gg_exprpool *pool, gg_window_obj **out)
{
	gg_window_obj *w;
	(void) e;
	if (!ggw_frame_supported(win->frameOptions)) { gg_set_error("mock: frame options 0x%x", win->frameOptions); return GG_ERR_UNSUPPORTED; }
	if (rows_desc->natts + win->numFuncs > GG_MAX_ATTS) { gg_set_error("mock: too many output columns"); return GG_ERR_UNSUPPORTED; }
	w = calloc(1, sizeof *w);
	if (!w) return GG_ERR_NOMEM;
	w->win = *win; w->pool = *pool; w->ncols = rows_desc->natts;
	for (int c = 0; c < w->ncols; c++) w->types[c] = rows_desc->attrs[c].atttypid;
	*out = w;
	return GG_OK;
}

int gg_window_run(gg_window_obj *w, gg_relation *rows, uint64_t nrows, gg_relation **out_view, uint64_t *nout)
{
	const uint64_t W2 = 1 + (uint64_t) w->ncols + (uint64_t) w->win.numFuncs;
	char err[256];
	int rc;
	gg_relation_free(w->out); gg_relation_free(w->view);
	w->out = w->view = NULL;
	rc = gg_relation_create(NULL, (nrows * W2 * 8 + 16 + GG_BLCKSZ - 1) / GG_BLCKSZ, &w->out);
	if (rc) return rc;
	rc = ref_window(&w->win, w->types, w->ncols, &w->pool, (const uint64_t *) rows->pages, nrows, (uint64_t *) w->out->owned, nout, err, sizeof err);
	if (rc) { gg_set_error("%s", err); return rc; }
	rc = gg_relation_attach_rows(NULL, w->out->owned, *nout, (int) W2 - 1, &w->view);
	if (rc) return rc;
	*out_view = w->view;
	return GG_OK;
}

void gg_window_free(gg_window_obj *w)
{
	if (!w) return;
	gg_relation_free(w->out); gg_relation_free(w->view);
	free(w);
}
