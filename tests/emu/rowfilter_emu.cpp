/*
 * rowfilter_emu.cpp — the per-row step of the row filter (gg_rowfilter, an Agg's HAVING) compiled for the host: the plan
 * compiler's ggp_compile_filter and gg_device.cuh's datumrow_passes, run row by row over datum rows in an emulated shared
 * memory (tests/test_having_compile.py holds it to the oracle's qual evaluation).
 */
#include "gg_host_emu.h"
#include "../../greengage_b200/csrc/gg_device.cuh"

uint8_t gg_emu_smem[GG_EMU_SMEM_BYTES];

extern "C" {

/* compile only: the return code, the message and the program listing */
int emu_filter_compile(const gg_tupdesc *desc, int32_t qual, const gg_exprpool *pool, char *listing, int cap, char *err, int errlen)
{
	static ggp_program prog;
	gg_scan scan;
	memset(&scan, 0, sizeof scan);
	scan.desc = *desc;
	scan.qual = qual;
	const int rc = ggp_compile_filter(&scan, pool, &prog, err, errlen);
	if (listing && cap > 0) { listing[0] = 0; if (rc == 0) ggp_disasm(&prog, listing, cap); }
	return rc;
}

/* rows: n datum rows of 1 + desc->natts words; pass[i] = whether row i passes; *errflags = the OR of the rows' error flags */
int emu_filter_run(const gg_tupdesc *desc, int32_t qual, const gg_exprpool *pool, const uint64_t *rows, uint64_t n, uint8_t *pass,
                   uint32_t *errflags, char *err, int errlen)
{
	static ggp_program prog;
	gg_scan scan;
	memset(&scan, 0, sizeof scan);
	scan.desc = *desc;
	scan.qual = qual;
	const int rc = ggp_compile_filter(&scan, pool, &prog, err, errlen);
	if (rc) return rc;
	const uint64_t W = 1 + (uint64_t) desc->natts;
	uint32_t e = 0;
	for (uint64_t i = 0; i < n; i++)
	{
		memcpy(gg_emu_smem, rows + i * W, W * 8);
		pass[i] = ggd::datumrow_passes(prog, 0, true, 0, e) ? 1 : 0;
	}
	*errflags = e;
	return 0;
}

}
