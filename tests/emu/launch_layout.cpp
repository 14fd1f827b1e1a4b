/*
 * launch_layout.cpp — TEST INFRASTRUCTURE.  The product's plan compiler (gg_compile.cpp) and launch configuration rules
 * (gg_launch.h) on the CPU: tests/test_launch_layout.py pins the configuration every role of the scan kernel is launched with.
 * out[] = threads, ctas, nstage, team, gcap, regslots, scratch_per_warp, scratch_off, cnt_off, acc_off, smem.
 */
#include "../../greengage_b200/csrc/gg_launch.h"

void gg_set_error(const char *, ...) {}

static void put(const gg_launch &c, int64_t *out)
{
	const int64_t v[] = { c.threads, c.ctas, c.nstage, c.team, c.gcap, c.regslots, c.scratch_per_warp, c.scratch_off, c.cnt_off, c.acc_off,
	                      (int64_t) c.smem };
	for (int i = 0; i < 11; i++) out[i] = v[i];
}

/* the scan+agg pipeline's kernel in variant `mode`; regslots_rule: what gg_priv_regslots says for the plan */
extern "C" int layout_scanagg(const gg_scan *scan, const gg_agg *agg, const gg_exprpool *pool, int mode, int chunks_per_page,
                              int items_per_page, int regslots_rule, int64_t smem_optin, int64_t *out)
{
	ggp_program P;
	ggp_aggmap aggmap[GG_MAX_AGGS];
	char msg[256];
	if (ggp_compile_scanagg(scan, agg, pool, &P, aggmap, msg, sizeof msg)) return -1;
	gg_launch c;
	if (!gg_scan_config(c, mode, false, P, chunks_per_page, items_per_page, regslots_rule, (size_t) smem_optin)) return -2;
	put(c, out);
	return 0;
}

/* a join: its probe kernel in variant `mode` (gg_joinagg_create's program), its build kernel (gg_joinagg_build's scratch) */
extern "C" int layout_join(const gg_scan *outer, const gg_scan *inner, const gg_hashjoin *hj, const gg_agg *agg, const gg_exprpool *pool,
                           int mode, int chunks_per_page, int64_t smem_optin, int64_t *probe, int64_t *build)
{
	ggp_joinprog jp;
	ggp_aggmap aggmap[GG_MAX_AGGS];
	char msg[256];
	if (ggp_compile_join(outer, inner, hj, agg, pool, &jp, aggmap, msg, sizeof msg)) return -1;
	ggp_program P = jp.probe;
	P.nullable = P.nullable || jp.build.nullable;
	gg_launch c;
	if (!gg_scan_config(c, mode, true, P, chunks_per_page, 0, 0, (size_t) smem_optin)) return -2;
	put(c, probe);
	put(gg_np_launch(2, ((jp.build.outer.ncols * 64 + 15) & ~15) + 16), build);
	return 0;
}

/* the sending Motion's kernel (gg_partition_rows's scratch: column offsets + the warp's claim windows) */
extern "C" int layout_motion(const gg_scan *scan, const gg_exprpool *pool, const int32_t *hashkeys, int nkeys, const int32_t *payload,
                             int npayload, int64_t *out)
{
	ggp_program P;
	uint8_t hashtype[GG_MAX_KEYS];
	char msg[256];
	if (ggp_compile_motion(scan, pool, hashkeys, nkeys, payload, npayload, &P, hashtype, msg, sizeof msg)) return -1;
	put(gg_np_launch(2, ((P.outer.ncols * 64 + 15) & ~15) + 512 + 16), out);
	return 0;
}
