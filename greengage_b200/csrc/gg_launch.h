/*
 * gg_launch.h — launch configuration of the scan kernel body (gg_scanagg_kernel.cuh) in each of its roles: block size, ring
 * stages, teams, group capacity, register slots and the dynamic shared-memory layout.  Arithmetic only, no CUDA, so that a
 * CPU test compiles it (tests/test_launch_layout.py).
 */
#pragma once
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include "gg_program.h"

/* kernel roles: the MODE_* of gg_scanagg_kernel.cuh (gg_scanagg.cu checks that they agree) */
enum { GGL_PRIV = 0, GGL_TR = 1, GGL_TRN = 2, GGL_BUILD = 3, GGL_PART = 4, GGL_HASH = 5 };

/* Launch configuration of the kernels that run two small blocks per SM by default (hash build, Motion send, general
 * HashAggregate, the transposed / nullable scan and probe variants): consumer warps per block, ring stages, team size
 * (ScanAggParams.team) and blocks per SM.  GGB200_NP_CONFIG="ncons,stages,team,ctas" overrides it for experiments; block
 * sizes other than the default need the run-time specialised kernel (the interpreter kernels are built for 256 threads). */
struct gg_npconfig { int ncons, nstage, team, ctas; bool forced; };
static inline gg_npconfig gg_np_config(int ncons, int nstage)
{
	gg_npconfig c = { ncons, nstage, 0, 2, false };
	const char *env = getenv("GGB200_NP_CONFIG");
	int a, b, t = 0, k = 2;
	if (env && sscanf(env, "%d,%d,%d,%d", &a, &b, &t, &k) >= 2 && a >= 1 && a <= 30 && b >= 2 && b <= 6 && t >= 0 && t <= a && k >= 1 && k <= 4)
	{ c.ncons = a; c.nstage = b; c.team = t; c.ctas = k; c.forced = true; }
	/* at most one team per ring slot (a team's pages arrive on its own barrier set, BlockTable::teamfull) */
	if (c.team > 0 && c.ncons / c.team > c.nstage) c.ncons = c.team * c.nstage;
	return c;
}

/* one launch shape of the scan kernel body */
struct gg_launch {
	int threads = 0, ctas = 2, nstage = 0;
	int team = 0;                   /* consumer warps per team (ScanAggParams.team); 0: chunks dealt across all warps */
	int gcap = 0;                   /* groups a block holds on chip */
	int regslots = -1;              /* private-accumulator variant: trailing value slots kept in registers (-1: not decided) */
	int scratch_per_warp = 0;
	bool forced = false;            /* the shape came from GGB200_NP_CONFIG */
	uint32_t scratch_off = 0, cnt_off = 0, acc_off = 0;
	size_t smem = 0;
};

#define GG_BLOCKTABLE_BYTES 1448          /* sizeof(ggd::BlockTable); gg_scanagg.cu checks it */

/* ring[nstage][32 KB] | full/empty mbarriers | BlockTable | per-warp scratch: where the scratch starts, and the fixed part of
 * the dynamic shared memory (everything up to the end of the scratch) */
struct gg_ring { uint32_t scratch_off; size_t fixed; };
static inline gg_ring gg_ring_layout(int nstage, int ncons, int scratch_per_warp)
{
	const size_t off = ((size_t) nstage * GG_BLCKSZ + (size_t) nstage * 16 + GG_BLOCKTABLE_BYTES + 15) & ~(size_t) 15;
	return { (uint32_t) off, off + (size_t) ncons * scratch_per_warp };
}

/* a role that runs two small blocks per SM: gg_np_config's shape on the ring layout, nothing behind the scratch */
static inline gg_launch gg_np_launch(int nstage, int scratch_per_warp)
{
	const gg_npconfig nc = gg_np_config(7, nstage);
	gg_launch c;
	c.ctas = nc.ctas;
	c.threads = (nc.ncons + 1) * 32;
	c.nstage = nc.nstage;
	c.team = nc.team;
	c.forced = nc.forced;
	c.regslots = 0;
	c.scratch_per_warp = scratch_per_warp;
	const gg_ring r = gg_ring_layout(c.nstage, nc.ncons, scratch_per_warp);
	c.scratch_off = r.scratch_off;
	c.smem = r.fixed;
	return c;
}

/* Launch configuration of the scan+agg pipeline's kernel (the probe kernel when `join`) in variant `mode`, for pages of
 * `chunks_per_page` 32-row chunks and `items_per_page` line pointers (0: not sampled).  c.regslots < 0: not decided yet, then
 * `regslots_rule` (gg_priv_regslots) and the page density decide.  The layout:
 *   ring[nstage][32 KB] | full/empty mbarriers | BlockTable | per-warp scratch | (PRIV) counts | (PRIV) sums
 * Returns false when the plan needs more shared memory than a block has. */
static inline bool gg_scan_config(gg_launch &c, int mode, bool join, const ggp_program &P, int chunks_per_page, int items_per_page,
                                  int regslots_rule, size_t smem_optin)
{
	const int V = P.nslots > 0 ? P.nslots : 1;
	int scr = (P.outer.ncols * 64 + 15) & ~15;                   /* column offsets [ncols][32] u16 */
	if (mode == GGL_TR || mode == GGL_TRN) scr += V * 33 * 8 + 128 + 128;      /* + transposed values, group ids, null masks */
	if (mode == GGL_PART) scr += 512;                            /* + the warp's row claim windows (the probe that writes rows) */
	scr = (scr + 15) & ~15;
	/* datum-row plans can be fed from column files (gg_scanagg_run_aocs): 32 staged rows per warp at the tail of its scratch */
	if (P.outer.rowwords) scr += 32 * ((P.outer.rowwords | 1) * 8);
	const int spw = (scr + 15) & ~15;
	if (mode != GGL_PRIV)
	{
		/* 2 CTAs/SM x (7 consumer warps + producer = 8 warps) unless configured otherwise */
		c = gg_np_launch(3, spw);
		const size_t per_cta = (smem_optin + 1024) / (size_t) c.ctas - 1024;   /* 1 KB reserved per CTA */
		if (c.smem > per_cta && !c.forced) c = gg_np_launch(2, spw);
		if (c.smem > per_cta) return false;
		const int ncons = c.threads / 32 - 1;
		c.gcap = GGP_MAX_PAIRS / V < GGP_FAST_GROUPS ? GGP_MAX_PAIRS / V : GGP_FAST_GROUPS;
		if (c.smem < 32 * 1024) c.smem = 32 * 1024;             /* the epilogue reuses the ring as reduction scratch */
		if ((size_t) ncons * GGP_MAX_PAIRS * 24 > c.smem) c.smem = (size_t) ncons * GGP_MAX_PAIRS * 24;    /* Red[ncons][GGP_MAX_PAIRS] */
		return true;
	}
	/* shared memory of `w` consumer warps on a ring of `stages` with private accumulators for 4 groups of `nslots` value slots
	 * (+ 40 bytes: the alignment slack the rules below were measured with) */
	auto need = [&](int stages, int w, int nslots) {
		return gg_ring_layout(stages, w, spw).fixed + 40 + (size_t) w * 32 * (8 * nslots + 4) * 4;
	};
	/* value slots that need shared memory: the private-accumulator variant keeps the last few in registers when a
	 * plan-specialised kernel is available and the planner expects no more groups than the registers hold */
	if (c.regslots < 0)
	{
		/* Measured with scripts/dev_regs.sh (10^8-row lineitem-wide): register slots cost a few predicated adds per row
		 * but free shared memory — Q1 one-stage: 20 warps instead of 16 on the 4-page ring; Q1 PARTIAL stage (8 value
		 * slots): 16 warps / 4 pages instead of 13 / 3, both faster.  Dense pages run on a 3-page ring where everything
		 * fits anyway, and there the plain layout is faster. */
		c.regslots = regslots_rule;
		/* dense pages: plain layout whenever it leaves room for (nearly) all 20 warps on the 3-page ring */
		if (chunks_per_page >= 10 && need(3, 18, P.nslots) <= smem_optin) c.regslots = 0;
	}
	const int nslots = P.nslots - c.regslots;
	c.scratch_per_warp = spw;
	c.forced = false;
	c.nstage = 3;
	/* 1 CTA/SM: 14 consumer warps + producer.  What the ring and the scratch leave of the 227 KB goes to
	 * the per-thread private accumulators; that fixes how many groups this variant holds. */
	c.ctas = 1;
	/* Measured on 10^8-row lineitem (scripts/dev_sweep.sh): sparse pages (190 rows = 6 chunks of 32 line pointers)
	 * need pages in flight more than warps -> 16 consumer warps on a 4-page ring (faster than 20 warps / 3 pages);
	 * dense pages (430 rows = 14 chunks) keep every warp busy from fewer pages -> 20 warps on a 3-page ring
	 * (faster than 16 warps / 4 pages).  Fewer warps if the private accumulators of >= 4 groups need the room. */
	auto fit = [&](int stages, int want) {           /* most consumer warps (<= want) whose accumulators of 4 groups fit */
		int w = want;
		for (; w > 4; w--)
			if (need(stages, w, nslots) <= smem_optin) break;
		return w;
	};
	int ncons;
	if (chunks_per_page >= 10) { c.nstage = 3; ncons = fit(3, 20); }
	else
	{
		/* plans with many value slots (a PARTIAL-stage Q1 carries 8): when 4 stages leave room for fewer than 15
		 * warps, a 3-page ring with more warps measured faster (13 warps / 3 pages against 9 / 4) */
		c.nstage = 4; ncons = fit(4, c.regslots > 0 ? 20 : 16);
		/* a fifth page in flight when it costs no warp (measured faster for one-stage Q1 with register slots) */
		if (fit(5, ncons) >= ncons) c.nstage = 5;
		if (ncons < 15) { int w3 = fit(3, 16); if (w3 >= ncons + 3) { c.nstage = 3; ncons = w3; } }
	}
	{
		const char *cfg = getenv("GGB200_PRIV_CONFIG");     /* "conswarps,stages[,team[,ctas]]" for experiments */
		int a, b, t = 0, d = 1;
		c.team = 0;
		/* Teams (gg_scanagg_kernel.cuh): sparse pages — every chunk of a page gets its own warp, the teams work on different
		 * pages of the ring.  The team must cover the fullest page (a warp with two chunks holds its whole team back): the
		 * sampled page's line pointers + 8 %.  Measured on 10^8-row lineitem-wide (190 +- 6 rows per page, scripts/
		 * sweep_teams.py): 3 teams of 7 on a 5-page ring beat 20 warps dealt across pages, and teams of 6 (pages with 193+
		 * rows cost a warp two chunks) were slower than both. */
		if (chunks_per_page >= 2 && chunks_per_page <= 10 && items_per_page > 0 && !P.outer.rowwords && !join)
		{
			const int ts = (items_per_page + items_per_page / 12 + 31) / 32;
			int nteams = ts > 0 ? 21 / ts : 0;
			if (nteams > 5) nteams = 5;
			if (nteams >= 1 && ts <= 10)
			{
				const int want = ts * nteams;
				int st = 5;
				while (st > nteams && fit(st, want) < want) st--;
				if (st >= nteams && fit(st, want) >= want) { ncons = want; c.nstage = st; c.team = ts; }
			}
		}
		if (cfg && sscanf(cfg, "%d,%d,%d,%d", &a, &b, &t, &d) >= 2 && a >= 1 && a <= 30 && b >= 2 && b <= 6 && t >= 0 && t <= a && d >= 1 && d <= 2)
		{ ncons = a; c.nstage = b; c.team = t; c.ctas = d; }
		/* a team waits for ITS page's phase of a ring slot; an mbarrier tells the current phase from the previous one only,
		 * so no two teams may be queued on one slot: at most as many teams as stages */
		if (c.team > 0 && ncons / c.team > c.nstage) ncons = c.team * c.nstage;
	}
	c.threads = (ncons + 1) * 32;
	const int NT = ncons * 32;
	const gg_ring r = gg_ring_layout(c.nstage, ncons, spw);
	const size_t fixed = r.fixed + 24;                  /* + the alignment slack the group capacity was measured with */
	/* two blocks per SM (experiments: more warps in flight for the latency-bound probe): each gets half, 1 KB reserved per block */
	const size_t budget = c.ctas > 1 ? (smem_optin + 1024) / (size_t) c.ctas - 1024 : smem_optin;
	if (fixed + (size_t) NT * (8 * nslots + 4) > budget) return false;
	int gcap = (int) ((budget - fixed) / ((size_t) NT * (8 * nslots + 4)));
	if (gcap > GGP_FAST_GROUPS) gcap = GGP_FAST_GROUPS;
	if (c.regslots > 0 && gcap > 4 /* GG_REG_GROUPS */) gcap = 4;
	c.gcap = gcap;
	c.scratch_off = r.scratch_off;
	c.cnt_off = (uint32_t) r.fixed;
	c.acc_off = (c.cnt_off + (uint32_t) gcap * NT * 4 + 15) & ~15u;
	c.smem = c.acc_off + (size_t) gcap * nslots * NT * 8;
	return true;
}
