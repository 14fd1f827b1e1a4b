/*
 * gg_groups.h — device-resident group records: what an Agg pipeline holds before anything is fetched to the host, and
 * what a Motion of aggregate rows moves (include/ggb200.h gg_groups_*, gg_ic_motion_groups).
 *
 * The reference hands partial-aggregate rows from node to node as TupleTableSlots (nodeAgg.c:1736 agg_retrieve_hash_table
 * -> ExecMotion -> the FINAL Agg's advance_aggregates); here the rows of a slice stay on the device as ggp_grec records
 * in the layout of the pipeline that produced them (deduplicated accumulator columns, gg_program.h), and only the node at
 * the top of the slice turns them into Datums.
 */
#pragma once
#include <cuda_runtime.h>
#include "gg_engine.h"
#include "gg_program.h"

#define GG_IC_GROUP_CAP GGP_FAST_GROUPS      /* group records one segment sends in the fixed-size block of a Motion */

struct gg_groupstatus {                       /* same layout as gg_scanagg::Status */
	uint32_t err;
	int n;
	unsigned long long counters[2];
};

struct gg_groups {
	gg_engine *eng = nullptr;
	ggp_grec *recs = nullptr;                 /* device */
	int cap = 0;                              /* record slots */
	bool sparse = false;                      /* false: records [0, *d_n) are valid; true: a slot counts iff its `valid` is set */
	int *d_n = nullptr;                       /* dense only: device count (= &d_status->n) */
	gg_groupstatus *d_status = nullptr;       /* error flags / rows scanned / rows passed travelling with the records */
	int alloc_cap = 0;                        /* owned: record slots actually allocated (pooled buffers are GG_GROUPS_POOL_CAP wide) */
	int *scratch = nullptr;                   /* owned: 2 x alloc_cap ints for the merge kernel */
	bool empty_is_empty = false;              /* rows of a segment that does not receive the Gather: no empty-input aggregate row */
	bool owned = false;                       /* recs / d_status are this object's allocations (else: a view into a pipeline) */
	/* how to read the records (copied from the producing pipeline) */
	gg_agg agg;                               /* the Agg node that produced them (aggstage says what a row means) */
	ggp_aggmap aggmap[GG_MAX_AGGS];
	int nkeys = 0, nacc = 0;
	uint8_t keytype[GG_MAX_KEYS];
	uint8_t acckind[GGP_MAX_ACCS];
	int32_t keytypid[GG_MAX_KEYS];            /* type OIDs of the grouping columns */
	/* gg_groups_datumrows: the finalised groups as datum rows (owned by this object, also when it is a view) */
	gg_relation *rows_buf = nullptr;
	gg_relation *rows_view = nullptr;
	uint64_t rows_n = 0;
};

/* a new owned set with the metadata of `like` */
gg_groups *gg_groups_alloc(gg_engine *e, const gg_groups *like, int cap, bool sparse);
extern "C" void gg_groups_free(gg_groups *g);
