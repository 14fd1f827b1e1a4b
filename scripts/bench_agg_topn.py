"""ORDER BY ... LIMIT over an Agg with many groups: the groups finalised into device datum rows and selected by the bounded
device sort (the new path), against the sequence the executor ran before (every group fetched to the host as a gg_aggrow, turned
into host Datum rows, copied back for gg_sort_rows_bounded).  Prints the card and one JSON line.

Workload, on LI-narrow resident on the device (synthetic, 4 rows per order):
    SELECT l_orderkey, count(*), sum(l_extendedprice) FROM lineitem GROUP BY l_orderkey ORDER BY 3 DESC, 1 LIMIT 10
at each --rows size (default 2*10^7 and 10^8: 5*10^6 and 2.5*10^7 groups).

  new:       Limit <- Sort <- Agg <- SeqScan through the executor-node surface, end to end (host clock around ExecProcNode to end
             of stream after a ReScan; median of --reps after a warm-up)
  old:       gg_scanagg_fetch of all groups + host rows + gg_sort_rows_bounded, end to end (same clock); only up to 2^24 groups,
             the most the host path holds — "not run" above that
  finalise:  CUDA events around gg_scanagg_datumrows on a settled HashAggregate (its count, scan and write kernels, with the one
             host read of the group count in between), and the algorithmic bytes over that time: the hash table once
             (cap x stride x 8) + (1 + ncols) x 8 bytes written per group
  parity:    the new top 10 against the old one (keys and counts equal, sums within 1e-12 relative: the HashAggregate's float8
             sums depend on the order of its atomic adds)
Usage: python scripts/bench_agg_topn.py [--rows N ...] [--reps R]"""
import argparse
import json
import os
import statistics
import struct
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HOST_PATH_MAX_GROUPS = 1 << 24                         # the host path's row buffer stops growing there (GG_ERR_NOMEM)
AGGVAL = np.dtype([("f", "<f8", 3), ("i", "<i8"), ("isnull", "<i4"), ("pad", "<i4")])
AGGROW = np.dtype([("key", "<i8", 4), ("keylen", "<i4", 4), ("keyisnull", "<i4", 4), ("agg", AGGVAL, 16)])


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def plan(capi, tpch, ngroups):
    lc = tpch.LI_NARROW_COLS
    p = capi.ExprPool()
    scan = capi.make_scan(capi.synth_tupdesc(capi.TAB_LINEITEM_NARROW), -1)
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [p.var(lc["orderkey"], capi.INT8OID)],
                        [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_FLOAT8, p.var(lc["extendedprice"], capi.FLOAT8OID))], num_groups=ngroups)
    keys = [capi.make_sortkey(2, capi.FLOAT8OID, desc=True), capi.make_sortkey(0, capi.INT8OID)]
    return p, scan, agg, keys


def b2f(v):
    return struct.unpack("<d", struct.pack("<q", int(v)))[0]


def run_size(eng, nrows, reps):
    from greengage_b200 import capi, tpch, executor as ex
    from greengage_b200.engine import Relation, ScanAgg
    import ctypes as C
    norders = nrows // 4
    pages, nb, n = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, nrows, seed=3, norders=norders))
    rel = Relation(eng, host_pages=pages)
    del pages
    p, scan, agg, keys = plan(capi, tpch, norders)
    out = {"rows": n, "pages": nb}

    # new path: through the node surface
    b = ex.PlanBuilder()
    x = ex.Executor(eng, p.pool, [rel], b.limit(b.sort(b.agg(b.seqscan(0, scan.desc), agg), keys), 10))
    ts, new_top = [], None
    for i in range(reps + 1):
        if i:
            x.rescan()
        t0 = time.perf_counter()
        rows = x.rows()
        t = (time.perf_counter() - t0) * 1e3
        if i:
            ts.append(t)
        new_top = [(int(v[0]), int(v[1]), b2f(v[2])) for v, nl, ty, ln in rows]
    out["new_ms"] = round(statistics.median(ts), 3)
    out["locations"] = x.locations()
    x.end()

    # the finalise kernels alone, on a settled HashAggregate
    sa = ScanAgg(eng, scan, agg, p.pool)
    fin = []
    ngroups = 0
    for i in range(reps + 1):
        sa.reset()
        sa.run(rel)                                         # numGroups = the groups: the HashAggregate from the start, no replay
        eng.sync()
        eng.timer_start()
        h, cnt = C.c_void_p(), C.c_uint64(0)
        capi.check(capi.dev_lib().gg_scanagg_datumrows(sa.h, C.byref(h), C.byref(cnt)))
        ms = eng.timer_stop()
        ngroups = cnt.value
        if i:
            fin.append(ms)
    variant = sa.variant() & 15
    sa.free()
    cap = 65536
    while cap < 2 * norders:
        cap <<= 1
    stride = 4                                             # key, count, sum + the header word, on 32-byte sectors
    W = 1 + 1 + 2
    fbytes = cap * stride * 8 + ngroups * W * 8
    fms = statistics.median(fin)
    out["finalise"] = {"ms": round(fms, 3), "groups": ngroups, "hash_variant": variant == 5, "table_slots": cap,
                       "algorithmic_bytes": fbytes, "gb_per_s": round(fbytes / (fms / 1e3) / 1e9, 1)}

    # old path: fetch everything, host rows, bounded host-row sort
    if norders > HOST_PATH_MAX_GROUPS:
        out["old_ms"] = "not run: %d groups, the host path holds at most 2^24" % norders
        out["parity"] = "not checked (no old path)"
    else:
        sa = ScanAgg(eng, scan, agg, p.pool)
        ts, old_top = [], None
        for i in range(reps + 1):
            sa.reset()
            sa.run(rel)
            eng.sync()
            t0 = time.perf_counter()
            raw, m, _, _ = sa.fetch_raw(norders + 1024)
            a = np.frombuffer(raw, dtype=AGGROW, count=m)
            vals = np.empty((m, 3), dtype=np.int64)
            vals[:, 0] = a["key"][:, 0]
            vals[:, 1] = a["agg"][:, 0]["i"]
            vals[:, 2] = a["agg"][:, 1]["f"][:, 0].view(np.int64)
            ka = (capi.gg_sortkey * 2)(*keys)
            perm = np.zeros(10, dtype=np.uint64)
            nperm = C.c_uint64(0)
            capi.check(capi.dev_lib().gg_sort_rows_bounded(eng.h, ka, 2, 3, vals.ctypes.data, None, m, 10, perm.ctypes.data, C.byref(nperm)))
            t = (time.perf_counter() - t0) * 1e3
            if i:
                ts.append(t)
            old_top = [(int(vals[j, 0]), int(vals[j, 1]), b2f(vals[j, 2])) for j in perm[:nperm.value].astype(np.int64)]
        sa.free()
        out["old_ms"] = round(statistics.median(ts), 3)
        out["parity"] = len(new_top) == len(old_top) == 10 and all(
            a[0] == b[0] and a[1] == b[1] and abs(a[2] - b[2]) <= 1e-12 * abs(b[2]) for a, b in zip(new_top, old_top))
    out["top3"] = new_top[:3]
    rel.free()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, nargs="+", default=[2 * 10 ** 7, 10 ** 8])
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    from greengage_b200.engine import Engine
    c = card()
    print("card:", c, flush=True)
    eng = Engine(0)
    res = [run_size(eng, n, a.reps) for n in a.rows]
    eng.close()
    print(json.dumps({"bench": "agg_topn", "card": c, "sizes": res}))


if __name__ == "__main__":
    main()
