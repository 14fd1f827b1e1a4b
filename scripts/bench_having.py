"""GROUP BY ... HAVING at the top of a slice: the Agg's groups finalised into device datum rows and filtered on the device by the row
filter (gg_rowfilter_run), so that only the surviving groups come to the host.  Prints the card and one JSON line.

Workload, on LI-narrow resident on the device (synthetic, 4 rows per order):
    SELECT l_orderkey, sum(l_quantity) FROM lineitem GROUP BY l_orderkey HAVING sum(l_quantity) > T
at each --rows size (default 2*10^7 and 10^8: 5*10^6 and 2.5*10^7 groups), for three thresholds T taken from the data: below
every group's sum (all pass), the 99th percentile (about 1 % pass) and the largest sum (none pass).

  e2e_ms:     the plan through the executor-node surface, host clock around ExecProcNode to end of stream after a ReScan (median of
              --reps after a warm-up run)
  filter_ms:  CUDA events around gg_rowfilter_run over the settled Agg's datum rows (its count pass, scan, one host read of the
              total and the error word, write pass)
  bytes:      the filter's algorithmic bytes: n x W x 8 read + n / 8 of pass bits + 2 x s x W x 8 for the s survivors read and
              written (W = 3 words a row); GB/s over filter_ms, against the data sheet's 3.35 TB/s
  baseline:   (only where the host path can hold the groups, <= 2^24) the same Agg without HAVING, every group fetched to the host
              (gg_scanagg_fetch) and filtered in NumPy (same clock, from the fetch on), and whether both give the same rows
Usage: python scripts/bench_having.py [--rows N ...] [--reps R]"""
import argparse
import ctypes as C
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

HOST_PATH_MAX_GROUPS = 1 << 24
PEAK_BYTES = 3.35e12
AGGVAL = np.dtype([("f", "<f8", 3), ("i", "<i8"), ("isnull", "<i4"), ("pad", "<i4")])
AGGROW = np.dtype([("key", "<i8", 4), ("keylen", "<i4", 4), ("keyisnull", "<i4", 4), ("agg", AGGVAL, 16)])


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def b2f(v):
    return struct.unpack("<d", struct.pack("<q", int(v)))[0]


class _View:
    """a datum-row relation handle for RowFilter.run_raw"""
    def __init__(self, h, nrows):
        self.h, self.nrows = h, nrows


def timed_rows(x, reps):
    ts, rows = [], None
    for i in range(reps + 1):
        if i:
            x.rescan()
        t0 = time.perf_counter()
        rows = x.rows()
        if i:
            ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts), rows


def run_size(eng, nrows, reps):
    from greengage_b200 import capi, tpch, executor as ex
    from greengage_b200.engine import Relation, RowFilter, ScanAgg
    lc = tpch.LI_NARROW_COLS
    norders = nrows // 4
    pages, nb, n = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, nrows, seed=3, norders=norders))
    rel = Relation(eng, host_pages=pages)
    del pages
    p = capi.ExprPool()
    scan = capi.make_scan(capi.synth_tupdesc(capi.TAB_LINEITEM_NARROW), -1)
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [p.var(lc["orderkey"], capi.INT8OID)], [(capi.AGG_SUM_FLOAT8, p.var(lc["quantity"], capi.FLOAT8OID))],
                        num_groups=norders)
    out = {"rows": n, "pages": nb, "thresholds": []}
    # the groups' sums, to take the thresholds from the data
    sa = ScanAgg(eng, scan, agg, p.pool)
    sa.run(rel)
    vals, _ = sa.datumrows()
    ngroups = len(vals)
    sums = vals[:, 1].view(np.float64)
    out["groups"] = ngroups
    for label, t in (("all", float(sums.min()) - 1.0), ("1pct", float(np.quantile(sums, 0.99))), ("none", float(sums.max()))):
        q = p.func(capi.F_FLOAT8GT, capi.BOOLOID, p.var(2, capi.FLOAT8OID), p.const(capi.FLOAT8OID, t))
        r = {"T": t, "label": label}
        rows = None
        if label != "all":
            # (every group to Python slots one by one would time the interpreter, not the plan: "all" times the filter only)
            b = ex.PlanBuilder()
            x = ex.Executor(eng, p.pool, [rel], b.agg(b.seqscan(0, scan.desc), agg, having=q))
            r["e2e_ms"], rows = timed_rows(x, reps)
            x.end()
        # the filter call alone, over the settled Agg's rows
        h, cnt = C.c_void_p(), C.c_uint64(0)
        capi.check(capi.dev_lib().gg_scanagg_datumrows(sa.h, C.byref(h), C.byref(cnt)))
        f = RowFilter(eng, capi.rows_tupdesc([capi.INT8OID, capi.FLOAT8OID]), q, p.pool)
        fms = []
        for i in range(reps + 1):
            eng.sync()
            eng.timer_start()
            _, m = f.run_raw(_View(h, cnt.value))
            ms = eng.timer_stop()
            if i:
                fms.append(ms)
        f.free()
        s = m
        assert rows is None or len(rows) == s, (len(rows), s)
        r["survivors"], r["fraction"] = s, round(s / max(ngroups, 1), 5)
        W = 3
        fbytes = ngroups * W * 8 + ngroups // 8 + 2 * s * W * 8
        r["filter_ms"] = round(statistics.median(fms), 3)
        r["filter_bytes"] = fbytes
        r["filter_gb_per_s"] = round(fbytes / (r["filter_ms"] / 1e3) / 1e9, 1)
        r["filter_share_of_3.35TB/s"] = round(fbytes / (r["filter_ms"] / 1e3) / PEAK_BYTES, 3)
        if rows is None:
            r["e2e_ms"], r["baseline_host_filter_ms"], r["parity"] = "not measured", "not measured", "not checked"
            out["thresholds"].append(r)
            continue
        got = sorted((int(v[0]), b2f(v[1])) for v, nl, ty, ln in rows)
        if ngroups <= HOST_PATH_MAX_GROUPS:
            # what a caller has today: every group fetched to the host (gg_scanagg_fetch), then filtered in NumPy
            base = ScanAgg(eng, scan, agg, p.pool)
            ts = []
            for i in range(reps + 1):
                base.reset()
                base.run(rel)
                eng.sync()
                t0 = time.perf_counter()
                raw, m, _, _ = base.fetch_raw(norders + 1024)
                a = np.frombuffer(raw, dtype=AGGROW, count=m)
                k, sm = a["key"][:, 0], a["agg"][:, 0]["f"][:, 0]
                keep = sm > t
                kept = (k[keep].copy(), sm[keep].copy())
                if i:
                    ts.append((time.perf_counter() - t0) * 1e3)
            base.free()
            r["baseline_host_filter_ms"] = round(statistics.median(ts), 3)
            r["parity"] = got == sorted(zip(kept[0].tolist(), kept[1].tolist()))
        else:
            r["baseline_host_filter_ms"] = "not run: %d groups, the host path holds at most 2^24" % ngroups
            r["parity"] = "checked against gg_rowfilter_run's count only"
        r["e2e_ms"] = round(r["e2e_ms"], 3)
        out["thresholds"].append(r)
    sa.free()
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
    print(json.dumps({"bench": "having", "card": c, "sizes": res}))


if __name__ == "__main__":
    main()
