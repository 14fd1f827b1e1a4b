"""WindowAgg on the device over LI-narrow resident on the device (synthetic, 4 rows per order).  Prints the card and one JSON line.

Workloads, at each --rows size (default 2*10^7 and 10^8):
  (a) SELECT row_number() OVER (PARTITION BY l_orderkey ORDER BY l_extendedprice DESC) AS rn,
             sum(l_extendedprice) OVER (PARTITION BY l_orderkey)
      -- two WindowAgg nodes over one Sort (l_orderkey, l_extendedprice DESC); and the same with WHERE rn = 1 (top-1 per order),
      -- folded into the upper node's qual
  (b) SELECT sum(l_quantity) OVER (ORDER BY l_shipdate)
      -- one partition: one scan across every tile
The scan projects (l_orderkey, l_extendedprice, l_quantity, l_shipdate).

  window_ms:  CUDA events around gg_window_run (both calls for (a)) over the sorted rows: every kernel, the host read of the live
              count and of the error word (median of --reps after a warm-up)
  sort_ms:    CUDA events around gg_sort_datumrows of the same rows, for scale
  e2e_ms:     the plan through the executor-node surface with a Limit 10 on top (so that only ten rows cross to Python), host
              clock around ExecProcNode after a ReScan: scan projection, Sort, WindowAgg(s), qual
  bytes:      the window's algorithmic bytes, from shapes: the input rows read (n x W x 8), the output rows written (n x (W + f) x 8),
              and the scan arrays (each written once and read once: the packed partition / peer numbers, the two start arrays, per
              aggregate its prefix or segmented-scan array; sorted rows have no dead slot, so no compaction runs), W = 5 words (+ 1 for
              the upper window of (a)); GB/s over window_ms, against the data sheet's 3.35 TB/s
  baseline:   (at the first size only) the sorted rows fetched to the host and windowed by the row-at-a-time reference
              (tests/window_ref.c, compiled into a temporary directory), same clock; parity: integer and rank columns equal, float8
              sums within 1e-12 relative (positive inputs, different summation order)
Usage: python scripts/bench_window.py [--rows N ...] [--reps R]"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

PEAK_BYTES = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def window_bytes(n, W, funcs):
    """algorithmic bytes of one gg_window_run over n rows of W words with these (winfnoid, ...) functions"""
    from greengage_b200 import capi
    b = n * W * 8 + n * (W + len(funcs)) * 8
    b += 2 * n * 8 + 2 * 2 * n * 4             # packed partition / peer numbers + the two start arrays (a Sort's rows have no dead
                                               # slot, so the live positions and idx are not written)
    for fn, _, _ in funcs:
        if fn in (capi.AGG_SUM_FLOAT8, capi.AGG_AVG_FLOAT8, capi.AGG_MIN_FLOAT8, capi.AGG_MAX_FLOAT8):
            b += 2 * n * 8 + 2 * n * 8             # non-NULL count prefix + segmented scan
        elif fn in (capi.AGG_SUM_INT4,):
            b += 4 * n * 8
        elif fn == capi.AGG_COUNT_ANY:
            b += 2 * n * 8
    return b


def median_ms(fn, reps, eng):
    ts = []
    for i in range(reps + 1):
        eng.sync()
        eng.timer_start()
        fn()
        ms = eng.timer_stop()
        if i:
            ts.append(ms)
    return statistics.median(ts)


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


def run_size(eng, nrows, reps, baseline):
    from greengage_b200 import capi, tpch, executor as ex
    from greengage_b200.engine import Relation, RowRelation, Window, motion_partition
    lc = tpch.LI_NARROW_COLS
    pages, nb, n = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, nrows, seed=3, norders=nrows // 4))
    rel = Relation(eng, host_pages=pages)
    del pages
    desc = capi.synth_tupdesc(capi.TAB_LINEITEM_NARROW)
    names = ["orderkey", "extendedprice", "quantity", "shipdate"]
    types = [desc.attrs[lc[k] - 1].atttypid for k in names]
    p = capi.ExprPool()
    targets = [p.var(lc[k], types[i]) for i, k in enumerate(names)]
    W = 1 + len(names)
    out = {"rows": n, "pages": nb}
    # the scan's projected rows, as the row-producing SeqScan writes them (one destination)
    cap = n + n // 4 + 8192
    rows_buf = Relation(eng, nblocks=(cap * W * 8 + 64 + capi.GG_BLCKSZ - 1) // capi.GG_BLCKSZ)
    counts, _ = motion_partition(eng, capi.make_scan(desc, -1), p.pool, [targets[0]], targets, 1, rel, rows_buf.device_ptr(), cap)
    m = counts[0]
    sorted_buf = Relation(eng, nblocks=(m * W * 8 + 64 + capi.GG_BLCKSZ - 1) // capi.GG_BLCKSZ)
    L = capi.dev_lib()
    price, qty = p.var(2, capi.FLOAT8OID), p.var(3, capi.FLOAT8OID)
    rn = p.var(len(names) + 2, capi.INT8OID)     # row_number in the upper node's output: the 4 columns, the sum, then rn
    work = {
        "a_rownumber_and_partition_sum": ([capi.make_sortkey(0, types[0]), capi.make_sortkey(1, capi.FLOAT8OID, desc=True)],
                                          [([0], [], capi.FRAMEOPTION_DEFAULTS, [(capi.AGG_SUM_FLOAT8, capi.FLOAT8OID, [price])]),
                                           ([0], [1], capi.FRAMEOPTION_DEFAULTS, [(capi.WF_ROW_NUMBER, capi.INT8OID, [])])]),
        "b_running_sum_one_partition": ([capi.make_sortkey(3, types[3])],
                                        [([], [3], capi.FRAMEOPTION_DEFAULTS, [(capi.AGG_SUM_FLOAT8, capi.FLOAT8OID, [qty])])]),
    }
    for name, (keys, wins) in work.items():
        r = {}
        karr = (capi.gg_sortkey * len(keys))(*keys)
        nlive, passes = C.c_uint64(0), C.c_int(0)

        def do_sort():
            capi.check(L.gg_sort_datumrows(eng.h, karr, len(keys), len(names), C.c_void_p(rows_buf.device_ptr()), m,
                                           C.c_void_p(sorted_buf.device_ptr()), C.byref(nlive), C.byref(passes)))
        r["sort_ms"] = round(median_ms(do_sort, reps, eng), 3)
        srows = RowRelation(eng, sorted_buf.device_ptr(), nlive.value, len(names))
        # the window calls: the first over the sorted rows, the second (a) over the first's output
        objs, in_types = [], list(types)
        for part, order, frame, funcs in wins:
            objs.append((Window(eng, capi.rows_tupdesc(in_types), capi.make_window(part, order, frame, funcs), p.pool), funcs))
            in_types += [f[1] for f in funcs]
        views = []

        def do_window():
            src, cnt = srows, srows.nrows
            views.clear()
            for w, funcs in objs:
                h, k = w.run_raw(src, cnt)
                views.append((h, k))
                src, cnt = type("V", (), {"h": h, "nrows": k})(), k
        wms = median_ms(do_window, reps, eng)
        r["window_ms"] = round(wms, 3)
        wbytes, width = 0, W
        for w, funcs in objs:
            wbytes += window_bytes(srows.nrows, width, funcs)
            width += len(funcs)
        r["window_bytes"] = wbytes
        r["window_gb_per_s"] = round(wbytes / (wms / 1e3) / 1e9, 1)
        r["window_share_of_3.35TB/s"] = round(wbytes / (wms / 1e3) / PEAK_BYTES, 3)
        # end to end through the node surface, a Limit 10 on top; (a) also with WHERE rn = 1
        quals = [("", -1)] + ([("_top1", p.func(capi.F_INT8EQ, capi.BOOLOID, rn, p.const(capi.INT8OID, 1)))] if len(wins) == 2 else [])
        for suffix, qual in quals:
            b = ex.PlanBuilder()
            node = b.sort(b.seqscan(0, desc, -1, targets), keys)
            for i, (part, order, frame, funcs) in enumerate(wins):
                node = b.windowagg(node, part, order, frame, funcs, qual=qual if i == len(wins) - 1 else -1)
            x = ex.Executor(eng, p.pool, [rel], b.limit(node, 10))
            r["e2e_ms" + suffix], _ = timed_rows(x, reps)
            r["e2e_ms" + suffix] = round(r["e2e_ms" + suffix], 3)
            x.end()
        if baseline:
            import _window
            # the host path: sorted rows fetched, windowed by the row-at-a-time reference (both windows for (a))
            nbs = (srows.nrows * W * 8 + capi.GG_BLCKSZ - 1) // capi.GG_BLCKSZ
            t0 = time.perf_counter()
            host = sorted_buf.read(0, nbs).view(np.uint64)[:srows.nrows * W].reshape(-1, W)
            cur, ty = host, list(types)
            for (part, order, frame, funcs), (w, _) in zip(wins, objs):
                win = capi.make_window(part, order, frame, funcs)
                rc, cur, msg = _window.ref_window(win, ty, p.pool, cur)
                assert rc == 0, msg
                ty += [f[1] for f in funcs]
            r["baseline_host_ms"] = round((time.perf_counter() - t0) * 1e3, 3)
            h, k = views[-1]
            wid = cur.shape[1]
            nb2 = (k * wid * 8 + capi.GG_BLCKSZ - 1) // capi.GG_BLCKSZ
            dev = np.zeros(nb2 * capi.GG_BLCKSZ // 8, dtype=np.uint64)
            capi.check(L.gg_relation_read(h, 0, dev.ctypes.data, nb2))
            dev = dev[:k * wid].reshape(k, wid)
            fcols = [1 + c for c, t in enumerate(ty) if t == capi.FLOAT8OID and c >= len(names)]
            icols = [c for c in range(wid) if c not in fcols]
            ok = dev.shape == cur.shape and np.array_equal(dev[:, icols], cur[:, icols])
            if ok and fcols:
                a, b_ = dev[:, fcols].view(np.float64), cur[:, fcols].view(np.float64)
                ok = bool(np.all(np.abs(a - b_) <= 1e-12 * np.abs(b_)))
            r["parity"] = bool(ok)
        else:
            r["baseline_host_ms"], r["parity"] = "not measured", "not checked"
        for w, _ in objs:
            w.free()
        srows.free()
        out[name] = r
    sorted_buf.free()
    rows_buf.free()
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
    res = [run_size(eng, n, a.reps, baseline=(i == 0)) for i, n in enumerate(a.rows)]
    eng.close()
    print(json.dumps({"bench": "window", "card": c, "sizes": res}))


if __name__ == "__main__":
    main()
