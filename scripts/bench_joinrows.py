"""A HashJoin that writes its rows (gg_joinrows_create) against the same join fused with count(*) (gg_joinagg_create), on
LI-narrow ⋈ orders (synthetic: every lineitem row finds its order); prints one JSON line.

  rows:      build and probe kernel ms (CUDA events of the pipeline, gg_joinagg_stats) of the join writing
             (l_orderkey, l_extendedprice, o_orderdate) for every joined row, median of --reps runs after a warm-up run; rows
             joined per second of probe time; the algorithmic bytes (outer pages + (1 + ncols) * 8 bytes written per joined row)
             and the bound they give at the HBM bandwidth plus one random table access per outer row at the rate
             build/gather_peak measures on this GPU
  count:     the same join fused with count(*), the non-materialising baseline, measured the same way
The card's name and power limit come from the same run.
Usage: python scripts/bench_joinrows.py [--li-rows N] [--orders N] [--reps R]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DATASHEET_HBM_GBS = 3350.0          # H100 SXM data sheet, 700 W


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def hbm_peak():
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    try:
        return float(json.load(open(path))["hbm_gbs"]), "measured copy kernel (MEASURED_PEAKS.json)"
    except (OSError, KeyError, ValueError):
        return DATASHEET_HBM_GBS, "data sheet (not reached by any kernel here)"


def gather_rate():
    """random 32-byte-entry gathers per second this GPU sustains (build/gather_peak), or None"""
    exe = os.path.join(ROOT, "build", "gather_peak")
    if not os.path.exists(exe):
        return None
    try:
        out = subprocess.run([exe, "2048", "2e8"], capture_output=True, timeout=120, text=True)
        d = json.loads(out.stdout.strip().splitlines()[-1])
        return max(d["gather_g_per_s"].values()) * 1e9
    except (OSError, subprocess.SubprocessError, ValueError, KeyError):
        return None


def measure(make, orel, irel, reps):
    """(build ms, probe ms) medians over reps runs after one warm-up run, and the pipeline after the last run"""
    j = make()
    b, p = [], []
    for i in range(reps + 1):
        if i:
            j.reset()
        j.run(irel, orel)
        if hasattr(j, "rows_raw"):
            j.rows_raw()
        else:
            j.fetch()
        st = j.stats()
        if i:
            b.append(st["build_ms"])
            p.append(st["probe_ms"])
    return statistics.median(b), statistics.median(p), j


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--li-rows", type=int, default=10 ** 8)
    ap.add_argument("--orders", type=int, default=25_000_000)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    from greengage_b200 import capi, tpch
    from greengage_b200.engine import Engine, JoinAgg, JoinRows, Relation
    eng = Engine(0)
    li, li_nb, li_n = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, a.li_rows, seed=11, norders=a.orders))
    od, od_nb, od_n = tpch.synth_generate(tpch.synth_spec(capi.TAB_ORDERS, a.orders, seed=11))
    orel, irel = Relation(eng, host_pages=li), Relation(eng, host_pages=od)

    outer, inner, hj, agg, pool = tpch.join_plan(capi.TAB_LINEITEM_NARROW, "count")
    lc, oc = tpch.LI_NARROW_COLS, tpch.ORDERS_COLS
    p = capi.ExprPool()
    hj_rows = capi.make_hashjoin(capi.JOIN_INNER, [p.var(lc["orderkey"], capi.INT8OID, 0)], [p.var(oc["orderkey"], capi.INT8OID, 1)])
    targets = [p.var(lc["orderkey"], capi.INT8OID, 0), p.var(lc["extendedprice"], capi.FLOAT8OID, 0), p.var(oc["orderdate"], capi.DATEOID, 1)]

    rb_ms, rp_ms, jr = measure(lambda: JoinRows(eng, outer, inner, hj_rows, targets, p.pool), orel, irel, a.reps)
    _, nslots, live = jr.rows_raw()
    jr.free()
    cb_ms, cp_ms, ja = measure(lambda: JoinAgg(eng, outer, inner, hj, agg, pool), orel, irel, a.reps)
    crow, cjoined = ja.fetch()
    ja.free()
    orel.free()
    irel.free()
    eng.close()

    peak, peak_src = hbm_peak()
    rate = gather_rate()
    W = 1 + len(targets)
    bytes_rows = li_nb * capi.GG_BLCKSZ + live * W * 8
    bytes_count = li_nb * capi.GG_BLCKSZ

    def bound_ms(nbytes):
        ms = nbytes / (peak * 1e9) * 1e3
        return ms + (li_n / rate * 1e3 if rate else 0.0)

    print(json.dumps({
        "bench": "joinrows", "card": card(), "outer_rows": li_n, "inner_rows": od_n, "outer_pages": li_nb, "inner_pages": od_nb,
        "parity": live == cjoined == li_n and crow[0].agg[0].i == live,
        "rows": {"ncols": len(targets), "build_ms": round(rb_ms, 3), "probe_ms": round(rp_ms, 3), "rows_joined": live,
                 "row_slots": nslots, "rows_per_s": round(live / (rp_ms / 1e3), 1), "algorithmic_bytes": bytes_rows,
                 "probe_bound_ms": round(bound_ms(bytes_rows), 3), "probe_frac_of_bound": round(bound_ms(bytes_rows) / rp_ms, 3)},
        "count": {"build_ms": round(cb_ms, 3), "probe_ms": round(cp_ms, 3), "rows_joined": cjoined, "algorithmic_bytes": bytes_count,
                  "probe_bound_ms": round(bound_ms(bytes_count), 3), "probe_frac_of_bound": round(bound_ms(bytes_count) / cp_ms, 3)},
        "hbm_gbs": peak, "hbm_source": peak_src,
        "gather_per_s": rate, "gather_source": "build/gather_peak (scripts/gather_peak.cu), this run" if rate else "not available"}))


if __name__ == "__main__":
    main()
