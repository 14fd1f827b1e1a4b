"""Bounded Sort (ORDER BY ... LIMIT) on the device against the full sort; prints one JSON line.

  sort:  gg_sort_datumrows against gg_sort_datumrows_bounded over 10^8 datum rows (an int8 key, then a float8 key DESC) at
         bounds 10, 10^3, 10^6, n/4 (the last bound that selects) and n/2 (sorts everything: DESIGN §4.4): kernel ms from CUDA
         events on the engine's stream, passes, and whether the bounded rows are byte for byte the full sort's first rows
  e2e:   "scan LI-narrow, project (l_orderkey, l_extendedprice), ORDER BY l_extendedprice DESC LIMIT 100" through the
         executor-node surface, with the Limit node (bounded Sort, 100 rows copied) and without it (the caller stops after 100
         rows of the full sort), host wall clock around calls that end in a device synchronise
Usage: python scripts/bench_topn.py [--rows N] [--li-rows N] [--reps R]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def sort_section(eng, n, reps):
    import torch
    from greengage_b200 import capi
    L = capi.dev_lib()
    g = torch.Generator(device="cuda").manual_seed(7)
    words = torch.empty((n, 3), dtype=torch.int64, device="cuda")
    words[:, 0] = 0
    words[:, 1] = torch.randint(-2 ** 62, 2 ** 62, (n,), generator=g, device="cuda", dtype=torch.int64)
    words[:, 2] = torch.randn(n, generator=g, device="cuda", dtype=torch.float64).view(torch.int64)
    full_out = torch.empty((n + 1, 3), dtype=torch.int64, device="cuda")
    part_out = torch.empty((n + 1, 3), dtype=torch.int64, device="cuda")
    res = []
    for name, keys in (("int8", [capi.make_sortkey(0, capi.INT8OID)]), ("float8 desc", [capi.make_sortkey(1, capi.FLOAT8OID, True)])):
        ka = (capi.gg_sortkey * len(keys))(*keys)

        def timed(call):
            ms = C.c_float(0)
            call()                                                   # warm-up: scratch allocation, module load
            torch.cuda.synchronize()
            best = None
            for _ in range(reps):
                capi.check(L.gg_engine_timer_start(eng.h))
                call()
                capi.check(L.gg_engine_timer_stop(eng.h, C.byref(ms)))
                best = ms.value if best is None else min(best, ms.value)
            return best

        cnt, passes = C.c_uint64(0), C.c_int(0)
        full = lambda: capi.check(L.gg_sort_datumrows(eng.h, ka, len(keys), 2, C.c_void_p(words.data_ptr()), n,
                                                      C.c_void_p(full_out.data_ptr()), C.byref(cnt), C.byref(passes)))
        full_ms = timed(full)
        full_passes = passes.value
        for bound in (10, 1000, 10 ** 6, n // 4, n // 2):
            bcnt, bpasses = C.c_uint64(0), C.c_int(0)
            part = lambda: capi.check(L.gg_sort_datumrows_bounded(eng.h, ka, len(keys), 2, C.c_void_p(words.data_ptr()), n, bound,
                                                                  C.c_void_p(part_out.data_ptr()), C.byref(bcnt), C.byref(bpasses)))
            ms = timed(part)
            parity = bcnt.value == bound and bool(torch.equal(part_out[:bound], full_out[:bound]))
            res.append({"key": name, "bound": bound, "full_ms": round(full_ms, 3), "full_passes": full_passes,
                        "bounded_ms": round(ms, 3), "bounded_passes": bpasses.value, "speedup": round(full_ms / ms, 2),
                        "parity": parity})
    del words, full_out, part_out
    torch.cuda.empty_cache()
    return res


def e2e_section(eng, nrows, reps):
    from greengage_b200 import capi, executor as ex, tpch
    from greengage_b200.engine import Relation
    pages, nb, nr = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, nrows))
    rel = Relation(eng, host_pages=pages)
    c = tpch.LI_NARROW_COLS
    p = capi.ExprPool()
    targets = [p.var(c["orderkey"], capi.INT8OID), p.var(c["extendedprice"], capi.FLOAT8OID)]
    keys = [capi.make_sortkey(1, capi.FLOAT8OID, True)]
    desc = capi.synth_tupdesc(capi.TAB_LINEITEM_NARROW)
    out = {}
    rows = {}
    for variant in ("limit", "no_limit"):
        b = ex.PlanBuilder()
        sort = b.sort(b.seqscan(0, desc, -1, targets), keys)
        x = ex.Executor(eng, p.pool, [rel], b.limit(sort, 100) if variant == "limit" else sort)
        times = []
        for i in range(reps + 1):
            if i:
                x.rescan()
            t = time.perf_counter()
            got = x.rows() if variant == "limit" else x.rows(limit=100)
            times.append((time.perf_counter() - t) * 1e3)
        rows[variant] = [r[0][:2] for r in got]
        x.end()
        out[variant + "_ms"] = round(min(times[1:]), 3)
    rel.free()
    out["rows"] = nr
    # the scan hands its rows out in claim order, which varies between runs: ties of the price may come in another order, so
    # parity is the price column in order and the row count
    out["parity"] = [r[1] for r in rows["limit"]] == [r[1] for r in rows["no_limit"]] and len(rows["limit"]) == 100
    out["speedup"] = round(out["no_limit_ms"] / out["limit_ms"], 2)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10 ** 8)
    ap.add_argument("--li-rows", type=int, default=20_000_000)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    from greengage_b200.engine import Engine
    eng = Engine(0)
    sort = sort_section(eng, a.rows, a.reps)
    e2e = e2e_section(eng, a.li_rows, a.reps)
    eng.close()
    print(json.dumps({"bench": "topn", "card": card(), "rows": a.rows, "sort": sort,
                      "parity": all(r["parity"] for r in sort) and e2e["parity"],
                      "bytes_per_row_per_pass": {"radix_pass": 32, "select_histogram": 9},
                      "e2e_order_by_price_desc_limit_100": e2e}))


if __name__ == "__main__":
    main()
