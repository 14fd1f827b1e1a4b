"""Build tests/golden/window_expected.json from the reference's regression output src/test/regress/expected/window.out: the printed
rows of the window-function queries over tenk1 (and one small VALUES relation) that the device path runs — integer, rank,
distribution and value functions over int4 columns, count and sum(int4) — keyed by an id the GPU test maps to a plan.  The outputs
have no ORDER BY, so the test compares them as multisets; every query chosen here prints the same multiset however ties are
ordered.  Left out: empsalary (depname is longer than 8 bytes), anything that returns numeric (avg, sum over int8 / numeric /
money / interval), and expression arguments (ten * 2, four + 1).

With --tenk, it also writes tests/golden/tenk1.npz: the 13 int4 columns of src/test/regress/data/tenk.data (unique1 .. even), the
fixture the queries run over.

Usage: python tests/golden/make_window_golden.py <reference root> [--tenk]"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))

QUERIES = {
    "count_over_empty": "SELECT COUNT(*) OVER () FROM tenk1 WHERE unique2 < 10;",
    "sum_cumulative": "SELECT sum(four) OVER (PARTITION BY ten ORDER BY unique2) AS sum_1, ten, four FROM tenk1 WHERE unique2 < 10;",
    "row_number": "SELECT row_number() OVER (ORDER BY unique2) FROM tenk1 WHERE unique2 < 10;",
    "rank": "SELECT rank() OVER (PARTITION BY four ORDER BY ten) AS rank_1, ten, four FROM tenk1 WHERE unique2 < 10;",
    "dense_rank": "SELECT dense_rank() OVER (PARTITION BY four ORDER BY ten), ten, four FROM tenk1 WHERE unique2 < 10;",
    "percent_rank": "SELECT percent_rank() OVER (PARTITION BY four ORDER BY ten), ten, four FROM tenk1 WHERE unique2 < 10;",
    "cume_dist": "SELECT cume_dist() OVER (PARTITION BY four ORDER BY ten), ten, four FROM tenk1 WHERE unique2 < 10;",
    "ntile3": "SELECT ntile(3) OVER (ORDER BY ten, four), ten, four FROM tenk1 WHERE unique2 < 10;",
    "lag": "SELECT lag(ten) OVER (PARTITION BY four ORDER BY ten), ten, four FROM tenk1 WHERE unique2 < 10;",
    "lag_offset": "SELECT lag(ten, four) OVER (PARTITION BY four ORDER BY ten), ten, four FROM tenk1 WHERE unique2 < 10;",
    "lag_default": "SELECT lag(ten, four, 0) OVER (PARTITION BY four ORDER BY ten), ten, four FROM tenk1 WHERE unique2 < 10;",
    "lead": "SELECT lead(ten) OVER (PARTITION BY four ORDER BY ten), ten, four FROM tenk1 WHERE unique2 < 10;",
    "first_value": "SELECT first_value(ten) OVER (PARTITION BY four ORDER BY ten), ten, four FROM tenk1 WHERE unique2 < 10;",
    "last_value_order": "SELECT last_value(ten) OVER (ORDER BY ten), ten, four FROM tenk1 WHERE unique2 < 10;",
    "last_value_partition": "SELECT last_value(ten) OVER (PARTITION BY four ORDER BY ten), ten, four FROM",
    "count_partition_subquery": "SELECT count(*) OVER (PARTITION BY four), four FROM (SELECT * FROM tenk1 WHERE two = 1)s WHERE unique2 < 10;",
    "values_sum_int": "SELECT i,SUM(v::int) OVER (ORDER BY i ROWS BETWEEN CURRENT ROW AND UNBOUNDED FOLLOWING)",
    "values_count_v": "SELECT i,COUNT(v) OVER (ORDER BY i ROWS BETWEEN CURRENT ROW AND UNBOUNDED FOLLOWING)",
    "values_count_star": "SELECT i,COUNT(*) OVER (ORDER BY i ROWS BETWEEN CURRENT ROW AND UNBOUNDED FOLLOWING)",
}


def parse(lines, first):
    """the printed rows of the first statement that starts with `first`: [[cell, ...], ...] (cells stripped, NULL = "")"""
    i = next(k for k, ln in enumerate(lines) if ln.startswith(first))
    while not set(lines[i + 1].strip()) <= set("-+") or not lines[i + 1].strip():
        i += 1
    rows = []
    for ln in lines[i + 2:]:
        if ln.startswith("(") and ln.rstrip().endswith(("rows)", "row)")):
            break
        rows.append([c.strip() for c in ln.split("|")])
    return rows


def main():
    ref = sys.argv[1]
    reg = os.path.join(ref, "src", "test", "regress")
    lines = open(os.path.join(reg, "expected", "window.out")).read().splitlines()
    out = {k: parse(lines, q) for k, q in QUERIES.items()}
    with open(os.path.join(HERE, "window_expected.json"), "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
        f.write("\n")
    if "--tenk" in sys.argv:
        import numpy as np
        rows = [ln.split("\t")[:13] for ln in open(os.path.join(reg, "data", "tenk.data")).read().splitlines() if ln.strip()]
        cols = ["unique1", "unique2", "two", "four", "ten", "twenty", "hundred", "thousand", "twothousand", "fivethous", "tenthous",
                "odd", "even"]
        a = np.array(rows, dtype=np.int32)
        np.savez_compressed(os.path.join(HERE, "tenk1.npz"), **{c: a[:, i] for i, c in enumerate(cols)})


if __name__ == "__main__":
    main()
