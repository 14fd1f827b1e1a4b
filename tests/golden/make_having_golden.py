"""Generate tests/golden/having_expected.json from the reference's regression files (text only; no reference objects needed):

  test_having       the rows of expected/select_having.out's test_having table
  queries           the answers of its HAVING queries the device expresses: 1, 2, 4, 5 and 6 of the file (GROUP BY ... HAVING over
                    counts, keys and min / max, and the plain aggregate giving 0 and 1 rows); 3 applies lower(), which the device
                    does not evaluate
  q18               the two rows of TPC-H Q18 (mpph18) over the suite's heap_orders / heap_lineitem (output/rpt_tpch.source)

Usage: python tests/golden/make_having_golden.py [reference root, default /root/reference]"""
import json
import os
import re
import sys
from datetime import date

HERE = os.path.dirname(os.path.abspath(__file__))


def result_tables(lines):
    """every result table of a psql output file: {"cols": [...], "rows": [[text, ...], ...]}"""
    out, i = [], 0
    while i < len(lines):
        if re.match(r"^-+(\+-+)*$", lines[i]) and i > 0 and lines[i - 1].startswith(" "):          # a result table's header rule
            cols = [c.strip() for c in lines[i - 1].split("|")]
            body = []
            i += 1
            while not lines[i].startswith("("):
                body.append([x.strip() for x in lines[i].split("|")])
                i += 1
            assert lines[i] in ("(%d rows)" % len(body), "(%d row)" % len(body)), lines[i]
            out.append({"cols": cols, "rows": body})
        i += 1
    return out


def main(ref):
    out = open(os.path.join(ref, "src/test/regress/expected/select_having.out")).read().splitlines()
    rows = []
    for ln in out:
        if ln.startswith("INSERT INTO test_having VALUES ("):
            v = [x.strip() for x in ln[ln.index("(") + 1:ln.rindex(")")].split(",")]
            rows.append([int(v[0]), int(v[1]), v[2].strip("'"), v[3].strip("'")])
    answers = result_tables(out)
    picked = [answers[k] for k in (0, 1, 3, 4, 5)]
    for a in picked:
        a["rows"] = [[int(x) if x.lstrip("-").isdigit() else x for x in r] for r in a["rows"]]
    src = open(os.path.join(ref, "src/test/regress/output/rpt_tpch.source")).read().splitlines()
    k = next(n for n, ln in enumerate(src) if ln.startswith("select  'mpph18'"))
    while not src[k].startswith("----------+"):
        k += 1
    q18 = []
    k += 1
    while not src[k].startswith("("):
        f = [x.strip() for x in src[k].split("|")]
        m, d, y = (int(x) for x in f[4].split("-"))
        q18.append([int(f[2]), int(f[3]), date(y, m, d).isoformat(), f[5], f[6]])
        k += 1
    json.dump({"source": "src/test/regress/expected/select_having.out (test_having, queries 1 2 4 5 6), "
                         "src/test/regress/output/rpt_tpch.source (mpph18)",
               "test_having": rows, "queries": picked, "q18": q18},
              open(os.path.join(HERE, "having_expected.json"), "w"), indent=1)
    print("having_expected.json", [len(a["rows"]) for a in picked], q18)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "/root/reference")
