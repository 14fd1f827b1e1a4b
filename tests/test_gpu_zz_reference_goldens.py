"""The GPU path against the REFERENCE'S OWN golden answers (its regression suite's expected outputs over its own data):
TPC-H Q4 (semi join), Q12 (inner join) and Q6 (range predicates + plain aggregate) of output/rpt_tpch.source; the inner /
left / right / full join tables of expected/join.out; the ORDER BY answers of expected/sort.out; the integer and hashed
aggregates of expected/aggregates.out.  Same plans and fixtures as the tests/test_oracle_*golden* tests, which hold the oracle
to those answers on every CPU run.  (Q1's golden is tests/test_gpu_scanagg.py / test_gpu_executor.py.)"""
import numpy as np
import pytest

from _util import golden, tpch_join_fixture, tpch_q4_plan, tpch_q12_plan
from greengage_b200 import capi
from test_gpu_join import gpu_joinagg

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from greengage_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def test_q4_semi_join_counts_are_the_references(eng):
    li_desc, li_pages, ord_desc, ord_pages, shipmode_code, priority_code = tpch_join_fixture()
    exp = golden("tpch_join_expected.json")["q4"]
    outer, inner, hj, agg, pool = tpch_q4_plan(li_desc, ord_desc, exp)
    rows, nj, _ = gpu_joinagg(eng, outer, inner, hj, agg, pool, ord_pages, li_pages)
    got = {capi.unpack_str(r.key[0], r.keylen[0]): r.agg[0].i for r in rows}
    assert got == {priority_code[e["orderpriority"]]: e["order_count"] for e in exp["rows"]}
    assert nj == sum(e["order_count"] for e in exp["rows"])


def test_q12_inner_join_counts_are_the_references(eng):
    li_desc, li_pages, ord_desc, ord_pages, shipmode_code, priority_code = tpch_join_fixture()
    exp = golden("tpch_join_expected.json")["q12"]
    for high, col in ((True, "high_line_count"), (False, "low_line_count")):
        outer, inner, hj, agg, pool = tpch_q12_plan(li_desc, ord_desc, exp, shipmode_code, priority_code, high)
        rows, nj, _ = gpu_joinagg(eng, outer, inner, hj, agg, pool, li_pages, ord_pages)
        got = {capi.unpack_str(r.key[0], r.keylen[0]): r.agg[0].i for r in rows}
        assert got == {shipmode_code[e["shipmode"]]: e[col] for e in exp["rows"]}, (col, got)


def test_q6_revenue_is_the_references(eng):
    """Q6 ('mpph6'): scan -> five range predicates -> plain aggregate, against the reference's golden revenue and the oracle."""
    from _util import Q6_GOLDEN_REVENUE, lineitem_fixture_pages, tpch_q6_plan
    from oracle import pyoracle as po
    from test_gpu_scanagg import gpu_scanagg
    desc, pages, n = lineitem_fixture_pages()
    scan, agg, pool = tpch_q6_plan(desc)
    want, sc, ps = po.seqscan_agg(scan, agg, pool, pages)
    got, gsc, gps, _ = gpu_scanagg(eng, scan, agg, pool, pages)
    assert (gsc, gps) == (sc, ps) and len(got) == 1 and got[0].agg[1].i == want[0].agg[1].i
    assert abs(got[0].agg[0].f[0] - Q6_GOLDEN_REVENUE) <= 1e-6 * Q6_GOLDEN_REVENUE, got[0].agg[0].f[0]


@pytest.mark.parametrize("name", ["inner", "inner_i_eq_k", "left", "right", "full"])
def test_j1j2_joins_reduce_the_references_golden_tables(eng, name):
    """J1_TBL / J2_TBL of the reference's sql/join.sql and the golden inner / left / right / full tables of expected/join.out
    (NULL keys on both sides, duplicate inner keys), consumed by GROUP BY J1.i aggregates; tests/test_oracle_join_golden.py
    holds the oracle to the same tables row by row."""
    from _util import j1j2_agg, j1j2_check_groups, j1j2_fixture, j1j2_golden_groups, j1j2_join
    d1, p1, d2, p2, g = j1j2_fixture()
    p, outer, inner, hj = j1j2_join(d1, d2, name)
    rows, nj, _ = gpu_joinagg(eng, outer, inner, hj, j1j2_agg(p), p.pool, p1, p2)
    assert nj == len(g["queries"][name]["rows"])
    j1j2_check_groups(rows, j1j2_golden_groups(g, name))


def test_order_by_answers_are_the_references(eng):
    """Golden ORDER BY outputs of the reference's expected/sort.out through the device sort (gg_sort_rows)."""
    import numpy as np
    from _util import sort_golden_cases
    from greengage_b200.engine import sort_rows
    for name, keys, rows, nulls, want, wantnulls in sort_golden_cases():
        perm = sort_rows(eng, keys, rows, nulls).astype(np.int64)
        assert np.array_equal(rows[perm], want) and np.array_equal(nulls[perm], wantnulls), name


def test_onek_aggregates_are_the_references(eng):
    """expected/aggregates.out over onek: sum/max/count of an int4 column, and `ten, count(*), sum(four) GROUP BY ten`."""
    from _util import onek_check, onek_fixture, onek_plans
    from test_gpu_scanagg import gpu_scanagg
    desc, pages, exp = onek_fixture()
    plain, grouped = onek_plans(desc, exp)
    onek_check(exp, gpu_scanagg(eng, *plain, pages)[0], gpu_scanagg(eng, *grouped, pages)[0])


def test_gp_hashagg_text_key_answer_is_the_references(eng):
    """sql/gp_hashagg.sql MPP-2614: hashed aggregate with a text key behind a three-clause qual (expected/gp_hashagg.out:17-22)"""
    from _util import gp_hashagg_case
    from test_gpu_scanagg import gpu_scanagg
    desc, pages, scan, agg, pool, want = gp_hashagg_case()
    rows, sc, ps, _ = gpu_scanagg(eng, scan, agg, pool, pages)
    assert (sc, ps) == (6, 6)
    assert {capi.unpack_str(r.key[0], r.keylen[0]): r.agg[0].i for r in rows} == want


def test_and_or_skip_the_arm_that_would_raise(eng):
    """ExecEvalAnd / ExecEvalOr stop at the deciding arm (execQual.c:3385,3455): a division by zero in the arm they skip is
    not an error; every kernel variant (specialised, interpreter private / transposed)"""
    from test_gpu_scanagg import gpu_scanagg
    from test_oracle_float import short_circuit_case
    desc, pages, plans = short_circuit_case()
    for scan, agg, pool, want in plans:
        for variant in (None, "interp-priv", "interp-tr"):
            rows, sc, ps, _ = gpu_scanagg(eng, scan, agg, pool, pages, variant)
            assert (sc, ps, rows[0].agg[0].i) == (5, want, want)


# ---- AOCS column files -> datum rows on the device (csrc/gg_aocs.cu); the same device function runs through gcc against the
# reference-written files in tests/test_aocs_decode.py


def test_aocs_columns_decode_to_the_rows_the_oracle_reads(eng):
    import numpy as np
    from greengage_b200 import aocs, tpch
    from oracle import pyoracle as po
    spec = tpch.synth_spec(capi.TAB_LINEITEM_WIDE, 300_000, nsegs=2, seg=1)
    nb, nr = tpch.synth_measure(spec)
    desc = capi.synth_tupdesc(capi.TAB_LINEITEM_WIDE)
    cols = [0, 3, 4, 8, 10]                                   # int8, int4, float8, char(1), date
    files, nrows = aocs.synth_columns(spec, cols, nr)
    dc = aocs.DeviceColumns(eng, desc, cols, files)
    try:
        rel = dc.decode()
        rows = dc.read_rows()
        rel.free()
    finally:
        dc.free()
    assert rows.shape == (nr, 1 + len(cols)) and not rows[:, 0].any()
    for i, c in enumerate(cols):
        a = desc.attrs[c]
        v, nl, _, _ = po.aocs_read_column(a, files[c], nr)
        if a.attlen == -1:
            want = np.array([int(files[c][o + 1]) for o in v], dtype=np.int64)
        elif a.attlen == 4:
            want = v.astype(np.uint32).view(np.int32).astype(np.int64)
        else:
            want = v
        assert np.array_equal(rows[:, 1 + i], want), c


def test_aocs_q1_equals_the_heap_answer_and_the_references_golden(eng):
    from _util import assert_aggrows_match, golden, lineitem_fixture_pages
    from greengage_b200 import aocs, tpch
    from greengage_b200.engine import ScanAgg
    from oracle import pyoracle as po
    from test_oracle_aocs import lineitem_as_column_files
    from test_oracle_q1_golden import _check_against_golden
    names = dict(quantity=1, extendedprice=2, discount=3, tax=4, returnflag=5, linestatus=6, shipdate=7)
    cols = [4, 5, 6, 7, 8, 9, 10]

    def run(desc, files, interval_days):
        dc = aocs.DeviceColumns(eng, desc, cols, files)
        try:
            rel = dc.decode()
            scan, agg, pool = tpch.q1_plan(stage=capi.AGGSTAGE_NORMAL, interval_days=interval_days, desc=dc.rows_tupdesc([1] * len(cols)), cols=names)
            sa = ScanAgg(eng, scan, agg, pool)
            try:
                sa.run(rel)
                return sa.fetch()
            finally:
                sa.free()
                rel.free()
        finally:
            dc.free()

    # synthetic LI-wide segment: the oracle's answer over the heap pages of the same rows
    spec = tpch.synth_spec(capi.TAB_LINEITEM_WIDE, 400_000)
    pages, nb, nr = tpch.synth_generate(spec)
    files, _ = aocs.synth_columns(spec, cols, nr)
    got, sc, ps = run(capi.synth_tupdesc(capi.TAB_LINEITEM_WIDE), files, 90)
    scan_h, agg_h, pool_h = tpch.q1_plan(capi.TAB_LINEITEM_WIDE)
    want, wsc, wps, want_x = po.seqscan_agg(scan_h, agg_h, pool_h, pages, exact=True)
    assert (sc, ps) == (wsc, wps)
    assert_aggrows_match(got, want, agg_h, exact=want_x)
    # the reference's regression lineitem stored as column files: its golden Q1 answer (co_lineitem, rpt_tpch.source:5768-5795)
    desc, colvals, n = lineitem_as_column_files()
    files = {c: aocs.write_column(desc.attrs[c], colvals[c]) for c in cols}
    got, sc, ps = run(desc, files, golden("q1_expected.json")["interval_days"])
    assert sc == n
    _check_against_golden(got)


@pytest.mark.parametrize("variant", ["specialised", "interpreter"])
def test_fused_aocs_scan_equals_the_heap_answer_and_the_references_golden(eng, monkeypatch, variant):
    """SeqScan over column files fused with the Agg (gg_scanagg_run_aocs; aocs_getnext, aocsam.c:661): no rows are written
    back, a lane loads its row's referenced columns from the files.  Same answers as the heap pages of the same rows
    (oracle), as the two-pass decode, and as the reference's golden Q1 over co_lineitem (rpt_tpch.source:5768-5795)."""
    from _util import assert_aggrows_match, golden, lineitem_fixture_pages
    from greengage_b200 import aocs, tpch
    from greengage_b200.engine import ScanAgg
    from oracle import pyoracle as po
    from test_oracle_aocs import lineitem_as_column_files
    from test_oracle_q1_golden import _check_against_golden
    if variant == "interpreter":
        monkeypatch.setenv("GGB200_JIT", "0")
    names = dict(quantity=1, extendedprice=2, discount=3, tax=4, returnflag=5, linestatus=6, shipdate=7)
    cols = [4, 5, 6, 7, 8, 9, 10]

    def run(desc, files, interval_days, stage=capi.AGGSTAGE_NORMAL, twice=False):
        dc = aocs.DeviceColumns(eng, desc, cols, files)
        try:
            scan, agg, pool = tpch.q1_plan(stage=stage, interval_days=interval_days, desc=dc.rows_tupdesc([1] * len(cols)), cols=names)
            sa = ScanAgg(eng, scan, agg, pool)
            try:
                sa.run_aocs(dc)
                if twice:
                    sa.run_aocs(dc)                     # feeds accumulate like gg_scanagg_run
                return sa.fetch(), sa.variant()
            finally:
                sa.free()
        finally:
            dc.free()

    spec = tpch.synth_spec(capi.TAB_LINEITEM_WIDE, 400_000)
    pages, nb, nr = tpch.synth_generate(spec)
    files, _ = aocs.synth_columns(spec, cols, nr)
    (got, sc, ps), var = run(capi.synth_tupdesc(capi.TAB_LINEITEM_WIDE), files, 90)
    assert (var >= 16) == (variant == "specialised")
    scan_h, agg_h, pool_h = tpch.q1_plan(capi.TAB_LINEITEM_WIDE)
    want, wsc, wps, want_x = po.seqscan_agg(scan_h, agg_h, pool_h, pages, exact=True)
    assert (sc, ps) == (wsc, wps)
    assert_aggrows_match(got, want, agg_h, exact=want_x)
    (got2, sc2, ps2), _ = run(capi.synth_tupdesc(capi.TAB_LINEITEM_WIDE), files, 90, twice=True)
    assert (sc2, ps2) == (2 * wsc, 2 * wps) and sorted(r.agg[7].i for r in got2) == sorted(2 * r.agg[7].i for r in want)
    desc, colvals, n = lineitem_as_column_files()
    files = {c: aocs.write_column(desc.attrs[c], colvals[c]) for c in cols}
    (got, sc, ps), _ = run(desc, files, golden("q1_expected.json")["interval_days"])
    assert sc == n
    _check_against_golden(got)


def test_fused_aocs_scan_with_nulls_and_a_ragged_tail(eng):
    """NULL-bearing blocks (bitmap + prefix popcount), a row count that is no multiple of the tile, min / max / count(col):
    the nullable kernel variant over column files equals the oracle's AOCS scan."""
    from _util import assert_aggrows_match, make_desc
    from greengage_b200 import aocs
    from greengage_b200.capi import ExprPool
    from greengage_b200.engine import ScanAgg
    from oracle import pyoracle as po
    rng = np.random.default_rng(17)
    n = 70_001
    desc = make_desc([(capi.INT4OID, 4, "i", 1), (capi.FLOAT8OID, 8, "d", 1), (capi.BPCHAROID, -1, "i", 0), (capi.INT8OID, 8, "d", 1)])
    k = rng.integers(0, 7, n)
    x = rng.integers(-1000, 1000, n).astype(np.float64) / 4
    f = [bytes([65 + int(c)]) for c in rng.integers(0, 3, n)]
    y = rng.integers(-10**12, 10**12, n)
    nulls = [rng.random(n) < 0.2, rng.random(n) < 0.3, rng.random(n) < 0.1, np.zeros(n, bool)]
    vals = [[int(v) for v in k], [float(v) for v in x], f, [int(v) for v in y]]
    files = {c: aocs.write_column(desc.attrs[c], vals[c], nulls[c] if c < 3 else None) for c in range(4)}
    dc = aocs.DeviceColumns(eng, desc, [0, 1, 2, 3], files)
    try:
        p = ExprPool()
        kk, xx, ff, yy = p.var(1, capi.INT4OID), p.var(2, capi.FLOAT8OID), p.var(3, capi.BPCHAROID), p.var(4, capi.INT8OID)
        qual = p.func(capi.F_INT4GT, capi.BOOLOID, kk, p.const(capi.INT4OID, 0))
        agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [ff], [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_FLOAT8, xx), (capi.AGG_COUNT_ANY, xx),
                                                          (capi.AGG_MAX_INT8, yy), (capi.AGG_MIN_INT4, kk)])
        scan = capi.make_scan(dc.rows_tupdesc([0, 0, 0, 1]), qual)
        sa = ScanAgg(eng, scan, agg, p.pool)
        sa.run_aocs(dc)
        got, sc, ps = sa.fetch()
        sa.free()
        oscan = capi.make_scan(desc, qual)
        want, wsc, wps, want_x = po.aocs_seqscan_agg(oscan, agg, p.pool, [files[c] for c in range(4)], n, exact=True)
        assert (sc, ps) == (wsc, wps) and sc == n
        assert_aggrows_match(got, want, agg, exact=want_x)
    finally:
        dc.free()


@pytest.mark.parametrize("blocksize,file_shift", [(8192, 0), (32768, 0), (32768, 8)])
def test_fused_aocs_scan_staged_and_row_by_row_columns_mix(eng, blocksize, file_shift):
    """The fused scan stages a unit's values of a column in shared memory when the storage blocks it touches are plain
    (no NULL bitmap, one stride) and reads the column row by row otherwise: NULLs only in the middle third of the rows make
    both happen inside one column file, small storage blocks make a unit run over several of them, and files that do not
    start on a 16-byte boundary take the row-by-row path altogether.  Every combination equals the oracle's AOCS scan."""
    from _util import assert_aggrows_match, make_desc
    from greengage_b200 import aocs
    from greengage_b200.capi import ExprPool
    from greengage_b200.engine import ScanAgg
    from oracle import pyoracle as po
    rng = np.random.default_rng(23)
    n = 100_003
    desc = make_desc([(capi.INT4OID, 4, "i", 1), (capi.FLOAT8OID, 8, "d", 1), (capi.BPCHAROID, -1, "i", 0), (capi.INT8OID, 8, "d", 1),
                      (capi.BOOLOID, 1, "c", 1)])
    k = rng.integers(0, 9, n)
    x = rng.integers(-1000, 1000, n).astype(np.float64) / 8
    f = [bytes([65 + int(c)]) * 2 for c in rng.integers(0, 3, n)]
    y = rng.integers(-10**12, 10**12, n)
    t = rng.integers(0, 2, n)
    mid = (np.arange(n) > n // 3) & (np.arange(n) < 2 * n // 3)
    nulls = [mid & (rng.random(n) < 0.2), mid & (rng.random(n) < 0.3), np.zeros(n, bool), None, None]
    vals = [[int(v) for v in k], [float(v) for v in x], f, [int(v) for v in y], [int(v) for v in t]]
    files = {c: aocs.write_column(desc.attrs[c], vals[c], nulls[c], blocksize=blocksize) for c in range(5)}
    dc = aocs.DeviceColumns(eng, desc, [0, 1, 2, 3, 4], files, file_shift=file_shift)
    try:
        p = ExprPool()
        kk, xx, ff, yy, tt = (p.var(1, capi.INT4OID), p.var(2, capi.FLOAT8OID), p.var(3, capi.BPCHAROID), p.var(4, capi.INT8OID),
                              p.var(5, capi.BOOLOID))
        qual = p.func(capi.F_INT4GT, capi.BOOLOID, kk, p.const(capi.INT4OID, 1))
        agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [ff, tt], [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_FLOAT8, xx), (capi.AGG_COUNT_ANY, xx),
                                                              (capi.AGG_MAX_INT8, yy), (capi.AGG_MIN_INT4, kk)])
        scan = capi.make_scan(dc.rows_tupdesc([0, 0, 0, 1, 1]), qual)
        sa = ScanAgg(eng, scan, agg, p.pool)
        sa.run_aocs(dc)
        got, sc, ps = sa.fetch()
        sa.free()
        oscan = capi.make_scan(desc, qual)
        want, wsc, wps, want_x = po.aocs_seqscan_agg(oscan, agg, p.pool, [files[c] for c in range(5)], n, exact=True)
        assert (sc, ps) == (wsc, wps) and sc == n
        assert_aggrows_match(got, want, agg, exact=want_x)
    finally:
        dc.free()


def test_flattened_qual_gives_the_references_q6_revenue(eng):
    from _util import Q6_GOLDEN_REVENUE, lineitem_fixture_pages, tpch_q6_plan
    from oracle import pyoracle as po
    from test_gpu_scanagg import gpu_scanagg
    desc, pages, n = lineitem_fixture_pages()
    scan, agg, pool = tpch_q6_plan(desc)
    want, sc, ps = po.seqscan_agg(scan, agg, pool, pages)
    for variant in (None, "interp-priv", "interp-tr"):
        got, gsc, gps, _ = gpu_scanagg(eng, scan, agg, pool, pages, variant)
        assert (gsc, gps) == (sc, ps) and got[0].agg[1].i == want[0].agg[1].i
        assert abs(got[0].agg[0].f[0] - Q6_GOLDEN_REVENUE) <= 1e-6 * Q6_GOLDEN_REVENUE
    # and the rows where the skipped arm would have raised now pass like in the reference
    from test_oracle_float import short_circuit_case
    d2, p2, plans = short_circuit_case()
    scan2, agg2, pool2, want2 = plans[0]                      # b <> 0 AND a / b > 1
    rows, sc2, ps2, _ = gpu_scanagg(eng, scan2, agg2, pool2, p2)
    assert (sc2, ps2, rows[0].agg[0].i) == (5, want2, want2)


def test_partial_stage_without_sumsq_gives_the_references_q1(eng):
    from _util import golden, lineitem_fixture_pages
    from greengage_b200 import tpch
    from greengage_b200.engine import agg_final
    from test_gpu_scanagg import gpu_scanagg
    from test_oracle_q1_golden import _check_against_golden
    desc, pages, n = lineitem_fixture_pages()
    exp = golden("q1_expected.json")
    scan, part, pool = tpch.q1_plan(capi.TAB_LINEITEM_WIDE, capi.AGGSTAGE_PARTIAL, interval_days=exp["interval_days"], desc=desc,
                                    flags=capi.AGGF_DEVICE_FINAL)
    nb = pages.size // capi.GG_BLCKSZ
    parts = []
    for lo, hi in ((0, nb // 2), (nb // 2, nb)):              # two "segments"
        rows, _, _, _ = gpu_scanagg(eng, scan, part, pool, pages[lo * capi.GG_BLCKSZ:hi * capi.GG_BLCKSZ])
        assert all(r.agg[4].f[2] == 0.0 for r in rows)        # no sumX2 travels
        parts.extend(rows)
    _check_against_golden(agg_final(eng, tpch.q1_final_agg(part), parts))


def test_q1_over_numeric_columns_is_the_references_golden_answer_to_the_last_digit(eng):
    """The reference's regression lineitem with its measures as numeric(15,2) (input/rpt_tpch.source:16-35): on-disk base-10000
    digits decoded on the device, numeric_mul / _sub / _add as exact scaled-integer arithmetic, 128-bit sums, avg with
    numeric_div's scale and rounding — every digit of output/rpt_tpch.source:309-315, not float8 within 1e-6."""
    from greengage_b200 import tpch
    from greengage_b200.engine import Relation, ScanAgg
    from oracle import pyoracle as po
    from test_oracle_numeric import check_q1_numeric_golden, numeric_lineitem_pages
    desc, pages, n = numeric_lineitem_pages()
    scan, agg, pool = tpch.q1_plan_numeric(desc, interval_days=golden("q1_expected.json")["interval_days"])
    rel = Relation(eng, host_pages=pages)
    sa = ScanAgg(eng, scan, agg, pool)
    try:
        sa.run(rel)
        got, sc, ps = sa.fetch()
        assert sc == n
        check_q1_numeric_golden(got)
        want, wsc, wps = po.seqscan_agg(scan, agg, pool, pages)
        assert (sc, ps) == (wsc, wps)
        by = {(r.key[0], r.key[1]): r for r in want}
        for r in got:
            w = by[(r.key[0], r.key[1])]
            assert [capi.numeric_of_aggval(r.agg[i]) for i in range(7)] == [capi.numeric_of_aggval(w.agg[i]) for i in range(7)]
    finally:
        sa.free()
        rel.free()


def test_numeric_values_outside_the_device_range_are_refused_not_miscomputed(eng):
    """a product beyond 64 bits at its scale raises GG_ERR_UNSUPPORTED at fetch (the relation then runs on the CPU path)"""
    from greengage_b200.capi import ExprPool, GGError
    from greengage_b200.engine import Relation, ScanAgg
    from oracle import pyoracle as po
    NUM = capi.NUMERICOID
    desc = capi.gg_tupdesc()
    desc.natts = 2
    for i, (t, l, al, bv, tm) in enumerate([(capi.INT4OID, 4, "i", 1, -1), (NUM, -1, "i", 0, ((18 << 16) | 2) + 4)]):
        a = desc.attrs[i]
        a.atttypid, a.attlen, a.attalign, a.attbyval, a.atttypmod, a.attnotnull = t, l, ord(al), bv, tm, 1
    rows = [[i, capi.numeric_payload(10 ** 15 + i, 2)] for i in range(500)]
    pages = po.build_pages(desc, rows)
    p = ExprPool()
    x = p.var(2, NUM)
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [], [(capi.AGG_SUM_NUMERIC, p.func(capi.F_NUMERIC_MUL, NUM, x, x))])
    rel = Relation(eng, host_pages=pages)
    sa = ScanAgg(eng, capi.make_scan(desc, -1), agg, p.pool)
    try:
        sa.run(rel)
        with pytest.raises(GGError) as ei:
            sa.fetch()
        assert ei.value.code == -6
    finally:
        sa.free()
        rel.free()
