"""numeric(p,s) sum / avg on the GPU against exact arithmetic (tests/_numeric.py, held to the reference's numeric.o by
test_device_emu.py): every scan-agg kernel variant, feeds in pieces, expressions, joins, and a scale where the merge kernel
folds many blocks' halves.  A device answer is either the exact one — value and display scale, compared as numeric_out
text — or GG_ERR_UNSUPPORTED with the numeric message; `_numeric.refusal` says which of the two a case allows.  The
oracle gives a second opinion where it answers."""
import numpy as np
import pytest

import _numeric as nref
from greengage_b200 import capi
from greengage_b200.capi import ExprPool
from oracle import pyoracle as po
from test_gpu_scanagg import VARIANTS, env, gpu_scanagg

pytestmark = pytest.mark.gpu
NUM = capi.NUMERICOID


@pytest.fixture(scope="module")
def eng():
    from greengage_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def num_desc(spec):
    """spec: list of (typid, typmod or None, notnull)"""
    d = capi.gg_tupdesc()
    d.natts = len(spec)
    for i, (t, tm, nn) in enumerate(spec):
        a = d.attrs[i]
        a.atttypid, a.atttypmod, a.attnotnull = t, -1 if tm is None else tm, nn
        ln, al, bv = {capi.INT4OID: (4, "i", 1), capi.FLOAT8OID: (8, "d", 1), NUM: (-1, "i", 0)}[t]
        a.attlen, a.attalign, a.attbyval = ln, ord(al), bv
    return d


# ---- the numeric edge relation ----
# columns: g int4 | a numeric(20,0) | b numeric(15,2) | c numeric(24,4) | d numeric(38,15) | e numeric(28,8)
COLS = [(20, 0), (15, 2), (24, 4), (38, 15), (28, 8)]
SCALES = [s for _, s in COLS]

NUM_EDGE_GROUPS = {
    0: "zero (no digits)", 1: "+-1 unit in the last place", 2: "negative weights: 0.01, 0.0001, 0.00000001",
    3: "stripped trailing zero digits: 10000, 10^8, 1.0000", 4: "4-digit boundaries: 9999, 10000, 9999.9999, 0.9999",
    5: "+-(2^63 - 1), the largest magnitude that fits", 6: "values near 2^62 that cancel to exactly 0",
    7: "sum crosses 2^64", 8: "sum crosses -2^64", 9: "3000 values with low 32 bits 0xFFFFFFFF",
    10: "avg ties half away from zero (positive)", 11: "avg ties (negative)", 12: "avg with sum's first digit = N's first digit",
    13: "N = 9999", 14: "N = 10000", 15: "N = 10001", 16: "one row", 17: "31 rows", 18: "32 rows", 19: "33 rows",
    20: "2000 rows across a page boundary", 21: "every input NULL", 22: "NULLs mixed with values",
    # refusal groups: each one runs in a plan of its own (WHERE g = k)
    100: "2^64 + 1 at scale 0 (digits carry past 2^64)", 101: "-(2^64 + 2792) at scale 0", 102: "2^64 + 7 unscaled at scale 4",
    103: "the integer 2^64 + 8383 at scale 4", 104: "-(2^64 + 100) unscaled at scale 8", 105: "nine base-10000 digits",
    106: "2^63 at scale 0", 107: "-2^63 at scale 0 (refused conservatively, or exact)", 108: "2^63 unscaled at scale 4",
}
REFUSAL_GROUPS = [g for g in NUM_EDGE_GROUPS if g >= 100]


def _edge_rows(rng):
    """[(g, [a, b, c, d, e] unscaled or None)]"""
    R = []
    full = lambda g, v: R.append((g, [v] * 5))
    small = lambda: [int(rng.integers(-10 ** 9, 10 ** 9)) for _ in range(5)]
    for _ in range(5):
        full(0, 0)
    for v in (1, -1, 1):
        full(1, v)
    R += [(2, [0, 1, 1, 10 ** 7, 1]), (2, [0, -1, 10 ** 4, 10 ** 11, 10 ** 4])]
    R += [(3, [10 ** 4, 10 ** 6, 10 ** 4, 10 ** 15, 10 ** 8]), (3, [10 ** 8, 10 ** 10, 10 ** 12, 10 ** 18, 10 ** 16])]
    R += [(4, [9999, 9999, 99999999, 9999 * 10 ** 11, 999999999999]), (4, [10000, 999999, 9999, 10 ** 15, 9999 * 10 ** 4])]
    m = 2 ** 63 - 1
    R += [(5, [m, 10 ** 15 - 1, m, m, m]), (5, [-m, -(10 ** 15 - 1), -m, -m, -m]), (5, [m, 10 ** 15 - 1, m, m, m])]
    x6 = [[int(rng.integers(2 ** 61, 2 ** 62)) * int(rng.choice([-1, 1])) for _ in range(5)] for _ in range(40)]
    for r in x6:
        r[1] = r[1] % 10 ** 15
    R += [(6, r) for r in x6] + [(6, [-v for v in r]) for r in x6]
    for g, sgn in ((7, 1), (8, -1)):
        R += [(g, [sgn * (2 ** 62 - int(rng.integers(0, 2 ** 40))) if c != 1 else sgn * (10 ** 15 - 1) for c in range(5)]) for _ in range(9)]
    R += [(9, [int(rng.integers(0, 2 ** 30)) * 2 ** 32 + 0xFFFFFFFF if c != 1 else int(rng.integers(0, 2 ** 17)) * 2 ** 32 + 0xFFFFFFFF
               for c in range(5)]) for _ in range(3000)]
    for g, s in ((10, 1), (11, -1)):     # a, c, e: sum 3*10^16 + 1 unscaled over 2 rows, a tie at the result scale 0, 4, 8
        R += [(g, [s * 15 * 10 ** 15, s * 1, s * 15 * 10 ** 15, s * 10 ** 15, s * 15 * 10 ** 15]),
              (g, [s * (15 * 10 ** 15 + 1), 0, s * (15 * 10 ** 15 + 1), 0, s * (15 * 10 ** 15 + 1)])]
    R += [(12, [10 ** 16, 1, 10 ** 16, 1, 10 ** 16]), (12, [10 ** 16 + 1, 0, 10 ** 16 + 1, 0, 10 ** 16 + 1])]
    for g, n in ((13, 9999), (14, 10000), (15, 10001), (16, 1), (17, 31), (18, 32), (19, 33)):
        R += [(g, small()) for _ in range(n)]
    for _ in range(4):
        R.append((21, [None] * 5))
    for _ in range(30):
        R.append((22, [v if rng.random() < 0.6 else None for v in small()]))
    R += [(100, [2 ** 64 + 1, 0, 0, 0, 0]), (100, [3, 0, 0, 0, 0]), (101, [-(2 ** 64 + 2792), 0, 0, 0, 0]), (102, [0, 0, 2 ** 64 + 7, 0, 0]), (102, [0, 0, 3, 0, 0]), (103, [0, 0, (2 ** 64 + 8383) * 10 ** 4, 0, 0]),
          (104, [0, 0, 0, 0, -(2 ** 64 + 100)]), (105, [0, 0, 0, 10 ** 32 + 10, 0]), (106, [2 ** 63, 0, 0, 0, 0]),
          (107, [-(2 ** 63), 0, 0, 0, 0]), (108, [0, 0, 2 ** 63, 0, 0])]
    return R


_cache = {}


def numeric_edge_relation(nullable=True, pad=0, long_headers=False):
    """(desc, pages, rows): the NUM_EDGE_GROUPS rows, seeded and shuffled over several pages, group 20 contiguous in the
    middle so that it straddles a page boundary.  nullable=False: rows with a NULL dropped, columns NOT NULL.  pad: float8
    columns (all 0) after e, for wide tuples.  long_headers: every third value with the 4-byte NumericLong header."""
    key = (nullable, pad, long_headers)
    if key in _cache:
        return _cache[key]
    rng = np.random.default_rng(1700)
    rows = _edge_rows(rng)
    order = rng.permutation(len(rows))
    rows = [rows[i] for i in order]
    mid = len(rows) // 2
    rows = rows[:mid] + [(20, [int(rng.integers(-2 ** 40, 2 ** 40)) for _ in range(5)]) for _ in range(2000)] + rows[mid:]
    if not nullable:
        rows = [r for r in rows if None not in r[1]]
    desc = num_desc([(capi.INT4OID, None, 1)] + [(NUM, nref.typmod(p, s), 0 if nullable else 1) for p, s in COLS] + [(capi.FLOAT8OID, None, 1)] * pad)
    tuples, nulls = [], []
    for i, (g, vals) in enumerate(rows):
        enc = [b"" if v is None else (nref.long_header_payload(v, s) if long_headers and (i + c) % 3 == 0 else capi.numeric_payload(v, s))
               for c, (v, s) in enumerate(zip(vals, SCALES))]
        tuples.append([g] + enc + [0.0] * pad)
        nulls.append([False] + [v is None for v in vals] + [False] * pad)
    pages = po.build_pages(desc, tuples, nulls)
    _cache[key] = (desc, pages, rows)
    return _cache[key]


def in_groups(p, gvar, groups):
    q = -1
    for x in groups:
        eq = p.func(capi.F_INT4EQ, capi.BOOLOID, gvar, p.const(capi.INT4OID, x))
        q = eq if q < 0 else p.boolop(capi.E_OR, q, eq)
    return q


def edge_plan(desc, groups=None, cols=range(5), count_x=True, num_groups=0):
    """[WHERE g IN groups | g < 100] GROUP BY g: count(*), then per column sum(x), avg(x)[, count(x)]"""
    p = ExprPool()
    g = p.var(1, capi.INT4OID)
    q = in_groups(p, g, groups) if groups is not None else p.func(capi.F_INT4LT, capi.BOOLOID, g, p.const(capi.INT4OID, 100))
    aggs = [(capi.AGG_COUNT_STAR, -1)]
    for c in cols:
        x = p.var(2 + c, NUM)
        aggs += [(capi.AGG_SUM_NUMERIC, x), (capi.AGG_AVG_NUMERIC, x)] + ([(capi.AGG_COUNT_ANY, x)] if count_x else [])
    return capi.make_scan(desc, q), capi.make_agg(capi.AGGSTAGE_NORMAL, [g], aggs, num_groups=num_groups), p.pool


def expected_edge(rows, groups=None, cols=range(5), count_x=True):
    """{g: [count(*), sum, avg[, count] per column]} with numeric results as text (None: NULL)"""
    by = {}
    for g, vals in rows:
        if (groups is None and g < 100) or (groups is not None and g in groups):
            by.setdefault(g, []).append(vals)
    want = {}
    for g, vs in by.items():
        out = [len(vs)]
        for c in cols:
            col = [v[c] for v in vs]
            out += [nref.sum_text(col, SCALES[c]), nref.avg_text(col, SCALES[c])] + ([sum(v is not None for v in col)] if count_x else [])
        want[g] = out
    return want


def got_rows(rows, agg):
    """device / oracle rows -> {g: [...]} in expected_edge's form"""
    out = {}
    for r in rows:
        vals = []
        for i in range(agg.numAggs):
            fn, v = agg.aggs[i].aggfnoid, r.agg[i]
            if fn in (capi.AGG_SUM_NUMERIC, capi.AGG_AVG_NUMERIC):
                vals.append(None if v.isnull else capi.numeric_of_aggval(v))
            else:
                vals.append(int(v.i))
        out[None if r.keyisnull[0] else int(r.key[0])] = vals
    return out


def assert_exact(rows, agg, want):
    got = got_rows(rows, agg)
    assert set(got) == set(want), (sorted(got), sorted(want))
    for k in want:
        assert got[k] == want[k], (k, NUM_EDGE_GROUPS.get(k), got[k], want[k])


def run_or_refusal(fn):
    """fn() -> rows; a refusal comes back as None (and must carry the numeric message)"""
    try:
        return fn()
    except capi.GGError as e:
        assert nref.is_numeric_refusal(e), str(e)
        return None


def edge_rule(rows, groups):
    vals = [v for g, vs in rows if g in groups for v in vs if v is not None]
    return nref.refusal(vals, [])


# ---- every scan-agg kernel variant ----

@pytest.mark.parametrize("nullable", [True, False])
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_numeric_edges_on_every_variant(eng, variant, nullable):
    """sum / avg / count of every column over the edge groups (refusal groups filtered out by the qual): the exact answer on
    every kernel variant, with the oracle agreeing; the oracle reads the same pages"""
    desc, pages, rows = numeric_edge_relation(nullable)
    scan, agg, pool = edge_plan(desc)
    got, sc, ps, _ = gpu_scanagg(eng, scan, agg, pool, pages, variant)
    want = expected_edge(rows)
    assert sc == len(rows) and ps == sum(want[g][0] for g in want)
    assert_exact(got, agg, want)
    orows, _, _ = po.seqscan_agg(scan, agg, pool, pages)
    assert got_rows(orows, agg) == want


@pytest.mark.parametrize("reg_slots", ["3", "0"])
@pytest.mark.parametrize("variant", ["specialised-priv", "nvrtc-priv", "interp-priv"])
def test_numeric_sums_on_the_private_accumulator_kernels(eng, monkeypatch, variant, reg_slots):
    """NOT NULL sums on the private-accumulator kernels, both halves per thread in shared memory or (plan-specialised, wide
    tuples, at most 4 groups) in registers: the carries of the 2^64 crossing, the 0xFFFFFFFF low halves, +-(2^63 - 1)"""
    monkeypatch.setenv("GGB200_REG_SLOTS", reg_slots)
    desc, pages, rows = numeric_edge_relation(nullable=False, pad=12)
    for groups in ((5, 7, 8, 9), (6, 10, 11, 12)):
        scan, agg, pool = edge_plan(desc, groups, count_x=False)
        got, sc, ps, var = gpu_scanagg(eng, scan, agg, pool, pages, variant)
        assert var % 16 == 0, "private-accumulator kernel expected, got variant %d" % var
        assert (var >= 16) == (variant != "interp-priv"), var
        assert_exact(got, agg, expected_edge(rows, groups, count_x=False))


def test_numeric_edges_on_the_general_hash_aggregate(eng):
    """the group table in HBM: from the start (a large planner estimate), and grown from a low one on more groups than the
    private accumulators hold (group k = row number, so the table has to grow)"""
    from greengage_b200.engine import Relation, ScanAgg
    desc, pages, rows = numeric_edge_relation()
    scan, agg, pool = edge_plan(desc, num_groups=1 << 20)
    got, _, _, var = gpu_scanagg(eng, scan, agg, pool, pages)
    assert var % 16 == 5, var
    assert_exact(got, agg, expected_edge(rows))
    # 150 000 distinct keys against an estimate of 100
    rng = np.random.default_rng(5)
    d2 = num_desc([(capi.INT4OID, None, 1), (NUM, nref.typmod(24, 4), 1)])
    vals = [int(rng.integers(2 ** 61, 2 ** 62)) * (1 if i % 3 else -1) for i in range(300_000)]
    keys = [i % 150_000 for i in range(300_000)]
    pg = po.build_pages(d2, [[k, capi.numeric_payload(v, 4)] for k, v in zip(keys, vals)])
    p = ExprPool()
    g, x = p.var(1, capi.INT4OID), p.var(2, NUM)
    agg2 = capi.make_agg(capi.AGGSTAGE_NORMAL, [g], [(capi.AGG_SUM_NUMERIC, x), (capi.AGG_AVG_NUMERIC, x)], num_groups=100)
    with env(GGB200_SCAN_MODE="5"):
        sa = ScanAgg(eng, capi.make_scan(d2, -1), agg2, p.pool)
    rel = Relation(eng, host_pages=pg)
    try:
        sa.run(rel)
        out, _, _ = sa.fetch(cap=200_000)
    finally:
        sa.free()
        rel.free()
    by = {}
    for k, v in zip(keys, vals):
        by.setdefault(k, []).append(v)
    assert len(out) == len(by)
    for r in out:
        vs = by[int(r.key[0])]
        assert [capi.numeric_of_aggval(r.agg[0]), capi.numeric_of_aggval(r.agg[1])] == [nref.sum_text(vs, 4), nref.avg_text(vs, 4)]


@pytest.mark.parametrize("variant", ["specialised-priv", "interp-priv", "interp-tr", "specialised-tr"])
def test_numeric_values_past_the_device_range_are_refused(eng, variant):
    """each refusal group on its own: the 2^64 carry family at scales 0, 4 and 8, nine base-10000 digits and 2^63 must come
    back as GG_ERR_UNSUPPORTED, never as a number; -2^63 may be refused or exact"""
    desc, pages, rows = numeric_edge_relation(nullable=variant.endswith("tr"))
    outcomes = {}
    for k in REFUSAL_GROUPS:
        scan, agg, pool = edge_plan(desc, (k,))
        got = run_or_refusal(lambda: gpu_scanagg(eng, scan, agg, pool, pages, variant)[0])
        rule = edge_rule(rows, (k,))
        outcomes[k] = got is None
        if rule == nref.REQUIRED:
            assert got is None, (k, NUM_EDGE_GROUPS[k], got_rows(got, agg))
        else:
            assert rule == nref.EITHER and k == 107
            if got is not None:
                assert_exact(got, agg, expected_edge(rows, (k,)))
    assert sum(outcomes.values()) >= len(REFUSAL_GROUPS) - 1


def test_numeric_long_headers_wide_tuples_and_feeds_in_pieces(eng):
    """the NumericLong header form mixed with short headers, wide tuples, and the same pages fed as several block ranges or
    from host memory: each equals the exact answer, as one resident run does"""
    for nullable, pad, lh in ((True, 0, True), (False, 6, True), (True, 9, False)):
        desc, pages, rows = numeric_edge_relation(nullable, pad, lh)
        scan, agg, pool = edge_plan(desc)
        want = expected_edge(rows)
        nb = pages.size // capi.GG_BLCKSZ
        assert nb >= 8
        for kw in ({}, {"ranges": [(0, 1), (1, nb // 2), (nb // 2, nb)]}, {"host": True}):
            got, sc, ps, _ = gpu_scanagg(eng, scan, agg, pool, pages, **kw)
            assert sc == len(rows), kw
            assert_exact(got, agg, want)


def test_numeric_plain_aggregate_over_no_rows_and_partial_stage(eng):
    """a plain aggregate whose qual passes nothing: one row, count 0, sum and avg NULL; and a numeric aggregate at PARTIAL
    stage is still refused when the pipeline is created"""
    desc, pages, rows = numeric_edge_relation()
    p = ExprPool()
    x = p.var(3, NUM)
    q = p.func(capi.F_INT4LT, capi.BOOLOID, p.var(1, capi.INT4OID), p.const(capi.INT4OID, -5))
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [], [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_NUMERIC, x), (capi.AGG_AVG_NUMERIC, x), (capi.AGG_COUNT_ANY, x)])
    for variant in ("specialised-priv", "interp-tr"):
        got, sc, ps, _ = gpu_scanagg(eng, capi.make_scan(desc, q), agg, p.pool, pages, variant)
        assert len(got) == 1 and ps == 0
        assert got[0].agg[0].i == 0 and got[0].agg[1].isnull and got[0].agg[2].isnull and got[0].agg[3].i == 0
    part = capi.make_agg(capi.AGGSTAGE_PARTIAL, [p.var(1, capi.INT4OID)], [(capi.AGG_SUM_NUMERIC, x)])
    with pytest.raises(capi.GGError) as e:
        gpu_scanagg(eng, capi.make_scan(desc, -1), part, p.pool, pages)
    assert e.value.code == -6


# ---- expressions ----

def _expr_relation(rows):
    """(k int4, x numeric(15,2), y numeric(12,4), z numeric(10,0)), NOT NULL; rows: (k, x, y, z) unscaled"""
    d = num_desc([(capi.INT4OID, None, 1), (NUM, nref.typmod(15, 2), 1), (NUM, nref.typmod(12, 4), 1), (NUM, nref.typmod(10, 0), 1)])
    return d, po.build_pages(d, [[k, capi.numeric_payload(x, 2), capi.numeric_payload(y, 4), capi.numeric_payload(z, 0)] for k, x, y, z in rows])


def test_numeric_expressions_equal_exact_arithmetic(eng):
    """x*y (scale 6), x+y with mixed scales (4), x - 7.5, 7.5 - x (the reversed subtract), under quals that compare across
    scales (1.0 = 1.00, a scale-0 column against 1.5)"""
    rng = np.random.default_rng(31)
    rows = [(int(rng.integers(0, 3)), int(rng.choice([100, 10 ** 6, int(rng.integers(-10 ** 9, 10 ** 9))])), int(rng.integers(-10 ** 9, 10 ** 9)),
             int(rng.integers(-5, 6))) for _ in range(20000)]
    desc, pages = _expr_relation(rows)
    p = ExprPool()
    k, x, y, z = p.var(1, capi.INT4OID), p.var(2, NUM), p.var(3, NUM), p.var(4, NUM)
    c75 = p.const(NUM, "7.5")
    exprs = [(p.func(capi.F_NUMERIC_MUL, NUM, x, y), 6, lambda r: r[1] * r[2]),
             (p.func(capi.F_NUMERIC_ADD, NUM, x, y), 4, lambda r: r[1] * 100 + r[2]),
             (p.func(capi.F_NUMERIC_SUB, NUM, x, c75), 2, lambda r: r[1] - 750),
             (p.func(capi.F_NUMERIC_SUB, NUM, c75, x), 2, lambda r: 750 - r[1])]
    quals = [(p.func(capi.F_NUMERIC_EQ, capi.BOOLOID, x, p.const(NUM, "10000.0")), lambda r: r[1] == 10 ** 6),      # 10000.0 = 10000.00
             (p.func(capi.F_NUMERIC_LT, capi.BOOLOID, z, p.const(NUM, "1.5")), lambda r: r[3] < 1.5),
             (p.func(capi.F_NUMERIC_GE, capi.BOOLOID, y, x), lambda r: r[2] >= r[1] * 100)]
    for qi, (q, qf) in enumerate(quals):
        agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [k], [(capi.AGG_COUNT_STAR, -1)] + [(f, e) for e, _, _ in exprs for f in (capi.AGG_SUM_NUMERIC, capi.AGG_AVG_NUMERIC)])
        by = {}
        for r in rows:
            if qf(r):
                by.setdefault(r[0], []).append(r)
        want = {g: [len(rs)] + [t for _, s, f in exprs for t in (nref.sum_text([f(r) for r in rs], s), nref.avg_text([f(r) for r in rs], s))]
                for g, rs in by.items()}
        assert all(len(v) > 0 for v in by.values()) and len(by) == 3, qi
        for variant in ("specialised-tr", "interp-tr"):
            got, sc, ps, _ = gpu_scanagg(eng, capi.make_scan(desc, q), agg, p.pool, pages, variant)
            assert_exact(got, agg, want)
        orows, _, _ = po.seqscan_agg(capi.make_scan(desc, q), agg, p.pool, pages)
        assert got_rows(orows, agg) == want


def test_numeric_product_just_below_and_just_above_2_63(eng):
    """x*y at scale 6: 92233720.36 * 100000.0000 (9223372036 * 10^9 unscaled, 854775808 below 2^63) is exact, and so is its
    negative; 92233720.37 * 100000.0000 is past 2^63 and refused"""
    assert 9223372036 * 10 ** 9 < 2 ** 63 < 9223372037 * 10 ** 9
    for xv, yv, must_refuse in ((9223372036, 10 ** 9, False), (-9223372036, 10 ** 9, False), (9223372037, 10 ** 9, True)):
        desc, pages = _expr_relation([(0, xv, yv, 0), (0, 1, 1, 0)])
        p = ExprPool()
        prod = p.func(capi.F_NUMERIC_MUL, NUM, p.var(2, NUM), p.var(3, NUM))
        agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [], [(capi.AGG_SUM_NUMERIC, prod)])
        assert nref.refusal([xv, yv, xv * yv], []) == (nref.REQUIRED if must_refuse else nref.EITHER)
        for variant in ("specialised-priv", "interp-tr"):
            got = run_or_refusal(lambda: gpu_scanagg(eng, capi.make_scan(desc, -1), agg, p.pool, pages, variant)[0])
            if must_refuse:
                assert got is None, variant
            else:                            # above 2^62, so a refusal would be allowed; the device takes it exactly
                assert got is not None and capi.numeric_of_aggval(got[0].agg[0]) == nref.text(xv * yv + 1, 6), variant


def test_numeric_sums_of_two_million_values_near_2_62(eng):
    """2 048 000 rows of mixed-sign values near 2^62 over 4 groups: the merge kernel folds the halves of many blocks, and the
    sums pass 2^64 several times over"""
    rng = np.random.default_rng(62)
    d = num_desc([(capi.INT4OID, None, 1), (NUM, nref.typmod(24, 4), 1)])
    one = []
    while True:
        v = int(rng.integers(2 ** 61, 2 ** 62)) * (1 if rng.random() < 0.7 else -1)
        one.append((len(one) % 4, v))
        pg = po.build_pages(d, [[g, capi.numeric_payload(x, 4)] for g, x in one])
        if pg.size > capi.GG_BLCKSZ:
            one.pop()
            break
    pg = po.build_pages(d, [[g, capi.numeric_payload(x, 4)] for g, x in one])
    reps = -(-2_000_000 // len(one))
    pages = np.tile(pg, reps)
    p = ExprPool()
    g, x = p.var(1, capi.INT4OID), p.var(2, NUM)
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [g], [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_NUMERIC, x), (capi.AGG_AVG_NUMERIC, x)])
    want = {}
    for k in range(4):
        vs = [v for gg, v in one if gg == k]
        s, n = sum(vs) * reps, len(vs) * reps
        assert abs(s) > 2 ** 64
        want[k] = [n, nref.text(s, 4), nref.text(*nref.avg(s, 4, n))]
    for variant in ("specialised-priv", "interp-tr"):
        got, sc, ps, _ = gpu_scanagg(eng, capi.make_scan(d, -1), agg, p.pool, pages, variant)
        assert sc == len(one) * reps >= 2_000_000
        assert_exact(got, agg, want)


# ---- joins ----

JOIN_VARIANTS = {"specialised": {}, "interp": {"GGB200_JIT": "0"}}


def _join_relations(rng, big_inner=False):
    """outer (k int4, g int4, x numeric(15,2) nullable), inner (k int4, n numeric(12,4) nullable, y numeric(10,0));
    inner keys 0..299 with duplicates, outer keys 0..399 (some without a partner)"""
    od = num_desc([(capi.INT4OID, None, 1), (capi.INT4OID, None, 1), (NUM, nref.typmod(15, 2), 0)])
    idd = num_desc([(capi.INT4OID, None, 1), (NUM, nref.typmod(12, 4), 0), (NUM, nref.typmod(10, 0), 1)])
    orows = [(int(rng.integers(0, 400)), int(rng.integers(0, 3)), None if rng.random() < 0.1 else int(rng.integers(-10 ** 12, 10 ** 12))) for _ in range(6000)]
    irows = [(int(rng.integers(0, 300)), None if rng.random() < 0.1 else int(rng.integers(-10 ** 14, 10 ** 14)), int(rng.integers(-10 ** 6, 10 ** 6))) for _ in range(900)]
    if big_inner:
        irows[17] = (irows[17][0], 2 ** 63 + 5, irows[17][2])
    enc = lambda v, s: b"" if v is None else capi.numeric_payload(v, s)
    opages = po.build_pages(od, [[k, g, enc(x, 2)] for k, g, x in orows], [[False, False, x is None] for _, _, x in orows])
    ipages = po.build_pages(idd, [[k, enc(n, 4), enc(y, 0)] for k, n, y in irows], [[False, n is None, False] for _, n, _ in irows])
    return od, idd, orows, irows, opages, ipages


def _join_expected(orows, irows, jointype, pred, cols):
    """GROUP BY outer.g of the joined rows (a LEFT join's null-extended rows have inner values None): per col fn -> values"""
    ib = {}
    for r in irows:
        ib.setdefault(r[0], []).append(r)
    groups = {}
    for o in orows:
        matched = [i for i in ib.get(o[0], []) if pred(o, i)]
        outs = [(o, i) for i in matched]
        if not matched and jointype == capi.JOIN_LEFT:
            outs = [(o, None)]
        for o2, i in outs:
            groups.setdefault(o2[1], []).append((o2, i))
    want = {}
    for g, prs in groups.items():
        row = [len(prs)]
        for f, s in cols:
            vs = [f(o, i) for o, i in prs]
            row += [nref.sum_text(vs, s), nref.avg_text(vs, s), sum(v is not None for v in vs)]
        want[g] = row
    return want


def _gpu_join(eng, outer, inner, hj, agg, pool, opages, ipages, variant, work_mem=0):
    from greengage_b200.engine import JoinAgg, Relation
    with env(**JOIN_VARIANTS[variant]):
        ja = JoinAgg(eng, outer, inner, hj, agg, pool)
        orel, irel = Relation(eng, host_pages=opages), Relation(eng, host_pages=ipages)
        try:
            if work_mem:
                ja.set_work_mem(work_mem)
                ja.run(irel, orel)
            else:
                ja.build(irel)
                ja.probe(orel)
            return ja.fetch()[0]
        finally:
            ja.free()
            orel.free()
            irel.free()


def _mul(a, b):
    return None if a is None or b is None else a * b


@pytest.mark.parametrize("variant", list(JOIN_VARIANTS))
@pytest.mark.parametrize("jointype", [capi.JOIN_INNER, capi.JOIN_LEFT])
def test_numeric_inner_columns_above_a_join(eng, variant, jointype):
    """sum / avg / count of an inner numeric column (NULLs among them, and a LEFT join's null-extended rows), of
    outer.x * inner.y, and under a join qual comparing an outer and an inner numeric at different scales, both ways round"""
    od, idd, orows, irows, opages, ipages = _join_relations(np.random.default_rng(40))
    for qi in range(3):
        p = ExprPool()
        ok, og, ox = p.var(1, capi.INT4OID, 0), p.var(2, capi.INT4OID, 0), p.var(3, NUM, 0)
        ik, inn, iy = p.var(1, capi.INT4OID, 1), p.var(2, NUM, 1), p.var(3, NUM, 1)
        if qi == 0:
            jq, pred = -1, lambda o, i: True
        elif qi == 1:        # outer scale 2 < inner scale 4: the outer side is loaded at scale 4
            jq, pred = p.func(capi.F_NUMERIC_LT, capi.BOOLOID, ox, inn), lambda o, i: o[2] is not None and i[1] is not None and o[2] * 100 < i[1]
        else:                # inner scale 0 against outer scale 2: the inner payload is rescaled by 100
            jq, pred = p.func(capi.F_NUMERIC_GE, capi.BOOLOID, iy, ox), lambda o, i: o[2] is not None and i[2] * 100 >= o[2]
        hj = capi.make_hashjoin(jointype, [ok], [ik], jq)
        prod = p.func(capi.F_NUMERIC_MUL, NUM, ox, iy)
        aggs = [(capi.AGG_COUNT_STAR, -1)]
        for e in (inn, prod):
            aggs += [(capi.AGG_SUM_NUMERIC, e), (capi.AGG_AVG_NUMERIC, e), (capi.AGG_COUNT_ANY, e)]
        agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [og], aggs)
        cols = [(lambda o, i: None if i is None else i[1], 4), (lambda o, i: None if i is None else _mul(o[2], i[2]), 2)]
        want = _join_expected(orows, irows, jointype, pred, cols)
        outer, inner = capi.make_scan(od, -1), capi.make_scan(idd, -1)
        got = _gpu_join(eng, outer, inner, hj, agg, p.pool, opages, ipages, variant)
        assert_exact(got, agg, want)
        orow, _ = po.hashjoin_agg(outer, inner, hj, agg, p.pool, opages, ipages)
        assert got_rows(orow, agg) == want, qi


def test_numeric_inner_value_past_the_range_and_batched_joins_are_refused(eng):
    """an inner value >= 2^63 is refused by the build (and stays refused through the probe's escalations); a join that has to
    run in batches moves columns as datum rows, which numeric does not travel as yet, so it is refused — never wrong"""
    od, idd, orows, irows, opages, ipages = _join_relations(np.random.default_rng(41), big_inner=True)
    p = ExprPool()
    hj = capi.make_hashjoin(capi.JOIN_INNER, [p.var(1, capi.INT4OID, 0)], [p.var(1, capi.INT4OID, 1)])
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [p.var(2, capi.INT4OID, 0)], [(capi.AGG_SUM_NUMERIC, p.var(2, NUM, 1))])
    for variant in JOIN_VARIANTS:
        with pytest.raises(capi.GGError) as e:
            _gpu_join(eng, capi.make_scan(od, -1), capi.make_scan(idd, -1), hj, agg, p.pool, opages, ipages, variant)
        assert nref.is_numeric_refusal(e.value), str(e.value)
    od, idd, orows, irows, opages, ipages = _join_relations(np.random.default_rng(42))
    with pytest.raises(capi.GGError) as e:
        _gpu_join(eng, capi.make_scan(od, -1), capi.make_scan(idd, -1), hj, agg, p.pool, opages, ipages, "specialised", work_mem=8192)
    assert e.value.code == -6 and "numeric" in str(e.value), str(e.value)
