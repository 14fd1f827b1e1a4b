"""An Agg's HAVING (plan.qual) on the device: the row filter over datum rows (gg_rowfilter_*) and the executor paths that use it.

ABI: the rows that pass are the oracle's (the qual evaluated by or_eval over the same rows written as heap pages), in input order,
dead slots dropped, for every output type, NULLs and float8 edge values; the errors are the oracle's, and an arm that AND / OR
skip raises nothing.  Node surface: an Agg with HAVING at the top of the slice, under Sort / Limit, under a Gather, on either side
of a HashJoin, as the FINAL stage over device groups and over host rows, as a plain Agg, in every kernel variant and after a
ReScan, against the same Agg without HAVING filtered by the oracle; the select_having goldens; TPC-H Q18; more than 2^24 groups."""
import json
import os
import struct
from collections import Counter

import numpy as np
import pytest

from greengage_b200 import capi, executor as ex
from greengage_b200.capi import ExprPool
from oracle import pyoracle as po
from test_gpu_agg_rows import TYPES, VARIANTS, _two_stage, datum_words, full_agg, key_exprs, load_rows, make_data
from test_join_tree_reference import rows_pages

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
STRINGS = (capi.BPCHAROID, capi.VARCHAROID, capi.TEXTOID)
DEAD = np.uint64(1 << 63)


@pytest.fixture(scope="module")
def eng():
    from greengage_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def f8(bits):
    return struct.unpack("<d", struct.pack("<q", int(bits)))[0]


def py_value(t, v, isnull):
    if isnull:
        return None
    if t == capi.FLOAT8OID:
        return f8(v)
    if t in STRINGS:
        return (int(v) & 0xFFFFFFFFFFFFFFFF).to_bytes(8, "little").rstrip(b"\0")
    return int(v)


def oracle_passes(types, rows, pool, qual):
    """which rows (Python values) pass `qual`: the oracle's scan qual over them as heap pages (a row id column appended, grouped
    on); raises po.OracleError as the oracle does"""
    if not rows:
        return []
    n = len(types)
    pages = rows_pages(list(types) + [capi.INT8OID], [list(r) + [i] for i, r in enumerate(rows)])
    from test_join_tree_reference import rows_desc
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [pool_var(pool, n + 1)], [(capi.AGG_COUNT_STAR, -1)])
    got, _, _ = po.seqscan_agg(capi.make_scan(rows_desc(list(types) + [capi.INT8OID]), qual), agg, pool.pool, pages, cap=len(rows) + 1)
    ok = {int(r.key[0]) for r in got}
    return [i in ok for i in range(len(rows))]


def pool_var(pool, attno):
    return pool.var(attno, capi.INT8OID)


# ---- ABI ----
ABI_TYPES = [capi.INT4OID, capi.INT8OID, capi.DATEOID, capi.FLOAT8OID, capi.BPCHAROID]


def abi_rows(n, seed):
    rng = np.random.default_rng(seed)
    vals = np.zeros((n, 5), dtype=np.int64)
    vals[:, 0] = rng.integers(-5, 5, n)
    vals[:, 1] = rng.integers(-10**6, 10**6, n)
    vals[:, 2] = rng.integers(-200, 200, n)
    f = rng.integers(-40, 40, n).astype(np.float64) / 4
    sp = rng.random(n)
    f[sp < 0.03] = -0.0
    f[(sp >= 0.03) & (sp < 0.05)] = np.inf
    f[(sp >= 0.05) & (sp < 0.07)] = -np.inf
    f[(sp >= 0.07) & (sp < 0.09)] = np.nan
    f[(sp >= 0.09) & (sp < 0.10)] = 1e300
    vals[:, 3] = f.view(np.int64)
    strs = np.array([int.from_bytes(s, "little") for s in (b"A", b"BB", b"CCC", b"DDDDDDDD")], dtype=np.int64)
    vals[:, 4] = strs[rng.integers(0, 4, n)]
    nulls = rng.random((n, 5)) < 0.08
    vals[nulls] = 0
    return vals, nulls


def abi_quals(p):
    i4, i8, d, f, c = (p.var(k + 1, t) for k, t in enumerate(ABI_TYPES))
    F, K = p.func, p.const
    gt = lambda fn, a, t, v: F(fn, capi.BOOLOID, a, K(t, v))
    return {
        "f_gt": gt(capi.F_FLOAT8GT, f, capi.FLOAT8OID, 1.5),
        "f_eq_zero": gt(capi.F_FLOAT8EQ, f, capi.FLOAT8OID, 0.0),
        "i8_or_fnull": p.boolop(capi.E_OR, gt(capi.F_INT8GT, i8, capi.INT8OID, 100), p.boolop(capi.E_ISNULL, f)),
        "not_and": p.boolop(capi.E_AND, p.boolop(capi.E_NOT, gt(capi.F_INT4EQ, i4, capi.INT4OID, 3)), gt(capi.F_DATE_LT, d, capi.DATEOID, 50)),
        "str_or_i4null": p.boolop(capi.E_OR, F(capi.F_BPCHAREQ, capi.BOOLOID, c, K(capi.BPCHAROID, "BB")), p.boolop(capi.E_ISNULL, i4)),
        "arith": gt(capi.F_FLOAT8LT, F(capi.F_FLOAT8MI, capi.FLOAT8OID, F(capi.F_I8TOD, capi.FLOAT8OID, i8), f), capi.FLOAT8OID, 0.0),
        # errors: the second arm overflows (f * 1e308) or divides by zero, but only where the first arm lets it run
        # (a NULL first clause of the top-level AND stops ExecQual's clause list, but not the oracle's AND: both decide here)
        "skipped_overflow": p.boolop(capi.E_AND, p.boolop(capi.E_AND, p.boolop(capi.E_ISNOTNULL, i4), gt(capi.F_INT4LT, i4, capi.INT4OID, -100)),
                                     gt(capi.F_FLOAT8GT, F(capi.F_FLOAT8MUL, capi.FLOAT8OID, f, K(capi.FLOAT8OID, 1e308)), capi.FLOAT8OID, 0.0)),
        "or_divzero": p.boolop(capi.E_OR, p.boolop(capi.E_ISNOTNULL, i4),
                               gt(capi.F_FLOAT8GT, F(capi.F_FLOAT8DIV, capi.FLOAT8OID, f, K(capi.FLOAT8OID, 0.0)), capi.FLOAT8OID, 0.0)),
        "overflow": p.boolop(capi.E_AND, p.boolop(capi.E_ISNOTNULL, i4),
                             gt(capi.F_FLOAT8GT, F(capi.F_FLOAT8MUL, capi.FLOAT8OID, f, K(capi.FLOAT8OID, 1e308)), capi.FLOAT8OID, 0.0)),
        "divzero": gt(capi.F_FLOAT8GT, F(capi.F_FLOAT8DIV, capi.FLOAT8OID, f, K(capi.FLOAT8OID, 0.0)), capi.FLOAT8OID, 0.0),
    }


@pytest.mark.parametrize("n", [1, 300, 70_000])
def test_rowfilter_equals_the_oracle(eng, n):
    from greengage_b200.engine import RowFilter
    vals, nulls = abi_rows(n, seed=n)
    rel, rows = load_rows(eng, vals, nulls)
    words = datum_words(vals, nulls)
    pyrows = [tuple(py_value(t, vals[r, c], nulls[r, c]) for c, t in enumerate(ABI_TYPES)) for r in range(n)]
    p = ExprPool()
    try:
        for name, q in abi_quals(p).items():
            f = RowFilter(eng, capi.rows_tupdesc(ABI_TYPES), q, p.pool)
            try:
                try:
                    ok = oracle_passes(ABI_TYPES, pyrows, p, q)
                    want_err = None
                except po.OracleError as e:
                    want_err = e.code
                if want_err is not None:
                    with pytest.raises(capi.GGError) as e:
                        f.run(rows)
                    assert e.value.code == want_err, name
                    continue
                got = f.run(rows)
                assert np.array_equal(got, words[np.array(ok, dtype=bool)]), name          # same rows, same order
                assert np.array_equal(f.run(rows), got)                                    # a second run: the same bytes
            finally:
                f.free()
    finally:
        rows.free(); rel.free()


def test_rowfilter_errors_dead_slots_and_prefix(eng):
    from greengage_b200.engine import RowFilter
    vals, nulls = abi_rows(5000, seed=7)
    nulls[:, 0] = False                                                          # i4 decides the first arm on every row
    vals[:, 3] = np.where(nulls[:, 3], 0, np.float64(2.0).view(np.int64))       # every non-NULL f overflows when multiplied by 1e308
    rel, rows = load_rows(eng, vals, nulls)
    p = ExprPool()
    qs = abi_quals(p)
    try:
        f = RowFilter(eng, capi.rows_tupdesc(ABI_TYPES), qs["overflow"], p.pool)
        with pytest.raises(capi.GGError) as e:
            f.run(rows)
        assert e.value.code == -2                            # GG_ERR_FLOAT_OVERFLOW
        f.free()
        f = RowFilter(eng, capi.rows_tupdesc(ABI_TYPES), qs["skipped_overflow"], p.pool)
        assert f.run(rows).shape == (0, 6)                   # i4 is never < -100: the product is never computed
        f.free()
        f = RowFilter(eng, capi.rows_tupdesc(ABI_TYPES), qs["divzero"], p.pool)
        with pytest.raises(capi.GGError) as e:
            f.run(rows)
        assert e.value.code == -4                            # GG_ERR_DIV_ZERO
        f.free()
        # dead slots are dropped; nrows filters a prefix; nrows == 0 gives nothing
        words = datum_words(vals, nulls)
        dead = np.zeros(5000, dtype=bool)
        dead[::7] = True
        buf = np.zeros(rel.nblocks * capi.GG_BLCKSZ // 8, dtype=np.uint64)
        w2 = words.copy()
        w2[dead, 0] |= DEAD
        buf[:w2.size] = w2.ravel()
        rel.load(0, buf.view(np.uint8))
        f = RowFilter(eng, capi.rows_tupdesc(ABI_TYPES), qs["i8_or_fnull"], p.pool)
        ok = np.array(oracle_passes(ABI_TYPES, [tuple(py_value(t, vals[r, c], nulls[r, c]) for c, t in enumerate(ABI_TYPES))
                                                for r in range(5000)], p, qs["i8_or_fnull"]))
        assert np.array_equal(f.run(rows), words[ok & ~dead])
        assert np.array_equal(f.run(rows, 1234), words[:1234][(ok & ~dead)[:1234]])
        assert f.run(rows, 0).shape == (0, 6)
        f.free()
        with pytest.raises(capi.GGError):
            f = RowFilter(eng, capi.rows_tupdesc(ABI_TYPES[:4]), qs["str_or_i4null"], p.pool)      # Var 5 of 4 columns
    finally:
        rows.free(); rel.free()


def test_rowfilter_refusals(eng):
    from greengage_b200.engine import RowFilter
    p = ExprPool()
    desc = capi.rows_tupdesc(ABI_TYPES)
    bad = p.func(9999, capi.BOOLOID, p.var(1, capi.INT4OID), p.const(capi.INT4OID, 1))
    with pytest.raises(capi.GGError) as e:
        RowFilter(eng, desc, bad, p.pool)
    assert e.value.code == -6                                 # GG_ERR_UNSUPPORTED
    with pytest.raises(capi.GGError) as e:
        RowFilter(eng, desc, p.pool.nnodes + 3, p.pool)
    assert e.value.code == -10                                # GG_ERR_ARG
    nd = capi.rows_tupdesc([capi.INT4OID, capi.NUMERICOID])
    q = p.func(capi.F_NUMERIC_GT, capi.BOOLOID, p.var(2, capi.NUMERICOID), p.const(capi.NUMERICOID, "1.5"))
    with pytest.raises(capi.GGError) as e:
        RowFilter(eng, nd, q, p.pool)
    assert e.value.code == -6


# ---- node surface ----
def agg_rows_py(x):
    """a finished Executor's slot rows as Python values, and the column types"""
    out, types = [], None
    for vals, nl, ty, ln in x.rows():
        types = list(ty)
        out.append(tuple(py_value(t, v, n) for v, n, t in zip(vals, nl, ty)))
    return out, types


def tok(r):
    """a row as a hashable token: float8 by its bits, but every NaN one token and the zeros one token (the sign of a zero min / max
    of a group with zeros of both signs is left to the order the HashAggregate's atomics ran in)"""
    return tuple(("nan" if x != x else "zero" if x == 0 else struct.pack("<d", x)) if isinstance(x, float) else x for x in r)


def expected_having(eng, pool, rels, plan_fn, qual, interconnect=None):
    """the same plan without HAVING, at the top, filtered by the oracle: (rows, types)"""
    b = ex.PlanBuilder()
    x = ex.Executor(eng, pool.pool, rels, plan_fn(b, -1), interconnect=interconnect)
    try:
        rows, types = agg_rows_py(x)
    finally:
        x.end()
    if not rows:
        return [], types
    ok = oracle_passes(types, rows, pool, qual)
    return [r for r, k in zip(rows, ok) if k], types


def check_top(eng, pool, rels, plan_fn, qual, interconnect=None, rescan=True, min_rows=1):
    want, _ = expected_having(eng, pool, rels, plan_fn, qual, interconnect)
    b = ex.PlanBuilder()
    x = ex.Executor(eng, pool.pool, rels, plan_fn(b, qual), interconnect=interconnect)
    try:
        got, _ = agg_rows_py(x)
        assert Counter(map(tok, got)) == Counter(map(tok, want))
        assert len(want) >= min_rows
        ins = dict(x.instrumentation())
        top = x.locations()[0][0]
        assert ins[top].ntuples == len(want)
        if rescan:
            x.rescan()
            again, _ = agg_rows_py(x)
            assert Counter(map(tok, again)) == Counter(map(tok, got))
    finally:
        x.end()
    return want


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_having_at_the_top_in_every_variant(eng, variant):
    keys, g3, ng, n, nullable = VARIANTS[variant]
    vals, nulls = make_data(n, g3, seed=len(variant) + 40, nullable=nullable)
    rel, rows = load_rows(eng, vals, nulls)
    p = ExprPool()
    agg = full_agg(p, key_exprs(p, keys), ng)
    nk = agg.numCols
    desc = capi.rows_tupdesc(TYPES, notnull=None if nullable else [1] * 7)
    # count(*) > 3 OR the float sum is NULL, AND max(i) >= -900000 (keys and aggregates of several types)
    cnt, fsum, maxi = p.var(nk + 1, capi.INT8OID), p.var(nk + 3, capi.FLOAT8OID), p.var(nk + 9, capi.INT4OID)
    q = p.boolop(capi.E_AND, p.boolop(capi.E_OR, p.func(capi.F_INT8GT, capi.BOOLOID, cnt, p.const(capi.INT8OID, 3)), p.boolop(capi.E_ISNULL, fsum)),
                 p.func(capi.F_INT4GE, capi.BOOLOID, maxi, p.const(capi.INT4OID, -900000)))
    try:
        check_top(eng, p, [rows], lambda b, qq: b.agg(b.seqscan(0, desc), agg, having=qq), q)
    finally:
        rows.free(); rel.free()


def test_having_under_sort_limit_and_gather(eng):
    vals, nulls = make_data(60000, 500, seed=51)
    rel, rows = load_rows(eng, vals, nulls)
    p = ExprPool()
    agg = full_agg(p, key_exprs(p, "many"), 0)
    desc = capi.rows_tupdesc(TYPES)
    q = p.func(capi.F_INT8GT, capi.BOOLOID, p.var(3, capi.INT8OID), p.const(capi.INT8OID, 40))          # count(*) > 40
    keys = [capi.make_sortkey(2, capi.INT8OID, desc=True), capi.make_sortkey(0, capi.INT8OID), capi.make_sortkey(1, capi.INT4OID)]
    plan = lambda b, qq: b.agg(b.seqscan(0, desc), agg, having=qq)
    try:
        want = check_top(eng, p, [rows], plan, q, min_rows=10)
        srt = sorted(want, key=lambda r: (-r[2], r[0], r[1] if r[1] is not None else 1 << 40))
        assert 0 < len(want) < 2000
        for count, offset in ((None, None), (10, 3), (len(want) + 5, None)):
            b = ex.PlanBuilder()
            top = b.sort(plan(b, q), keys) if count is None else b.limit(b.sort(plan(b, q), keys), count, offset)
            x = ex.Executor(eng, p.pool, [rows], top)
            try:
                got, _ = agg_rows_py(x)
                lo = offset or 0
                assert [tok(r) for r in got] == [tok(r) for r in (srt if count is None else srt[lo:lo + count])]
                assert ("scanagg", "device-rows") in x.locations()
            finally:
                x.end()
        # under a Gather Motion (one segment, no interconnect: the host-row path takes the survivors)
        check_top(eng, p, [rows], lambda b, qq: b.motion(plan(b, qq), ex.MOTION_GATHER), q, rescan=False)
    finally:
        rows.free(); rel.free()


@pytest.mark.parametrize("path", ["device-groups", "host-rows"])
def test_having_on_the_final_stage(eng, path):
    from greengage_b200.engine import Interconnect
    vals, nulls = make_data(40000, 300, seed=61)
    rel, rows = load_rows(eng, vals, nulls)
    p = ExprPool()
    desc = capi.rows_tupdesc(TYPES)
    ic = Interconnect(eng, 1, 0) if path == "device-groups" else None
    # "tiny": 5 groups, which a Motion block carries; count(*) > 9500 OR the key IS NULL keeps 3 of them
    q = p.boolop(capi.E_OR, p.func(capi.F_INT8GT, capi.BOOLOID, p.var(2, capi.INT8OID), p.const(capi.INT8OID, 9500)), p.boolop(capi.E_ISNULL, p.var(1, capi.BPCHAROID)))

    def plan(b, qq):
        top = _two_stage(b, desc, p, "tiny")
        top.plan.qual = qq
        return top
    try:
        want = check_top(eng, p, [rows], plan, q, interconnect=ic, rescan=False)
        assert 0 < len(want) < 5
    finally:
        if ic:
            ic.close()
        rows.free(); rel.free()


def test_plain_agg_with_having_gives_zero_or_one_row(eng):
    vals, nulls = make_data(3000, 1, seed=71)
    rel, rows = load_rows(eng, vals, nulls)
    p = ExprPool()
    desc = capi.rows_tupdesc(TYPES)
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [], [(capi.AGG_COUNT_STAR, -1), (capi.AGG_MIN_INT4, p.var(5, capi.INT4OID)),
                                                   (capi.AGG_MAX_INT4, p.var(5, capi.INT4OID))])
    never = p.func(capi.F_INT4LT, capi.BOOLOID, p.var(1, capi.INT4OID), p.const(capi.INT4OID, -100))
    mn, mx, cnt = p.var(2, capi.INT4OID), p.var(3, capi.INT4OID), p.var(1, capi.INT8OID)
    cases = [(-1, p.func(capi.F_INT4LT, capi.BOOLOID, mn, mx), 1), (-1, p.func(capi.F_INT4EQ, capi.BOOLOID, mn, mx), 0),
             (never, p.func(capi.F_INT8EQ, capi.BOOLOID, cnt, p.const(capi.INT8OID, 0)), 1),       # the count = 0 row over no input
             (never, p.boolop(capi.E_ISNOTNULL, mn), 0)]
    try:
        for scanq, q, n in cases:
            b = ex.PlanBuilder()
            x = ex.Executor(eng, p.pool, [rows], b.agg(b.seqscan(0, desc, qual=scanq), agg, having=q))
            try:
                got, _ = agg_rows_py(x)
                assert len(got) == n, (scanq, q)
                if n and scanq != -1:
                    assert got == [(0, None, None)]
            finally:
                x.end()
    finally:
        rows.free(); rel.free()


def _join_case(eng, having_side, use_having):
    """HashJoin[targets](outer, Hash(inner)) with an Agg over rows on one side, against a Python join of the Agg's rows"""
    vals, nulls = make_data(30000, 800, seed=81)
    rel, rows = load_rows(eng, vals, nulls)
    p = ExprPool()
    desc = capi.rows_tupdesc(TYPES)
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [p.var(3, capi.INT8OID)], [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_INT4, p.var(5, capi.INT4OID))])
    q = p.func(capi.F_INT8GT, capi.BOOLOID, p.var(2, capi.INT8OID), p.const(capi.INT8OID, 37)) if use_having else -1
    hj = capi.gg_hashjoin()
    hj.jointype, hj.nkeys, hj.joinqual = capi.JOIN_INNER, 1, -1
    side_rows = 0 if having_side == "outer" else 1
    # the base side projects (k3, g); the Agg side is (k3, count, sum)
    k_agg, k_base = p.var(1, capi.INT8OID, varno=side_rows), p.var(3, capi.INT8OID, varno=1 - side_rows)
    hj.outerkey[0], hj.innerkey[0] = (k_agg, k_base) if side_rows == 0 else (k_base, k_agg)
    targets = [p.var(1, capi.INT8OID, varno=side_rows), p.var(2, capi.INT8OID, varno=side_rows), p.var(7, capi.INT8OID, varno=1 - side_rows)]
    try:
        b = ex.PlanBuilder()
        x = ex.Executor(eng, p.pool, [rows], b.agg(b.seqscan(0, desc), agg))
        aggrows, types = agg_rows_py(x)
        x.end()
        if use_having:
            ok = oracle_passes(types, aggrows, p, q)
            aggrows = [r for r, k in zip(aggrows, ok) if k]
        cnt = {r[0]: r[1] for r in aggrows if r[0] is not None}
        want = Counter((int(vals[i, 2]), cnt[int(vals[i, 2])], int(vals[i, 6])) for i in range(len(vals)) if int(vals[i, 2]) in cnt)
        b = ex.PlanBuilder()
        a = b.agg(b.seqscan(0, desc), agg, having=q)
        base = b.seqscan(0, desc)
        top = b.hashjoin(a, b.hash(base), hj, targets) if side_rows == 0 else b.hashjoin(base, b.hash(a), hj, targets)
        x = ex.Executor(eng, p.pool, [rows], top)
        try:
            got = Counter(tuple(int(v) for v in vals_) for vals_, nl, ty, ln in x.rows())
            assert got == want and len(want) > 100
            kinds = [k for k, _ in x.locations()]
            assert kinds[0] == "joinrows" and (side_rows == 1 or kinds[1] == "scanagg"), kinds
            x.rescan()
            assert Counter(tuple(int(v) for v in vals_) for vals_, nl, ty, ln in x.rows()) == want
        finally:
            x.end()
    finally:
        rows.free(); rel.free()


@pytest.mark.parametrize("side", ["outer", "inner"])
@pytest.mark.parametrize("use_having", [True, False])
def test_agg_as_an_input_of_a_hashjoin(eng, side, use_having):
    _join_case(eng, side, use_having)


# ---- goldens ----
def test_select_having_goldens(eng):
    from greengage_b200.engine import Relation
    g = json.load(open(os.path.join(HERE, "golden", "having_expected.json")))
    th = g["test_having"]
    types = [capi.INT4OID, capi.INT4OID, capi.BPCHAROID, capi.BPCHAROID]
    from test_join_tree_reference import rows_desc
    desc = rows_desc(types)
    pages = rows_pages(types, [[a, b, c.encode(), d.encode()] for a, b, c, d in th])
    rel = Relation(eng, host_pages=pages)
    p = ExprPool()
    a, bb, c = p.var(1, capi.INT4OID), p.var(2, capi.INT4OID), p.var(3, capi.BPCHAROID)
    I8, I4 = capi.INT8OID, capi.INT4OID
    q1 = (capi.make_agg(capi.AGGSTAGE_NORMAL, [bb, c], [(capi.AGG_COUNT_STAR, -1)]),
          p.func(capi.F_INT8EQ, capi.BOOLOID, p.var(3, I8), p.const(I8, 1)), 2)
    q2 = (capi.make_agg(capi.AGGSTAGE_NORMAL, [bb, c], []), p.func(capi.F_INT4EQ, capi.BOOLOID, p.var(1, I4), p.const(I4, 3)), 2)
    # SELECT c, max(a) ... HAVING count(*) > 2 OR min(a) = max(a): count and min are hidden aggregates the node above ignores
    q4 = (capi.make_agg(capi.AGGSTAGE_NORMAL, [c], [(capi.AGG_MAX_INT4, a), (capi.AGG_COUNT_STAR, -1), (capi.AGG_MIN_INT4, a)]),
          p.boolop(capi.E_OR, p.func(capi.F_INT8GT, capi.BOOLOID, p.var(3, I8), p.const(I8, 2)),
                   p.func(capi.F_INT4EQ, capi.BOOLOID, p.var(4, I4), p.var(2, I4))), 2)
    q5 = (capi.make_agg(capi.AGGSTAGE_NORMAL, [], [(capi.AGG_MIN_INT4, a), (capi.AGG_MAX_INT4, a)]),
          p.func(capi.F_INT4EQ, capi.BOOLOID, p.var(1, I4), p.var(2, I4)), 2)
    q6 = (q5[0], p.func(capi.F_INT4LT, capi.BOOLOID, p.var(1, I4), p.var(2, I4)), 2)
    try:
        for (agg, q, width), want in zip((q1, q2, q4, q5, q6), g["queries"]):
            b = ex.PlanBuilder()
            x = ex.Executor(eng, p.pool, [rel], b.agg(b.seqscan(0, desc), agg, having=q))
            try:
                got, _ = agg_rows_py(x)
                got = sorted(tuple(v.decode() if isinstance(v, bytes) else v for v in r[:width]) for r in got)
                assert got == sorted(tuple(r) for r in want["rows"]), want
            finally:
                x.end()
    finally:
        rel.free()


def _q18(eng, li_pages, od_pages, li_desc, od_desc, c_li_key, c_li_qty, c_od_key, c_od_cust, c_od_date, c_od_price, threshold=300.0):
    """Limit 100 <- Sort(totalprice DESC, orderdate) <- Agg(GROUP BY custkey, orderkey, orderdate, totalprice; sum(quantity))
         <- HashJoin(lineitem, Hash(HashJoin[targets](orders, Hash(Agg(GROUP BY l_orderkey; sum(l_quantity)) HAVING sum > 300))))"""
    from greengage_b200.engine import Relation
    rels = [Relation(eng, host_pages=li_pages), Relation(eng, host_pages=od_pages)]
    p = ExprPool()
    I8, F8 = capi.INT8OID, capi.FLOAT8OID
    lkey_t = li_desc.attrs[c_li_key - 1].atttypid
    okey_t = od_desc.attrs[c_od_key - 1].atttypid
    sub = capi.make_agg(capi.AGGSTAGE_NORMAL, [p.var(c_li_key, lkey_t)], [(capi.AGG_SUM_FLOAT8, p.var(c_li_qty, F8))])
    having = p.func(capi.F_FLOAT8GT, capi.BOOLOID, p.var(2, F8), p.const(F8, threshold))
    semi = capi.gg_hashjoin()                       # orders ⋈ the big orders: o_orderkey IN (...), as the planner's inner join
    semi.jointype, semi.nkeys, semi.joinqual = capi.JOIN_INNER, 1, -1
    semi.outerkey[0], semi.innerkey[0] = p.var(c_od_key, okey_t), p.var(1, lkey_t, varno=1)
    ctype, dtype_ = od_desc.attrs[c_od_cust - 1].atttypid, od_desc.attrs[c_od_date - 1].atttypid
    otargets = [p.var(c_od_key, okey_t), p.var(c_od_cust, ctype), p.var(c_od_date, dtype_), p.var(c_od_price, F8)]
    top = capi.gg_hashjoin()
    top.jointype, top.nkeys, top.joinqual = capi.JOIN_INNER, 1, -1
    top.outerkey[0], top.innerkey[0] = p.var(c_li_key, lkey_t), p.var(1, okey_t, varno=1)
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [p.var(2, ctype, varno=1), p.var(1, okey_t, varno=1), p.var(3, dtype_, varno=1), p.var(4, F8, varno=1)],
                        [(capi.AGG_SUM_FLOAT8, p.var(c_li_qty, F8))])
    keys = [capi.make_sortkey(3, F8, desc=True), capi.make_sortkey(2, dtype_)]
    b = ex.PlanBuilder()
    inner = b.hashjoin(b.seqscan(1, od_desc), b.hash(b.agg(b.seqscan(0, li_desc), sub, having=having)), semi, otargets)
    plan = b.limit(b.sort(b.agg(b.hashjoin(b.seqscan(0, li_desc), b.hash(inner), top), agg), keys), 100)
    x = ex.Executor(eng, p.pool, rels, plan)
    try:
        got = [(int(v[0]), int(v[1]), int(v[2]), f8(v[3]), f8(v[4])) for v, nl, ty, ln in x.rows()]
        kinds = x.locations()
    finally:
        x.end()
        for r in rels:
            r.free()
    return got, kinds


def test_q18_over_the_regression_tables(eng):
    from datetime import date
    g = json.load(open(os.path.join(HERE, "golden", "having_expected.json")))["q18"]
    li = np.load(os.path.join(HERE, "golden", "lineitem_q1.npz"))
    od = np.load(os.path.join(HERE, "golden", "orders_tpch.npz"))
    I4, I8, F8, D = capi.INT4OID, capi.INT8OID, capi.FLOAT8OID, capi.DATEOID
    from test_join_tree_reference import rows_desc
    lt, ot = [I8, F8], [I8, I4, D, F8]
    lpages = rows_pages(lt, [[int(k), float(q)] for k, q in zip(li["orderkey"], li["quantity"])])
    opages = rows_pages(ot, [[int(k), int(c), int(d), float(pr)] for k, c, d, pr in zip(od["orderkey"], od["custkey"], od["orderdate"], od["totalprice"])])
    got, kinds = _q18(eng, lpages, opages, rows_desc(lt), rows_desc(ot), 1, 2, 1, 2, 3, 4)
    epoch = date(2000, 1, 1).toordinal()
    want = [(c, o, date.fromisoformat(d).toordinal() - epoch, float(pr), float(s)) for c, o, d, pr, s in g]
    assert [(c, o, d, round(pr, 2), s) for c, o, d, pr, s in got] == want
    assert all(k in ("limit", "sort", "joinagg", "joinrows", "scanagg", "hash") for k, _ in kinds), kinds


def test_q18_shape_at_scale(eng):
    """the Q18 plan over synthetic LI-narrow ⋈ orders, against NumPy"""
    n, no = 600_000, 150_000
    rng = np.random.default_rng(18)
    lkey = rng.integers(1, no + 1, n).astype(np.int64)
    qty = rng.integers(1, 51, n).astype(np.float64)
    okey = np.arange(1, no + 1, dtype=np.int64)
    cust = rng.integers(1, 50_000, no).astype(np.int64)
    odate = rng.integers(0, 3000, no).astype(np.int64)
    price = rng.integers(100, 10**8, no).astype(np.float64) / 100
    I4, I8, F8, D = capi.INT4OID, capi.INT8OID, capi.FLOAT8OID, capi.DATEOID
    lt, ot = [I8, F8], [I8, I4, D, F8]
    lpages = po.build_pages(_heap(lt), [[int(k), float(q)] for k, q in zip(lkey, qty)])
    opages = po.build_pages(_heap(ot), [[int(k), int(c), int(d), float(pr)] for k, c, d, pr in zip(okey, cust, odate, price)])
    got, _ = _q18(eng, lpages, opages, _heap(lt), _heap(ot), 1, 2, 1, 2, 3, 4, threshold=150.0)
    s = np.bincount(lkey, weights=qty, minlength=no + 1)
    big = np.nonzero(s > 150.0)[0]
    assert len(big) > 100
    rows = [(int(cust[k - 1]), int(k), int(odate[k - 1]), float(price[k - 1]), float(s[k])) for k in big]
    rows.sort(key=lambda r: (-r[3], r[2]))
    assert got == rows[:100]


def _heap(types):
    from test_join_tree_reference import rows_desc
    return rows_desc(types)


def test_more_than_2_24_groups_with_a_selective_having(eng):
    n = (1 << 24) + 1_000_000
    rng = np.random.default_rng(24)
    key = rng.permutation(n).astype(np.int64) * 3 + 1
    price = rng.integers(1, 10**6, n).astype(np.float64) / 100
    vals = np.stack([key, price.view(np.int64)], axis=1)
    rel, rows = load_rows(eng, vals, np.zeros_like(vals, dtype=bool))
    p = ExprPool()
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [p.var(1, capi.INT8OID)], [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_FLOAT8, p.var(2, capi.FLOAT8OID))])
    q = p.func(capi.F_FLOAT8GT, capi.BOOLOID, p.var(3, capi.FLOAT8OID), p.const(capi.FLOAT8OID, 9999.0))
    desc = capi.rows_tupdesc([capi.INT8OID, capi.FLOAT8OID], notnull=[1, 1])
    b = ex.PlanBuilder()
    x = ex.Executor(eng, p.pool, [rows], b.agg(b.seqscan(0, desc), agg, having=q))
    try:
        got = sorted((int(v[0]), int(v[1]), f8(v[2])) for v, nl, ty, ln in x.rows())
        sel = price > 9999.0
        want = sorted(zip(key[sel].tolist(), [1] * int(sel.sum()), price[sel].tolist()))
        assert got == want and 0 < len(want) < 5000
    finally:
        x.end(); rows.free(); rel.free()
