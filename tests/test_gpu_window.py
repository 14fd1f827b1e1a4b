"""WindowAgg on the device (gg_window_* and the executor's WindowAgg node) against the row-at-a-time reference (tests/window_ref.c).

Kernels: every function over every supported frame and key type (int4, int8, date, bool, float8 with -0 / NaN, packed strings;
NULLs), dead slots, partitions at the tile bounds, one partition over more than 2^24 rows; integer results exact; float8 sums and
averages bit-identical across runs and within the exact-sum bound; overflow; the ntile / nth_value errors.  Node surface: over
scan rows, join rows and an Agg's rows, with a top-N qual, under a Limit and a Sort, stacked, after ReScan."""
import numpy as np
import pytest

from _window import FRAMES, all_funcs, random_rows, ref_window
from greengage_b200 import capi, executor as ex
from greengage_b200.capi import ExprPool

pytestmark = pytest.mark.gpu
DEAD = np.uint64(1 << 63)


@pytest.fixture(scope="module")
def eng():
    from greengage_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def load_words(eng, rows):
    """datum-row words uint64 [n][W] resident on the device: (owning Relation, RowRelation)"""
    from greengage_b200.engine import Relation, RowRelation
    n, W = rows.shape
    nb = max(1, (n * W * 8 + 16 + capi.GG_BLCKSZ - 1) // capi.GG_BLCKSZ)
    buf = np.zeros(nb * capi.GG_BLCKSZ // 8, dtype=np.uint64)
    buf[:n * W] = rows.reshape(-1)
    rel = Relation(eng, nblocks=nb)
    rel.load(0, buf.view(np.uint8))
    return rel, RowRelation(eng, rel.device_ptr(), n, W - 1)


def device_window(eng, rows, types, win, pool):
    from greengage_b200.engine import Window
    rel, rr = load_words(eng, rows)
    w = Window(eng, capi.rows_tupdesc(types), win, pool)
    try:
        return w.run(rr)
    finally:
        w.free()
        rr.free()
        rel.free()


def check(eng, rows, types, win, pool):
    rc, want, msg = ref_window(win, types, pool, rows)
    assert rc == 0, msg
    got = device_window(eng, rows, types, win, pool)
    assert got.shape == want.shape
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert len(bad) == 0, (len(bad), got[bad[:3]], want[bad[:3]])
    return got


KEYS = {"int4": [capi.INT4OID], "int8_float8": [capi.INT8OID, capi.FLOAT8OID], "date": [capi.DATEOID],
        "bool_text": [capi.BOOLOID, capi.TEXTOID], "float8": [capi.FLOAT8OID]}


@pytest.mark.parametrize("frame", sorted(FRAMES))
@pytest.mark.parametrize("keys", sorted(KEYS))
def test_kernels_equal_the_reference(eng, frame, keys):
    """the value columns hold multiples of 1/8 below 2^10 in magnitude: every partial float8 sum is exact, so the device's sums
    and averages equal the reference's left-to-right ones bit for bit"""
    rng = np.random.default_rng(sorted(FRAMES).index(frame) * 10 + sorted(KEYS).index(keys))
    ktypes = KEYS[keys]
    rows, types = random_rows(rng, 3000, ktypes, [capi.FLOAT8OID, capi.INT4OID, capi.INT8OID], dead=0.05)
    ncols = len(types)
    kcols = list(range(len(ktypes)))
    for part, order in ((kcols[:1], kcols[1:]), ([], kcols), (kcols, [])):
        for g in range(3):
            pool = ExprPool()
            funcs = all_funcs(pool, ncols, types, kcols, list(range(len(ktypes), ncols)))[g]
            check(eng, rows, types, capi.make_window(part, order, FRAMES[frame], funcs), pool.pool)


def sorted_rows(rng, sizes, peer_every=3, dead=0.0):
    """partitions of the given sizes (key column 0 = partition number, column 1 = an order key with ties), a float8 value of
    multiples of 1/8 and an int4 value, both with NULLs"""
    n = int(sum(sizes))
    rows = np.zeros((n, 5), dtype=np.uint64)
    rows[:, 1] = np.repeat(np.arange(len(sizes), dtype=np.int64), sizes).view(np.uint64)
    rows[:, 2] = (np.concatenate([np.arange(s) for s in sizes]) // peer_every).astype(np.int64).view(np.uint64) if n else 0
    rows[:, 3] = (rng.integers(-1000, 1000, n) / 8.0).view(np.uint64)
    rows[:, 4] = rng.integers(-2 ** 31, 2 ** 31, n).astype(np.int64).view(np.uint64)
    nl = rng.random((n, 2)) < 0.1
    rows[:, 3] = np.where(nl[:, 0], np.uint64(0), rows[:, 3])
    rows[:, 4] = np.where(nl[:, 1], np.uint64(0), rows[:, 4])
    rows[:, 0] = (nl[:, 0].astype(np.uint64) << np.uint64(2)) | (nl[:, 1].astype(np.uint64) << np.uint64(3))
    if dead:
        rows[rng.random(n) < dead, 0] |= DEAD
    return rows, [capi.INT8OID, capi.INT8OID, capi.FLOAT8OID, capi.INT4OID]


def scan_funcs(pool, cheap=False):
    x, i = pool.var(3, capi.FLOAT8OID), pool.var(4, capi.INT4OID)
    f = [(capi.WF_ROW_NUMBER, capi.INT8OID, []), (capi.WF_RANK, capi.INT8OID, []), (capi.WF_DENSE_RANK, capi.INT8OID, []),
         (capi.AGG_SUM_FLOAT8, capi.FLOAT8OID, [x]), (capi.AGG_SUM_INT4, capi.INT8OID, [i]), (capi.AGG_COUNT_ANY, capi.INT8OID, [x]),
         (capi.AGG_MAX_FLOAT8, capi.FLOAT8OID, [x]), (capi.WF_LAG, capi.INT4OID, [i])]
    return f[:6] if cheap else f


@pytest.mark.parametrize("frame", ["range_up_cr", "rows_cr_uf", "range_cr_cr", "rows_up_uf"])
def test_partitions_at_the_tile_bounds(eng, frame):
    rng = np.random.default_rng(3)
    sizes = [1, 2047, 2048, 2049, 1, 4095, 4096, 4097, 1, 1, 3, 6143, 6145]
    rows, types = sorted_rows(rng, sizes, dead=0.02)
    pool = ExprPool()
    check(eng, rows, types, capi.make_window([0], [1], FRAMES[frame], scan_funcs(pool)), pool.pool)


def test_one_partition_above_2_24_rows(eng):
    """one partition of 1.72 * 10^7 slots (more than 2^24 rows) in one ordered scan across every tile; dead slots included"""
    rng = np.random.default_rng(4)
    rows, types = sorted_rows(rng, [17_200_000], peer_every=5, dead=0.01)
    pool = ExprPool()
    for frame in ("range_up_cr", "rows_up_cr"):
        check(eng, rows, types, capi.make_window([0], [1], FRAMES[frame], scan_funcs(pool, cheap=True)), pool.pool)


def test_float8_sums_are_deterministic_and_within_the_exact_bound(eng):
    """arbitrary magnitudes: the sums are bit-identical run to run, and each is within gamma(k-1) * sum|x| of the exact sum, as the
    reference's left-to-right sum is"""
    import math
    from fractions import Fraction
    rng = np.random.default_rng(8)
    sizes = [5000, 1, 3, 20000, 777]
    rows, types = sorted_rows(rng, sizes)
    x = rng.standard_normal(len(rows)) * 10.0 ** rng.integers(-20, 20, len(rows))
    rows[:, 3] = x.view(np.uint64)
    rows[:, 0] &= ~np.uint64(4)
    pool = ExprPool()
    xv = pool.var(3, capi.FLOAT8OID)
    for frame in ("range_up_cr", "rows_cr_uf", "range_up_uf"):
        win = capi.make_window([0], [1], FRAMES[frame], [(capi.AGG_SUM_FLOAT8, capi.FLOAT8OID, [xv]), (capi.AGG_AVG_FLOAT8, capi.FLOAT8OID, [xv])])
        a = device_window(eng, rows, types, win, pool.pool)
        b = device_window(eng, rows, types, win, pool.pool)
        assert np.array_equal(a, b)
        from _window import bounds
        ps, pe, gs, ge = bounds(win, types, rows)
        eps = 2.0 ** -53
        for j in list(rng.integers(0, len(rows), 300)) + [0, len(rows) - 1]:
            rowsmode = FRAMES[frame] & capi.FRAMEOPTION_ROWS
            head = ps[j] if FRAMES[frame] & capi.FRAMEOPTION_START_UNBOUNDED_PRECEDING else (j if rowsmode else gs[j])
            tail = pe[j] - 1 if FRAMES[frame] & capi.FRAMEOPTION_END_UNBOUNDED_FOLLOWING else (j if rowsmode else ge[j] - 1)
            vals = x[head:tail + 1]
            k = len(vals)
            exact = sum(Fraction(float(v)) for v in vals)
            bound = (k - 1) * eps / (1 - (k - 1) * eps) * float(np.abs(vals).sum()) if k > 1 else 0.0
            s = a[j, 5].view(np.float64)
            assert abs(Fraction(float(s)) - exact) <= Fraction(bound) * (1 + 1e-12), (frame, j, k, s, float(exact))
            avg = a[j, 6].view(np.float64)
            assert math.isclose(avg, float(s) / k, rel_tol=4 * eps) or (avg == 0 and s == 0)


def test_overflow_and_argument_errors(eng):
    from greengage_b200.engine import Window
    rows = np.zeros((6, 3), dtype=np.uint64)
    rows[:, 2] = np.array([1e308, 1e308, -1.0, 2.0, 3.0, np.inf]).view(np.uint64)
    types = [capi.INT4OID, capi.FLOAT8OID]
    pool = ExprPool()
    x = pool.var(2, capi.FLOAT8OID)
    for frame in ("range_up_cr", "rows_cr_cr"):
        win = capi.make_window([], [], FRAMES[frame], [(capi.AGG_SUM_FLOAT8, capi.FLOAT8OID, [x])])
        if frame == "range_up_cr":
            with pytest.raises(capi.GGError, match="overflow"):
                device_window(eng, rows[:5], types, win, pool.pool)
            got = device_window(eng, rows, types, win, pool.pool)     # an infinite input: +inf, as float8pl gives it
            assert np.isinf(got[:, 3].view(np.float64)).all()
        else:
            device_window(eng, rows[:5], types, win, pool.pool)      # every row its own frame: no sum overflows
    for fn, args, ty in ((capi.WF_NTILE, [pool.const(capi.INT4OID, 0)], capi.INT4OID),
                         (capi.WF_NTH_VALUE, [x, pool.const(capi.INT4OID, 0)], capi.FLOAT8OID)):
        win = capi.make_window([0], [], capi.FRAMEOPTION_DEFAULTS, [(fn, ty, args)])
        with pytest.raises(capi.GGError, match="must be greater than zero") as e:
            device_window(eng, rows, types, win, pool.pool)
        assert e.value.args[0].startswith("ggb200 error %d" % capi.ERR_WINDOW_ARG)
        assert device_window(eng, rows[:0], types, win, pool.pool).shape == (0, 4)
        dead = rows.copy()
        dead[:, 0] |= DEAD
        assert device_window(eng, dead, types, win, pool.pool).shape == (0, 4)
    # refusals at create
    desc = capi.rows_tupdesc(types)
    value_offset = capi.FRAMEOPTION_NONDEFAULT | capi.FRAMEOPTION_ROWS | capi.FRAMEOPTION_BETWEEN | capi.FRAMEOPTION_START_VALUE_PRECEDING | capi.FRAMEOPTION_END_CURRENT_ROW
    cases = [capi.make_window([], [], value_offset, [(capi.WF_ROW_NUMBER, capi.INT8OID, [])]),
             capi.make_window([], [], capi.FRAMEOPTION_DEFAULTS, [(capi.AGG_SUM_NUMERIC, capi.NUMERICOID, [x])]),
             capi.make_window([], [], capi.FRAMEOPTION_DEFAULTS, [(capi.WF_LAG, capi.FLOAT8OID, [pool.func(capi.F_FLOAT8PL, capi.FLOAT8OID, x, x)])]),
             capi.make_window([], [], capi.FRAMEOPTION_DEFAULTS, [(capi.WF_NTILE, capi.INT4OID, [pool.var(1, capi.INT4OID)])])]
    for win in cases:
        with pytest.raises(capi.GGError) as e:
            Window(eng, desc, win, pool.pool)
        assert e.value.args[0].startswith("ggb200 error -6"), e.value.args[0]


# ---- the node surface ----

@pytest.fixture(scope="module")
def li(eng):
    from greengage_b200 import tpch
    from greengage_b200.engine import Relation
    pages, nb, nr = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, 200_000, seed=3, norders=40_000))
    rel = Relation(eng, host_pages=pages)
    yield rel, capi.synth_tupdesc(capi.TAB_LINEITEM_NARROW)
    rel.free()


def _scan(b, pool, desc):
    from greengage_b200 import tpch
    c = tpch.LI_NARROW_COLS
    names = ["orderkey", "extendedprice", "quantity", "shipdate"]
    targets = [pool.var(c[k], desc.attrs[c[k] - 1].atttypid) for k in names]
    types = [desc.attrs[c[k] - 1].atttypid for k in names]
    return b.seqscan(0, desc, -1, targets), types


def _rows(x):
    return [tuple(v if not nl else None for v, nl in zip(vals, nulls)) for vals, nulls, ty, ln in x.rows()]


def _words(rows, ncols):
    out = np.zeros((len(rows), 1 + ncols), dtype=np.uint64)
    for r, t in enumerate(rows):
        for c, v in enumerate(t):
            if v is None:
                out[r, 0] |= np.uint64(1 << c)
            else:
                out[r, 1 + c] = np.uint64(v & 0xFFFFFFFFFFFFFFFF)
    return out


def _as_tuples(words, ncols):
    return [tuple(None if (int(r[0]) >> c) & 1 else int(np.uint64(r[1 + c]).view(np.int64)) for c in range(ncols)) for r in words]


def _f(v):
    return float(np.array([v], dtype=np.int64).view(np.float64)[0])


def assert_rows(got, want, fcols):
    """the same rows in the same order: float8 columns fcols within 1e-12 relative (the device sums in its own fixed order, and an
    Agg's float8 sums below may differ in the last bits run to run), every other column exact"""
    assert len(got) == len(want)
    for j, (g, w) in enumerate(zip(got, want)):
        for c, (a, b) in enumerate(zip(g, w)):
            if c in fcols and a is not None and b is not None:
                assert abs(_f(a) - _f(b)) <= 1e-12 * abs(_f(b)), (j, c, _f(a), _f(b))
            else:
                assert a == b, (j, c, a, b)


def _win_funcs(pool, types):
    price = pool.var(2, types[1])
    return [(capi.WF_ROW_NUMBER, capi.INT8OID, []), (capi.AGG_SUM_FLOAT8, capi.FLOAT8OID, [price]), (capi.WF_RANK, capi.INT8OID, []),
            (capi.WF_LAG, types[1], [price])]


def test_node_over_scan_rows_with_qual_limit_sort_stack_and_rescan(eng, li):
    rel, desc = li
    pool = ExprPool()
    b = ex.PlanBuilder()
    scan, types = _scan(b, pool, desc)
    keys = [capi.make_sortkey(0, types[0]), capi.make_sortkey(1, types[1], desc=True)]
    part, order = [0], [1]
    funcs = _win_funcs(pool, types)
    frame = capi.FRAMEOPTION_DEFAULTS
    # the Sort's rows, windowed by the reference
    x = ex.Executor(eng, pool.pool, [rel], b.sort(scan, keys))
    sorted_rows = _rows(x)
    x.end()
    win = capi.make_window(part, order, frame, funcs)
    rc, want, msg = ref_window(win, types, pool.pool, _words(sorted_rows, 4))
    assert rc == 0, msg
    want = _as_tuples(want, 8)
    fc = (1, 2, 5, 7)
    x = ex.Executor(eng, pool.pool, [rel], b.windowagg(b.sort(scan, keys), part, order, frame, funcs))
    assert_rows(_rows(x), want, fc)
    ins = dict(x.instrumentation())
    assert x.kind() == "windowagg" and ins["windowagg"].ntuples == len(want) and ins["windowagg"].kernel_ms > 0
    x.rescan()
    assert_rows(_rows(x), want, fc)
    assert dict(x.instrumentation())["windowagg"].nloops == 2
    x.end()
    # top-1 per order: WHERE rn = 1 folded into the node's qual
    rn = pool.var(5, capi.INT8OID)
    qual = pool.func(capi.F_INT8EQ, capi.BOOLOID, rn, pool.const(capi.INT8OID, 1))
    x = ex.Executor(eng, pool.pool, [rel], b.windowagg(b.sort(scan, keys), part, order, frame, funcs, qual=qual))
    top1 = [r for r in want if r[4] == 1]
    assert_rows(_rows(x), top1, fc)
    assert dict(x.instrumentation())["windowagg"].ntuples == len(top1)
    x.end()
    # under a Limit: only its window comes back
    x = ex.Executor(eng, pool.pool, [rel], b.limit(b.windowagg(b.sort(scan, keys), part, order, frame, funcs), 25, 10))
    assert_rows(_rows(x), want[10:35], fc)
    x.end()
    # under a Sort (ORDER BY the window sum DESC, orderkey, row_number)
    k2 = [capi.make_sortkey(5, capi.FLOAT8OID, desc=True), capi.make_sortkey(0, types[0]), capi.make_sortkey(4, capi.INT8OID)]
    x = ex.Executor(eng, pool.pool, [rel], b.sort(b.windowagg(b.sort(scan, keys), part, order, frame, funcs), k2))
    got = _rows(x)
    x.end()
    by_key = lambda r: (r[0], r[4])                                             # noqa: E731 (orderkey, row_number)
    assert_rows(sorted(got, key=by_key), sorted(want, key=by_key), fc)
    assert all(_f(got[i][5]) >= _f(got[i + 1][5]) for i in range(len(got) - 1))
    # stacked: a second WindowAgg through a Sort on a column the first one produced
    funcs2 = [(capi.AGG_COUNT_STAR, capi.INT8OID, []), (capi.WF_DENSE_RANK, capi.INT8OID, [])]
    k3 = [capi.make_sortkey(4, capi.INT8OID), capi.make_sortkey(3, types[3])]
    inner = b.windowagg(b.sort(scan, keys), part, order, frame, funcs)
    x = ex.Executor(eng, pool.pool, [rel], b.sort(inner, k3))
    mid = _rows(x)
    x.end()
    win2 = capi.make_window([4], [3], frame, funcs2)
    rc, want2, msg = ref_window(win2, types + [capi.INT8OID, capi.FLOAT8OID, capi.INT8OID, types[1]], pool.pool, _words(mid, 8))
    assert rc == 0, msg
    x = ex.Executor(eng, pool.pool, [rel], b.windowagg(b.sort(inner, k3), [4], [3], frame, funcs2))
    assert_rows(_rows(x), _as_tuples(want2, 10), fc)
    x.end()
    # the order below is checked: a Sort on other columns is refused
    with pytest.raises(ex.ExecError) as e:
        ex.Executor(eng, pool.pool, [rel], b.windowagg(b.sort(scan, [capi.make_sortkey(1, types[1])]), part, order, frame, funcs))
    assert e.value.args[0].startswith("ggb200 error -6")


def test_node_over_agg_rows_and_join_rows(eng, li):
    from greengage_b200 import tpch
    from greengage_b200.engine import Relation
    rel, desc = li
    c = tpch.LI_NARROW_COLS
    # over an Agg's rows: rank() OVER (ORDER BY count(*) DESC) of GROUP BY orderkey (the float8 sums below may differ in the last
    # bits run to run, so they order nothing here)
    pool = ExprPool()
    okey = pool.var(c["orderkey"], desc.attrs[c["orderkey"] - 1].atttypid)
    price = pool.var(c["extendedprice"], capi.FLOAT8OID)
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [okey], [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_FLOAT8, price)], num_groups=40_000)
    b = ex.PlanBuilder()
    a = b.agg(b.seqscan(0, desc, -1), agg)
    keys = [capi.make_sortkey(1, capi.INT8OID, desc=True), capi.make_sortkey(0, desc.attrs[c["orderkey"] - 1].atttypid)]
    x = ex.Executor(eng, pool.pool, [rel], b.sort(a, keys))
    srows = _rows(x)
    x.end()
    types = [desc.attrs[c["orderkey"] - 1].atttypid, capi.INT8OID, capi.FLOAT8OID]
    funcs = [(capi.WF_RANK, capi.INT8OID, []), (capi.WF_NTILE, capi.INT4OID, [pool.const(capi.INT4OID, 10)]),
             (capi.AGG_COUNT_ANY, capi.INT8OID, [pool.var(3, capi.FLOAT8OID)])]
    win = capi.make_window([], [1], capi.FRAMEOPTION_DEFAULTS, funcs)
    rc, want, msg = ref_window(win, types, pool.pool, _words(srows, 3))
    assert rc == 0, msg
    x = ex.Executor(eng, pool.pool, [rel], b.windowagg(b.sort(a, keys), [], [1], capi.FRAMEOPTION_DEFAULTS, funcs))
    assert_rows(_rows(x), _as_tuples(want, 6), (2,))
    x.end()
    # over join rows: lineitem ⋈ orders, lag(price) OVER (PARTITION BY custkey ORDER BY orderkey)
    od, _, _ = tpch.synth_generate(tpch.synth_spec(capi.TAB_ORDERS, 40_000, seed=3))
    orel = Relation(eng, host_pages=od)
    try:
        odesc = capi.synth_tupdesc(capi.TAB_ORDERS)
        oc = tpch.ORDERS_COLS
        jpool = ExprPool()
        hj = capi.make_hashjoin(capi.JOIN_INNER, [jpool.var(c["orderkey"], capi.INT8OID, varno=0)], [jpool.var(oc["orderkey"], capi.INT8OID, varno=1)])
        t_cust = jpool.var(oc["custkey"], capi.INT4OID, varno=1)
        t_okey = jpool.var(c["orderkey"], capi.INT8OID, varno=0)
        t_price = jpool.var(c["extendedprice"], capi.FLOAT8OID, varno=0)
        b = ex.PlanBuilder()
        j = b.hashjoin(b.seqscan(0, desc, -1), b.hash(b.seqscan(1, odesc, -1)), hj, [t_cust, t_okey, t_price])
        jtypes = [capi.INT4OID, capi.INT8OID, capi.FLOAT8OID]
        keys = [capi.make_sortkey(0, jtypes[0]), capi.make_sortkey(1, jtypes[1]), capi.make_sortkey(2, capi.FLOAT8OID)]
        x = ex.Executor(eng, jpool.pool, [rel, orel], b.sort(j, keys))
        srows = _rows(x)
        x.end()
        assert len(srows) > 1000
        funcs = [(capi.WF_LAG, capi.FLOAT8OID, [jpool.var(3, capi.FLOAT8OID)]), (capi.WF_ROW_NUMBER, capi.INT8OID, [])]
        win = capi.make_window([0], [1], capi.FRAMEOPTION_DEFAULTS, funcs)
        rc, want, msg = ref_window(win, jtypes, jpool.pool, _words(srows, 3))
        assert rc == 0, msg
        x = ex.Executor(eng, jpool.pool, [rel, orel], b.windowagg(b.sort(j, keys), [0], [1], capi.FRAMEOPTION_DEFAULTS, funcs))
        assert_rows(_rows(x), _as_tuples(want, 5), (2, 3))
        x.end()
    finally:
        orel.free()


def test_window_out_goldens(eng):
    """the reference's window.out rows for the tenk1 and VALUES queries the device runs, as multisets of the printed tuples"""
    from collections import Counter
    from _window import golden_cases, printed
    n = 0
    for gid, win, types, pool, rows, items, want in golden_cases():
        out = device_window(eng, rows, types, win, pool.pool)
        assert Counter(map(tuple, printed(win, out, len(types), items))) == Counter(map(tuple, want)), gid
        n += 1
    assert n == 19
