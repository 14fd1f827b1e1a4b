"""A HashJoin with a target list on the GPU (gg_joinrows_create / gg_joinagg_rows and the executor's "joinrows" node): the rows
it returns, as a multiset, against the reference's golden join tables and against the oracle's join pairs; the one re-probe of
an output that overflows; batched (hybrid) joins; a three-table TPC-H Q3-shaped plan through the node surface; Sort, Limit,
ReScan, squelch and a Gather Motion over join rows; and a device error inside a target expression."""
import struct
from collections import Counter

import numpy as np
import pytest

from _util import j1j2_fixture, j1j2_golden_rows, make_desc, J1J2_QUERIES
from greengage_b200 import capi, executor as ex, tpch
from oracle import pyoracle as po
from test_oracle_join import join_nodes, small_relations

pytestmark = pytest.mark.gpu

INT4 = (capi.INT4OID, 4, "i", 1)
JOINTYPES = [capi.JOIN_INNER, capi.JOIN_LEFT, capi.JOIN_RIGHT, capi.JOIN_FULL, capi.JOIN_SEMI, capi.JOIN_ANTI, capi.JOIN_LASJ_NOTIN]
BOTH_SIDES = (capi.JOIN_INNER, capi.JOIN_LEFT, capi.JOIN_RIGHT, capi.JOIN_FULL)
STRINGS = (capi.BPCHAROID, capi.VARCHAROID, capi.TEXTOID)


@pytest.fixture(scope="module")
def eng():
    from greengage_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def datum(v, isnull, typid):
    """one Datum word of a row, as a Python value"""
    if isnull:
        return None
    v = int(v) & 0xFFFFFFFFFFFFFFFF
    if typid in (capi.INT4OID, capi.DATEOID):
        v &= 0xFFFFFFFF
        return v - (1 << 32) if v >> 31 else v
    if typid == capi.FLOAT8OID:
        return struct.unpack("<d", struct.pack("<Q", v))[0]
    if typid in STRINGS:
        return v.to_bytes(8, "little").rstrip(b"\0")
    return v - (1 << 64) if v >> 63 else v


def slot_rows(rows):
    return [tuple(datum(v, n, t) for v, n, t in zip(vals, nl, ty)) for vals, nl, ty, ln in rows]


def device_rows(jr, typids):
    vals, nulls, live = jr.rows()
    assert vals.shape[0] == live
    return [tuple(datum(v, n, t) for v, n, t in zip(vals[r], nulls[r], typids)) for r in range(vals.shape[0])]


def run_joinrows(eng, outer, inner, hj, targets, pool, opages, ipages, work_mem=0):
    from greengage_b200.engine import JoinRows, Relation
    jr = JoinRows(eng, outer, inner, hj, targets, pool)
    orel, irel = Relation(eng, host_pages=opages), Relation(eng, host_pages=ipages)
    try:
        jr.set_work_mem(work_mem)
        nbatch = jr.run(irel, orel)
        return device_rows(jr, [pool.nodes[t].rettype for t in targets]), nbatch
    finally:
        jr.free()
        orel.free()
        irel.free()


# ---- 1. the reference's golden join tables, rows and all ----
@pytest.mark.parametrize("name", sorted(J1J2_QUERIES))
def test_reference_join_goldens_as_rows(eng, name):
    from greengage_b200.engine import Relation
    d1, p1, d2, p2, g = j1j2_fixture()
    jt, inner_att = J1J2_QUERIES[name]
    p = capi.ExprPool()
    hj = capi.make_hashjoin(jt, [p.var(1, capi.INT4OID, 0)], [p.var(inner_att, capi.INT4OID, 1)], -1)
    targets = [p.var(1, capi.INT4OID, 0), p.var(2, capi.INT4OID, 0), p.var(3, capi.TEXTOID, 0), p.var(1, capi.INT4OID, 1),
               p.var(2, capi.INT4OID, 1)]
    b = ex.PlanBuilder()
    plan = b.hashjoin(b.seqscan(0, d1), b.hash(b.seqscan(1, d2)), hj, targets)
    r1, r2 = Relation(eng, host_pages=p1), Relation(eng, host_pages=p2)
    x = ex.Executor(eng, p.pool, [r1, r2], plan)
    try:
        assert x.kind() == "joinrows"
        got = slot_rows(x.rows())
        assert x.locations() == [("joinrows", "host")]
    finally:
        x.end()
        r1.free()
        r2.free()
    got = [(i1, j, None if t is None else t.decode(), i2, k) for i1, j, t, i2, k in got]
    if name == "inner_i_eq_k":
        have = Counter(got)
    else:                                        # JOIN ... USING (i): i = coalesce(J1.i, J2.i)
        have = Counter((i1 if i1 is not None else i2, j, t, k) for i1, j, t, i2, k in got)
    assert have == Counter(j1j2_golden_rows(g, name)), name


# ---- 2. every join type against the oracle's pairs ----
def _pair_rows(pairs, orows, onulls, irows, inulls, ocols, icols):
    def col(rows, nulls, i, c):
        if i < 0 or nulls[i][c]:
            return None
        v = rows[i][c]
        return v.rstrip(b" ") if isinstance(v, bytes) else v
    out = []
    for a, b_ in pairs:
        oi = ((int(a) & 0xFFFF) - 1) if a >= 0 else -1           # one page per relation: offnum - 1 = row index
        ii = ((int(b_) & 0xFFFF) - 1) if b_ >= 0 else -1
        out.append(tuple(col(orows, onulls, oi, c) for c in ocols) + tuple(col(irows, inulls, ii, c) for c in icols))
    return out


@pytest.mark.parametrize("jointype", JOINTYPES)
@pytest.mark.parametrize("nkeys", [1, 2])
@pytest.mark.parametrize("with_qual", [False, True])
def test_every_join_type_against_the_oracle_pairs(eng, jointype, nkeys, with_qual):
    odesc, idesc, orows, onulls, irows, inulls, opages, ipages = small_relations()
    p, outer, inner, hj = join_nodes(odesc, idesc, jointype, nkeys, with_qual)
    targets = [p.var(1, capi.INT4OID, 0), p.var(2, capi.BPCHAROID, 0), p.var(3, capi.FLOAT8OID, 0)]
    icols = []
    if jointype in BOTH_SIDES:
        targets += [p.var(1, capi.INT4OID, 1), p.var(3, capi.INT4OID, 1)]
        icols = [0, 2]
    got, _ = run_joinrows(eng, outer, inner, hj, targets, p.pool, opages, ipages)
    pairs = po.hashjoin_tids(outer, inner, hj, p.pool, opages, ipages)
    want = _pair_rows(pairs, orows, onulls, irows, inulls, [0, 1, 2], icols)
    assert Counter(got) == Counter(want)


# ---- 3. an output larger than the outer side: grown once, probed once more ----
def _many_to_many(nouter=2000, ninner=200, inner_keys=10):
    d = make_desc([INT4, INT4])
    orows = [[i % 10, i] for i in range(nouter)]
    irows = [[i % inner_keys, 100000 + i] for i in range(ninner)]
    return d, orows, irows, po.build_pages(d, orows), po.build_pages(d, irows)


@pytest.mark.parametrize("jointype", [capi.JOIN_INNER, capi.JOIN_FULL])
def test_output_overflow_is_probed_exactly_once_more(eng, jointype):
    from greengage_b200.engine import JoinRows, Relation
    d, orows, irows, opages, ipages = _many_to_many(inner_keys=12)
    p = capi.ExprPool()
    hj = capi.make_hashjoin(jointype, [p.var(1, capi.INT4OID, 0)], [p.var(1, capi.INT4OID, 1)], -1)
    targets = [p.var(2, capi.INT4OID, 0), p.var(2, capi.INT4OID, 1)]
    want = [(o[1], i[1]) for o in orows for i in irows if o[0] == i[0]]
    if jointype == capi.JOIN_FULL:
        want += [(None, i[1]) for i in irows if i[0] >= 10]
    assert len(want) >= 10 * len(orows)
    jr = JoinRows(eng, capi.make_scan(d), capi.make_scan(d), hj, targets, p.pool)
    orel, irel = Relation(eng, host_pages=opages), Relation(eng, host_pages=ipages)
    try:
        jr.run(irel, orel)
        before = eng.launch_count()
        _, n, live = jr.rows_raw()
        reprobe = eng.launch_count() - before
        got = device_rows(jr, [capi.INT4OID, capi.INT4OID])
        assert live == len(want) and n >= live
        assert Counter(got) == Counter(want)
        if jointype == capi.JOIN_INNER:
            assert reprobe == 1                                    # the one probe launch of the replay, nothing else
        # a rescan into the grown buffer needs no second probe
        jr.reset()
        jr.probe(orel)
        before = eng.launch_count()
        jr.rows_raw()
        assert eng.launch_count() - before == (0 if jointype == capi.JOIN_INNER else 1)      # (the fill-inner pass of FULL)
        assert Counter(device_rows(jr, [capi.INT4OID, capi.INT4OID])) == Counter(want)
    finally:
        jr.free()
        orel.free()
        irel.free()


# ---- 4. hybrid hash join: the batches' rows are the one-table run's ----
@pytest.mark.parametrize("jointype,nkeys,with_qual", [(capi.JOIN_INNER, 2, False), (capi.JOIN_LEFT, 1, True), (capi.JOIN_RIGHT, 1, False),
                                                      (capi.JOIN_FULL, 1, True), (capi.JOIN_ANTI, 1, False)])
def test_hybrid_join_rows_equal_one_table(eng, jointype, nkeys, with_qual):
    odesc, idesc, orows, onulls, irows, inulls, opages, ipages = small_relations(seed=21, nouter=6000, ninner=2000)
    p, outer, inner, hj = join_nodes(odesc, idesc, jointype, nkeys, with_qual)
    targets = [p.var(1, capi.INT4OID, 0), p.var(3, capi.FLOAT8OID, 0)]
    if jointype in BOTH_SIDES:
        targets += [p.var(2, capi.BPCHAROID, 1), p.var(3, capi.INT4OID, 1)]
    one, nb1 = run_joinrows(eng, outer, inner, hj, targets, p.pool, opages, ipages)
    many, nb = run_joinrows(eng, outer, inner, hj, targets, p.pool, opages, ipages, work_mem=32768)
    assert nb1 == 1 and nb > 1
    assert len(one) > 0 and Counter(many) == Counter(one)


# ---- 5. TPC-H Q3 shape: customer ⋈ orders ⋈ lineitem through the node surface ----
D = tpch.D_1995_03_15


@pytest.fixture(scope="module")
def q3_data():
    oc, lc = tpch.ORDERS_COLS, tpch.LI_NARROW_COLS
    od, _, _ = tpch.synth_generate(tpch.synth_spec(capi.TAB_ORDERS, 20000, seed=3))
    li, _, _ = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, 80000, seed=4, norders=20000))
    odesc, ldesc = capi.synth_tupdesc(capi.TAB_ORDERS), capi.synth_tupdesc(capi.TAB_LINEITEM_NARROW)
    orders = [r for b in range(od.size // capi.GG_BLCKSZ) for r in po.deform_page(odesc, od, b)]
    lines = [r for b in range(li.size // capi.GG_BLCKSZ) for r in po.deform_page(ldesc, li, b)]
    custkeys = sorted({r[oc["custkey"] - 1] for r in orders})
    rng = np.random.default_rng(8)
    seg = {k: ["BUILDING", "MACHINE", "HOUSE"][int(rng.integers(0, 3))] for k in custkeys}
    cdesc = make_desc([INT4, (capi.BPCHAROID, -1, "i", 1)])
    cpages = po.build_pages(cdesc, [[k, seg[k].encode()] for k in custkeys])
    # the answer in NumPy terms: orders of BUILDING customers before D, their lineitems shipped after D
    okeys = {r[oc["orderkey"] - 1] for r in orders if r[oc["orderdate"] - 1] < D and seg[r[oc["custkey"] - 1]] == "BUILDING"}
    lk = np.array([r[lc["orderkey"] - 1] for r in lines], dtype=np.int64)
    price = np.array([r[lc["extendedprice"] - 1] for r in lines])
    disc = np.array([r[lc["discount"] - 1] for r in lines])
    ship = np.array([r[lc["shipdate"] - 1] for r in lines])
    m = (ship > D) & np.isin(lk, np.array(sorted(okeys), dtype=np.int64))
    rev = price[m] * (1.0 - disc[m])
    keys, inv = np.unique(lk[m], return_inverse=True)
    sums = np.zeros(keys.size)
    np.add.at(sums, inv, rev)
    counts = np.bincount(inv, minlength=keys.size)
    order = np.lexsort((keys, -sums))[:10]
    want = [(int(keys[i]), float(sums[i]), int(counts[i])) for i in order]
    assert len(want) == 10
    return od, li, cpages, odesc, ldesc, cdesc, want


def _q3_plan(rows_side, odesc, ldesc, cdesc):
    oc, lc = tpch.ORDERS_COLS, tpch.LI_NARROW_COLS
    p = capi.ExprPool()
    b = ex.PlanBuilder()
    # orders ⋈ customer: the rows (o_orderkey, o_orderdate) of BUILDING customers' orders before D
    oqual = p.func(capi.F_DATE_LT, capi.BOOLOID, p.var(oc["orderdate"], capi.DATEOID, 0), p.const(capi.DATEOID, D))
    cqual = p.func(capi.F_BPCHAREQ, capi.BOOLOID, p.var(2, capi.BPCHAROID, 1), p.const(capi.BPCHAROID, "BUILDING"))
    lower = b.hashjoin(b.seqscan(0, odesc, oqual), b.hash(b.seqscan(2, cdesc, cqual)),
                       capi.make_hashjoin(capi.JOIN_INNER, [p.var(oc["custkey"], capi.INT4OID, 0)], [p.var(1, capi.INT4OID, 1)]),
                       [p.var(oc["orderkey"], capi.INT8OID, 0), p.var(oc["orderdate"], capi.DATEOID, 0)])
    li_side, rows_varno = (0, 1) if rows_side == "inner" else (1, 0)
    lqual = p.func(capi.F_DATE_GT, capi.BOOLOID, p.var(lc["shipdate"], capi.DATEOID, li_side), p.const(capi.DATEOID, D))
    lscan = b.seqscan(1, ldesc, lqual)
    lkey, okey = p.var(lc["orderkey"], capi.INT8OID, li_side), p.var(1, capi.INT8OID, rows_varno)
    rev = p.func(capi.F_FLOAT8MUL, capi.FLOAT8OID, p.var(lc["extendedprice"], capi.FLOAT8OID, li_side),
                 p.func(capi.F_FLOAT8MI, capi.FLOAT8OID, p.const(capi.FLOAT8OID, 1.0), p.var(lc["discount"], capi.FLOAT8OID, li_side)))
    if rows_side == "inner":
        upper = b.hashjoin(lscan, b.hash(lower), capi.make_hashjoin(capi.JOIN_INNER, [lkey], [okey]))
    else:
        upper = b.hashjoin(lower, b.hash(lscan), capi.make_hashjoin(capi.JOIN_INNER, [okey], [lkey]))
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [okey if rows_side == "outer" else lkey],
                        [(capi.AGG_SUM_FLOAT8, rev), (capi.AGG_COUNT_STAR, -1)], num_groups=20000)
    top = b.limit(b.sort(b.agg(upper, agg), [capi.make_sortkey(1, capi.FLOAT8OID, desc=True), capi.make_sortkey(0, capi.INT8OID)]), 10)
    return p, top


@pytest.mark.parametrize("rows_side", ["inner", "outer"])
def test_q3_shape_three_tables(eng, q3_data, rows_side):
    from greengage_b200.engine import Relation
    od, li, cpages, odesc, ldesc, cdesc, want = q3_data
    p, top = _q3_plan(rows_side, odesc, ldesc, cdesc)
    rels = [Relation(eng, host_pages=od), Relation(eng, host_pages=li), Relation(eng, host_pages=cpages)]
    x = ex.Executor(eng, p.pool, rels, top)
    try:
        got = [(int(v[0]), struct.unpack("<d", struct.pack("<q", v[1]))[0], int(v[2])) for v, nl, ty, ln in x.rows()]
        L = ex.exec_lib()
        join = L.GgExecOuterPlanState(L.GgExecOuterPlanState(x.state))              # Limit -> Sort -> the Agg's join
        lower = L.GgExecInnerPlanState(join) if rows_side == "inner" else L.GgExecOuterPlanState(join)
        assert L.GgExecNodeKind(join).decode() == "joinagg" and L.GgExecNodeKind(lower).decode() == "joinrows"
        assert [g[0] for g in got] == [w[0] for w in want] and [g[2] for g in got] == [w[2] for w in want]
        for g, w in zip(got, want):
            assert abs(g[1] - w[1]) <= 1e-6 * abs(w[1]), (g, w)
    finally:
        x.end()
        for r in rels:
            r.free()


# ---- 6. Sort / Limit / ReScan / squelch / Gather Motion over join rows ----
@pytest.fixture(scope="module")
def left_join():
    odesc, idesc, orows, onulls, irows, inulls, opages, ipages = small_relations(seed=17, nouter=3000, ninner=900)
    p, outer, inner, hj = join_nodes(odesc, idesc, capi.JOIN_LEFT, 1, True)
    targets = [p.var(1, capi.INT4OID, 0), p.var(3, capi.FLOAT8OID, 0), p.var(3, capi.INT4OID, 1)]
    return odesc, idesc, opages, ipages, p, hj, targets


def _left_plan(b, lj):
    odesc, idesc, opages, ipages, p, hj, targets = lj
    return b.hashjoin(b.seqscan(0, odesc), b.hash(b.seqscan(1, idesc)), hj, targets)


def test_sort_and_limit_over_join_rows(eng, left_join):
    from greengage_b200.engine import Relation
    odesc, idesc, opages, ipages, p, hj, targets = left_join
    rels = [Relation(eng, host_pages=opages), Relation(eng, host_pages=ipages)]
    # NULLs in col 2; rows equal on all three keys are equal rows, so the order is one whatever order the probe wrote them in
    keys = [capi.make_sortkey(2, capi.INT4OID, desc=True), capi.make_sortkey(1, capi.FLOAT8OID), capi.make_sortkey(0, capi.INT4OID)]
    try:
        b = ex.PlanBuilder()
        x = ex.Executor(eng, p.pool, rels, b.sort(_left_plan(b, left_join), keys))
        full = x.rows()
        assert x.locations()[1][0] == "joinrows"
        x.end()
        assert len(full) > 1000
        for count in (1, 10, 333, len(full) + 5):
            b = ex.PlanBuilder()
            x = ex.Executor(eng, p.pool, rels, b.limit(b.sort(_left_plan(b, left_join), keys), count))
            assert x.rows() == full[:count], count                 # byte for byte the prefix of the full device sort
            x.end()
    finally:
        for r in rels:
            r.free()


def test_rescan_squelch_and_gather_over_join_rows(eng, left_join):
    from greengage_b200.engine import Relation
    odesc, idesc, opages, ipages, p, hj, targets = left_join
    rels = [Relation(eng, host_pages=opages), Relation(eng, host_pages=ipages)]
    try:
        b = ex.PlanBuilder()
        x = ex.Executor(eng, p.pool, rels, _left_plan(b, left_join))
        first = Counter(slot_rows(x.rows()))
        ins = dict(x.instrumentation())["joinrows"]
        assert ins.hash_batches == 1 and ins.ntuples == sum(first.values()) and ins.kernel_ms > 0
        x.rescan()                                                   # the table is kept; the outer side is probed again
        assert Counter(slot_rows(x.rows())) == first
        x.rescan()
        part = x.rows(limit=5)                                       # squelched after five rows
        assert len(part) == 5 and exec_slot_is_end(x)
        x.end()
        b = ex.PlanBuilder()
        x = ex.Executor(eng, p.pool, rels, b.motion(_left_plan(b, left_join), ex.MOTION_GATHER))
        assert Counter(slot_rows(x.rows())) == first and x.kind() == "motion"
        x.end()
    finally:
        for r in rels:
            r.free()


def exec_slot_is_end(x):
    return not ex.exec_lib().GgExecProcNode(x.state)


# ---- 7. a device error inside a target expression ----
def test_error_in_a_target_expression_surfaces_with_its_code(eng):
    from greengage_b200.engine import Relation
    odesc, idesc, orows, onulls, irows, inulls, opages, ipages = small_relations()
    p, outer, inner, hj = join_nodes(odesc, idesc, capi.JOIN_INNER, 1, False)
    bad = p.func(capi.F_FLOAT8DIV, capi.FLOAT8OID, p.var(3, capi.FLOAT8OID, 0), p.const(capi.FLOAT8OID, 0.0))
    b = ex.PlanBuilder()
    plan = b.hashjoin(b.seqscan(0, odesc), b.hash(b.seqscan(1, idesc)), hj, [p.var(1, capi.INT4OID, 0), bad])
    rels = [Relation(eng, host_pages=opages), Relation(eng, host_pages=ipages)]
    x = ex.Executor(eng, p.pool, rels, plan)
    try:
        with pytest.raises(ex.ExecError) as e:
            x.rows()
        assert e.value.code == -4 and "division by zero" in str(e.value)       # GG_ERR_DIV_ZERO
    finally:
        x.end()
        for r in rels:
            r.free()


# ---- windowed claims: outputs large enough that every warp claims rows a window at a time ----
@pytest.fixture(scope="module")
def fk_join():
    """LI-narrow (3·10^6 rows over 150 000 orders) and orders (200 000 rows: 50 000 of them with no lineitem), and the
    oracle's l_orderkey -> (count, sum(l_extendedprice))"""
    li, _, nli = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, 3_000_000, seed=5, norders=150_000))
    od, _, nod = tpch.synth_generate(tpch.synth_spec(capi.TAB_ORDERS, 200_000, seed=5))
    lc, oc = tpch.LI_NARROW_COLS, tpch.ORDERS_COLS
    p = capi.ExprPool()
    lkey, price = p.var(lc["orderkey"], capi.INT8OID, 0), p.var(lc["extendedprice"], capi.FLOAT8OID, 0)
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [lkey], [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_FLOAT8, price)])
    rows, scanned, _ = po.seqscan_agg(capi.make_scan(capi.synth_tupdesc(capi.TAB_LINEITEM_NARROW)), agg, p.pool, li, cap=200_000)
    assert scanned == nli == 3_000_000
    keys = np.array([r.key[0] for r in rows], dtype=np.int64)
    counts = np.array([r.agg[0].i for r in rows], dtype=np.int64)
    order = np.argsort(keys)
    hj = capi.make_hashjoin(capi.JOIN_INNER, [lkey], [p.var(oc["orderkey"], capi.INT8OID, 1)])
    targets = [lkey, p.var(oc["orderkey"], capi.INT8OID, 1), price]
    return li, od, nod, p, hj, targets, keys[order], counts[order], sum(r.agg[1].f[0] for r in rows)


@pytest.mark.parametrize("jointype,work_mem", [(capi.JOIN_INNER, 0), (capi.JOIN_INNER, 9 << 20), (capi.JOIN_RIGHT, 0)])
def test_windowed_claims_need_no_second_probe(eng, fk_join, jointype, work_mem):
    from greengage_b200.engine import JoinRows, Relation
    li, od, nod, p, hj, targets, keys, counts, price_sum = fk_join
    hj.jointype = jointype
    desc_li, desc_od = capi.synth_tupdesc(capi.TAB_LINEITEM_NARROW), capi.synth_tupdesc(capi.TAB_ORDERS)
    jr = JoinRows(eng, capi.make_scan(desc_li), capi.make_scan(desc_od), hj, targets, p.pool)
    orel, irel = Relation(eng, host_pages=li), Relation(eng, host_pages=od)
    try:
        jr.set_work_mem(work_mem)
        nbatch = jr.run(irel, orel)
        assert (nbatch > 1) == (work_mem > 0)
        before = eng.launch_count()
        _, nslots, live = jr.rows_raw()
        # no re-probe: nothing but the fill-inner pass of the right join is launched here
        assert eng.launch_count() - before == (1 if jointype == capi.JOIN_RIGHT and nbatch == 1 else 0)
        unmatched = nod - keys.size
        assert live == counts.sum() + (unmatched if jointype == capi.JOIN_RIGHT else 0)
        assert nslots > live                          # the tails of the warps' windows are there, marked dead
        vals, nulls, live2 = jr.rows()
        assert vals.shape[0] == live2 == live
        m = ~nulls[:, 0]
        assert not nulls[:, 1].any() and np.array_equal(vals[m, 0], vals[m, 1])
        k, c = np.unique(vals[m, 0], return_counts=True)
        assert np.array_equal(k, keys) and np.array_equal(c, counts)
        got_sum = vals[m, 2].view(np.float64).sum()
        assert abs(got_sum - price_sum) <= 1e-9 * abs(price_sum)
        if jointype == capi.JOIN_RIGHT:
            assert (~m).sum() == unmatched and not np.isin(vals[~m, 1], keys).any() and nulls[~m, 2].all()
    finally:
        jr.free()
        orel.free()
        irel.free()
        hj.jointype = capi.JOIN_INNER


def test_sort_skips_the_dead_slots_of_windowed_join_rows(eng, fk_join):
    from greengage_b200.engine import Relation
    li, od, nod, p, hj, targets, keys, counts, price_sum = fk_join
    b = ex.PlanBuilder()
    join = b.hashjoin(b.seqscan(0, capi.synth_tupdesc(capi.TAB_LINEITEM_NARROW)), b.hash(b.seqscan(1, capi.synth_tupdesc(capi.TAB_ORDERS))),
                      hj, targets)
    top = b.limit(b.sort(join, [capi.make_sortkey(0, capi.INT8OID)]), 1000)
    rels = [Relation(eng, host_pages=li), Relation(eng, host_pages=od)]
    x = ex.Executor(eng, p.pool, rels, top)
    try:
        got = [v[0] for v, nl, ty, ln in x.rows()]
        assert got == np.repeat(keys, counts)[:1000].tolist()
    finally:
        x.end()
        for r in rels:
            r.free()
