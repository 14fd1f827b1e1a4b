"""The executor-node surface end to end on the GPU: plans are built the way the Postgres-side translator builds
them, run through GgExecInitNode / GgExecProcNode / GgExecEndNode, and checked against the reference's golden Q1
answer (ORDER BY included) and the oracle.  The golden answer is printed to fewer digits than a float8 holds, so it is
met within 1e-6; float8 sums and averages are held to the oracle's exact record of the same pages
(_util.assert_aggrows_match with exact=)."""
import ctypes as C

import numpy as np
import pytest

from _util import assert_aggrows_match, golden, lineitem_fixture_pages
from greengage_b200 import capi, executor as ex, tpch
from oracle import pyoracle as po

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from greengage_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def b2f(v):
    return np.int64(v).view(np.float64).item()


FLOAT_AGGS = (capi.AGG_SUM_FLOAT8, capi.AGG_AVG_FLOAT8, capi.AGG_MIN_FLOAT8, capi.AGG_MAX_FLOAT8)


def as_aggrows(rows, want, agg, row_key, want_key):
    """executor rows (grouping columns, then one column per aggregate) as gg_aggrows, keyed by the oracle row of the same
    group so that assert_aggrows_match compares them; row_key(v, ln) and want_key(aggrow) name a group the same way"""
    by = {want_key(w): w for w in want}
    out = []
    for v, nl, ty, ln in rows:
        r = capi.gg_aggrow()
        C.memmove(C.byref(r), C.byref(by[row_key(v, ln)]), C.sizeof(r))       # the keys, in the oracle's encoding
        for i in range(agg.numAggs):
            col = agg.numCols + i
            r.agg[i].isnull = nl[col]
            if agg.aggs[i].aggfnoid in FLOAT_AGGS:
                r.agg[i].f[0] = b2f(v[col])
            else:
                r.agg[i].i = v[col]
        out.append(r)
    return out


def q1_oracle(desc, pages, exp):
    """(agg, oracle rows, exact record) of the one-stage Q1 over the pages: what a one- or two-stage plan must meet"""
    scan, agg, pool = tpch.q1_plan(capi.TAB_LINEITEM_WIDE, capi.AGGSTAGE_NORMAL, interval_days=exp["interval_days"], desc=desc)
    want, _, _, want_x = po.seqscan_agg(scan, agg, pool, pages, exact=True)
    return agg, want, want_x


def check_q1_exact(rows, oracle):
    agg, want, want_x = oracle
    key = lambda a, la, b, lb: (capi.unpack_str(a, la), capi.unpack_str(b, lb))
    got = as_aggrows(rows, want, agg, lambda v, ln: key(v[0], ln[0], v[1], ln[1]), lambda w: key(w.key[0], w.keylen[0], w.key[1], w.keylen[1]))
    assert_aggrows_match(got, want, agg, exact=want_x)


def q1_sorted_plan(b, scan, agg, two_stage):
    keys = [capi.make_sortkey(0, capi.BPCHAROID), capi.make_sortkey(1, capi.BPCHAROID)]
    ss = b.seqscan(0, scan.desc, scan.qual)
    if not two_stage:
        return b.sort(b.agg(ss, agg), keys)
    part = capi.gg_agg.from_buffer_copy(bytes(agg))
    part.aggstage = capi.AGGSTAGE_PARTIAL
    fin = tpch.q1_final_agg(part)
    # Gather Motion <- Sort <- Agg(FINAL) <- Redistribute Motion <- Agg(PARTIAL) <- SeqScan   (tpch500GB.out:1771-1782)
    return b.motion(b.sort(b.agg(b.motion(b.agg(ss, part), ex.MOTION_HASH, [0, 1], 1), fin), keys), ex.MOTION_GATHER, [], 2,
                    merge_keys=keys)          # Gather Motion with Merge Key: l_returnflag, l_linestatus


@pytest.mark.parametrize("two_stage", [False, True])
def test_q1_end_to_end_matches_the_reference_answer(eng, two_stage):
    from greengage_b200.engine import Relation
    desc, pages, n = lineitem_fixture_pages()
    exp = golden("q1_expected.json")
    scan, agg, pool = tpch.q1_plan(capi.TAB_LINEITEM_WIDE, capi.AGGSTAGE_NORMAL, interval_days=exp["interval_days"], desc=desc)
    rel = Relation(eng, host_pages=pages)
    b = ex.PlanBuilder()
    x = ex.Executor(eng, pool, [rel], q1_sorted_plan(b, scan, agg, two_stage))
    try:
        assert x.kind() == ("motion" if two_stage else "sort")
        rows = x.rows()
        want = exp["rows"]
        assert len(rows) == len(want)
        for (v, nl, ty, ln), w in zip(rows, want):                 # ORDER BY l_returnflag, l_linestatus
            assert capi.unpack_str(v[0], ln[0]) == w["returnflag"] and capi.unpack_str(v[1], ln[1]) == w["linestatus"]
            assert v[9] == w["count_order"]
            for col, name in ((2, "sum_qty"), (3, "sum_base_price"), (4, "sum_disc_price"), (5, "sum_charge"),
                              (6, "avg_qty"), (7, "avg_price"), (8, "avg_disc")):
                assert abs(b2f(v[col]) - float(w[name])) <= 1e-6 * abs(float(w[name])), (name, b2f(v[col]), w[name])
        check_q1_exact(rows, q1_oracle(desc, pages, exp))           # two stages: one tree over the same inputs, same bound
        assert x.rows() == []                                       # end of stream stays end of stream
        x.rescan()
        assert len(x.rows()) == len(want)                           # ExecReScan runs the slice again
        x.rescan()
        assert len(x.rows(limit=2)) == 2 and x.rows() == []          # squelched after LIMIT
    finally:
        x.end()
        rel.free()


def test_join_through_the_node_surface(eng):
    from greengage_b200.engine import Relation
    li, _, _ = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, 100_000, seed=6, norders=20_000))
    od, _, _ = tpch.synth_generate(tpch.synth_spec(capi.TAB_ORDERS, 15_000, seed=6))
    outer, inner, hj, agg, pool = tpch.join_plan(capi.TAB_LINEITEM_NARROW, "q3ish", capi.JOIN_INNER)
    want, _, want_x = po.hashjoin_agg(outer, inner, hj, agg, pool, li, od, exact=True)
    lrel, orel = Relation(eng, host_pages=li), Relation(eng, host_pages=od)
    b = ex.PlanBuilder()
    plan = b.sort(b.agg(b.hashjoin(b.seqscan(0, outer.desc, outer.qual), b.hash(b.seqscan(1, inner.desc, inner.qual)), hj), agg),
                  [capi.make_sortkey(0, capi.BPCHAROID, desc=True)])
    x = ex.Executor(eng, pool, [lrel, orel], plan)
    try:
        rows = x.rows()
        keys = [capi.unpack_str(v[0], ln[0]) for v, nl, ty, ln in rows]
        assert keys == sorted(keys, reverse=True) and len(rows) == len(want)
        assert_aggrows_match(as_aggrows(rows, want, agg, lambda v, ln: v[0], lambda w: w.key[0]), want, agg, exact=want_x)
    finally:
        x.end()
        lrel.free()
        orel.free()


def test_device_errors_surface_through_exec_proc_node(eng):
    from _util import make_desc
    from greengage_b200.capi import ExprPool
    from greengage_b200.engine import Relation
    desc = make_desc([(capi.FLOAT8OID, 8, "d", 1, 1), (capi.FLOAT8OID, 8, "d", 1, 1)])
    pages = po.build_pages(desc, [[1.0, 0.0]])
    p = ExprPool()
    agg = capi.make_agg(0, [], [(capi.AGG_SUM_FLOAT8, p.func(capi.F_FLOAT8DIV, capi.FLOAT8OID, p.var(1, capi.FLOAT8OID), p.var(2, capi.FLOAT8OID)))])
    rel = Relation(eng, host_pages=pages)
    b = ex.PlanBuilder()
    x = ex.Executor(eng, p.pool, [rel], b.agg(b.seqscan(0, desc), agg))
    try:
        with pytest.raises(ex.ExecError) as e:
            x.rows()
        assert e.value.code == -4 and "division by zero" in str(e.value)
    finally:
        x.end()
        rel.free()


# ---- results that stay on the device between the nodes of a slice (gg_groups / datum rows) and the C interconnect ----

def _check_q1_rows(rows, exp, oracle):
    by = {(capi.unpack_str(v[0], ln[0]), capi.unpack_str(v[1], ln[1])): v for v, nl, ty, ln in rows}
    assert len(by) == len(rows) == len(exp["rows"])
    for w in exp["rows"]:
        v = by[(w["returnflag"], w["linestatus"])]
        assert v[9] == w["count_order"]
        for col, name in ((2, "sum_qty"), (3, "sum_base_price"), (4, "sum_disc_price"), (5, "sum_charge"),
                          (6, "avg_qty"), (7, "avg_price"), (8, "avg_disc")):
            assert abs(b2f(v[col]) - float(w[name])) <= 1e-6 * abs(float(w[name])), (name, b2f(v[col]), w[name])
    check_q1_exact(rows, oracle)


def test_two_stage_q1_stays_on_the_device_through_the_interconnect(eng):
    """Gather <- Agg(FINAL) <- Redistribute <- Agg(PARTIAL) <- SeqScan with the C interconnect (one segment: loopback, the
    same pack / route / combine kernels as over NCCL): the partial rows never leave the device until the top node is asked
    for tuples, and the answer is the reference's golden Q1."""
    from greengage_b200.engine import Interconnect, Relation
    desc, pages, n = lineitem_fixture_pages()
    exp = golden("q1_expected.json")
    rel = Relation(eng, host_pages=pages)
    ic = Interconnect(eng, 1, 0)
    b = ex.PlanBuilder()
    plan, pool = tpch.q1_exec_plan(b, two_stage=True, interval_days=exp["interval_days"], desc=desc)
    x = ex.Executor(eng, pool, [rel], plan, interconnect=ic)
    oracle = q1_oracle(desc, pages, exp)      # the device FINAL against the exact record of the one-stage scan of the pages
    try:
        rows = x.rows()
        _check_q1_rows(rows, exp, oracle)
        loc = x.locations()
        assert [k for k, _ in loc] == ["motion", "aggfinal", "motion", "scanagg"]
        assert loc[1][1] == "device-groups" and loc[2][1] == "device-groups"      # FINAL Agg and Redistribute: no host rows
        x.rescan()
        _check_q1_rows(x.rows(), exp, oracle)
    finally:
        x.end()
        ic.close()
        rel.free()


def test_scan_of_a_relation_in_host_memory(eng):
    """GgEState.host_pages: the SeqScan's pages are in (pinned) host memory and are streamed to the device inside the
    pipeline — the end-to-end path bench.py times"""
    from greengage_b200.engine import host_alloc, host_free
    desc, pages, n = lineitem_fixture_pages()
    exp = golden("q1_expected.json")
    addr, view = host_alloc(pages.size)
    view[:] = pages
    b = ex.PlanBuilder()
    plan, pool = tpch.q1_exec_plan(b, two_stage=False, interval_days=exp["interval_days"], desc=desc)
    x = ex.Executor(eng, pool, [(addr, pages.size // capi.GG_BLCKSZ)], plan)
    try:
        _check_q1_rows(x.rows(), exp, q1_oracle(desc, pages, exp))
    finally:
        x.end()
        host_free(addr)


@pytest.mark.parametrize("kind", ["q3ish", "survey"])
@pytest.mark.parametrize("redistribute", [True, False])
def test_redistribute_hashjoin_plan(eng, kind, redistribute):
    """BASELINE config 3's plan through the node surface on one segment: both sides projected by their scans, partitioned on
    the join key (device Motion), joined over the delivered datum rows, aggregated in two stages — equal to the oracle's join
    over the heap pages."""
    from greengage_b200.engine import Interconnect, Relation
    li, _, _ = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, 120_000, seed=9, norders=30_000))
    od, _, _ = tpch.synth_generate(tpch.synth_spec(capi.TAB_ORDERS, 25_000, seed=9))
    outer, inner, hj, agg, pool0 = tpch.join_plan(capi.TAB_LINEITEM_NARROW, kind, capi.JOIN_INNER)
    want, nj, want_x = po.hashjoin_agg(outer, inner, hj, agg, pool0, li, od, exact=True)
    lrel, orel = Relation(eng, host_pages=li), Relation(eng, host_pages=od)
    ic = Interconnect(eng, 1, 0)
    b = ex.PlanBuilder()
    plan, pool, _, _ = tpch.rjoin_exec_plan(b, kind, redistribute=redistribute)
    x = ex.Executor(eng, pool, [lrel, orel], plan, interconnect=ic)
    try:
        rows = x.rows()
        assert len(rows) == len(want)
        if kind == "survey":
            v = rows[0][0]
            w = want[0]
            assert v[0] == w.agg[0].i == nj and v[1] == w.agg[1].i               # count(*), sum(o_custkey): bit-exact
            got = as_aggrows(rows, want, agg, lambda v, ln: (), lambda w: ())
        else:
            got = as_aggrows(rows, want, agg, lambda v, ln: v[0], lambda w: w.key[0])
        assert_aggrows_match(got, want, agg, exact=want_x)
        if redistribute:
            L = ex.exec_lib()
            join_state = L.GgExecOuterPlanState(L.GgExecOuterPlanState(x.state))      # Agg(FINAL) -> Gather -> Agg over the join
            assert L.GgExecNodeKind(join_state) == b"joinagg"
            assert L.GgExecNodeResultLocation(L.GgExecOuterPlanState(join_state)) == b"device-rows"
            assert L.GgExecNodeResultLocation(L.GgExecInnerPlanState(join_state)) == b"device-rows"
    finally:
        x.end()
        ic.close()
        lrel.free()
        orel.free()


def test_bare_seqscan_with_a_target_list_returns_its_rows(eng):
    """ExecSeqScan proper (nodeSeqscan.c:128): qual + projection, tuples handed to the caller one slot at a time"""
    from greengage_b200.capi import ExprPool
    from greengage_b200.engine import Relation
    li, _, nr = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, 20_000, seed=3))
    c = tpch.LI_NARROW_COLS
    desc = capi.synth_tupdesc(capi.TAB_LINEITEM_NARROW)
    p = ExprPool()
    key, price, flag = p.var(c["orderkey"], capi.INT8OID), p.var(c["extendedprice"], capi.FLOAT8OID), p.var(c["returnflag"], capi.BPCHAROID)
    qual = p.func(capi.F_FLOAT8GT, capi.BOOLOID, p.var(c["quantity"], capi.FLOAT8OID), p.const(capi.FLOAT8OID, 25.0))
    agg = capi.make_agg(0, [], [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_FLOAT8, price), (capi.AGG_SUM_FLOAT8, p.func(capi.F_I8TOD, capi.FLOAT8OID, key))])
    want, sc, ps = po.seqscan_agg(capi.make_scan(desc, qual), agg, p.pool, li)
    rel = Relation(eng, host_pages=li)
    b = ex.PlanBuilder()
    x = ex.Executor(eng, p.pool, [rel], b.seqscan(0, desc, qual, targets=[key, price, flag]))
    try:
        assert x.kind() == "scanrows"
        rows = x.rows()
        assert len(rows) == ps == want[0].agg[0].i
        assert rows[0][2] == [capi.INT8OID, capi.FLOAT8OID, capi.BPCHAROID]
        assert sorted(capi.unpack_str(v[2], ln[2]) for v, nl, ty, ln in rows[:200]) <= ["R"] * 200
        assert abs(sum(b2f(v[1]) for v, nl, ty, ln in rows) - want[0].agg[1].f[0]) <= 1e-9 * want[0].agg[1].f[0]
        assert sum(v[0] for v, nl, ty, ln in rows) == int(want[0].agg[2].f[0])
    finally:
        x.end()
        rel.free()


def test_sort_over_a_row_producing_seqscan_stays_on_the_device(eng):
    """Sort <- SeqScan(targets) (nodeSort.c:48 over nodeSeqscan.c:128): the scan leaves datum rows on the device, the Sort orders
    them there (comparator of tuplesort_mk.c:2816: DESC, then ASC on the second key) and the rows come to the host once."""
    import numpy as np
    from greengage_b200.capi import ExprPool
    from greengage_b200.engine import Relation
    li, _, nr = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, 30_000, seed=11))
    c = tpch.LI_NARROW_COLS
    desc = capi.synth_tupdesc(capi.TAB_LINEITEM_NARROW)
    p = ExprPool()
    key, price, flag, date = (p.var(c["orderkey"], capi.INT8OID), p.var(c["extendedprice"], capi.FLOAT8OID),
                              p.var(c["returnflag"], capi.BPCHAROID), p.var(c["shipdate"], capi.DATEOID))
    qual = p.func(capi.F_FLOAT8GT, capi.BOOLOID, p.var(c["quantity"], capi.FLOAT8OID), p.const(capi.FLOAT8OID, 10.0))
    rel = Relation(eng, host_pages=li)
    b = ex.PlanBuilder()
    scan = b.seqscan(0, desc, qual, targets=[key, price, flag, date])
    x0 = ex.Executor(eng, p.pool, [rel], scan)
    x = ex.Executor(eng, p.pool, [rel], b.sort(b.seqscan(0, desc, qual, targets=[key, price, flag, date]),
                                                 [capi.make_sortkey(2, capi.BPCHAROID, desc=True), capi.make_sortkey(1, capi.FLOAT8OID),
                                                  capi.make_sortkey(0, capi.INT8OID)]))
    try:
        plain = x0.rows()
        rows = x.rows()
        assert len(rows) == len(plain) > 20_000
        assert sorted(tuple(v) for v, nl, ty, ln in rows) == sorted(tuple(v) for v, nl, ty, ln in plain)      # same multiset of rows
        keys = [(-ord(capi.unpack_str(v[2], ln[2])), b2f(v[1]), v[0]) for v, nl, ty, ln in rows]
        assert keys == sorted(keys)
        assert len({k[0] for k in keys}) == 3
    finally:
        x.end()
        x0.end()
        rel.free()


def test_es_snapshot_reaches_the_scans_of_the_slice(eng):
    """EState.es_snapshot -> heap_beginscan -> HeapTupleSatisfiesMVCC (execMain.c / heapam.c:1573 / tqual.c:997): the join's
    two scans both judge their tuples against the query's snapshot"""
    from _util import mvcc_snapshot, stamp_visibility
    from greengage_b200.engine import Relation
    li, _, nli = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, 40_000, norders=10_000, seed=4))
    od, _, nod = tpch.synth_generate(tpch.synth_spec(capi.TAB_ORDERS, 10_000, seed=4))
    li, vli = stamp_visibility(li, all_visible_every=5)
    od, vod = stamp_visibility(od)
    outer, inner, hj, agg, pool = tpch.join_plan(capi.TAB_LINEITEM_NARROW, "survey", capi.JOIN_INNER)
    snap = mvcc_snapshot()
    po.set_snapshot(snap)
    try:
        want, wj = po.hashjoin_agg(outer, inner, hj, agg, pool, li, od)
    finally:
        po.set_snapshot(None)
    assert 0 < wj < sum(vli)
    rl, ro = Relation(eng, host_pages=li), Relation(eng, host_pages=od)
    b = ex.PlanBuilder()
    plan = b.agg(b.hashjoin(b.seqscan(0, outer.desc, outer.qual), b.hash(b.seqscan(1, inner.desc, inner.qual)), hj), agg)
    x = ex.Executor(eng, pool, [rl, ro], plan, snapshot=snap)
    try:
        rows = x.rows()
        assert len(rows) == 1 and rows[0][0][0] == wj == want[0].agg[0].i
        assert rows[0][0][1] == want[0].agg[1].i
    finally:
        x.end()
    x = ex.Executor(eng, pool, [rl, ro], plan)                  # no snapshot: the relation is not the GPU's to scan
    try:
        with pytest.raises(ex.ExecError) as e:
            x.rows()
        assert e.value.code == -7
    finally:
        x.end()
        rl.free(); ro.free()
