"""GPU parity tests for SeqScan ⋈ Hash(SeqScan) -> Agg through the C-ABI (gg_joinagg_*), against the oracle's
Hash / HashJoin restatement (oracle/or_join.c; pinned by tests/test_oracle_join.py).
Bar: joined-row counts, keys and integer aggregates bit-exact; float8 sums within 1e-6 relative."""
import numpy as np
import pytest

from _util import assert_aggrows_match
from greengage_b200 import capi, tpch
from oracle import pyoracle as po
from test_oracle_join import join_nodes, small_relations

pytestmark = pytest.mark.gpu

JOINTYPES = [capi.JOIN_INNER, capi.JOIN_LEFT, capi.JOIN_RIGHT, capi.JOIN_FULL, capi.JOIN_SEMI, capi.JOIN_ANTI, capi.JOIN_LASJ_NOTIN]
BOTH_SIDES = (capi.JOIN_INNER, capi.JOIN_LEFT, capi.JOIN_RIGHT, capi.JOIN_FULL)      # join types whose output carries inner columns


@pytest.fixture(scope="module")
def eng():
    from greengage_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def gpu_joinagg(eng, outer, inner, hj, agg, pool, opages, ipages, host=False, twice=False):
    from greengage_b200.engine import JoinAgg, Relation
    ja = JoinAgg(eng, outer, inner, hj, agg, pool)
    orel = Relation(eng, host_pages=opages) if opages.size else Relation(eng, nblocks=0)
    irel = Relation(eng, host_pages=ipages) if ipages.size else Relation(eng, nblocks=0)
    try:
        ja.build(irel)
        if host:
            ja.probe_host(opages.ctypes.data, opages.size // capi.GG_BLCKSZ)
        else:
            ja.probe(orel)
        rows, nj = ja.fetch()
        if twice:                                   # rescan with the hash table kept
            ja.reset()
            ja.probe(orel)
            rows2, nj2 = ja.fetch()
            assert nj2 == nj and len(rows2) == len(rows)
        return rows, nj, ja.stats()
    finally:
        ja.free()
        orel.free()
        irel.free()


@pytest.mark.parametrize("jointype", JOINTYPES)
@pytest.mark.parametrize("nkeys", [1, 2])
@pytest.mark.parametrize("with_qual", [False, True])
def test_small_relations_duplicates_and_nulls(eng, jointype, nkeys, with_qual):
    odesc, idesc, orows, onulls, irows, inulls, opages, ipages = small_relations()
    p, outer, inner, hj = join_nodes(odesc, idesc, jointype, nkeys, with_qual)
    grp = [p.var(2, capi.BPCHAROID, 1)] if jointype in BOTH_SIDES else [p.var(2, capi.BPCHAROID, 0)]
    aggs = [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_FLOAT8, p.var(3, capi.FLOAT8OID, 0))]
    if jointype in BOTH_SIDES:
        aggs += [(capi.AGG_SUM_INT4, p.var(3, capi.INT4OID, 1)), (capi.AGG_COUNT_ANY, p.var(1, capi.INT4OID, 1))]
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, grp, aggs)
    want, nj_want, want_x = po.hashjoin_agg(outer, inner, hj, agg, p.pool, opages, ipages, exact=True)
    got, nj, st = gpu_joinagg(eng, outer, inner, hj, agg, p.pool, opages, ipages)
    assert nj == nj_want
    assert_aggrows_match(got, want, agg, exact=want_x)


@pytest.mark.parametrize("kind,jointype", [("count", capi.JOIN_INNER), ("q3ish", capi.JOIN_INNER), ("q3ish", capi.JOIN_LEFT),
                                           ("count", capi.JOIN_ANTI), ("count", capi.JOIN_SEMI)])
def test_lineitem_orders_synth_vs_oracle(eng, kind, jointype):
    """BASELINE config 2 shape at a size the oracle finishes in seconds: lineitem ⋈ orders on int64 keys.
    orders holds fewer rows than lineitem references, so outer rows without a partner exist."""
    li, _, nli = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, 300_000, seed=3, norders=60_000))
    od, _, nod = tpch.synth_generate(tpch.synth_spec(capi.TAB_ORDERS, 45_000, seed=3))
    outer, inner, hj, agg, pool = tpch.join_plan(capi.TAB_LINEITEM_NARROW, kind, jointype)
    want, nj_want, want_x = po.hashjoin_agg(outer, inner, hj, agg, pool, li, od, exact=True)
    got, nj, st = gpu_joinagg(eng, outer, inner, hj, agg, pool, li, od, twice=True)
    assert st["rows_built"] <= nod
    assert nj == nj_want and nj > 0
    assert_aggrows_match(got, want, agg, exact=want_x)
    got_h, nj_h, _ = gpu_joinagg(eng, outer, inner, hj, agg, pool, li, od, host=True)
    assert nj_h == nj_want
    assert_aggrows_match(got_h, want, agg, exact=want_x)


@pytest.mark.parametrize("nkeys", [1, 2])
def test_lasj_notin_with_a_null_free_inner_side(eng, nkeys):
    """NOT IN over an inner side without NULL keys: an anti join that also drops outer rows with NULL keys; and
    against an empty inner side every outer row qualifies."""
    odesc, idesc, orows, onulls, irows, inulls, opages, ipages = small_relations(seed=12)
    inulls = [[False, False, n[2]] for n in inulls]
    ipages = po.build_pages(idesc, irows, inulls)
    p, outer, inner, hj = join_nodes(odesc, idesc, capi.JOIN_LASJ_NOTIN, nkeys, False)
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [p.var(2, capi.BPCHAROID, 0)], [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_FLOAT8, p.var(3, capi.FLOAT8OID, 0))])
    for ip in (ipages, np.zeros(0, dtype=np.uint8)):
        want, nj_want, want_x = po.hashjoin_agg(outer, inner, hj, agg, p.pool, opages, ip, exact=True)
        got, nj, _ = gpu_joinagg(eng, outer, inner, hj, agg, p.pool, opages, ip, twice=True)
        assert nj == nj_want and nj > 0
        assert_aggrows_match(got, want, agg, exact=want_x)


@pytest.mark.parametrize("jointype", [capi.JOIN_RIGHT, capi.JOIN_FULL])
def test_right_and_full_join_synth(eng, jointype):
    """orders holds keys no lineitem references and lineitem references orders that are missing: both sides have
    unmatched rows.  Rescan (hash table kept) must forget the match marks."""
    li, _, nli = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, 200_000, seed=4, norders=40_000))
    od_all, _, nod = tpch.synth_generate(tpch.synth_spec(capi.TAB_ORDERS, 60_000, seed=4))
    outer, inner, hj, agg, pool = tpch.join_plan(capi.TAB_LINEITEM_NARROW, "q3ish", jointype)
    want, nj_want, want_x = po.hashjoin_agg(outer, inner, hj, agg, pool, li, od_all, exact=True)
    got, nj, st = gpu_joinagg(eng, outer, inner, hj, agg, pool, li, od_all, twice=True)
    assert nj == nj_want
    assert_aggrows_match(got, want, agg, exact=want_x)
    got_h, nj_h, _ = gpu_joinagg(eng, outer, inner, hj, agg, pool, li, od_all, host=True)
    assert nj_h == nj_want
    assert_aggrows_match(got_h, want, agg, exact=want_x)


def test_join_with_a_high_cardinality_aggregate(eng):
    """HashJoin feeding the general HashAggregate: GROUP BY l_orderkey above the join."""
    from greengage_b200.capi import ExprPool
    from greengage_b200.engine import JoinAgg, Relation
    li, _, nli = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, 150_000, seed=2, norders=30_000))
    od, _, nod = tpch.synth_generate(tpch.synth_spec(capi.TAB_ORDERS, 24_000, seed=2))
    c, oc = tpch.LI_NARROW_COLS, tpch.ORDERS_COLS
    p = ExprPool()
    lkey, okey = p.var(c["orderkey"], capi.INT8OID, 0), p.var(oc["orderkey"], capi.INT8OID, 1)
    outer = capi.make_scan(capi.synth_tupdesc(capi.TAB_LINEITEM_NARROW), -1)
    inner = capi.make_scan(capi.synth_tupdesc(capi.TAB_ORDERS), -1)
    hj = capi.make_hashjoin(capi.JOIN_LEFT, [lkey], [okey])
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [lkey], [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_FLOAT8, p.var(c["extendedprice"], capi.FLOAT8OID, 0)),
                                                      (capi.AGG_MIN_DATE, p.var(oc["orderdate"], capi.DATEOID, 1))], num_groups=30_000)
    want, nj_want, want_x = po.hashjoin_agg(outer, inner, hj, agg, p.pool, li, od, cap=100_000, exact=True)
    ja = JoinAgg(eng, outer, inner, hj, agg, p.pool)
    lrel, orel = Relation(eng, host_pages=li), Relation(eng, host_pages=od)
    try:
        ja.build(orel)
        ja.probe(lrel)
        got, nj = ja.fetch(cap=100_000)
        assert nj == nj_want and len(got) == len(want) > 20_000
        assert_aggrows_match(got, want, agg, exact=want_x)
    finally:
        ja.free(); lrel.free(); orel.free()


def test_empty_sides(eng):
    li, _, _ = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, 5000, seed=4))
    od, _, _ = tpch.synth_generate(tpch.synth_spec(capi.TAB_ORDERS, 1250, seed=4))
    empty = np.zeros(0, dtype=np.uint8)
    for jt in (capi.JOIN_INNER, capi.JOIN_LEFT):
        outer, inner, hj, agg, pool = tpch.join_plan(capi.TAB_LINEITEM_NARROW, "count", jt)
        for op, ip in ((li, empty), (empty, od)):
            want, nj_want, want_x = po.hashjoin_agg(outer, inner, hj, agg, pool, op, ip, exact=True)
            got, nj, _ = gpu_joinagg(eng, outer, inner, hj, agg, pool, op, ip)
            assert nj == nj_want
            assert_aggrows_match(got, want, agg, exact=want_x)


def test_unsupported_join_shapes_are_refused(eng):
    from greengage_b200.engine import JoinAgg
    outer, inner, hj, agg, pool = tpch.join_plan(capi.TAB_LINEITEM_NARROW, "count")
    hj.jointype = 7                                   # JOIN_UNIQUE_OUTER: a planner-internal code, the CPU node keeps it
    with pytest.raises(capi.GGError) as e:
        JoinAgg(eng, outer, inner, hj, agg, pool)
    assert e.value.code == -6


def gpu_join_batched(eng, outer, inner, hj, agg, pool, opages, ipages, work_mem):
    from greengage_b200.engine import JoinAgg, Relation
    ja = JoinAgg(eng, outer, inner, hj, agg, pool)
    orel = Relation(eng, host_pages=opages) if opages.size else Relation(eng, nblocks=0)
    irel = Relation(eng, host_pages=ipages) if ipages.size else Relation(eng, nblocks=0)
    try:
        ja.set_work_mem(work_mem)
        nbatch = ja.run(irel, orel)
        rows, nj = ja.fetch()
        ja.reset()                                   # ExecReScanHashJoin: the same answer again, batches and all
        nbatch2 = ja.run(irel, orel)
        rows2, nj2 = ja.fetch()
        assert nbatch2 == nbatch and nj2 == nj and len(rows2) == len(rows)
        return rows, nj, nbatch, ja.stats()
    finally:
        ja.free()
        orel.free()
        irel.free()


@pytest.mark.parametrize("jointype", [capi.JOIN_INNER, capi.JOIN_LEFT, capi.JOIN_RIGHT, capi.JOIN_FULL, capi.JOIN_SEMI, capi.JOIN_ANTI])
@pytest.mark.parametrize("nkeys", [1, 2])
def test_hybrid_hash_join_batches_small_relations(eng, jointype, nkeys):
    """A hash table that does not fit the operator's memory (artificially tiny here): both sides are split by the batch bits of
    the reference's hash value and joined batch by batch — duplicates, NULL keys, a join qual, every join type that has a
    probe side; the answer is the one-table oracle's (nodeHash.c:713,1132; nodeHashjoin.c:906)."""
    odesc, idesc, orows, onulls, irows, inulls, opages, ipages = small_relations()
    p, outer, inner, hj = join_nodes(odesc, idesc, jointype, nkeys, True)
    grp = [p.var(2, capi.BPCHAROID, 1)] if jointype in BOTH_SIDES else [p.var(2, capi.BPCHAROID, 0)]
    aggs = [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_FLOAT8, p.var(3, capi.FLOAT8OID, 0))]
    if jointype in BOTH_SIDES:
        aggs += [(capi.AGG_SUM_INT4, p.var(3, capi.INT4OID, 1)), (capi.AGG_COUNT_ANY, p.var(1, capi.INT4OID, 1))]
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, grp, aggs)
    want, nj_want, want_x = po.hashjoin_agg(outer, inner, hj, agg, p.pool, opages, ipages, exact=True)
    got, nj, nbatch, st = gpu_join_batched(eng, outer, inner, hj, agg, p.pool, opages, ipages, work_mem=8192)
    assert nbatch >= 2
    assert nj == nj_want
    assert_aggrows_match(got, want, agg, exact=want_x)


@pytest.mark.parametrize("kind,jointype", [("survey", capi.JOIN_INNER), ("q3ish", capi.JOIN_INNER), ("q3ish", capi.JOIN_LEFT), ("count", capi.JOIN_ANTI)])
def test_hybrid_hash_join_build_side_larger_than_the_budget(eng, kind, jointype):
    """lineitem ⋈ orders with the operator's memory at a fraction of the hash table the inner side needs: 4 to 16 batches."""
    li, _, nli = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, 400_000, seed=5, norders=90_000))
    od, _, nod = tpch.synth_generate(tpch.synth_spec(capi.TAB_ORDERS, 70_000, seed=5))
    outer, inner, hj, agg, pool = tpch.join_plan(capi.TAB_LINEITEM_NARROW, kind, jointype)
    want, nj_want, want_x = po.hashjoin_agg(outer, inner, hj, agg, pool, li, od, exact=True)
    one, nj_one, _ = gpu_joinagg(eng, outer, inner, hj, agg, pool, li, od)
    table_bytes = _["table_bytes"]
    got, nj, nbatch, st = gpu_join_batched(eng, outer, inner, hj, agg, pool, li, od, work_mem=table_bytes // 5)
    assert 4 <= nbatch <= 16
    assert nj == nj_want == nj_one and nj > 0
    assert_aggrows_match(got, want, agg, exact=want_x)
    # and with memory to spare nothing is batched
    got1, nj1, nbatch1, _ = gpu_join_batched(eng, outer, inner, hj, agg, pool, li, od, work_mem=table_bytes * 2)
    assert nbatch1 == 1 and nj1 == nj_want
