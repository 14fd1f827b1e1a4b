"""GPU parity tests for the SeqScan -> qual -> Agg path, through the C-ABI (libggb200.so), against the
oracle (oracle/) and the reference's golden Q1 answer.  Every kernel variant is exercised: private
accumulators / transposed accumulate, interpreter / plan-specialised (build-time cache and NVRTC).
Bar: keys, counts and integer aggregates bit-exact; float8 SUM/AVG against the oracle's exact sums (_util.assert_aggrows_match
with exact=): bit for bit where every summation order is exact, else within the proven bound γ(n-1)·Σ|x|."""
import ctypes as C
import os

import numpy as np
import pytest

from _util import assert_aggrows_match, golden, lineitem_fixture_pages, make_desc
from greengage_b200 import capi, tpch
from greengage_b200.capi import ExprPool
from oracle import pyoracle as po

pytestmark = pytest.mark.gpu

VARIANTS = {
    "specialised-priv": {},
    "nvrtc-priv": {"GGB200_PLAN_CACHE": "0"},
    "interp-priv": {"GGB200_JIT": "0"},
    "specialised-tr": {"GGB200_SCAN_MODE": "1"},
    "interp-tr": {"GGB200_JIT": "0", "GGB200_SCAN_MODE": "1"},
}


@pytest.fixture(scope="module")
def eng():
    from greengage_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


class env:
    def __init__(self, **kw):
        self.kw = kw

    def __enter__(self):
        self.old = {k: os.environ.get(k) for k in ("GGB200_JIT", "GGB200_SCAN_MODE", "GGB200_PLAN_CACHE")}
        for k in self.old:
            os.environ.pop(k, None)
        os.environ.update(self.kw)

    def __exit__(self, *a):
        for k, v in self.old.items():
            os.environ.pop(k, None)
            if v is not None:
                os.environ[k] = v


def gpu_scanagg(eng, scan, agg, pool, pages, variant=None, ranges=None, host=False):
    from greengage_b200.engine import Relation, ScanAgg
    # the variant's environment stays in force for the whole pipeline life: the kernel is (re)chosen at the first run too
    with env(**(VARIANTS[variant] if variant else {})):
        sa = ScanAgg(eng, scan, agg, pool)
        rel = Relation(eng, host_pages=pages) if pages.size else Relation(eng, nblocks=0)
        nb = pages.size // capi.GG_BLCKSZ
        try:
            if host:
                sa.run_host(pages.ctypes.data, nb)
            elif ranges:
                for a, b in ranges:
                    sa.run(rel, a, b - a)
            else:
                sa.run(rel)
            rows, sc, ps = sa.fetch()
            return rows, sc, ps, sa.variant()
        finally:
            sa.free()
            rel.free()


# ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("variant", list(VARIANTS))
def test_q1_reference_fixture_all_variants(eng, variant):
    """The reference's own regression data and golden answer (rpt_tpch.source:288-315)."""
    desc, pages, n = lineitem_fixture_pages()
    exp = golden("q1_expected.json")
    scan, agg, pool = tpch.q1_plan(capi.TAB_LINEITEM_WIDE, capi.AGGSTAGE_NORMAL, interval_days=exp["interval_days"], desc=desc)
    rows, sc, ps, var = gpu_scanagg(eng, scan, agg, pool, pages, variant)
    if variant.startswith("specialised") or variant.startswith("nvrtc"):
        assert var >= 16, "plan-specialised kernel expected, got variant %d" % var
    else:
        assert var < 16
    assert sc == n and ps == sum(e["count_order"] for e in exp["rows"])
    got = {(capi.unpack_str(r.key[0], r.keylen[0]), capi.unpack_str(r.key[1], r.keylen[1])): r for r in rows}
    assert len(got) == 4
    for e in exp["rows"]:
        r = got[(e["returnflag"], e["linestatus"])]
        assert r.agg[7].i == e["count_order"]
        for i, name in enumerate(["sum_qty", "sum_base_price", "sum_disc_price", "sum_charge", "avg_qty", "avg_price", "avg_disc"]):
            want = float(e[name])
            assert abs(r.agg[i].f[0] - want) <= 1e-6 * abs(want), (name, r.agg[i].f[0], want)
    want, _, _, want_x = po.seqscan_agg(scan, agg, pool, pages, exact=True)
    assert_aggrows_match(rows, want, agg, exact=want_x)


@pytest.mark.parametrize("table", [capi.TAB_LINEITEM_WIDE, capi.TAB_LINEITEM_NARROW])
@pytest.mark.parametrize("stage", [capi.AGGSTAGE_NORMAL, capi.AGGSTAGE_PARTIAL])
def test_q1_synthetic_vs_oracle(eng, table, stage):
    pages, nb, nr = tpch.synth_generate(tpch.synth_spec(table, 400000, seed=7))
    scan, agg, pool = tpch.q1_plan(table, stage)
    for variant in ("specialised-priv", "interp-tr"):
        rows, sc, ps, _ = gpu_scanagg(eng, scan, agg, pool, pages, variant)
        want, wsc, wps, want_x = po.seqscan_agg(scan, agg, pool, pages, exact=True)
        assert (sc, ps) == (wsc, wps) == (nr, wps)
        assert_aggrows_match(rows, want, agg, exact=want_x)


@pytest.mark.parametrize("nullable", [True, False])
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_edge_relation_all_variants(eng, variant, nullable):
    """_util.EDGE_GROUPS (all -0, mixed zeros, infinities, NaN, cancellation inside the exact regime, groups of 1/31/32/33,
    NULLs) at NORMAL and PARTIAL stage: float8 sums against the exact sums — bit for bit where every order is exact, the
    sign of a zero sum included.  The plan has MIN/MAX, so the '-priv' variants run the transposed kernels here; see
    test_edge_sums_on_the_private_accumulator_kernels for those."""
    from _util import edge_plan, edge_relation
    desc, pages, n = edge_relation(nullable)
    for stage in (capi.AGGSTAGE_NORMAL, capi.AGGSTAGE_PARTIAL):
        scan, agg, pool = edge_plan(desc, stage)
        rows, sc, ps, _ = gpu_scanagg(eng, scan, agg, pool, pages, variant)
        want, wsc, wps, want_x = po.seqscan_agg(scan, agg, pool, pages, exact=True)
        assert (sc, ps) == (wsc, wps) == (n, n)
        assert_aggrows_match(rows, want, agg, exact=want_x)


@pytest.mark.parametrize("reg_slots", ["3", "0"])
@pytest.mark.parametrize("variant", ["specialised-priv", "nvrtc-priv", "interp-priv"])
def test_edge_sums_on_the_private_accumulator_kernels(eng, monkeypatch, variant, reg_slots):
    """The edge groups' sums through the private-accumulator kernels at NORMAL and PARTIAL stage: per-thread sums in shared
    memory, and in the plan-specialised kernels on wide tuples with at most 4 groups the trailing value slots in registers
    (GGB200_REG_SLOTS=0: every slot in shared memory).  A group of only -0 inputs sums to -0, every other sum is exact to
    the bit."""
    from _util import edge_relation, edge_sum_plan
    monkeypatch.setenv("GGB200_REG_SLOTS", reg_slots)
    desc, pages, n = edge_relation(nullable=False, pad=12)
    groups = (0, 1, 5, 15)                      # all -0, mixed zeros, cancellation in the exact regime, -0 with positives
    for stage in (capi.AGGSTAGE_NORMAL, capi.AGGSTAGE_PARTIAL):
        scan, agg, pool = edge_sum_plan(desc, groups, stage)
        rows, sc, ps, var = gpu_scanagg(eng, scan, agg, pool, pages, variant)
        assert var % 16 == 0, "private-accumulator kernel expected, got variant %d" % var
        assert (var >= 16) == (variant != "interp-priv"), var
        want, wsc, wps, want_x = po.seqscan_agg(scan, agg, pool, pages, exact=True)
        assert (sc, ps) == (wsc, wps) and len(want) == len(groups)
        assert_aggrows_match(rows, want, agg, exact=want_x)


def test_edge_relation_hash_aggregate_and_two_stages(eng):
    """the same edges through the general HashAggregate (group table in HBM, atomics) and through PARTIAL over two halves
    + the device FINAL, held to the exact record of the one-stage scan"""
    from _util import edge_plan, edge_relation, exact_by_key
    from greengage_b200.engine import agg_final
    desc, pages, n = edge_relation()
    scan, agg, pool = edge_plan(desc)
    want, _, _, want_x = po.seqscan_agg(scan, agg, pool, pages, exact=True)
    hagg = capi.make_agg(agg.aggstage, [agg.grpCol[0]], [(agg.aggs[i].aggfnoid, agg.aggs[i].arg) for i in range(agg.numAggs)], num_groups=1 << 20)
    rows, sc, ps, _ = gpu_scanagg(eng, scan, hagg, pool, pages)
    assert (sc, ps) == (n, n)
    assert_aggrows_match(rows, want, agg, exact=want_x)
    pscan, pagg, ppool = edge_plan(desc, capi.AGGSTAGE_PARTIAL)
    nb = pages.size // capi.GG_BLCKSZ
    parts = []
    for a, b in ((0, nb // 2), (nb // 2, nb)):
        r, _, _, _ = gpu_scanagg(eng, pscan, pagg, ppool, pages, ranges=[(a, b)])
        parts += r
    fin = capi.gg_agg()
    C.memmove(C.byref(fin), C.byref(pagg), C.sizeof(capi.gg_agg))
    fin.aggstage, fin.grpCol[0] = capi.AGGSTAGE_FINAL, capi.INT4OID     # a FINAL Agg's grpCol carries key type OIDs
    final = agg_final(eng, fin, parts)
    assert_aggrows_match(final, want, agg, exact=exact_by_key(want, want_x, 1))


def test_runs_accumulate_and_host_path_equals_resident(eng):
    pages, nb, nr = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, 300000, seed=3))
    scan, agg, pool = tpch.q1_plan(capi.TAB_LINEITEM_NARROW)
    whole, sc, ps, _ = gpu_scanagg(eng, scan, agg, pool, pages)
    parts, sc2, ps2, _ = gpu_scanagg(eng, scan, agg, pool, pages, ranges=[(0, 100), (100, 101), (101, nb)])
    host, sc3, ps3, _ = gpu_scanagg(eng, scan, agg, pool, pages, host=True)
    assert (sc, ps) == (sc2, ps2) == (sc3, ps3)
    assert_aggrows_match(parts, whole, agg, rel=1e-12)
    assert_aggrows_match(host, whole, agg, float_exact=True)         # same kernels, same order: identical bits
    again, _, _, _ = gpu_scanagg(eng, scan, agg, pool, pages)
    assert_aggrows_match(again, whole, agg, float_exact=True)        # deterministic run to run


def _nullable_relation(n=5000, seed=11):
    """int4 k (nullable), bpchar(1) f (nullable), float8 x (nullable), int4 i (nullable), date d"""
    rng = np.random.RandomState(seed)
    desc = make_desc([(capi.INT4OID, 4, 'i', 1), (capi.BPCHAROID, -1, 'i', 0), (capi.FLOAT8OID, 8, 'd', 1),
                      (capi.INT4OID, 4, 'i', 1), (capi.DATEOID, 4, 'i', 1, 1)])
    rows, nulls = [], []
    for r in range(n):
        k = int(rng.randint(0, 3))
        row = [k, bytes([65 + rng.randint(0, 3)]), float(rng.randint(-50, 50)) / 4.0, int(rng.randint(-1000, 1000)), int(rng.randint(-3000, 0))]
        nl = [int(rng.rand() < 0.1), int(rng.rand() < 0.1), int(rng.rand() < 0.2), int(rng.rand() < 0.2), 0]
        rows.append(row)
        nulls.append(nl)
    return desc, po.build_pages(desc, rows, nulls)


def test_nulls_in_keys_and_arguments(eng):
    desc, pages = _nullable_relation()
    p = ExprPool()
    k, f, x, i, d = p.var(1, capi.INT4OID), p.var(2, capi.BPCHAROID), p.var(3, capi.FLOAT8OID), p.var(4, capi.INT4OID), p.var(5, capi.DATEOID)
    qual = p.boolop(capi.E_OR, p.func(capi.F_DATE_GT, capi.BOOLOID, d, p.const(capi.DATEOID, -2500)),
                    p.boolop(capi.E_ISNULL, x))
    scan = capi.make_scan(desc, qual)
    aggs = [(capi.AGG_COUNT_STAR, -1), (capi.AGG_COUNT_ANY, x), (capi.AGG_SUM_FLOAT8, x), (capi.AGG_AVG_FLOAT8, x),
            (capi.AGG_MIN_FLOAT8, x), (capi.AGG_MAX_FLOAT8, x), (capi.AGG_SUM_INT4, i), (capi.AGG_MIN_INT4, i),
            (capi.AGG_MAX_INT4, i), (capi.AGG_MAX_DATE, d), (capi.AGG_COUNT_ANY, i)]
    for stage in (capi.AGGSTAGE_NORMAL, capi.AGGSTAGE_PARTIAL):
        agg = capi.make_agg(stage, [k, f], aggs)
        want, wsc, wps, want_x = po.seqscan_agg(scan, agg, p.pool, pages, exact=True)
        for variant in ("interp-priv", "specialised-priv"):          # both must fall to the NULL-tracking transposed kernel
            rows, sc, ps, var = gpu_scanagg(eng, scan, agg, p.pool, pages, variant)
            assert var % 16 == 2 and (sc, ps) == (wsc, wps)
            assert any(r.keyisnull[0] for r in rows) and any(r.keyisnull[1] for r in rows)
            assert_aggrows_match(rows, want, agg, exact=want_x)


def test_empty_and_ragged_relations(eng):
    desc = capi.synth_tupdesc(capi.TAB_LINEITEM_NARROW)
    scan, agg, pool = tpch.q1_plan(capi.TAB_LINEITEM_NARROW)
    # no blocks at all: a hashed aggregate returns no rows, a plain one exactly one row (count 0, sums NULL)
    rows, sc, ps, _ = gpu_scanagg(eng, scan, agg, pool, np.zeros(0, dtype=np.uint8))
    assert rows == [] and sc == 0
    p = ExprPool()
    x = p.var(2, capi.FLOAT8OID)
    plain = capi.make_agg(capi.AGGSTAGE_NORMAL, [], [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_FLOAT8, x), (capi.AGG_AVG_FLOAT8, x)])
    rows, sc, ps, _ = gpu_scanagg(eng, capi.make_scan(desc, -1), plain, p.pool, np.zeros(0, dtype=np.uint8))
    assert len(rows) == 1 and rows[0].agg[0].i == 0 and rows[0].agg[1].isnull and rows[0].agg[2].isnull
    # ragged: 1-row page, an all-zero (new) page, a page with dead and unused line pointers, a full page
    mk = lambda n, base: [[base + j, 1.0 + j, 10.0 * j, 0.05, 0.02, b"AN"[j % 2:j % 2 + 1], b"F", -1000 - j] for j in range(n)]
    p1 = po.build_pages(desc, mk(1, 0))
    p2 = np.zeros(capi.GG_BLCKSZ, dtype=np.uint8)
    p3 = po.build_pages(desc, mk(100, 10))
    lps = p3[24:24 + 400].view(np.uint32)
    lps[5] = (lps[5] & ~np.uint32(3 << 15)) | np.uint32(3 << 15)      # LP_DEAD
    lps[6] = 0                                                      # LP_UNUSED
    lps[7] = (lps[7] & ~np.uint32(3 << 15)) | np.uint32(2 << 15)      # LP_REDIRECT
    p4 = po.build_pages(desc, mk(430, 1000))
    pages = np.concatenate([p1, p2, p3, p4])
    want, wsc, wps, want_x = po.seqscan_agg(scan, agg, pool, pages, exact=True)
    assert wsc == 1 + 97 + 430
    for variant in ("specialised-priv", "interp-priv", "interp-tr"):
        rows, sc, ps, _ = gpu_scanagg(eng, scan, agg, pool, pages, variant)
        assert (sc, ps) == (wsc, wps)
        assert_aggrows_match(rows, want, agg, exact=want_x)


def test_visibility_rules(eng):
    desc = capi.synth_tupdesc(capi.TAB_LINEITEM_NARROW)
    scan, agg, pool = tpch.q1_plan(capi.TAB_LINEITEM_NARROW)
    rows_in = [[j, 2.0, 10.0, 0.0, 0.0, b"A", b"F", -2000] for j in range(50)]
    pg = po.build_pages(desc, rows_in, all_visible=False)
    # frozen tuples on a page without PD_ALL_VISIBLE: visible through the hint bits
    want, wsc, _, want_x = po.seqscan_agg(scan, agg, pool, pg, exact=True)
    rows, sc, ps, _ = gpu_scanagg(eng, scan, agg, pool, pg)
    assert sc == wsc == 50
    assert_aggrows_match(rows, want, agg, exact=want_x)
    # an aborted inserter (HEAP_XMIN_INVALID, not committed): invisible to everyone
    lp = int(pg[24:28].view(np.uint32)[0]) & 0x7FFF
    pg2 = pg.copy()
    pg2[lp + 20:lp + 22].view(np.uint16)[0] = (int(pg2[lp + 20:lp + 22].view(np.uint16)[0]) & ~0x0300) | 0x0200
    rows, sc, ps, _ = gpu_scanagg(eng, scan, agg, pool, pg2)
    assert sc == 49 == po.seqscan_agg(scan, agg, pool, pg2)[1]
    # a tuple whose visibility needs clog/snapshot: refused, like the oracle
    pg3 = pg.copy()
    pg3[lp + 20:lp + 22].view(np.uint16)[0] = int(pg3[lp + 20:lp + 22].view(np.uint16)[0]) & ~0x0300
    with pytest.raises(capi.GGError) as e:
        gpu_scanagg(eng, scan, agg, pool, pg3)
    assert e.value.code == -7
    with pytest.raises(po.OracleError):
        po.seqscan_agg(scan, agg, pool, pg3)


def test_scan_against_a_snapshot(eng):
    """HeapTupleSatisfiesMVCC on the device (tqual.c:997-1238; tests/test_mvcc.py pins the rule to the reference's tqual.o):
    committed / aborted / in-progress inserters and deleters around a snapshot, all-visible pages in between.  Every kernel
    variant and the join / Motion kernels share the front end; here: the specialised, the run-time compiled and the interpreter
    scan over wide and narrow pages."""
    from _util import mvcc_snapshot, stamp_visibility
    snap = mvcc_snapshot()
    for table in (capi.TAB_LINEITEM_NARROW, capi.TAB_LINEITEM_WIDE):
        pages, nb, nr = tpch.synth_generate(tpch.synth_spec(table, 60_000, seed=9))
        pg, vis = stamp_visibility(pages, all_visible_every=4)
        scan, agg, pool = tpch.q1_plan(table)
        po.set_snapshot(snap)
        try:
            want, wsc, wps, want_x = po.seqscan_agg(scan, agg, pool, pg, exact=True)
        finally:
            po.set_snapshot(None)
        assert wsc == sum(vis) and 0 < wsc < nr
        eng.set_snapshot(snap)
        try:
            for variant in ("specialised-priv", "nvrtc-priv", "interp-priv"):
                rows, sc, ps, _ = gpu_scanagg(eng, scan, agg, pool, pg, variant)
                assert (sc, ps) == (wsc, wps), variant
                assert_aggrows_match(rows, want, agg, exact=want_x)
        finally:
            eng.set_snapshot(None)
        with pytest.raises(capi.GGError) as e:                 # the same pages without a snapshot: refused, not guessed
            gpu_scanagg(eng, scan, agg, pool, pg)
        assert e.value.code == -7


def test_more_groups_than_private_accumulators_hold(eng):
    """7 x 3 groups: the private-accumulator kernel overflows and the input is replayed on the transposed kernel."""
    pages, nb, nr = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_WIDE, 120000, seed=5))
    desc = capi.synth_tupdesc(capi.TAB_LINEITEM_WIDE)
    p = ExprPool()
    ln, flag = p.var(4, capi.INT4OID), p.var(9, capi.BPCHAROID)
    price, tax = p.var(6, capi.FLOAT8OID), p.var(8, capi.FLOAT8OID)
    scan = capi.make_scan(desc, p.func(capi.F_INT4GT, capi.BOOLOID, p.var(2, capi.INT4OID), p.const(capi.INT4OID, 100)))
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [ln, flag], [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_FLOAT8, price),
                                                            (capi.AGG_AVG_FLOAT8, p.func(capi.F_FLOAT8MUL, capi.FLOAT8OID, price, tax))])
    want, wsc, wps, want_x = po.seqscan_agg(scan, agg, p.pool, pages, exact=True)
    assert len(want) == 21
    for variant in ("specialised-priv", "nvrtc-priv", "interp-priv"):
        rows, sc, ps, var = gpu_scanagg(eng, scan, agg, p.pool, pages, variant)
        assert var % 16 == 1 and (sc, ps) == (wsc, wps)        # ended on the transposed variant
        assert_aggrows_match(rows, want, agg, exact=want_x)
    # with the planner's estimate the wide variant is chosen up front
    agg.numGroups = 21
    rows, sc, ps, var = gpu_scanagg(eng, scan, agg, p.pool, pages)
    assert var % 16 == 1
    assert_aggrows_match(rows, want, agg, exact=want_x)


def _many_groups_plan(table, num_groups):
    cols = tpch.LI_NARROW_COLS
    desc = capi.synth_tupdesc(table)
    p = ExprPool()
    price = p.var(cols["extendedprice"], capi.FLOAT8OID)
    agg = capi.make_agg(capi.AGGSTAGE_PARTIAL, [p.var(cols["orderkey"], capi.INT8OID)],
                        [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_FLOAT8, price), (capi.AGG_AVG_FLOAT8, p.var(cols["quantity"], capi.FLOAT8OID)),
                         (capi.AGG_MIN_DATE, p.var(cols["shipdate"], capi.DATEOID)), (capi.AGG_MAX_FLOAT8, price)], num_groups=num_groups)
    return capi.make_scan(desc, -1), agg, p


@pytest.mark.parametrize("hint", [0, 60_000])
def test_group_by_with_tens_of_thousands_of_groups(eng, hint):
    """GROUP BY l_orderkey: the general HashAggregate (HBM hash table).  Without a planner estimate the on-chip
    variants overflow first and the input is replayed; with one the table is used from the start."""
    from greengage_b200.engine import Relation, ScanAgg
    pages, nb, nr = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, 200_000, seed=5))
    scan, agg, p = _many_groups_plan(capi.TAB_LINEITEM_NARROW, hint)
    want, sc, ps, want_x = po.seqscan_agg(scan, agg, p.pool, pages, cap=100_000, exact=True)
    assert len(want) > 40_000
    rel = Relation(eng, host_pages=pages)
    sa = ScanAgg(eng, scan, agg, p.pool)
    try:
        half = rel.nblocks // 2
        sa.run(rel, 0, half)                          # two runs accumulate into the same table
        sa.run(rel, half, rel.nblocks - half)
        got, gsc, gps = sa.fetch(cap=100_000)
        assert sa.variant() % 16 == 5                 # the general HashAggregate (plan-specialised or not)
        assert (gsc, gps) == (sc, ps)
        assert_aggrows_match(got, want, agg, exact=want_x)
        with pytest.raises(capi.GGError) as e:        # the caller's buffer is too small: said so, not truncated
            sa.fetch(cap=1000)
        assert e.value.code == -8
    finally:
        sa.free()
        rel.free()


def test_group_table_grows_when_the_estimate_was_low(eng):
    from greengage_b200.engine import Relation, ScanAgg
    pages, nb, nr = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, 600_000, seed=9, norders=400_000))
    scan, agg, p = _many_groups_plan(capi.TAB_LINEITEM_NARROW, 100)          # the planner said 100 groups; there are ~300 k
    want, sc, ps, want_x = po.seqscan_agg(scan, agg, p.pool, pages, cap=500_000, exact=True)
    assert len(want) > 65_536
    with env(GGB200_SCAN_MODE="5"):
        sa = ScanAgg(eng, scan, agg, p.pool)
    rel = Relation(eng, host_pages=pages)
    try:
        sa.run(rel)
        got, gsc, gps = sa.fetch(cap=500_000)
        assert (gsc, gps) == (sc, ps)
        assert_aggrows_match(got, want, agg, exact=want_x)
    finally:
        sa.free()
        rel.free()


def test_nullable_keys_and_int_aggregates_in_the_general_hashagg(eng):
    rng = np.random.default_rng(3)
    desc = make_desc([(capi.INT4OID, 4, "i", 1), (capi.BPCHAROID, -1, "i", 0), (capi.FLOAT8OID, 8, "d", 1), (capi.INT4OID, 4, "i", 1)])
    rows, nulls = [], []
    for i in range(20_000):
        rows.append([int(rng.integers(0, 300)), bytes([65 + int(rng.integers(0, 6))]), float(rng.normal()) * 10, int(rng.integers(-9, 9))])
        nulls.append([rng.random() < 0.05, rng.random() < 0.05, rng.random() < 0.1, rng.random() < 0.1])
    pages = po.build_pages(desc, rows, nulls)
    p = ExprPool()
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [p.var(1, capi.INT4OID), p.var(2, capi.BPCHAROID)],
                        [(capi.AGG_COUNT_STAR, -1), (capi.AGG_COUNT_ANY, p.var(3, capi.FLOAT8OID)), (capi.AGG_SUM_FLOAT8, p.var(3, capi.FLOAT8OID)),
                         (capi.AGG_MIN_FLOAT8, p.var(3, capi.FLOAT8OID)), (capi.AGG_SUM_INT4, p.var(4, capi.INT4OID)),
                         (capi.AGG_MAX_INT4, p.var(4, capi.INT4OID)), (capi.AGG_AVG_FLOAT8, p.var(3, capi.FLOAT8OID))], num_groups=2000)
    scan = capi.make_scan(desc, -1)
    want, sc, ps, want_x = po.seqscan_agg(scan, agg, p.pool, pages, cap=10_000, exact=True)
    from greengage_b200.engine import Relation, ScanAgg
    rel = Relation(eng, host_pages=pages)
    sa = ScanAgg(eng, scan, agg, p.pool)
    try:
        sa.run(rel)
        got, gsc, gps = sa.fetch(cap=10_000)
        assert sa.variant() % 16 == 5 and len(got) == len(want) > 1500
        assert_aggrows_match(got, want, agg, exact=want_x)
    finally:
        sa.free()
        rel.free()


def _f8_relation(values):
    desc = make_desc([(capi.FLOAT8OID, 8, 'd', 1, 1), (capi.FLOAT8OID, 8, 'd', 1, 1)])
    return desc, po.build_pages(desc, [[v, w] for v, w in values])


def test_float_errors_match_reference_semantics(eng):
    p = ExprPool()
    a, b = p.var(1, capi.FLOAT8OID), p.var(2, capi.FLOAT8OID)
    # float8mul overflow inside the expression: "value out of range: overflow"
    desc, pages = _f8_relation([(1.0, 2.0), (1e200, 1e200), (3.0, 4.0)])
    scan = capi.make_scan(desc, -1)
    agg = capi.make_agg(0, [], [(capi.AGG_SUM_FLOAT8, p.func(capi.F_FLOAT8MUL, capi.FLOAT8OID, a, b))])
    for variant in ("specialised-priv", "interp-priv", "interp-tr"):
        with pytest.raises(capi.GGError) as e:
            gpu_scanagg(eng, scan, agg, p.pool, pages, variant)
        assert e.value.code == -2
    with pytest.raises(po.OracleError):
        po.seqscan_agg(scan, agg, p.pool, pages)
    # underflow, division by zero
    desc, pages = _f8_relation([(1e-200, 1e-200)])
    with pytest.raises(capi.GGError) as e:
        gpu_scanagg(eng, capi.make_scan(desc, -1), agg, p.pool, pages)
    assert e.value.code == -3
    desc, pages = _f8_relation([(1.0, 0.0)])
    aggd = capi.make_agg(0, [], [(capi.AGG_SUM_FLOAT8, p.func(capi.F_FLOAT8DIV, capi.FLOAT8OID, a, b))])
    with pytest.raises(capi.GGError) as e:
        gpu_scanagg(eng, capi.make_scan(desc, -1), aggd, p.pool, pages)
    assert e.value.code == -4
    # a sum that overflows although every input is finite is an ERROR (float8pl) ...
    desc, pages = _f8_relation([(1.7e308, 0.0), (1.7e308, 0.0)])
    aggs = capi.make_agg(0, [], [(capi.AGG_SUM_FLOAT8, a)])
    with pytest.raises(capi.GGError) as e:
        gpu_scanagg(eng, capi.make_scan(desc, -1), aggs, p.pool, pages)
    assert e.value.code == -2
    with pytest.raises(po.OracleError):
        po.seqscan_agg(capi.make_scan(desc, -1), aggs, p.pool, pages)
    # ... while an infinite input makes an infinite sum legitimately
    desc, pages = _f8_relation([(float("inf"), 0.0), (1.0, 0.0)])
    rows, _, _, _ = gpu_scanagg(eng, capi.make_scan(desc, -1), aggs, p.pool, pages)
    want, _, _, want_x = po.seqscan_agg(capi.make_scan(desc, -1), aggs, p.pool, pages, exact=True)
    assert rows[0].agg[0].f[0] == want[0].agg[0].f[0] == float("inf")
    assert_aggrows_match(rows, want, aggs, exact=want_x)
    # the overflow ERROR where every summation order agrees on it: required when all inputs share a sign and the sum is past
    # the overflow threshold even after the largest rounding any order can make, absent when no order can reach it.  The
    # exact record comes from sum(v * 2^-16), which cannot overflow (scaling by a power of two is exact here).
    from _util import sum_overflow_rule
    big = 1.7976931348623157e308
    sums16 = capi.make_agg(0, [], [(capi.AGG_SUM_FLOAT8, p.func(capi.F_FLOAT8MUL, capi.FLOAT8OID, a, p.const(capi.FLOAT8OID, 2.0 ** -16)))])
    for vals, rule in (([0.7 * big] * 3, True), ([0.3 * big] * 3, False), ([-0.45 * big, -0.5 * big], False),
                       ([0.7 * big, 0.7 * big, -0.7 * big], None)):
        desc, pages = _f8_relation([(v, 0.0) for v in vals])
        _, _, _, x16 = po.seqscan_agg(capi.make_scan(desc, -1), sums16, p.pool, pages, exact=True)
        assert sum_overflow_rule(x16[0][0], scale_exp=16) is rule, vals
        if rule is None:
            continue                                      # order-dependent: not asserted
        for variant in ("specialised-priv", "interp-tr"):
            if rule:
                with pytest.raises(capi.GGError) as e:
                    gpu_scanagg(eng, capi.make_scan(desc, -1), aggs, p.pool, pages, variant)
                assert e.value.code == -2
            else:
                rows, _, _, _ = gpu_scanagg(eng, capi.make_scan(desc, -1), aggs, p.pool, pages, variant)
                want, _, _, want_x = po.seqscan_agg(capi.make_scan(desc, -1), aggs, p.pool, pages, exact=True)
                assert_aggrows_match(rows, want, aggs, exact=want_x)


def test_filters_and_casts(eng):
    pages, nb, nr = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_WIDE, 60000, seed=9))
    desc = capi.synth_tupdesc(capi.TAB_LINEITEM_WIDE)
    p = ExprPool()
    qty, disc = p.var(5, capi.FLOAT8OID), p.var(7, capi.FLOAT8OID)
    flag, status, ln, okey = p.var(9, capi.BPCHAROID), p.var(10, capi.BPCHAROID), p.var(4, capi.INT4OID), p.var(1, capi.INT8OID)
    shipdate, commitdate = p.var(11, capi.DATEOID), p.var(12, capi.DATEOID)
    q = p.boolop(capi.E_AND,
                 p.boolop(capi.E_OR, p.func(capi.F_BPCHAREQ, capi.BOOLOID, flag, p.const(capi.BPCHAROID, "R ")),
                          p.boolop(capi.E_NOT, p.func(capi.F_BPCHARNE, capi.BOOLOID, status, p.const(capi.BPCHAROID, "O")))),
                 p.boolop(capi.E_AND, p.func(capi.F_FLOAT8LT, capi.BOOLOID, disc, p.const(capi.FLOAT8OID, 0.07)),
                          p.boolop(capi.E_AND, p.func(capi.F_DATE_LT, capi.BOOLOID, shipdate, commitdate),
                                   p.func(capi.F_INT8GT, capi.BOOLOID, okey, p.func(capi.F_INT48, capi.INT8OID, ln)))))
    scan = capi.make_scan(desc, q)
    agg = capi.make_agg(0, [status], [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_FLOAT8, p.func(capi.F_FLOAT8MUL, capi.FLOAT8OID, qty, p.func(capi.F_I4TOD, capi.FLOAT8OID, ln))),
                                      (capi.AGG_SUM_INT4, ln), (capi.AGG_MIN_DATE, shipdate), (capi.AGG_MAX_FLOAT8, qty)])
    want, wsc, wps, want_x = po.seqscan_agg(scan, agg, p.pool, pages, exact=True)
    assert 0 < wps < wsc
    for variant in ("specialised-tr", "interp-tr"):
        rows, sc, ps, _ = gpu_scanagg(eng, scan, agg, p.pool, pages, variant)
        assert (sc, ps) == (wsc, wps)
        assert_aggrows_match(rows, want, agg, exact=want_x)


def test_final_stage_combine(eng):
    from greengage_b200.engine import agg_final
    parts, segs = [], []
    scan, part, pool = tpch.q1_plan(capi.TAB_LINEITEM_NARROW, capi.AGGSTAGE_PARTIAL)
    for s in range(3):
        pages, nb, nr = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, 90000, nsegs=3, seg=s))
        segs.append(pages)
        rows, _, _, _ = gpu_scanagg(eng, scan, part, pool, pages)
        want, _, _, want_x = po.seqscan_agg(scan, part, pool, pages, exact=True)
        assert_aggrows_match(rows, want, part, exact=want_x)
        parts.extend(rows)
    fin = tpch.q1_final_agg(part)
    got = agg_final(eng, fin, parts)
    want = po.agg_final(fin, parts)
    n1, a1, p1 = tpch.q1_plan(capi.TAB_LINEITEM_NARROW)
    assert_aggrows_match(got, want, a1, rel=1e-12)
    # and the device FINAL against the exact record of a one-stage scan of all three segments' pages
    one, _, _, one_x = po.seqscan_agg(n1, a1, p1, np.concatenate(segs), exact=True)
    assert_aggrows_match(got, one, a1, exact=one_x)
    # FINAL over nothing: no groups
    assert agg_final(eng, fin, []) == []


def test_large_relation_properties(eng):
    """2 x 10^7 rows: counts are exact, halves add up to the whole, rows scanned == rows generated."""
    pages, nb, nr = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, 20_000_000, seed=42))
    scan, agg, pool = tpch.q1_plan(capi.TAB_LINEITEM_NARROW)
    whole, sc, ps, _ = gpu_scanagg(eng, scan, agg, pool, pages)
    assert sc == nr == 20_000_000 and sum(r.agg[7].i for r in whole) == ps
    a, _, pa, _ = gpu_scanagg(eng, scan, agg, pool, pages, ranges=[(0, nb // 2)])
    b, _, pb, _ = gpu_scanagg(eng, scan, agg, pool, pages, ranges=[(nb // 2, nb)])
    assert pa + pb == ps
    ka = {(r.key[0], r.key[1]): r for r in a}
    kb = {(r.key[0], r.key[1]): r for r in b}
    for r in whole:
        k = (r.key[0], r.key[1])
        assert ka[k].agg[7].i + kb[k].agg[7].i == r.agg[7].i
        for i in range(4):
            s = ka[k].agg[i].f[0] + kb[k].agg[i].f[0]
            assert abs(s - r.agg[i].f[0]) <= 1e-9 * abs(r.agg[i].f[0])
    # and an answer that does not come from the GPU: the oracle's exact record of the same pages (about 10 s single-threaded)
    want, wsc, wps, want_x = po.seqscan_agg(scan, agg, pool, pages, exact=True)
    assert (wsc, wps) == (sc, ps)
    assert_aggrows_match(whole, want, agg, exact=want_x)


def test_four_byte_varlena_headers_and_alignment_padding(eng):
    """Short strings normally carry 1-byte headers; a 4-byte (big-endian, GPDB) header is aligned like an int with zero
    pad bytes in front — att_align_pointer's peek (tupmacs.h:149) decides per value.  Tuples are crafted byte by byte
    (header copied from a tuple the oracle formed); both header kinds are mixed on one page and followed by an aligned
    float8, so every offset after the string depends on the decision."""
    desc = make_desc([(capi.INT4OID, 4, "i", 1, 1), (capi.BPCHAROID, -1, "i", 0, 1), (capi.FLOAT8OID, 8, "d", 1, 1)])
    rng = np.random.default_rng(17)
    L = po.lib()
    page = np.zeros(capi.GG_BLCKSZ, dtype=np.uint8)
    L.or_page_init(page.ctypes.data)
    L.or_page_set_all_visible(page.ctypes.data)
    n = 0
    for i in range(500):
        a = int(rng.integers(0, 1000))
        s = bytes([65 + int(rng.integers(0, 4))]) + (b"x " if i % 3 == 0 else b"  ")        # char(3), blank padded
        c = float(rng.integers(1, 100)) / 4
        t = bytearray(po.form_tuple(desc, [a, s, c]))
        if i % 2:
            # same row with a 4-byte header: data = int4 | 00 00 00 07 | 3 bytes | pad to 8 | float8
            data = a.to_bytes(4, "little", signed=True) + (7).to_bytes(4, "big") + s + b"\0" * 5 + np.float64(c).tobytes()
            t = t[:24] + data
        tb = (C.c_uint8 * len(t)).from_buffer_copy(bytes(t))
        assert L.or_page_add_item(page.ctypes.data, tb, len(t)) > 0
        n += 1
    p = ExprPool()
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [p.var(2, capi.BPCHAROID)],
                        [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_FLOAT8, p.var(3, capi.FLOAT8OID)), (capi.AGG_SUM_INT4, p.var(1, capi.INT4OID))])
    scan = capi.make_scan(desc, -1)
    want, sc, ps, want_x = po.seqscan_agg(scan, agg, p.pool, page, exact=True)
    assert sc == n and len(want) == 8                      # 4 letters x {"Ax", "A"}
    for variant in ("interp-tr", "specialised-tr"):
        got, gsc, gps, _ = gpu_scanagg(eng, scan, agg, p.pool, page, variant)
        assert (gsc, gps) == (sc, ps)
        assert_aggrows_match(got, want, agg, exact=want_x)


def test_limits_of_the_accelerated_subset(eng):
    """The widest plan the subset allows: a 32-attribute relation (GG_MAX_ATTS), 4 grouping keys (GG_MAX_KEYS) of four
    different types, 16 aggregates (GG_MAX_AGGS) over nullable columns, PARTIAL stage (avg carries its sum of squares)."""
    rng = np.random.default_rng(23)
    spec = []
    for i in range(32):
        spec.append([(capi.INT4OID, 4, "i", 1), (capi.FLOAT8OID, 8, "d", 1), (capi.BPCHAROID, -1, "i", 0), (capi.INT8OID, 8, "d", 1),
                     (capi.DATEOID, 4, "i", 1)][i % 5])
    desc = make_desc(spec)
    rows, nulls = [], []
    for r in range(6000):
        row, nl = [], []
        for i in range(32):
            k = i % 5
            if k == 0: v = int(rng.integers(0, 2)) if i == 0 else int(rng.integers(-1000, 1000))
            elif k == 1: v = float(rng.integers(-500, 500)) / 8
            elif k == 2: v = bytes([65 + int(rng.integers(0, 2))]) + b" " * 3
            elif k == 3: v = int(rng.integers(0, 2)) if i == 3 else int(rng.integers(-10**12, 10**12))
            else: v = int(rng.integers(7000, 7002)) if i == 4 else int(rng.integers(-3000, 9000))
            row.append(v)
            nl.append(bool(rng.random() < 0.07))
        rows.append(row)
        nulls.append(nl)
    pages = po.build_pages(desc, rows, nulls)
    p = ExprPool()
    keys = [p.var(1, capi.INT4OID), p.var(3, capi.BPCHAROID), p.var(4, capi.INT8OID), p.var(5, capi.DATEOID)]
    f = lambda a: p.var(a, capi.FLOAT8OID)
    aggs = [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_FLOAT8, f(2)), (capi.AGG_AVG_FLOAT8, f(7)), (capi.AGG_MIN_FLOAT8, f(12)),
            (capi.AGG_MAX_FLOAT8, f(17)), (capi.AGG_SUM_INT4, p.var(6, capi.INT4OID)), (capi.AGG_MIN_INT4, p.var(11, capi.INT4OID)),
            (capi.AGG_MAX_INT4, p.var(16, capi.INT4OID)), (capi.AGG_MIN_INT8, p.var(9, capi.INT8OID)), (capi.AGG_MAX_INT8, p.var(14, capi.INT8OID)),
            (capi.AGG_MIN_DATE, p.var(10, capi.DATEOID)), (capi.AGG_MAX_DATE, p.var(15, capi.DATEOID)), (capi.AGG_COUNT_ANY, f(22)),
            (capi.AGG_AVG_FLOAT8, f(27)), (capi.AGG_SUM_FLOAT8, p.func(capi.F_FLOAT8MUL, capi.FLOAT8OID, f(32), f(2))),
            (capi.AGG_COUNT_ANY, p.var(31, capi.INT4OID))]
    assert len(aggs) == capi.GG_MAX_AGGS
    agg = capi.make_agg(capi.AGGSTAGE_PARTIAL, keys, aggs, num_groups=81)
    scan = capi.make_scan(desc, -1)
    want, sc, ps, want_x = po.seqscan_agg(scan, agg, p.pool, pages, exact=True)
    assert 30 < len(want) <= 81                              # 3^4 combinations of {value, value, NULL}
    got, gsc, gps, var = gpu_scanagg(eng, scan, agg, p.pool, pages)
    assert (gsc, gps) == (sc, ps)
    assert_aggrows_match(got, want, agg, exact=want_x)
    agg.numGroups = 0                                        # no planner estimate: the on-chip variants overflow, then the HBM table
    got2, _, _, var2 = gpu_scanagg(eng, scan, agg, p.pool, pages)
    assert_aggrows_match(got2, want, agg, exact=want_x)


def test_plain_aggregate_on_the_general_hashagg(eng):
    """numCols == 0 with a planner estimate that sends the plan to the HBM group table: the single group's entry has no
    key words (found by the randomised join test)."""
    pages, nb, nr = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, 80_000, seed=2))
    c = tpch.LI_NARROW_COLS
    p = ExprPool()
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [], [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_FLOAT8, p.var(c["quantity"], capi.FLOAT8OID)),
                                                   (capi.AGG_MIN_DATE, p.var(c["shipdate"], capi.DATEOID))], num_groups=500)
    scan = capi.make_scan(capi.synth_tupdesc(capi.TAB_LINEITEM_NARROW), -1)
    want, sc, ps, want_x = po.seqscan_agg(scan, agg, p.pool, pages, exact=True)
    got, gsc, gps, var = gpu_scanagg(eng, scan, agg, p.pool, pages)
    assert var % 16 == 5 and (gsc, gps) == (sc, ps) and len(got) == 1
    assert_aggrows_match(got, want, agg, exact=want_x)
