"""Size-independent properties at 10^7 rows: the answers of the GPU path must be consistent with themselves and with what
the generator knows — row counts, range additivity (bit-identical), one-stage == two-stage aggregation, join cardinality
identities, sortedness — and Q1 must be within the proven rounding bound of the oracle's exact sums over the same pages."""
import numpy as np
import pytest

from _util import assert_aggrows_match
from greengage_b200 import capi, tpch

pytestmark = pytest.mark.gpu
N = 10_000_000


@pytest.fixture(scope="module")
def eng():
    from greengage_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def lineitem(eng):
    from greengage_b200.engine import Relation
    pages, nb, nr = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, N, seed=21, norders=N // 4))
    rel = Relation(eng, host_pages=pages)
    yield rel, nb, nr, pages
    rel.free()


@pytest.fixture(scope="module")
def q1_exact(lineitem):
    """the oracle's Q1 over the same pages with its exact record: an answer that does not come from the GPU (about 5 s)"""
    from oracle import pyoracle as po
    scan, agg, pool = tpch.q1_plan(capi.TAB_LINEITEM_NARROW, capi.AGGSTAGE_NORMAL)
    want, sc, ps, want_x = po.seqscan_agg(scan, agg, pool, lineitem[3], exact=True)
    return want, sc, ps, want_x


def run_q1(eng, rel, stage, ranges):
    from greengage_b200.engine import ScanAgg
    scan, agg, pool = tpch.q1_plan(capi.TAB_LINEITEM_NARROW, stage)
    sa = ScanAgg(eng, scan, agg, pool)
    try:
        for a, b in ranges:
            sa.run(rel, a, b - a)
        rows, sc, ps = sa.fetch()
        return rows, sc, ps, agg
    finally:
        sa.free()


def test_counts_and_range_additivity(eng, lineitem, q1_exact):
    rel, nb, nr, _ = lineitem
    whole, sc, ps, agg = run_q1(eng, rel, capi.AGGSTAGE_NORMAL, [(0, nb)])
    assert sc == nr and sum(r.agg[7].i for r in whole) == ps and 0 < ps <= nr
    want, wsc, wps, want_x = q1_exact
    assert (wsc, wps) == (sc, ps)
    assert_aggrows_match(whole, want, agg, exact=want_x)
    again, sc2, ps2, _ = run_q1(eng, rel, capi.AGGSTAGE_NORMAL, [(0, nb)])
    assert [bytes(r) for r in sorted(again, key=lambda r: (r.key[0], r.key[1]))] == \
           [bytes(r) for r in sorted(whole, key=lambda r: (r.key[0], r.key[1]))]          # run to run: bit-identical
    parts, sc3, ps3, _ = run_q1(eng, rel, capi.AGGSTAGE_NORMAL, [(0, nb // 3), (nb // 3, nb // 2), (nb // 2, nb)])
    assert (sc3, ps3) == (sc, ps)
    assert_aggrows_match(parts, whole, agg, rel=1e-12)                                   # fed in pieces: same sums
    assert_aggrows_match(parts, want, agg, exact=want_x)


def test_two_stage_equals_one_stage(eng, lineitem, q1_exact):
    from greengage_b200.engine import agg_final
    rel, nb, nr, _ = lineitem
    whole, sc, ps, agg = run_q1(eng, rel, capi.AGGSTAGE_NORMAL, [(0, nb)])
    partial_rows = []
    cuts = [0, nb // 4, nb // 2, nb]
    for a, b in zip(cuts[:-1], cuts[1:]):                                                 # three "segments"
        rows, _, _, pagg = run_q1(eng, rel, capi.AGGSTAGE_PARTIAL, [(a, b)])
        partial_rows += rows
    final = agg_final(eng, tpch.q1_final_agg(pagg), partial_rows)
    assert_aggrows_match(final, whole, agg, rel=1e-12)
    assert_aggrows_match(final, q1_exact[0], agg, exact=q1_exact[3])                       # one tree over the same inputs


def test_join_cardinality_identities(eng, lineitem):
    """inner + anti = outer rows; left = inner + anti; semi + anti = outer rows (orders has unique keys)."""
    from greengage_b200.engine import JoinAgg, Relation
    rel, nb, nr, _ = lineitem
    od, _, nod = tpch.synth_generate(tpch.synth_spec(capi.TAB_ORDERS, (N // 4) * 3 // 4, seed=21))       # a quarter of the orders are missing
    orel = Relation(eng, host_pages=od)
    counts = {}
    try:
        for name, jt in (("inner", capi.JOIN_INNER), ("left", capi.JOIN_LEFT), ("semi", capi.JOIN_SEMI), ("anti", capi.JOIN_ANTI)):
            outer, inner, hj, agg, pool = tpch.join_plan(capi.TAB_LINEITEM_NARROW, "count", jt)
            ja = JoinAgg(eng, outer, inner, hj, agg, pool)
            try:
                ja.build(orel)
                ja.probe(rel)
                rows, nj = ja.fetch()
                assert len(rows) == 1 and rows[0].agg[0].i == nj
                assert ja.stats()["rows_built"] == nod
                counts[name] = nj
            finally:
                ja.free()
    finally:
        orel.free()
    assert 0 < counts["anti"] < nr
    assert counts["inner"] + counts["anti"] == nr
    assert counts["left"] == nr
    assert counts["semi"] == counts["inner"]


def test_sorted_at_scale(eng):
    from greengage_b200.engine import sort_rows
    rng = np.random.default_rng(5)
    rows = np.stack([rng.integers(0, 1000, N // 2), rng.normal(size=N // 2).view(np.int64)], axis=1).astype(np.int64)
    keys = [capi.make_sortkey(0, capi.INT8OID, desc=True), capi.make_sortkey(1, capi.FLOAT8OID)]
    perm = sort_rows(eng, keys, rows).astype(np.int64)
    assert np.array_equal(np.sort(perm), np.arange(N // 2))
    k0 = rows[perm, 0]
    k1 = rows[perm, 1].view(np.float64)
    assert np.all(np.diff(k0) <= 0)
    same = np.diff(k0) == 0
    assert np.all(np.diff(k1)[same] >= 0)
