"""GPU parity tests for the sending side of a Redistribute Motion (gg_motion_partition) and for operators
that consume the rows a Motion delivers (GG_FMT_DATUMROWS), through the C-ABI.
Oracle: or_motion_route (evalHashKey + cdbhash + jump consistent hash, pinned against the reference's own
cdbhash.o / hashfunc.o in tests/test_oracle_hash.py) for placement — bit-exact; the heap-page answers of the
oracle's scan/agg/join for what the consumers compute from the redistributed rows."""
import ctypes as C

import numpy as np
import pytest

from _util import assert_aggrows_match, make_desc
from greengage_b200 import capi, tpch
from greengage_b200.capi import ExprPool
from oracle import pyoracle as po

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from greengage_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


class DevBuf:
    """device scratch of `nwords` 64-bit words (+ slack), readable back as numpy"""

    def __init__(self, eng, nwords):
        from greengage_b200.engine import Relation
        self.nwords = nwords
        self.rel = Relation(eng, nblocks=(nwords * 8 + 64 + capi.GG_BLCKSZ - 1) // capi.GG_BLCKSZ)
        self.ptr = self.rel.device_ptr()

    def read(self):
        return self.rel.read().view(np.int64)[:self.nwords]

    def free(self):
        self.rel.free()


def partition(eng, scan, pool, hashkeys, payload, nsegs, pages, cap_total):
    from greengage_b200.engine import Relation, motion_partition
    rel = Relation(eng, host_pages=pages)
    W = 1 + len(payload)
    buf = DevBuf(eng, cap_total * W)
    try:
        counts, offs = motion_partition(eng, scan, pool.pool, hashkeys, payload, nsegs, rel, buf.ptr, cap_total)
        words = buf.read().reshape(-1, W)
        return counts, offs, words, buf
    finally:
        rel.free()


def li_motion_nodes():
    desc = capi.synth_tupdesc(capi.TAB_LINEITEM_NARROW)
    c = tpch.LI_NARROW_COLS
    p = ExprPool()
    key = p.var(c["orderkey"], capi.INT8OID)
    payload = [key, p.var(c["quantity"], capi.FLOAT8OID), p.var(c["extendedprice"], capi.FLOAT8OID),
               p.var(c["discount"], capi.FLOAT8OID), p.var(c["tax"], capi.FLOAT8OID),
               p.var(c["returnflag"], capi.BPCHAROID), p.var(c["linestatus"], capi.BPCHAROID), p.var(c["shipdate"], capi.DATEOID)]
    types = [capi.INT8OID, capi.FLOAT8OID, capi.FLOAT8OID, capi.FLOAT8OID, capi.FLOAT8OID, capi.BPCHAROID, capi.BPCHAROID, capi.DATEOID]
    return desc, p, key, payload, types


@pytest.mark.parametrize("nsegs", [1, 3, 8])
def test_redistribute_placement_is_bit_exact(eng, nsegs):
    li, _, nli = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, 120_000, seed=11))
    desc, p, key, payload, types = li_motion_nodes()
    scan = capi.make_scan(desc, -1)
    cap = 2 * ((nli // nsegs) * 2 + 1024) * nsegs
    counts, offs, words, buf = partition(eng, scan, p, [key], payload, nsegs, li, cap)
    try:
        dest = po.motion_route(scan, p.pool, [key], nsegs, li)
        # whether warps claim rows one at a time or a window at a time depends on the region size per warp of this GPU;
        # windows leave dead slots (mask bit 63), which are not rows
        DEAD = np.int64(-2**63)
        live = [words[offs[d]:offs[d] + counts[d]] for d in range(nsegs)]
        live = [reg[(reg[:, 0] & DEAD) == 0] for reg in live]
        assert len(dest) == nli and sum(len(reg) for reg in live) == nli
        assert [len(reg) for reg in live] == np.bincount(dest, minlength=nsegs).tolist()
        # every delivered row sits in the region of the segment the reference would send it to, and the multiset
        # of rows is the relation's: compare the distribution keys region by region
        for d in range(nsegs):
            reg = live[d]
            assert np.all(reg[:, 0] == 0)                                   # no NULLs in synthetic lineitem
            t = (C.c_int32 * 1)(capi.INT8OID)
            ln = (C.c_int32 * 1)(8)
            nn = (C.c_int32 * 1)(0)
            for k in reg[::97, 1]:                                          # a sample through the oracle's router
                v = (C.c_int64 * 1)(int(k))
                assert po.lib().or_route_datums(t, v, ln, nn, 1, nsegs) == d
    finally:
        buf.free()


def test_null_keys_qual_and_null_payload(eng):
    """NULL distribution keys hash as if absent (cdbhash.c:215), the scan qual filters before routing, NULL
    columns travel as mask bits."""
    rng = np.random.default_rng(2)
    desc = make_desc([(capi.INT4OID, 4, "i", 1), (capi.BPCHAROID, -1, "i", 0), (capi.FLOAT8OID, 8, "d", 1)])
    rows, nulls = [], []
    for i in range(3000):
        rows.append([int(rng.integers(-100, 100)), bytes([65 + int(rng.integers(0, 5))]), float(rng.integers(0, 100))])
        nulls.append([rng.random() < 0.2, rng.random() < 0.2, rng.random() < 0.3])
    pages = po.build_pages(desc, rows, nulls)
    p = ExprPool()
    k0, k1, v = p.var(1, capi.INT4OID), p.var(2, capi.BPCHAROID), p.var(3, capi.FLOAT8OID)
    qual = p.func(capi.F_INT4GT, capi.BOOLOID, k0, p.const(capi.INT4OID, -50))
    scan = capi.make_scan(desc, qual)
    nsegs = 5
    counts, offs, words, buf = partition(eng, scan, p, [k0, k1], [k0, k1, v], nsegs, pages, 4000 * nsegs)
    try:
        dest = po.motion_route(scan, p.pool, [k0, k1], nsegs, pages)
        assert counts == np.bincount(dest, minlength=nsegs).tolist()
        want = {d: [] for d in range(nsegs)}
        passing = [(r, n) for r, n in zip(rows, nulls) if not n[0] and r[0] > -50]
        assert len(passing) == len(dest)
        for (r, n), d in zip(passing, dest):
            mask = (2 if n[1] else 0) | (4 if n[2] else 0)
            want[int(d)].append((mask, r[0], 0 if n[1] else r[1][0], 0 if n[2] else np.float64(r[2]).view(np.int64).item()))
        for d in range(nsegs):
            got = sorted(tuple(int(x) for x in w) for w in words[offs[d]:offs[d] + counts[d]])
            assert got == sorted(want[d])
    finally:
        buf.free()


def test_region_overflow_is_reported(eng):
    li, _, nli = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, 20_000, seed=1))
    desc, p, key, payload, types = li_motion_nodes()
    with pytest.raises(capi.GGError) as e:
        partition(eng, capi.make_scan(desc, -1), p, [key], payload, 4, li, 4 * 1000)
    assert e.value.code == -8


def test_q1_over_redistributed_rows(eng):
    """SeqScan -> Agg over datum rows = the answer over the heap pages they came from."""
    from greengage_b200.engine import RowRelation, ScanAgg
    li, _, nli = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, 150_000, seed=5))
    desc, p, key, payload, types = li_motion_nodes()
    counts, offs, words, buf = partition(eng, capi.make_scan(desc, -1), p, [key], payload, 1, li, 2 * nli + 1024)
    try:
        assert counts == [nli]
        rdesc = capi.rows_tupdesc(types, notnull=[1] * len(types))
        cols = dict(orderkey=1, quantity=2, extendedprice=3, discount=4, tax=5, returnflag=6, linestatus=7, shipdate=8)
        scan_r, agg_r, pool_r = tpch.q1_plan(stage=capi.AGGSTAGE_NORMAL, desc=rdesc, cols=cols)
        scan_h, agg_h, pool_h = tpch.q1_plan(capi.TAB_LINEITEM_NARROW)
        want, sc, ps, want_x = po.seqscan_agg(scan_h, agg_h, pool_h, li, exact=True)
        rel = RowRelation(eng, buf.ptr, nli, len(types))
        sa = ScanAgg(eng, scan_r, agg_r, pool_r)
        try:
            sa.run(rel)
            got, gsc, gps = sa.fetch()
        finally:
            sa.free()
            rel.free()
        assert (gsc, gps) == (sc, ps)
        assert_aggrows_match(got, want, agg_h, exact=want_x)
    finally:
        buf.free()


@pytest.mark.parametrize("jointype", [capi.JOIN_INNER, capi.JOIN_LEFT])
def test_join_over_redistributed_rows(eng, jointype):
    """Redistribute both sides on the join key, then HashJoin -> Agg over what arrived (BASELINE config 3 on one
    segment): every destination joins its share; the shares' partial results combine to the heap-page answer."""
    from greengage_b200.engine import JoinAgg, RowRelation
    li, _, nli = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, 200_000, seed=8, norders=40_000))
    od, _, nod = tpch.synth_generate(tpch.synth_spec(capi.TAB_ORDERS, 30_000, seed=8))
    nsegs = 3
    ldesc, lp, lkey, lpayload, ltypes = li_motion_nodes()
    odesc = capi.synth_tupdesc(capi.TAB_ORDERS)
    op = ExprPool()
    okey = op.var(tpch.ORDERS_COLS["orderkey"], capi.INT8OID)
    opayload = [okey, op.var(tpch.ORDERS_COLS["orderdate"], capi.DATEOID), op.var(tpch.ORDERS_COLS["orderstatus"], capi.BPCHAROID)]
    otypes = [capi.INT8OID, capi.DATEOID, capi.BPCHAROID]
    lc, lo, lw, lbuf = partition(eng, capi.make_scan(ldesc, -1), lp, [lkey], lpayload, nsegs, li, 2 * (nli // nsegs + 4096) * nsegs)
    oc, oo, ow, obuf = partition(eng, capi.make_scan(odesc, -1), op, [okey], opayload, nsegs, od, 2 * (nod // nsegs + 4096) * nsegs)
    try:
        lrd = capi.rows_tupdesc(ltypes, notnull=[1] * len(ltypes))
        ord_ = capi.rows_tupdesc(otypes, notnull=[1] * len(otypes))
        li_cols = dict(orderkey=1, quantity=2, extendedprice=3, discount=4, tax=5, returnflag=6, linestatus=7, shipdate=8)
        ord_cols = dict(orderkey=1, orderdate=2, orderstatus=3)
        outer_r, inner_r, hj_r, agg_r, pool_r = tpch.join_plan(kind="q3ish", jointype=jointype, li_desc=lrd, ord_desc=ord_,
                                                               li_cols=li_cols, ord_cols=ord_cols)
        outer_h, inner_h, hj_h, agg_h, pool_h = tpch.join_plan(capi.TAB_LINEITEM_NARROW, "q3ish", jointype)
        want, nj_want, want_x = po.hashjoin_agg(outer_h, inner_h, hj_h, agg_h, pool_h, li, od, exact=True)
        parts, nj = [], 0
        Wl, Wo = 1 + len(ltypes), 1 + len(otypes)
        for d in range(nsegs):
            lrel = RowRelation(eng, lbuf.ptr + lo[d] * Wl * 8, lc[d], len(ltypes))
            orel = RowRelation(eng, obuf.ptr + oo[d] * Wo * 8, oc[d], len(otypes))
            ja = JoinAgg(eng, outer_r, inner_r, hj_r, agg_r, pool_r)
            try:
                ja.build(orel)
                ja.probe(lrel)
                rows, n = ja.fetch()
            finally:
                ja.free(); lrel.free(); orel.free()
            parts.append(rows)
            nj += n
        assert nj == nj_want
        # combine the per-destination results: count / sum / min are their own combine functions here
        merged = {}
        for rows in parts:
            for r in rows:
                k = (r.key[0], r.keyisnull[0])
                m = merged.setdefault(k, [0, None, None])
                m[0] += r.agg[0].i
                if not r.agg[1].isnull:                   # float8pl's combine: the first partial sum as it is
                    m[1] = r.agg[1].f[0] if m[1] is None else m[1] + r.agg[1].f[0]
                if not r.agg[2].isnull:
                    m[2] = r.agg[2].i if m[2] is None else min(m[2], r.agg[2].i)
        assert len(merged) == len(want)
        got = []
        for r in want:
            m = merged[(r.key[0], r.keyisnull[0])]
            g = capi.gg_aggrow.from_buffer_copy(bytes(r))
            g.agg[0].i = m[0]
            g.agg[1].isnull, g.agg[1].f[0] = m[1] is None, 0.0 if m[1] is None else m[1]
            g.agg[2].isnull, g.agg[2].i = m[2] is None, 0 if m[2] is None else m[2]
            got.append(g)
        # the per-destination sums added up: one more level of the same summation tree, same bound
        assert_aggrows_match(got, want, agg_h, exact=want_x)
    finally:
        lbuf.free(); obuf.free()


@pytest.mark.parametrize("nsegs,window", [(1, 256), (3, 64), (8, 32)])
def test_windowed_claims_leave_dead_slots_that_every_consumer_skips(eng, monkeypatch, nsegs, window):
    """Large inputs: a warp claims rows of a region a window at a time (one atomic on the region cursor per window instead of
    one per 32 rows); what it claimed and did not fill is marked dead (mask bit 63).  The live rows of every region are exactly
    the rows the reference routes there, and a scan over a region (Q1 here) sees only them."""
    from greengage_b200.engine import RowRelation, ScanAgg
    monkeypatch.setenv("GGB200_MOTION_WINDOW", str(window))
    li, _, nli = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, 150_000, seed=13))
    desc, p, key, payload, types = li_motion_nodes()
    scan = capi.make_scan(desc, -1)
    cap = (nli // nsegs + 2200 * window + 4096) * nsegs           # room for every warp's unused tail
    counts, offs, words, buf = partition(eng, scan, p, [key], payload, nsegs, li, cap)
    try:
        dest = po.motion_route(scan, p.pool, [key], nsegs, li)
        want_counts = np.bincount(dest, minlength=nsegs)
        DEAD = np.int64(-2**63)
        total_dead = 0
        for d in range(nsegs):
            reg = words[offs[d]:offs[d] + counts[d]]
            dead = (reg[:, 0] & DEAD) != 0
            total_dead += int(dead.sum())
            assert int((~dead).sum()) == int(want_counts[d])
            assert np.all(reg[~dead, 0] == 0)
        assert total_dead > 0                                       # the path under test was taken
        # a consumer over one region: the same Q1 as over the heap pages of exactly the rows routed there
        d = nsegs - 1
        names = dict(orderkey=1, quantity=2, extendedprice=3, discount=4, tax=5, returnflag=6, linestatus=7, shipdate=8)
        rdesc = capi.rows_tupdesc(types, notnull=[1] * len(types))
        rscan, ragg, rpool = tpch.q1_plan(capi.TAB_LINEITEM_NARROW, desc=rdesc, cols=names)
        rows_rel = RowRelation(eng, buf.ptr + offs[d] * (1 + len(payload)) * 8, counts[d], len(payload))
        sa = ScanAgg(eng, rscan, ragg, rpool)
        sa.run(rows_rel)
        got, scanned, passed = sa.fetch()
        sa.free()
        rows_rel.free()
        assert scanned == int(want_counts[d])
        hscan, hagg, hpool = tpch.q1_plan(capi.TAB_LINEITEM_NARROW)
        whole, _, _ = po.seqscan_agg(hscan, hagg, hpool, li)
        assert sum(r.agg[7].i for r in got) <= sum(r.agg[7].i for r in whole)
        # exact check: recompute Q1 on the host from the live rows of the region
        reg = words[offs[d]:offs[d] + counts[d]]
        reg = reg[(reg[:, 0] & DEAD) == 0]
        cutoff = tpch.D_1998_12_01 - 90
        sel = reg[reg[:, 8].astype(np.int64) <= cutoff]
        for r in got:
            m = (sel[:, 6] == r.key[0]) & (sel[:, 7] == r.key[1])
            assert int(m.sum()) == r.agg[7].i
            q = sel[m, 2].view(np.float64)
            assert abs(q.sum() - r.agg[0].f[0]) <= 1e-9 * abs(q.sum())
    finally:
        buf.free()
