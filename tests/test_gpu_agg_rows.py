"""An Agg's groups finalised on the device into datum rows (gg_scanagg_datumrows / gg_joinagg_datumrows / gg_groups_datumrows)
and the executor path that uses them: a Sort or a Limit directly over an Agg sorts / windows the rows where they are.

ABI: the rows equal what *_fetch returns, word for word — in the same order for merged group records and group sets, as the same
multiset from the general HashAggregate's table — for every non-numeric aggregate, NULL and string keys, float8 edge values and
every kernel variant; errors are fetch's.  Node surface: Limit <- Sort <- Agg over a SeqScan, a HashJoin and the two-stage plan
against a host sort of the same Agg's rows under a total order; the host fallbacks; more than 2^24 groups."""
import struct

import numpy as np
import pytest

from greengage_b200 import capi, executor as ex, tpch
from greengage_b200.capi import ExprPool

pytestmark = pytest.mark.gpu

AGGVAL = np.dtype([("f", "<f8", 3), ("i", "<i8"), ("isnull", "<i4"), ("pad", "<i4")])
AGGROW = np.dtype([("key", "<i8", 4), ("keylen", "<i4", 4), ("keyisnull", "<i4", 4), ("agg", AGGVAL, 16)])
FLOAT_RESULTS = (capi.AGG_SUM_FLOAT8, capi.AGG_AVG_FLOAT8, capi.AGG_MIN_FLOAT8, capi.AGG_MAX_FLOAT8)
HASH = 5                                                     # gg_scanagg_variant & 15 of the general HashAggregate


@pytest.fixture(scope="module")
def eng():
    from greengage_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def aggrow_words(buf, n, agg):
    """gg_aggrow[] (fetch_raw's bytes) -> uint64 [n][1 + numCols + numAggs]: what a datum row of the group holds"""
    a = np.frombuffer(buf, dtype=AGGROW, count=n)
    nk, na = agg.numCols, agg.numAggs
    out = np.zeros((n, 1 + nk + na), dtype=np.uint64)
    mask = np.zeros(n, dtype=np.uint64)
    for c in range(nk):
        out[:, 1 + c] = a["key"][:, c].view(np.uint64)
        mask |= (a["keyisnull"][:, c] != 0).astype(np.uint64) << np.uint64(c)
    for i in range(na):
        v = a["agg"][:, i]
        out[:, 1 + nk + i] = (v["f"][:, 0].view(np.uint64) if agg.aggs[i].aggfnoid in FLOAT_RESULTS else v["i"].view(np.uint64))
        mask |= (v["isnull"] != 0).astype(np.uint64) << np.uint64(nk + i)
    out[:, 0] = mask
    return out


def datum_words(vals, nulls):
    n, ncols = vals.shape
    out = np.zeros((n, 1 + ncols), dtype=np.uint64)
    out[:, 1:] = vals.view(np.uint64)
    out[:, 0] = (nulls.astype(np.uint64) << np.arange(ncols, dtype=np.uint64)).sum(axis=1, dtype=np.uint64) if ncols else 0
    return out


def as_multiset(words):
    return words[np.lexsort(words.T[::-1])] if len(words) else words


def load_rows(eng, vals, nulls):
    """datum rows (int64 [n][ncols] + NULL flags) resident on the device: (owning Relation, RowRelation)"""
    from greengage_b200.engine import Relation, RowRelation
    n, ncols = vals.shape
    W = 1 + ncols
    nb = (n * W * 8 + 16 + capi.GG_BLCKSZ - 1) // capi.GG_BLCKSZ
    buf = np.zeros(nb * capi.GG_BLCKSZ // 8, dtype=np.uint64)
    buf[:n * W].reshape(n, W)[:] = datum_words(vals, nulls)
    rel = Relation(eng, nblocks=nb)
    rel.load(0, buf.view(np.uint8))
    return rel, RowRelation(eng, rel.device_ptr(), n, ncols)


# ---- the relation: k1 int4 (NULLs), k2 bpchar (NULLs), k3 int8, f float8 (NULLs, edges), i int4 (NULLs), d date, g int8 ----
TYPES = [capi.INT4OID, capi.BPCHAROID, capi.INT8OID, capi.FLOAT8OID, capi.INT4OID, capi.DATEOID, capi.INT8OID]


def make_data(n, ngroups3, seed, nullable=True):
    rng = np.random.default_rng(seed)
    vals = np.zeros((n, 7), dtype=np.int64)
    nulls = np.zeros((n, 7), dtype=bool)
    vals[:, 0] = rng.integers(0, 3, n)
    strs = np.array([int.from_bytes(s, "little") for s in (b"A", b"BB", b"CCC", b"DDDDDDDD")], dtype=np.int64)
    vals[:, 1] = strs[rng.integers(0, 4, n)]
    vals[:, 2] = rng.integers(0, ngroups3, n) * 7919 - 10**9
    f = rng.integers(-40, 40, n).astype(np.float64) / 4
    special = rng.random(n)
    f[special < 0.01] = -0.0
    f[(special >= 0.01) & (special < 0.013)] = np.inf
    f[(special >= 0.013) & (special < 0.016)] = -np.inf
    f[(special >= 0.016) & (special < 0.018)] = np.nan
    vals[:, 3] = f.view(np.int64)
    vals[:, 4] = rng.integers(-10**6, 10**6, n)
    vals[:, 5] = rng.integers(-4000, 4000, n)
    vals[:, 6] = rng.integers(-10**15, 10**15, n)
    if nullable:
        for c, p in ((0, 0.05), (1, 0.05), (3, 0.1), (4, 0.1)):
            nulls[:, c] = rng.random(n) < p
        vals[nulls] = 0
    # a group whose inputs are all NULL, and one whose float sum is -0
    vals[:4, 0], vals[:4, 1], vals[:4, 2] = 99, strs[0], 5
    if nullable:
        nulls[:2, 3] = nulls[:2, 4] = True
    vals[2:4, 3] = np.float64(-0.0).view(np.int64)
    nulls[:4, :3] = False
    return vals, nulls


def full_agg(p, keys, num_groups, stage=capi.AGGSTAGE_NORMAL):
    f, i, d, g = p.var(4, capi.FLOAT8OID), p.var(5, capi.INT4OID), p.var(6, capi.DATEOID), p.var(7, capi.INT8OID)
    aggs = [(capi.AGG_COUNT_STAR, -1), (capi.AGG_COUNT_ANY, f), (capi.AGG_SUM_FLOAT8, f), (capi.AGG_AVG_FLOAT8, f),
            (capi.AGG_MIN_FLOAT8, f), (capi.AGG_MAX_FLOAT8, f), (capi.AGG_SUM_INT4, i), (capi.AGG_MIN_INT4, i),
            (capi.AGG_MAX_INT4, i), (capi.AGG_MIN_DATE, d), (capi.AGG_MAX_DATE, d), (capi.AGG_MIN_INT8, g), (capi.AGG_MAX_INT8, g)]
    return capi.make_agg(stage, keys, aggs, num_groups=num_groups)


def key_exprs(p, which):
    return {"none": [], "small": [p.var(1, capi.INT4OID), p.var(2, capi.BPCHAROID)],
            "many": [p.var(3, capi.INT8OID), p.var(1, capi.INT4OID)], "tiny": [p.var(2, capi.BPCHAROID)]}[which]


def fetch_words(pipe, agg, cap):
    buf, n, _, _ = pipe.fetch_raw(cap)
    return aggrow_words(buf.tobytes(), n, agg)


# keys, groups of k3, numGroups, rows, NOT NULL inputs: the private-accumulator, transposed, HashAggregate variants, the
# escalation from a block table into the hash table and the hash table's growth (65 536 slots -> x 8)
VARIANTS = {
    "priv": ("tiny", 1, 0, 20000, False),
    "trn": ("tiny", 1, 0, 20000, True),
    "plain": ("none", 1, 0, 5000, True),
    "escalate": ("many", 3000, 0, 40000, True),
    "hash": ("many", 20000, 50000, 100000, True),
    "growth": ("many", 150000, 20000, 400000, True),
}


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_scanagg_datumrows_equal_fetch(eng, variant):
    from greengage_b200.engine import ScanAgg
    keys, g3, ng, n, nullable = VARIANTS[variant]
    vals, nulls = make_data(n, g3, seed=len(variant), nullable=nullable)
    rel, rows = load_rows(eng, vals, nulls)
    p = ExprPool()
    agg = full_agg(p, key_exprs(p, keys), ng)
    scan = capi.make_scan(capi.rows_tupdesc(TYPES, notnull=None if nullable else [1] * 7), -1)
    b = ScanAgg(eng, scan, agg, p.pool)
    try:
        b.run(rows)
        got = datum_words(*b.datumrows())
        want = fetch_words(b, agg, 400000)                     # the same settled state, read the old way
        assert len(want) > 0 and got.shape == want.shape
        if b.variant() & 15 == HASH:
            assert variant in ("escalate", "hash", "growth")
            assert np.array_equal(as_multiset(got), as_multiset(want))
        else:
            assert variant in ("priv", "trn", "plain")
            assert np.array_equal(got, want)                      # record order: fetch's
        # the view is kept until the reset; a reset and a second run give the same rows (but for the sign of a zero min / max of
        # a group with zeros of both signs, which the HashAggregate's atomics leave to the order they ran in)
        assert np.array_equal(datum_words(*b.datumrows()), got)
        b.reset()
        b.run(rows)
        again = datum_words(*b.datumrows())
        for w in (got, again):
            for col in (1 + agg.numCols + 4, 1 + agg.numCols + 5):
                w[w[:, col] == np.uint64(1 << 63), col] = 0
        assert np.array_equal(as_multiset(again), as_multiset(got))
    finally:
        b.free(); rows.free(); rel.free()


def test_plain_agg_over_no_rows_gives_one_row(eng):
    from greengage_b200.engine import ScanAgg
    vals, nulls = make_data(1000, 1, seed=3)
    rel, rows = load_rows(eng, vals, nulls)
    p = ExprPool()
    agg = full_agg(p, [], 0)
    never = p.func(capi.F_INT4LT, capi.BOOLOID, p.var(1, capi.INT4OID), p.const(capi.INT4OID, -100))
    sa = ScanAgg(eng, capi.make_scan(capi.rows_tupdesc(TYPES), never), agg, p.pool)
    try:
        sa.run(rows)
        v, nl = sa.datumrows()
        assert v.shape == (1, agg.numAggs) and v[0, 0] == 0 and v[0, 1] == 0 and nl[0].tolist() == [False, False] + [True] * 11
        assert np.array_equal(datum_words(v, nl), fetch_words(sa, agg, 4))
    finally:
        sa.free(); rows.free(); rel.free()


def test_stage_and_numeric_refusals(eng):
    from greengage_b200.engine import ScanAgg
    vals, nulls = make_data(1000, 1, seed=4)
    rel, rows = load_rows(eng, vals, nulls)
    p = ExprPool()
    scan = capi.make_scan(capi.rows_tupdesc(TYPES), -1)
    part = ScanAgg(eng, scan, full_agg(p, key_exprs(p, "small"), 0, capi.AGGSTAGE_PARTIAL), p.pool)
    try:
        part.run(rows)
        with pytest.raises(capi.GGError) as e:
            part.datumrows()
        assert e.value.code == -6
    finally:
        part.free(); rows.free(); rel.free()


# ---- errors: fetch's code and message, at the ABI and through a Sort over the Agg ----
def _error_plan(p, kind):
    a, b = p.var(1, capi.FLOAT8OID), p.var(2, capi.FLOAT8OID)
    arg = p.func(capi.F_FLOAT8DIV, capi.FLOAT8OID, a, b) if kind == "div0" else a
    return capi.make_agg(capi.AGGSTAGE_NORMAL, [p.var(3, capi.INT8OID)], [(capi.AGG_SUM_FLOAT8, arg), (capi.AGG_COUNT_STAR, -1)],
                         num_groups=100000 if kind == "overflow_hash" else 0)


@pytest.mark.parametrize("kind", ["overflow", "overflow_hash", "div0"])
def test_errors_equal_fetch(eng, kind):
    from greengage_b200.engine import ScanAgg
    n = 5000
    vals = np.zeros((n, 3), dtype=np.int64)
    vals[:, 0] = np.full(n, 1e308 if kind.startswith("overflow") else 1.0).view(np.int64)
    vals[:, 1] = np.full(n, 0.0 if kind == "div0" else 2.0).view(np.int64)
    vals[:, 2] = np.arange(n) % 7
    rel, rows = load_rows(eng, vals, np.zeros_like(vals, dtype=bool))
    p = ExprPool()
    agg = _error_plan(p, kind)
    scan = capi.make_scan(capi.rows_tupdesc([capi.FLOAT8OID, capi.FLOAT8OID, capi.INT8OID]), -1)
    a, b = ScanAgg(eng, scan, agg, p.pool), ScanAgg(eng, scan, agg, p.pool)
    try:
        a.run(rows)
        b.run(rows)
        with pytest.raises(capi.GGError) as ef:
            a.fetch(64)
        with pytest.raises(capi.GGError) as ed:
            b.datumrows()
        assert ef.value.code == ed.value.code == (-4 if kind == "div0" else -2) and str(ef.value) == str(ed.value)
        bl = ex.PlanBuilder()
        x = ex.Executor(eng, p.pool, [rows], bl.limit(bl.sort(bl.agg(bl.seqscan(0, scan.desc), agg), [capi.make_sortkey(1, capi.INT8OID)]), 3))
        try:
            with pytest.raises(ex.ExecError) as ee:
                x.rows()
            assert ee.value.code == ef.value.code and ("division by zero" if kind == "div0" else "overflow") in str(ee.value)
        finally:
            x.end()
    finally:
        a.free(); b.free(); rows.free(); rel.free()


# ---- joins: inner / left / right / full, in one batch and batched ----
def _join_plan(p, jointype, floats=True):
    lc, oc = tpch.LI_NARROW_COLS, tpch.ORDERS_COLS
    outer = capi.make_scan(capi.synth_tupdesc(capi.TAB_LINEITEM_NARROW), -1)
    inner = capi.make_scan(capi.synth_tupdesc(capi.TAB_ORDERS), -1)
    hj = capi.make_hashjoin(jointype, [p.var(lc["orderkey"], capi.INT8OID, 0)], [p.var(oc["orderkey"], capi.INT8OID, 1)])
    price = p.var(lc["extendedprice"], capi.FLOAT8OID, 0)
    # float sums of a HashAggregate depend on the order its atomics ran in: the runs compared across executors leave them out
    aggs = [(capi.AGG_COUNT_STAR, -1)] + ([(capi.AGG_SUM_FLOAT8, price), (capi.AGG_AVG_FLOAT8, price)] if floats else []) + \
        [(capi.AGG_MAX_DATE, p.var(lc["shipdate"], capi.DATEOID, 0)), (capi.AGG_COUNT_ANY, price)]
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [p.var(oc["orderstatus"], capi.BPCHAROID, 1), p.var(oc["custkey"], capi.INT4OID, 1)],
                        aggs, num_groups=2000)
    return outer, inner, hj, agg


@pytest.fixture(scope="module")
def li_orders():
    li, _, _ = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, 120_000, seed=21, norders=40_000))
    od, _, _ = tpch.synth_generate(tpch.synth_spec(capi.TAB_ORDERS, 30_000, seed=21))
    return li, od


@pytest.mark.parametrize("work_mem", [0, 64 << 10])
@pytest.mark.parametrize("jointype", [capi.JOIN_INNER, capi.JOIN_LEFT, capi.JOIN_RIGHT, capi.JOIN_FULL])
def test_joinagg_datumrows_equal_fetch(eng, li_orders, jointype, work_mem):
    from greengage_b200.engine import JoinAgg, Relation
    li, od = li_orders
    p = ExprPool()
    outer, inner, hj, agg = _join_plan(p, jointype)
    lrel, orel = Relation(eng, host_pages=li), Relation(eng, host_pages=od)
    j = JoinAgg(eng, outer, inner, hj, agg, p.pool)
    try:
        j.set_work_mem(work_mem)
        nb = j.run(orel, lrel)
        assert (nb > 1) == (work_mem > 0)
        got = datum_words(*j.datumrows())
        buf_rows, _ = j.fetch(200000)                           # the same settled state, read the old way
        want = np.array([aggrow_words(bytes(r), 1, agg)[0] for r in buf_rows], dtype=np.uint64)
        assert len(want) > 100
        if capi.dev_lib().gg_joinagg_variant(j.h) & 15 == HASH:
            assert np.array_equal(as_multiset(got), as_multiset(want))      # one table, read in slot order / in claim order
        else:
            assert np.array_equal(got, want)
    finally:
        j.free(); lrel.free(); orel.free()


def test_final_group_set_equals_fetch(eng):
    """a FINAL set from gg_groups_final: the combined PARTIAL records, finalised on the device, equal gg_groups_fetch"""
    from greengage_b200.engine import Groups, ScanAgg
    vals, nulls = make_data(30000, 1, seed=8)
    rel, rows = load_rows(eng, vals, nulls)
    p = ExprPool()
    part = full_agg(p, key_exprs(p, "tiny"), 0, capi.AGGSTAGE_PARTIAL)
    sa = ScanAgg(eng, capi.make_scan(capi.rows_tupdesc(TYPES), -1), part, p.pool)
    try:
        sa.run(rows)
        sa.fetch(4096)                                           # settles the pipeline, as the executor does before a Motion
        g = Groups.of(sa)
        fin = g.final()
        fin2 = g.final()
        want, _, _ = fin.fetch(4096)
        normal = capi.gg_agg.from_buffer_copy(bytes(part))
        normal.aggstage = capi.AGGSTAGE_NORMAL
        want = np.array([aggrow_words(bytes(r), 1, normal)[0] for r in want], dtype=np.uint64)
        got = datum_words(*fin2.datumrows(part.numCols + part.numAggs))
        assert len(want) == 5 and np.array_equal(got, want)          # 4 strings and NULL
        for x in (fin, fin2, g):
            x.free()
    finally:
        sa.free(); rows.free(); rel.free()


# ---- the node surface: Limit <- Sort <- Agg ----
def host_rows(rows):
    return [tuple(int(v) for v in vals) + tuple(int(n) for n in nl) for vals, nl, ty, ln in rows]


def np_sorted(rows, keys):
    """a NumPy-free Python sort of host slot rows under the Sort's keys (ints / floats / packed strings)"""
    def keyfn(r):
        out = []
        for k in keys:
            v, isnull = r[0][k.col], r[1][k.col]
            t = k.typid or r[2][k.col]
            if t == capi.FLOAT8OID:
                x = struct.unpack("<d", struct.pack("<q", v))[0]
                x = (1, 0.0) if x != x else (0, x + 0.0)
            elif t in (capi.BPCHAROID, capi.VARCHAROID, capi.TEXTOID):
                x = (v & 0xFFFFFFFFFFFFFFFF).to_bytes(8, "little").rstrip(b"\0")
            else:
                x = v
            nullkey = (0 if isnull else 1) if k.nulls_first else (1 if isnull else 0)
            if k.desc:
                x = _Desc(x)
            out.append((nullkey, None if isnull else x))
        return out
    return sorted(rows, key=keyfn)


class _Desc:
    def __init__(self, x):
        self.x = x

    def __lt__(self, o):
        return o.x < self.x

    def __eq__(self, o):
        return self.x == o.x


def slot_rows(x):
    return [(vals, nl, ty) for vals, nl, ty, ln in x.rows()]


def check_windows(eng, pool, rels, agg_plan_fn, keys, kinds, interconnect=None, expect_device=True):
    """Limit <- Sort <- Agg for windows of 0, 1, n, > n, LIMIT ALL and OFFSETs, against the sorted rows of the Agg at the top"""
    b = ex.PlanBuilder()
    x = ex.Executor(eng, pool, rels, agg_plan_fn(b), interconnect=interconnect)
    try:
        base = np_sorted(slot_rows(x), keys)
    finally:
        x.end()
    n = len(base)
    assert n > 0
    for count, offset in ((0, None), (1, None), (n, None), (n + 7, None), (None, None), (10, 3), (5, n - 2), (None, n // 2)):
        b = ex.PlanBuilder()
        x = ex.Executor(eng, pool, rels, b.limit(b.sort(agg_plan_fn(b), keys), count, offset), interconnect=interconnect)
        try:
            got = slot_rows(x)
            lo = offset or 0
            hi = n if count is None else min(n, lo + count)
            assert got == base[lo:hi], (count, offset)
            want_loc = [("limit", "host"), ("sort", "device-rows"), (kinds, "device-rows")]
            if count != 0 and expect_device:
                assert x.locations()[:3] == want_loc, x.locations()
            if count == 10:
                x.rescan()
                assert slot_rows(x) == base[lo:hi]
                if expect_device:
                    assert x.locations()[:3] == want_loc
        finally:
            x.end()
    return base


def test_limit_sort_agg_over_seqscan(eng):
    vals, nulls = make_data(60000, 500, seed=11)
    rel, rows = load_rows(eng, vals, nulls)
    p = ExprPool()
    agg = full_agg(p, key_exprs(p, "many"), 0)
    desc = capi.rows_tupdesc(TYPES)
    # count(*) DESC, then the grouping keys: a total order
    keys = [capi.make_sortkey(2, capi.INT8OID, desc=True), capi.make_sortkey(4, capi.FLOAT8OID), capi.make_sortkey(0, capi.INT8OID),
            capi.make_sortkey(1, capi.INT4OID)]
    try:
        check_windows(eng, p.pool, [rows], lambda b: b.agg(b.seqscan(0, desc), agg), keys, "scanagg")
        # a Limit directly over the Agg: a window of distinct groups
        b = ex.PlanBuilder()
        x = ex.Executor(eng, p.pool, [rows], b.limit(b.agg(b.seqscan(0, desc), agg), 50, 7))
        try:
            got = slot_rows(x)
            assert len(got) == 50 and len({tuple(r[0][:2]) + tuple(r[1][:2]) for r in got}) == 50
            assert x.locations()[:2] == [("limit", "host"), ("scanagg", "device-rows")]
            ins = dict(x.instrumentation())["scanagg"]
            assert ins.ntuples == 57
        finally:
            x.end()
    finally:
        rows.free(); rel.free()


def test_limit_sort_agg_over_hashjoin(eng, li_orders):
    from greengage_b200.engine import Relation
    li, od = li_orders
    p = ExprPool()
    outer, inner, hj, agg = _join_plan(p, capi.JOIN_LEFT, floats=False)
    keys = [capi.make_sortkey(2, capi.INT8OID, desc=True), capi.make_sortkey(0, capi.BPCHAROID), capi.make_sortkey(1, capi.INT4OID)]
    rels = [Relation(eng, host_pages=li), Relation(eng, host_pages=od)]
    try:
        check_windows(eng, p.pool, rels, lambda b: b.agg(b.hashjoin(b.seqscan(0, outer.desc), b.hash(b.seqscan(1, inner.desc)), hj), agg),
                      keys, "joinagg")
    finally:
        for r in rels:
            r.free()


def _two_stage(b, desc, p, keys_which):
    part = full_agg(p, key_exprs(p, keys_which), 0, capi.AGGSTAGE_PARTIAL)
    fin = capi.gg_agg.from_buffer_copy(bytes(part))
    fin.aggstage = capi.AGGSTAGE_FINAL
    for c in range(part.numCols):
        fin.grpCol[c] = p.pool.nodes[part.grpCol[c]].rettype          # a FINAL Agg's grpCol carries the key type OIDs
    return b.agg(b.motion(b.agg(b.seqscan(0, desc), part), ex.MOTION_HASH, list(range(part.numCols)), 1), fin)


@pytest.mark.parametrize("groups", ["few", "many"])
def test_limit_sort_agg_two_stage(eng, groups):
    """two stages over the loopback interconnect: a FINAL Agg that combines device group records hands up device rows; with more
    groups than a Motion block carries, every segment retries with host rows (GG_ERR_RETRY_HOST) and the answer is the same"""
    from greengage_b200.engine import Interconnect
    vals, nulls = make_data(40000, 300, seed=13)
    rel, rows = load_rows(eng, vals, nulls)
    p = ExprPool()
    desc = capi.rows_tupdesc(TYPES)
    ic = Interconnect(eng, 1, 0)
    # "tiny": 5 groups, within the 32 records a Motion block carries; "many": thousands
    which = "tiny" if groups == "few" else "many"
    keys = [capi.make_sortkey(1, capi.INT8OID, desc=True), capi.make_sortkey(0, capi.BPCHAROID)] if which == "tiny" else \
        [capi.make_sortkey(2, capi.INT8OID, desc=True), capi.make_sortkey(0, capi.INT8OID), capi.make_sortkey(1, capi.INT4OID)]
    try:
        check_windows(eng, p.pool, [rows], lambda b: _two_stage(b, desc, p, which), keys, "aggfinal", interconnect=ic,
                      expect_device=groups == "few")
    finally:
        ic.close(); rows.free(); rel.free()


def test_numeric_aggregate_keeps_host_rows(eng):
    """an Agg with a numeric aggregate under a Sort / Limit keeps the host path, with the same answer"""
    import _numeric as nref
    from oracle import pyoracle as po
    from test_gpu_numeric import NUM, num_desc
    from greengage_b200.engine import Relation
    rng = np.random.default_rng(9)
    desc = num_desc([(capi.INT4OID, None, 1), (NUM, nref.typmod(15, 2), 1)])
    data = [(int(rng.integers(0, 40)), int(rng.integers(-10**9, 10**9))) for _ in range(5000)]
    pages = po.build_pages(desc, [[k, capi.numeric_payload(v, 2)] for k, v in data])
    p = ExprPool()
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [p.var(1, capi.INT4OID)], [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_NUMERIC, p.var(2, NUM))])
    rel = Relation(eng, host_pages=pages)
    keys = [capi.make_sortkey(0, capi.INT4OID, desc=True)]
    try:
        b = ex.PlanBuilder()
        x = ex.Executor(eng, p.pool, [rel], b.agg(b.seqscan(0, desc), agg))
        base = np_sorted(slot_rows(x), keys)
        x.end()
        b = ex.PlanBuilder()
        x = ex.Executor(eng, p.pool, [rel], b.limit(b.sort(b.agg(b.seqscan(0, desc), agg), keys), 7, 2))
        try:
            assert slot_rows(x) == base[2:9]
            assert x.locations()[:3] == [("limit", "host"), ("sort", "host"), ("scanagg", "host")]
        finally:
            x.end()
    finally:
        rel.free()


def test_more_than_2_24_groups_under_limit_sort(eng):
    """GROUP BY over 2^24 + 10^6 distinct keys, ORDER BY sum DESC, key LIMIT 10: the host path stopped at 2^24 groups"""
    n = (1 << 24) + 1_000_000
    rng = np.random.default_rng(5)
    key = rng.permutation(n).astype(np.int64) * 3 + 1
    price = rng.integers(1, 10**6, n).astype(np.float64) / 100
    vals = np.stack([key, price.view(np.int64)], axis=1)
    rel, rows = load_rows(eng, vals, np.zeros_like(vals, dtype=bool))
    p = ExprPool()
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [p.var(1, capi.INT8OID)],
                        [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_FLOAT8, p.var(2, capi.FLOAT8OID))])
    desc = capi.rows_tupdesc([capi.INT8OID, capi.FLOAT8OID], notnull=[1, 1])
    b = ex.PlanBuilder()
    x = ex.Executor(eng, p.pool, [rows], b.limit(b.sort(b.agg(b.seqscan(0, desc), agg),
                                                      [capi.make_sortkey(2, capi.FLOAT8OID, desc=True), capi.make_sortkey(0, capi.INT8OID)]), 10))
    try:
        got = [(v[0], v[1], struct.unpack("<d", struct.pack("<q", v[2]))[0]) for v, nl, ty, ln in x.rows()]
        order = np.lexsort((key, -price))[:10]                  # one row per key: the sum is the price itself
        assert got == [(int(key[i]), 1, float(price[i])) for i in order]
        assert x.locations()[:3] == [("limit", "host"), ("sort", "device-rows"), ("scanagg", "device-rows")]
    finally:
        x.end(); rows.free(); rel.free()
