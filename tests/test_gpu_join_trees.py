"""Multi-level join plans on the GPU through the executor-node surface (PlanBuilder / Executor), against the row-at-a-time
reference of test_join_tree_reference.py: a HashJoin whose input is the datum rows of another join, on either side, under
every consumer of join rows — another join, an Agg fused with a join, Sort, Sort + Limit, a Gather Motion and the caller.

Seeded random trees draw join types, sides, key pairs (cross-type included, keys from null-extended columns included), join
quals, target lists, the top node and the operator's memory; a shape the executor refuses must be refused with
GG_ERR_UNSUPPORTED.  Targeted tests pin what the random trees may miss: dead slots of windowed claims in every consumer,
NULL keys from null-extension (NOT IN included), NOT NULL through null-extension, cross-type keys between levels, an
overflowing lower join under an upper one, and ReScan / squelch of a two-level tree."""
import ctypes as C
from collections import Counter

import numpy as np
import pytest

from _util import make_desc
from greengage_b200 import capi, executor as ex
from oracle import pyoracle as po
from test_gpu_join_rows import datum
from test_gpu_keys import COLS, TYPID, col, key_relation
from test_join_tree_reference import (BOTH_SIDES, Join, Scan, aggregate, check_groups, check_limit, check_sort, join_pairs, page_rows,
                                      plan_of, row_token, rows_of)

pytestmark = pytest.mark.gpu

UNSUPPORTED = -6                                          # GG_ERR_UNSUPPORTED
OUTER_ONLY = (capi.JOIN_SEMI, capi.JOIN_ANTI, capi.JOIN_LASJ_NOTIN)
INT4 = (capi.INT4OID, 4, "i", 1, 1)                       # NOT NULL


@pytest.fixture(scope="module")
def eng():
    from greengage_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


class Rels:
    """base relations: host pages, descriptors, reference rows and the device copies (relid = index)"""
    def __init__(self, eng, tables):
        from greengage_b200.engine import Relation
        self.desc = [d for d, _ in tables]
        self.pages = [pg for _, pg in tables]
        self.rows = [page_rows(d, pg) for d, pg in tables]
        self.dev = [Relation(eng, host_pages=pg) for pg in self.pages]

    def scan(self, relid, qual=-1):
        return Scan(relid, self.desc[relid], self.rows[relid], qual)

    def free(self):
        for r in self.dev:
            r.free()


@pytest.fixture(scope="module")
def key_rels(eng):
    tables = []
    for n, seed in ((60, 41), (40, 42), (30, 43), (24, 44)):
        d, pg, _, _ = key_relation(n, seed)
        tables.append((d, pg))
    r = Rels(eng, tables)
    yield r
    r.free()


def slot_rows(rows):
    return [tuple(datum(v, n, t) for v, n, t in zip(vals, nl, ty)) for vals, nl, ty, ln in rows]


def join_states(x):
    """[(node kind, hash batches)] of every join in the executor tree, top down, outer before inner"""
    L = ex.exec_lib()
    L.GgExecNodeInstrumentation.argtypes = [C.c_void_p, C.POINTER(ex.GgInstrumentation)]
    out = []

    def walk(st):
        if not st:
            return
        kind = L.GgExecNodeKind(st).decode()
        if kind in ("joinrows", "joinagg"):
            ins = ex.GgInstrumentation()
            capi.check(L.GgExecNodeInstrumentation(st, C.byref(ins)))
            out.append((kind, ins.hash_batches))
        walk(L.GgExecOuterPlanState(st))
        walk(L.GgExecInnerPlanState(st))
    walk(x.state)
    return out


def execute(eng, pool, rels, plan, operator_mem=0, limit=None):
    """(device rows as Python values, [(join kind, hash batches)])"""
    x = ex.Executor(eng, pool, rels, plan, operator_mem=operator_mem)
    try:
        rows = slot_rows(x.rows(limit))
        return rows, join_states(x)
    finally:
        x.end()


def agg_rows(rows, agg):
    """Agg slots (grouping columns, then one column per aggregate) as check_groups' (keys, values)"""
    return [(list(r[:agg.numCols]), list(r[agg.numCols:])) for r in rows]


# ---- random trees ----

STRINGS = (capi.BPCHAROID, capi.VARCHAROID, capi.TEXTOID)


def partners(t):
    """the key types a key of type t joins with"""
    if t in (capi.INT4OID, capi.INT8OID):
        return (capi.INT4OID, capi.INT8OID)
    if t in (capi.VARCHAROID, capi.TEXTOID):
        return (capi.VARCHAROID, capi.TEXTOID)
    return (t,)


class Side:
    """what one input of a join offers: its column types, which float8 columns are small finite values (safe in + - *)"""
    def __init__(self, node, safe):
        self.node, self.types, self.safe = node, node.types, safe


def base_side(rels, relid):
    s = rels.scan(relid)
    return Side(s, [c == "v" for c in COLS])


def draw_join(rng, p, outer, inner, budget, top_agg):
    """one HashJoin over two Sides; None when no key pair exists"""
    jt = int(rng.integers(0, 7))
    pairs = [(a, b) for a, ta in enumerate(outer.types) for b, tb in enumerate(inner.types) if tb in partners(ta)]
    if not pairs:
        return None
    nk = int(rng.integers(1, 3))
    idx = rng.choice(len(pairs), size=min(nk, len(pairs)), replace=False)
    ok = [p.var(pairs[i][0] + 1, outer.types[pairs[i][0]], 0) for i in idx]
    ik = [p.var(pairs[i][1] + 1, inner.types[pairs[i][1]], 1) for i in idx]
    qual = -1
    if rng.random() < 0.4:
        side, varno = (outer, 0) if rng.random() < 0.5 else (inner, 1)
        f8 = [c for c, t in enumerate(side.types) if t == capi.FLOAT8OID]
        i4 = [c for c, t in enumerate(side.types) if t == capi.INT4OID]
        if f8 and (not i4 or rng.random() < 0.5):
            c = int(rng.choice(f8))
            qual = p.func(capi.F_FLOAT8GT, capi.BOOLOID, p.var(c + 1, capi.FLOAT8OID, varno), p.const(capi.FLOAT8OID, float(rng.choice([-10.0, 0.0]))))
        elif i4:
            c = int(rng.choice(i4))
            qual = p.func(capi.F_INT4LT, capi.BOOLOID, p.var(c + 1, capi.INT4OID, varno), p.const(capi.INT4OID, int(rng.choice([0, 2, 1000]))))
    targets, safe = [], []
    if not top_agg:
        cols = [(0, c) for c in range(len(outer.types))] + ([(1, c) for c in range(len(inner.types))] if jt not in OUTER_ONLY else [])
        n = int(min(rng.integers(1, 17), budget - p.pool.nnodes - 2))
        for k in rng.choice(len(cols), size=min(max(n, 1), len(cols)), replace=False):
            if p.pool.nnodes >= budget - 1:
                break
            varno, c = cols[k]
            side = outer if varno == 0 else inner
            v = p.var(c + 1, side.types[c], varno)
            if side.safe[c] and rng.random() < 0.5 and p.pool.nnodes < budget - 4:
                f = int(rng.choice([capi.F_FLOAT8PL, capi.F_FLOAT8MI, capi.F_FLOAT8MUL]))
                v = p.func(f, capi.FLOAT8OID, v, p.const(capi.FLOAT8OID, float(rng.choice([0.5, -2.0, 0.0]))))
            targets.append(v)
            safe.append(bool(side.safe[c]))
    node = Join(outer.node, inner.node, jt, ok, ik, qual, targets, p.pool)
    return Side(node, safe) if targets else node


def draw_agg(rng, p, node):
    """an Agg fused with the join `node`: 1–2 group keys from either input, null-extended ones included"""
    o, i = node.outer.types, node.inner.types
    cols = [(0, c, t) for c, t in enumerate(o)] + ([(1, c, t) for c, t in enumerate(i)] if node.jointype not in OUTER_ONLY else [])
    pick = lambda pred: [x for x in cols if pred(x[2])]
    keys = [p.var(c + 1, t, v) for v, c, t in (cols[k] for k in rng.choice(len(cols), size=int(rng.integers(1, 3)), replace=False))]
    aggs = [(capi.AGG_COUNT_STAR, -1)]
    v, c, t = cols[int(rng.integers(0, len(cols)))]
    aggs.append((capi.AGG_COUNT_ANY, p.var(c + 1, t, v)))
    for types, fns in (((capi.INT4OID,), (capi.AGG_SUM_INT4, capi.AGG_MIN_INT4, capi.AGG_MAX_INT4)),
                       ((capi.INT8OID,), (capi.AGG_MIN_INT8, capi.AGG_MAX_INT8)), ((capi.DATEOID,), (capi.AGG_MIN_DATE, capi.AGG_MAX_DATE))):
        xs = pick(lambda tt: tt in types)
        if xs:
            v, c, t = xs[int(rng.integers(0, len(xs)))]
            aggs.append((int(rng.choice(fns)), p.var(c + 1, t, v)))
    safe = [(0, c) for c in range(len(o)) if node.outer_safe[c]] + \
           ([(1, c) for c in range(len(i)) if node.inner_safe[c]] if node.jointype not in OUTER_ONLY else [])
    if safe:
        v, c = safe[int(rng.integers(0, len(safe)))]
        aggs += [(capi.AGG_SUM_FLOAT8, p.var(c + 1, capi.FLOAT8OID, v)), (capi.AGG_AVG_FLOAT8, p.var(c + 1, capi.FLOAT8OID, v))]
    return capi.make_agg(capi.AGGSTAGE_NORMAL, keys, aggs, num_groups=int(rng.choice([0, 10, 500])))


def random_tree(rng, rels):
    """(pool, reference top, executor plan builder fn, top kind, extra) for one seed; None when the draw got too large"""
    p = capi.ExprPool()
    nlev = int(rng.integers(2, 4))
    order = [int(x) for x in rng.permutation(4)[:nlev + 1]]
    top = str(rng.choice(["rows", "agg", "sort", "limit", "gather"]))
    cur = base_side(rels, order[0])
    for lev in range(nlev):
        other = base_side(rels, order[lev + 1])
        outer, inner = (cur, other) if rng.random() < 0.5 else (other, cur)
        last = lev == nlev - 1
        got = draw_join(rng, p, outer, inner, 64 if not last else 80, last and top == "agg")
        if got is None:
            return None
        if isinstance(got, Join):                                  # the top join of an Agg
            got.outer_safe, got.inner_safe = outer.safe, inner.safe
            return p, got, top, draw_agg(rng, p, got)
        if len(rows_of(p.pool, got.node)) > 20000:
            return None
        cur = got
    node = cur.node
    extra = None
    if top in ("sort", "limit"):
        nk = int(rng.integers(1, min(4, len(node.types)) + 1))
        extra = [capi.make_sortkey(int(c), node.types[int(c)], bool(rng.random() < 0.5), bool(rng.random() < 0.5))
                 for c in rng.choice(len(node.types), size=nk, replace=False)]
    return p, node, top, extra


def run_tree(eng, rels, p, node, top, extra, operator_mem):
    b = ex.PlanBuilder()
    if top == "agg":
        plan = b.agg(plan_of(b, node), extra)
    elif top == "sort":
        plan = b.sort(plan_of(b, node), extra)
    elif top == "limit":
        plan = b.limit(b.sort(plan_of(b, node), extra), 17)
    elif top == "gather":
        plan = b.motion(plan_of(b, node), ex.MOTION_GATHER)
    else:
        plan = plan_of(b, node)
    return execute(eng, p.pool, rels.dev, plan, operator_mem)


def check_tree(p, node, top, extra, got, ctx):
    if top == "agg":
        check_groups(agg_rows(got, extra), aggregate(p.pool, extra, join_pairs(p.pool, node)), extra, p.pool, ctx)
        return
    want = rows_of(p.pool, node)
    if top == "sort":
        check_sort(got, want, extra, ctx)
    elif top == "limit":
        check_limit(got, want, extra, 17, ctx)
    else:
        assert Counter(map(row_token, got)) == Counter(map(row_token, want)), ctx


SEEDS = list(range(30))
_outcomes = {}


@pytest.mark.parametrize("seed", SEEDS)
def test_random_join_trees(eng, key_rels, seed):
    rng = np.random.default_rng(1000 + seed)
    drawn = None
    for _ in range(8):
        drawn = random_tree(rng, key_rels)
        if drawn is not None:
            break
    assert drawn is not None, seed
    p, node, top, extra = drawn
    operator_mem = int(rng.choice([0, 0, 16384, 65536]))
    ctx = (seed, top, operator_mem)
    try:
        got, joins = run_tree(eng, key_rels, p, node, top, extra, operator_mem)
    except ex.ExecError as e:
        assert e.code == UNSUPPORTED, (ctx, e.code, str(e))
        _outcomes[seed] = ("refused", str(e))
        pytest.skip("refused with GG_ERR_UNSUPPORTED: %s" % e)
    assert len(joins) >= 2, joins
    if operator_mem == 0:
        assert all(nb == 1 for _, nb in joins), joins
    _outcomes[seed] = ("ran", top, [nb for _, nb in joins])
    check_tree(p, node, top, extra, got, ctx)


def test_most_random_trees_run():
    """after the seeds: most of them ran on the device rather than being refused, and some ran batched"""
    if len(_outcomes) < len(SEEDS):
        pytest.skip("judges the seeds of test_random_join_trees, which did not all run")
    ran = [o for o in _outcomes.values() if o[0] == "ran"]
    assert len(ran) >= 0.8 * len(SEEDS), _outcomes
    assert any(max(o[2]) > 1 for o in ran), _outcomes


# ---- 1. dead slots of windowed claims into every consumer ----

@pytest.fixture(scope="module")
def wide(eng):
    """A(a, k = a % 100) 100 000 rows ⋈ B(b, k = b % 100) 2 000 rows on k: 2·10^6 rows, enough that the probe's warps claim
    rows a window at a time; C(c) 5 000 ids of A, duplicates and misses included"""
    rng = np.random.default_rng(3)
    d2 = make_desc([INT4, INT4])
    A = np.arange(100_000)
    B = np.arange(2000)
    Cc = rng.integers(0, 110_000, 5000)
    Cc[0] = 0                                             # a dead slot read as a row of zeros would match it
    pages = [po.build_pages(d2, [[int(a), int(a % 100)] for a in A]), po.build_pages(d2, [[int(b), int(b % 100)] for b in B]),
             po.build_pages(d2, [[int(c), int(c % 7)] for c in Cc])]
    r = Rels.__new__(Rels)
    from greengage_b200.engine import Relation
    r.desc, r.pages, r.rows = [d2] * 3, pages, [None] * 3
    r.dev = [Relation(eng, host_pages=pg) for pg in pages]
    yield r, A, B, Cc
    r.free()


def _lower_wide(b, p):
    """A ⋈ Hash(B) on k, projecting (a, b, k)"""
    d = make_desc([INT4, INT4])
    hj = capi.make_hashjoin(capi.JOIN_INNER, [p.var(2, capi.INT4OID, 0)], [p.var(2, capi.INT4OID, 1)])
    return b.hashjoin(b.seqscan(0, d), b.hash(b.seqscan(1, d)), hj, [p.var(1, capi.INT4OID, 0), p.var(1, capi.INT4OID, 1), p.var(2, capi.INT4OID, 0)])


def test_wide_lower_join_leaves_dead_slots(eng, wide):
    from greengage_b200.engine import JoinRows
    r, A, B, Cc = wide
    p = capi.ExprPool()
    d = r.desc[0]
    hj = capi.make_hashjoin(capi.JOIN_INNER, [p.var(2, capi.INT4OID, 0)], [p.var(2, capi.INT4OID, 1)])
    jr = JoinRows(eng, capi.make_scan(d), capi.make_scan(d), hj, [p.var(1, capi.INT4OID, 0), p.var(1, capi.INT4OID, 1), p.var(2, capi.INT4OID, 0)], p.pool)
    try:
        assert jr.run(r.dev[1], r.dev[0]) == 1
        _, nslots, live = jr.rows_raw()
        assert live == A.size * 20 and nslots > live, (nslots, live)
    finally:
        jr.free()


@pytest.mark.parametrize("operator_mem", [0, 200_000])
@pytest.mark.parametrize("consumer", ["hash", "outer", "agg", "limit"])
def test_dead_slots_into_every_consumer(eng, wide, consumer, operator_mem):
    r, A, B, Cc = wide
    if consumer == "limit" and operator_mem:
        pytest.skip("no upper join to batch")
    p = capi.ExprPool()
    b = ex.PlanBuilder()
    d = r.desc[0]
    lower = _lower_wide(b, p)
    bs = {k: B[B % 100 == k] for k in range(100)}
    hit = Cc[Cc < A.size]
    want_pairs = Counter((int(c), int(x)) for c in hit for x in bs[int(c % 100)])
    if consumer == "hash":          # C ⋈ Hash(lower rows) on c = a
        hj = capi.make_hashjoin(capi.JOIN_INNER, [p.var(1, capi.INT4OID, 0)], [p.var(1, capi.INT4OID, 1)])
        plan = b.hashjoin(b.seqscan(2, d), b.hash(lower), hj, [p.var(1, capi.INT4OID, 0), p.var(2, capi.INT4OID, 1)])
    else:                           # lower rows ⋈ Hash(C) on a = c
        hj = capi.make_hashjoin(capi.JOIN_INNER, [p.var(1, capi.INT4OID, 0)], [p.var(1, capi.INT4OID, 1)])
        if consumer == "outer":
            plan = b.hashjoin(lower, b.hash(b.seqscan(2, d)), hj, [p.var(1, capi.INT4OID, 0), p.var(2, capi.INT4OID, 0)])
        elif consumer == "agg":
            # a LEFT join: every row the upper join reads reaches the Agg, whatever its values
            agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [p.var(3, capi.INT4OID, 0)], [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_INT4, p.var(2, capi.INT4OID, 0))],
                                num_groups=100)
            hj.jointype = capi.JOIN_LEFT
            plan = b.agg(b.hashjoin(lower, b.hash(b.seqscan(2, d)), hj), agg)
        else:
            plan = b.limit(b.sort(lower, [capi.make_sortkey(1, capi.INT4OID, desc=True), capi.make_sortkey(0, capi.INT4OID)]), 100)
    got, joins = execute(eng, p.pool, r.dev, plan, operator_mem)
    if operator_mem:
        assert joins[-1][1] == 1 and joins[0][1] > 1, joins            # the upper join batched, the wide lower one not
    else:
        assert all(nb == 1 for _, nb in joins), joins
    if consumer in ("hash", "outer"):
        assert Counter(got) == want_pairs
    elif consumer == "agg":
        mult = np.maximum(np.bincount(Cc, minlength=110_000)[:A.size], 1)       # rows per lower row: its matches, or one
        want = {k: [20 * int(mult[A % 100 == k].sum()), int(mult[A % 100 == k].sum()) * int(B[B % 100 == k].sum())] for k in range(100)}
        assert {g[0]: [g[1], g[2]] for g in got} == want
    else:
        top = A[A % 100 == 99][:100]
        assert got == [(int(a), 1999, 99) for a in top]


# ---- 2. NULL keys from null-extension ----

def small_tables(eng):
    """A(id NOT NULL, z NOT NULL in 0..2, v) 200 rows; B(id NOT NULL, z NOT NULL in 0..2) 50 rows; C(id NOT NULL, w) 120 rows"""
    rng = np.random.default_rng(5)
    F8 = (capi.FLOAT8OID, 8, "d", 1, 0)
    da, db, dc = make_desc([INT4, INT4, F8]), make_desc([INT4, INT4]), make_desc([INT4, (capi.INT8OID, 8, "d", 1, 0)])
    ta = (da, po.build_pages(da, [[i, int(rng.integers(0, 3)), float(rng.integers(-40, 40)) / 4] for i in range(200)]))
    tb = (db, po.build_pages(db, [[i, i % 3] for i in range(50)]))
    tc = (dc, po.build_pages(dc, [[int(rng.integers(0, 60)), int(rng.integers(-5, 5))] for i in range(120)]))
    return Rels(eng, [ta, tb, tc])


@pytest.fixture(scope="module")
def small(eng):
    r = small_tables(eng)
    yield r
    r.free()


def left_lower(p, rels, bqual_max):
    """A LEFT JOIN (B where B.z < bqual_max) on z: (A.id, B.id, B.z, A.z); B.id / B.z NULL where nothing matched"""
    bq = p.func(capi.F_INT4LT, capi.BOOLOID, p.var(2, capi.INT4OID, 1), p.const(capi.INT4OID, bqual_max))
    return Join(rels.scan(0), rels.scan(1, bq), capi.JOIN_LEFT, [p.var(2, capi.INT4OID, 0)], [p.var(2, capi.INT4OID, 1)],
                targets=[p.var(1, capi.INT4OID, 0), p.var(1, capi.INT4OID, 1), p.var(2, capi.INT4OID, 1), p.var(2, capi.INT4OID, 0)], pool=p.pool)


@pytest.mark.parametrize("upper", ["inner", "notin", "notin-matched", "full-outer", "right-inner"])
def test_null_extended_column_as_an_upper_key(eng, small, upper):
    p = capi.ExprPool()
    lower = left_lower(p, small, 3 if upper == "notin-matched" else 2)
    lrows = rows_of(p.pool, lower)
    has_null = any(r[1] is None for r in lrows)
    assert has_null == (upper != "notin-matched")
    cscan = small.scan(2)
    if upper == "inner":
        node = Join(lower, cscan, capi.JOIN_INNER, [p.var(2, capi.INT4OID, 0)], [p.var(1, capi.INT4OID, 1)],
                    targets=[p.var(1, capi.INT4OID, 0), p.var(2, capi.INT4OID, 0), p.var(2, capi.INT8OID, 1)], pool=p.pool)
    elif upper.startswith("notin"):          # C.id NOT IN (lower B.id)
        node = Join(cscan, lower, capi.JOIN_LASJ_NOTIN, [p.var(1, capi.INT4OID, 0)], [p.var(2, capi.INT4OID, 1)],
                    targets=[p.var(1, capi.INT4OID, 0), p.var(2, capi.INT8OID, 0)], pool=p.pool)
    elif upper == "full-outer":
        node = Join(lower, cscan, capi.JOIN_FULL, [p.var(2, capi.INT4OID, 0)], [p.var(1, capi.INT4OID, 1)],
                    targets=[p.var(1, capi.INT4OID, 0), p.var(2, capi.INT4OID, 0), p.var(1, capi.INT4OID, 1)], pool=p.pool)
    else:                                     # C RIGHT JOIN lower rows: the NULL-keyed lower rows come back unmatched
        node = Join(cscan, lower, capi.JOIN_RIGHT, [p.var(1, capi.INT4OID, 0)], [p.var(2, capi.INT4OID, 1)],
                    targets=[p.var(1, capi.INT4OID, 0), p.var(1, capi.INT4OID, 1), p.var(2, capi.INT4OID, 1)], pool=p.pool)
    want = rows_of(p.pool, node)
    b = ex.PlanBuilder()
    got, joins = execute(eng, p.pool, small.dev, plan_of(b, node))
    assert len(joins) == 2
    assert Counter(map(row_token, got)) == Counter(map(row_token, want))
    if upper == "notin":
        assert want == []
    elif upper == "notin-matched":
        assert 0 < len(want) < len(small.rows[2])
    elif upper == "full-outer":
        assert any(r[1] is None and r[0] is not None for r in want)
    elif upper == "right-inner":
        assert any(r[0] is None and r[1] is not None and r[2] is None for r in want)


# ---- 3. NOT NULL through null-extension ----

@pytest.mark.parametrize("jointype", [capi.JOIN_LEFT, capi.JOIN_RIGHT, capi.JOIN_FULL])
def test_not_null_columns_of_a_null_extended_side(eng, small, jointype):
    p = capi.ExprPool()
    bq = p.func(capi.F_INT4LT, capi.BOOLOID, p.var(2, capi.INT4OID, 1), p.const(capi.INT4OID, 2))
    aq = p.func(capi.F_INT4GT, capi.BOOLOID, p.var(2, capi.INT4OID, 0), p.const(capi.INT4OID, 0))
    # (A.id, A.z, B.id, B.z): every base column NOT NULL; A's come out NULL under RIGHT / FULL, B's under LEFT / FULL
    lower = Join(small.scan(0, aq), small.scan(1, bq), jointype, [p.var(2, capi.INT4OID, 0)], [p.var(2, capi.INT4OID, 1)],
                 targets=[p.var(1, capi.INT4OID, 0), p.var(2, capi.INT4OID, 0), p.var(1, capi.INT4OID, 1), p.var(2, capi.INT4OID, 1)], pool=p.pool)
    lrows = rows_of(p.pool, lower)
    ext = [2, 3] if jointype == capi.JOIN_LEFT else [0, 1] if jointype == capi.JOIN_RIGHT else [0, 1, 2, 3]
    assert all(any(r[c] is None for r in lrows) for c in ext)
    # an Agg fused with an upper join over the lower rows: group keys, count(x), min / max of the null-extended columns
    cscan = small.scan(2)
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [p.var(4, capi.INT4OID, 0), p.var(2, capi.INT4OID, 0)],
                        [(capi.AGG_COUNT_STAR, -1), (capi.AGG_COUNT_ANY, p.var(3, capi.INT4OID, 0)), (capi.AGG_MIN_INT4, p.var(3, capi.INT4OID, 0)),
                         (capi.AGG_MAX_INT4, p.var(1, capi.INT4OID, 0)), (capi.AGG_COUNT_ANY, p.var(1, capi.INT4OID, 0))], num_groups=10)
    # an INNER upper join that reads NOT NULL columns only, so nothing but the rows' descriptor says a column can be NULL (an
    # upper join that null-extends would make the consumer's program nullable on its own)
    for key in (1, 3):                       # the upper key: A.id (NULL under RIGHT / FULL) or B.id (NULL under LEFT / FULL)
        upper = Join(lower, cscan, capi.JOIN_INNER, [p.var(key, capi.INT4OID, 0)], [p.var(1, capi.INT4OID, 1)], pool=p.pool)
        b = ex.PlanBuilder()
        got, joins = execute(eng, p.pool, small.dev, b.agg(plan_of(b, upper), agg))
        check_groups(agg_rows(got, agg), aggregate(p.pool, agg, join_pairs(p.pool, upper)), agg, p.pool, (jointype, key))
    # a NULLS FIRST sort over the lower rows, on a null-extended NOT NULL column
    keys = [capi.make_sortkey(ext[-1], capi.INT4OID, False, True), capi.make_sortkey(0, capi.INT4OID, True, True), capi.make_sortkey(2, capi.INT4OID)]
    b = ex.PlanBuilder()
    got, _ = execute(eng, p.pool, small.dev, b.sort(plan_of(b, lower), keys))
    check_sort(got, lrows, keys, (jointype,))
    assert got[0][ext[-1]] is None


# ---- 4. cross-type keys between levels ----

@pytest.mark.parametrize("pair", [("int4", "int8"), ("int8", "int4"), ("varchar", "text"), ("text", "varchar"), ("bpchar", "bpchar"),
                                  ("float8", "f0"), ("f0", "float8")], ids=lambda x: "%s=%s" % x)
@pytest.mark.parametrize("rows_side", ["outer", "inner"])
def test_cross_type_keys_between_levels(eng, key_rels, pair, rows_side):
    """rows of the lower join (A ⋈ B on z, projecting B's columns) keyed against C's pages; the relation's int4 -1 / int8 2^32-1,
    'A' / 'A ' and ±0 / NaN make a wrong equality change the answer"""
    rk, ck = pair
    p = capi.ExprPool()
    lt = [p.var(col(c), TYPID[c], 1) for c in ("id", rk, "z")]
    lower = Join(key_rels.scan(0), key_rels.scan(1), capi.JOIN_INNER, [p.var(col("z"), capi.INT4OID, 0)], [p.var(col("z"), capi.INT4OID, 1)],
                 targets=lt, pool=p.pool)
    rv = 0 if rows_side == "outer" else 1
    lkey, ckey = p.var(2, TYPID[rk], rv), p.var(col(ck), TYPID[ck], 1 - rv)
    targets = [p.var(1, capi.INT4OID, rv), p.var(2, TYPID[rk], rv), p.var(col("id"), capi.INT4OID, 1 - rv), p.var(col(ck), TYPID[ck], 1 - rv)]
    cscan = key_rels.scan(2)
    node = Join(lower, cscan, capi.JOIN_FULL, [lkey], [ckey], targets=targets, pool=p.pool) if rv == 0 else \
        Join(cscan, lower, capi.JOIN_FULL, [ckey], [lkey], targets=targets, pool=p.pool)
    want = rows_of(p.pool, node)
    assert any(r[0] is not None and r[2] is not None for r in want)
    b = ex.PlanBuilder()
    got, _ = execute(eng, p.pool, key_rels.dev, plan_of(b, node))
    assert Counter(map(row_token, got)) == Counter(map(row_token, want))


# ---- 5. an overflowing lower join under an upper join and an Agg ----

def test_overflowing_lower_join_replays_once_under_an_upper_join(eng):
    """lower: outer 2000 rows ⋈ inner 200 rows on k, ten inner rows per key (20 000 rows, ten times its first sizing) or one per
    key (no overflow); the launches of the whole plan differ by the one replay of the lower probe"""
    from greengage_b200.engine import Relation
    d = make_desc([INT4, INT4])
    opages = po.build_pages(d, [[i % 10, i] for i in range(2000)])
    cpages = po.build_pages(d, [[i, i % 4] for i in range(0, 2000, 3)])
    counts = {}
    for name, ikey in (("many", lambda i: i % 10), ("one", lambda i: i if i < 10 else 1000 + i)):
        ipages = po.build_pages(d, [[ikey(i), 100000 + i] for i in range(200)])
        rels = [Relation(eng, host_pages=pg) for pg in (opages, ipages, cpages)]
        p = capi.ExprPool()
        b = ex.PlanBuilder()
        lower = b.hashjoin(b.seqscan(0, d), b.hash(b.seqscan(1, d)),
                           capi.make_hashjoin(capi.JOIN_INNER, [p.var(1, capi.INT4OID, 0)], [p.var(1, capi.INT4OID, 1)]),
                           [p.var(2, capi.INT4OID, 0), p.var(2, capi.INT4OID, 1)])
        hj = capi.make_hashjoin(capi.JOIN_INNER, [p.var(1, capi.INT4OID, 0)], [p.var(1, capi.INT4OID, 1)])
        agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [], [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_INT4, p.var(2, capi.INT4OID, 0))])
        try:
            before = eng.launch_count()
            got, joins = execute(eng, p.pool, rels, b.agg(b.hashjoin(lower, b.hash(b.seqscan(2, d)), hj), agg))
            counts[name] = eng.launch_count() - before
        finally:
            for r in rels:
                r.free()
        irows = [ikey(i) for i in range(200)]
        want = [(o, 100000 + i) for o in range(2000) for i in range(200) if irows[i] == o % 10 and o % 3 == 0]
        assert got == [(len(want), sum(x for _, x in want))], name
        if name == "many":
            assert len(want) > 2000
    assert counts["many"] == counts["one"] + 1, counts


# ---- 6. ReScan and squelch of a two-level tree ----

@pytest.mark.parametrize("operator_mem", [0, 16384])
def test_rescan_and_squelch_of_a_two_level_tree(eng, key_rels, operator_mem):
    p = capi.ExprPool()
    lower = Join(key_rels.scan(0), key_rels.scan(1), capi.JOIN_LEFT, [p.var(col("int8"), capi.INT8OID, 0)], [p.var(col("int4"), capi.INT4OID, 1)],
                 targets=[p.var(col("id"), capi.INT4OID, 0), p.var(col("text"), capi.TEXTOID, 1), p.var(col("float8"), capi.FLOAT8OID, 0)], pool=p.pool)
    upper = Join(key_rels.scan(2), lower, capi.JOIN_INNER, [p.var(col("varchar"), capi.VARCHAROID, 0)], [p.var(2, capi.TEXTOID, 1)],
                 targets=[p.var(col("id"), capi.INT4OID, 0), p.var(1, capi.INT4OID, 1), p.var(3, capi.FLOAT8OID, 1)], pool=p.pool)
    want = Counter(map(row_token, rows_of(p.pool, upper)))
    assert sum(want.values()) > 5
    b = ex.PlanBuilder()
    x = ex.Executor(eng, p.pool, key_rels.dev, plan_of(b, upper), operator_mem=operator_mem)
    try:
        first = Counter(map(row_token, slot_rows(x.rows())))
        joins = join_states(x)
        assert first == want
        assert [nb > 1 for _, nb in joins] == [operator_mem > 0] * 2, joins
        for _ in range(2):
            x.rescan()
            assert Counter(map(row_token, slot_rows(x.rows()))) == want
        x.rescan()
        part = slot_rows(x.rows(limit=3))
        assert len(part) == 3 and not (Counter(map(row_token, part)) - want)
    finally:
        x.end()
