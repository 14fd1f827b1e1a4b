"""A row-at-a-time reference for the join trees the executor accepts — SeqScan, HashJoin of every join type with or without a
target list, an Agg over a join, Sort and Limit — and its pin to the oracle (oracle/: the reference's HashJoin and grouping
restated), so that tests/test_gpu_join_trees.py can judge multi-level plans on the device with it.

Values are Python values: int4 / int8 / date / timestamp / bool as int, float8 as float, strings as bytes, NULL as None.  A
bpchar value is kept blank-stripped, as the datum rows a join writes hold it.  Key equality follows each key's hash
opfamily: integers by value (int4 = int8 across types), float8 with -0 = +0 and NaN = NaN, bpchar ignoring trailing blanks,
varchar / text by bytes.  NULL keys match nothing."""
import functools
import math
import struct
from collections import Counter

import numpy as np
import pytest

from _util import check_float8_agg, make_desc
from greengage_b200 import capi, executor as ex
from oracle import pyoracle as po
from test_gpu_keys import COLS, SPEC, TYPID, col, key_relation
from test_oracle_join import ALL_JOINTYPES, join_nodes, small_relations

STRINGS = (capi.BPCHAROID, capi.VARCHAROID, capi.TEXTOID)
BOTH_SIDES = (capi.JOIN_INNER, capi.JOIN_LEFT, capi.JOIN_RIGHT, capi.JOIN_FULL)
# key pairs a hash join accepts: every device key type with itself, int4 = int8 and varchar = text both ways
KEYPAIRS = [(t, t) for t in ("int4", "int8", "date", "timestamp", "bool", "float8", "bpchar", "varchar", "text")] + \
           [("int4", "int8"), ("int8", "int4"), ("varchar", "text"), ("text", "varchar")]


def key_class(typid, x):
    """the equality class of a key value under its hash opfamily (None: a NULL key, which matches nothing)"""
    if x is None:
        return None
    if typid == capi.FLOAT8OID:
        return "nan" if x != x else (0.0 if x == 0 else x)
    if typid == capi.BPCHAROID:
        return x.rstrip(b" ")
    return x


def token(x):
    """a value as a hashable token for multisets: float8 by its bits (every NaN one token)"""
    if isinstance(x, float):
        return "nan" if x != x else struct.unpack("<q", struct.pack("<d", x))[0]
    return x


def row_token(r):
    return tuple(token(x) for x in r)


# ---- inputs ----

def page_rows(desc, pages):
    """the tuples of heap pages in page order, bpchar blank-stripped"""
    out = []
    for b in range(pages.size // capi.GG_BLCKSZ):
        for r in po.deform_page(desc, pages, b):
            out.append(tuple(x.rstrip(b" ") if (x is not None and desc.attrs[a].atttypid == capi.BPCHAROID) else x
                             for a, x in enumerate(r)))
    return out


def rows_desc(typids):
    """a heap descriptor for rows of these types (every column nullable)"""
    return make_desc([(t,) + SPEC[t] for t in typids])


def rows_pages(typids, rows):
    """heap pages holding rows of these types"""
    return po.build_pages(rows_desc(typids), [[0 if x is None else x for x in r] for r in rows],
                          [[x is None for x in r] for r in rows])


# ---- expressions ----

def _fcmp(a, b):
    """float8_cmp_internal: NaN above everything, NaN = NaN, -0 = +0"""
    if a != a or b != b:
        return (a != a) - (b != b)
    return (a > b) - (a < b)


ERR_DIV_ZERO = -4                                         # GG_ERR_DIV_ZERO


class RefError(Exception):
    """an ERROR the reference raises; code: the GG_ERR_* the device raises for it"""
    def __init__(self, code, msg):
        super().__init__(code, msg)
        self.code = code


def _float8div(a, b):
    if b == 0:
        raise RefError(ERR_DIV_ZERO, "division by zero")
    return a / b


FUNCS = {
    capi.F_FLOAT8PL: lambda a, b: a + b, capi.F_FLOAT8MI: lambda a, b: a - b, capi.F_FLOAT8MUL: lambda a, b: a * b,
    capi.F_FLOAT8DIV: _float8div,
    capi.F_FLOAT8LT: lambda a, b: _fcmp(a, b) < 0, capi.F_FLOAT8GT: lambda a, b: _fcmp(a, b) > 0,
    capi.F_FLOAT8LE: lambda a, b: _fcmp(a, b) <= 0, capi.F_FLOAT8GE: lambda a, b: _fcmp(a, b) >= 0,
    capi.F_FLOAT8EQ: lambda a, b: _fcmp(a, b) == 0, capi.F_FLOAT8NE: lambda a, b: _fcmp(a, b) != 0,
    capi.F_INT4GT: lambda a, b: a > b, capi.F_INT4LT: lambda a, b: a < b, capi.F_INT4EQ: lambda a, b: a == b,
    capi.F_INT4NE: lambda a, b: a != b, capi.F_INT4LE: lambda a, b: a <= b, capi.F_INT4GE: lambda a, b: a >= b,
    capi.F_INT8GT: lambda a, b: a > b, capi.F_INT8LT: lambda a, b: a < b, capi.F_INT8EQ: lambda a, b: a == b,
    capi.F_INT8NE: lambda a, b: a != b, capi.F_INT8LE: lambda a, b: a <= b, capi.F_INT8GE: lambda a, b: a >= b,
    capi.F_DATE_LT: lambda a, b: a < b, capi.F_DATE_GT: lambda a, b: a > b, capi.F_I8TOD: float, capi.F_I4TOD: float,
    capi.F_BPCHAREQ: lambda a, b: a.rstrip(b" ") == b.rstrip(b" "), capi.F_BPCHARNE: lambda a, b: a.rstrip(b" ") != b.rstrip(b" "),
}


def evaluate(pool, i, o, n):
    """expression node i of the pool over an outer row o (varno 0) and an inner row n (varno 1); None is NULL"""
    e = pool.nodes[i]
    if e.kind == capi.E_VAR:
        return (o if e.varno == 0 else n)[e.varattno - 1]
    if e.kind == capi.E_CONST:
        if e.constisnull:
            return None
        if e.rettype == capi.FLOAT8OID:
            return struct.unpack("<d", struct.pack("<q", e.constvalue))[0]
        if e.rettype in STRINGS:
            return (e.constvalue & 0xFFFFFFFFFFFFFFFF).to_bytes(8, "little")[:e.constlen]
        return int(e.constvalue)
    if e.kind == capi.E_FUNC:
        args = [evaluate(pool, e.args[k], o, n) for k in range(e.nargs)]
        return None if any(a is None for a in args) else FUNCS[e.funcid](*args)
    if e.kind in (capi.E_AND, capi.E_OR):
        a, b = evaluate(pool, e.args[0], o, n), evaluate(pool, e.args[1], o, n)
        stop = e.kind == capi.E_OR                      # three-valued: OR is true if either is, AND false if either is
        if a is stop or b is stop or (a is not None and bool(a) == stop) or (b is not None and bool(b) == stop):
            return stop
        return None if (a is None or b is None) else (not stop)
    if e.kind == capi.E_NOT:
        a = evaluate(pool, e.args[0], o, n)
        return None if a is None else not a
    if e.kind in (capi.E_ISNULL, capi.E_ISNOTNULL):
        return (evaluate(pool, e.args[0], o, n) is None) == (e.kind == capi.E_ISNULL)
    raise AssertionError("expression kind %d is not in the reference" % e.kind)


def passes(pool, q, o, n):
    return q < 0 or evaluate(pool, q, o, n) is True


# ---- plan nodes ----

class Scan:
    """SeqScan of relation `relid` (rows: page_rows of its pages) with a qual (its Vars take the varno of the join side the
    scan feeds); targets: the expressions a row-producing scan projects (Vars varno 0), () for the relation's own columns"""
    def __init__(self, relid, desc, rows, qual=-1, targets=(), pool=None):
        self.relid, self.desc, self.rows, self.qual, self.targets = relid, desc, rows, qual, list(targets)
        self.types = [pool.nodes[t].rettype for t in self.targets] if self.targets else [desc.attrs[a].atttypid for a in range(desc.natts)]


class Join:
    """HashJoin(outer, Hash(inner)): keys are (outer expr, inner expr) pairs; targets () fuse it with an Agg above"""
    def __init__(self, outer, inner, jointype, okeys, ikeys, qual=-1, targets=(), pool=None):
        self.outer, self.inner, self.jointype, self.qual = outer, inner, jointype, qual
        self.okeys, self.ikeys, self.targets = list(okeys), list(ikeys), list(targets)
        self.hj = capi.make_hashjoin(jointype, okeys, ikeys, qual)
        self.types = [pool.nodes[t].rettype for t in self.targets] if pool is not None else []


def plan_of(b, node):
    """the executor plan of a reference tree (PlanBuilder b)"""
    if isinstance(node, Scan):
        return b.seqscan(node.relid, node.desc, node.qual, node.targets)
    if isinstance(node, Agg):
        if not node.two_stage:
            return b.agg(plan_of(b, node.child), node.agg, having=node.having)
        return b.agg(b.motion(b.agg(plan_of(b, node.child), node.partial), ex.MOTION_GATHER), node.agg, having=node.having)
    if isinstance(node, Window):
        w = node.win
        return b.windowagg(plan_of(b, node.child), list(w.partColIdx[:w.partNumCols]), list(w.ordColIdx[:w.ordNumCols]), w.frameOptions,
                           node.funcs, qual=node.qual)
    if isinstance(node, Sort):
        return b.sort(plan_of(b, node.child), node.keys)
    if isinstance(node, Limit):
        return b.limit(plan_of(b, node.child), node.count, node.offset)
    if isinstance(node, Gather):
        return b.motion(plan_of(b, node.child), ex.MOTION_GATHER)
    return b.hashjoin(plan_of(b, node.outer), b.hash(plan_of(b, node.inner)), node.hj, node.targets)


def rows_of(pool, node):
    """the rows a node delivers: a Scan's qualifying tuples (projected when it has targets), a Join's target list over its pairs,
    an Agg's finalised groups that pass its HAVING, a WindowAgg's rows, a Sort's in order, a Limit's window of them, what a
    Gather passes through.  A caller that computed a node's rows may keep them as node.cached"""
    if getattr(node, "cached", None) is not None:
        return node.cached
    if isinstance(node, Scan):
        rows = [r for r in node.rows if passes(pool, node.qual, r, r)]
        return [tuple(evaluate(pool, t, r, r) for t in node.targets) for r in rows] if node.targets else rows
    if isinstance(node, Agg):
        return agg_rows(pool, node)
    if isinstance(node, Window):
        return window_rows(pool, node)
    if isinstance(node, Sort):
        return sorted(rows_of(pool, node.child), key=functools.cmp_to_key(sort_cmp(node.keys)))
    if isinstance(node, Limit):
        rows = rows_of(pool, node.child)[node.offset or 0:]
        return rows if node.count is None else rows[:node.count]
    if isinstance(node, Gather):
        return rows_of(pool, node.child)
    return [tuple(evaluate(pool, t, o, n) for t in node.targets) for o, n in join_pairs(pool, node)]


def join_pairs(pool, node):
    """(outer row, inner row) per joined row; the side a join null-extends is a row of NULLs"""
    outer, inner = rows_of(pool, node.outer), rows_of(pool, node.inner)
    return hashjoin(pool, outer, inner, node.jointype, node.okeys, node.ikeys, node.qual,
                    len(width_of(node.outer)), len(width_of(node.inner)))


def width_of(node):
    return node.types


def hashjoin(pool, outer, inner, jt, okeys, ikeys, qual, owidth, iwidth):
    """brute() of test_oracle_join generalised to any key expressions and types, with a hash table on the key classes"""
    otypes = [pool.nodes[k].rettype for k in okeys]
    itypes = [pool.nodes[k].rettype for k in ikeys]
    fill_outer = jt in (capi.JOIN_LEFT, capi.JOIN_FULL, capi.JOIN_ANTI, capi.JOIN_LASJ_NOTIN)
    fill_inner = jt in (capi.JOIN_RIGHT, capi.JOIN_FULL)
    anti = jt in (capi.JOIN_ANTI, capi.JOIN_LASJ_NOTIN)
    onull, inull = (None,) * owidth, (None,) * iwidth
    table, inner_keynull = {}, False
    for ii, r in enumerate(inner):
        k = tuple(key_class(t, evaluate(pool, e, r, r)) for t, e in zip(itypes, ikeys))
        if None in k:
            inner_keynull = True
            continue
        table.setdefault(k, []).append(ii)
    if jt == capi.JOIN_LASJ_NOTIN and inner_keynull:
        return []                                                   # x NOT IN (.., NULL, ..) is never true
    out, inner_matched = [], [False] * len(inner)
    for o in outer:
        k = tuple(key_class(t, evaluate(pool, e, o, o)) for t, e in zip(otypes, okeys))
        if None in k:
            if fill_outer and not (jt == capi.JOIN_LASJ_NOTIN and inner):     # NULL NOT IN (non-empty set) is not true
                out.append((o, inull))
            continue
        matched = False
        for ii in table.get(k, ()):
            if not passes(pool, qual, o, inner[ii]):
                continue
            matched = True
            inner_matched[ii] = True
            if anti:
                break
            out.append((o, inner[ii]))
            if jt == capi.JOIN_SEMI:
                break
        if not matched and fill_outer:
            out.append((o, inull))
    if fill_inner:
        out += [(onull, inner[ii]) for ii in range(len(inner)) if not inner_matched[ii]]
    return out


# ---- Agg ----

INT_AGGS = (capi.AGG_SUM_INT4, capi.AGG_MIN_INT4, capi.AGG_MAX_INT4, capi.AGG_MIN_INT8, capi.AGG_MAX_INT8, capi.AGG_MIN_DATE,
            capi.AGG_MAX_DATE)


def aggregate(pool, agg, pairs):
    """{key classes: (zero signs seen per float8 key position, [inputs per aggregate])} over (outer, inner) rows"""
    ktypes = [pool.nodes[agg.grpCol[j]].rettype for j in range(agg.numCols)]
    groups = {}
    for o, n in pairs:
        kv = [evaluate(pool, agg.grpCol[j], o, n) for j in range(agg.numCols)]
        g = tuple(key_class(t, v) for t, v in zip(ktypes, kv))
        signs, inputs = groups.setdefault(g, ({}, [[] for _ in range(agg.numAggs)]))
        for j, (t, v) in enumerate(zip(ktypes, kv)):
            if t == capi.FLOAT8OID and v == 0:
                signs.setdefault(j, set()).add(math.copysign(1, v) < 0)
        for i in range(agg.numAggs):
            a = agg.aggs[i]
            x = 1 if a.aggfnoid == capi.AGG_COUNT_STAR else evaluate(pool, a.arg, o, n)
            if x is not None:
                inputs[i].append(x)
    return groups


def check_groups(got, want, agg, pool, ctx=()):
    """got: [(group key values, aggregate values)] from the device or the oracle, against aggregate()'s groups.  Keys: the
    classes equal; a float8 zero key -0 when every zero of its group was -0 and +0 when every one was +0.  count / int
    aggregates exact; float8 SUM / AVG by _util.check_float8_agg"""
    ktypes = [pool.nodes[agg.grpCol[j]].rettype for j in range(agg.numCols)]
    seen = set()
    for keys, vals in got:
        g = tuple(key_class(t, v) for t, v in zip(ktypes, keys))
        assert g in want and g not in seen, ("group", g) + tuple(ctx)
        seen.add(g)
        signs, inputs = want[g]
        for j, s in signs.items():
            if len(s) == 1:
                assert math.copysign(1, keys[j]) < 0 if s == {True} else math.copysign(1, keys[j]) > 0, ("zero key sign", g) + tuple(ctx)
        for i in range(agg.numAggs):
            fn, xs, x = agg.aggs[i].aggfnoid, inputs[i], vals[i]
            if fn in (capi.AGG_COUNT_STAR, capi.AGG_COUNT_ANY):
                assert x == len(xs), (g, i, x, len(xs)) + tuple(ctx)
                continue
            if not xs:
                assert x is None, (g, i, x) + tuple(ctx)
                continue
            assert x is not None, (g, i) + tuple(ctx)
            if fn == capi.AGG_SUM_INT4:
                assert x == sum(xs), (g, i, x, sum(xs)) + tuple(ctx)
            elif fn in (capi.AGG_MIN_INT4, capi.AGG_MIN_INT8, capi.AGG_MIN_DATE):
                assert x == min(xs), (g, i, x, min(xs)) + tuple(ctx)
            elif fn in (capi.AGG_MAX_INT4, capi.AGG_MAX_INT8, capi.AGG_MAX_DATE):
                assert x == max(xs), (g, i, x, max(xs)) + tuple(ctx)
            else:
                check_float8_agg(fn, x, xs, (g, i) + tuple(ctx))
    assert seen == set(want), ("groups missing", set(want) - seen) + tuple(ctx)


# ---- Sort / Limit ----

def _sort_value(typid, x):
    if typid == capi.FLOAT8OID:
        return (1, 0.0) if x != x else (0, x + 0.0)
    if typid == capi.BPCHAROID:
        return x.rstrip(b" ")
    return x


def sort_cmp(keys):
    """the comparator of Sort keys (col, typid, desc, nulls_first) over rows"""
    def cmp(a, b):
        for k in keys:
            x, y = a[k.col], b[k.col]
            if x is None or y is None:
                if x is None and y is None:
                    continue
                return (-1 if x is None else 1) * (1 if k.nulls_first else -1)
            x, y = _sort_value(k.typid, x), _sort_value(k.typid, y)
            c = (x > y) - (x < y)
            if c:
                return -c if k.desc else c
        return 0
    return cmp


def sort_key_token(keys, r):
    return tuple(None if r[k.col] is None else token(_sort_value(k.typid, r[k.col])) for k in keys)


def zero_token(r, cols):
    """row_token with both float8 zeros one token in the columns `cols`: those whose zeros may carry either sign (a float8 group
    key, a min / max over zeros of both signs, and what is copied or summed from them; the key sign rule is test_gpu_keys').
    Every other column is compared by its bits"""
    return tuple("zero" if c in cols and isinstance(x, float) and x == 0 else token(x) for c, x in enumerate(r))


def check_sort(got, want, keys, ctx=(), tok=row_token):
    """a full Sort: the key sequence is the reference's, and the rows are its multiset"""
    ref = sorted(want, key=functools.cmp_to_key(sort_cmp(keys)))
    assert [sort_key_token(keys, r) for r in got] == [sort_key_token(keys, r) for r in ref], ("key order",) + tuple(ctx)
    assert Counter(map(tok, got)) == Counter(map(tok, want)), ("rows",) + tuple(ctx)


def check_limit(got, want, keys, n, ctx=(), offset=0, tok=row_token):
    """Sort + Limit n (OFFSET offset): the key sequence is that of the reference's sorted rows offset .. offset + n, the rows come
    from the reference multiset, and every reference row whose key sorts strictly inside the window's first and last keys
    (before the last, without an offset) is there as often as in the reference"""
    cmp = sort_cmp(keys)
    ref = sorted(want, key=functools.cmp_to_key(cmp))[offset:offset + n]
    assert len(got) == len(ref), (len(got), n, offset, len(want)) + tuple(ctx)
    assert all(cmp(a, b) <= 0 for a, b in zip(got, got[1:])), ("not sorted",) + tuple(ctx)
    assert [sort_key_token(keys, r) for r in got] == [sort_key_token(keys, r) for r in ref], ("key order",) + tuple(ctx)
    have, pool = Counter(map(tok, got)), Counter(map(tok, want))
    assert not (have - pool), ("rows not in the reference", list((have - pool).items())[:3]) + tuple(ctx)
    if got:
        first, last = got[0], got[-1]
        inside = Counter(tok(r) for r in want if cmp(r, last) < 0 and (not offset or cmp(r, first) > 0))
        assert not (inside - have), ("rows inside the window's keys missing", list((inside - have).items())[:3]) + tuple(ctx)


# ---- Agg over any rows, HAVING, WindowAgg, Sort, Limit, Gather ----

def agg_type(fn):
    """the result type of an aggregate (gg_executor.c agg_result_type)"""
    if fn in (capi.AGG_COUNT_STAR, capi.AGG_COUNT_ANY, capi.AGG_SUM_INT4, capi.AGG_MIN_INT8, capi.AGG_MAX_INT8):
        return capi.INT8OID
    if fn in (capi.AGG_MIN_INT4, capi.AGG_MAX_INT4):
        return capi.INT4OID
    if fn in (capi.AGG_MIN_DATE, capi.AGG_MAX_DATE):
        return capi.DATEOID
    return capi.FLOAT8OID


def _stage(agg, stage):
    a = capi.gg_agg.from_buffer_copy(bytes(agg))
    a.aggstage = stage
    return a


class Agg:
    """Agg over a node's rows: its Vars read the rows of the node below (varno 0), or, when a Join is below, the join's (outer,
    inner) pairs (the executor fuses the two).  having: a qual over the finalised row (Vars varno 0: the grouping columns, then
    one per aggregate), -1 none.  two_stage: the plan is a PARTIAL Agg under a Gather under the FINAL one; the reference's rows
    are the same either way, so only the device tells the two plans apart"""
    def __init__(self, child, agg, having=-1, two_stage=False, pool=None):
        self.child, self.spec, self.having, self.two_stage = child, agg, having, two_stage
        self.types = [pool.nodes[agg.grpCol[j]].rettype for j in range(agg.numCols)] + [agg_type(agg.aggs[i].aggfnoid) for i in range(agg.numAggs)]
        self.agg = agg
        if two_stage:
            self.partial = _stage(agg, capi.AGGSTAGE_PARTIAL)
            self.agg = _stage(agg, capi.AGGSTAGE_FINAL)
            for j in range(agg.numCols):
                self.agg.grpCol[j] = self.types[j]                   # a FINAL Agg's grpCol carries the key type OIDs


def _fmin(xs, largest):
    best = xs[0]
    for x in xs[1:]:
        c = _fcmp(x, best)
        if (c > 0) if largest else (c < 0):
            best = x
    return best


def finalise(fn, xs):
    """an aggregate over its non-NULL inputs, exactly: float8 sums by math.fsum, which the device's sum equals bit for bit when
    every partial sum is exact (the inputs the random plans feed it), -0 when every input is -0; avg that sum over the count"""
    if fn in (capi.AGG_COUNT_STAR, capi.AGG_COUNT_ANY):
        return len(xs)
    if not xs:
        return None
    if fn == capi.AGG_SUM_INT4:
        return sum(xs)
    if fn in (capi.AGG_SUM_FLOAT8, capi.AGG_AVG_FLOAT8):
        s = math.fsum(xs)
        if s == 0 and all(x == 0 and math.copysign(1, x) < 0 for x in xs):
            s = -0.0                                   # float8pl: -0 + -0 is -0 (fsum gives +0)
        return s if fn == capi.AGG_SUM_FLOAT8 else s / len(xs)
    if fn in (capi.AGG_MIN_FLOAT8, capi.AGG_MAX_FLOAT8):
        return _fmin(xs, fn == capi.AGG_MAX_FLOAT8)
    if fn in (capi.AGG_MAX_INT4, capi.AGG_MAX_INT8, capi.AGG_MAX_DATE):
        return max(xs)
    if fn in (capi.AGG_MIN_INT4, capi.AGG_MIN_INT8, capi.AGG_MIN_DATE):
        return min(xs)
    raise AssertionError("aggregate %d is not in the reference" % fn)


def agg_input(pool, node):
    """the (outer, inner) rows an Agg reads"""
    if isinstance(node.child, Join):
        return join_pairs(pool, node.child)
    return [(r, r) for r in rows_of(pool, node.child)]


def agg_rows(pool, node):
    """an Agg's finalised groups (grouping values, then one value per aggregate) whose HAVING is true.  A float8 zero key is -0
    when every zero of its group was -0; a group of zeros of both signs gets +0 (the device may give either: compare such rows
    with zero_token).  An Agg without grouping columns gives one row, over no input too"""
    a = node.spec
    groups = aggregate(pool, a, agg_input(pool, node))
    if not groups and a.numCols == 0:
        groups[()] = ({}, [[] for _ in range(a.numAggs)])
    out = []
    for g, (signs, inputs) in groups.items():
        keys = []
        for j, k in enumerate(g):
            if k == "nan":
                k = float("nan")
            elif node.types[j] == capi.FLOAT8OID and k == 0:
                k = -0.0 if signs.get(j) == {True} else 0.0
            keys.append(k)
        out.append(tuple(keys) + tuple(finalise(a.aggs[i].aggfnoid, inputs[i]) for i in range(a.numAggs)))
    return [r for r in out if passes(pool, node.having, r, r)]


MASK64 = (1 << 64) - 1


def datum_word(typid, x):
    """a non-NULL value as its datum-row word: int4 / date sign-extended, int8 / timestamp, float8 bits, bool 0 / 1, a string of
    at most 8 bytes packed LSB-first (bpchar blank-stripped, as the rows hold it)"""
    if typid == capi.FLOAT8OID:
        return struct.unpack("<Q", struct.pack("<d", x))[0]
    if typid in STRINGS:
        assert len(x) <= 8, x
        return int.from_bytes(x.ljust(8, b"\0"), "little")
    return int(x) & MASK64


def word_value(typid, u):
    """datum_word's inverse"""
    u = int(u)
    if typid == capi.FLOAT8OID:
        return struct.unpack("<d", struct.pack("<Q", u))[0]
    if typid in STRINGS:
        return u.to_bytes(8, "little").rstrip(b"\0")
    if typid in (capi.INT4OID, capi.DATEOID):
        u &= 0xFFFFFFFF
        return u - (1 << 32) if u >> 31 else u
    return u - (1 << 64) if u >> 63 else u


def encode_rows(types, rows):
    """rows of Python values -> datum-row words uint64 [n][1 + ncols] (word 0 the NULL mask)"""
    out = np.zeros((len(rows), 1 + len(types)), dtype=np.uint64)
    for i, r in enumerate(rows):
        mask = 0
        for c, (t, x) in enumerate(zip(types, r)):
            if x is None:
                mask |= 1 << c
            else:
                out[i, 1 + c] = datum_word(t, x)
        out[i, 0] = mask
    return out


def decode_rows(types, words):
    return [tuple(None if (int(w[0]) >> c) & 1 else word_value(t, w[1 + c]) for c, t in enumerate(types)) for w in words]


class Window:
    """WindowAgg over the rows of `child` in their order (a Sort on part + order, possibly under other WindowAggs; none when it
    has no keys): part / order 0-based columns, frame FRAMEOPTION_* bits, funcs (winfnoid, wintype, [arg roots]); qual over the
    output row (the child's columns, then one per function; Vars varno 0), -1 none"""
    def __init__(self, child, part, order, frame, funcs, qual=-1):
        self.child, self.funcs, self.qual = child, list(funcs), qual
        self.win = capi.make_window(part, order, frame, self.funcs)
        self.types = list(child.types) + [f[1] for f in self.funcs]


def window_rows(pool, node):
    """the child's rows encoded as datum rows, windowed by tests/window_ref.c, decoded, then through the qual; a window_ref ERROR
    (ntile / nth_value of a Const <= 0 over at least one row) raises RefError with the device's code"""
    from _window import ref_window
    rows = rows_of(pool, node.child)
    rc, out, msg = ref_window(node.win, node.child.types, pool, encode_rows(node.child.types, rows))
    if rc:
        raise RefError(rc, msg)
    return [r for r in decode_rows(node.types, out) if passes(pool, node.qual, r, r)]


class Sort:
    def __init__(self, child, keys):
        self.child, self.keys, self.types = child, list(keys), child.types


class Limit:
    """LIMIT count OFFSET offset over the node below (None: no count / no offset)"""
    def __init__(self, child, count, offset=None):
        self.child, self.count, self.offset, self.types = child, count, offset, child.types


class Gather:
    """a Gather Motion at one segment: the rows below, as host rows"""
    def __init__(self, child):
        self.child, self.types = child, child.types


# ---- the pin: single joins against the oracle's pairs and aggregates ----

def tid_index(pages):
    """tid (block << 16 | offnum) -> row index in page_rows order"""
    idx, k = {}, 0
    for b in range(pages.size // capi.GG_BLCKSZ):
        for off in range(1, po.lib().or_page_nitems(po._ptr(pages[b * capi.GG_BLCKSZ:(b + 1) * capi.GG_BLCKSZ])) + 1):
            idx[(b << 16) | off] = k
            k += 1
    return idx


def oracle_rows(pool, node, opages, ipages):
    """the oracle's pairs of a single join (po.hashjoin_tids), through the same target list"""
    orows, irows = node.outer.rows, node.inner.rows
    oi, ii = tid_index(opages), tid_index(ipages)
    onull, inull = (None,) * node.outer.desc.natts, (None,) * node.inner.desc.natts
    pairs = po.hashjoin_tids(capi.make_scan(node.outer.desc, node.outer.qual), capi.make_scan(node.inner.desc, node.inner.qual),
                             node.hj, pool, opages, ipages)
    out = []
    for a, b in pairs:
        o = orows[oi[int(a)]] if a >= 0 else onull
        n = irows[ii[int(b)]] if (b >= 0 and node.jointype not in (capi.JOIN_SEMI, capi.JOIN_ANTI, capi.JOIN_LASJ_NOTIN)) else inull
        out.append(tuple(evaluate(pool, t, o, n) for t in node.targets))
    return out


def aggrow_values(pool, agg, r):
    """an oracle gg_aggrow as (key values, aggregate values)"""
    keys = []
    for j in range(agg.numCols):
        t = pool.nodes[agg.grpCol[j]].rettype
        if r.keyisnull[j]:
            keys.append(None)
        elif t == capi.FLOAT8OID:
            keys.append(struct.unpack("<d", struct.pack("<q", r.key[j]))[0])
        elif t in STRINGS:
            keys.append(capi.unpack_str(r.key[j], r.keylen[j]).encode("latin1"))
        elif t in (capi.INT4OID, capi.DATEOID):
            keys.append(int(np.uint32(r.key[j] & 0xFFFFFFFF).astype(np.int32)))
        else:
            keys.append(int(r.key[j]))
    vals = []
    for i in range(agg.numAggs):
        a = r.agg[i]
        fn = agg.aggs[i].aggfnoid
        if a.isnull:
            vals.append(None)
        elif agg_type(fn) == capi.FLOAT8OID:
            vals.append(a.f[0])
        else:
            vals.append(int(a.i))
    return keys, vals


def _key_rel(n, seed):
    desc, pages, _, _ = key_relation(n, seed)
    return desc, pages, page_rows(desc, pages)


@pytest.fixture(scope="module")
def key_rels():
    return _key_rel(150, 31), _key_rel(64, 32), _key_rel(44, 33)


def key_targets(p, side, jt):
    """every column of the outer side, and of the inner side where the join type has one"""
    t = [p.var(col(c), TYPID[c], 0) for c in COLS]
    if jt in BOTH_SIDES:
        t += [p.var(col(c), TYPID[c], 1) for c in COLS]
    return t


def key_agg(p, jt):
    aggs = [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_FLOAT8, p.var(col("v"), capi.FLOAT8OID, 0)),
            (capi.AGG_AVG_FLOAT8, p.var(col("v"), capi.FLOAT8OID, 0)), (capi.AGG_MIN_DATE, p.var(col("date"), capi.DATEOID, 0)),
            (capi.AGG_SUM_INT4, p.var(col("int4"), capi.INT4OID, 0))]
    if jt in BOTH_SIDES:
        aggs += [(capi.AGG_COUNT_ANY, p.var(col("w"), capi.INT8OID, 1)), (capi.AGG_MAX_INT8, p.var(col("w"), capi.INT8OID, 1)),
                 (capi.AGG_MAX_INT4, p.var(col("int4"), capi.INT4OID, 1))]
    return capi.make_agg(capi.AGGSTAGE_NORMAL, [p.var(col("z"), capi.INT4OID, 0), p.var(col("float8"), capi.FLOAT8OID, 0)], aggs)


@pytest.mark.parametrize("pair", KEYPAIRS, ids=["%s=%s" % kp for kp in KEYPAIRS])
def test_single_joins_over_the_key_relation_match_the_oracle(key_rels, pair):
    (od, opages, orows), (idesc, ipages, irows), _ = key_rels
    ok, ik = pair
    for jt in ALL_JOINTYPES:
        for nkeys in (1, 2):
            p = capi.ExprPool()
            okeys, ikeys = [p.var(col(ok), TYPID[ok], 0)], [p.var(col(ik), TYPID[ik], 1)]
            qual = -1
            if nkeys == 2:
                okeys.append(p.var(col("z"), capi.INT4OID, 0))
                ikeys.append(p.var(col("z"), capi.INT4OID, 1))
                qual = p.func(capi.F_FLOAT8GT, capi.BOOLOID, p.var(col("v"), capi.FLOAT8OID, 1), p.const(capi.FLOAT8OID, -20.0))
            node = Join(Scan(0, od, orows), Scan(1, idesc, irows), jt, okeys, ikeys, qual, key_targets(p, 0, jt), p.pool)
            ctx = (pair, jt, nkeys)
            want = Counter(map(row_token, rows_of(p.pool, node)))
            assert want == Counter(map(row_token, oracle_rows(p.pool, node, opages, ipages))), ctx
            agg = key_agg(p, jt)
            orc, _ = po.hashjoin_agg(capi.make_scan(od), capi.make_scan(idesc, -1), node.hj, agg, p.pool, opages, ipages)
            check_groups([aggrow_values(p.pool, agg, r) for r in orc], aggregate(p.pool, agg, join_pairs(p.pool, node)), agg, p.pool, ctx)


@pytest.mark.parametrize("jointype", ALL_JOINTYPES)
def test_single_joins_over_small_relations_match_the_oracle(jointype):
    odesc, idesc, _, _, _, _, opages, ipages = small_relations()
    orows, irows = page_rows(odesc, opages), page_rows(idesc, ipages)
    for nkeys in (1, 2):
        for with_qual in (False, True):
            p, _, _, hj = join_nodes(odesc, idesc, jointype, nkeys, with_qual)
            okeys = [hj.outerkey[k] for k in range(nkeys)]
            ikeys = [hj.innerkey[k] for k in range(nkeys)]
            targets = [p.var(a + 1, odesc.attrs[a].atttypid, 0) for a in range(3)]
            if jointype in BOTH_SIDES:
                targets += [p.var(a + 1, idesc.attrs[a].atttypid, 1) for a in range(3)]
            node = Join(Scan(0, odesc, orows), Scan(1, idesc, irows), jointype, okeys, ikeys, hj.joinqual, targets, p.pool)
            ctx = (jointype, nkeys, with_qual)
            assert Counter(map(row_token, rows_of(p.pool, node))) == Counter(map(row_token, oracle_rows(p.pool, node, opages, ipages))), ctx
            agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [p.var(2, capi.BPCHAROID, 0)],
                                [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_FLOAT8, p.var(3, capi.FLOAT8OID, 0)), (capi.AGG_COUNT_ANY, p.var(3, capi.FLOAT8OID, 0))]
                                + ([(capi.AGG_SUM_INT4, p.var(3, capi.INT4OID, 1)), (capi.AGG_MIN_INT4, p.var(1, capi.INT4OID, 1))] if jointype in BOTH_SIDES else []))
            orc, _ = po.hashjoin_agg(capi.make_scan(odesc), capi.make_scan(idesc), node.hj, agg, p.pool, opages, ipages)
            check_groups([aggrow_values(p.pool, agg, r) for r in orc], aggregate(p.pool, agg, join_pairs(p.pool, node)), agg, p.pool, ctx)


# ---- the pin: two-level trees against the oracle's single join over the lower join's rows as pages ----

LOWER_COLS = ["int4", "int8", "float8", "bpchar", "varchar", "text", "date", "z", "id"]


@pytest.mark.parametrize("lower_jt", [capi.JOIN_INNER, capi.JOIN_LEFT, capi.JOIN_RIGHT, capi.JOIN_FULL])
@pytest.mark.parametrize("rows_side", ["outer", "inner"])
def test_two_level_trees_match_the_oracle_over_the_lower_rows(key_rels, lower_jt, rows_side):
    (ad, apages, arows), (bd, bpages, brows), (cd, cpages, crows) = key_rels
    def lower_of(p):
        # lower: A ⋈ B on int8, projecting A's columns and (null-extended under LEFT / FULL) B's
        targets = [p.var(col(c), TYPID[c], 0) for c in LOWER_COLS[:5]] + [p.var(col(c), TYPID[c], 1) for c in LOWER_COLS]
        return Join(Scan(0, ad, arows), Scan(1, bd, brows), lower_jt, [p.var(col("int8"), capi.INT8OID, 0)],
                    [p.var(col("int8"), capi.INT8OID, 1)], targets=targets, pool=p.pool)
    p = capi.ExprPool()
    lower = lower_of(p)
    lrows = rows_of(p.pool, lower)
    lpages = rows_pages(lower.types, lrows)
    lrows_paged = page_rows(rows_desc(lower.types), lpages)
    assert Counter(map(row_token, lrows_paged)) == Counter(map(row_token, lrows))
    for upper_jt in ALL_JOINTYPES:
        for okey, ckey in (("int4", "int8"), ("float8", "float8"), ("bpchar", "bpchar"), ("varchar", "text")):
            p = capi.ExprPool()
            lower = lower_of(p)
            # upper key: the lower rows' B column (position 5 + index) against C's column
            lv, cs = 5 + LOWER_COLS.index(okey), 2 if rows_side == "outer" else 0
            rv = 0 if rows_side == "outer" else 1
            lkey, ckey_e = p.var(lv + 1, lower.types[lv], rv), p.var(col(ckey), TYPID[ckey], 1 - rv)
            ut = [p.var(k + 1, lower.types[k], rv) for k in (0, 2, 5, lv)]
            ct = [p.var(col(c), TYPID[c], 1 - rv) for c in ("id", "float8", "varchar")]
            cscan = Scan(cs, cd, crows)
            if rows_side == "outer":
                upper = Join(lower, cscan, upper_jt, [lkey], [ckey_e], targets=ut + (ct if upper_jt in BOTH_SIDES else []), pool=p.pool)
                flat = Join(Scan(0, rows_desc(lower.types), lrows_paged), cscan, upper_jt, [lkey], [ckey_e], targets=upper.targets, pool=p.pool)
                pages = (lpages, cpages)
            else:
                upper = Join(cscan, lower, upper_jt, [ckey_e], [lkey], targets=ct + (ut if upper_jt in BOTH_SIDES else []), pool=p.pool)
                flat = Join(cscan, Scan(1, rows_desc(lower.types), lrows_paged), upper_jt, [ckey_e], [lkey], targets=upper.targets, pool=p.pool)
                pages = (cpages, lpages)
            ctx = (lower_jt, rows_side, upper_jt, okey, ckey)
            want = Counter(map(row_token, rows_of(p.pool, upper)))
            assert want == Counter(map(row_token, oracle_rows(p.pool, flat, *pages))), ctx


# ---- the pin: Agg over any rows, HAVING and WindowAgg ----

def test_agg_and_having_reproduce_the_select_having_goldens():
    """the reference's select_having rows that test_gpu_having.py runs on the device"""
    import json
    import os
    g = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "having_expected.json")))
    types = [capi.INT4OID, capi.INT4OID, capi.BPCHAROID, capi.BPCHAROID]
    rows = page_rows(rows_desc(types), rows_pages(types, [[a, b, c.encode(), d.encode()] for a, b, c, d in g["test_having"]]))
    p = capi.ExprPool()
    a, bb, c = p.var(1, capi.INT4OID), p.var(2, capi.INT4OID), p.var(3, capi.BPCHAROID)
    I8, I4 = capi.INT8OID, capi.INT4OID
    q5 = capi.make_agg(capi.AGGSTAGE_NORMAL, [], [(capi.AGG_MIN_INT4, a), (capi.AGG_MAX_INT4, a)])
    queries = [(capi.make_agg(capi.AGGSTAGE_NORMAL, [bb, c], [(capi.AGG_COUNT_STAR, -1)]), p.func(capi.F_INT8EQ, capi.BOOLOID, p.var(3, I8), p.const(I8, 1))),
               (capi.make_agg(capi.AGGSTAGE_NORMAL, [bb, c], []), p.func(capi.F_INT4EQ, capi.BOOLOID, p.var(1, I4), p.const(I4, 3))),
               (capi.make_agg(capi.AGGSTAGE_NORMAL, [c], [(capi.AGG_MAX_INT4, a), (capi.AGG_COUNT_STAR, -1), (capi.AGG_MIN_INT4, a)]),
                p.boolop(capi.E_OR, p.func(capi.F_INT8GT, capi.BOOLOID, p.var(3, I8), p.const(I8, 2)), p.func(capi.F_INT4EQ, capi.BOOLOID, p.var(4, I4), p.var(2, I4)))),
               (q5, p.func(capi.F_INT4EQ, capi.BOOLOID, p.var(1, I4), p.var(2, I4))),
               (q5, p.func(capi.F_INT4LT, capi.BOOLOID, p.var(1, I4), p.var(2, I4)))]
    for (agg, q), want in zip(queries, g["queries"]):
        got = rows_of(p.pool, Agg(Scan(0, rows_desc(types), rows), agg, q, pool=p.pool))
        got = sorted(tuple(v.decode() if isinstance(v, bytes) else v for v in r[:2]) for r in got)
        assert got == sorted(tuple(r) for r in want["rows"]), want


def _rows_agg(p, types):
    """an Agg over rows of these types: grouped by the first int4 / bool / float8 / string columns; count, count(x), int4 sum and
    min / max, float8 min / max, and the float8 sum / avg of `exact` (a column of multiples of 1/4)"""
    v = lambda c: p.var(c + 1, types[c])                                        # noqa: E731
    first = lambda ts: next(c for c, t in enumerate(types) if t in ts)          # noqa: E731
    keys = [v(first((capi.INT4OID,))), v(first((capi.BOOLOID, capi.BPCHAROID, capi.TEXTOID, capi.FLOAT8OID)))]
    i4, f8 = first((capi.INT4OID,)), first((capi.FLOAT8OID,))
    ex_ = len(types) - 1
    aggs = [(capi.AGG_COUNT_STAR, -1), (capi.AGG_COUNT_ANY, v(f8)), (capi.AGG_SUM_INT4, v(i4)), (capi.AGG_MIN_INT4, v(i4)),
            (capi.AGG_MAX_INT4, v(i4)), (capi.AGG_MIN_FLOAT8, v(f8)), (capi.AGG_MAX_FLOAT8, v(f8)),
            (capi.AGG_SUM_FLOAT8, v(ex_)), (capi.AGG_AVG_FLOAT8, v(ex_))]
    return capi.make_agg(capi.AGGSTAGE_NORMAL, keys, aggs)


@pytest.mark.parametrize("rows_kind", ["scan", "join", "window"])
def test_agg_over_rows_matches_the_oracle(key_rels, rows_kind):
    """the reference Agg over scan rows, join rows and window rows equals the oracle's grouping over the same rows written as
    heap pages (the last column of every row set is an exact float8 column: its sums are exact, in any order)"""
    (ad, _, arows), (bd, _, brows), _ = key_rels
    p = capi.ExprPool()
    names = ["id", "int4", "bool", "float8", "bpchar", "date", "v"]
    scan = Scan(0, ad, arows, targets=[p.var(col(c), TYPID[c]) for c in names], pool=p.pool)
    if rows_kind == "scan":
        node = scan
    elif rows_kind == "join":
        node = Join(Scan(0, ad, arows), Scan(1, bd, brows), capi.JOIN_FULL, [p.var(col("z"), capi.INT4OID, 0)], [p.var(col("z"), capi.INT4OID, 1)],
                    targets=[p.var(col("int4"), capi.INT4OID, 1), p.var(col("text"), capi.TEXTOID, 0), p.var(col("float8"), capi.FLOAT8OID, 1),
                             p.func(capi.F_FLOAT8MUL, capi.FLOAT8OID, p.var(col("v"), capi.FLOAT8OID, 0), p.const(capi.FLOAT8OID, -2.0))], pool=p.pool)
    else:
        keys = [capi.make_sortkey(2, capi.BOOLOID), capi.make_sortkey(1, capi.INT4OID), capi.make_sortkey(0, capi.INT4OID)]
        x = p.var(7, capi.FLOAT8OID)
        node = Window(Sort(scan, keys), [2], [1], capi.FRAMEOPTION_DEFAULTS,
                      [(capi.WF_RANK, capi.INT8OID, []), (capi.WF_LAG, capi.INT4OID, [p.var(2, capi.INT4OID)]), (capi.AGG_SUM_FLOAT8, capi.FLOAT8OID, [x])])
    rows = rows_of(p.pool, node)
    types = node.types
    if rows_kind == "window":                       # the window's int4 lag, then its exact sum last
        types, rows = types[:7] + [types[8], types[9]], [r[:7] + (r[8], r[9]) for r in rows]
    agg = _rows_agg(p, types)
    desc = rows_desc(types)
    want = rows_of(p.pool, Agg(Scan(0, desc, rows), agg, pool=p.pool))
    orc, _, _ = po.seqscan_agg(capi.make_scan(desc), agg, p.pool, rows_pages(types, rows), cap=len(rows) + 1)
    got = [tuple(k) + tuple(v) for k, v in (aggrow_values(p.pool, agg, r) for r in orc)]
    assert len(want) > 3
    mm = {agg.numCols + 5, agg.numCols + 6}          # min / max(float8): the sign of a zero over zeros of both signs is open
    assert Counter(zero_token(r, mm) for r in got) == Counter(zero_token(r, mm) for r in want)


@pytest.mark.parametrize("frame", ["range_up_cr", "rows_up_cr", "range_cr_uf", "rows_cr_cr"])
def test_window_step_matches_the_naive_statement(frame):
    """the reference's WindowAgg step (rows sorted by the reference Sort, encoded, windowed, decoded) over order keys with ties,
    NULLs, -0 and NaN, against _window.naive_window's statement of each function over the same sorted rows"""
    from _window import FRAMES, all_funcs, naive_window
    from test_window_rules import _same
    rng = np.random.default_rng(len(frame))
    fl = [-0.0, 0.0, 1.5, float("nan"), -2.0, float("-inf")]
    strs = [b"", b"a", b"ab", b"abcdefgh"]
    types = [capi.INT4OID, capi.FLOAT8OID, capi.BPCHAROID, capi.FLOAT8OID, capi.INT4OID, capi.INT8OID]
    rows = [(None if rng.random() < 0.1 else int(rng.integers(-2, 2)), None if rng.random() < 0.1 else fl[int(rng.integers(0, 6))],
             strs[int(rng.integers(0, 4))], None if rng.random() < 0.2 else float(rng.integers(-400, 400)) / 4,
             None if rng.random() < 0.2 else int(rng.integers(-2 ** 31, 2 ** 31)), int(rng.integers(-2 ** 62, 2 ** 62))) for _ in range(700)]
    src = Scan(0, rows_desc(types), rows)
    for part, order in (([0], [1]), ([], [1, 2]), ([2], [])):
        keys = [capi.make_sortkey(c, types[c], bool(rng.random() < 0.5), bool(rng.random() < 0.5)) for c in part + order]
        for g in range(3):
            p = capi.ExprPool()
            funcs = all_funcs(p, len(types), types, [0, 1, 2], [3, 4, 5])[g]
            child = Sort(src, keys) if keys else src
            node = Window(child, part, order, FRAMES[frame], funcs)
            err, want = naive_window(node.win, types, p.pool, encode_rows(types, rows_of(p.pool, child)))
            if err:
                with pytest.raises(RefError) as e:
                    rows_of(p.pool, node)
                assert e.value.code == capi.ERR_WINDOW_ARG
                continue
            got = rows_of(p.pool, node)
            assert len(got) == len(want) == len(rows)
            for j, (r, w) in enumerate(zip(got, want)):
                for i, b in enumerate(w):
                    fn, t = funcs[i][0], funcs[i][1]
                    if isinstance(b, int) and capi.WF_LAG <= fn <= capi.WF_NTH_VALUE:
                        b = word_value(t, b)                   # the naive statement returns a value function's input word
                    assert _same(r[len(types) + i], b, fn), (part, order, g, j, i, fn, r[len(types) + i], b)


def test_plan_tree_generator_draws_every_composition():
    """every seed of test_gpu_plan_trees.py drawn here, with its reference answer: no draw fails, and each composition the
    device run must cover is drawn by at least two seeds"""
    import test_gpu_plan_trees as g
    seen = Counter()
    for seed in g.SEEDS:
        d, top, want = g.draw_plan(seed, g.host_rels())
        assert want[0] == "rows" or want[1] in (ERR_DIV_ZERO, capi.ERR_WINDOW_ARG), (seed, want)
        seen.update(d.tags)
    assert all(seen[c] >= 2 for c in g.COMPOSITIONS), seen
