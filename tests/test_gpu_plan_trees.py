"""Random plans of Agg (with or without HAVING, one-stage or PARTIAL -> Gather -> FINAL), WindowAgg, HashJoin, Sort, Limit and
Gather on the device, through the executor-node surface, against the row-at-a-time reference of test_join_tree_reference.py.

Each seed builds its plan around one composition of these nodes (COMPOSITIONS: where one node hands its rows to another) and
stacks random nodes above it, over base relations of the key relation at join-tree sizes and, for about a quarter of the seeds, a
50 000-row one whose partitions and groups run past the window tiles and the row filter's blocks.  Rules that make every answer
exactly checkable: float8 sums and averages read only exact columns (multiples of 1/4 and their sums, far below 2^53), and a
WindowAgg draws an order-dependent function only when the Sort below it orders its rows totally (unique columns appended).  A
plan the executor refuses must be refused with GG_ERR_UNSUPPORTED; a reference ERROR must surface with the same code.  Each seed
draws the operator's memory as the join trees do, so that joins run batched and Sorts of host rows in runs under the new
compositions.  Each plan that runs is checked, its top node's instrumentation must count the rows it returned, and after a ReScan
the rows pass the same check and are the first run's, bit for bit (under a Limit, which rows tied at the window's edge come back
is the run's choice).  Rows are compared by their bits, except that both float8 zeros are one value in the columns whose zero
sign is open: a float8 group key or min / max over zeros of both signs, and what is copied or summed from one."""
import ctypes as C
from collections import Counter

import numpy as np
import pytest

from greengage_b200 import capi, executor as ex
from test_gpu_join_rows import datum
from test_gpu_join_trees import join_states
from test_gpu_keys import COLS, TYPID, col, key_relation
from test_join_tree_reference import (Agg, Gather, Join, Limit, RefError, Scan, Sort, Window, check_limit, check_sort,
                                      page_rows, plan_of, row_token, rows_of, zero_token)

pytestmark = pytest.mark.gpu

UNSUPPORTED = -6                                          # GG_ERR_UNSUPPORTED
OUTER_ONLY = (capi.JOIN_SEMI, capi.JOIN_ANTI, capi.JOIN_LASJ_NOTIN)
SMALL = ((60, 41), (40, 42), (30, 43), (24, 44))          # relids 0..3
LARGE = (50_000, 45)                                      # relid 4
MAX_ROWS = 60_000
SEEDS = list(range(40))
# the compositions every run of the seeds must cover (each seed's plan is built around COMPOSITIONS[seed % len])
COMPOSITIONS = ["win/scan", "win/join", "win/agg", "win/having-sort", "win/having-nokeys", "win/win-prefix", "win/gather",
                "winqual/limit", "winqual/sort", "agg/win", "having/win", "join/win-outer", "join/win-inner", "join/having-win",
                "final-having/sort-win", "gather/win", "gather/having"]
RANGE_FRAMES = ("range_up_cr", "range_up_uf", "range_cr_uf", "range_cr_cr")
FRAMES_ALL = RANGE_FRAMES + ("rows_up_cr", "rows_up_uf", "rows_cr_uf", "rows_cr_cr")
EXACT_V = (100.0, 0.25)                                   # v: |x| <= 100, multiples of 1/4


# ---- base relations (host side; the device copies are made by the fixture) ----

class HostRels:
    def __init__(self, large):
        tables = [key_relation(n, s)[:2] for n, s in SMALL + ((LARGE,) if large else ())]
        self.desc = [d for d, _ in tables]
        self.pages = [pg for _, pg in tables]
        self.rows = [page_rows(d, pg) for d, pg in tables]


_host = {}


def host_rels():
    if "r" not in _host:
        _host["r"] = HostRels(True)
    return _host["r"]


# ---- drawing ----

class R:
    """a drawn node with what the drawing rules need: its exact float8 columns {col: (bound, ulp)}, the columns that make its
    rows unique (None: none known), what kind of node it is, and the float8 columns whose zeros may carry either sign (amb)"""
    def __init__(self, node, exact, uniq, kind, amb=()):
        self.node, self.exact, self.uniq, self.kind, self.amb = node, exact, uniq, kind, frozenset(amb)
        self.types = node.types


class Redraw(Exception):
    pass


class PoolFull(Exception):
    pass


class Pool(capi.ExprPool):
    """an ExprPool that says it is full with PoolFull, so that a plan too large for it is drawn again"""
    def _new(self):
        if self.pool.nnodes >= capi.GG_MAX_EXPR_NODES:
            raise PoolFull()
        return super()._new()


MINMAX_F8 = (capi.AGG_MIN_FLOAT8, capi.AGG_MAX_FLOAT8)
FOLLOWS_ARG = tuple(range(capi.WF_LAG, capi.WF_NTH_VALUE + 1)) + (capi.AGG_SUM_FLOAT8, capi.AGG_AVG_FLOAT8)


def sign_token(amb):
    """the row token of a node's rows: float8 by their bits, but both zeros one token in the columns amb"""
    return lambda r: zero_token(r, amb)


def _exact_ok(b):
    return b[0] / b[1] < 2.0 ** 50


def rows(p, r):
    """the reference rows of a drawn node, computed once (a RefError propagates); Redraw past MAX_ROWS"""
    n = r.node if isinstance(r, R) else r
    if getattr(n, "cached", None) is None:
        got = rows_of(p.pool, n)
        if len(got) > MAX_ROWS:
            raise Redraw()
        n.cached = got
    return n.cached


class Draw:
    def __init__(self, rng, rels, large):
        self.rng, self.rels, self.large, self.p = rng, rels, large, Pool()
        self.tags, self.ops, self.failed = set(), [], False

    def size(self, r):
        """r, after its reference rows are computed once (Redraw past MAX_ROWS); after a reference ERROR nothing above is computed"""
        if not self.failed:
            try:
                rows(self.p, r)
            except RefError:
                self.failed = True
        return r

    def pick(self, xs):
        return xs[int(self.rng.integers(0, len(xs)))]

    def chance(self, x):
        return bool(self.rng.random() < x)

    def relid(self):
        return 4 if self.large and self.chance(0.6) else int(self.rng.integers(0, 4))

    # bases
    def scan_rows(self, relid=None):
        relid = self.relid() if relid is None else relid
        others = [c for c in COLS if c != "id"]
        cols = ["id"] + [others[int(k)] for k in self.rng.choice(len(others), size=int(self.rng.integers(3, 8)), replace=False)]
        t = [self.p.var(col(c), TYPID[c]) for c in cols]
        node = Scan(relid, self.rels.desc[relid], self.rels.rows[relid], targets=t, pool=self.p.pool)
        return R(node, {i: EXACT_V for i, c in enumerate(cols) if c == "v"}, [0], "scan")

    def plain_scan(self, relid=None):
        relid = self.relid() if relid is None else relid
        node = Scan(relid, self.rels.desc[relid], self.rels.rows[relid])
        return R(node, {col("v") - 1: EXACT_V}, [col("id") - 1], "base")

    # HashJoin
    def join(self, outer, inner, fused=False):
        p, jt = self.p, int(self.rng.integers(0, 7))
        ot, it = outer.types, inner.types
        pairs = [(a, b) for a, ta in enumerate(ot) for b, tb in enumerate(it) if tb in partners(ta)]
        if not pairs:
            raise Redraw()
        ids = [(a, b) for a, b in pairs if (outer.uniq and a in outer.uniq) or (inner.uniq and b in inner.uniq)]
        if ids and (self.large or self.chance(0.3)):
            pairs = ids                                             # unique columns as keys keep the large joins small
        idx = self.rng.choice(len(pairs), size=min(int(self.rng.integers(1, 3)), len(pairs)), replace=False)
        ok = [p.var(pairs[i][0] + 1, ot[pairs[i][0]], 0) for i in idx]
        ik = [p.var(pairs[i][1] + 1, it[pairs[i][1]], 1) for i in idx]
        qual = -1
        if self.chance(0.3):
            side, varno = (outer, 0) if self.chance(0.5) else (inner, 1)
            i4 = [c for c, t in enumerate(side.types) if t == capi.INT4OID]
            if i4:
                qual = p.func(capi.F_INT4LT, capi.BOOLOID, p.var(self.pick(i4) + 1, capi.INT4OID, varno), p.const(capi.INT4OID, self.pick([0, 2, 1000])))
        if fused:
            return Join(outer.node, inner.node, jt, ok, ik, qual, (), p.pool), outer, inner, jt
        both = jt not in OUTER_ONLY
        want = [(0, c) for c in (outer.uniq or [])] + ([(1, c) for c in (inner.uniq or [])] if both else [])
        rest = [(0, c) for c in range(len(ot))] + ([(1, c) for c in range(len(it))] if both else [])
        rest = [x for x in rest if x not in want]
        extra = [rest[int(k)] for k in self.rng.choice(len(rest), size=min(len(rest), int(self.rng.integers(1, 8))), replace=False)]
        targets, exact, uniq, amb = [], {}, [], set()
        for varno, c in want + extra:
            side = outer if varno == 0 else inner
            v = p.var(c + 1, side.types[c], varno)
            if c in side.amb:
                amb.add(len(targets))
            if c in side.exact:
                b = side.exact[c]
                if self.chance(0.4):
                    f, k = self.pick([(capi.F_FLOAT8PL, 0.5), (capi.F_FLOAT8MUL, 0.5), (capi.F_FLOAT8MUL, -2.0), (capi.F_FLOAT8MI, 0.25)])
                    v = p.func(f, capi.FLOAT8OID, v, p.const(capi.FLOAT8OID, k))
                    b = (b[0] * 2 + 1, min(b[1], 0.25) / (2 if k == 0.5 and f == capi.F_FLOAT8MUL else 1))
                exact[len(targets)] = b
            if (varno, c) in want:
                uniq.append(len(targets))
            targets.append(v)
        node = Join(outer.node, inner.node, jt, ok, ik, qual, targets, p.pool)
        self.ops.append("join")
        return self.size(R(node, exact, uniq if (outer.uniq is not None and (inner.uniq is not None or not both)) else None, "join", amb))

    # Agg
    def agg(self, src, having=False, two_stage=False, nkeys=None):
        """an Agg over src (an R; a Join is fused: its columns are the two sides' with varno 0 / 1)"""
        p = self.p
        if isinstance(src, tuple):
            j, o, i, jt = src
            cols = [(0, c, t, o.exact.get(c)) for c, t in enumerate(o.types)] + \
                   ([(1, c, t, i.exact.get(c)) for c, t in enumerate(i.types)] if jt not in OUTER_ONLY else [])
            child, sides = j, (o, i)
        else:
            cols = [(0, c, t, src.exact.get(c)) for c, t in enumerate(src.types)]
            child, sides = src.node, (src,)
        nk = int(self.rng.integers(1 if two_stage else 0, 3)) if nkeys is None else nkeys
        keyc = [cols[int(k)] for k in self.rng.choice(len(cols), size=min(nk, len(cols)), replace=False)]
        if self.large and nk and self.chance(0.5):
            ids = [x for x in cols if x[2] == capi.INT4OID]
            keyc[0] = ids[0] if ids else keyc[0]
        keys = [p.var(c + 1, t, v) for v, c, t, _ in keyc]
        aggs, exact = [(capi.AGG_COUNT_STAR, -1)], {}
        v, c, t, _ = self.pick(cols)
        aggs.append((capi.AGG_COUNT_ANY, p.var(c + 1, t, v)))
        for types, fns in (((capi.INT4OID,), (capi.AGG_SUM_INT4, capi.AGG_MIN_INT4, capi.AGG_MAX_INT4)),
                           ((capi.INT8OID,), (capi.AGG_MIN_INT8, capi.AGG_MAX_INT8)), ((capi.DATEOID,), (capi.AGG_MIN_DATE, capi.AGG_MAX_DATE)),
                           ((capi.FLOAT8OID,), (capi.AGG_MIN_FLOAT8, capi.AGG_MAX_FLOAT8))):
            xs = [x for x in cols if x[2] in types]
            if xs and self.chance(0.7):
                v, c, t, _ = self.pick(xs)
                aggs.append((self.pick(fns), p.var(c + 1, t, v)))
        ex_cols = [x for x in cols if x[3] is not None]
        if ex_cols:
            v, c, t, b = self.pick(ex_cols)
            if _exact_ok((b[0] * MAX_ROWS, b[1])):
                exact[len(keys) + len(aggs)] = (b[0] * MAX_ROWS, b[1])
                aggs += [(capi.AGG_SUM_FLOAT8, p.var(c + 1, capi.FLOAT8OID, v)), (capi.AGG_AVG_FLOAT8, p.var(c + 1, capi.FLOAT8OID, v))]
        a = capi.make_agg(capi.AGGSTAGE_NORMAL, keys, aggs, num_groups=int(self.pick([0, 10, 500])))
        q = -1
        if having:
            cnt = p.var(len(keys) + 1, capi.INT8OID)
            q = p.func(capi.F_INT8GT, capi.BOOLOID, cnt, p.const(capi.INT8OID, self.pick([0, 0, 1, 2])))
            if self.chance(0.3):
                cany = p.var(len(keys) + 2, capi.INT8OID)
                q = p.boolop(capi.E_OR, q, p.func(capi.F_INT8LE, capi.BOOLOID, cany, p.const(capi.INT8OID, 1)))
            elif ex_cols and exact and self.chance(0.08):
                s = p.var(len(keys) + len(aggs) - 1, capi.FLOAT8OID)      # sum(x) / 0.0 > 0: division by zero over any non-NULL sum
                q = p.func(capi.F_FLOAT8GT, capi.BOOLOID, p.func(capi.F_FLOAT8DIV, capi.FLOAT8OID, s, p.const(capi.FLOAT8OID, 0.0)),
                           p.const(capi.FLOAT8OID, 0.0))
        node = Agg(child, a, q, two_stage, p.pool)
        self.ops.append("agg")
        kind = ("final" if two_stage else "agg") + ("-having" if having else "")
        # a float8 group key is -0 or +0 over zeros of both signs, so is a float8 min / max; a sum follows its input
        amb = {j for j, k in enumerate(keys) if p.pool.nodes[k].rettype == capi.FLOAT8OID}
        for i, (fn, arg) in enumerate(aggs):
            e = p.pool.nodes[arg] if arg >= 0 else None
            if fn in MINMAX_F8 or (fn in FOLLOWS_ARG and e.varattno - 1 in sides[e.varno].amb):
                amb.add(len(keys) + i)
        return self.size(R(node, exact, list(range(len(keys))), kind, amb))

    # WindowAgg
    def funcs(self, r, od, n, frame_rows):
        p, types = self.p, r.types
        v = lambda c: p.var(c + 1, types[c])                                   # noqa: E731
        nonstr = [c for c, t in enumerate(types) if t not in (capi.BPCHAROID, capi.VARCHAROID, capi.TEXTOID)]
        cands = [lambda: (capi.WF_RANK, capi.INT8OID, []), lambda: (capi.WF_DENSE_RANK, capi.INT8OID, []),
                 lambda: (capi.WF_PERCENT_RANK, capi.FLOAT8OID, []), lambda: (capi.WF_CUME_DIST, capi.FLOAT8OID, [])]
        aggs = [lambda: (capi.AGG_COUNT_STAR, capi.INT8OID, [])]
        c_any = self.pick(range(len(types)))
        aggs.append(lambda: (capi.AGG_COUNT_ANY, capi.INT8OID, [v(c_any)]))
        for t, fns in ((capi.INT4OID, (capi.AGG_SUM_INT4, capi.AGG_MIN_INT4, capi.AGG_MAX_INT4)), (capi.INT8OID, (capi.AGG_MIN_INT8, capi.AGG_MAX_INT8)),
                       (capi.DATEOID, (capi.AGG_MIN_DATE, capi.AGG_MAX_DATE)), (capi.FLOAT8OID, (capi.AGG_MIN_FLOAT8, capi.AGG_MAX_FLOAT8))):
            cs = [c for c in nonstr if types[c] == t]
            for fn in fns:
                if cs:
                    c = self.pick(cs)
                    aggs.append(lambda fn=fn, c=c: (fn, capi.INT8OID if fn == capi.AGG_SUM_INT4 else types[c], [v(c)]))
        exact_cols = [c for c, b in r.exact.items() if _exact_ok((b[0] * MAX_ROWS, b[1]))]
        for c in exact_cols:
            aggs += [lambda c=c: (capi.AGG_SUM_FLOAT8, capi.FLOAT8OID, [v(c)]), lambda c=c: (capi.AGG_AVG_FLOAT8, capi.FLOAT8OID, [v(c)])]
        if od or not frame_rows:
            cands += aggs
        if od:
            bad = self.chance(0.05)                     # ntile(0) / nth_value(x, 0): an ERROR over at least one row
            c0 = self.pick(range(len(types)))
            cands += [lambda: (capi.WF_ROW_NUMBER, capi.INT8OID, []),
                      lambda: (capi.WF_NTILE, capi.INT4OID, [p.const(capi.INT4OID, 0 if bad else self.pick([1, 3, 7]))]),
                      lambda: (self.pick([capi.WF_LAG, capi.WF_LEAD]), types[c0], [v(c0)]),
                      lambda: (self.pick([capi.WF_LAG_OFFSET, capi.WF_LEAD_OFFSET]), types[c0], [v(c0), p.const(capi.INT4OID, self.pick([-1, 0, 2, 3]))]),
                      lambda: (self.pick([capi.WF_LAG_DEFAULT, capi.WF_LEAD_DEFAULT]), types[c0], [v(c0), p.const(capi.INT4OID, 2), v(c0)]),
                      lambda: (self.pick([capi.WF_FIRST_VALUE, capi.WF_LAST_VALUE]), types[c0], [v(c0)]),
                      lambda: (capi.WF_NTH_VALUE, types[c0], [v(c0), p.const(capi.INT4OID, 0 if bad else self.pick([1, 2, 3]))])]
        fs = [self.pick(cands)() for _ in range(n)]
        ex_out = {}
        for i, f in enumerate(fs):
            if f[0] == capi.AGG_SUM_FLOAT8:
                b = r.exact[p.pool.nodes[f[2][0]].varattno - 1]
                ex_out[len(types) + i] = (b[0] * MAX_ROWS, b[1])
        return fs, ex_out

    def window(self, r, keys=None, over_window=None, qual=None, kind=None):
        """WindowAgg over r: a Sort below on part + order (+ r's unique columns when that orders it totally), or none without keys;
        over_window: (the WindowAgg below, its Sort's keys) for a WindowAgg whose keys are a prefix of that Sort's"""
        from _window import FRAMES
        types, p = r.types, self.p
        if over_window is not None:
            sk = over_window
            m = int(self.rng.integers(1, len(sk) + 1))
            npart = int(self.rng.integers(0, min(m, 2) + 1))
            part, order = [k.col for k in sk[:npart]], [k.col for k in sk[npart:m]]
            od = r.kind == "total"
            child = r
        else:
            if keys is None:
                keys = int(self.rng.integers(0, 3)) + int(self.rng.integers(0, 2))
            pick = [int(c) for c in self.rng.choice(len(types), size=min(keys, len(types), 3), replace=False)]
            npart = int(self.rng.integers(0, min(len(pick), 1) + 1))
            part, order = pick[:npart], pick[npart:]
            tail = [u for u in (r.uniq or []) if u not in pick]
            od = r.uniq is not None and len(pick) + len(tail) <= 4 and (pick or not tail)
            if pick:
                sk = [capi.make_sortkey(c, types[c], self.chance(0.3), self.chance(0.3)) for c in pick + (tail if od else [])]
                child = R(Sort(r.node, sk), r.exact, r.uniq, "total" if od else "sort", r.amb)
            else:
                sk, child = [], r
                od = r.kind == "total"
        frame = self.pick(FRAMES_ALL if od else RANGE_FRAMES)
        fs, ex_out = self.funcs(child, od, int(self.rng.integers(1, 9)), "rows" in frame)
        q = -1
        want_qual = self.chance(0.3) if qual is None else qual
        if want_qual:
            rk = [i for i, f in enumerate(fs) if f[0] in (capi.WF_ROW_NUMBER, capi.WF_RANK, capi.WF_DENSE_RANK, capi.AGG_COUNT_STAR)]
            if not rk:
                fs[0] = (capi.WF_RANK, capi.INT8OID, [])
                rk = [0]
            q = p.func(capi.F_INT8LE, capi.BOOLOID, p.var(len(types) + rk[0] + 1, capi.INT8OID), p.const(capi.INT8OID, self.pick([1, 2, 5])))
        node = Window(child.node, part, order, FRAMES[frame], fs, q)
        exact = dict(r.exact)
        exact.update(ex_out)
        amb = set(r.amb)
        for i, (fn, _, args) in enumerate(fs):
            if fn in MINMAX_F8 or (fn in FOLLOWS_ARG and p.pool.nodes[args[0]].varattno - 1 in r.amb):
                amb.add(len(types) + i)
        self.ops.append("window")
        out = R(node, exact, r.uniq, "total" if od and q == -1 else "window", amb)
        out.sort_keys = sk
        return self.size(out)

    def gather(self, r):
        self.ops.append("gather")
        return self.size(R(Gather(r.node), r.exact, r.uniq, "gather", r.amb))

    def sort(self, r, total=False):
        types = r.types
        n = int(self.rng.integers(1, min(3, len(types)) + 1))
        cs = [int(c) for c in self.rng.choice(len(types), size=n, replace=False)]
        if total and r.uniq is not None:
            cs += [u for u in r.uniq if u not in cs]
        cs = cs[:4]
        return Sort(r.node, [capi.make_sortkey(c, types[c], self.chance(0.4), self.chance(0.4)) for c in cs])


def partners(t):
    if t in (capi.INT4OID, capi.INT8OID):
        return (capi.INT4OID, capi.INT8OID)
    if t in (capi.VARCHAROID, capi.TEXTOID):
        return (capi.VARCHAROID, capi.TEXTOID)
    return (t,)


# ---- one plan per seed ----

def agg_source(d):
    """what an Agg reads: scan rows, or a HashJoin of two base relations fused with it"""
    return d.scan_rows() if d.chance(0.5) else d.join(d.plain_scan(), d.plain_scan(), fused=True)


def rows_node(d):
    """a node whose rows a WindowAgg, a join or a Gather reads: scan rows or join rows"""
    return d.scan_rows() if d.chance(0.5) else d.join(d.plain_scan(), d.plain_scan())


def build(d, theme):
    """the composition `theme`, then up to two random nodes, then the top: (top node, what checks it)"""
    r, top = None, None
    if theme == "win/scan":
        r = d.window(d.scan_rows(), keys=int(d.rng.integers(1, 4)))
    elif theme == "win/join":
        r = d.window(d.join(d.plain_scan(), d.plain_scan()), keys=int(d.rng.integers(1, 4)))
    elif theme in ("win/agg", "win/having-sort", "final-having/sort-win"):
        a = d.agg(agg_source(d), having=theme != "win/agg", two_stage=theme.startswith("final"))
        r = d.window(a, keys=int(d.rng.integers(1, 3)))
    elif theme == "win/having-nokeys":
        r = d.window(d.agg(agg_source(d), having=True), keys=0)
    elif theme == "win/win-prefix":
        w = d.window(rows_node(d), keys=int(d.rng.integers(1, 4)), qual=False)
        r = d.window(w, over_window=w.sort_keys)
    elif theme == "win/gather":
        r = d.window(d.gather(rows_node(d)), keys=int(d.rng.integers(1, 3)))
    elif theme == "winqual/limit":
        w = d.window(rows_node(d), qual=True)
        top = ("limit", Limit(d.sort(w, total=d.chance(0.5)), int(d.pick([1, 5, 17, 100])), d.pick([None, 3, 10])), w.amb)
    elif theme == "winqual/sort":
        w = d.window(rows_node(d), qual=True)
        top = ("sort", d.sort(w), w.amb)
    elif theme in ("agg/win", "having/win"):
        r = d.agg(d.window(rows_node(d)), having=theme == "having/win", two_stage=d.chance(0.3))
    elif theme in ("join/win-outer", "join/win-inner"):
        w, o = d.window(rows_node(d)), d.plain_scan()
        r = d.join(w, o) if theme.endswith("outer") else d.join(o, w)
    elif theme == "join/having-win":
        a, w = d.agg(d.scan_rows(), having=True, nkeys=int(d.rng.integers(1, 3))), d.window(d.scan_rows())
        r = d.join(a, w) if d.chance(0.5) else d.join(w, a)
    elif theme == "gather/win":
        r = d.gather(d.window(rows_node(d)))
    elif theme == "gather/having":
        r = d.gather(d.agg(agg_source(d), having=True, two_stage=d.chance(0.3)))
    d.tags.add(theme)
    if top is None:
        for _ in range(int(d.rng.integers(0, 3))):
            ops = ["window", "gather"] + (["agg"] if r.kind in ("scan", "window", "total") else []) + \
                  (["join"] if r.kind in ("scan", "join", "window", "total", "agg", "agg-having", "final-having") else [])
            op = d.pick(ops if r.kind != "gather" else ["window"])
            r = {"window": lambda: d.window(r), "gather": lambda: d.gather(r), "agg": lambda: d.agg(r, having=d.chance(0.5)),
                 "join": lambda: d.join(r, d.plain_scan()) if d.chance(0.5) else d.join(d.plain_scan(), r)}[op]()
            d.size(r)
        end = d.pick(["rows", "sort", "limit"])
        if end == "sort":
            top = ("sort", d.sort(r), r.amb)
        elif end == "limit":
            top = ("limit", Limit(d.sort(r, total=d.chance(0.5)), int(d.pick([1, 5, 17, 100])), d.pick([None, 3, 10])), r.amb)
        else:
            top = ("agg" if isinstance(r.node, Agg) else "rows", r.node, r.amb)
    return top


def draw_plan(seed, rels):
    """(Draw, (check kind, top node, its sign-ambiguous columns), expected: ("rows", rows) or ("error", code)) of one seed"""
    rng = np.random.default_rng(7000 + seed)
    theme = COMPOSITIONS[seed % len(COMPOSITIONS)]
    large = bool(rng.random() < 0.25)
    for attempt in range(16):
        d = Draw(rng, rels, large)
        try:
            top = build(d, theme)
            try:
                want = ("rows", rows(d.p, top[1]))
            except RefError as e:
                want = ("error", e.code)
            if want[0] == "rows" and not want[1] and attempt < 10:
                continue                              # an empty answer checks little: draw again
            return d, top, want
        except (Redraw, PoolFull):                   # too many reference rows, or the expression pool is full
            continue
    raise AssertionError("seed %d: no plan drawn" % seed)


def check(p, top, got, want, ctx):
    """the device's rows of the top node against the reference's: a Limit against every row of the Sort below it"""
    kind, node, amb = top
    tok = sign_token(amb)
    if kind == "sort":
        check_sort(got, want, node.keys, ctx, tok=tok)
    elif kind == "limit":
        check_limit(got, rows(p, node.child), node.child.keys, node.count, ctx, offset=node.offset or 0, tok=tok)
    else:
        assert Counter(map(tok, got)) == Counter(map(tok, want)), ctx


# ---- on the device ----

@pytest.fixture(scope="module")
def eng():
    from greengage_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def dev_rels(eng):
    from greengage_b200.engine import Relation
    rels = host_rels()
    dev = [Relation(eng, host_pages=pg) for pg in rels.pages]
    yield rels, dev
    for r in dev:
        r.free()


def slot_rows(rows):
    return [tuple(datum(v, n, t) for v, n, t in zip(vals, nl, ty)) for vals, nl, ty, ln in rows]


def sort_runs(x):
    """the most sorted runs of any Sort in the executor tree (more than one: an external sort of host rows)"""
    L = ex.exec_lib()
    L.GgExecNodeInstrumentation.argtypes = [C.c_void_p, C.POINTER(ex.GgInstrumentation)]
    most = 0

    def walk(st):
        nonlocal most
        if not st:
            return
        if L.GgExecNodeKind(st).decode() == "sort":
            ins = ex.GgInstrumentation()
            capi.check(L.GgExecNodeInstrumentation(st, C.byref(ins)))
            most = max(most, ins.sort_runs)
        walk(L.GgExecOuterPlanState(st))
        walk(L.GgExecInnerPlanState(st))
    walk(x.state)
    return most


_outcomes = {}


@pytest.mark.parametrize("seed", SEEDS)
def test_random_plans(eng, dev_rels, seed):
    rels, dev = dev_rels
    d, top, want = draw_plan(seed, rels)
    operator_mem = int(np.random.default_rng(9000 + seed).choice([0, 0, 16384, 65536]))
    ctx = (seed, sorted(d.tags), d.ops, top[0], operator_mem)
    b = ex.PlanBuilder()
    try:
        x = ex.Executor(eng, d.p.pool, dev, plan_of(b, top[1]), operator_mem=operator_mem)
    except ex.ExecError as e:
        assert e.code == UNSUPPORTED, (ctx, e.code, str(e))
        _outcomes[seed] = ("refused", str(e))
        pytest.skip("refused with GG_ERR_UNSUPPORTED: %s" % e)
    try:
        if want[0] == "error":
            with pytest.raises(ex.ExecError) as e:
                x.rows()
            assert e.value.code == want[1], (ctx, e.value.code, str(e.value))
            _outcomes[seed] = ("error", want[1])
            return
        got = slot_rows(x.rows())
        check(d.p, top, got, want[1], ctx)
        assert x.instrumentation()[0][1].ntuples == len(got), ctx
        batches, runs = [nb for _, nb in join_states(x)], sort_runs(x)
        if operator_mem == 0:
            assert all(nb == 1 for nb in batches) and runs <= 1, (ctx, batches, runs)
        x.rescan()
        again = slot_rows(x.rows())
        # the same check again (under a Limit, which rows tied at the window's edge come back is the run's choice), and, but
        # for that choice, the same rows as the first run, bit for bit outside the columns whose zero sign is open
        check(d.p, top, again, want[1], ctx + ("rescan",))
        if top[0] != "limit":
            tok = sign_token(top[2])
            assert Counter(map(tok, again)) == Counter(map(tok, got)), ctx
        _outcomes[seed] = ("ran", sorted(d.tags), len(got), operator_mem, max(batches, default=0), runs)
    finally:
        x.end()


def test_most_random_plans_run(capsys):
    """after the seeds: at least 80% of them ran on the device (an expected ERROR included) rather than being refused, some ran
    a batched join, some sorted host rows in more than one run, and every composition ran at least once"""
    if len(_outcomes) < len(SEEDS):
        pytest.skip("judges the seeds of test_random_plans, which did not all run")
    ran = {s: o for s, o in _outcomes.items() if o[0] in ("ran", "error")}
    with capsys.disabled():
        print("\nrandom plans: %d ran, %d raised the reference's ERROR, %d refused; %d ran a batched join, %d sorted in runs" % (
            sum(o[0] == "ran" for o in ran.values()), sum(o[0] == "error" for o in ran.values()), len(_outcomes) - len(ran),
            sum(o[0] == "ran" and o[4] > 1 for o in ran.values()), sum(o[0] == "ran" and o[5] > 1 for o in ran.values())))
    assert len(ran) >= 0.8 * len(SEEDS), _outcomes
    done = {t for o in ran.values() if o[0] == "ran" for t in o[1]}
    assert any(o[0] == "ran" and o[4] > 1 for o in ran.values()), ("no seed ran a batched join", _outcomes)
    assert any(o[0] == "ran" and o[5] > 1 for o in ran.values()), ("no seed sorted host rows in runs", _outcomes)
    assert set(COMPOSITIONS) <= done, (set(COMPOSITIONS) - done, _outcomes)


# ---- a WindowAgg over an Agg's HAVING survivors ----

@pytest.mark.parametrize("shape", ["sort", "no-keys", "final-sort"])
def test_window_over_having_survivors(eng, dev_rels, shape):
    """rank() OVER (ORDER BY count(*) DESC) ... GROUP BY z, bool HAVING count(*) > 1: the Sort (or, without window keys, the
    WindowAgg itself) reads the rows the HAVING filter kept, one-stage or as the FINAL stage over a Gather at one segment"""
    rels, dev = dev_rels
    p = capi.ExprPool()
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [p.var(col("z"), capi.INT4OID), p.var(col("bool"), capi.BOOLOID)],
                        [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_FLOAT8, p.var(col("v"), capi.FLOAT8OID)), (capi.AGG_MIN_INT4, p.var(col("int4"), capi.INT4OID))])
    having = p.func(capi.F_INT8GT, capi.BOOLOID, p.var(3, capi.INT8OID), p.const(capi.INT8OID, 1))
    a = Agg(Scan(0, rels.desc[0], rels.rows[0]), agg, having, two_stage=shape == "final-sort", pool=p.pool)
    s = p.var(4, capi.FLOAT8OID)
    if shape == "no-keys":
        node = Window(a, [], [], capi.FRAMEOPTION_DEFAULTS, [(capi.AGG_COUNT_STAR, capi.INT8OID, []), (capi.WF_RANK, capi.INT8OID, []),
                                                             (capi.AGG_SUM_FLOAT8, capi.FLOAT8OID, [s])])
    else:
        keys = [capi.make_sortkey(2, capi.INT8OID, desc=True), capi.make_sortkey(0, capi.INT4OID), capi.make_sortkey(1, capi.BOOLOID)]
        node = Window(Sort(a, keys), [], [2], capi.FRAMEOPTION_DEFAULTS,
                      [(capi.WF_RANK, capi.INT8OID, []), (capi.WF_ROW_NUMBER, capi.INT8OID, []), (capi.AGG_SUM_FLOAT8, capi.FLOAT8OID, [s]),
                       (capi.WF_LAG, capi.INT4OID, [p.var(5, capi.INT4OID)])])
    want = rows_of(p.pool, node)
    every = rows_of(p.pool, Agg(Scan(0, rels.desc[0], rels.rows[0]), agg, pool=p.pool))
    assert 0 < len(want) < len(every)
    b = ex.PlanBuilder()
    x = ex.Executor(eng, p.pool, dev, plan_of(b, node))
    try:
        got = slot_rows(x.rows())
        if shape == "no-keys":
            assert Counter(map(row_token, got)) == Counter(map(row_token, want))
        else:
            assert [row_token(r) for r in got] == [row_token(r) for r in want]            # a total order: the same sequence
        assert x.instrumentation()[0][1].ntuples == len(want)
        x.rescan()
        assert Counter(map(row_token, slot_rows(x.rows()))) == Counter(map(row_token, got))
    finally:
        x.end()
