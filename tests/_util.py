"""Shared helpers for the test-suite: golden vectors, fixture relations, result comparison."""
import ctypes as C
import json
import os
import struct
from fractions import Fraction

import numpy as np

from greengage_b200 import capi, tpch
from oracle import pyoracle as po

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")


def golden(name):
    return json.load(open(os.path.join(GOLD, name)))


def ref_live_kat():
    """What the reference's own objects answered for the seeded inputs below and for the product's Motion chunks
    (tests/golden/ref_live_kat.npz, written by tests/golden/make_golden.py::ref_live_kat)"""
    z = np.load(os.path.join(GOLD, "ref_live_kat.npz"))
    return {k: z[k] for k in z.files}


def hash_live_inputs():
    """20000 seeded (bytes for hash_any, int8 value, segment count) triples"""
    import random
    rng = random.Random(7)
    for _ in range(20000):
        n = rng.randint(0, 48)
        b = bytes(rng.getrandbits(8) for _ in range(n))
        v = rng.getrandbits(64) - (1 << 63)
        ns = rng.choice([1, 2, 3, 5, 8, 13, 64, 999])
        yield b, v, ns


def aocs_live_cases(types):
    """seeded random columns of every type in `types`: (name, values, nulls or None), 40000 rows (4000 for text, up to
    3000 bytes each), null fractions 0, 0.5 and 1"""
    rng = np.random.default_rng(77)
    n = 40000
    for name in types:
        if name == "text":
            vals = [bytes(rng.integers(97, 123, int(ln)).astype(np.uint8)) for ln in rng.choice([0, 3, 126, 127, 500, 3000], 4000)]
        elif name == "bpchar1":
            vals = [bytes([65 + int(x)]) for x in rng.integers(0, 3, n)]
        elif name == "float8":
            vals = [float(x) for x in rng.normal(size=n)]
        else:
            vals = [int(x) for x in rng.integers(-2**31, 2**31, n)]
        for nullfrac in (0.0, 0.5, 1.0):
            nulls = (rng.random(len(vals)) < nullfrac).astype(np.uint8) if nullfrac else None
            yield name, vals, nulls, nullfrac


def digest(*arrays):
    """SHA-256 over the bytes of the arrays, in order"""
    import hashlib
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def b2f(bits):
    return struct.unpack("<d", struct.pack("<q", int(bits)))[0]


def f2b(x):
    return struct.unpack("<q", struct.pack("<d", x))[0]


def make_desc(spec):
    """spec: list of (typid, attlen, attalign, byval[, notnull])"""
    d = capi.gg_tupdesc()
    d.natts = len(spec)
    for i, sp in enumerate(spec):
        a = d.attrs[i]
        a.atttypid, a.attlen, a.attalign, a.attbyval = sp[0], sp[1], ord(sp[2]), sp[3]
        a.attnotnull = sp[4] if len(sp) > 4 else 0
        a.atttypmod = -1
    return d


_fixture_cache = {}


def lineitem_fixture_pages():
    """The reference's own regression lineitem data (tests/golden/lineitem_q1.npz) as LI-wide heap pages
    (float8 in place of numeric), built with the oracle's heap_form_tuple / PageAddItem restatement."""
    if "li" in _fixture_cache:
        return _fixture_cache["li"]
    zf = np.load(os.path.join(GOLD, "lineitem_q1.npz"))
    z = {k: zf[k] for k in zf.files}          # NpzFile decompresses on every access: materialise once
    desc = capi.synth_tupdesc(capi.TAB_LINEITEM_WIDE)
    instr = [str(x) for x in z["shipinstruct_names"]]
    modes = [str(x) for x in z["shipmode_names"]]
    n = len(z["orderkey"])
    rows = []
    for i in range(n):
        rows.append([int(z["orderkey"][i]), int(z["partkey"][i]), int(z["suppkey"][i]), int(z["linenumber"][i]),
                     float(z["quantity"][i]), float(z["extendedprice"][i]), float(z["discount"][i]), float(z["tax"][i]),
                     bytes([z["returnflag"][i]]), bytes([z["linestatus"][i]]),
                     int(z["shipdate"][i]), int(z["commitdate"][i]), int(z["receiptdate"][i]),
                     instr[z["shipinstruct"][i]].ljust(25).encode(), modes[z["shipmode"][i]].ljust(10).encode(),
                     b"c" * int(z["comment_len"][i])])
    pages = po.build_pages(desc, rows)
    _fixture_cache["li"] = (desc, pages, n)
    return _fixture_cache["li"]


def rows_by_key(rows, nkeys=2):
    out = {}
    for r in rows:
        k = tuple((r.key[i], r.keylen[i], r.keyisnull[i]) for i in range(nkeys))
        assert k not in out, "duplicate group in output"
        out[k] = r
    return out


def exact_by_key(rows, states, nkeys):
    """the oracle's exact records (po.seqscan_agg(..., exact=True)[-1]) keyed like rows_by_key, for comparing another
    stage's rows (a FINAL over the same inputs) with them"""
    return {k: states[i] for i, k in enumerate(rows_by_key(rows, nkeys))}


_U = Fraction(1, 1 << 53)                  # unit roundoff of binary64


def _gamma(k):
    """γ(k) = k·u / (1 - k·u): |fl(Σ) - Σ| <= γ(n-1)·Σ|x| for any summation tree over n values (Higham, ASNA §4.2)"""
    return k * _U / (1 - k * _U)


def _exact_regime(total_abs, lowbit):
    """every partial sum of every order is representable: all inputs are multiples of g = 2^lowbit and Σ|x| < 2^53·g"""
    return lowbit is None or total_abs < (1 << (53 + lowbit + po.EXACT_SCALE))


def _check_exact_sum(x, n, s, a, lowbit, nan, pinf, ninf, zero, ctx):
    """one float8 sum `x` of n inputs against their exact sum s and Σ|x| a (integers in units of 2^-EXACT_SCALE).
    zero: the float a zero sum must be (its sign)"""
    if nan or (pinf and ninf):
        assert x != x, ("NaN expected",) + ctx
        return
    if pinf or ninf:
        assert x == (float("inf") if pinf else -float("inf")), ("infinity expected", x) + ctx
        return
    scale = 1 << po.EXACT_SCALE
    if _exact_regime(a, lowbit):
        want = zero if s == 0 else s / scale            # int / int: correctly rounded, and exact here
        assert f2b(x) == f2b(want), ("not the exact sum", x, want) + ctx
        return
    assert abs(x) != float("inf") and x == x, ("finite sum expected", x) + ctx
    err = abs(Fraction(x) - Fraction(s, scale))
    bound = _gamma(n - 1) * Fraction(a, scale)
    assert err <= bound, ("sum outside γ(n-1)·Σ|x|", x, float(Fraction(s, scale)), float(err), float(bound)) + ctx


_OVERFLOW = Fraction((1 << 1024) - (1 << 970))        # sums at or past this round to infinity (DBL_MAX + half an ulp)


def sum_overflow_rule(e, scale_exp=0):
    """Whether float8pl's overflow ERROR is the same in every summation order of the finite inputs `e` records (an Exact of
    values scaled by 2^-scale_exp): True every order overflows — all inputs share a sign and even the smallest sum any order
    can compute, (1 - γ(n-1))·|s|, is past the overflow threshold; False no order does — the largest any order can compute,
    (1 + γ(n-1))·Σ|x|, stays below it; None it depends on the order, and nothing may be asserted."""
    scale = Fraction(1 << scale_exp, 1 << po.EXACT_SCALE)
    s, a, g = abs(Fraction(e.s) * scale), Fraction(e.a) * scale, _gamma(e.n - 1)
    if s == a and (1 - g) * s >= _OVERFLOW:
        return True
    if (1 + g) * a < _OVERFLOW:
        return False
    return None


def _check_exact(fn, partial, j, x, e, ctx):
    nan, pinf, ninf = bool(e.flags & po.XF_NAN), bool(e.flags & po.XF_PINF), bool(e.flags & po.XF_NINF)
    if fn == capi.AGG_SUM_FLOAT8:
        # float8pl with a NULL initcond takes the first input as it is: -0 exactly when every input was -0, in any order
        _check_exact_sum(x, e.n, e.s, e.a, e.lowbit, nan, pinf, ninf, -0.0 if e.flags & po.XF_ALL_NEGZERO else 0.0, ctx)
    elif partial and j == 1:                        # float8_accum's sumX starts from the +0 of "{0,0,0}"
        _check_exact_sum(x, e.n, e.s, e.a, e.lowbit, nan, pinf, ninf, 0.0, ctx)
    elif partial and j == 2:                        # sumX2 over fl(x*x) >= 0: an infinite input squares to +inf
        _check_exact_sum(x, e.n, e.q, e.q, e.lowbit_sq, nan, pinf or ninf, False, 0.0, ctx)
    else:                                           # float8_avg: sumX / N
        if nan or pinf or ninf:
            _check_exact_sum(x, e.n, e.s, e.a, e.lowbit, nan, pinf, ninf, 0.0, ctx)
            return
        scale = 1 << po.EXACT_SCALE
        if _exact_regime(e.a, e.lowbit):
            want = (e.s / scale + 0.0) / e.n            # the exact sum, then one correctly rounded division
            assert f2b(x) == f2b(want), ("not fl(s/n)", x, want) + ctx
            return
        assert abs(x) != float("inf") and x == x, ("finite avg expected", x) + ctx
        s, a, g = Fraction(e.s, scale), Fraction(e.a, scale), _gamma(e.n - 1)
        err = abs(Fraction(x) - s / e.n)
        bound = g * a / e.n + _U * (abs(s) + g * a) / e.n
        assert err <= bound, ("avg outside its bound", x, float(s / e.n), float(err), float(bound)) + ctx


def assert_aggrows_match(got, want, agg, rel=1e-6, float_exact=False, exact=None):
    """Integer results and keys bit-exact; float8 sums/avgs within `rel` (the tolerance BASELINE.json states).

    exact: the oracle's exact records of the same inputs (po.seqscan_agg / hashjoin_agg / aocs_seqscan_agg with exact=True:
    a list aligned with `want`, or exact_by_key's dict).  Then every float8 SUM/AVG is held to what any summation order
    provably gives instead of `rel`: bit for bit the exact answer where every partial sum is representable, else within
    γ(n-1)·Σ|x| of the exact sum; NaN / ±inf as the non-finite inputs dictate."""
    nkeys = agg.numCols
    g, w = rows_by_key(got, nkeys), rows_by_key(want, nkeys)
    assert set(g) == set(w), (sorted(g), sorted(w))
    if isinstance(exact, list):
        exact = dict(zip(w, exact))
    partial = agg.aggstage == capi.AGGSTAGE_PARTIAL
    for k in w:
        for i in range(agg.numAggs):
            a, b = g[k].agg[i], w[k].agg[i]
            assert a.isnull == b.isnull, (k, i, a.isnull, b.isnull)
            if a.isnull:
                continue
            fn = agg.aggs[i].aggfnoid
            if fn in (capi.AGG_COUNT_STAR, capi.AGG_COUNT_ANY, capi.AGG_SUM_INT4, capi.AGG_MAX_INT4, capi.AGG_MIN_INT4,
                      capi.AGG_MAX_INT8, capi.AGG_MIN_INT8, capi.AGG_MAX_DATE, capi.AGG_MIN_DATE):
                assert a.i == b.i, (k, i, a.i, b.i)
            else:
                nf = 3 if (fn == capi.AGG_AVG_FLOAT8 and partial) else 1
                e = exact[k][i] if exact is not None else None
                for j in range(nf):
                    x, y = a.f[j], b.f[j]
                    if fn in (capi.AGG_MAX_FLOAT8, capi.AGG_MIN_FLOAT8):
                        if e is not None and x == 0 and y == 0 and e.flags & po.XF_POSZERO and e.flags & po.XF_NEGZERO:
                            # float8larger/smaller keep the later argument of a tie, so with both zeros in the group the
                            # reference's sign depends on scan order; a parallel scan has none, either sign is right
                            continue
                        assert f2b(x) == f2b(y) or (x != x and y != y), (k, i, j, x, y)
                    elif float_exact or (nf == 3 and j == 0):
                        assert f2b(x) == f2b(y) or (x != x and y != y), (k, i, j, x, y)
                    elif e is not None:
                        _check_exact(fn, partial, j, x, e, (k, i, j))
                    elif y == 0 or y != y or abs(y) == float("inf"):
                        assert x == y or (x != x and y != y), (k, i, j, x, y)
                    else:
                        assert abs(x - y) <= rel * abs(y), (k, i, j, x, y)


# ---- a relation built for the edges of float8 summation ----

EDGE_GROUPS = {
    0: "every input -0", 1: "+0 and -0 mixed", 2: "+inf alone", 3: "+inf with -inf", 4: "NaN among finite values",
    5: "multiples of 2^-10, heavy cancellation, sum|x| just under 2^43 (exact in any order)",
    6: "non-dyadic values that cancel: sum|x| >> |sum|", 7: "one input", 8: "31 inputs", 9: "32 inputs", 10: "33 inputs",
    11: "2000 inputs laid out across a page boundary", 12: "every input NULL", 13: "-inf alone, with NULLs",
    14: "zeros of both signs and negative values (min ties at neither zero)", 15: "-0 and positive values (min is -0)",
}


def edge_relation(nullable=True, pad=0):
    """(desc, pages, nrows): (g int4, v float8) rows of the EDGE_GROUPS, seeded, most groups shuffled over ~10 pages;
    NULL v is mixed into several groups.  nullable=False: the same rows without the NULL ones, v declared NOT NULL.
    pad: that many float8 columns (all 0, never aggregated) after v, for tuples wide enough that a page holds fewer than
    10 chunks of 32 rows — the shape on which the private-accumulator kernels keep sums in registers."""
    if ("edge", nullable, pad) in _fixture_cache:
        return _fixture_cache[("edge", nullable, pad)]
    rng = np.random.default_rng(2024)
    rows = []
    rows += [(0, -0.0)] * 200
    rows += [(1, z) for z in rng.choice([0.0, -0.0], 300)]
    rows += [(2, float("inf"))]
    rows += [(3, float("inf")), (3, -float("inf"))] + [(3, float(x)) for x in rng.normal(size=20)]
    rows += [(4, float("nan"))] + [(4, float(x)) for x in rng.normal(size=60)]
    n5 = 3000
    half = rng.integers((1 << 53) // n5 // 2, (1 << 53) // n5 - 8, n5 // 2, dtype=np.int64) * rng.choice([-1, 1], n5 // 2)
    k = np.concatenate([half, -half])                        # the total cancels but for the few units added here
    k[0] += 3 if k[0] > 0 else -3
    k[1] -= 1 if k[1] > 0 else -1
    assert (1 << 52) < int(np.abs(k).sum()) < 1 << 53
    rows += [(5, float(int(v)) * 2.0 ** -10) for v in k]
    x6 = rng.normal(size=600) * 1e8
    rows += [(6, float(v)) for v in np.concatenate([x6, -x6 * (1 + 1e-12), [0.1]])]
    rows += [(7, 0.3)]
    for gid, n in ((8, 31), (9, 32), (10, 33)):
        rows += [(gid, float(v)) for v in rng.normal(size=n) / 3]
    rows += [(14, v) for v in (0.0, -0.0, -1.5, 0.0, -2.25)]
    rows += [(15, v) for v in (1.0, -0.0, 0.5)]
    nulls = [False] * len(rows)
    rows += [(12, 0.0)] * 7
    nulls += [True] * 7
    rows += [(13, -float("inf")), (13, 0.0), (13, 0.0)]
    nulls += [False, True, True]
    for gid in (1, 4, 5, 8):                                # NULLs mixed into groups that have values
        rows += [(gid, 0.0)] * 5
        nulls += [True] * 5
    order = rng.permutation(len(rows))
    rows, nulls = [rows[i] for i in order], [nulls[i] for i in order]
    # group 11 kept contiguous in the middle of the relation, so that it straddles a page boundary
    mid = len(rows) // 2
    g11 = [(11, float(v)) for v in rng.normal(size=2000) * 7.25]
    rows, nulls = rows[:mid] + g11 + rows[mid:], nulls[:mid] + [False] * len(g11) + nulls[mid:]
    if not nullable:
        rows, nulls = [r for r, isn in zip(rows, nulls) if not isn], [False] * (len(rows) - sum(nulls))
    desc = make_desc([(capi.INT4OID, 4, "i", 1, 1), (capi.FLOAT8OID, 8, "d", 1, 0 if nullable else 1)] + [(capi.FLOAT8OID, 8, "d", 1, 1)] * pad)
    pages = po.build_pages(desc, [list(r) + [0.0] * pad for r in rows], [[False, n] + [False] * pad for n in nulls])
    _fixture_cache[("edge", nullable, pad)] = (desc, pages, len(rows))
    return _fixture_cache[("edge", nullable, pad)]


def edge_plan(desc, stage=capi.AGGSTAGE_NORMAL):
    """GROUP BY g: count(*), sum(v), avg(v), min(v), max(v), count(v), sum(v * 0.5)"""
    p = capi.ExprPool()
    g, v = p.var(1, capi.INT4OID), p.var(2, capi.FLOAT8OID)
    half = p.func(capi.F_FLOAT8MUL, capi.FLOAT8OID, v, p.const(capi.FLOAT8OID, 0.5))
    agg = capi.make_agg(stage, [g], [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_FLOAT8, v), (capi.AGG_AVG_FLOAT8, v), (capi.AGG_MIN_FLOAT8, v),
                                     (capi.AGG_MAX_FLOAT8, v), (capi.AGG_COUNT_ANY, v), (capi.AGG_SUM_FLOAT8, half)])
    return capi.make_scan(desc, -1), agg, p.pool


def edge_sum_plan(desc, groups, stage=capi.AGGSTAGE_NORMAL, num_groups=0):
    """WHERE g IN (groups) GROUP BY g: sum(v), avg(v), sum(v * 0.5) — sums only, so that a NOT NULL v runs on the
    private-accumulator kernels (which take no MIN/MAX); `groups` should leave out the non-finite ones, whose private sums
    are replayed on the interpreter kernel"""
    p = capi.ExprPool()
    g, v = p.var(1, capi.INT4OID), p.var(2, capi.FLOAT8OID)
    q = -1
    for x in groups:
        eq = p.func(capi.F_INT4EQ, capi.BOOLOID, g, p.const(capi.INT4OID, x))
        q = eq if q < 0 else p.boolop(capi.E_OR, q, eq)
    half = p.func(capi.F_FLOAT8MUL, capi.FLOAT8OID, v, p.const(capi.FLOAT8OID, 0.5))
    agg = capi.make_agg(stage, [g], [(capi.AGG_SUM_FLOAT8, v), (capi.AGG_AVG_FLOAT8, v), (capi.AGG_SUM_FLOAT8, half), (capi.AGG_COUNT_STAR, -1)],
                        num_groups=num_groups)
    return capi.make_scan(desc, q), agg, p.pool


# ---- the reference's regression lineitem / orders as join-shaped relations (tests/golden/*.npz) ----

def tpch_join_fixture():
    """(li_desc, li_pages, ord_desc, ord_pages, shipmode_code, priority_code): the reference's heap_lineitem / heap_orders
    regression data, projected to the columns its Q4 and Q12 touch.  Strings longer than 8 bytes become 1-character
    codes in 1:1 correspondence (l_shipmode -> 'a'.., o_orderpriority -> its first character), so grouping on the code
    is grouping on the value."""
    if "join" in _fixture_cache:
        return _fixture_cache["join"]
    zl = np.load(os.path.join(GOLD, "lineitem_q1.npz"))
    li = {k: zl[k] for k in ("orderkey", "shipdate", "commitdate", "receiptdate", "shipmode")}
    modes = [str(x) for x in zl["shipmode_names"]]
    zo = np.load(os.path.join(GOLD, "orders_tpch.npz"))
    od = {k: zo[k] for k in ("orderkey", "orderdate", "orderpriority")}
    prios = [str(x) for x in zo["orderpriority_names"]]
    li_desc = make_desc([(capi.INT8OID, 8, "d", 1, 1), (capi.DATEOID, 4, "i", 1, 1), (capi.DATEOID, 4, "i", 1, 1), (capi.DATEOID, 4, "i", 1, 1),
                         (capi.BPCHAROID, -1, "i", 0, 1)])
    ord_desc = make_desc([(capi.INT8OID, 8, "d", 1, 1), (capi.DATEOID, 4, "i", 1, 1), (capi.BPCHAROID, -1, "i", 0, 1)])
    shipmode_code = {m: chr(ord("a") + i) for i, m in enumerate(modes)}
    priority_code = {p: p[0] for p in prios}
    li_rows = [[int(li["orderkey"][i]), int(li["shipdate"][i]), int(li["commitdate"][i]), int(li["receiptdate"][i]),
                shipmode_code[modes[li["shipmode"][i]]].encode()] for i in range(len(li["orderkey"]))]
    ord_rows = [[int(od["orderkey"][i]), int(od["orderdate"][i]), priority_code[prios[od["orderpriority"][i]]].encode()]
                for i in range(len(od["orderkey"]))]
    _fixture_cache["join"] = (li_desc, po.build_pages(li_desc, li_rows), ord_desc, po.build_pages(ord_desc, ord_rows), shipmode_code, priority_code)
    return _fixture_cache["join"]


def tpch_q4_plan(li_desc, ord_desc, exp):
    """Q4: orders SEMI JOIN lineitem (l_commitdate < l_receiptdate) on the order key, orders filtered on o_orderdate,
    GROUP BY o_orderpriority, count(*)  (output/rpt_tpch.source, 'mpph4')."""
    p = capi.ExprPool()
    okey, odate, oprio = p.var(1, capi.INT8OID, 0), p.var(2, capi.DATEOID, 0), p.var(3, capi.BPCHAROID, 0)
    lkey, lcommit, lreceipt = p.var(1, capi.INT8OID, 1), p.var(3, capi.DATEOID, 1), p.var(4, capi.DATEOID, 1)
    oqual = p.boolop(capi.E_AND, p.func(capi.F_DATE_GE, capi.BOOLOID, odate, p.const(capi.DATEOID, exp["orderdate_from"])),
                     p.func(capi.F_DATE_LT, capi.BOOLOID, odate, p.const(capi.DATEOID, exp["orderdate_to"])))
    iqual = p.func(capi.F_DATE_LT, capi.BOOLOID, lcommit, lreceipt)
    outer, inner = capi.make_scan(ord_desc, oqual), capi.make_scan(li_desc, iqual)
    hj = capi.make_hashjoin(capi.JOIN_SEMI, [okey], [lkey])
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [oprio], [(capi.AGG_COUNT_STAR, -1)])
    return outer, inner, hj, agg, p.pool


def tpch_q12_plan(li_desc, ord_desc, exp, shipmode_code, priority_code, high):
    """Q12's join: lineitem (its five quals) INNER JOIN orders on the order key, GROUP BY l_shipmode, count(*); the orders
    side keeps the high-priority orders (high=True: Q12's high_line_count) or the others (low_line_count)."""
    p = capi.ExprPool()
    lkey, lship, lcommit, lreceipt, lmode = (p.var(1, capi.INT8OID, 0), p.var(2, capi.DATEOID, 0), p.var(3, capi.DATEOID, 0),
                                             p.var(4, capi.DATEOID, 0), p.var(5, capi.BPCHAROID, 0))
    okey, oprio = p.var(1, capi.INT8OID, 1), p.var(3, capi.BPCHAROID, 1)
    m1, m2 = (shipmode_code[m] for m in exp["shipmodes"])
    q = p.boolop(capi.E_OR, p.func(capi.F_BPCHAREQ, capi.BOOLOID, lmode, p.const(capi.BPCHAROID, m1)),
                 p.func(capi.F_BPCHAREQ, capi.BOOLOID, lmode, p.const(capi.BPCHAROID, m2)))
    for cond in (p.func(capi.F_DATE_LT, capi.BOOLOID, lcommit, lreceipt), p.func(capi.F_DATE_LT, capi.BOOLOID, lship, lcommit),
                 p.func(capi.F_DATE_GE, capi.BOOLOID, lreceipt, p.const(capi.DATEOID, exp["receipt_from"])),
                 p.func(capi.F_DATE_LT, capi.BOOLOID, lreceipt, p.const(capi.DATEOID, exp["receipt_to"]))):
        q = p.boolop(capi.E_AND, q, cond)
    h1, h2 = (priority_code[x] for x in exp["high_priorities"])
    if high:
        iq = p.boolop(capi.E_OR, p.func(capi.F_BPCHAREQ, capi.BOOLOID, oprio, p.const(capi.BPCHAROID, h1)),
                      p.func(capi.F_BPCHAREQ, capi.BOOLOID, oprio, p.const(capi.BPCHAROID, h2)))
    else:
        iq = p.boolop(capi.E_AND, p.func(capi.F_BPCHARNE, capi.BOOLOID, oprio, p.const(capi.BPCHAROID, h1)),
                      p.func(capi.F_BPCHARNE, capi.BOOLOID, oprio, p.const(capi.BPCHAROID, h2)))
    outer, inner = capi.make_scan(li_desc, q), capi.make_scan(ord_desc, iq)
    hj = capi.make_hashjoin(capi.JOIN_INNER, [lkey], [okey])
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [lmode], [(capi.AGG_COUNT_STAR, -1)])
    return outer, inner, hj, agg, p.pool


def tpch_q6_plan(desc):
    """Q6 over the reference's regression lineitem (output/rpt_tpch.source 'mpph6', golden revenue 740117.7050):
    sum(l_extendedprice * l_discount) where l_shipdate in 1996, l_discount between 0.03 and 0.05, l_quantity < 24."""
    from datetime import date
    p = capi.ExprPool()
    qty, price, disc, shipdate = p.var(5, capi.FLOAT8OID), p.var(6, capi.FLOAT8OID), p.var(7, capi.FLOAT8OID), p.var(11, capi.DATEOID)
    d0 = (date(1996, 1, 1) - date(2000, 1, 1)).days
    d1 = (date(1997, 1, 1) - date(2000, 1, 1)).days
    q = p.func(capi.F_DATE_GE, capi.BOOLOID, shipdate, p.const(capi.DATEOID, d0))
    for cond in (p.func(capi.F_DATE_LT, capi.BOOLOID, shipdate, p.const(capi.DATEOID, d1)),
                 p.func(capi.F_FLOAT8GE, capi.BOOLOID, disc, p.const(capi.FLOAT8OID, 0.03)),
                 p.func(capi.F_FLOAT8LE, capi.BOOLOID, disc, p.const(capi.FLOAT8OID, 0.05)),
                 p.func(capi.F_FLOAT8LT, capi.BOOLOID, qty, p.const(capi.FLOAT8OID, 24.0))):
        q = p.boolop(capi.E_AND, q, cond)
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [], [(capi.AGG_SUM_FLOAT8, p.func(capi.F_FLOAT8MUL, capi.FLOAT8OID, price, disc)), (capi.AGG_COUNT_STAR, -1)])
    return capi.make_scan(desc, q), agg, p.pool


Q6_GOLDEN_REVENUE = 740117.7050          # src/test/regress/output/rpt_tpch.source:531 (numeric; float8 columns here: <= 1e-6 relative)


def j1j2_fixture():
    """(j1_desc, j1_pages, j2_desc, j2_pages, golden): J1_TBL(i int4, j int4, t text) / J2_TBL(i int4, k int4) of the
    reference's sql/join.sql:6-38 and its expected/join.out answers (tests/golden/join_j1j2.json)."""
    if "j1j2" not in _fixture_cache:
        g = golden("join_j1j2.json")
        d1 = make_desc([(capi.INT4OID, 4, "i", 1), (capi.INT4OID, 4, "i", 1), (capi.TEXTOID, -1, "i", 0)])
        d2 = make_desc([(capi.INT4OID, 4, "i", 1), (capi.INT4OID, 4, "i", 1)])
        r1 = [[r[0] or 0, r[1] or 0, (r[2] or "").encode()] for r in g["j1"]]
        r2 = [[r[0] or 0, r[1] or 0] for r in g["j2"]]
        n1 = [[v is None for v in r] for r in g["j1"]]
        n2 = [[v is None for v in r] for r in g["j2"]]
        _fixture_cache["j1j2"] = (d1, po.build_pages(d1, r1, n1), d2, po.build_pages(d2, r2, n2), g)
    return _fixture_cache["j1j2"]


J1J2_QUERIES = {"inner": (capi.JOIN_INNER, 1), "inner_i_eq_k": (capi.JOIN_INNER, 2), "left": (capi.JOIN_LEFT, 1),
                "right": (capi.JOIN_RIGHT, 1), "full": (capi.JOIN_FULL, 1)}      # name -> (jointype, J2 key attno)


def j1j2_join(d1, d2, name):
    """J1_TBL <jointype> JOIN J2_TBL ON J1.i = J2.<i|k> -> (pool, outer scan, inner scan, hashjoin)"""
    jt, inner_att = J1J2_QUERIES[name]
    p = capi.ExprPool()
    hj = capi.make_hashjoin(jt, [p.var(1, capi.INT4OID, 0)], [p.var(inner_att, capi.INT4OID, 1)], -1)
    return p, capi.make_scan(d1, -1), capi.make_scan(d2, -1), hj


def j1j2_golden_rows(g, name):
    """the golden table as (J1.i-or-coalesced i, j, t, k) tuples; for ON (J1.i = J2.k) the extra J2.i column is kept last"""
    q = g["queries"][name]
    return [tuple(r) for r in q["rows"]]


def j1j2_agg(p):
    """GROUP BY J1.i: count(*), sum(J1.j), count(J1.j), sum(J2.k), count(J2.k) — what a join that is never materialised can
    be held to against the golden table (the row multiset per group, reduced)."""
    return capi.make_agg(capi.AGGSTAGE_NORMAL, [p.var(1, capi.INT4OID, 0)],
                         [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_INT4, p.var(2, capi.INT4OID, 0)), (capi.AGG_COUNT_ANY, p.var(2, capi.INT4OID, 0)),
                          (capi.AGG_SUM_INT4, p.var(2, capi.INT4OID, 1)), (capi.AGG_COUNT_ANY, p.var(2, capi.INT4OID, 1))])


def j1j2_golden_groups(g, name):
    """{J1.i or None: [count, sum_j or None, count_j, sum_k or None, count_k]} from the golden table.  J1.i of a row is
    recovered from its t column (unique per J1 row up to the two 'zero' rows, which differ in i IS NULL <=> j = 0)."""
    groups = {}
    for r in j1j2_golden_rows(g, name):
        i, j, t, k = r[0], r[1], r[2], r[-1]
        j1_i = None if t is None else next(x[0] for x in g["j1"] if x[2] == t and x[1] == j)
        a = groups.setdefault(j1_i, [0, None, 0, None, 0])
        a[0] += 1
        if j is not None:
            a[1], a[2] = (a[1] or 0) + j, a[2] + 1
        if k is not None:
            a[3], a[4] = (a[3] or 0) + k, a[4] + 1
    return groups


def j1j2_check_groups(rows, want):
    got = {}
    for r in rows:
        key = None if r.keyisnull[0] else int(np.int32(r.key[0] & 0xFFFFFFFF))
        got[key] = [r.agg[0].i, None if r.agg[1].isnull else r.agg[1].i, r.agg[2].i, None if r.agg[3].isnull else r.agg[3].i, r.agg[4].i]
    assert got == want, (got, want)


def sort_golden_cases():
    """[(name, keys, shuffled input rows [n,1] int64, nulls [n,1], golden rows in order, golden nulls)] from the reference's
    expected/sort.out (tests/golden/sort_golden.json): input = the golden values in a fixed shuffled order."""
    g = golden("sort_golden.json")
    typid = {"int8": capi.INT8OID, "int4": capi.INT4OID, "date": capi.DATEOID, "float8": capi.FLOAT8OID, "bpchar": capi.BPCHAROID}

    def datum(t, v):
        if v is None:
            return 0
        if t == "float8":
            return f2b(v)
        if t in ("bpchar", "text"):
            return capi.pack_str(v)[0]
        return int(v)

    def case(name, t, oid, want, desc, nulls_first):
        rng = np.random.default_rng(len(name) * 7 + desc)
        order = rng.permutation(len(want))
        w = np.array([[datum(t, v)] for v in want], dtype=np.int64)
        wn = np.array([[v is None] for v in want], dtype=np.uint8)
        return (name, [capi.make_sortkey(0, oid, desc, nulls_first)], w[order], wn[order], w, wn)

    cases = []
    for col, c in g["alltypes"].items():
        cases.append(case(col + "-asc", c["type"], typid[c["type"]], c["asc"], False, None))
        cases.append(case(col + "-desc", c["type"], typid[c["type"]], c["desc"], True, None))
    cases.append(case("colltest-nulls-last", "text", capi.TEXTOID, g["colltest"]["nulls_last"], False, None))
    cases.append(case("colltest-nulls-first", "text", capi.TEXTOID, g["colltest"]["nulls_first"], False, True))
    return cases


def onek_fixture():
    """(desc, pages, expected): the regression suite's onek table (13 int4 columns, 1000 rows) and the golden aggregates of
    expected/aggregates.out over it (tests/golden/onek.npz, onek_agg_expected.json)."""
    if "onek" not in _fixture_cache:
        ints = np.load(os.path.join(GOLD, "onek.npz"))["ints"]
        desc = make_desc([(capi.INT4OID, 4, "i", 1)] * ints.shape[1])
        _fixture_cache["onek"] = (desc, po.build_pages(desc, [[int(v) for v in r] for r in ints]), golden("onek_agg_expected.json"))
    return _fixture_cache["onek"]


def onek_plans(desc, exp):
    """-> (plain, grouped): `sum(four), max(four), count(four)` and `ten, count(*), sum(four) GROUP BY ten`
    (sql/aggregates.sql:22,27,70,73)"""
    four, ten = exp["columns"].index("four") + 1, exp["columns"].index("ten") + 1
    p = capi.ExprPool()
    plain = capi.make_agg(capi.AGGSTAGE_NORMAL, [], [(capi.AGG_SUM_INT4, p.var(four, capi.INT4OID)), (capi.AGG_MAX_INT4, p.var(four, capi.INT4OID)),
                                                     (capi.AGG_COUNT_ANY, p.var(four, capi.INT4OID))])
    grouped = capi.make_agg(capi.AGGSTAGE_NORMAL, [p.var(ten, capi.INT4OID)], [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_INT4, p.var(four, capi.INT4OID))])
    return (capi.make_scan(desc, -1), plain, p.pool), (capi.make_scan(desc, -1), grouped, p.pool)


def onek_check(exp, plain_rows, grouped_rows):
    assert len(plain_rows) == 1
    a = plain_rows[0].agg
    assert (a[0].i, a[1].i, a[2].i) == (exp["sum_four"], exp["max_four"], exp["count_four"])
    got = sorted([int(np.int32(r.key[0] & 0xFFFFFFFF)), r.agg[0].i, r.agg[1].i] for r in grouped_rows)
    assert got == exp["by_ten"], got


def gp_hashagg_case():
    """MPP-2614 of the reference's sql/gp_hashagg.sql:4-28 (hashed aggregate with a text key behind a three-clause qual;
    golden answer expected/gp_hashagg.out:17-22: hi 9, there 6).  -> (desc, pages, scan, agg, pool, expected {grp: sum})"""
    from datetime import date
    d = lambda m, dd: (date(2006, m, dd) - date(2000, 1, 1)).days
    desc = make_desc([(capi.INT4OID, 4, "i", 1), (capi.INT4OID, 4, "i", 1), (capi.DATEOID, 4, "i", 1), (capi.TEXTOID, -1, "i", 0),
                      (capi.INT4OID, 4, "i", 1)])
    rows = [[1, 1, d(1, 1), b"there", 1], [1, 1, d(1, 2), b"there", 2], [1, 1, d(1, 3), b"there", 3],
            [1, 1, d(1, 1), b"hi", 2], [1, 1, d(1, 2), b"hi", 3], [1, 1, d(1, 3), b"hi", 4]]        # the six INSERTs
    p = capi.ExprPool()
    id1, id2, day, grp, v = (p.var(i + 1, desc.attrs[i].atttypid) for i in range(5))
    q = p.func(capi.F_INT4EQ, capi.BOOLOID, id1, p.const(capi.INT4OID, 1))
    for cond in (p.func(capi.F_INT4EQ, capi.BOOLOID, id2, p.const(capi.INT4OID, 1)),
                 p.func(capi.F_DATE_GE, capi.BOOLOID, day, p.const(capi.DATEOID, d(1, 1))),
                 p.func(capi.F_DATE_LE, capi.BOOLOID, day, p.const(capi.DATEOID, d(1, 31)))):
        q = p.boolop(capi.E_AND, q, cond)
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [grp], [(capi.AGG_SUM_INT4, v)])
    return desc, po.build_pages(desc, rows), capi.make_scan(desc, q), agg, p.pool, {"hi": 9, "there": 6}


# (xmin, xmax, visibility bits of t_infomask) patterns over the xids of mvcc_snapshot() below, and what HeapTupleSatisfiesMVCC
# (tqual.c:997) answers for each: frozen; committed before the snapshot; aborted; in progress; in the snapshot's xip; committed
# after xmin but not in xip; deleted by a committed-after-snapshot-start xact not in xip (gone); deleted by an xip member (still
# there); deleted by an aborted xact; deleted, hinted committed
MVCC_PATTERNS = [(2, 0, 0x0B00, 1), (1001, 0, 0x0800, 1), (1002, 0, 0x0800, 0), (1003, 0, 0x0800, 0), (1004, 0, 0x0800, 0), (1005, 0, 0x0800, 1),
                 (1001, 1005, 0x0000, 0), (1001, 1004, 0x0000, 1), (1001, 1002, 0x0000, 1), (1001, 1001, 0x0500, 0)]


def mvcc_snapshot():
    """xids 1001 committed, 1002 aborted, 1003 in progress, 1004 committed but in progress at snapshot time (xip), 1005 committed"""
    from greengage_b200 import capi
    base, clog = 1000, bytearray(16)
    for x, st in {1001: 1, 1002: 2, 1003: 0, 1004: 1, 1005: 1}.items():
        clog[(x - base) >> 2] |= st << (((x - base) & 3) * 2)
    return capi.make_snapshot(1004, 1006, [1004], 0, 0, base, bytes(clog))


def stamp_visibility(pages, all_visible_every=0):
    """Rewrite xmin / xmax / hint bits of every tuple with MVCC_PATTERNS in turn and clear PD_ALL_VISIBLE (kept on every
    all_visible_every-th page, where heapgetpage then skips the rule, heapam.c:391).  Returns (pages, [visible per tuple])."""
    import struct
    import numpy as np
    pg = np.frombuffer(pages, dtype=np.uint8).copy() if not isinstance(pages, np.ndarray) else pages.copy()
    vis, k = [], 0
    for b in range(len(pg) // 32768):
        page = pg[b * 32768:(b + 1) * 32768]
        keep = all_visible_every and b % all_visible_every == 0
        flags = struct.unpack("<H", page[10:12].tobytes())[0]
        page[10:12] = np.frombuffer(struct.pack("<H", (flags | 0x0004) if keep else (flags & ~0x0004)), dtype=np.uint8)
        lower = struct.unpack("<H", page[12:14].tobytes())[0]
        for i in range((lower - 24) // 4):
            lp = struct.unpack("<I", page[24 + 4 * i:28 + 4 * i].tobytes())[0]
            if (lp >> 15) & 3 != 1:
                continue
            off = lp & 0x7FFF
            xmin, xmax, mask, v = MVCC_PATTERNS[k % len(MVCC_PATTERNS)]
            page[off:off + 8] = np.frombuffer(struct.pack("<II", xmin, xmax), dtype=np.uint8)
            im = struct.unpack("<H", page[off + 20:off + 22].tobytes())[0]
            page[off + 20:off + 22] = np.frombuffer(struct.pack("<H", (im & 0x000F) | mask), dtype=np.uint8)
            vis.append(1 if keep else v)
            k += 1
    return pg, vis
