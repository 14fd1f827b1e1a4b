"""Shared by the window-function tests: the row-at-a-time reference (tests/window_ref.c) through ctypes, a direct statement of the
SQL semantics in Python, and random sorted datum rows with NULLs, ties and float8 -0 / NaN keys."""
import ctypes as C
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from greengage_b200 import capi  # noqa: E402

_libs = {}


def _build(name, src):
    if name not in _libs:
        d = tempfile.mkdtemp(prefix="ggwin")
        so = os.path.join(d, name + ".so")
        subprocess.check_call(["gcc", "-O2", "-Wall", "-Wextra", "-shared", "-fPIC", "-o", so, os.path.join(HERE, src), "-lm"])
        _libs[name] = C.CDLL(so)
    return _libs[name]


def ref_lib():
    L = _build("libwinref", "window_ref.c")
    L.ref_window.argtypes = [C.POINTER(capi.gg_window), C.POINTER(C.c_int32), C.c_int, C.POINTER(capi.gg_exprpool), C.c_void_p,
                             C.c_uint64, C.c_void_p, C.POINTER(C.c_uint64), C.c_char_p, C.c_int]
    return L


def rules_lib():
    L = _build("libwinrules", "window_rules_harness.c")
    L.ntile_mismatches.restype = C.c_int64
    L.ntile_mismatches.argtypes = [C.c_int64, C.c_int32]
    p64 = C.c_void_p
    L.rules_rows.argtypes = [C.c_int32, C.c_int64] + [p64] * 10 + [C.c_int32, p64, C.c_int64, p64]
    return L


def ref_window(win, types, pool, rows):
    """rows: uint64 [n][1 + ncols] (dead slots allowed) -> (rc, out uint64 [m][1 + ncols + nfuncs], message)"""
    rows = np.ascontiguousarray(rows, dtype=np.uint64)
    n, W = rows.shape
    W2 = W + win.numFuncs
    out = np.zeros((max(n, 1), W2), dtype=np.uint64)
    nout = C.c_uint64(0)
    err = C.create_string_buffer(256)
    ty = (C.c_int32 * len(types))(*types)
    rc = ref_lib().ref_window(C.byref(win), ty, len(types), C.byref(pool), rows.ctypes.data, n, out.ctypes.data, C.byref(nout), err, 256)
    return rc, out[:nout.value].copy(), err.value.decode()


def f2u(x):
    return int(np.array([x], dtype=np.float64).view(np.uint64)[0])


def u2f(u):
    return float(np.array([u], dtype=np.uint64).view(np.float64)[0])


KEYVALS = {
    capi.INT4OID: lambda rng, k: rng.integers(-3, 3, k),
    capi.INT8OID: lambda rng, k: rng.integers(-2 ** 40, -2 ** 40 + 4, k),
    capi.DATEOID: lambda rng, k: rng.integers(7000, 7004, k),
    capi.BOOLOID: lambda rng, k: rng.integers(0, 2, k),
}


def _key_words(rng, typ, k, nkeys):
    """k values of a key column of `typ` with few distinct values (ties), as (words, isnull)"""
    if typ == capi.FLOAT8OID:
        pool = np.array([-0.0, 0.0, 1.5, float("nan"), -2.0, float("-inf")])
        v = pool[rng.integers(0, min(len(pool), nkeys + 2), k)]
        if rng.random() < 0.5:                                         # NaNs with different payloads are still equal
            nan2 = np.array([0x7ff8000000000123], dtype=np.uint64).view(np.float64)[0]
            v = np.where(np.isnan(v) & (rng.random(k) < 0.5), nan2, v)
        w = v.view(np.uint64)
    elif typ in (capi.BPCHAROID, capi.TEXTOID, capi.VARCHAROID):
        strs = ["", "a", "ab", "abcdefgh", "zz"]
        w = np.array([capi.pack_str(strs[i], False)[0] & 0xFFFFFFFFFFFFFFFF for i in rng.integers(0, min(len(strs), nkeys + 1), k)],
                     dtype=np.uint64)
    else:
        w = KEYVALS[typ](rng, k).astype(np.int64).view(np.uint64)
    return w, rng.random(k) < 0.15


def sort_key(typ, w, isnull):
    """an order-preserving key of one column (NULLs last), for sorting the generated rows the way a Sort would"""
    if isnull:
        return (1, 0)
    if typ == capi.FLOAT8OID:
        x = u2f(int(w))
        return (0, (1, 0.0) if x != x else (0, x + 0.0))
    if typ in (capi.BPCHAROID, capi.TEXTOID, capi.VARCHAROID):
        return (0, int(w).to_bytes(8, "little"))
    return (0, int(np.uint64(w).view(np.int64)))


def random_rows(rng, n, ktypes, vtypes, dead=0.0, nkeys=3):
    """n rows: key columns of ktypes, then value columns of vtypes; sorted on all key columns; some slots dead.  Returns
    (rows uint64 [n][1 + ncols], types)"""
    types = list(ktypes) + list(vtypes)
    ncols = len(types)
    rows = np.zeros((n, 1 + ncols), dtype=np.uint64)
    for c, t in enumerate(types):
        if c < len(ktypes):
            w, nl = _key_words(rng, t, n, nkeys)
        elif t == capi.FLOAT8OID:
            w = (rng.integers(-1000, 1000, n) / 8.0).astype(np.float64).view(np.uint64)
            nl = rng.random(n) < 0.2
        elif t == capi.INT4OID:
            w = rng.integers(-2 ** 31, 2 ** 31, n).astype(np.int64).view(np.uint64)
            nl = rng.random(n) < 0.2
        else:
            w = rng.integers(-2 ** 62, 2 ** 62, n).astype(np.int64).view(np.uint64)
            nl = rng.random(n) < 0.2
        w = np.where(nl, np.uint64(0), w)
        rows[:, 1 + c] = w
        rows[:, 0] |= nl.astype(np.uint64) << np.uint64(c)
    order = sorted(range(n), key=lambda r: tuple(sort_key(types[c], rows[r, 1 + c], (int(rows[r, 0]) >> c) & 1) for c in range(len(ktypes))))
    rows = rows[order]
    if dead:
        rows[rng.random(n) < dead, 0] |= np.uint64(1 << 63)
    return rows, types


# ---- the SQL semantics stated directly, row by row ----

def _match(a, b, cols, types):
    for c in cols:
        na, nb = (int(a[0]) >> c) & 1, (int(b[0]) >> c) & 1
        if na != nb:
            return False
        if na:
            continue
        if types[c] == capi.FLOAT8OID:
            x, y = u2f(int(a[1 + c])), u2f(int(b[1 + c]))
            if (x != x) != (y != y) or (x == x and x != y):
                return False
        elif a[1 + c] != b[1 + c]:
            return False
    return True


def bounds(win, types, rows):
    """per live row: its partition [ps, pe) and peer group [gs, ge), as runs of the sorted input"""
    live = [r for r in rows if not int(r[0]) >> 63]
    m = len(live)
    pstart, gstart = [0] * m, [0] * m
    for j in range(1, m):
        pstart[j] = pstart[j - 1] if _match(live[j], live[j - 1], list(win.partColIdx[:win.partNumCols]), types) else j
        gstart[j] = gstart[j - 1] if pstart[j] == pstart[j - 1] and _match(live[j], live[j - 1], list(win.ordColIdx[:win.ordNumCols]), types) else j
    pend, gend = [m] * m, [m] * m
    for j in range(m - 2, -1, -1):
        pend[j] = pend[j + 1] if pstart[j + 1] == pstart[j] else j + 1
        gend[j] = gend[j + 1] if gstart[j + 1] == gstart[j] else j + 1
    return pstart, pend, gstart, gend


def naive_window(win, types, pool, rows):
    """(error or None, [[value or None, ...] per live row]) — each result from its definition: the partition is every row equal
    on the partition columns, the peers those also equal on the order columns, the frame the rows the frame clause names"""
    live = [r for r in rows if not int(r[0]) >> 63]
    m = len(live)
    pstart, pend, gstart, gend = bounds(win, types, rows)
    opt = win.frameOptions
    rowsmode = bool(opt & capi.FRAMEOPTION_ROWS)
    out = []

    def arg(i, a, r):
        root = win.funcs[i].arg[a]
        nd = pool.nodes[root]
        if nd.kind == capi.E_VAR:
            c = nd.varattno - 1
            return None if (int(r[0]) >> c) & 1 else int(r[1 + c])
        return None if nd.constisnull else int(nd.constvalue) & 0xFFFFFFFFFFFFFFFF

    def s32(u):
        u &= 0xFFFFFFFF
        return u - (1 << 32) if u >= 1 << 31 else u

    def s64(u):
        u &= 0xFFFFFFFFFFFFFFFF
        return u - (1 << 64) if u >= 1 << 63 else u

    for j in range(m):
        ps, pe, gs, ge = pstart[j], pend[j], gstart[j], gend[j]
        head = ps if opt & capi.FRAMEOPTION_START_UNBOUNDED_PRECEDING else (j if rowsmode else gs)
        tail = pe - 1 if opt & capi.FRAMEOPTION_END_UNBOUNDED_FOLLOWING else (j if rowsmode else ge - 1)
        res = []
        for i in range(win.numFuncs):
            fn = win.funcs[i].winfnoid
            total = pe - ps
            rank = gs - ps + 1
            if fn == capi.WF_ROW_NUMBER:
                v = j - ps + 1
            elif fn == capi.WF_RANK:
                v = rank
            elif fn == capi.WF_DENSE_RANK:
                v = len({gstart[k] for k in range(ps, j + 1)})
            elif fn == capi.WF_PERCENT_RANK:
                v = 0.0 if total <= 1 else (rank - 1) / (total - 1)
            elif fn == capi.WF_CUME_DIST:
                v = (ge - ps) / total
            elif fn == capi.WF_NTILE:
                nb = arg(i, 0, live[j])
                if nb is None:
                    v = None
                elif s32(nb) <= 0:
                    return "ntile", None
                else:
                    # bucket sizes: total // n each, the first total % n one more
                    nb = s32(nb)
                    sizes = [total // nb + (1 if b < total % nb else 0) for b in range(nb)]
                    k, b = j - ps, 0
                    while k >= sizes[b]:
                        k -= sizes[b]
                        b += 1
                    v = b + 1
            elif capi.WF_LAG <= fn <= capi.WF_LEAD_DEFAULT:
                off = 1
                if win.funcs[i].arg[1] >= 0:
                    off = arg(i, 1, live[j])
                    off = None if off is None else s32(off)
                if off is None:
                    v = None
                else:
                    t = j + off if fn >= capi.WF_LEAD else j - off
                    if ps <= t < pe:
                        v = arg(i, 0, live[t])
                    else:
                        v = arg(i, 2, live[j]) if win.funcs[i].arg[2] >= 0 else None
            elif fn == capi.WF_FIRST_VALUE:
                v = arg(i, 0, live[head])
            elif fn == capi.WF_LAST_VALUE:
                v = arg(i, 0, live[tail])
            elif fn == capi.WF_NTH_VALUE:
                nth = arg(i, 1, live[j])
                if nth is None:
                    v = None
                elif s32(nth) <= 0:
                    return "nth_value", None
                else:
                    t = head + s32(nth) - 1
                    v = arg(i, 0, live[t]) if t <= tail else None
            else:
                frame = live[head:tail + 1]
                xs = [] if fn == capi.AGG_COUNT_STAR else [x for x in (arg(i, 0, r) for r in frame) if x is not None]
                if fn == capi.AGG_COUNT_STAR:
                    v = len(frame)
                elif fn == capi.AGG_COUNT_ANY:
                    v = len(xs)
                elif not xs:
                    v = None
                elif fn == capi.AGG_SUM_INT4:
                    v = sum(s64(x) for x in xs)
                elif fn in (capi.AGG_SUM_FLOAT8, capi.AGG_AVG_FLOAT8):
                    s = u2f(xs[0]) if fn == capi.AGG_SUM_FLOAT8 else 0.0 + u2f(xs[0])
                    for x in xs[1:]:
                        s += u2f(x)
                    v = s if fn == capi.AGG_SUM_FLOAT8 else s / len(xs)
                elif fn in (capi.AGG_MIN_FLOAT8, capi.AGG_MAX_FLOAT8):
                    fs = [u2f(x) for x in xs]
                    key = [(1, 0.0) if f != f else (0, f) for f in fs]
                    best = max(key) if fn == capi.AGG_MAX_FLOAT8 else min(key)
                    v = float("nan") if best[0] else best[1]
                else:
                    ints = [s64(x) for x in xs]
                    v = max(ints) if fn in (capi.AGG_MAX_INT4, capi.AGG_MAX_INT8, capi.AGG_MAX_DATE) else min(ints)
            res.append(v)
        out.append(res)
    return None, out


def decode(win, types, out, ncols):
    """reference / device output rows -> [[value or None, ...]] of the function columns, floats as Python floats, ints signed"""
    res = []
    for r in out:
        row = []
        for i in range(win.numFuncs):
            if (int(r[0]) >> (ncols + i)) & 1:
                row.append(None)
                continue
            u = int(r[1 + ncols + i])
            t = win.funcs[i].wintype
            if t == capi.FLOAT8OID:
                row.append(u2f(u))
            elif t in (capi.INT4OID, capi.DATEOID, capi.INT8OID, capi.BOOLOID):
                row.append(u - (1 << 64) if u >= 1 << 63 else u)
            else:
                row.append(u)
        res.append(row)
    return res


FRAMES = {
    "range_up_cr": capi.FRAMEOPTION_DEFAULTS,
    "rows_up_cr": capi.FRAMEOPTION_NONDEFAULT | capi.FRAMEOPTION_ROWS | capi.FRAMEOPTION_START_UNBOUNDED_PRECEDING | capi.FRAMEOPTION_END_CURRENT_ROW,
    "range_up_uf": capi.FRAMEOPTION_NONDEFAULT | capi.FRAMEOPTION_RANGE | capi.FRAMEOPTION_BETWEEN | capi.FRAMEOPTION_START_UNBOUNDED_PRECEDING |
    capi.FRAMEOPTION_END_UNBOUNDED_FOLLOWING,
    "rows_up_uf": capi.FRAMEOPTION_NONDEFAULT | capi.FRAMEOPTION_ROWS | capi.FRAMEOPTION_BETWEEN | capi.FRAMEOPTION_START_UNBOUNDED_PRECEDING |
    capi.FRAMEOPTION_END_UNBOUNDED_FOLLOWING,
    "range_cr_uf": capi.FRAMEOPTION_NONDEFAULT | capi.FRAMEOPTION_RANGE | capi.FRAMEOPTION_BETWEEN | capi.FRAMEOPTION_START_CURRENT_ROW |
    capi.FRAMEOPTION_END_UNBOUNDED_FOLLOWING,
    "rows_cr_uf": capi.FRAMEOPTION_NONDEFAULT | capi.FRAMEOPTION_ROWS | capi.FRAMEOPTION_BETWEEN | capi.FRAMEOPTION_START_CURRENT_ROW |
    capi.FRAMEOPTION_END_UNBOUNDED_FOLLOWING,
    "range_cr_cr": capi.FRAMEOPTION_NONDEFAULT | capi.FRAMEOPTION_RANGE | capi.FRAMEOPTION_BETWEEN | capi.FRAMEOPTION_START_CURRENT_ROW |
    capi.FRAMEOPTION_END_CURRENT_ROW,
    "rows_cr_cr": capi.FRAMEOPTION_NONDEFAULT | capi.FRAMEOPTION_ROWS | capi.FRAMEOPTION_BETWEEN | capi.FRAMEOPTION_START_CURRENT_ROW |
    capi.FRAMEOPTION_END_CURRENT_ROW,
}


def all_funcs(pool, ncols, types, kcols, vcols):
    """one plan's worth of functions per group (at most 8 each): ranking, value and aggregate functions over the columns"""
    f8 = [c for c in vcols if types[c] == capi.FLOAT8OID]
    i4 = [c for c in vcols if types[c] == capi.INT4OID]
    i8 = [c for c in vcols if types[c] == capi.INT8OID]
    v = lambda c: pool.var(c + 1, types[c])                                  # noqa: E731
    ranking = [(capi.WF_ROW_NUMBER, capi.INT8OID, []), (capi.WF_RANK, capi.INT8OID, []), (capi.WF_DENSE_RANK, capi.INT8OID, []),
               (capi.WF_PERCENT_RANK, capi.FLOAT8OID, []), (capi.WF_CUME_DIST, capi.FLOAT8OID, []),
               (capi.WF_NTILE, capi.INT4OID, [pool.const(capi.INT4OID, 3)]), (capi.WF_NTILE, capi.INT4OID, [pool.const(capi.INT4OID, 7)])]
    c0 = (f8 + i4 + i8)[0]
    value = [(capi.WF_LAG, types[c0], [v(c0)]), (capi.WF_LEAD, types[c0], [v(c0)]),
             (capi.WF_LAG_DEFAULT, types[c0], [v(c0), pool.const(capi.INT4OID, 2), v(c0)]),
             (capi.WF_FIRST_VALUE, types[c0], [v(c0)]), (capi.WF_LAST_VALUE, types[c0], [v(c0)]),
             (capi.WF_NTH_VALUE, types[c0], [v(c0), pool.const(capi.INT4OID, 2)])]
    if i4:
        value += [(capi.WF_LEAD_OFFSET, types[c0], [v(c0), v(i4[0])])]
    aggs = [(capi.AGG_COUNT_STAR, capi.INT8OID, [])]
    if f8:
        aggs += [(capi.AGG_SUM_FLOAT8, capi.FLOAT8OID, [v(f8[0])]), (capi.AGG_AVG_FLOAT8, capi.FLOAT8OID, [v(f8[0])]),
                 (capi.AGG_MIN_FLOAT8, capi.FLOAT8OID, [v(f8[0])]), (capi.AGG_MAX_FLOAT8, capi.FLOAT8OID, [v(f8[0])]),
                 (capi.AGG_COUNT_ANY, capi.INT8OID, [v(f8[0])])]
    if i4:
        aggs += [(capi.AGG_SUM_INT4, capi.INT8OID, [v(i4[0])]), (capi.AGG_MIN_INT4, capi.INT4OID, [v(i4[0])])]
    if i8:
        aggs += [(capi.AGG_MAX_INT8, capi.INT8OID, [v(i8[0])])]
    return [ranking, value, aggs[:8]]


# ---- the window.out goldens (tests/golden/window_expected.json over tests/golden/tenk1.npz) ----
# input columns of tenk1: 0 unique2, 1 two, 2 four, 3 ten (int4); of the VALUES relation: 0 i, 1 v
_T = dict(unique2=0, two=1, four=2, ten=3)
GOLDEN = {
    # id: (relation, filter, partition, order, frame, [(fn, type, [arg columns or ("const", v)])], printed items)
    "count_over_empty": ("tenk1", "u10", [], [], "range_up_cr", [(capi.AGG_COUNT_STAR, capi.INT8OID, [])], ["f0"]),
    "sum_cumulative": ("tenk1", "u10", [3], [0], "range_up_cr", [(capi.AGG_SUM_INT4, capi.INT8OID, [2])], ["f0", "c3", "c2"]),
    "row_number": ("tenk1", "u10", [], [0], "range_up_cr", [(capi.WF_ROW_NUMBER, capi.INT8OID, [])], ["f0"]),
    "rank": ("tenk1", "u10", [2], [3], "range_up_cr", [(capi.WF_RANK, capi.INT8OID, [])], ["f0", "c3", "c2"]),
    "dense_rank": ("tenk1", "u10", [2], [3], "range_up_cr", [(capi.WF_DENSE_RANK, capi.INT8OID, [])], ["f0", "c3", "c2"]),
    "percent_rank": ("tenk1", "u10", [2], [3], "range_up_cr", [(capi.WF_PERCENT_RANK, capi.FLOAT8OID, [])], ["f0", "c3", "c2"]),
    "cume_dist": ("tenk1", "u10", [2], [3], "range_up_cr", [(capi.WF_CUME_DIST, capi.FLOAT8OID, [])], ["f0", "c3", "c2"]),
    "ntile3": ("tenk1", "u10", [], [3, 2], "range_up_cr", [(capi.WF_NTILE, capi.INT4OID, [("const", 3)])], ["f0", "c3", "c2"]),
    "lag": ("tenk1", "u10", [2], [3], "range_up_cr", [(capi.WF_LAG, capi.INT4OID, [3])], ["f0", "c3", "c2"]),
    "lag_offset": ("tenk1", "u10", [2], [3], "range_up_cr", [(capi.WF_LAG_OFFSET, capi.INT4OID, [3, 2])], ["f0", "c3", "c2"]),
    "lag_default": ("tenk1", "u10", [2], [3], "range_up_cr", [(capi.WF_LAG_DEFAULT, capi.INT4OID, [3, 2, ("const", 0)])], ["f0", "c3", "c2"]),
    "lead": ("tenk1", "u10", [2], [3], "range_up_cr", [(capi.WF_LEAD, capi.INT4OID, [3])], ["f0", "c3", "c2"]),
    "first_value": ("tenk1", "u10", [2], [3], "range_up_cr", [(capi.WF_FIRST_VALUE, capi.INT4OID, [3])], ["f0", "c3", "c2"]),
    "last_value_order": ("tenk1", "u10", [], [3], "range_up_cr", [(capi.WF_LAST_VALUE, capi.INT4OID, [3])], ["f0", "c3", "c2"]),
    "last_value_partition": ("tenk1", "u10", [2], [3], "range_up_cr", [(capi.WF_LAST_VALUE, capi.INT4OID, [3])], ["f0", "c3", "c2"]),
    "count_partition_subquery": ("tenk1", "u10_two1", [2], [], "range_up_cr", [(capi.AGG_COUNT_STAR, capi.INT8OID, [])], ["f0", "c2"]),
    "values_sum_int": ("values", None, [], [0], "rows_cr_uf", [(capi.AGG_SUM_INT4, capi.INT8OID, [1])], ["c0", "f0"]),
    "values_count_v": ("values", None, [], [0], "rows_cr_uf", [(capi.AGG_COUNT_ANY, capi.INT8OID, [1])], ["c0", "f0"]),
    "values_count_star": ("values", None, [], [0], "rows_cr_uf", [(capi.AGG_COUNT_STAR, capi.INT8OID, [])], ["c0", "f0"]),
}


def golden_cases():
    """(id, gg_window, input types, ExprPool, sorted input rows uint64 [n][W], printed items, the expected printed rows)"""
    import json
    expected = json.load(open(os.path.join(HERE, "golden", "window_expected.json")))
    t = np.load(os.path.join(HERE, "golden", "tenk1.npz"))
    tenk = np.stack([t[k].astype(np.int64) for k in ("unique2", "two", "four", "ten")], axis=1)
    for gid, (relname, flt, part, order, frame, funcs, items) in sorted(GOLDEN.items()):
        if relname == "tenk1":
            keep = tenk[:, 0] < 10
            if flt == "u10_two1":
                keep &= tenk[:, 1] == 1
            vals, nulls = tenk[keep], np.zeros((int(keep.sum()), 4), dtype=bool)
        else:
            vals = np.array([[1, 1], [2, 2], [3, 0], [4, 0]], dtype=np.int64)
            nulls = np.array([[0, 0], [0, 0], [0, 1], [0, 1]], dtype=bool)
        ncols = vals.shape[1]
        types = [capi.INT4OID] * ncols
        # the Sort below the WindowAgg: partition columns, then order columns (stable)
        keys = [vals[:, c] for c in reversed(part + order)]
        idx = np.lexsort(keys) if keys else np.arange(len(vals))
        rows = np.zeros((len(vals), 1 + ncols), dtype=np.uint64)
        rows[:, 1:] = vals[idx].view(np.uint64)
        for c in range(ncols):
            rows[:, 0] |= nulls[idx, c].astype(np.uint64) << np.uint64(c)
            rows[nulls[idx, c], 1 + c] = 0
        pool = capi.ExprPool()
        fl = [(fn, ty, [pool.const(capi.INT4OID, a[1]) if isinstance(a, tuple) else pool.var(a + 1, capi.INT4OID) for a in args])
              for fn, ty, args in funcs]
        yield gid, capi.make_window(part, order, FRAMES[frame], fl), types, pool, rows, items, expected[gid]


def printed(win, out, ncols, items):
    """output rows as the reference prints them: integers as they are, float8 with 15 significant digits, NULL empty"""
    vals = decode(win, None, out, ncols)
    res = []
    for r, fv in zip(out, vals):
        row = []
        for it in items:
            if it[0] == "f":
                v = fv[int(it[1:])]
                row.append("" if v is None else ("%.15g" % v if isinstance(v, float) else str(v)))
            else:
                c = int(it[1:])
                row.append("" if (int(r[0]) >> c) & 1 else str(int(np.uint64(r[1 + c]).view(np.int64))))
        res.append(row)
    return res
