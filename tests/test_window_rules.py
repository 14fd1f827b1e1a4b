"""WindowAgg without a GPU: the row-at-a-time reference (tests/window_ref.c) against a direct statement of the SQL semantics, and the
per-row rules the kernels share (greengage_b200/csrc/gg_window.h, compiled with gcc) against the reference and windowfuncs.c."""
import math

import numpy as np
import pytest

from _window import FRAMES, all_funcs, bounds, decode, naive_window, random_rows, ref_window, rules_lib, u2f
from greengage_b200 import capi


def test_ntile_closed_form_equals_the_windowfuncs_loop():
    assert rules_lib().ntile_mismatches(2000, 64) == 0


def _same(a, b, fn):
    if a is None or b is None:
        return a is None and b is None
    if isinstance(a, float) or isinstance(b, float):
        if a != a or b != b:
            return a != a and b != b
        if fn in (capi.AGG_MIN_FLOAT8, capi.AGG_MAX_FLOAT8, capi.WF_FIRST_VALUE, capi.WF_LAST_VALUE) and a == 0 and b == 0:
            return True
        return math.copysign(1, a) == math.copysign(1, b) and a == b if a == 0 else a == b
    return a == b


def _check_against_naive(win, types, pool, rows, ncols):
    rc, out, msg = ref_window(win, types, pool, rows)
    err, want = naive_window(win, types, pool, rows)
    if err:
        assert rc == capi.ERR_WINDOW_ARG and err in msg, (rc, msg, err)
        return
    assert rc == 0, msg
    got = decode(win, types, out, ncols)
    # value functions over float8 columns decode their bits as floats; the naive statement returns the raw words
    for j, (g, w) in enumerate(zip(got, want)):
        for i, (a, b) in enumerate(zip(g, w)):
            fn = win.funcs[i].winfnoid
            if win.funcs[i].wintype == capi.FLOAT8OID and isinstance(b, int):
                b = u2f(b)
            elif win.funcs[i].wintype in (capi.INT4OID, capi.INT8OID, capi.DATEOID) and isinstance(b, int) and b >= 1 << 63:
                b -= 1 << 64
            assert _same(a, b, fn), (j, i, fn, a, b)
    assert len(got) == len(want)


KEYS = [[capi.INT4OID], [capi.INT8OID, capi.FLOAT8OID], [capi.DATEOID], [capi.BOOLOID, capi.TEXTOID], [capi.FLOAT8OID]]


@pytest.mark.parametrize("frame", sorted(FRAMES))
@pytest.mark.parametrize("keys", range(len(KEYS)))
def test_reference_equals_the_sql_semantics(frame, keys):
    rng = np.random.default_rng(sorted(FRAMES).index(frame) * 10 + keys)
    ktypes = KEYS[keys]
    vtypes = [capi.FLOAT8OID, capi.INT4OID, capi.INT8OID]
    for n, npart, dead in ((0, 1, 0.0), (1, 1, 0.0), (150, 1, 0.1), (150, len(ktypes), 0.0), (60, len(ktypes), 0.3)):
        rows, types = random_rows(rng, n, ktypes, vtypes, dead=dead)
        ncols = len(types)
        kcols = list(range(len(ktypes)))
        vcols = list(range(len(ktypes), ncols))
        for funcs_of in range(3):
            pool = capi.ExprPool()
            funcs = all_funcs(pool, ncols, types, kcols, vcols)[funcs_of]
            part, order = kcols[:npart], kcols[npart:]
            if npart == len(ktypes) and len(ktypes) == 1 and n > 100:
                part, order = [], kcols                              # one partition, ordered
            win = capi.make_window(part, order, FRAMES[frame], funcs)
            _check_against_naive(win, types, pool.pool, rows, ncols)


def test_one_row_partitions_and_no_order():
    rng = np.random.default_rng(5)
    rows, types = random_rows(rng, 80, [capi.INT8OID], [capi.FLOAT8OID, capi.INT4OID, capi.INT8OID], nkeys=80)
    rows[:, 1] = np.arange(80, dtype=np.uint64)                         # every partition a single row
    rows[:, 0] &= ~np.uint64(1)
    for frame in FRAMES.values():
        for g in range(3):
            pool = capi.ExprPool()
            win = capi.make_window([0], [], frame, all_funcs(pool, 4, types, [0], [1, 2, 3])[g])
            _check_against_naive(win, types, pool.pool, rows, 4)


def test_errors_of_ntile_and_nth_value_need_a_row():
    rng = np.random.default_rng(9)
    rows, types = random_rows(rng, 20, [capi.INT4OID], [capi.FLOAT8OID])
    for fn, args, word in ((capi.WF_NTILE, lambda p: [p.const(capi.INT4OID, 0)], "ntile"),
                           (capi.WF_NTH_VALUE, lambda p: [p.var(2, capi.FLOAT8OID), p.const(capi.INT4OID, -1)], "nth_value")):
        pool = capi.ExprPool()
        ty = capi.INT4OID if fn == capi.WF_NTILE else capi.FLOAT8OID
        win = capi.make_window([0], [], capi.FRAMEOPTION_DEFAULTS, [(fn, ty, args(pool))])
        rc, out, msg = ref_window(win, types, pool.pool, rows)
        assert rc == capi.ERR_WINDOW_ARG and msg == "argument of %s must be greater than zero" % word
        rc, out, msg = ref_window(win, types, pool.pool, rows[:0])
        assert rc == 0 and len(out) == 0


def test_float8_sum_overflow_raises():
    rows = np.zeros((4, 3), dtype=np.uint64)
    rows[:, 2] = np.array([1e308, 1e308, -1.0, 2.0]).view(np.uint64)
    pool = capi.ExprPool()
    x = pool.var(2, capi.FLOAT8OID)
    for fn in (capi.AGG_SUM_FLOAT8, capi.AGG_AVG_FLOAT8):
        win = capi.make_window([], [], capi.FRAMEOPTION_DEFAULTS, [(fn, capi.FLOAT8OID, [x])])
        rc, out, msg = ref_window(win, [capi.INT4OID, capi.FLOAT8OID], pool.pool, rows)
        assert rc == -2, (fn, rc)          # GG_ERR_FLOAT_OVERFLOW


@pytest.mark.parametrize("frame", sorted(FRAMES))
def test_rules_equal_the_reference(frame):
    """ranks, percent_rank, cume_dist, ntile, the frame's first and last row and lag's row from gg_window.h, given each row's
    partition and peer group, against the reference's values over a column holding the row's position"""
    rng = np.random.default_rng(11)
    rows, types = random_rows(rng, 400, [capi.INT4OID, capi.FLOAT8OID], [capi.INT8OID], dead=0.1)
    live = ~(rows[:, 0] >> np.uint64(63)).astype(bool)
    rows[live, 3] = np.arange(int(live.sum()), dtype=np.uint64)         # the row's position among the live rows
    rows[:, 0] &= ~np.uint64(4)
    pool = capi.ExprPool()
    pos = pool.var(3, capi.INT8OID)
    funcs = [(capi.WF_ROW_NUMBER, capi.INT8OID, []), (capi.WF_RANK, capi.INT8OID, []), (capi.WF_PERCENT_RANK, capi.FLOAT8OID, []),
             (capi.WF_CUME_DIST, capi.FLOAT8OID, []), (capi.WF_NTILE, capi.INT4OID, [pool.const(capi.INT4OID, 5)]),
             (capi.WF_FIRST_VALUE, capi.INT8OID, [pos]), (capi.WF_LAST_VALUE, capi.INT8OID, [pos]),
             (capi.WF_LAG_OFFSET, capi.INT8OID, [pos, pool.const(capi.INT4OID, -2)])]
    win = capi.make_window([0], [1], FRAMES[frame], funcs)
    rc, out, msg = ref_window(win, types, pool.pool, rows)
    assert rc == 0, msg
    ps, pe, gs, ge = (np.array(a, dtype=np.int64) for a in bounds(win, types, rows))
    m = len(ps)
    res = {k: np.zeros(m, dtype=np.int64) for k in ("rownum", "rank", "head", "tail", "lagrow")}
    prank, cdist, ntile = np.zeros(m), np.zeros(m), np.zeros(m, dtype=np.int32)
    rules_lib().rules_rows(FRAMES[frame], m, ps.ctypes.data, pe.ctypes.data, gs.ctypes.data, ge.ctypes.data, res["rownum"].ctypes.data,
                           res["rank"].ctypes.data, prank.ctypes.data, cdist.ctypes.data, res["head"].ctypes.data, res["tail"].ctypes.data,
                           5, ntile.ctypes.data, -2, res["lagrow"].ctypes.data)
    f = out[:, 4:].view(np.int64)
    assert np.array_equal(f[:, 0], res["rownum"]) and np.array_equal(f[:, 1], res["rank"])
    assert np.array_equal(out[:, 6].view(np.float64), prank) and np.array_equal(out[:, 7].view(np.float64), cdist)
    assert np.array_equal(f[:, 4], ntile.astype(np.int64))
    assert np.array_equal(f[:, 5], res["head"]) and np.array_equal(f[:, 6], res["tail"])
    lagnull = ((out[:, 0] >> np.uint64(3 + 7)) & np.uint64(1)).astype(bool)
    assert np.array_equal(lagnull, res["lagrow"] < 0) and np.array_equal(f[~lagnull, 7], res["lagrow"][~lagnull])


def test_reference_reproduces_the_window_out_goldens():
    from collections import Counter
    from _window import golden_cases, printed
    n = 0
    for gid, win, types, pool, rows, items, want in golden_cases():
        rc, out, msg = ref_window(win, types, pool.pool, rows)
        assert rc == 0, (gid, msg)
        assert Counter(map(tuple, printed(win, out, len(types), items))) == Counter(map(tuple, want)), gid
        n += 1
    assert n == 19
