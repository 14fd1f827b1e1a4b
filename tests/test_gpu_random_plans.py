"""Randomised plans: expression trees drawn at random (arithmetic, comparisons, three-valued AND/OR/NOT, NULL tests,
casts, date and string comparisons) over a relation with NULLs, evaluated as scan quals and aggregate arguments on
the GPU (interpreter and plan-specialised kernels) and by the oracle.  Where the oracle raises an arithmetic ERROR
(overflow, underflow, division by zero) the GPU must raise one too."""
import numpy as np
import pytest

from _util import assert_aggrows_match, make_desc
from greengage_b200 import capi
from greengage_b200.capi import ExprPool
from oracle import pyoracle as po
from test_gpu_scanagg import env, gpu_scanagg  # noqa: F401

pytestmark = pytest.mark.gpu
ARITH_ERRORS = {-2, -3, -4, -5, -11}


@pytest.fixture(scope="module")
def eng():
    from greengage_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def relation():
    rng = np.random.default_rng(77)
    # g int4 (group), a int4, b int4 NULLable, x float8, y float8 NULLable, s bpchar(2) NULLable, d date, k int8
    desc = make_desc([(capi.INT4OID, 4, "i", 1, 1), (capi.INT4OID, 4, "i", 1, 1), (capi.INT4OID, 4, "i", 1, 0), (capi.FLOAT8OID, 8, "d", 1, 1),
                      (capi.FLOAT8OID, 8, "d", 1, 0), (capi.BPCHAROID, -1, "i", 0, 0), (capi.DATEOID, 4, "i", 1, 1), (capi.INT8OID, 8, "d", 1, 1)])
    rows, nulls = [], []
    for _ in range(20_000):
        rows.append([int(rng.integers(0, 5)), int(rng.integers(-20, 20)), int(rng.integers(-5, 5)), float(rng.integers(-40, 40)) / 4,
                     float(rng.choice([0.0, -0.0, 0.5, -1.25, 3.0, 1e-3, float(rng.integers(-9, 9))])), bytes([65 + int(rng.integers(0, 3))]) + b" ",
                     int(rng.integers(-400, 400)), int(rng.integers(-10**9, 10**9))])
        nulls.append([False, False, rng.random() < 0.15, False, rng.random() < 0.15, rng.random() < 0.1, False, False])
    return desc, po.build_pages(desc, rows, nulls)


class Gen:
    def __init__(self, rng, p):
        self.rng, self.p = rng, p

    def f8(self, depth):
        r, p = self.rng, self.p
        c = r.integers(0, 6 if depth > 0 else 3)
        if c == 0: return p.var(4, capi.FLOAT8OID)
        if c == 1: return p.var(5, capi.FLOAT8OID)
        if c == 2: return p.const(capi.FLOAT8OID, float(r.choice([0.0, 1.0, -2.5, 0.125, 100.0])), isnull=bool(r.random() < 0.05))
        if c == 3: return p.func(capi.F_I4TOD, capi.FLOAT8OID, p.var(int(r.choice([2, 3])), capi.INT4OID))
        fn = int(r.choice([capi.F_FLOAT8PL, capi.F_FLOAT8MI, capi.F_FLOAT8MUL, capi.F_FLOAT8DIV]))
        return p.func(fn, capi.FLOAT8OID, self.f8(depth - 1), self.f8(depth - 1))

    def boolean(self, depth):
        r, p = self.rng, self.p
        c = r.integers(0, 9 if depth > 0 else 5)
        if c == 0:
            fn = int(r.choice([capi.F_FLOAT8EQ, capi.F_FLOAT8NE, capi.F_FLOAT8LT, capi.F_FLOAT8LE, capi.F_FLOAT8GT, capi.F_FLOAT8GE]))
            return p.func(fn, capi.BOOLOID, self.f8(1), self.f8(1))
        if c == 1:
            fn = int(r.choice([capi.F_INT4EQ, capi.F_INT4NE, capi.F_INT4LT, capi.F_INT4LE, capi.F_INT4GT, capi.F_INT4GE]))
            rhs = p.var(3, capi.INT4OID) if r.random() < 0.5 else p.const(capi.INT4OID, int(r.integers(-5, 5)))
            return p.func(fn, capi.BOOLOID, p.var(2, capi.INT4OID), rhs)
        if c == 2:
            fn = int(r.choice([capi.F_DATE_LT, capi.F_DATE_GE, capi.F_DATE_EQ, capi.F_DATE_NE]))
            return p.func(fn, capi.BOOLOID, p.var(7, capi.DATEOID), p.const(capi.DATEOID, int(r.integers(-300, 300))))
        if c == 3:
            fn = int(r.choice([capi.F_BPCHAREQ, capi.F_BPCHARNE]))
            return p.func(fn, capi.BOOLOID, p.var(6, capi.BPCHAROID), p.const(capi.BPCHAROID, str(r.choice(["A", "B", "C "]))))
        if c == 4:
            fn = int(r.choice([capi.F_INT8GT, capi.F_INT8LE]))
            return p.func(fn, capi.BOOLOID, p.var(8, capi.INT8OID), p.const(capi.INT8OID, int(r.integers(-10**9, 10**9))))
        if c == 5: return p.boolop(capi.E_AND, self.boolean(depth - 1), self.boolean(depth - 1))
        if c == 6: return p.boolop(capi.E_OR, self.boolean(depth - 1), self.boolean(depth - 1))
        if c == 7: return p.boolop(capi.E_NOT, self.boolean(depth - 1))
        arg = self.f8(1) if r.random() < 0.5 else p.var(int(r.choice([3, 5, 6])), {3: capi.INT4OID, 5: capi.FLOAT8OID, 6: capi.BPCHAROID}[int(r.choice([3, 5, 6]))])
        return p.boolop(capi.E_ISNULL if r.random() < 0.5 else capi.E_ISNOTNULL, arg)


@pytest.mark.parametrize("seed", list(range(24)))
def test_random_plan(eng, relation, seed):
    desc, pages = relation
    rng = np.random.default_rng(1000 + seed)
    p = ExprPool()
    g = Gen(rng, p)
    qual = g.boolean(2) if rng.random() < 0.8 else -1
    aggs = [(capi.AGG_COUNT_STAR, -1)]
    for _ in range(int(rng.integers(1, 5))):
        fn = int(rng.choice([capi.AGG_SUM_FLOAT8, capi.AGG_AVG_FLOAT8, capi.AGG_MIN_FLOAT8, capi.AGG_MAX_FLOAT8, capi.AGG_COUNT_ANY]))
        aggs.append((fn, g.f8(2)))
    if rng.random() < 0.5:
        aggs.append((int(rng.choice([capi.AGG_SUM_INT4, capi.AGG_MIN_INT4, capi.AGG_MAX_INT4])), p.var(int(rng.choice([2, 3])), capi.INT4OID)))
    keys = [[], [p.var(1, capi.INT4OID)], [p.var(1, capi.INT4OID), p.var(6, capi.BPCHAROID)]][int(rng.integers(0, 3))]
    stage = capi.AGGSTAGE_PARTIAL if rng.random() < 0.3 else capi.AGGSTAGE_NORMAL
    agg = capi.make_agg(stage, keys, aggs, num_groups=int(rng.choice([0, 20, 500])))      # 500: straight to the HBM group table
    scan = capi.make_scan(desc, qual)
    try:
        want, sc, ps, want_x = po.seqscan_agg(scan, agg, p.pool, pages, exact=True)
        oracle_error = None
    except Exception as e:                                        # noqa: BLE001 - the oracle's ERROR is the expectation
        oracle_error = e
    for variant in ("interp-tr", None):          # the interpreter on the transposed kernel; whatever the library picks by itself
        if oracle_error is not None:
            with pytest.raises(capi.GGError) as e:
                gpu_scanagg(eng, scan, agg, p.pool, pages, variant)
            assert e.value.code in ARITH_ERRORS, (str(oracle_error), e.value.code)
        else:
            got, gsc, gps, _ = gpu_scanagg(eng, scan, agg, p.pool, pages, variant)
            assert (gsc, gps) == (sc, ps)
            assert_aggrows_match(got, want, agg, exact=want_x)
