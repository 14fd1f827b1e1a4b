"""The bounded Sort on the device (gg_sort_datumrows_bounded / gg_sort_rows_bounded: radix select on the first key's prefix,
then the radix sort of the survivors) and the Limit node above it.  The contract is exact: the bounded result is byte for byte
the first min(bound, live) rows of the unbounded sort, ties included, so every check here compares bytes or row numbers."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from greengage_b200 import capi  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from greengage_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def datum_rows(cols, nulls=None, dead=None):
    """GG_FMT_DATUMROWS words: NULL mask (bit 63: a dead slot), then the columns"""
    n = len(cols[0])
    mask = np.zeros(n, dtype=np.int64)
    if nulls is not None:
        for c in range(nulls.shape[1]):
            mask |= nulls[:, c].astype(np.int64) << c
    if dead is not None:
        mask[dead] = np.int64(-2 ** 63)
    return np.stack([mask] + [np.asarray(c, dtype=np.int64) for c in cols], axis=1)


class Sorter:
    """one device copy of the rows; full() and bounded() return the output rows as int64 words"""

    def __init__(self, eng, words):
        from greengage_b200.engine import Relation
        self.eng, self.n, self.W = eng, words.shape[0], words.shape[1]
        nbytes = words.nbytes
        self.nbl = (nbytes + 64 + capi.GG_BLCKSZ - 1) // capi.GG_BLCKSZ
        host = np.zeros(self.nbl * capi.GG_BLCKSZ, dtype=np.uint8)
        host[:nbytes] = words.view(np.uint8).reshape(-1)
        self.src, self.dst = Relation(eng, host_pages=host), Relation(eng, nblocks=self.nbl)

    def _out(self, cnt):
        nb = (cnt * self.W * 8 + capi.GG_BLCKSZ - 1) // capi.GG_BLCKSZ
        if nb == 0:
            return np.zeros((0, self.W), dtype=np.int64)
        return self.dst.read(0, nb).view(np.int64)[:cnt * self.W].reshape(-1, self.W).copy()

    def full(self, keys):
        ka = (capi.gg_sortkey * len(keys))(*keys)
        cnt, passes = C.c_uint64(0), C.c_int(0)
        capi.check(capi.dev_lib().gg_sort_datumrows(self.eng.h, ka, len(keys), self.W - 1, C.c_void_p(self.src.device_ptr()), self.n,
                                                    C.c_void_p(self.dst.device_ptr()), C.byref(cnt), C.byref(passes)))
        return self._out(cnt.value)

    def bounded(self, keys, bound):
        ka = (capi.gg_sortkey * len(keys))(*keys)
        cnt, passes = C.c_uint64(12345), C.c_int(0)
        capi.check(capi.dev_lib().gg_sort_datumrows_bounded(self.eng.h, ka, len(keys), self.W - 1, C.c_void_p(self.src.device_ptr()), self.n,
                                                            bound, C.c_void_p(self.dst.device_ptr()), C.byref(cnt), C.byref(passes)))
        return self._out(cnt.value)

    def check(self, keys, bounds):
        full = self.full(keys)
        live = full.shape[0]
        for b in bounds(live) if callable(bounds) else bounds:
            got = self.bounded(keys, b)
            assert got.shape[0] == min(b, live), (b, live, got.shape)
            assert got.tobytes() == full[:got.shape[0]].tobytes(), (b, live)
        return full

    def free(self):
        self.src.free()
        self.dst.free()


def _bounds(live):
    return sorted({0, 1, 7, 1000, max(live - 1, 0), live, live + 5})


@pytest.mark.parametrize("name", ["int4", "int8", "date", "timestamp", "bool", "float8", "bpchar", "text"])
def test_bounded_datumrows_are_the_prefix_of_the_full_sort_for_every_type(eng, name):
    """20 000 rows of the type's edge values (float8: NaN, +-0, +-inf), 5 % NULLs and 10 % dead slots between the rows;
    ASC / DESC x NULLS FIRST / LAST; bounds 0, 1, 7, 1000, live - 1, live, > live"""
    from test_gpu_keys import TYPID, datums
    rng = np.random.default_rng(len(name) * 7)
    n = 20_000
    k = datums(name, n, rng)
    nulls = np.zeros((n, 2), dtype=np.uint8)
    nulls[:, 0] = rng.random(n) < 0.05
    s = Sorter(eng, datum_rows([k, np.arange(n)], nulls, rng.random(n) < 0.1))
    try:
        for desc in (False, True):
            for nf in (False, True):
                full = s.check([capi.make_sortkey(0, TYPID[name], desc, nf)], _bounds)
                assert np.all(full[:, 0] >= 0)                                  # no dead slot comes out
    finally:
        s.free()


def test_heavy_ties_in_the_first_key_are_decided_by_the_later_keys(eng):
    """a first key of three values (so every row survives the selection's first digits) under 1-4 keys of mixed types; the
    ties of the last key keep input order in both results"""
    from test_gpu_keys import datums
    rng = np.random.default_rng(11)
    n = 200_000
    cols = [rng.integers(0, 3, n), datums("float8", n, rng), datums("text", n, rng), rng.integers(-50, 50, n), np.arange(n)]
    nulls = (rng.random((n, 5)) < 0.02).astype(np.uint8)
    nulls[:, 4] = 0
    s = Sorter(eng, datum_rows(cols, nulls, rng.random(n) < 0.01))
    keys = [capi.make_sortkey(0, capi.INT4OID, True), capi.make_sortkey(1, capi.FLOAT8OID, False, True),
            capi.make_sortkey(2, capi.TEXTOID, True, False), capi.make_sortkey(3, capi.INT8OID)]
    try:
        for nk in (1, 2, 3, 4):
            s.check(keys[:nk], lambda live: [1, 7, 1000, live // 5, live // 3, live // 2, live - 1, live])
    finally:
        s.free()


@pytest.mark.parametrize("n", [1, 2, 4095, 4097, 10_000_000])
def test_bounded_datumrows_at_every_size(eng, n):
    """n from one row to 10^7 (an int8 key over the whole range, then a float8 key), no dead slots"""
    rng = np.random.default_rng(n)
    k8 = rng.integers(-2 ** 63, 2 ** 63 - 1, n, dtype=np.int64)
    f8 = rng.standard_normal(n).view(np.int64)
    s = Sorter(eng, datum_rows([k8, f8]))
    try:
        bounds = _bounds if n < 10 ** 6 else (lambda live: [1, 1000, live // 5, live // 2, live - 1])
        s.check([capi.make_sortkey(0, capi.INT8OID)], bounds)
        s.check([capi.make_sortkey(1, capi.FLOAT8OID, True), capi.make_sortkey(0, capi.INT8OID)], bounds)
    finally:
        s.free()


def test_bounded_host_rows_give_the_prefix_of_the_permutation(eng):
    from greengage_b200.engine import sort_rows
    rng = np.random.default_rng(5)
    n = 100_000
    rows = np.stack([rng.integers(0, 50, n), rng.standard_normal(n).view(np.int64), np.arange(n)], axis=1).astype(np.int64)
    nulls = (rng.random(rows.shape) < 0.05).astype(np.uint8)
    keys = [capi.make_sortkey(0, capi.INT8OID, True, False), capi.make_sortkey(1, capi.FLOAT8OID)]
    whole = sort_rows(eng, keys, rows, nulls)
    ka = (capi.gg_sortkey * len(keys))(*keys)
    for bound in (0, 1, 7, 1000, n // 2, n - 1, n, n + 3):
        perm, cnt = np.zeros(n, dtype=np.uint64), C.c_uint64(0)
        capi.check(capi.dev_lib().gg_sort_rows_bounded(eng.h, ka, len(keys), 3, rows.ctypes.data, nulls.ctypes.data, n, bound,
                                                       perm.ctypes.data, C.byref(cnt)))
        assert cnt.value == min(bound, n) and np.array_equal(perm[:cnt.value], whole[:cnt.value]), bound


# ---- the Limit node over device rows ----

def _onek_plan(eng, quals, desc, count, offset):
    from _util import onek_fixture
    from greengage_b200 import executor as ex
    from greengage_b200.engine import Relation
    d, pages, exp = onek_fixture()
    u1, u2 = exp["columns"].index("unique1") + 1, exp["columns"].index("unique2") + 1
    p = capi.ExprPool()
    fn = {">": capi.F_INT4GT, "<": capi.F_INT4LT}
    qual = -1
    for op, v in quals:
        q = p.func(fn[op], capi.BOOLOID, p.var(u1, capi.INT4OID), p.const(capi.INT4OID, v))
        qual = q if qual < 0 else p.boolop(capi.E_AND, qual, q)
    b = ex.PlanBuilder()
    scan = b.seqscan(0, d, qual, [p.var(u1, capi.INT4OID), p.var(u2, capi.INT4OID)])
    lim = b.limit(b.sort(scan, [capi.make_sortkey(0, capi.INT4OID, desc)]), count, offset)
    rel = Relation(eng, host_pages=pages)
    return ex.Executor(eng, p.pool, [rel], lim), lim, rel


def test_reference_limit_goldens(eng):
    """the nine onek queries of sql/limit.sql as Limit <- Sort <- SeqScan(qual, targets unique1, unique2): expected/limit.out"""
    from _util import golden
    for q in golden("limit_expected.json")["queries"]:
        x, lim, rel = _onek_plan(eng, q["quals"], q["desc"], q["limit"], q["offset"])
        try:
            assert [r[0][:2] for r in x.rows()] == q["rows"], q
            assert x.locations()[:2] == [("limit", "host"), ("sort", "device-rows")]
        finally:
            x.end()
            rel.free()


def test_variable_limit_through_rescan(eng):
    """limit.sql:112 (LIMIT 1 OFFSET s - 1 with s from an outer query): every ReScan recomputes the limits and the bound, and
    returns the s-th row of the whole sort"""
    x, lim, rel = _onek_plan(eng, [], False, 1, 0)
    try:
        for s in list(range(1, 11)) + [500, 1000, 1001]:
            lim.limitOffset = s - 1
            x.rescan()
            assert [r[0][0] for r in x.rows()] == ([s - 1] if s <= 1000 else [])
    finally:
        x.end()
        rel.free()


def test_preliminary_limit_plan_on_one_gpu(eng):
    """Limit <- Gather Motion(merge) <- Limit <- Sort <- SeqScan with targets on one segment (loopback), and a Limit straight
    over the rows node: a window of the scan's rows, copied from the device without the rest of the buffer"""
    from _util import onek_fixture
    from greengage_b200 import executor as ex
    from greengage_b200.engine import Relation
    d, pages, exp = onek_fixture()
    u1, u2 = exp["columns"].index("unique1") + 1, exp["columns"].index("unique2") + 1
    p = capi.ExprPool()
    keys = [capi.make_sortkey(1, capi.INT4OID, True)]
    rel = Relation(eng, host_pages=pages)
    try:
        def run(build):
            b = ex.PlanBuilder()
            x = ex.Executor(eng, p.pool, [rel], build(b, b.seqscan(0, d, -1, [p.var(u1, capi.INT4OID), p.var(u2, capi.INT4OID)])))
            rows = [tuple(r[0][:2]) for r in x.rows()]
            x.end()
            return rows
        full = run(lambda b, s: b.sort(s, keys))
        plain = run(lambda b, s: s)
        assert len(full) == len(plain) == 1000
        got = run(lambda b, s: b.limit(b.motion(b.limit(b.sort(s, keys), 15), ex.MOTION_GATHER, [], 1, merge_keys=keys), 10, 5))
        assert got == full[5:15]
        # without ORDER BY any rows are the answer (the scan hands rows out in the order its warps claim them): the count, and
        # distinct rows of the relation
        for count, offset in ((30, 970), (3, 2), (50, 990)):
            got = run(lambda b, s: b.limit(s, count, offset))
            assert len(got) == min(count, 1000 - offset) and len(set(got)) == len(got) and set(got) <= set(plain)
    finally:
        rel.free()
