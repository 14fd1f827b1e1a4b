"""An Agg's HAVING without a GPU: the row filter's program (ggp_compile_filter), its refusals, the per-row step of the device
(gg_device.cuh datumrow_passes, compiled for the host as tests/test_device_emu.py does) held to the oracle's qual evaluation over
rows with NULLs, -0, +-inf and NaN, and the executor over the oracle-backed stand-in library, which has no row filter."""
import ctypes as C
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from greengage_b200 import capi
from greengage_b200.capi import ExprPool
from oracle import pyoracle as po

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
EF_CODES = ((0x01, -2), (0x02, -3), (0x04, -4), (0x200, -5), (0x80, -11))      # GGP_EF_* -> GG_ERR_* (gg_errflags_to_code's order)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("rfemu") / "librfemu.so")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-ffp-contract=off", "-DGG_HOST_EMU", "-I", os.path.join(HERE, "emu"),
                           "-shared", "-o", so, os.path.join(HERE, "emu", "rowfilter_emu.cpp"),
                           os.path.join(ROOT, "greengage_b200", "csrc", "gg_compile.cpp")])
    L = C.CDLL(so)
    L.emu_filter_compile.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_char_p, C.c_int, C.c_char_p, C.c_int]
    L.emu_filter_run.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.POINTER(C.c_uint32),
                                 C.c_char_p, C.c_int]
    return L


def compile_filter(L, desc, qual, pool):
    listing, err = C.create_string_buffer(8192), C.create_string_buffer(256)
    rc = L.emu_filter_compile(C.byref(desc), qual, C.byref(pool), listing, 8192, err, 256)
    return rc, listing.value.decode(), err.value.decode()


def ops(listing):
    return [ln.split()[1] for ln in listing.splitlines()]


AGG_TYPES = [capi.INT4OID, capi.BPCHAROID, capi.INT8OID, capi.FLOAT8OID, capi.DATEOID]     # keys, count / sum, avg, min(date)


def test_program_shape(emu):
    desc = capi.rows_tupdesc(AGG_TYPES)
    p = ExprPool()
    k, s, cnt, avg, dmin = (p.var(i + 1, t) for i, t in enumerate(AGG_TYPES))
    over_key = p.func(capi.F_INT4EQ, capi.BOOLOID, k, p.const(capi.INT4OID, 3))
    over_agg = p.func(capi.F_INT8GT, capi.BOOLOID, cnt, p.const(capi.INT8OID, 2))
    # a top-level AND is an implicit-AND list: one FILTER per clause
    both = p.boolop(capi.E_AND, over_key, p.boolop(capi.E_OR, over_agg, p.boolop(capi.E_NOT, p.boolop(capi.E_ISNULL, avg))))
    rc, lst, _ = compile_filter(emu, desc, over_key, p.pool)
    assert rc == 0 and lst.count("FILTER") == 1 and ops(lst)[-1] == "END" and "off=0" in lst       # the first key: at the row's word 1
    rc, lst, _ = compile_filter(emu, desc, over_agg, p.pool)
    assert rc == 0 and lst.count("FILTER") == 1 and "off=16" in lst            # column 3 of the row: word 1 + 2, offset 16 past the mask
    rc, lst, _ = compile_filter(emu, desc, both, p.pool)
    o = ops(lst)
    assert rc == 0 and lst.count("FILTER") == 2 and "GUARD_OR" in o and "UNGUARD" in o and "ISNULL" in o and "NOT" in o and o[-1] == "END"
    # string and date comparisons, float8 arithmetic over an aggregate
    q = p.boolop(capi.E_AND, p.func(capi.F_BPCHAREQ, capi.BOOLOID, s, p.const(capi.BPCHAROID, "AB")),
                 p.func(capi.F_FLOAT8GT, capi.BOOLOID, p.func(capi.F_FLOAT8MUL, capi.FLOAT8OID, avg, p.const(capi.FLOAT8OID, 2.0)),
                        p.const(capi.FLOAT8OID, 1.0)))
    rc, lst, _ = compile_filter(emu, desc, q, p.pool)
    assert rc == 0 and "CMPS_K" in ops(lst) and "MUL_K" in ops(lst) and lst.count("FILTER") == 2


def test_refusals(emu):
    desc = capi.rows_tupdesc(AGG_TYPES)
    p = ExprPool()
    unknown = p.func(9999, capi.BOOLOID, p.var(1, capi.INT4OID), p.const(capi.INT4OID, 1))
    rc, _, msg = compile_filter(emu, desc, unknown, p.pool)
    assert rc == -6 and "9999" in msg
    rc, _, msg = compile_filter(emu, desc, p.func(capi.F_INT4EQ, capi.BOOLOID, p.var(6, capi.INT4OID), p.const(capi.INT4OID, 1)), p.pool)
    assert rc == -10 and "out of range" in msg
    rc, _, msg = compile_filter(emu, desc, p.pool.nnodes + 5, p.pool)
    assert rc == -10 and "not in the pool" in msg
    rc, _, msg = compile_filter(emu, desc, -1, p.pool)
    assert rc == -10
    nd = capi.rows_tupdesc([capi.INT4OID, capi.NUMERICOID])
    q = p.func(capi.F_NUMERIC_GT, capi.BOOLOID, p.var(2, capi.NUMERICOID), p.const(capi.NUMERICOID, "1.5"))
    rc, _, msg = compile_filter(emu, nd, q, p.pool)
    assert rc == -6 and "numeric" in msg
    heap = capi.synth_tupdesc(capi.TAB_LINEITEM_NARROW)
    rc, _, msg = compile_filter(emu, heap, p.func(capi.F_INT4EQ, capi.BOOLOID, p.var(1, capi.INT4OID), p.const(capi.INT4OID, 1)), p.pool)
    assert rc == -10 and "datum rows" in msg


@pytest.mark.parametrize("seed", range(4))
def test_per_row_step_matches_the_oracle(emu, seed):
    sys.path.insert(0, HERE)
    from test_gpu_having import ABI_TYPES, abi_quals, abi_rows, oracle_passes, py_value
    from test_gpu_agg_rows import datum_words
    n = 2000
    vals, nulls = abi_rows(n, seed=100 + seed)
    words = np.ascontiguousarray(datum_words(vals, nulls))
    pyrows = [tuple(py_value(t, vals[r, c], nulls[r, c]) for c, t in enumerate(ABI_TYPES)) for r in range(n)]
    desc = capi.rows_tupdesc(ABI_TYPES)
    p = ExprPool()
    for name, q in abi_quals(p).items():
        pas = np.zeros(n, dtype=np.uint8)
        ef = C.c_uint32(0)
        err = C.create_string_buffer(256)
        assert emu.emu_filter_run(C.byref(desc), q, C.byref(p.pool), words.ctypes.data, n, pas.ctypes.data, C.byref(ef), err, 256) == 0
        try:
            want = oracle_passes(ABI_TYPES, pyrows, p, q)
            assert ef.value == 0, (name, hex(ef.value))
            assert pas.astype(bool).tolist() == want, name
        except po.OracleError as e:
            got = next((code for bit, code in EF_CODES if ef.value & bit), 0)
            assert got == e.code, (name, hex(ef.value), e.code)


# ---- the executor over the stand-in library (no gg_rowfilter_*): an Agg with a qual is refused at init, never run without it ----
NODE_SCRIPT = textwrap.dedent("""
    import ctypes as C, sys
    sys.path.insert(0, %(root)r); sys.path.insert(0, %(here)r)
    from greengage_b200 import capi, executor as ex
    from test_executor_multiseg import MockRel
    from test_executor_limit import _li_agg
    L = ex.bind(C.CDLL(%(mock)r))
    L.mock_engine.restype = C.c_void_p
    L.mock_relation.restype = C.c_void_p
    L.mock_relation.argtypes = [C.c_void_p, C.c_uint64]
    ex._lib = L
    eng = L.mock_engine()
    li, scan, agg, p = _li_agg()
    rel = MockRel(L, li)
    out = []
    def attempt(having, stage=None, var=1):
        a = capi.gg_agg.from_buffer_copy(bytes(agg))
        if stage is not None:
            a.aggstage = stage
        b = ex.PlanBuilder()
        q = -1 if having is None else p.func(capi.F_INT8GT, capi.BOOLOID, p.var(var, capi.INT8OID), p.const(capi.INT8OID, 0))
        try:
            x = ex.Executor(eng, p.pool, [rel], b.agg(b.seqscan(0, scan.desc, scan.qual), a, having=q))
        except ex.ExecError as e:
            return ("refused", e.code, str(e))
        n = len(x.rows()); x.end()
        return ("ran", n)
    print(repr([attempt(None), attempt(1), attempt(1, stage=capi.AGGSTAGE_PARTIAL), attempt(1, var=40)]))
""")


def test_executor_refuses_having_without_a_row_filter(tmp_path):
    sys.path.insert(0, HERE)
    from test_executor_multiseg import build_mock
    mock = build_mock(str(tmp_path))
    r = subprocess.run([sys.executable, "-c", NODE_SCRIPT % {"root": ROOT, "here": HERE, "mock": mock}], capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr
    plain, having, partial, badvar = eval(r.stdout.strip().splitlines()[-1])
    assert plain[0] == "ran" and plain[1] > 0                         # qual = -1: as before
    assert having[:2] == ("refused", -6) and "row filter" in having[2]
    assert partial[:2] == ("refused", -6) and "PARTIAL" in partial[2]
    assert badvar[:2] == ("refused", -6)         # refused before the qual is even compiled
