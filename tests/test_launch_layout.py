"""The launch configuration of every role of the scan kernel, on the CPU: tests/emu/launch_layout.cpp compiles the product's plan
compiler and its configuration rules (greengage_b200/csrc/gg_launch.h) with g++, and the configuration each plan gets — block
size, blocks per SM, ring stages, team, group capacity, register slots and shared-memory offsets — is pinned for an H100 (132
SMs, 232 448 bytes of opt-in shared memory per block).  A change to these numbers changes what the GPU runs: it wants a
measurement, not only a new expectation here."""
import ctypes as C
import os
import subprocess

import pytest

from _util import make_desc
from greengage_b200 import capi, tpch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OPTIN = 232448
FIELDS = ("threads", "ctas", "nstage", "team", "gcap", "regslots", "scratch_per_warp", "scratch_off", "cnt_off", "acc_off", "smem")
PRIV, TR, TRN, HASH = 0, 1, 2, 5


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("layout") / "liblayout.so")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emu", "launch_layout.cpp"),
                           os.path.join(ROOT, "greengage_b200", "csrc", "gg_compile.cpp")])
    return C.CDLL(so)


def out():
    return (C.c_int64 * len(FIELDS))()


def cfg(o):
    return dict(zip(FIELDS, list(o)))


def scanagg(lib, plan, mode, chunks, items, rule):
    scan, agg, pool = plan
    o = out()
    assert lib.layout_scanagg(C.byref(scan), C.byref(agg), C.byref(pool), mode, chunks, items, rule, C.c_int64(OPTIN), o) == 0
    return cfg(o)


def nullable_plan():
    """SELECT k, sum(x) GROUP BY k over (k int4 NOT NULL, x float8 NULL)"""
    p = capi.ExprPool()
    k, x = p.var(1, capi.INT4OID), p.var(2, capi.FLOAT8OID)
    desc = make_desc([(capi.INT4OID, 4, "i", 1, 1), (capi.FLOAT8OID, 8, "d", 1, 0)])
    return capi.make_scan(desc, -1), capi.make_agg(capi.AGGSTAGE_NORMAL, [k], [(capi.AGG_SUM_FLOAT8, x)]), p.pool


WIDE, NARROW = capi.TAB_LINEITEM_WIDE, capi.TAB_LINEITEM_NARROW
NORMAL, PARTIAL = capi.AGGSTAGE_NORMAL, capi.AGGSTAGE_PARTIAL

# (table, stage, variant, chunks of 32 line pointers per page, line pointers of the sampled page, gg_priv_regslots's value) ->
# the configuration.  Q1 on lineitem-wide (~190 rows per page): 3 teams of 7 on a 5-page ring (DESIGN §4.1); on lineitem-narrow
# (~430 rows per page): 20 warps on a 3-page ring, one-stage with everything in shared memory.  0 chunks: pages not sampled.
Q1_CASES = [
    ((WIDE, NORMAL, PRIV, 6, 190, 3),
     dict(threads=704, ctas=1, nstage=5, team=7, gcap=4, regslots=3, scratch_per_warp=448, scratch_off=165376, cnt_off=174784, acc_off=185536, smem=228544)),
    ((WIDE, PARTIAL, PRIV, 6, 190, 3),
     dict(threads=704, ctas=1, nstage=3, team=7, gcap=4, regslots=3, scratch_per_warp=448, scratch_off=99808, cnt_off=109216, acc_off=119968, smem=227488)),
    ((NARROW, NORMAL, PRIV, 14, 430, 3),
     dict(threads=672, ctas=1, nstage=3, team=0, gcap=4, regslots=0, scratch_per_warp=448, scratch_off=99808, cnt_off=108768, acc_off=119008, smem=221408)),
    ((NARROW, PARTIAL, PRIV, 14, 430, 3),
     dict(threads=672, ctas=1, nstage=3, team=0, gcap=4, regslots=3, scratch_per_warp=448, scratch_off=99808, cnt_off=108768, acc_off=119008, smem=221408)),
    ((WIDE, NORMAL, PRIV, 0, 0, 3),
     dict(threads=672, ctas=1, nstage=5, team=0, gcap=4, regslots=3, scratch_per_warp=448, scratch_off=165376, cnt_off=174336, acc_off=184576, smem=225536)),
    ((WIDE, NORMAL, TR, 6, 190, 0),
     dict(threads=256, ctas=2, nstage=3, team=0, gcap=25, regslots=0, scratch_per_warp=2032, scratch_off=99808, cnt_off=0, acc_off=0, smem=114032)),
    ((WIDE, NORMAL, HASH, 6, 190, 0),
     dict(threads=256, ctas=2, nstage=3, team=0, gcap=25, regslots=0, scratch_per_warp=448, scratch_off=99808, cnt_off=0, acc_off=0, smem=102944)),
]


@pytest.mark.parametrize("case,want", Q1_CASES, ids=["-".join(map(str, c)) for c, _ in Q1_CASES])
def test_q1_launch_configuration(lib, case, want):
    table, stage, mode, chunks, items, rule = case
    assert scanagg(lib, tpch.q1_plan(table, stage), mode, chunks, items, rule) == want


def test_nullable_plan_launch_configuration(lib):
    assert scanagg(lib, nullable_plan(), TRN, 1, 20, 0) == dict(
        threads=256, ctas=2, nstage=3, team=0, gcap=32, regslots=0, scratch_per_warp=656, scratch_off=99808, cnt_off=0, acc_off=0,
        smem=104400)


@pytest.mark.parametrize("mode,want", [
    (TR, dict(threads=256, ctas=2, nstage=3, team=0, gcap=32, regslots=0, scratch_per_warp=1040, scratch_off=99808, cnt_off=0, acc_off=0, smem=107088)),
    (HASH, dict(threads=256, ctas=2, nstage=3, team=0, gcap=32, regslots=0, scratch_per_warp=256, scratch_off=99808, cnt_off=0, acc_off=0, smem=101600)),
])
def test_join_probe_and_build_launch_configuration(lib, mode, want):
    outer, inner, hj, agg, pool = tpch.join_plan(NARROW, "q3ish", capi.JOIN_INNER)
    probe, build = out(), out()
    assert lib.layout_join(C.byref(outer), C.byref(inner), C.byref(hj), C.byref(agg), C.byref(pool), mode, 14, C.c_int64(OPTIN), probe, build) == 0
    assert cfg(probe) == want
    assert cfg(build) == dict(threads=256, ctas=2, nstage=2, team=0, gcap=0, regslots=0, scratch_per_warp=208, scratch_off=67024, cnt_off=0,
                              acc_off=0, smem=68480)


def test_motion_send_launch_configuration(lib):
    p = capi.ExprPool()
    key = p.var(1, capi.INT8OID)
    scan = capi.make_scan(capi.synth_tupdesc(NARROW), -1)
    keys = (C.c_int32 * 1)(key)
    o = out()
    assert lib.layout_motion(C.byref(scan), C.byref(p.pool), keys, 1, keys, 1, o) == 0
    assert cfg(o) == dict(threads=256, ctas=2, nstage=2, team=0, gcap=0, regslots=0, scratch_per_warp=592, scratch_off=67024, cnt_off=0,
                          acc_off=0, smem=71168)
