"""The finalisation rule shared by the host's finalize_rows and the device's datum-row writer (greengage_b200/csrc/gg_aggfinal.h),
compiled by gcc and run over the group records the device interpreter produces (tests/emu/device_emu.cpp) for the random plans
of test_device_emu.py and the float8 edge relation: every aggregate's word and NULL flag equal the oracle's finalised rows bit
for bit — groups whose inputs are all NULL, -0 sums and +-inf / NaN inputs included."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from _util import edge_plan, edge_relation, f2b
from greengage_b200 import capi
from oracle import pyoracle as po
from test_device_emu import emu, random_plan, relation, run_emu  # noqa: F401  (fixtures)

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def rule(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("aggfinal") / "libaggfinal.so")
    subprocess.check_call(["gcc", "-std=c11", "-O2", "-Wall", "-Wextra", "-Werror", "-ffp-contract=off", "-fPIC", "-shared", "-o", so,
                           os.path.join(HERE, "aggfinal_harness.c")])
    L = C.CDLL(so)
    L.harness_aggfinal.argtypes = [C.c_int32, C.c_uint64, C.c_uint64, C.c_uint64, C.POINTER(C.c_int)]
    L.harness_aggfinal.restype = C.c_uint64
    L.harness_covers.argtypes = L.harness_is_float8.argtypes = [C.c_int32]
    return L


def u64(x):
    return int(np.float64(x).view(np.uint64))


def check_groups(L, groups, aggcol, want, agg, exact):
    """every aggregate of every group through the rule, against the oracle's finalised row; returns the values checked"""
    by = {}
    for g in groups:
        by[tuple((None if (g.keynull >> c) & 1 else int(np.uint64(g.key[c]).astype(np.int64))) for c in range(agg.numCols))] = g
    assert len(by) == len(want)
    checked = 0
    for ri, r in enumerate(want):
        g = by[tuple(None if r.keyisnull[c] else r.key[c] for c in range(agg.numCols))]
        for i in range(agg.numAggs):
            fn, col, v = agg.aggs[i].aggfnoid, aggcol[i], r.agg[i]
            assert L.harness_covers(fn)
            isnull = C.c_int(0)
            w = L.harness_aggfinal(fn, g.count, g.n[col] if col >= 0 else 0, u64(g.sum[col]) if col >= 0 else 0, C.byref(isnull))
            assert bool(isnull.value) == bool(v.isnull), (fn, isnull.value, v.isnull)
            checked += 1
            if v.isnull:
                assert w == 0
            elif L.harness_is_float8(fn):
                got = float(np.uint64(w).view(np.float64))
                # float8larger/smaller keep the later argument of a tie, the device's fold the first: with zeros of both signs in
                # a group the sign of a zero extreme is the scan order's (test_device_emu.check has the same exception)
                both_zeros = got == 0 and fn in (capi.AGG_MIN_FLOAT8, capi.AGG_MAX_FLOAT8) and \
                    exact[ri][i].flags & po.XF_POSZERO and exact[ri][i].flags & po.XF_NEGZERO
                if not both_zeros:
                    assert f2b(got) == f2b(v.f[0]) or (got != got and v.f[0] != v.f[0]), (fn, got, v.f[0])
            else:
                assert np.uint64(w).astype(np.int64) == v.i, (fn, w, v.i)
    return checked


def test_rule_over_the_float8_edge_relation(rule, emu):  # noqa: F811
    for nullable in (True, False):
        desc, pages, n = edge_relation(nullable)
        scan, agg, pool = edge_plan(desc, capi.AGGSTAGE_NORMAL)
        want, sc, ps, exact = po.seqscan_agg(scan, agg, pool, pages, exact=True)
        groups, aggcol, gsc, gps, err = run_emu(emu, scan, agg, pool, pages)
        assert err & ~0x800 == 0
        assert check_groups(rule, groups, aggcol, want, agg, exact) > 0


def test_rule_over_random_plans(rule, emu, relation):  # noqa: F811
    desc, pages = relation
    checked = plans = 0
    for seed in range(300):
        scan, agg, p = random_plan(desc, seed)
        if agg.aggstage != capi.AGGSTAGE_NORMAL:
            continue
        try:
            want, sc, ps, exact = po.seqscan_agg(scan, agg, p.pool, pages, exact=True)
        except po.OracleError:
            continue
        groups, aggcol, gsc, gps, err = run_emu(emu, scan, agg, p.pool, pages)
        if err & ~0x800:
            continue
        checked += check_groups(rule, groups, aggcol, want, agg, exact)
        plans += 1
    assert plans > 150 and checked > 1000, (plans, checked)
