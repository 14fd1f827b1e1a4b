"""Differential test of the plan compiler + the device interpreter on the CPU: tests/emu/device_emu.cpp compiles
greengage_b200/csrc/gg_device.cuh for the host (-DGG_HOST_EMU: shared memory becomes a byte array, nothing else changes) and
runs walk_tuple + run_prog tuple by tuple over heap pages for plans built by the same random generator the GPU tests use;
the groups must equal the oracle's.  Sequential on both sides, so float8 sums are compared bit for bit.  Covers what a
program MEANS (operand decoding, NULL tracking, three-valued logic, comparisons, casts, key normalisation, error flags);
the parallel machinery around it is the GPU tests' job."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from _util import edge_plan, edge_relation, f2b, make_desc
from greengage_b200 import capi, tpch
from greengage_b200.capi import ExprPool
from oracle import pyoracle as po
import test_gpu_random_plans as rp

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
ARITH = 0x01 | 0x02 | 0x04 | 0x80 | 0x200            # GGP_EF_FLOAT_OVERFLOW | UNDERFLOW | DIV_ZERO | DATE_RANGE | INT_OVERFLOW


class EmuGroup(C.Structure):
    _fields_ = [("key", C.c_uint64 * capi.GG_MAX_KEYS), ("keynull", C.c_uint32), ("pad", C.c_uint32), ("count", C.c_uint64),
                ("sum", C.c_double * 16), ("sumsq", C.c_double * 16), ("n", C.c_uint64 * 16)]


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emu") / "libemu.so")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-ffp-contract=off", "-I", os.path.join(HERE, "emu"), "-shared", "-o", so,
                           os.path.join(HERE, "emu", "device_emu.cpp"), os.path.join(ROOT, "greengage_b200", "csrc", "gg_compile.cpp")])
    L = C.CDLL(so)
    L.emu_scanagg.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_int, C.POINTER(C.c_int),
                              C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), C.c_char_p, C.c_int]
    return L


@pytest.fixture(scope="module")
def relation():
    rng = np.random.default_rng(77)
    desc = make_desc([(capi.INT4OID, 4, "i", 1, 1), (capi.INT4OID, 4, "i", 1, 1), (capi.INT4OID, 4, "i", 1, 0), (capi.FLOAT8OID, 8, "d", 1, 1),
                      (capi.FLOAT8OID, 8, "d", 1, 0), (capi.BPCHAROID, -1, "i", 0, 0), (capi.DATEOID, 4, "i", 1, 1), (capi.INT8OID, 8, "d", 1, 1)])
    rows, nulls = [], []
    for _ in range(4000):
        rows.append([int(rng.integers(0, 5)), int(rng.integers(-20, 20)), int(rng.integers(-5, 5)), float(rng.integers(-40, 40)) / 4,
                     float(rng.choice([0.0, -0.0, 0.5, -1.25, 3.0, 1e-3, float(rng.integers(-9, 9))])), bytes([65 + int(rng.integers(0, 3))]) + b" ",
                     int(rng.integers(-400, 400)), int(rng.integers(-10**9, 10**9))])
        nulls.append([False, False, rng.random() < 0.15, False, rng.random() < 0.15, rng.random() < 0.1, False, False])
    return desc, po.build_pages(desc, rows, nulls)


def run_emu(L, scan, agg, pool, pages, cap=4096, nrows=None):
    """pages: heap pages (uint8), or with nrows the datum rows (uint64 [nrows, 1 + ncols]) of a GG_FMT_DATUMROWS descriptor"""
    out = (EmuGroup * cap)()
    n, sc, ps, err = C.c_int(0), C.c_uint64(0), C.c_uint64(0), C.c_uint32(0)
    aggcol, accsq = (C.c_int32 * capi.GG_MAX_AGGS)(), (C.c_int32 * 16)()
    msg = C.create_string_buffer(256)
    rc = L.emu_scanagg(C.byref(scan), C.byref(agg), C.byref(pool), pages.ctypes.data, pages.size // capi.GG_BLCKSZ if nrows is None else nrows, out, cap, C.byref(n),
                       aggcol, accsq, C.byref(sc), C.byref(ps), C.byref(err), msg, 256)
    assert rc == 0, (rc, msg.value)
    return [out[i] for i in range(n.value)], list(aggcol), sc.value, ps.value, err.value


def check(groups, aggcol, want, agg, exact=None):
    """exact: the oracle's exact records aligned with `want` (po.seqscan_agg(..., exact=True)), for the one float result
    that may differ from the oracle's: a zero min/max of a group with zeros of both signs"""
    by = {}
    for g in groups:
        by[tuple((None if (g.keynull >> c) & 1 else int(np.uint64(g.key[c]).astype(np.int64))) for c in range(agg.numCols))] = g
    assert len(by) == len(want)
    partial = agg.aggstage == capi.AGGSTAGE_PARTIAL
    for ri, r in enumerate(want):
        g = by[tuple(None if r.keyisnull[c] else r.key[c] for c in range(agg.numCols))]
        for i in range(agg.numAggs):
            fn, col, v = agg.aggs[i].aggfnoid, aggcol[i], r.agg[i]
            if col < 0:
                assert v.i == g.count
                continue
            nn, s = g.n[col], g.sum[col]
            ibits = int(np.float64(s).view(np.int64))
            # float results by their bits, so that the sign of a zero counts; the avg and its PARTIAL state are finalised as
            # the product's host finalisation does (gg_scanagg.cu finalize_rows: float8_accum's "{0,0,0}" start is + 0.0)
            same = lambda x, y: f2b(x) == f2b(y) or (x != x and y != y)
            if fn == capi.AGG_COUNT_ANY:
                assert v.i == nn
            elif fn == capi.AGG_AVG_FLOAT8:
                if partial:
                    assert v.f[0] == float(nn) and same(v.f[1], s + 0.0) and same(v.f[2], g.sumsq[col] + 0.0), (v.f[1], s, v.f[2], g.sumsq[col])
                elif nn == 0:
                    assert v.isnull
                else:
                    assert same(v.f[0], (s + 0.0) / nn), (v.f[0], s, nn)
            elif fn in (capi.AGG_SUM_FLOAT8, capi.AGG_MIN_FLOAT8, capi.AGG_MAX_FLOAT8):
                assert bool(v.isnull) == (nn == 0)
                # float8larger/smaller keep the later argument of a tie, the device's fold the first: with zeros of both
                # signs in a group the sign of a zero extreme is the scan order's, not the result's
                both_zeros = exact is not None and v.f[0] == 0 and s == 0 and fn != capi.AGG_SUM_FLOAT8 and \
                    exact[ri][i].flags & po.XF_POSZERO and exact[ri][i].flags & po.XF_NEGZERO
                if nn and not both_zeros:
                    assert same(v.f[0], s), (fn, v.f[0], s)
            else:
                assert bool(v.isnull) == (nn == 0)
                if nn:
                    assert v.i == ibits, (fn, v.i, ibits)


def test_edge_relation_through_the_device_interpreter(emu):
    """the float8 edges (all -0, mixed zeros, infinities, NaN, cancellation, NULLs, groups of 1/31/32/33) at NORMAL and
    PARTIAL stage: sequential on both sides, so every float result equals the oracle's bit for bit, the sign of zero
    included (sum over all -0 is -0, as float8pl's first input taken as it is)"""
    for (desc, pages, n), stage in [(edge_relation(nullable), stage) for nullable in (True, False)
                                    for stage in (capi.AGGSTAGE_NORMAL, capi.AGGSTAGE_PARTIAL)]:
        scan, agg, pool = edge_plan(desc, stage)
        want, sc, ps, exact = po.seqscan_agg(scan, agg, pool, pages, exact=True)
        groups, aggcol, gsc, gps, err = run_emu(emu, scan, agg, pool, pages)
        assert err == 0 and (gsc, gps) == (sc, ps) == (n, n), (hex(err), gsc, gps, sc, ps)
        check(groups, aggcol, want, agg, exact)


def random_plan(desc, seed, depth=2):
    rng = np.random.default_rng(1000 + seed)
    p = ExprPool()
    g = rp.Gen(rng, p)
    qual = g.boolean(depth) if rng.random() < 0.8 else -1
    aggs = [(capi.AGG_COUNT_STAR, -1)]
    for _ in range(int(rng.integers(1, 5))):
        fn = int(rng.choice([capi.AGG_SUM_FLOAT8, capi.AGG_AVG_FLOAT8, capi.AGG_MIN_FLOAT8, capi.AGG_MAX_FLOAT8, capi.AGG_COUNT_ANY]))
        aggs.append((fn, g.f8(depth)))
    if rng.random() < 0.5:
        aggs.append((int(rng.choice([capi.AGG_SUM_INT4, capi.AGG_MIN_INT4, capi.AGG_MAX_INT4])), p.var(int(rng.choice([2, 3])), capi.INT4OID)))
    keys = [[], [p.var(1, capi.INT4OID)], [p.var(1, capi.INT4OID), p.var(6, capi.BPCHAROID)]][int(rng.integers(0, 3))]
    stage = capi.AGGSTAGE_PARTIAL if rng.random() < 0.3 else capi.AGGSTAGE_NORMAL
    return capi.make_scan(desc, qual), capi.make_agg(stage, keys, aggs, num_groups=int(rng.choice([0, 20, 500]))), p


def differential(emu, relation, seeds, stats):
    desc, pages = relation
    for seed in seeds:
        scan, agg, p = random_plan(desc, seed)
        try:
            want, sc, ps, exact = po.seqscan_agg(scan, agg, p.pool, pages, exact=True)
            oracle_error = None
        except po.OracleError as e:
            oracle_error = e
        groups, aggcol, gsc, gps, err = run_emu(emu, scan, agg, p.pool, pages)
        if oracle_error is not None:
            assert err & ARITH, (seed, str(oracle_error), hex(err))
            stats["errors"] += 1
        else:
            # an arm ExecEvalAnd / ExecEvalOr would have skipped must not raise on the device either (GGP_GUARD_*)
            assert not (err & ARITH), (seed, hex(err))
            assert err == 0 or not (err & ~0x800), (seed, hex(err))
            assert (gsc, gps) == (sc, ps), seed
            check(groups, aggcol, want, agg, exact)
            stats["equal"] += 1


def test_random_plans_mean_what_the_oracle_computes(emu, relation):
    stats = {"equal": 0, "errors": 0}
    differential(emu, relation, range(300), stats)
    assert stats["equal"] > 200 and stats["errors"] > 0, stats


def test_partial_stage_for_a_device_final_keeps_everything_but_sumsq(emu, relation):
    """GG_AGGF_DEVICE_FINAL: a PARTIAL stage without sumX2 against the same oracle answers"""
    desc, pages = relation
    for seed in range(60):
        scan, agg, p = random_plan(desc, seed)
        if agg.aggstage != capi.AGGSTAGE_PARTIAL:
            continue
        agg.flags = capi.AGGF_DEVICE_FINAL
        try:
            want, sc, ps, exact = po.seqscan_agg(scan, agg, p.pool, pages, exact=True)
        except po.OracleError:
            continue
        groups, aggcol, gsc, gps, err = run_emu(emu, scan, agg, p.pool, pages)
        if err & ARITH:
            continue
        for g in groups:
            assert not any(g.sumsq[j] for j in range(16))
        for r in want:                                   # everything but sumX2 is unchanged
            for i in range(agg.numAggs):
                if agg.aggs[i].aggfnoid == capi.AGG_AVG_FLOAT8:
                    r.agg[i].f[2] = 0.0
        check(groups, aggcol, want, agg, exact)


def test_reference_golden_plans_through_the_device_interpreter(emu):
    """the scan/aggregate plans of the reference-golden GPU tests (Q1, Q6, onek, gp_hashagg), compiled by the product and run
    by the product's interpreter on the CPU: the reference's own answers"""
    from _util import Q6_GOLDEN_REVENUE, golden, gp_hashagg_case, lineitem_fixture_pages, onek_fixture, onek_plans, tpch_q6_plan
    from greengage_b200 import tpch
    desc, pages, n = lineitem_fixture_pages()
    scan, agg, pool = tpch_q6_plan(desc)
    groups, aggcol, sc, ps, err = run_emu(emu, scan, agg, pool, pages)
    assert err == 0 and sc == n and len(groups) == 1
    assert abs(groups[0].sum[aggcol[0]] - Q6_GOLDEN_REVENUE) <= 1e-6 * Q6_GOLDEN_REVENUE and groups[0].count == ps
    exp = golden("q1_expected.json")
    scan, agg, pool = tpch.q1_plan(capi.TAB_LINEITEM_WIDE, capi.AGGSTAGE_NORMAL, interval_days=exp["interval_days"], desc=desc)
    groups, aggcol, sc, ps, err = run_emu(emu, scan, agg, pool, pages)
    by = {(chr(g.key[0] & 0xFF), chr(g.key[1] & 0xFF)): g for g in groups}
    assert err == 0 and len(by) == 4
    for e in exp["rows"]:
        g = by[(e["returnflag"], e["linestatus"])]
        assert g.count == e["count_order"]
        for i, name in enumerate(("sum_qty", "sum_base_price", "sum_disc_price", "sum_charge")):
            assert abs(g.sum[aggcol[i]] - float(e[name])) <= 1e-6 * float(e[name])
        assert abs(g.sum[aggcol[4]] / g.n[aggcol[4]] - float(e["avg_qty"])) <= 1e-6 * float(e["avg_qty"])
    d, pg, oexp = onek_fixture()
    plain, grouped = onek_plans(d, oexp)
    groups, aggcol, sc, ps, err = run_emu(emu, *plain, pg)
    f8i = lambda x: int(np.float64(x).view(np.int64))
    assert err == 0 and (f8i(groups[0].sum[aggcol[0]]), f8i(groups[0].sum[aggcol[1]]), groups[0].n[aggcol[2]]) == (oexp["sum_four"], oexp["max_four"], oexp["count_four"])
    groups, aggcol, sc, ps, err = run_emu(emu, *grouped, pg)
    assert err == 0 and sorted([int(np.int32(g.key[0] & 0xFFFFFFFF)), g.count, f8i(g.sum[aggcol[1]])] for g in groups) == oexp["by_ten"]
    d, pg, scan, agg, pool, want = gp_hashagg_case()
    groups, aggcol, sc, ps, err = run_emu(emu, scan, agg, pool, pg)
    assert err == 0 and {capi.unpack_str(g.key[0], 8).rstrip("\0"): f8i(g.sum[aggcol[0]]) for g in groups} == want


def test_aocs_column_files_to_q1_with_product_source_only(emu):
    """The whole AOCS path as far as a CPU can run it with the product's own source: column files (host loader: directory, tile
    plan) -> the decode kernel's device function (tests/aocs_decode_harness.c) -> datum rows -> the product's compiler and
    interpreter on the row descriptor.  Same groups, bit for bit, as the interpreter over the heap pages of the same rows."""
    import test_aocs_decode as ad
    from greengage_b200 import aocs, tpch
    so = os.path.join(os.path.dirname(emu._name), "harness.so")
    subprocess.check_call(["gcc", "-O2", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "aocs_decode_harness.c")])
    H = C.CDLL(so)
    H.harness_decode_rows.restype = C.c_uint32
    H.harness_decode_rows.argtypes = [C.c_void_p, C.c_int, C.c_uint64, C.c_int32, C.c_void_p]
    spec = tpch.synth_spec(capi.TAB_LINEITEM_WIDE, 40000, nsegs=2, seg=0)
    pages, nb, nr = tpch.synth_generate(spec)
    desc = capi.synth_tupdesc(capi.TAB_LINEITEM_WIDE)
    cols = [4, 5, 6, 7, 8, 9, 10]
    files, nrows = aocs.synth_columns(spec, cols, nr)
    rows, err = ad.host_decode(H, [desc.attrs[c] for c in cols], [files[c] for c in cols], 1024)
    assert err == 0 and rows.shape == (nr, 8)
    rdesc = capi.rows_tupdesc([desc.attrs[c].atttypid for c in cols], notnull=[1] * len(cols))
    names = dict(quantity=1, extendedprice=2, discount=3, tax=4, returnflag=5, linestatus=6, shipdate=7)
    scan_r, agg_r, pool_r = tpch.q1_plan(stage=capi.AGGSTAGE_NORMAL, desc=rdesc, cols=names)
    got, aggcol_r, sc, ps, e1 = run_emu(emu, scan_r, agg_r, pool_r, np.ascontiguousarray(rows), nrows=nr)
    scan_h, agg_h, pool_h = tpch.q1_plan(capi.TAB_LINEITEM_WIDE)
    want, aggcol_h, hsc, hps, e2 = run_emu(emu, scan_h, agg_h, pool_h, pages)
    assert e1 == 0 and e2 == 0 and (sc, ps) == (hsc, hps) == (nr, ps) and aggcol_r == aggcol_h
    key = lambda g: (g.key[0], g.key[1])
    for a, b in zip(sorted(got, key=key), sorted(want, key=key)):
        assert key(a) == key(b) and a.count == b.count
        assert [a.sum[j] for j in range(8)] == [b.sum[j] for j in range(8)] and [a.n[j] for j in range(8)] == [b.n[j] for j in range(8)]
    # and that answer is the oracle's
    owant, osc, ops, oexact = po.seqscan_agg(scan_h, agg_h, pool_h, pages, exact=True)
    check(want, aggcol_h, owant, agg_h, oexact)


def test_device_hash_and_routing_functions_equal_the_references(emu):
    """hash_uint32 / hashint8 / hashfloat8 / hash_any (<= 8 bytes) / cdbhash + jump_consistent_hash as written for the device
    (gg_device.cuh), against tests/golden/hash_kat.json — computed by the reference's own hashfunc.o, varchar.o and cdbhash.o"""
    from _util import golden
    K = golden("hash_kat.json")
    emu.emu_hash_uint32.restype = emu.emu_hashint8.restype = emu.emu_hashfloat8.restype = emu.emu_hash_any_le8.restype = C.c_uint32
    emu.emu_hash_uint32.argtypes = [C.c_uint32]
    emu.emu_hashint8.argtypes = [C.c_int64]
    emu.emu_hashfloat8.argtypes = [C.c_uint64]
    emu.emu_hash_any_le8.argtypes = [C.c_uint64, C.c_int]
    emu.emu_route.argtypes = [C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int, C.c_int]
    for v, want in K["hash_uint32"]:
        assert emu.emu_hash_uint32(v) == want
    for v, want in K["hashint4"]:
        assert emu.emu_hash_uint32(v & 0xFFFFFFFF) == want             # hashint4 = hash_uint32 of the value (hashfunc.c:46)
    for v, want in K["hashint8"]:
        assert emu.emu_hashint8(int(v)) == want
    for bits, want in K["hashfloat8"]:
        assert emu.emu_hashfloat8(int(bits) & 0xFFFFFFFFFFFFFFFF) == want
    short = 0
    for hexs, want in K["hash_any"]:
        b = bytes.fromhex(hexs)
        if len(b) <= 8:
            assert emu.emu_hash_any_le8(int.from_bytes(b.ljust(8, b"\0"), "little"), len(b)) == want
            short += 1
    for hexs, want in K["hashbpchar"]:
        b = bytes.fromhex(hexs).rstrip(b" ")                             # bcTruelen: the packed form is already stripped
        if len(b) <= 8:
            assert emu.emu_hash_any_le8(int.from_bytes(b.ljust(8, b"\0"), "little"), len(b)) == want
            short += 1
    assert short > 100
    routed = 0
    for r in K["route"]:
        n = len(r["typ"])
        if any(t in (capi.BPCHAROID, capi.VARCHAROID, capi.TEXTOID) and ln > 8 for t, ln in zip(r["typ"], r["len"])):
            continue
        t = (C.c_int32 * n)(*r["typ"])
        v = (C.c_int64 * n)(*[int(x) for x in r["val"]])
        ln = (C.c_int32 * n)(*r["len"])
        nn = (C.c_int32 * n)(*r["null"])
        assert emu.emu_route(t, v, ln, nn, n, r["nsegs"]) == r["seg"], r
        routed += 1
    assert routed > 1000


def test_device_routing_of_every_key_type_equals_the_oracle(emu):
    """key_hash + cdbhash (the one hash dispatch the sending Motion and the group-record Motion run) against the oracle's
    or_route_datums, which test_oracle_hash.py pins to the reference's cdbhash.o: every device key type — bool (hashchar),
    date (hashint4), timestamp (hashint8), float8 ±0 / NaN / ±inf, bpchar stripped and varchar / text with their blanks —
    alone and in keys of 2..4 columns with NULLs anywhere, over segment counts from 1 to 1024."""
    import random
    emu.emu_route.argtypes = [C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int, C.c_int]
    rng = random.Random(17)
    f8 = [0.0, -0.0, float("inf"), -float("inf"), float("nan"), 5e-324, 1.7976931348623157e308, 1.0, 1.0000000000000002, -2.5]
    strs = [b"", b" ", b"A", b"A ", b"ABCDEFGH", b"ABCDEFG ", b"\x80\xff", b"ab", b"abc  "]

    def value(t):
        if t == capi.BOOLOID:
            return rng.choice([0, 1]), 0
        if t in (capi.INT4OID, capi.DATEOID):
            return rng.choice([0, 1, -1, -2**31, 2**31 - 1, rng.randint(-2**31, 2**31 - 1)]), 0
        if t in (capi.INT8OID, capi.TIMESTAMPOID):
            return rng.choice([0, 2**32 + 1, -1, 2**32 - 1, -2**63, 2**63 - 1, rng.randint(-2**63, 2**63 - 1)]), 0
        if t == capi.FLOAT8OID:
            return f2b(rng.choice(f8)), 0
        b = rng.choice(strs)
        if t == capi.BPCHAROID:
            b = b.rstrip(b" ")                                           # packed bpchar is blank-stripped
        return int.from_bytes(b.ljust(8, b"\0"), "little", signed=True), len(b)

    types = [capi.BOOLOID, capi.INT4OID, capi.DATEOID, capi.INT8OID, capi.TIMESTAMPOID, capi.FLOAT8OID, capi.BPCHAROID,
             capi.VARCHAROID, capi.TEXTOID]
    seen = set()
    for it in range(6000):
        n = 1 if it < 2000 else rng.randint(2, 4)
        typ = [types[it % len(types)]] if n == 1 else [rng.choice(types) for _ in range(n)]
        vl = [value(t) for t in typ]
        nul = [0] * n if n == 1 and it % 10 else [int(rng.random() < 0.3) for _ in range(n)]
        nsegs = rng.choice([1, 2, 3, 7, 8, 64, 1024])
        t, v = (C.c_int32 * n)(*typ), (C.c_int64 * n)(*[x for x, _ in vl])
        ln, nn = (C.c_int32 * n)(*[x for _, x in vl]), (C.c_int32 * n)(*nul)
        want = po.lib().or_route_datums(t, v, ln, nn, n, nsegs)
        assert emu.emu_route(t, v, ln, nn, n, nsegs) == want, (typ, vl, nul, nsegs)
        seen.add(typ[0])
    assert seen == set(types)


def test_device_tuple_walk_equals_the_references_deform(emu):
    """walk_tuple (the GPU's slot_deform_tuple) over the 180 tuples the reference's heap_form_tuple built
    (tests/golden/heap_kat.json: NULL bitmaps, 1-byte and big-endian 4-byte varlena headers, alignment padding): every
    attribute's NULL flag, value or datum offset equals what the reference's heap_deform_tuple returned — on the
    constant-offset fast path and on the stored-offset path"""
    from _util import golden
    K = golden("heap_kat.json")
    emu.emu_walk.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_uint8), C.POINTER(C.c_uint32)]
    checked = 0
    for case in K["cases"]:
        d = K["descs"][case["desc"]]
        if len(d) > capi.GG_MAX_AGGS:
            continue
        desc = make_desc([(t, ln, al, bv) for t, ln, al, bv in d])
        tup = np.frombuffer(bytes.fromhex(case["tuple"]), dtype=np.uint8).copy()
        for force_slow in (0, 1):
            v, nu, err = (C.c_int64 * desc.natts)(), (C.c_uint8 * desc.natts)(), C.c_uint32(0)
            rc = emu.emu_walk(C.byref(desc), tup.ctypes.data, tup.size, force_slow, v, nu, C.byref(err))
            if rc == -6:
                break                                  # a column type the plan compiler does not take: not this test's subject
            assert rc == 0 and err.value == 0, (case["desc"], rc, err.value)
            assert [int(x) for x in nu] == case["deform_null"], case["desc"]
            for i in range(desc.natts):
                if not nu[i]:
                    want = int(case["deform"][i])
                    if desc.attrs[i].attlen == 4:
                        want = int(np.array([want & 0xFFFFFFFF], dtype=np.uint32).view(np.int32)[0])
                    assert int(v[i]) == want, (case["desc"], i, force_slow)
            checked += 1
    assert checked >= 300, checked


def test_device_arithmetic_and_comparisons_equal_the_references(emu):
    """float8pl / mi / mul / div with their overflow / underflow / division-by-zero ERRORs, float8 comparisons (NaN ordering,
    signed zeros) and date-vs-timestamp comparisons with "date out of range", as the device interpreter computes them,
    against tests/golden/float_kat.json — answers of the reference's own float.o / date.o.  Column-column, column-constant
    and constant-column operand forms of every case (different op codes of the accumulator machine)."""
    from _util import golden
    K = golden("float_kat.json")
    FN = {"pl": capi.F_FLOAT8PL, "mi": capi.F_FLOAT8MI, "mul": capi.F_FLOAT8MUL, "div": capi.F_FLOAT8DIV}
    ERR = {0x01, 0x02, 0x04}
    b2f = lambda x: float(np.int64(int(x)).view(np.float64))
    f2b = lambda x: int(np.float64(x).view(np.int64))
    d2 = make_desc([(capi.FLOAT8OID, 8, 'd', 1, 1), (capi.FLOAT8OID, 8, 'd', 1, 1)])

    def operands(p, form, a, b):
        x, y = p.var(1, capi.FLOAT8OID), p.var(2, capi.FLOAT8OID)
        if form == 1:
            y = p.const(capi.FLOAT8OID, 0.0); p.pool.nodes[y].constvalue = int(b)
        elif form == 2:
            x = p.const(capi.FLOAT8OID, 0.0); p.pool.nodes[x].constvalue = int(a)
        return x, y

    pages_cache = {}

    def pages_of(a, b):
        key = (a, b)
        if key not in pages_cache:
            pages_cache[key] = po.build_pages(d2, [[b2f(a), b2f(b)]])
        return pages_cache[key]

    n = 0
    for fn, a, b, err, r, _msg in K["arith"][::4]:
        for form in (0, 1, 2):
            p = ExprPool()
            x, y = operands(p, form, a, b)
            agg = capi.make_agg(0, [], [(capi.AGG_MIN_FLOAT8, p.func(FN[fn], capi.FLOAT8OID, x, y))])
            groups, aggcol, sc, ps, e = run_emu(emu, capi.make_scan(d2, -1), agg, p.pool, pages_of(a, b))
            if err:
                assert e & 0x07, (fn, b2f(a), b2f(b), form, hex(e))
            else:
                assert not (e & 0x07), (fn, b2f(a), b2f(b), form, hex(e))
                got, want = groups[0].sum[aggcol[0]], b2f(r)
                assert f2b(got) == int(r) or (got != got and want != want), (fn, b2f(a), b2f(b), form, got, want)
            n += 1
    for a, b, eq, lt, le, cmp3 in K["cmp"][::2]:
        for fid, want in ((capi.F_FLOAT8EQ, eq), (capi.F_FLOAT8LT, lt), (capi.F_FLOAT8LE, le), (capi.F_FLOAT8NE, 1 - eq),
                          (capi.F_FLOAT8GT, 1 - le), (capi.F_FLOAT8GE, 1 - lt)):
            for form in (0, 1, 2):
                p = ExprPool()
                x, y = operands(p, form, a, b)
                agg = capi.make_agg(0, [], [(capi.AGG_COUNT_STAR, -1)])
                groups, aggcol, sc, ps, e = run_emu(emu, capi.make_scan(d2, p.func(fid, capi.BOOLOID, x, y)), agg, p.pool, pages_of(a, b))
                assert e == 0 and ps == want, (fid, b2f(a), b2f(b), form, ps, want)
                n += 1
    dd = make_desc([(capi.DATEOID, 4, 'i', 1, 1)])
    FD = [capi.F_DATE_LT_TIMESTAMP, capi.F_DATE_LE_TIMESTAMP, capi.F_DATE_EQ_TIMESTAMP, capi.F_DATE_GT_TIMESTAMP, capi.F_DATE_GE_TIMESTAMP,
          capi.F_DATE_NE_TIMESTAMP]
    dpages = {}
    for op, d, ts, err, res in K["date_ts"][::3]:
        if d not in dpages:
            dpages[d] = po.build_pages(dd, [[d]])
        p = ExprPool()
        q = p.func(FD[op], capi.BOOLOID, p.var(1, capi.DATEOID), p.const(capi.TIMESTAMPOID, int(ts)))
        groups, aggcol, sc, ps, e = run_emu(emu, capi.make_scan(dd, q), capi.make_agg(0, [], [(capi.AGG_COUNT_STAR, -1)]), p.pool, dpages[d])
        if err:
            assert e & 0x80, (op, d, ts)
        else:
            assert e == 0 and ps == res, (op, d, ts, ps, res)
        n += 1
    assert n > 2500, n


def test_random_plans_over_datum_rows(emu):
    """the same random plans compiled for the GG_FMT_DATUMROWS descriptor (what a receiving Motion and the AOCS decode
    deliver: NULL-mask word + one 64-bit Datum per column, constant offsets) and run over the same rows in that format"""
    rng = np.random.default_rng(78)
    types = [capi.INT4OID, capi.INT4OID, capi.INT4OID, capi.FLOAT8OID, capi.FLOAT8OID, capi.BPCHAROID, capi.DATEOID, capi.INT8OID]
    notnull = [1, 1, 0, 1, 0, 0, 1, 1]
    hdesc = make_desc([(capi.INT4OID, 4, "i", 1, 1), (capi.INT4OID, 4, "i", 1, 1), (capi.INT4OID, 4, "i", 1, 0), (capi.FLOAT8OID, 8, "d", 1, 1),
                       (capi.FLOAT8OID, 8, "d", 1, 0), (capi.BPCHAROID, -1, "i", 0, 0), (capi.DATEOID, 4, "i", 1, 1), (capi.INT8OID, 8, "d", 1, 1)])
    rows, nulls = [], []
    for _ in range(2500):
        rows.append([int(rng.integers(0, 5)), int(rng.integers(-20, 20)), int(rng.integers(-5, 5)), float(rng.integers(-40, 40)) / 4,
                     float(rng.choice([0.0, -0.0, 0.5, -1.25, 3.0, 1e-3, float(rng.integers(-9, 9))])), bytes([65 + int(rng.integers(0, 3))]) + b" ",
                     int(rng.integers(-400, 400)), int(rng.integers(-10**9, 10**9))])
        nulls.append([False, False, rng.random() < 0.15, False, rng.random() < 0.15, rng.random() < 0.1, False, False])
    pages = po.build_pages(hdesc, rows, nulls)
    dr = np.zeros((len(rows), 9), dtype=np.int64)
    for i, (r, nl) in enumerate(zip(rows, nulls)):
        mask = 0
        for c, (v, isn) in enumerate(zip(r, nl)):
            if isn:
                mask |= 1 << c
            elif types[c] == capi.FLOAT8OID:
                dr[i, 1 + c] = np.float64(v).view(np.int64)
            elif types[c] == capi.BPCHAROID:
                dr[i, 1 + c] = capi.pack_str(v)[0]
            else:
                dr[i, 1 + c] = v
        dr[i, 0] = mask
    rdesc = capi.rows_tupdesc(types, notnull=notnull)
    stats = {"equal": 0, "errors": 0}
    for seed in range(200):
        scan_h, agg, p = random_plan(hdesc, seed)
        scan_r = capi.make_scan(rdesc, scan_h.qual)
        try:
            want, sc, ps, exact = po.seqscan_agg(scan_h, agg, p.pool, pages, exact=True)
        except po.OracleError:
            groups, aggcol, gsc, gps, err = run_emu(emu, scan_r, agg, p.pool, dr, nrows=len(rows))
            assert err & ARITH
            stats["errors"] += 1
            continue
        groups, aggcol, gsc, gps, err = run_emu(emu, scan_r, agg, p.pool, dr, nrows=len(rows))
        if err & ARITH:
            continue
        assert (gsc, gps) == (sc, ps), seed
        check(groups, aggcol, want, agg, exact)
        stats["equal"] += 1
    assert stats["equal"] > 120 and stats["errors"] > 10, stats


def test_avg_raises_what_float8_accum_raises_for_a_square_that_overflows(emu):
    """float8_accum squares every input (sumX2 += x*x, CHECKFLOATVAL: float.c:1895-1896): avg over a finite 1e200 is "value out
    of range: overflow" in the reference — also in a one-stage plan, which never ships sumX2.  sum() of the same column is fine."""
    desc = make_desc([(capi.INT4OID, 4, "i", 1, 1), (capi.FLOAT8OID, 8, "d", 1, 1)])
    pages = po.build_pages(desc, [[i % 3, 1e200 if i == 777 else float(i)] for i in range(2000)], None)
    for fn, raises in ((capi.AGG_AVG_FLOAT8, True), (capi.AGG_SUM_FLOAT8, False)):
        p = ExprPool()
        agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [p.var(1, capi.INT4OID)], [(fn, p.var(2, capi.FLOAT8OID))])
        scan = capi.make_scan(desc, -1)
        try:
            po.seqscan_agg(scan, agg, p.pool, pages)
            oracle_raised = False
        except po.OracleError:
            oracle_raised = True
        groups, aggcol, sc, ps, err = run_emu(emu, scan, agg, p.pool, pages)
        assert oracle_raised == raises and bool(err & 0x01) == raises, (fn, oracle_raised, hex(err))


def test_numeric_q1_through_the_device_interpreter_is_the_references_golden_answer(emu):
    """numeric(15,2) columns decoded from their on-disk digits and evaluated as scaled 64-bit integers by the product's
    compiler + interpreter (host build), the two halves of every sum folded the way the kernels fold them, finalised by the
    product's host code (gg_debug_numeric_final): the reference's golden Q1 over its numeric heap_lineitem, to the last digit —
    and the oracle's answer over the same pages."""
    from test_oracle_numeric import numeric_lineitem_pages
    from _util import golden
    desc, pages, n = numeric_lineitem_pages()
    exp = golden("q1_expected.json")
    scan, agg, pool = tpch.q1_plan_numeric(desc, interval_days=exp["interval_days"])
    groups, aggcol, sc, ps, err = run_emu(emu, scan, agg, pool, pages)
    assert err == 0 and sc == n
    want, wsc, wps = po.seqscan_agg(scan, agg, pool, pages)
    assert (sc, ps) == (wsc, wps)
    D = capi.dev_lib()
    D.gg_debug_numeric_final.argtypes = [C.c_int, C.c_int64, C.c_int64, C.c_int, C.c_uint64, C.POINTER(capi.gg_aggval)]
    scales = [2, 2, 4, 6, 2, 2, 2]
    by = {(int(g.key[0]), int(g.key[1])): g for g in groups}
    names = ["sum_qty", "sum_base_price", "sum_disc_price", "sum_charge", "avg_qty", "avg_price", "avg_disc"]
    for w, o in zip(exp["rows"], sorted(want, key=lambda r: (r.key[0], r.key[1]))):
        g = by[(capi.pack_str(w["returnflag"])[0], capi.pack_str(w["linestatus"])[0])]
        assert g.count == w["count_order"]
        for i, name in enumerate(names):
            col = aggcol[i]
            lo = int(np.float64(g.sum[col]).view(np.int64))
            hi = int(np.float64(g.sum[col + 1]).view(np.int64))
            v = capi.gg_aggval()
            assert D.gg_debug_numeric_final(1 if i >= 4 else 0, lo, hi, scales[i], g.n[col], C.byref(v)) == 0
            assert capi.numeric_of_aggval(v) == w[name], (name, capi.numeric_of_aggval(v), w[name])
            assert capi.numeric_of_aggval(v) == capi.numeric_of_aggval(o.agg[i])


def test_numeric_finalisation_equals_the_references_sum_and_avg():
    """the product's host finalisation of (low half, high half, N) against numeric_kat.json's sums and averages"""
    import json
    kat = json.load(open(os.path.join(HERE, "golden", "numeric_kat.json")))
    D = capi.dev_lib()
    D.gg_debug_numeric_final.argtypes = [C.c_int, C.c_int64, C.c_int64, C.c_int, C.c_uint64, C.POINTER(capi.gg_aggval)]
    for case in kat["sumavg"]:
        parsed = [capi.numeric_parse(t) for t in case["values"]]
        sc = max(s for _, s in parsed)
        lo = sum((v * 10 ** (sc - s)) & 0xFFFFFFFF for v, s in parsed)
        hi = sum((v * 10 ** (sc - s)) >> 32 for v, s in parsed)
        for which, name in ((0, "sum"), (1, "avg")):
            v = capi.gg_aggval()
            assert D.gg_debug_numeric_final(which, lo, hi, sc, len(parsed), C.byref(v)) == 0
            assert capi.numeric_of_aggval(v) == case[name], (name, capi.numeric_of_aggval(v), case[name])


def test_exact_numeric_reference_restates_the_references_sum_and_avg():
    """tests/_numeric.py (the exact reference the GPU numeric tests compare with) against numeric_kat.json's sums and
    averages, which the reference's own numeric.o computed: every digit and the display scale"""
    import json
    import _numeric as nref
    kat = json.load(open(os.path.join(HERE, "golden", "numeric_kat.json")))
    for case in kat["sumavg"]:
        parsed = [capi.numeric_parse(t) for t in case["values"]]
        sc = max(s for _, s in parsed)
        vals = [nref.rescale(v, s, sc) for v, s in parsed]
        assert nref.sum_text(vals, sc) == case["sum"]
        assert nref.avg_text(vals, sc) == case["avg"], (case["avg"], nref.avg_text(vals, sc))
    assert len(kat["sumavg"]) >= 60


def _numeric_sum_through_the_interpreter(emu, values, scale, precision=38):
    """sum(x) over rows of one numeric(precision, scale) column through the product's compiler + interpreter (host build):
    (error flags, the sum at `scale` or None)"""
    import _numeric as nref
    desc = capi.gg_tupdesc()
    desc.natts = 1
    a = desc.attrs[0]
    a.atttypid, a.attlen, a.attalign, a.attbyval, a.atttypmod, a.attnotnull = capi.NUMERICOID, -1, ord("i"), 0, nref.typmod(precision, scale), 1
    pages = po.build_pages(desc, [[capi.numeric_payload(v, scale)] for v in values])
    p = ExprPool()
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [], [(capi.AGG_SUM_NUMERIC, p.var(1, capi.NUMERICOID))])
    groups, aggcol, sc, ps, err = run_emu(emu, capi.make_scan(desc, -1), agg, p.pool, pages)
    assert sc == len(values) and len(groups) == 1
    col = aggcol[0]
    lo, hi = int(np.float64(groups[0].sum[col]).view(np.int64)), int(np.float64(groups[0].sum[col + 1]).view(np.int64))
    return err, hi * 2 ** 32 + lo


# the leading five base-10000 digits form an integer in [2^64, 2^64 + 8383]: v * 10000 + digit carries past 2^64
WRAP_FAMILY = [
    ([2 ** 64 + 1, 3], 0, 20),                              # the sum came back as 4
    ([2 ** 64 + 7, 3], 4, 20),                              # 1844674407370955.1623 + 0.0003 came back as 0.0010
    ([-(2 ** 64 + 2792) * 10 ** 4], 0, 24),                 # -184467440737095544080000 came back as -27920000
    ([(2 ** 64 + 8383) * 10 ** 4, 1], 4, 24),               # an integer at scale 4: its digits align with 10^(4k) all the same
    ([2 ** 64, -5], 0, 20), ([-(2 ** 64 + 100)], 8, 28), ([(2 ** 64 + 4000) * 10 ** 8], 8, 36),
]


def test_numeric_decoder_refuses_values_whose_digits_carry_past_2_64(emu):
    """The 2^64 wrap family through the interpreter must raise GGP_EF_NUMERIC_RANGE: every such value is >= 2^63 at its
    column scale, so no answer is right but a refusal.  With the carry of the last digit unchecked, the decoder wrapped to a
    small number and the sums above came back wrong without an error flag."""
    for values, scale, prec in WRAP_FAMILY:
        err, got = _numeric_sum_through_the_interpreter(emu, values, scale, prec)
        assert err & 0x8000, (values, scale, got)


def test_numeric_sums_near_the_64_bit_edges_are_exact_or_refused(emu):
    """Seeded pairs of values near 10^k, 2^63 and 2^64 (times 10^(4j), so that the base-10000 digits line up with the carry)
    at scales 0, 2, 4, 8 and 15: the interpreter's sum equals the exact one, or it is refused — a refusal when an input is >= 2^63
    at its scale, and an exact answer when every input is below 2^62."""
    import _numeric as nref
    rng = np.random.default_rng(64)
    stats = {nref.REQUIRED: 0, nref.FORBIDDEN: 0, nref.EITHER: 0, "refused": 0}
    for trial in range(300):
        scale = int(rng.choice([0, 2, 4, 8, 15]))
        vals = []
        for _ in range(2):
            kind = int(rng.integers(0, 4))
            if kind <= 1:
                base = 10 ** int(rng.integers(0, 27))
            elif kind == 2:
                base = 2 ** 63
            else:
                base = 2 ** 64 * 10 ** (4 * int(rng.integers(0, 3)))
            v = base + int(rng.integers(-9000, 9000))
            vals.append(v if rng.random() < 0.5 else -v)
        rule = nref.refusal(vals, [])
        stats[rule] += 1
        err, got = _numeric_sum_through_the_interpreter(emu, vals, scale)
        refused = bool(err & 0x8000)
        stats["refused"] += refused
        assert not (err & ~0x8000), (trial, hex(err))
        if rule == nref.REQUIRED:
            assert refused, (trial, vals, scale, got)
        elif rule == nref.FORBIDDEN:
            assert not refused and got == sum(vals), (trial, vals, scale, got)
        elif not refused:
            assert got == sum(vals), (trial, vals, scale, got)
    assert stats[nref.REQUIRED] > 100 and stats[nref.FORBIDDEN] > 20, stats


def test_random_numeric_expressions_mean_what_the_oracle_computes(emu):
    """numeric_add / _sub / _mul trees, comparisons in the qual, NULLs, columns of different scales: sums (both halves) and
    counts of the device interpreter equal the oracle's exact sums"""
    rng = np.random.default_rng(99)
    NUM = capi.NUMERICOID
    desc = capi.gg_tupdesc()
    spec = [(capi.INT4OID, 4, "i", 1, -1, 1), (NUM, -1, "i", 0, ((15 << 16) | 2) + 4, 0), (NUM, -1, "i", 0, ((12 << 16) | 0) + 4, 1),
            (NUM, -1, "i", 0, ((10 << 16) | 4) + 4, 0)]
    desc.natts = len(spec)
    for i, (t, l, al, bv, tm, nn) in enumerate(spec):
        a = desc.attrs[i]
        a.atttypid, a.attlen, a.attalign, a.attbyval, a.atttypmod, a.attnotnull = t, l, ord(al), bv, tm, nn
    rows, nulls = [], []
    for i in range(3000):
        rows.append([int(rng.integers(0, 4)), capi.numeric_payload(int(rng.integers(-10**7, 10**7)), 2), capi.numeric_payload(int(rng.integers(-500, 500)), 0),
                     capi.numeric_payload(int(rng.integers(-10**6, 10**6)), 4)])
        nulls.append([False, rng.random() < 0.1, False, rng.random() < 0.1])
    pages = po.build_pages(desc, rows, nulls)
    scale_of = {2: 2, 3: 0, 4: 4}

    def expr(p, depth):
        if depth == 0 or rng.random() < 0.3:
            if rng.random() < 0.25:
                sc = int(rng.integers(0, 3))
                return p.const(NUM, capi.numeric_text(int(rng.integers(-99, 99)), sc)), sc
            a = int(rng.integers(2, 5))
            return p.var(a, NUM), scale_of[a]
        (l, ls), (r, rs) = expr(p, depth - 1), expr(p, depth - 1)
        op = rng.choice(["+", "-", "*"])
        if op == "*" and ls + rs > 8:
            op = "+"
        f = {"+": capi.F_NUMERIC_ADD, "-": capi.F_NUMERIC_SUB, "*": capi.F_NUMERIC_MUL}[op]
        return p.func(f, NUM, l, r), (ls + rs if op == "*" else max(ls, rs))

    ran = 0
    for seed in range(40):
        p = ExprPool()
        args = [expr(p, 2) for _ in range(int(rng.integers(1, 4)))]
        (ql, _), (qr, _) = expr(p, 1), expr(p, 1)
        qual = p.func(int(rng.choice([capi.F_NUMERIC_LT, capi.F_NUMERIC_GE, capi.F_NUMERIC_NE])), capi.BOOLOID, ql, qr) if rng.random() < 0.7 else -1
        agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [p.var(1, capi.INT4OID)], [(capi.AGG_COUNT_STAR, -1)] + [(capi.AGG_SUM_NUMERIC, a) for a, _ in args])
        scan = capi.make_scan(desc, qual)
        want, wsc, wps = po.seqscan_agg(scan, agg, p.pool, pages)
        groups, aggcol, sc, ps, err = run_emu(emu, scan, agg, p.pool, pages)
        assert err == 0 and (sc, ps) == (wsc, wps), (seed, hex(err))
        by = {int(np.uint64(g.key[0]).astype(np.int64)): g for g in groups}
        for r in want:
            g = by[r.key[0]]
            assert g.count == r.agg[0].i
            for i, (a, asc) in enumerate(args):
                col = aggcol[1 + i]
                lo, hi = int(np.float64(g.sum[col]).view(np.int64)), int(np.float64(g.sum[col + 1]).view(np.int64))
                if r.agg[1 + i].isnull:
                    assert g.n[col] == 0
                else:
                    assert capi.numeric_text(hi * 2 ** 32 + lo, asc) == capi.numeric_of_aggval(r.agg[1 + i]), (seed, i)
        ran += 1
    assert ran == 40
