"""Plan compiler (host side, no GPU): expression trees -> accumulator-machine program; eligibility."""
import ctypes as C
import os

import pytest

from _util import make_desc
from greengage_b200 import capi, tpch
from greengage_b200.capi import ExprPool

L = capi.dev_lib()
L.gg_debug_disasm_scanagg.argtypes = [C.POINTER(capi.gg_scan), C.POINTER(capi.gg_agg), C.POINTER(capi.gg_exprpool), C.c_char_p, C.c_int]


def disasm(scan, agg, pool):
    buf = C.create_string_buffer(1 << 16)
    n = L.gg_debug_disasm_scanagg(C.byref(scan), C.byref(agg), C.byref(pool), buf, 1 << 16)
    if n < 0:
        raise capi.GGError(n, L.gg_last_error().decode())
    return buf.value.decode().splitlines()


def test_q1_program_shape():
    lines = disasm(*tpch.q1_plan(capi.TAB_LINEITEM_WIDE))
    ops = [ln.split()[1] for ln in lines]
    assert ops[:3] == ["LD_C4", "DATE2TS", "CMPI_K"] and "FILTER" in lines[2]
    assert "KEY0" in lines[3] and "KEY1" in lines[4] and "GROUP" in lines[4]
    # l_extendedprice*(1-l_discount) is computed once and reused for sum_charge
    assert sum(1 for o in ops if o == "SUB_C") == 1 and sum(1 for o in ops if o.startswith("MUL")) == 2
    # single-stage plan: float8_avg ignores sumX2, so no sums of squares are produced
    assert not any("OUTSQ" in ln for ln in lines)
    assert ops[-1] == "END"
    # constant offsets of the fixed-width prefix are baked in; l_linestatus/l_shipdate come from the walk
    assert "off=24" in lines[5] and "off=-1" in lines[4]
    part = disasm(*tpch.q1_plan(capi.TAB_LINEITEM_WIDE, capi.AGGSTAGE_PARTIAL))
    assert sum(1 for ln in part if "OUTSQ" in ln) == 3          # avg's transition state {N, sumX, sumX2}


def test_unsupported_plans_are_refused():
    desc = make_desc([(1700, -1, 'i', 0), (capi.FLOAT8OID, 8, 'd', 1)])       # numeric column
    p = ExprPool()
    scan = capi.make_scan(desc, -1)
    with pytest.raises(capi.GGError) as e:
        disasm(scan, capi.make_agg(0, [], [(capi.AGG_SUM_FLOAT8, p.var(1, 1700))]), p.pool)
    assert e.value.code == -6
    p = ExprPool()
    with pytest.raises(capi.GGError):
        disasm(scan, capi.make_agg(0, [], [(2114, p.var(2, capi.FLOAT8OID))]), p.pool)     # sum(numeric)
    p = ExprPool()
    with pytest.raises(capi.GGError):                                                       # float8 op on an int column without a cast
        disasm(capi.make_scan(make_desc([(capi.INT4OID, 4, 'i', 1)]), -1),
               capi.make_agg(0, [], [(capi.AGG_SUM_FLOAT8, p.func(capi.F_FLOAT8PL, capi.FLOAT8OID, p.var(1, capi.INT4OID), p.const(capi.FLOAT8OID, 1.0)))]), p.pool)


def test_deep_expression_uses_temporaries():
    desc = make_desc([(capi.FLOAT8OID, 8, 'd', 1, 1)] * 4)
    p = ExprPool()
    a, b, c, d = (p.var(i + 1, capi.FLOAT8OID) for i in range(4))
    e = p.func(capi.F_FLOAT8MI, capi.FLOAT8OID, p.func(capi.F_FLOAT8MUL, capi.FLOAT8OID, a, b),
               p.func(capi.F_FLOAT8DIV, capi.FLOAT8OID, c, d))
    lines = disasm(capi.make_scan(desc, -1), capi.make_agg(0, [], [(capi.AGG_SUM_FLOAT8, e)]), p.pool)
    ops = [ln.split()[1] for ln in lines]
    # a plain aggregate opens with the (key-less) GROUP action
    assert ops == ["NOP", "LD_C8", "MUL_C", "LD_C8", "DIV_C", "RSUB_T", "END"] and "GROUP" in lines[0] and "ST t0" in lines[2]


# ---- join pipelines and datum-row input -------------------------------------------------------------------------

L.gg_debug_disasm_join.argtypes = [C.POINTER(capi.gg_scan), C.POINTER(capi.gg_scan), C.POINTER(capi.gg_hashjoin), C.POINTER(capi.gg_agg),
                                   C.POINTER(capi.gg_exprpool), C.c_char_p, C.c_int]


def disasm_join(outer, inner, hj, agg, pool):
    buf = C.create_string_buffer(1 << 16)
    n = L.gg_debug_disasm_join(C.byref(outer), C.byref(inner), C.byref(hj), C.byref(agg), C.byref(pool), buf, 1 << 16)
    if n < 0:
        raise capi.GGError(n, L.gg_last_error().decode())
    text = buf.value.decode()
    build, probe = text.split("-- probe")
    return build.splitlines()[1:], probe.splitlines()[1:], text


def test_join_programs_shape():
    build, probe, text = disasm_join(*tpch.join_plan(kind="q3ish", jointype=capi.JOIN_INNER))
    assert "payload 2" in text
    # build: inner qual, then the join key claims the slot, then the payload columns in slot order
    assert "FILTER" in build[1] and "KEY0 GROUP" in build[2] and "OUT0" in build[3] and "OUT1" in build[4]
    # probe: the outer key completes the first piece; the per-match piece reads inner columns (idx >= 128) from the payload
    assert "KEY0 PROBE" in probe[0] and "per-match segment from pc 1" in text
    assert any("idx=128" in ln and "FILTER" in ln for ln in probe)           # the join qual l_shipdate > o_orderdate
    assert any("idx=129" in ln and "GROUP" in ln for ln in probe)            # GROUP BY o_orderstatus
    assert not any("off=" in ln and "idx=12" in ln and "off=-1" not in ln for ln in probe)   # no tuple offsets for payload reads


def test_join_carries_inner_numeric_columns_as_scaled_integers():
    """An inner numeric column above a join travels in the hash-table payload as its scaled 64-bit integer: the build program
    decodes it (LD_NUM at the column's declared scale, the scale shown as cc=) into an OUT slot, and the probe program reads
    the payload slot (idx >= 128), rescaled by a multiply where the expression needs a larger scale."""
    import _numeric as nref
    NUM = capi.NUMERICOID
    odesc = capi.gg_tupdesc()
    idesc = capi.gg_tupdesc()
    for d, spec in ((odesc, [(capi.INT4OID, -1), (NUM, nref.typmod(18, 4))]), (idesc, [(capi.INT4OID, -1), (NUM, nref.typmod(15, 2)), (NUM, nref.typmod(12, 0))])):
        d.natts = len(spec)
        for i, (t, tm) in enumerate(spec):
            a = d.attrs[i]
            a.atttypid, a.attlen, a.attalign, a.attbyval, a.atttypmod, a.attnotnull = t, 4 if t == capi.INT4OID else -1, ord("i"), int(t == capi.INT4OID), tm, 1
    p = ExprPool()
    ok, ik = p.var(1, capi.INT4OID, 0), p.var(1, capi.INT4OID, 1)
    x, y, z = p.var(2, NUM, 0), p.var(2, NUM, 1), p.var(3, NUM, 1)
    qual = p.func(capi.F_NUMERIC_LT, capi.BOOLOID, x, y)                        # outer scale 4 < inner scale 2: inner rescaled x100
    hj = capi.make_hashjoin(capi.JOIN_INNER, [ok], [ik], qual)
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [], [(capi.AGG_SUM_NUMERIC, y), (capi.AGG_SUM_NUMERIC, p.func(capi.F_NUMERIC_MUL, NUM, x, z))])
    build, probe, text = disasm_join(capi.make_scan(odesc, -1), capi.make_scan(idesc, -1), hj, agg, p.pool)
    ops = [ln.split() for ln in build]
    outs = [ln for ln in build if " OUT" in ln]
    assert len(outs) == 2 and all(ln.split()[1] == "LD_NUM" for ln in outs), build
    assert sorted(ln.split()[3] for ln in outs) == ["cc=0", "cc=2"], build       # each at its own column's scale
    assert not any(o[1] == "LD_BOOL" for o in ops), build
    inner_loads = [ln for ln in probe if ln.split()[1] == "LD_NUM" and int(ln.split()[2][4:]) >= 128]
    assert len(inner_loads) >= 3, probe                                          # qual, sum(y), x * z
    assert all("off=-1" in ln for ln in inner_loads), probe                       # from the payload, not from a tuple offset
    nxt = [probe[probe.index(ln) + 1].split()[1] for ln in inner_loads if "cc=2" in ln]
    assert "IMUL_K" in nxt, probe                                                 # y at scale 4 for the comparison


def test_join_shapes_outside_the_subset_are_refused():
    outer, inner, hj, agg, pool = tpch.join_plan(kind="count")
    hj.jointype = 7                                                          # JOIN_UNIQUE_OUTER (planner-internal)
    with pytest.raises(capi.GGError) as e:
        disasm_join(outer, inner, hj, agg, pool)
    assert e.value.code == -6
    outer, inner, hj, agg, pool = tpch.join_plan(kind="count")
    hj.nkeys = 3
    with pytest.raises(capi.GGError) as e:
        disasm_join(outer, inner, hj, agg, pool)
    assert e.value.code == -6
    # mismatched key classes (int8 = float8) have no common hash function
    p = ExprPool()
    li, od = capi.synth_tupdesc(capi.TAB_LINEITEM_NARROW), capi.synth_tupdesc(capi.TAB_ORDERS)
    hj = capi.make_hashjoin(capi.JOIN_INNER, [p.var(1, capi.INT8OID, 0)], [p.var(4, capi.FLOAT8OID, 1)])
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [], [(capi.AGG_COUNT_STAR, -1)])
    with pytest.raises(capi.GGError) as e:
        disasm_join(capi.make_scan(li, -1), capi.make_scan(od, -1), hj, agg, p.pool)
    assert e.value.code == -6 and "join key" in str(e.value)


KEY_TYPES = {"int4": (capi.INT4OID, 4, "i", 1), "int8": (capi.INT8OID, 8, "d", 1), "date": (capi.DATEOID, 4, "i", 1),
             "timestamp": (capi.TIMESTAMPOID, 8, "d", 1), "bool": (capi.BOOLOID, 1, "c", 1), "float8": (capi.FLOAT8OID, 8, "d", 1),
             "bpchar": (capi.BPCHAROID, -1, "i", 0), "varchar": (capi.VARCHAROID, -1, "i", 0), "text": (capi.TEXTOID, -1, "i", 0)}
# the pairs the reference can hash-join: one hash opfamily per pair (pg_amop.h:557-565).  integer_ops is the only cross-type
# family among these types; varchar has no operators of its own and uses text_ops.
HASH_JOINABLE = {frozenset(p) for p in (("int4",), ("int8",), ("int4", "int8"), ("date",), ("timestamp",), ("bool",), ("float8",),
                                         ("bpchar",), ("varchar",), ("text",), ("varchar", "text"))}


@pytest.mark.parametrize("nkeys", [1, 2])
def test_join_key_pairs_follow_the_reference_hash_opfamilies(nkeys):
    """Every (outer, inner) pair of device key types: compiled when the reference can hash-join it, GG_ERR_UNSUPPORTED with a
    message naming the join key otherwise — date = timestamp, bpchar = text, int4 = date, int4 = bool, float8 = int8 and the
    like must never compile into a bitwise comparison of unlike encodings.  With two keys the pair is the second key."""
    names = list(KEY_TYPES)
    desc = make_desc([KEY_TYPES[n] for n in names])
    for i, a in enumerate(names):
        for j, b in enumerate(names):
            p = ExprPool()
            ok, ik = [p.var(i + 1, KEY_TYPES[a][0], 0)], [p.var(j + 1, KEY_TYPES[b][0], 1)]
            if nkeys == 2:
                ok, ik = [p.var(1, capi.INT4OID, 0)] + ok, [p.var(1, capi.INT4OID, 1)] + ik
            hj = capi.make_hashjoin(capi.JOIN_INNER, ok, ik)
            agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [], [(capi.AGG_COUNT_STAR, -1)])
            args = (capi.make_scan(desc, -1), capi.make_scan(desc, -1), hj, agg, p.pool)
            if frozenset((a, b)) in HASH_JOINABLE:
                build, probe, text = disasm_join(*args)
                assert "KEY%d PROBE" % (nkeys - 1) in text, (a, b, text)
            else:
                with pytest.raises(capi.GGError) as e:
                    disasm_join(*args)
                assert e.value.code == -6 and "join key %d" % (nkeys - 1) in str(e.value), (a, b, str(e.value))


def test_datum_row_input_uses_constant_word_offsets():
    types = [capi.INT8OID, capi.FLOAT8OID, capi.BPCHAROID, capi.DATEOID]
    desc = capi.rows_tupdesc(types, notnull=[1, 1, 0, 1])
    p = ExprPool()
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [p.var(3, capi.BPCHAROID)], [(capi.AGG_SUM_FLOAT8, p.var(2, capi.FLOAT8OID)), (capi.AGG_MIN_DATE, p.var(4, capi.DATEOID))])
    lines = disasm(capi.make_scan(desc, -1), agg, p.pool)
    # every column is a 64-bit word: strings and dates are already in loaded form, offsets are 8 * attno
    assert "LD_C8" in lines[0] and "off=16" in lines[0] and "KEY0" in lines[0]
    assert "LD_C8" in lines[1] and "off=8" in lines[1]
    assert "LD_C8" in lines[2] and "off=24" in lines[2]


def test_generated_kernel_sources_compile_for_sm90a(tmp_path):
    """The plan-specialised translation units (what NVRTC compiles at run time) must be valid CUDA for every kernel
    role: checked here with nvcc, without a GPU."""
    import shutil
    import subprocess
    from greengage_b200.build import ARCH
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    L.gg_debug_jit_source_join.argtypes = [C.POINTER(capi.gg_scan), C.POINTER(capi.gg_scan), C.POINTER(capi.gg_hashjoin), C.POINTER(capi.gg_agg),
                                           C.POINTER(capi.gg_exprpool), C.c_int, C.c_int, C.c_char_p, C.c_int]
    outer, inner, hj, agg, pool = tpch.join_plan(kind="q3ish", jointype=capi.JOIN_FULL)
    csrc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "greengage_b200", "csrc")
    for which, mode, name in ((0, 3, "build"), (1, 2, "probe_transposed_nulls"), (1, 5, "probe_hashagg")):
        buf = C.create_string_buffer(1 << 18)
        n = L.gg_debug_jit_source_join(C.byref(outer), C.byref(inner), C.byref(hj), C.byref(agg), C.byref(pool), which, mode, buf, 1 << 18)
        assert n > 0, L.gg_last_error()
        src = tmp_path / (name + ".cu")
        src.write_text(buf.value.decode())
        r = subprocess.run([nvcc] + ARCH + ["-std=c++17", "-I", csrc, "-c", str(src), "-o", str(tmp_path / (name + ".o"))],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-2000:]


def test_q6_plan_compiles_to_five_filters_and_one_sum():
    """The Q6 plan the golden tests run (tests/_util.tpch_q6_plan): the five range predicates are the clauses of an
    implicit-AND qual, one FILTER each, in front of the single accumulate; no group key (private-accumulator kernel)."""
    from _util import lineitem_fixture_pages, tpch_q6_plan
    desc, _, _ = lineitem_fixture_pages()
    lines = disasm(*tpch_q6_plan(desc))
    assert sum(1 for ln in lines if "FILTER" in ln) == 5 and sum(1 for ln in lines if "AND_T" in ln) == 0
    assert sum(1 for ln in lines if "CMPF_K" in ln) == 3 and sum(1 for ln in lines if "CMPI_K" in ln) == 2
    assert sum(1 for ln in lines if "OUT" in ln and "OUTSQ" not in ln) == 1 and not any("KEY" in ln for ln in lines)
    assert lines[-1].split()[1] == "END"


def test_malformed_plans_are_error_codes_not_crashes():
    """What crosses the C-ABI is validated before anything indexes with it (gg_compile.cpp: valid_nodes): a plan whose
    expression indices, attribute numbers or counts are out of range comes back as GG_ERR_ARG with a message.  Found by
    fuzzing the plan compiler under AddressSanitizer (a child index past the pool used to be dereferenced)."""
    def refused(scan, agg, pool, code=-10):
        with pytest.raises(capi.GGError) as e:
            disasm(scan, agg, pool)
        assert e.value.code == code, (e.value.code, str(e.value))
        return str(e.value)

    def fresh():
        scan, agg, pool = tpch.q1_plan(capi.TAB_LINEITEM_WIDE)
        return (type(scan).from_buffer_copy(bytes(scan)), type(agg).from_buffer_copy(bytes(agg)), type(pool).from_buffer_copy(bytes(pool)))

    scan, agg, pool = fresh()
    assert disasm(scan, agg, pool)                                     # the copy compiles
    func = next(i for i in range(pool.nnodes) if pool.nodes[i].kind == 3)      # GG_E_FUNC
    for bad in (2 ** 31 - 1, -7, 4000, func):                          # child index: far out, negative, past the pool, itself (a cycle)
        scan, agg, pool = fresh()
        pool.nodes[func].args[0] = bad
        assert "children come before their parents" in refused(scan, agg, pool)
    scan, agg, pool = fresh()
    pool.nnodes = 10 ** 6
    assert "expression pool" in refused(scan, agg, pool)
    scan, agg, pool = fresh()
    var = next(i for i in range(pool.nnodes) if pool.nodes[i].kind == 1)
    pool.nodes[var].varattno = 99
    assert "attribute 99" in refused(scan, agg, pool)
    scan, agg, pool = fresh()
    pool.nodes[var].varno = 1                                          # an inner Var in a plan without an inner side
    assert "relation 1" in refused(scan, agg, pool)
    for field, bad in (("numCols", 77), ("numAggs", -3), ("numAggs", 10 ** 6)):
        scan, agg, pool = fresh()
        setattr(agg, field, bad)
        refused(scan, agg, pool)
    scan, agg, pool = fresh()
    agg.aggs[0].arg = 12345
    assert "aggregate argument" in refused(scan, agg, pool)
    scan, agg, pool = fresh()
    scan.qual = 500
    assert "scan qual" in refused(scan, agg, pool)
    scan, agg, pool = fresh()
    scan.desc.natts = 1000
    refused(scan, agg, pool)
    # nodes no root reaches are not looked at: a pool may hold other pipelines' expressions
    scan, agg, pool = fresh()
    n = pool.nnodes
    pool.nodes[n].kind, pool.nodes[n].varno, pool.nodes[n].varattno = 1, 1, 3
    pool.nnodes = n + 1
    assert disasm(scan, agg, pool)
    # the same validation guards the join compiler
    outer, inner, hj, jagg, jpool = tpch.join_plan(kind="q3ish", jointype=capi.JOIN_INNER)
    hj = type(hj).from_buffer_copy(bytes(hj))
    hj.innerkey[0] = -5
    with pytest.raises(capi.GGError) as e:
        disasm_join(outer, inner, hj, jagg, jpool)
    assert e.value.code == -10 and "inner join key" in str(e.value)


def test_qual_clauses_are_separate_filters_and_and_or_arms_are_guarded():
    """An implicit-AND qual compiles to one FILTER per clause (ExecQual's list walk, execQual.c:6260-6310); a nested AND / OR
    keeps its three-valued combinator but the second arm runs under a GUARD (ExecEvalAnd / ExecEvalOr stop at the deciding
    arm, execQual.c:3385,3455)."""
    from _util import lineitem_fixture_pages, tpch_q6_plan
    desc, _, _ = lineitem_fixture_pages()
    flat = disasm(*tpch_q6_plan(desc))
    assert sum(1 for ln in flat if "FILTER" in ln) == 5 and not any("AND_T" in ln or "GUARD" in ln for ln in flat)
    assert sum(1 for ln in disasm(*tpch.q1_plan(capi.TAB_LINEITEM_WIDE)) if "FILTER" in ln) == 1
    d = make_desc([(capi.FLOAT8OID, 8, 'd', 1), (capi.FLOAT8OID, 8, 'd', 1)])
    p = ExprPool()
    a, b = p.var(1, capi.FLOAT8OID), p.var(2, capi.FLOAT8OID)
    nz = p.func(capi.F_FLOAT8NE, capi.BOOLOID, b, p.const(capi.FLOAT8OID, 0.0))
    gt = p.func(capi.F_FLOAT8GT, capi.BOOLOID, p.func(capi.F_FLOAT8DIV, capi.FLOAT8OID, a, b), p.const(capi.FLOAT8OID, 1.0))
    inner = p.boolop(capi.E_OR, p.boolop(capi.E_NOT, nz), gt)            # NOT (b <> 0) OR a / b > 1
    lines = disasm(capi.make_scan(d, inner), capi.make_agg(0, [], [(capi.AGG_COUNT_STAR, -1)]), p.pool)
    ops = [ln.split()[1] for ln in lines]
    assert ops.count("GUARD_OR") == 1 and ops.count("UNGUARD") == 1 and ops.count("OR_T") == 1
    assert ops.index("GUARD_OR") < ops.index("DIV_C") < ops.index("UNGUARD") < ops.index("OR_T")


def test_partial_stage_ships_sumsq_unless_this_engine_combines_it():
    """avg's transition state is {N, sumX, sumX2} (float8_accum, float.c:1878); float8_avg never reads sumX2, so a PARTIAL
    stage whose rows go to this engine's own FINAL stage (GG_AGGF_DEVICE_FINAL) is the one-stage program"""
    part = disasm(*tpch.q1_plan(capi.TAB_LINEITEM_WIDE, capi.AGGSTAGE_PARTIAL))
    nosq = disasm(*tpch.q1_plan(capi.TAB_LINEITEM_WIDE, capi.AGGSTAGE_PARTIAL, flags=capi.AGGF_DEVICE_FINAL))
    assert sum(1 for ln in part if "OUTSQ" in ln) == 3 and not any("OUTSQ" in ln for ln in nosq)
    assert nosq == disasm(*tpch.q1_plan(capi.TAB_LINEITEM_WIDE, capi.AGGSTAGE_NORMAL))


def test_flattening_a_shared_and_chain_is_bounded():
    """a pool is a DAG: and(x, x) nested 60 deep would be 2^60 clauses if walked as a tree"""
    desc = make_desc([(capi.INT4OID, 4, 'i', 1)])
    p = ExprPool()
    q = p.func(capi.F_INT4GT, capi.BOOLOID, p.var(1, capi.INT4OID), p.const(capi.INT4OID, 0))
    for _ in range(60):
        q = p.boolop(capi.E_AND, q, q)
    with pytest.raises(capi.GGError) as e:
        disasm(capi.make_scan(desc, q), capi.make_agg(0, [], [(capi.AGG_COUNT_STAR, -1)]), p.pool)
    assert e.value.code == -6 and "too many clauses" in str(e.value)


def test_the_build_time_plan_cache_is_what_the_generator_writes(tmp_path):
    """csrc/plans/gg_plan_cache.cu holds the kernels specialised at build time for the registered plans; it is generated from the
    product's own compiler and source generator (scripts/gen_plan_cache.py) and must not lag behind them: a stale file would run
    yesterday's program for today's plan hash (the lookup compares program bytes, so it would simply stop hitting — and the bench
    would silently fall back to run-time compilation)."""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = tmp_path / "gg_plan_cache.cu"
    subprocess.check_call([sys.executable, os.path.join(root, "scripts", "gen_plan_cache.py"), str(out)], stdout=subprocess.DEVNULL)
    committed = open(os.path.join(root, "greengage_b200", "csrc", "plans", "gg_plan_cache.cu")).read()
    assert out.read_text() == committed
