"""A HashJoin with a target list on the host, no GPU: what the plan compiler makes of it (the probe's per-match piece claims a
row and writes one column per target; the build payload holds the inner columns the targets and the join qual read), what it
refuses, and how the executor-node surface treats such a join when linked against the stand-in device library
(tests/mock/ggb200_mock.c), which has no join that writes rows."""
import ctypes as C

import pytest

from _util import make_desc
from greengage_b200 import capi, executor as ex
from test_oracle_join import join_nodes

INT4 = (capi.INT4OID, 4, "i", 1)
F8 = (capi.FLOAT8OID, 8, "d", 1)
BP = (capi.BPCHAROID, -1, "i", 0)
NUM = (capi.NUMERICOID, -1, "i", 0)
ODESC = make_desc([INT4, BP, F8])
IDESC = make_desc([INT4, BP, INT4, F8, NUM])


def disasm(outer, inner, hj, targets, pool):
    L = capi.dev_lib()
    buf = C.create_string_buffer(1 << 16)
    t = (C.c_int32 * max(1, len(targets)))(*targets)
    n = L.gg_debug_disasm_joinrows(C.byref(outer), C.byref(inner), C.byref(hj), t, len(targets), C.byref(pool), buf, 1 << 16)
    if n < 0:
        raise capi.GGError(n, L.gg_last_error().decode())
    text = buf.value.decode()
    build, probe = text.split("-- probe")
    return build.splitlines(), probe.splitlines()


def test_probe_writes_one_row_of_the_targets_per_match():
    p, outer, inner, hj = join_nodes(ODESC, IDESC, capi.JOIN_LEFT, 1, True)      # join qual reads inner attribute 3
    expr = p.func(capi.F_FLOAT8MUL, capi.FLOAT8OID, p.var(3, capi.FLOAT8OID, 0), p.var(4, capi.FLOAT8OID, 1))
    targets = [p.var(1, capi.INT4OID, 0), p.var(2, capi.BPCHAROID, 1), expr]
    build, probe = disasm(outer, inner, hj, targets, p.pool)
    ops = [ln for ln in probe[1:] if ln.strip()]
    pc = int(probe[0].split("pc")[1].strip(" )"))
    tail = ops[pc:]
    # the per-match piece: the join qual FILTER, then GROUP (claim a row), then OUT0..OUT2 in target order, then END
    assert "FILTER" in " ".join(tail[:tail.index(next(ln for ln in tail if "GROUP" in ln))])
    g = next(i for i, ln in enumerate(tail) if "GROUP" in ln)
    outs = [ln for ln in tail[g:] if " OUT" in ln]
    assert [ln.split(" OUT")[1].split()[0] for ln in outs] == ["0", "1", "2"]
    assert tail[-1].split()[1] == "END" and not any(" KEY" in ln for ln in tail)
    # the build payload: exactly the inner columns read above the join (attributes 2, 3 and 4; not 5, the numeric)
    assert build[0].strip() == "-- build (payload 3)"
    assert sum(1 for ln in build[1:] if " OUT" in ln) == 3


def test_outer_only_targets_need_no_payload():
    p, outer, inner, hj = join_nodes(ODESC, IDESC, capi.JOIN_ANTI, 2, False)
    build, probe = disasm(outer, inner, hj, [p.var(3, capi.FLOAT8OID, 0)], p.pool)
    assert build[0].strip() == "-- build (payload 0)"
    assert sum(1 for ln in probe if " OUT" in ln) == 1


@pytest.mark.parametrize("case", ["numeric", "too_many", "none", "semi_inner", "anti_inner", "lasj_inner"])
def test_refusals(case):
    jt = {"semi_inner": capi.JOIN_SEMI, "anti_inner": capi.JOIN_ANTI, "lasj_inner": capi.JOIN_LASJ_NOTIN}.get(case, capi.JOIN_INNER)
    p, outer, inner, hj = join_nodes(ODESC, IDESC, jt, 1, False)
    targets = {"numeric": [p.var(1, capi.INT4OID, 0), p.var(5, capi.NUMERICOID, 1)],
               "too_many": [p.var(1, capi.INT4OID, 0)] * 17,
               "none": []}.get(case, [p.var(1, capi.INT4OID, 0), p.func(capi.F_INT4GT, capi.BOOLOID, p.var(3, capi.INT4OID, 1), p.const(capi.INT4OID, 0))])
    with pytest.raises(capi.GGError) as e:
        disasm(outer, inner, hj, targets, p.pool)
    assert e.value.code == -6                                         # GG_ERR_UNSUPPORTED
    msg = str(e.value)
    want = {"numeric": "numeric", "too_many": "17 columns", "none": "0 columns"}.get(case, "semi or anti join returns outer rows only")
    assert want in msg, msg


@pytest.fixture(scope="module")
def mock_exec(tmp_path_factory):
    """libggexec linked against the stand-in device library, bound in this process for the duration of the module"""
    from test_executor_multiseg import build_mock
    L = ex.bind(C.CDLL(build_mock(str(tmp_path_factory.mktemp("joinrows")))))
    L.mock_engine.restype = C.c_void_p
    saved, ex._lib = ex._lib, L
    yield L
    ex._lib = saved


def _join_plan(b, targets, p):
    p_, outer, inner, hj = join_nodes(ODESC, IDESC, capi.JOIN_INNER, 1, False) if p is None else p
    return b.hashjoin(b.seqscan(0, outer.desc), b.hash(b.seqscan(1, inner.desc)), hj, targets), p_


def test_executor_refuses_a_bare_join_without_targets_as_before(mock_exec):
    b = ex.PlanBuilder()
    plan, p = _join_plan(b, (), None)
    with pytest.raises(ex.ExecError) as e:
        ex.Executor(mock_exec.mock_engine(), p.pool, [None, None], plan)
    assert e.value.code == -6 and "only accelerated underneath an Agg (the join is never materialised)" in str(e.value)


def test_executor_with_targets_needs_the_device_entry_points(mock_exec):
    jp = join_nodes(ODESC, IDESC, capi.JOIN_INNER, 1, False)
    b = ex.PlanBuilder()
    plan, p = _join_plan(b, [jp[0].var(1, capi.INT4OID, 0)], jp)
    with pytest.raises(ex.ExecError) as e:
        ex.Executor(mock_exec.mock_engine(), p.pool, [None, None], plan)
    assert e.value.code == -6 and "no join that writes its rows" in str(e.value)
    # the same join under an Agg stays fused, targets or not: the refusal is about the relations, not the targets
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [], [(capi.AGG_COUNT_STAR, -1)])
    with pytest.raises(ex.ExecError) as e:
        ex.Executor(mock_exec.mock_engine(), p.pool, [None, None], b.agg(plan, agg))
    assert "no join that writes its rows" not in str(e.value)
