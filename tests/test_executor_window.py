"""The WindowAgg node through the executor-node surface on CPU: the product's host C linked against the oracle-backed stand-in for
the device library (tests/mock/ggb200_mock.c) and a stand-in for gg_window_* answered by the row-at-a-time reference
(tests/mock/ggb200_mock_window.c), one process per segment over gloo.  What runs for real is the node logic: the order check, the
descriptor of the rows below, the upload of host rows, the rows handed up to slots, a Limit, a Sort and another WindowAgg, ReScan,
squelch, Instrumentation, the refusals, and a WindowAgg above a Gather at 1-3 segments."""
import ctypes as C
import glob
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
RELATION_FNS = ("gg_relation_create", "gg_relation_attach_rows", "gg_relation_read", "gg_relation_device_ptr", "gg_relation_free",
                "gg_sort_datumrows")
ERR_UNSUPPORTED = -6


def build_window_mock(outdir):
    """(the executor over the stand-in with gg_window_*, the executor over the plain stand-in)"""
    sys.path.insert(0, HERE)
    from test_executor_multiseg import build_mock
    plain = build_mock(outdir)
    wdir = os.path.join(outdir, "window")
    os.makedirs(wdir, exist_ok=True)
    objs = []
    for src in glob.glob(os.path.join(outdir, "*.o")):
        if os.path.basename(src) != "ggb200_mock.c.o":
            objs.append(src)
    renames = ["-D%s=mockbase_%s" % (f, f[3:]) for f in RELATION_FNS]
    for src, extra in ((os.path.join(HERE, "mock", "ggb200_mock.c"), renames), (os.path.join(HERE, "mock", "ggb200_mock_window.c"), []),
                       (os.path.join(HERE, "window_ref.c"), [])):
        obj = os.path.join(wdir, os.path.basename(src) + ".o")
        subprocess.check_call(["gcc", "-O1", "-g", "-fPIC", "-Wall", "-Wextra", "-std=gnu11"] + extra + ["-c", src, "-o", obj])
        objs.append(obj)
    so = os.path.join(wdir, "libggexec_mock_window.so")
    subprocess.check_call(["g++", "-shared", "-o", so] + objs + ["-L", os.path.join(ROOT, "oracle"), "-lggoracle",
                                                                 "-Wl,-rpath," + os.path.join(ROOT, "oracle"), "-Wl,-z,defs", "-lm"])
    return so, plain


def _setup(mock):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    from greengage_b200 import executor as ex
    L = ex.bind(C.CDLL(mock))
    L.mock_engine.restype = C.c_void_p
    L.mock_relation.restype = C.c_void_p
    L.mock_relation.argtypes = [C.c_void_p, C.c_uint64]
    ex._lib = L
    return L, ex


def _funcs(capi, pool):
    price = pool.var(3, capi.FLOAT8OID)                               # the Agg's sum(extendedprice)
    return [(capi.WF_RANK, capi.INT8OID, []), (capi.WF_ROW_NUMBER, capi.INT8OID, []), (capi.AGG_SUM_FLOAT8, capi.FLOAT8OID, [price]),
            (capi.WF_LAG, capi.FLOAT8OID, [price]), (capi.WF_NTILE, capi.INT4OID, [pool.const(capi.INT4OID, 4)])]


def _words(rows, ncols):
    import numpy as np
    out = np.zeros((len(rows), 1 + ncols), dtype=np.uint64)
    for r, (vals, nulls) in enumerate(rows):
        for c in range(ncols):
            if nulls[c]:
                out[r, 0] |= np.uint64(1 << c)
            else:
                out[r, 1 + c] = np.uint64(vals[c] & 0xFFFFFFFFFFFFFFFF)
    return out


def _expected(win, types, pool, rows):
    import numpy as np
    from _window import ref_window
    rc, out, msg = ref_window(win, types, pool, _words(rows, len(types)))
    assert rc == 0, msg
    ncols = out.shape[1] - 1
    return [tuple(None if (int(r[0]) >> c) & 1 else int(np.uint64(r[1 + c]).view(np.int64)) for c in range(ncols)) for r in out]


def _tuples(x, limit=None):
    return [tuple(None if nl else v for v, nl in zip(vals, nulls)) for vals, nulls, ty, ln in x.rows(limit)]


def _nine(node):
    """a node that claims one function more than gg_window holds"""
    node.win.numFuncs = 9
    return node


def _single(mock):
    L, ex = _setup(mock)
    from greengage_b200 import capi
    from test_executor_limit import _li_agg
    from test_executor_multiseg import MockRel
    eng = L.mock_engine()
    li, scan, agg, p = _li_agg()
    rels = [MockRel(L, li)]
    types = [capi.INT8OID, capi.INT8OID, capi.FLOAT8OID]              # orderkey, count(*), sum(extendedprice)
    keys = [capi.make_sortkey(1, capi.INT8OID, desc=True), capi.make_sortkey(0, capi.INT8OID)]
    funcs = _funcs(capi, p)
    frame = capi.FRAMEOPTION_DEFAULTS
    done = []

    def plan(build):
        b = ex.PlanBuilder()
        return build(b, b.sort(b.agg(b.seqscan(0, scan.desc, scan.qual), agg), keys))

    x = ex.Executor(eng, p.pool, rels, plan(lambda b, s: s))
    srows = [(v, nl) for v, nl, ty, ln in x.rows()]
    x.end()
    want = _expected(capi.make_window([], [1], frame, funcs), types, p.pool, srows)
    x = ex.Executor(eng, p.pool, rels, plan(lambda b, s: b.windowagg(s, [], [1], frame, funcs)))
    assert _tuples(x) == want and len(want) > 4000
    ins = dict(x.instrumentation())
    assert x.kind() == "windowagg" and ins["windowagg"].ntuples == len(want) and ins["windowagg"].nloops == 1
    assert x.locations()[0] == ("windowagg", "host")                   # handed out through slots
    x.rescan()
    assert _tuples(x) == want and dict(x.instrumentation())["windowagg"].nloops == 2
    assert _tuples(x) == []
    x.end()
    done.append("over-sort-and-rescan")
    x = ex.Executor(eng, p.pool, rels, plan(lambda b, s: b.windowagg(s, [], [1], frame, funcs)))
    assert _tuples(x, 3) == want[:3]                                  # the caller stops after three rows: squelched
    assert _tuples(x) == []
    x.end()
    x = ex.Executor(eng, p.pool, rels, plan(lambda b, s: b.limit(b.windowagg(s, [], [1], frame, funcs), 7, 3)))
    assert _tuples(x) == want[3:10]
    ins = dict(x.instrumentation())
    assert ins["limit"].ntuples == 7 and ins["windowagg"].ntuples == 10
    x.end()
    done.append("squelch-and-limit")
    # stacked: PARTITION BY the first node's ntile, ORDER BY orderkey, through a Sort
    k2 = [capi.make_sortkey(7, capi.INT4OID), capi.make_sortkey(0, capi.INT8OID)]
    funcs2 = [(capi.AGG_COUNT_STAR, capi.INT8OID, []), (capi.WF_FIRST_VALUE, capi.INT8OID, [p.var(1, capi.INT8OID)])]
    x = ex.Executor(eng, p.pool, rels, plan(lambda b, s: b.sort(b.windowagg(s, [], [1], frame, funcs), k2)))
    mid = [(v, nl) for v, nl, ty, ln in x.rows()]
    x.end()
    want2 = _expected(capi.make_window([7], [0], frame, funcs2), types + [f[1] for f in funcs], p.pool, mid)
    x = ex.Executor(eng, p.pool, rels, plan(lambda b, s: b.windowagg(b.sort(b.windowagg(s, [], [1], frame, funcs), k2), [7], [0], frame, funcs2)))
    assert _tuples(x) == want2
    x.end()
    done.append("stacked")
    # refusals: each with its reason, at init
    value_offset = capi.FRAMEOPTION_NONDEFAULT | capi.FRAMEOPTION_ROWS | capi.FRAMEOPTION_BETWEEN | capi.FRAMEOPTION_START_VALUE_PRECEDING | \
        capi.FRAMEOPTION_END_CURRENT_ROW
    two = p.func(capi.F_FLOAT8PL, capi.FLOAT8OID, p.var(3, capi.FLOAT8OID), p.var(3, capi.FLOAT8OID))
    qual = p.func(capi.F_INT8EQ, capi.BOOLOID, p.var(5, capi.INT8OID), p.const(capi.INT8OID, 1))
    for what, build in (
            ("order", lambda b, s: b.windowagg(s, [0], [], frame, funcs)),
            ("frame", lambda b, s: b.windowagg(s, [], [1], value_offset, funcs)),
            ("numeric", lambda b, s: b.windowagg(s, [], [1], frame, [(capi.AGG_SUM_NUMERIC, capi.NUMERICOID, [p.var(3, capi.FLOAT8OID)])])),
            ("expression", lambda b, s: b.windowagg(s, [], [1], frame, [(capi.WF_LAG, capi.FLOAT8OID, [two])])),
            ("nine functions", lambda b, s: _nine(b.windowagg(s, [], [1], frame, (funcs * 2)[:8]))),
            ("qual without a row filter", lambda b, s: b.windowagg(s, [], [1], frame, funcs, qual=qual))):
        with pytest.raises(ex.ExecError) as e:
            ex.Executor(eng, p.pool, rels, plan(build))
        assert e.value.code == ERR_UNSUPPORTED, (what, str(e.value))
    done.append("refusals")
    return done


def _refused(mock):
    L, ex = _setup(mock)
    from greengage_b200 import capi
    from test_executor_limit import _li_agg
    from test_executor_multiseg import MockRel
    eng = L.mock_engine()
    li, scan, agg, p = _li_agg()
    b = ex.PlanBuilder()
    s = b.sort(b.agg(b.seqscan(0, scan.desc, scan.qual), agg), [capi.make_sortkey(1, capi.INT8OID)])
    try:
        ex.Executor(eng, p.pool, [MockRel(L, li)], b.windowagg(s, [], [1], capi.FRAMEOPTION_DEFAULTS, _funcs(capi, p)))
        return ("accepted",)
    except ex.ExecError as e:
        return (e.code, "no window functions" in str(e))


def _worker(rank, world, port, mock, case, q):
    try:
        dist = None
        if world > 1:
            os.environ["MASTER_ADDR"] = "127.0.0.1"
            os.environ["MASTER_PORT"] = str(port)
            import torch.distributed as dist
            dist.init_process_group("gloo", rank=rank, world_size=world)
        if case == "single":
            q.put(("ok", rank, _single(mock)))
            return
        if case == "refused":
            q.put(("ok", rank, _refused(mock)))
            return
        L, ex = _setup(mock)
        from greengage_b200 import capi
        from test_executor_limit import _li_agg
        from test_executor_multiseg import MockRel
        eng = L.mock_engine()
        li, scan, agg, p = _li_agg(rank, world)
        keys = [capi.make_sortkey(1, capi.INT8OID, desc=True), capi.make_sortkey(0, capi.INT8OID)]
        funcs = _funcs(capi, p)
        tr = ex.TorchTransport() if world > 1 else None

        def run(top):
            b = ex.PlanBuilder()
            s = b.sort(b.motion(b.agg(b.seqscan(0, scan.desc, scan.qual), agg), ex.MOTION_GATHER, [], 1), keys)
            x = ex.Executor(eng, p.pool, [MockRel(L, li)], top(b, s), nsegs=world, segindex=rank, transport=tr)
            rows = [(v, nl) for v, nl, ty, ln in x.rows()]
            again = None
            if top is not None:
                x.rescan()
                again = _tuples(x)
            x.end()
            return rows, again

        srows, _ = run(lambda b, s: s)
        got, again = run(lambda b, s: b.windowagg(s, [], [1], capi.FRAMEOPTION_DEFAULTS, funcs))
        want = _expected(capi.make_window([], [1], capi.FRAMEOPTION_DEFAULTS, funcs), [capi.INT8OID, capi.INT8OID, capi.FLOAT8OID], p.pool, srows) \
            if srows else []
        got = [tuple(None if n else v for v, n in zip(vals, nl)) for vals, nl in got]
        q.put(("ok", rank, (len(srows), got == want, again == want)))
        if dist is not None:
            dist.destroy_process_group()
    except Exception:  # pragma: no cover
        import traceback
        q.put(("err", rank, traceback.format_exc()))


def _run(world, case, tmp_path):
    import torch.multiprocessing as mp
    window, plain = build_window_mock(str(tmp_path))
    mock = plain if case == "refused" else window
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29870 + (os.getpid() * 7 + world * 13 + len(case)) % 40
    procs = [ctx.Process(target=_worker, args=(r, world, port, mock, case, q)) for r in range(world)]
    for pr in procs:
        pr.start()
    res = [q.get(timeout=300) for _ in procs]
    for pr in procs:
        pr.join(timeout=60)
    for r in res:
        assert r[0] == "ok", r[2]
    return {r[1]: r[2] for r in res}


def test_window_node_on_one_segment(tmp_path):
    assert _run(1, "single", tmp_path)[0] == ["over-sort-and-rescan", "squelch-and-limit", "stacked", "refusals"]


def test_a_library_without_window_functions_refuses_the_node(tmp_path):
    from greengage_b200 import capi
    assert _run(1, "refused", tmp_path)[0] == (ERR_UNSUPPORTED, True)


@pytest.mark.parametrize("world", [1, 2, 3])
def test_window_above_a_gather(world, tmp_path):
    res = _run(world, "gather", tmp_path)
    # the receiving segment windows every group; the others yield nothing
    assert res[0][0] > 4000 and res[0][1] and res[0][2]
    for r in range(1, world):
        assert res[r] == (0, True, True)
