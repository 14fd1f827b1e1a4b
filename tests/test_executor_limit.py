"""The Limit node and the bounded Sort below it, through the executor-node surface on CPU: the product's host C linked
against the oracle-backed stand-in for the device library (tests/mock/ggb200_mock.c), one process per segment over gloo.
What runs for real is the node logic: recompute_limits / the window (nodeLimit.c:44-230, 258), pass_down_bound (:345), the
bounded Sort over host rows in memory and through external runs, the squelch of what lies below, and the preliminary-limit
plan of the MPP planner (Limit <- Gather Motion(merge) <- Limit <- Sort <- Agg, planner.c:5829) at 1-3 segments."""
import ctypes as C
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def _li_agg(seg=0, nsegs=1):
    """LI-narrow (hash-distributed on the order key) and `orderkey, count(*), sum(extendedprice) GROUP BY orderkey`"""
    from greengage_b200 import capi, tpch
    li, _, _ = tpch.synth_generate(tpch.synth_spec(capi.TAB_LINEITEM_NARROW, 30_000, seed=6, norders=6_000, nsegs=nsegs, seg=seg,
                                                   policy=capi.DIST_HASH), nthreads=1)
    p = capi.ExprPool()
    c = tpch.LI_NARROW_COLS
    okey, price = p.var(c["orderkey"], capi.INT8OID), p.var(c["extendedprice"], capi.FLOAT8OID)
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [okey], [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_FLOAT8, price)], num_groups=6000)
    return li, capi.make_scan(capi.synth_tupdesc(capi.TAB_LINEITEM_NARROW), -1), agg, p


def _keys(total):
    from greengage_b200 import capi
    if total:                                        # count DESC, orderkey: a total order
        return [capi.make_sortkey(1, capi.INT8OID, desc=True), capi.make_sortkey(0, capi.INT8OID)]
    return [capi.make_sortkey(1, capi.INT8OID)]      # count only: heavy ties, kept in input order


def _setup(mock):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    from greengage_b200 import executor as ex
    L = ex.bind(C.CDLL(mock))
    L.mock_engine.restype = C.c_void_p
    L.mock_relation.restype = C.c_void_p
    L.mock_relation.argtypes = [C.c_void_p, C.c_uint64]
    L.GgExecSortRuns.argtypes = [C.c_void_p]
    ex._lib = L
    return L, ex


def _single(mock):
    L, ex = _setup(mock)
    from greengage_b200 import capi
    from test_executor_multiseg import MockRel
    eng = L.mock_engine()
    li, scan, agg, p = _li_agg()
    done = []

    def run(build, mem=0):
        b = ex.PlanBuilder()
        x = ex.Executor(eng, p.pool, [MockRel(L, li)], build(b, b.agg(b.seqscan(0, scan.desc, scan.qual), agg)), operator_mem=mem)
        rows = [tuple(v) for v, nl, ty, ln in x.rows()]
        return x, rows

    for total in (True, False):
        keys = _keys(total)
        x, full = run(lambda b, a: b.sort(a, keys))
        x.end()
        n = len(full)
        assert n > 4000
        for count, offset in ((10, None), (5, 3), (1, 0), (0, None), (0, 7), (None, None), (None, 100), (7, n - 3), (7, n + 5),
                              (n, 0), (n + 10, 1)):
            x, rows = run(lambda b, a: b.limit(b.sort(a, keys), count, offset))
            o = offset or 0
            want = full[o:] if count is None else full[o:o + count]
            assert rows == want, (total, count, offset)
            ins = dict(x.instrumentation())
            assert x.kind() == "limit" and ins["limit"].ntuples == len(want)
            # the Sort handed up only what the window needed: never more than the bound (and nothing for an empty window)
            bound = n if count is None else min(n, count + o)
            assert ins["sort"].ntuples == (0 if count == 0 else bound), (count, offset, ins["sort"].ntuples)
            x.rescan()                                        # ReScan: the limits are recomputed, the same rows come back
            assert [tuple(v) for v, nl, ty, ln in x.rows()] == want
            assert dict(x.instrumentation())["limit"].nloops == 2
            x.end()
        done.append("window-total" if total else "window-ties")
        # host rows beyond the operator's memory (16 KB: 420 rows a run): a bound that fits sorts once without runs; one that
        # does not keeps the external path, each run bounded, the merge stopped after `bound` rows
        for count, offset, ext in ((10, 5, False), (400, 0, False), (2000, 100, True), (None, 10, True)):
            x, rows = run(lambda b, a: b.limit(b.sort(a, keys), count, offset), mem=16 * 1024)
            o = offset or 0
            assert rows == (full[o:] if count is None else full[o:o + count]), (count, offset)
            sort_state = L.GgExecOuterPlanState(x.state)
            runs = L.GgExecSortRuns(sort_state)
            assert (runs >= 10) if ext else (runs == 1), (count, offset, runs)
            assert dict(x.instrumentation())["sort"].sort_runs == runs
            x.end()
        done.append("external-total" if total else "external-ties")
    keys = _keys(True)
    x, full = run(lambda b, a: b.sort(a, keys))
    x.end()
    # the bound reaches a Sort directly below only: through a Motion the Sort sorts everything (external under 16 KB); a
    # count + offset that overflows is no bound
    for count, offset, through_motion, bounded in ((10, None, False, True), (10, None, True, False), (2 ** 62, 2 ** 62, False, False),
                                                   (2 ** 63 - 1, 5, False, False)):
        def build(b, a):
            s = b.sort(a, keys)
            return b.limit(b.motion(s, ex.MOTION_GATHER, [], 1) if through_motion else s, count, offset)
        x, rows = run(build, mem=16 * 1024)
        o = offset or 0
        assert rows == full[o:o + count], (count, offset)
        sort_runs = dict(x.instrumentation())["sort"].sort_runs
        assert (sort_runs == 1) if bounded else (sort_runs >= 10), (count, offset, through_motion, sort_runs)
        x.end()
    done.append("bound-only-to-sort")
    # a Limit over an Agg (no ORDER BY) or over a Motion: the window of whatever order the node below hands up
    x, plain = run(lambda b, a: a)
    x.end()
    for build in (lambda b, a: b.limit(a, 25, 40), lambda b, a: b.limit(b.motion(a, ex.MOTION_GATHER, [], 1), 25, 40)):
        x, rows = run(build)
        assert rows == plain[40:65]
        x.end()
    done.append("limit-over-agg-and-motion")
    # negative values: the reference's errors
    for count, offset, msg in ((-1, None, "LIMIT must not be negative"), (5, -2, "OFFSET must not be negative")):
        b = ex.PlanBuilder()
        x = ex.Executor(eng, p.pool, [MockRel(L, li)], b.limit(b.sort(b.agg(b.seqscan(0, scan.desc, scan.qual), agg), keys), count, offset))
        with pytest.raises(ex.ExecError) as e:
            x.rows()
        assert e.value.code == -10 and msg in str(e.value)
        x.end()
    done.append("negative")
    # the bounded host-row sort itself: the prefix of the whole sort's permutation
    import numpy as np
    rng = np.random.default_rng(3)
    vals = np.stack([rng.integers(0, 20, 5000), rng.integers(-10 ** 9, 10 ** 9, 5000)], axis=1).astype(np.int64)
    nulls = (rng.random(vals.shape) < 0.1).astype(np.uint8)
    ka = (capi.gg_sortkey * 2)(capi.make_sortkey(0, capi.INT8OID, desc=True), capi.make_sortkey(1, capi.INT8OID, nulls_first=True))
    L.gg_sort_rows.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]
    L.gg_sort_rows_bounded.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p,
                                       C.POINTER(C.c_uint64)]
    whole = np.zeros(5000, dtype=np.uint64)
    assert L.gg_sort_rows(eng, ka, 2, 2, vals.ctypes.data, nulls.ctypes.data, 5000, whole.ctypes.data) == 0
    for bound in (0, 1, 7, 1000, 4999, 5000, 9000):
        part, cnt = np.zeros(5000, dtype=np.uint64), C.c_uint64(99)
        assert L.gg_sort_rows_bounded(eng, ka, 2, 2, vals.ctypes.data, nulls.ctypes.data, 5000, bound, part.ctypes.data, C.byref(cnt)) == 0
        assert cnt.value == min(bound, 5000) and np.array_equal(part[:cnt.value], whole[:cnt.value])
    done.append("bounded-perm")
    return done


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
        from test_executor_multiseg import MockRel
        eng = L.mock_engine()
        li, scan, agg, p = _li_agg(rank, world)
        keys = _keys(True)
        count, offset = (5, None) if case == "limit0" else (12, 3)
        b = ex.PlanBuilder()
        # the reference's MPP plan of ORDER BY ... LIMIT c OFFSET o: every segment sorts and keeps its first c + o rows, the
        # Gather merges them on segment 0, the top Limit cuts the window (limit0: LIMIT 0 there, on segment 0 only)
        sorted_rows = b.sort(b.agg(b.seqscan(0, scan.desc, scan.qual), agg), keys)
        gather = b.motion(b.limit(sorted_rows, count + (offset or 0)), ex.MOTION_GATHER, [], 1, merge_keys=keys)
        plan = b.limit(gather, 0 if (case == "limit0" and rank == 0) else count, offset)
        x = ex.Executor(eng, p.pool, [MockRel(L, li)], plan, nsegs=world, segindex=rank, transport=ex.TorchTransport() if world > 1 else None)
        rows = [tuple(v) for v, nl, ty, ln in x.rows()]
        again = None
        if case == "mpp":
            x.rescan()                                        # every segment takes part in the rescan's exchange
            again = [tuple(v) for v, nl, ty, ln in x.rows()]
        x.end()
        q.put(("ok", rank, (rows, again)))
        if dist is not None:
            dist.destroy_process_group()
    except Exception:  # pragma: no cover
        import traceback
        q.put(("err", rank, traceback.format_exc()))


def _refused(mock):
    """the stand-in without the bounded sorts: a Limit over a Sort is refused at init (the caller keeps its CPU nodes), a Limit
    over an Agg still runs"""
    L, ex = _setup(mock)
    from test_executor_multiseg import MockRel
    eng = L.mock_engine()
    li, scan, agg, p = _li_agg()
    b = ex.PlanBuilder()
    try:
        ex.Executor(eng, p.pool, [MockRel(L, li)], b.limit(b.sort(b.agg(b.seqscan(0, scan.desc, scan.qual), agg), _keys(True)), 5))
        return ("accepted",)
    except ex.ExecError as e:
        refused = (e.code, "bounded sort" in str(e))
    b = ex.PlanBuilder()
    x = ex.Executor(eng, p.pool, [MockRel(L, li)], b.limit(b.agg(b.seqscan(0, scan.desc, scan.qual), agg), 5))
    n = len(x.rows())
    x.end()
    return refused, n


def build_topn_mock(outdir):
    """the executor linked against the oracle-backed stand-in plus its bounded sorts (tests/mock/ggb200_mock_topn.c)"""
    import glob
    import subprocess
    from test_executor_multiseg import build_mock
    plain = build_mock(outdir)                      # compiles the objects of the stand-in (and links it without the bounded sorts)
    obj = os.path.join(outdir, "ggb200_mock_topn.c.o")
    subprocess.check_call(["gcc", "-O1", "-g", "-fPIC", "-Wall", "-Wextra", "-std=gnu11", "-c",
                           os.path.join(HERE, "mock", "ggb200_mock_topn.c"), "-o", obj])
    so = os.path.join(outdir, "libggexec_mock_topn.so")
    subprocess.check_call(["g++", "-shared", "-o", so] + sorted(glob.glob(os.path.join(outdir, "*.o"))) +
                          ["-L", os.path.join(ROOT, "oracle"), "-lggoracle", "-Wl,-rpath," + os.path.join(ROOT, "oracle"), "-Wl,-z,defs", "-lm"])
    return so, plain


def _run(world, case, tmp_path):
    import torch.multiprocessing as mp
    topn, plain = build_topn_mock(str(tmp_path))
    mock = plain if case == "refused" else topn
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29950 + (os.getpid() * 7 + world * 13 + len(case)) % 40
    procs = [ctx.Process(target=_worker, args=(r, world, port, mock, case, q)) for r in range(world)]
    for pr in procs:
        pr.start()
    res = [q.get(timeout=300) for _ in procs]
    for pr in procs:
        pr.join(timeout=60)
    for r in res:
        assert r[0] == "ok", r[2]
    return {r[1]: r[2] for r in res}


def test_limit_window_bound_and_external_sort_on_one_segment(tmp_path):
    """OFFSET past the end, LIMIT 0, LIMIT ALL, negative values, the bound reaching only a Sort, the bounded sort in memory and
    through external runs, the Sort's Instrumentation, ReScan"""
    by = _run(1, "single", tmp_path)
    assert by[0] == ["window-total", "external-total", "window-ties", "external-ties", "bound-only-to-sort",
                     "limit-over-agg-and-motion", "negative", "bounded-perm"]


@pytest.mark.parametrize("world", [1, 2, 3])
def test_preliminary_limit_under_a_gather_gives_the_top_n(world, tmp_path):
    """Limit <- Gather Motion(merge) <- Limit <- Sort <- Agg over hash-distributed segments: segment 0 returns rows 3..14 of
    the whole table's order, the others nothing; a ReScan returns the same rows"""
    sys.path.insert(0, ROOT)
    from oracle import pyoracle as po
    by = _run(world, "mpp", tmp_path)
    li, scan, agg, p = _li_agg()
    want = po.seqscan_agg(scan, agg, p.pool, li, cap=65536)[0]
    want = sorted(((r.key[0], r.agg[0].i) for r in want), key=lambda t: (-t[1], t[0]))[3:15]
    rows, again = by[0]
    assert [(r[0], r[1]) for r in rows] == want and again == rows
    for r in range(1, world):
        assert by[r] == ([], [])


def test_limit_over_a_sort_is_refused_without_the_bounded_sorts(tmp_path):
    """a device library without gg_sort_rows_bounded / gg_sort_datumrows_bounded: GG_ERR_UNSUPPORTED at init for Limit <- Sort,
    never another sort in their place; a Limit over an Agg needs neither and runs"""
    by = _run(1, "refused", tmp_path)
    assert by[0] == ((-6, True), 5)


def test_limit_zero_on_the_receiver_still_finishes_every_segment(tmp_path):
    """LIMIT 0 on segment 0 over the Gather: its Limit never runs the child, but the squelch runs the Motion there, so the
    senders are not left in the exchange and every segment finishes"""
    by = _run(2, "limit0", tmp_path)
    assert by[0] == ([], None) and by[1] == ([], None)
