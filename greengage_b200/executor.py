"""ctypes mirror of include/gg_executor.h (libggexec.so): plan-tree builders and the node-at-a-time driver.

This is the stub a test or bench uses in place of the C module of INTEGRATION.md: it builds the GgPlan tree a
Postgres-side translator would build, calls GgExecInitNode / GgExecProcNode / GgExecEndNode, and (for more than
one segment) plugs a torch.distributed transport under the Motion nodes.
"""
import ctypes as C
import os

import numpy as np

from . import capi

_HERE = os.path.dirname(os.path.abspath(__file__))
T_SeqScan, T_Agg, T_Hash, T_HashJoin, T_Sort, T_Motion, T_Limit, T_WindowAgg = 1, 2, 3, 4, 5, 6, 7, 8
MOTION_GATHER, MOTION_HASH, MOTION_BROADCAST = 0, 1, 2
GG_MAX_SORTKEYS = 4
GG_MAX_OUTCOLS = capi.GG_MAX_KEYS + 3 * capi.GG_MAX_AGGS
GG_MAX_RELATIONS = 16


class GgPlan(C.Structure):
    pass


GgPlan._fields_ = [("type", C.c_int), ("lefttree", C.POINTER(GgPlan)), ("righttree", C.POINTER(GgPlan)), ("qual", C.c_int32)]


class GgSeqScan(C.Structure):
    _fields_ = [("plan", GgPlan), ("scanrelid", C.c_int32), ("desc", capi.gg_tupdesc),
                ("numTargets", C.c_int32), ("targets", C.c_int32 * GG_MAX_OUTCOLS)]


class GgAgg(C.Structure):
    _fields_ = [("plan", GgPlan), ("agg", capi.gg_agg)]


class GgHash(C.Structure):
    _fields_ = [("plan", GgPlan)]


class GgHashJoin(C.Structure):
    _fields_ = [("plan", GgPlan), ("hj", capi.gg_hashjoin), ("numTargets", C.c_int32), ("targets", C.c_int32 * GG_MAX_OUTCOLS)]


class GgSort(C.Structure):
    _fields_ = [("plan", GgPlan), ("numCols", C.c_int32), ("keys", capi.gg_sortkey * GG_MAX_SORTKEYS)]


class GgMotion(C.Structure):
    _fields_ = [("plan", GgPlan), ("motionType", C.c_int32), ("numHashCols", C.c_int32),
                ("hashCol", C.c_int32 * capi.GG_MAX_KEYS), ("motionID", C.c_int32),
                ("numSortCols", C.c_int32), ("sortKeys", capi.gg_sortkey * GG_MAX_SORTKEYS)]


class GgLimit(C.Structure):
    _fields_ = [("plan", GgPlan), ("hasOffset", C.c_int32), ("hasCount", C.c_int32), ("limitOffset", C.c_int64),
                ("limitCount", C.c_int64)]


class GgWindowAgg(C.Structure):
    _fields_ = [("plan", GgPlan), ("win", capi.gg_window)]


class GgTupleTableSlot(C.Structure):
    _fields_ = [("tts_nvalid", C.c_int32), ("tts_isempty", C.c_int32), ("tts_values", C.c_int64 * GG_MAX_OUTCOLS),
                ("tts_isnull", C.c_uint8 * GG_MAX_OUTCOLS), ("tts_typid", C.c_int32 * GG_MAX_OUTCOLS),
                ("tts_len", C.c_int32 * GG_MAX_OUTCOLS)]


class GgInstrumentation(C.Structure):
    _fields_ = [("ntuples", C.c_double), ("nloops", C.c_double), ("kernel_ms", C.c_float), ("sort_runs", C.c_int32),
                ("hash_batches", C.c_int32), ("pad", C.c_int32)]


class GgRowBatch(C.Structure):
    _fields_ = [("ncols", C.c_int32), ("nrows", C.c_int64), ("values", C.POINTER(C.c_int64)), ("isnull", C.POINTER(C.c_uint8))]


EXCHANGE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.c_int, C.POINTER(GgRowBatch), C.POINTER(C.c_int32), C.POINTER(GgRowBatch))


class GgMotionTransport(C.Structure):
    _fields_ = [("ctx", C.c_void_p), ("exchange", EXCHANGE_FN)]


class GgEState(C.Structure):
    _fields_ = [("engine", C.c_void_p), ("pool", C.POINTER(capi.gg_exprpool)), ("relations", C.c_void_p * GG_MAX_RELATIONS),
                ("nsegs", C.c_int32), ("segindex", C.c_int32), ("transport", C.POINTER(GgMotionTransport)),
                ("es_processed", C.c_uint64), ("interconnect", C.c_void_p),
                ("host_pages", C.c_void_p * GG_MAX_RELATIONS), ("host_nblocks", C.c_uint64 * GG_MAX_RELATIONS),
                ("motion_on_host", C.c_int32), ("pad", C.c_int32), ("es_operator_mem", C.c_uint64),
                ("es_snapshot", C.POINTER(capi.gg_snapshot))]


_lib = None


def exec_lib():
    """libggexec.so.  Loading needs no GPU; running a plan does."""
    global _lib
    if _lib is None:
        path = os.path.join(_HERE, "libggexec.so")
        if not os.path.exists(path):
            raise ImportError("greengage_b200/libggexec.so is not built: run `python -c 'import __graft_entry__ as g; g.build()'`")
        capi.dev_lib()
        _lib = bind(C.CDLL(path))
    return _lib


def bind(L):
    """ctypes signatures of include/gg_executor.h on a loaded library"""
    L.GgExecInitNode.restype = C.c_void_p
    L.GgExecInitNode.argtypes = [C.POINTER(GgPlan), C.POINTER(GgEState), C.c_int]
    L.GgExecProcNode.restype = C.POINTER(GgTupleTableSlot)
    L.GgExecProcNode.argtypes = [C.c_void_p]
    L.GgExecEndNode.restype = None
    L.GgExecEndNode.argtypes = [C.c_void_p]
    L.GgExecReScan.argtypes = [C.c_void_p]
    L.GgExecSquelchNode.restype = None
    L.GgExecSquelchNode.argtypes = [C.c_void_p]
    L.GgExecLastError.restype = C.c_char_p
    L.GgExecLastErrorCode.restype = C.c_int
    L.GgExecNodeKind.restype = C.c_char_p
    L.GgExecNodeKind.argtypes = [C.c_void_p]
    L.GgExecNodeResultLocation.restype = C.c_char_p
    L.GgExecNodeResultLocation.argtypes = [C.c_void_p]
    L.GgExecPipelineKernelMs.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_float)]
    L.GgExecOuterPlanState.restype = C.c_void_p
    L.GgExecOuterPlanState.argtypes = [C.c_void_p]
    L.GgExecInnerPlanState.restype = C.c_void_p
    L.GgExecInnerPlanState.argtypes = [C.c_void_p]
    return L


class ExecError(capi.GGError):
    pass


def _as_plan(node):
    return C.cast(C.pointer(node), C.POINTER(GgPlan))


class PlanBuilder:
    """Keeps the ctypes nodes alive while the tree is in use."""

    def __init__(self):
        self.nodes = []

    def _keep(self, n):
        self.nodes.append(n)
        return n

    def seqscan(self, scanrelid, desc, qual=-1, targets=()):
        """targets: expression roots the scan projects (rows stay on the device for the node above); () = fused"""
        n = self._keep(GgSeqScan())
        n.plan.type, n.plan.qual, n.scanrelid = T_SeqScan, qual, scanrelid
        C.memmove(C.byref(n.desc), C.byref(desc), C.sizeof(capi.gg_tupdesc))
        n.numTargets = len(targets)
        for i, t in enumerate(targets):
            n.targets[i] = t
        return n

    def agg(self, child, agg, having=-1):
        """having: the HAVING qual's expression root (Vars varno 0, varattno = 1-based output column of the Agg: grouping keys,
        then one per aggregate); -1 = none"""
        n = self._keep(GgAgg())
        n.plan.type, n.plan.qual, n.plan.lefttree = T_Agg, having, _as_plan(child)
        C.memmove(C.byref(n.agg), C.byref(agg), C.sizeof(capi.gg_agg))
        return n

    def hash(self, child):
        n = self._keep(GgHash())
        n.plan.type, n.plan.qual, n.plan.lefttree = T_Hash, -1, _as_plan(child)
        return n

    def hashjoin(self, outer, hashnode, hj, targets=()):
        """targets: expression roots the join projects (varno 0 outer, 1 inner; its rows stay on the device for the node
        above); () = fused with the Agg above"""
        n = self._keep(GgHashJoin())
        n.plan.type, n.plan.qual, n.plan.lefttree, n.plan.righttree = T_HashJoin, -1, _as_plan(outer), _as_plan(hashnode)
        C.memmove(C.byref(n.hj), C.byref(hj), C.sizeof(capi.gg_hashjoin))
        n.numTargets = len(targets)
        for i, t in enumerate(targets):
            n.targets[i] = t
        return n

    def sort(self, child, keys):
        n = self._keep(GgSort())
        n.plan.type, n.plan.qual, n.plan.lefttree, n.numCols = T_Sort, -1, _as_plan(child), len(keys)
        for i, k in enumerate(keys):
            n.keys[i] = k
        return n

    def limit(self, child, count=None, offset=None):
        """LIMIT count OFFSET offset; None = LIMIT ALL / no OFFSET (the translator's evaluated constants)"""
        n = self._keep(GgLimit())
        n.plan.type, n.plan.qual, n.plan.lefttree = T_Limit, -1, _as_plan(child)
        n.hasCount, n.limitCount = (0, 0) if count is None else (1, count)
        n.hasOffset, n.limitOffset = (0, 0) if offset is None else (1, offset)
        return n

    def windowagg(self, child, part, ord, frame, funcs, qual=-1):
        """WindowAgg over `child` (a Sort on the partition columns, then the order columns): part / ord are 0-based columns of
        the child's rows, frame the FRAMEOPTION_* bits, funcs (winfnoid, wintype, [arg roots]) each; qual: a SubqueryScan's qual
        over the output row (the child's columns, then one per function; Vars varno 0, 1-based), -1 = none"""
        n = self._keep(GgWindowAgg())
        n.plan.type, n.plan.qual, n.plan.lefttree = T_WindowAgg, qual, _as_plan(child)
        w = capi.make_window(part, ord, frame, funcs)
        C.memmove(C.byref(n.win), C.byref(w), C.sizeof(capi.gg_window))
        return n

    def motion(self, child, motion_type, hash_cols=(), motion_id=1, merge_keys=()):
        n = self._keep(GgMotion())
        n.plan.type, n.plan.qual, n.plan.lefttree = T_Motion, -1, _as_plan(child)
        n.motionType, n.numHashCols, n.motionID = motion_type, len(hash_cols), motion_id
        for i, c in enumerate(hash_cols):
            n.hashCol[i] = c
        n.numSortCols = len(merge_keys)                 # sendSorted: the receiver merges on these keys
        for i, k in enumerate(merge_keys):
            n.sortKeys[i] = k
        return n


class Executor:
    """One slice on one segment: ExecInitNode at construction, rows() drives ExecProcNode to end of stream."""

    def __init__(self, eng, pool, relations, plan, nsegs=1, segindex=0, transport=None, interconnect=None, operator_mem=0, snapshot=None):
        """relations[i]: a device-resident Relation, or (host address, nblocks) for pages in host memory, or None"""
        L = exec_lib()
        self.es = GgEState()
        self.es.es_operator_mem = int(operator_mem)
        self._snapshot = snapshot                       # capi.make_snapshot(...): kept alive with the executor
        if snapshot is not None:
            self.es.es_snapshot = C.pointer(snapshot)
        self.es.engine = eng.h if hasattr(eng, "h") else eng
        self._pool = pool
        self.es.pool = C.pointer(pool)
        for i, r in enumerate(relations):
            if isinstance(r, tuple):
                self.es.host_pages[i], self.es.host_nblocks[i] = r
            else:
                self.es.relations[i] = r.h if r is not None else None
        if interconnect is not None:
            self.es.interconnect = interconnect.h if hasattr(interconnect, "h") else interconnect
        self.es.nsegs, self.es.segindex = nsegs, segindex
        self._transport = transport
        if transport is not None:
            self.es.transport = C.pointer(transport.struct)
        self._plan = plan
        self.state = L.GgExecInitNode(_as_plan(plan), C.byref(self.es), 0)
        if not self.state:
            raise ExecError(L.GgExecLastErrorCode(), L.GgExecLastError().decode("utf-8", "replace"))

    def kind(self):
        return exec_lib().GgExecNodeKind(self.state).decode()

    def locations(self):
        """[(node kind, where its result lives)] from the top node down the outer children"""
        L = exec_lib()
        out, st = [], self.state
        while st:
            out.append((L.GgExecNodeKind(st).decode(), L.GgExecNodeResultLocation(st).decode()))
            st = L.GgExecOuterPlanState(st)
        return out

    def instrumentation(self):
        """[(node kind, GgInstrumentation)] from the top node down the outer children: what EXPLAIN ANALYZE would print"""
        L = exec_lib()
        L.GgExecNodeInstrumentation.argtypes = [C.c_void_p, C.POINTER(GgInstrumentation)]
        out, st = [], self.state
        while st:
            ins = GgInstrumentation()
            capi.check(L.GgExecNodeInstrumentation(st, C.byref(ins)))
            out.append((L.GgExecNodeKind(st).decode(), ins))
            st = L.GgExecOuterPlanState(st)
        return out

    def kernel_ms(self):
        """(scan/probe kernel ms since the last rescan, launches, kernel variant, join build ms) of the slice's pipeline"""
        ms, n, v, b = C.c_float(0), C.c_int(0), C.c_int(0), C.c_float(0)
        capi.check(exec_lib().GgExecPipelineKernelMs(self.state, C.byref(ms), C.byref(n), C.byref(v), C.byref(b)))
        return ms.value, n.value, v.value, b.value

    def drain(self):
        """ExecProcNode to end of stream without building Python rows; returns the row count (benchmarks)"""
        L = exec_lib()
        n = 0
        while L.GgExecProcNode(self.state):
            n += 1
        code = L.GgExecLastErrorCode()
        if code:
            raise ExecError(code, L.GgExecLastError().decode("utf-8", "replace"))
        return n

    def rows(self, limit=None):
        """[(values, isnull, typids, lens)] one per ExecProcNode call"""
        L = exec_lib()
        out = []
        while limit is None or len(out) < limit:
            slot = L.GgExecProcNode(self.state)
            if not slot:
                code = L.GgExecLastErrorCode()
                if code:
                    raise ExecError(code, L.GgExecLastError().decode("utf-8", "replace"))
                break
            s = slot.contents
            n = s.tts_nvalid
            out.append((list(s.tts_values[:n]), list(s.tts_isnull[:n]), list(s.tts_typid[:n]), list(s.tts_len[:n])))
        if limit is not None and len(out) >= limit:
            L.GgExecSquelchNode(self.state)
        return out

    def rescan(self):
        capi.check(exec_lib().GgExecReScan(self.state))

    def end(self):
        if self.state:
            exec_lib().GgExecEndNode(self.state)
            self.state = None


class TorchTransport:
    """The interconnect under Motion nodes: count exchange + all-to-all-v of fixed-width rows over one
    torch.distributed communicator with rank = segment (NCCL over NVLink on the GPU box, gloo in CPU tests).
    Replaces the UDP interconnect's send/receive loops (cdbmotion.c:378-532, ic_udpifc.c); end of stream is the
    completion of the collective."""

    def __init__(self, device=None, group=None):
        import torch.distributed as dist
        self.device, self.group = device, group
        self.nsegs = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        self._libc = C.CDLL(None)
        self._libc.malloc.restype = C.c_void_p
        self._libc.malloc.argtypes = [C.c_size_t]
        self._cb = EXCHANGE_FN(self._exchange)
        self.struct = GgMotionTransport()
        self.struct.ctx = None
        self.struct.exchange = self._cb
        self.error = None

    def exchange_arrays(self, values, isnull, dest, motion_type):
        """values [n][ncols] int64, isnull [n][ncols] uint8, dest [n] int32 (-1 = every segment) -> received arrays"""
        import torch
        import torch.distributed as dist
        n, ncols = values.shape
        rec = np.zeros((n, ncols * 9), dtype=np.uint8)           # one record = ncols Datums + ncols null bytes
        rec[:, :ncols * 8] = values.view(np.uint8).reshape(n, ncols * 8)
        rec[:, ncols * 8:] = isnull
        if motion_type == MOTION_BROADCAST:
            send = np.concatenate([rec] * self.nsegs) if n else rec
            counts = np.full(self.nsegs, n, dtype=np.int64)
        else:
            order = np.argsort(dest, kind="stable")
            send = rec[order]
            counts = np.bincount(dest, minlength=self.nsegs).astype(np.int64)
        dev = self.device
        sc = torch.from_numpy(counts.copy())
        sc = sc.to(dev) if dev is not None else sc
        rc = torch.empty_like(sc)
        dist.all_to_all_single(rc, sc, group=self.group)
        rcounts = rc.cpu().numpy()
        w = ncols * 9
        st = torch.from_numpy(np.ascontiguousarray(send).reshape(-1))
        st = st.to(dev) if dev is not None else st
        rt = torch.empty(int(rcounts.sum()) * w, dtype=torch.uint8, device=st.device)
        dist.all_to_all_single(rt, st, output_split_sizes=[int(c) * w for c in rcounts],
                               input_split_sizes=[int(c) * w for c in counts], group=self.group)
        got = rt.cpu().numpy().reshape(-1, w)
        m = got.shape[0]
        rv = np.ascontiguousarray(got[:, :ncols * 8]).view(np.int64).reshape(m, ncols)
        rn = np.ascontiguousarray(got[:, ncols * 8:])
        return rv, rn

    def _exchange(self, ctx, motion_id, motion_type, send, dest, out):
        try:
            s = send.contents
            n, ncols = int(s.nrows), int(s.ncols)
            import torch
            import torch.distributed as dist
            # every segment says whether its slice below the Motion failed (nrows = -1) before any row moves: a failed
            # segment takes part with no rows and every segment comes back with GG_ERR_PEER
            flag = torch.tensor([1 if n < 0 else 0], dtype=torch.int32)
            flag = flag.to(self.device) if self.device is not None else flag
            dist.all_reduce(flag, op=dist.ReduceOp.MAX, group=self.group)
            if int(flag.item()):
                return -12
            if n:
                values = np.ctypeslib.as_array(s.values, shape=(n, ncols)).copy()
                isnull = np.ctypeslib.as_array(s.isnull, shape=(n, ncols)).copy()
                d = np.ctypeslib.as_array(dest, shape=(n,)).copy()
            else:
                values = np.zeros((0, ncols), dtype=np.int64)
                isnull = np.zeros((0, ncols), dtype=np.uint8)
                d = np.zeros(0, dtype=np.int32)
            rv, rn = self.exchange_arrays(values, isnull, d, motion_type)
            m = rv.shape[0]
            o = out.contents
            o.ncols, o.nrows = ncols, m
            pv = self._libc.malloc(max(m * ncols * 8, 8))
            pn = self._libc.malloc(max(m * ncols, 8))
            if m:
                C.memmove(pv, rv.ctypes.data, m * ncols * 8)
                C.memmove(pn, rn.ctypes.data, m * ncols)
            o.values = C.cast(pv, C.POINTER(C.c_int64))
            o.isnull = C.cast(pn, C.POINTER(C.c_uint8))
            return 0
        except Exception as exc:                                  # noqa: BLE001 - reported through the C return code
            self.error = exc
            return 1
