"""ctypes mirror of include/gg_plan.h, include/ggb200.h and include/gg_synth.h.

Plumbing only: every call below lands in libggb200.so (CUDA engine, C-ABI) or
libgghost.so (host C: synthetic loader + executor-node surface).  There is no
Python or CPU implementation of any operator here; if the CUDA library is
missing or no GPU is present the calls fail loudly.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))

GG_BLCKSZ = 32768
GG_MAX_ATTS = 32
GG_MAX_EXPR_NODES = 96
GG_MAX_AGGS = 16
GG_MAX_KEYS = 4

# type OIDs (pg_type.h)
BOOLOID, INT8OID, INT4OID, TEXTOID, FLOAT8OID = 16, 20, 23, 25, 701
BPCHAROID, VARCHAROID, DATEOID, TIMESTAMPOID = 1042, 1043, 1082, 1114
NUMERICOID = 1700

# function OIDs (pg_proc.h), see gg_plan.h
F_INT4EQ, F_INT4LT, F_INT4NE, F_INT4GT, F_INT4LE, F_INT4GE = 65, 66, 144, 147, 149, 150
F_FLOAT8MUL, F_FLOAT8DIV, F_FLOAT8PL, F_FLOAT8MI = 216, 217, 218, 219
F_FLOAT8EQ, F_FLOAT8NE, F_FLOAT8LT, F_FLOAT8LE, F_FLOAT8GT, F_FLOAT8GE = 293, 294, 295, 296, 297, 298
F_I4TOD, F_INT48, F_I8TOD = 316, 481, 482
F_INT8EQ, F_INT8NE, F_INT8LT, F_INT8GT, F_INT8LE, F_INT8GE = 467, 468, 469, 470, 471, 472
F_BPCHAREQ, F_BPCHARNE = 1048, 1053
F_NUMERIC_EQ, F_NUMERIC_NE, F_NUMERIC_GT, F_NUMERIC_GE, F_NUMERIC_LT, F_NUMERIC_LE = 1718, 1719, 1720, 1721, 1722, 1723
F_NUMERIC_ADD, F_NUMERIC_SUB, F_NUMERIC_MUL = 1724, 1725, 1726
F_DATE_EQ, F_DATE_LT, F_DATE_LE, F_DATE_GT, F_DATE_GE, F_DATE_NE = 1086, 1087, 1088, 1089, 1090, 1091
F_DATE_LT_TIMESTAMP, F_DATE_LE_TIMESTAMP, F_DATE_EQ_TIMESTAMP = 2338, 2339, 2340
F_DATE_GT_TIMESTAMP, F_DATE_GE_TIMESTAMP, F_DATE_NE_TIMESTAMP = 2341, 2342, 2343

AGG_AVG_FLOAT8, AGG_SUM_INT4, AGG_SUM_FLOAT8 = 2105, 2108, 2111
AGG_MAX_INT8, AGG_MAX_INT4, AGG_MAX_FLOAT8, AGG_MAX_DATE = 2115, 2116, 2120, 2122
AGG_MIN_INT8, AGG_MIN_INT4, AGG_MIN_FLOAT8, AGG_MIN_DATE = 2131, 2132, 2136, 2138
AGG_COUNT_ANY, AGG_COUNT_STAR = 2147, 2803
AGG_AVG_NUMERIC, AGG_SUM_NUMERIC = 2103, 2114

AGGSTAGE_NORMAL, AGGSTAGE_PARTIAL, AGGSTAGE_FINAL = 0, 1, 3

# window functions (pg_proc.h:4874-4902) and frame options (parsenodes.h:495-517)
WF_ROW_NUMBER, WF_RANK, WF_DENSE_RANK, WF_PERCENT_RANK, WF_CUME_DIST, WF_NTILE = 3100, 3101, 3102, 3103, 3104, 3105
WF_LAG, WF_LAG_OFFSET, WF_LAG_DEFAULT, WF_LEAD, WF_LEAD_OFFSET, WF_LEAD_DEFAULT = 3106, 3107, 3108, 3109, 3110, 3111
WF_FIRST_VALUE, WF_LAST_VALUE, WF_NTH_VALUE = 3112, 3113, 3114
GG_MAX_WINFUNCS = 8
FRAMEOPTION_NONDEFAULT, FRAMEOPTION_RANGE, FRAMEOPTION_ROWS, FRAMEOPTION_BETWEEN = 0x1, 0x2, 0x4, 0x8
FRAMEOPTION_START_UNBOUNDED_PRECEDING, FRAMEOPTION_END_UNBOUNDED_PRECEDING = 0x10, 0x20
FRAMEOPTION_START_UNBOUNDED_FOLLOWING, FRAMEOPTION_END_UNBOUNDED_FOLLOWING = 0x40, 0x80
FRAMEOPTION_START_CURRENT_ROW, FRAMEOPTION_END_CURRENT_ROW = 0x100, 0x200
FRAMEOPTION_START_VALUE_PRECEDING, FRAMEOPTION_END_VALUE_PRECEDING = 0x400, 0x800
FRAMEOPTION_START_VALUE_FOLLOWING, FRAMEOPTION_END_VALUE_FOLLOWING = 0x1000, 0x2000
FRAMEOPTION_DEFAULTS = FRAMEOPTION_RANGE | FRAMEOPTION_START_UNBOUNDED_PRECEDING | FRAMEOPTION_END_CURRENT_ROW
ERR_WINDOW_ARG = -14
JOIN_INNER, JOIN_LEFT, JOIN_FULL, JOIN_RIGHT, JOIN_SEMI, JOIN_ANTI, JOIN_LASJ_NOTIN = 0, 1, 2, 3, 4, 5, 6
E_VAR, E_CONST, E_FUNC, E_AND, E_OR, E_NOT, E_ISNULL, E_ISNOTNULL = 1, 2, 3, 4, 5, 6, 7, 8

TAB_LINEITEM_WIDE, TAB_LINEITEM_NARROW, TAB_ORDERS = 1, 2, 3
DIST_RANDOM, DIST_HASH = 0, 1


class gg_attr(C.Structure):
    _fields_ = [("atttypid", C.c_int32), ("atttypmod", C.c_int32), ("attlen", C.c_int16),
                ("attalign", C.c_int8), ("attbyval", C.c_int8), ("attnotnull", C.c_int8),
                ("pad", C.c_int8 * 3)]


class gg_tupdesc(C.Structure):
    _fields_ = [("natts", C.c_int32), ("format", C.c_int32), ("attrs", gg_attr * GG_MAX_ATTS)]


class gg_expr(C.Structure):
    _fields_ = [("kind", C.c_int32), ("funcid", C.c_int32), ("rettype", C.c_int32),
                ("varno", C.c_int16), ("varattno", C.c_int16), ("nargs", C.c_int32),
                ("args", C.c_int32 * 2), ("constisnull", C.c_int32), ("constlen", C.c_int32),
                ("constvalue", C.c_int64)]


class gg_exprpool(C.Structure):
    _fields_ = [("nnodes", C.c_int32), ("pad", C.c_int32), ("nodes", gg_expr * GG_MAX_EXPR_NODES)]


class gg_aggref(C.Structure):
    _fields_ = [("aggfnoid", C.c_int32), ("arg", C.c_int32)]


class gg_aggval(C.Structure):
    _fields_ = [("f", C.c_double * 3), ("i", C.c_int64), ("isnull", C.c_int32), ("pad", C.c_int32)]


class gg_aggrow(C.Structure):
    _fields_ = [("key", C.c_int64 * GG_MAX_KEYS), ("keylen", C.c_int32 * GG_MAX_KEYS),
                ("keyisnull", C.c_int32 * GG_MAX_KEYS), ("agg", gg_aggval * GG_MAX_AGGS)]


class gg_scan(C.Structure):
    _fields_ = [("desc", gg_tupdesc), ("qual", C.c_int32), ("pad", C.c_int32)]


class gg_agg(C.Structure):
    _fields_ = [("aggstage", C.c_int32), ("numCols", C.c_int32), ("grpCol", C.c_int32 * GG_MAX_KEYS),
                ("numAggs", C.c_int32), ("flags", C.c_int32), ("aggs", gg_aggref * GG_MAX_AGGS),
                ("numGroups", C.c_int64)]


class gg_hashjoin(C.Structure):
    _fields_ = [("jointype", C.c_int32), ("nkeys", C.c_int32), ("outerkey", C.c_int32 * GG_MAX_KEYS),
                ("innerkey", C.c_int32 * GG_MAX_KEYS), ("joinqual", C.c_int32), ("pad", C.c_int32)]


class gg_sortkey(C.Structure):
    _fields_ = [("col", C.c_int32), ("typid", C.c_int32), ("desc", C.c_int32), ("nulls_first", C.c_int32)]


class gg_winfunc(C.Structure):
    _fields_ = [("winfnoid", C.c_int32), ("wintype", C.c_int32), ("arg", C.c_int32 * 3), ("pad", C.c_int32)]


class gg_window(C.Structure):
    _fields_ = [("partNumCols", C.c_int32), ("partColIdx", C.c_int32 * GG_MAX_KEYS), ("ordNumCols", C.c_int32),
                ("ordColIdx", C.c_int32 * GG_MAX_KEYS), ("frameOptions", C.c_int32), ("numFuncs", C.c_int32),
                ("funcs", gg_winfunc * GG_MAX_WINFUNCS)]


def make_window(part, order, frame, funcs):
    """part / order: 0-based input columns; frame: FRAMEOPTION_* bits; funcs: (winfnoid, wintype, [arg roots]) each"""
    w = gg_window()
    w.partNumCols, w.ordNumCols, w.frameOptions, w.numFuncs = len(part), len(order), frame, len(funcs)
    for i, c in enumerate(part):
        w.partColIdx[i] = c
    for i, c in enumerate(order):
        w.ordColIdx[i] = c
    for i, (fn, ty, args) in enumerate(funcs):
        w.funcs[i].winfnoid, w.funcs[i].wintype = fn, ty
        for a in range(3):
            w.funcs[i].arg[a] = args[a] if a < len(args) else -1
    return w


class gg_snapshot(C.Structure):
    """include/gg_plan.h gg_snapshot; make_snapshot() below keeps the arrays it points to alive"""
    _fields_ = [("xmin", C.c_uint32), ("xmax", C.c_uint32), ("xcnt", C.c_uint32), ("curcid", C.c_uint32), ("own_xid", C.c_uint32),
                ("clog_base", C.c_uint32), ("clog_n", C.c_uint32), ("suboverflowed", C.c_uint8), ("takenDuringRecovery", C.c_uint8),
                ("haveDistribSnapshot", C.c_uint8), ("pad", C.c_uint8), ("xip", C.POINTER(C.c_uint32)), ("clog", C.POINTER(C.c_uint8))]


def make_snapshot(xmin, xmax, xip=(), curcid=0, own_xid=0, clog_base=0, clog=b"", clog_n=None):
    """clog: the pg_clog bytes covering xids clog_base .. (2 bits per xid, clog.h:25-28)"""
    s = gg_snapshot()
    s.xmin, s.xmax, s.xcnt, s.curcid, s.own_xid = xmin, xmax, len(xip), curcid, own_xid
    s.clog_base, s.clog_n = clog_base, len(clog) * 4 if clog_n is None else clog_n
    s._xip = (C.c_uint32 * max(1, len(xip)))(*xip)
    s._clog = (C.c_uint8 * max(1, len(clog))).from_buffer_copy(bytes(clog) if clog else b"\0")
    s.xip = C.cast(s._xip, C.POINTER(C.c_uint32))
    s.clog = C.cast(s._clog, C.POINTER(C.c_uint8))
    return s


class gg_synth_spec(C.Structure):
    _fields_ = [("table", C.c_int32), ("policy", C.c_int32), ("seed", C.c_uint64), ("ncand", C.c_uint64),
                ("norders", C.c_uint64), ("nsegs", C.c_int32), ("seg", C.c_int32)]


class GGError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("ggb200 error %d: %s" % (code, msg))
        self.code = code


_dev = None
_host = None


def host_lib():
    """libgghost.so: host C (synthetic loader, executor-node surface). No GPU needed."""
    global _host
    if _host is None:
        path = os.path.join(_HERE, "libgghost.so")
        if not os.path.exists(path):
            raise ImportError("greengage_b200/libgghost.so is not built: run `python -c 'import __graft_entry__ as g; g.build()'`")
        L = C.CDLL(path)
        L.gg_synth_tupdesc.argtypes = [C.c_int, C.POINTER(gg_tupdesc)]
        L.gg_synth_measure.argtypes = [C.POINTER(gg_synth_spec), C.c_int, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        L.gg_synth_generate.argtypes = [C.POINTER(gg_synth_spec), C.c_int, C.c_void_p, C.c_uint64,
                                        C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        L.gg_synth_row.argtypes = [C.POINTER(gg_synth_spec), C.c_uint64, C.POINTER(C.c_int64), C.POINTER(C.c_int32),
                                   C.c_char_p, C.c_int, C.POINTER(C.c_int)]
        L.gg_synth_aocs_generate.argtypes = [C.POINTER(gg_synth_spec), C.c_int, C.POINTER(C.c_int32), C.c_int, C.POINTER(C.c_void_p),
                                             C.POINTER(C.c_int64), C.c_int, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_uint64)]
        L.gg_aocs_crc32c.restype = C.c_uint32
        L.gg_aocs_crc32c.argtypes = [C.c_void_p, C.c_int64]
        L.gg_aocs_index_column.argtypes = [C.POINTER(gg_attr), C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_int64,
                                           C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
        L.gg_aocs_plan_tiles.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_void_p, C.c_int64]
        L.gg_aocs_writer_create.argtypes = [C.POINTER(gg_attr), C.c_int, C.c_int, C.c_int64, C.c_void_p, C.c_int64, C.POINTER(C.c_void_p)]
        L.gg_aocs_writer_put.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_int]
        L.gg_aocs_writer_finish.argtypes = [C.c_void_p, C.POINTER(C.c_int64)]
        L.gg_aocs_file_bound.restype = C.c_int64
        L.gg_aocs_file_bound.argtypes = [C.POINTER(gg_attr), C.c_int64, C.c_int32, C.c_int, C.c_int]
        L.gg_synth_orderkey.argtypes = [C.c_uint64]
        L.gg_synth_orderkey.restype = C.c_int64
        L.gg_cdbhash_route.argtypes = [C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_int32),
                                       C.POINTER(C.c_int32), C.c_int, C.c_int]
        L.gg_cdbhash_route_aggrows.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int32), C.c_int, C.c_int, C.c_void_p]
        L.gg_cdbhash_route_aggrows.restype = None
        L.gg_hash_any.argtypes = [C.c_char_p, C.c_int]
        L.gg_hash_any.restype = C.c_uint32
        _host = L
    return _host


def dev_lib():
    """libggb200.so: the CUDA engine behind the C-ABI.  Loading needs no GPU; running does."""
    global _dev
    if _dev is None:
        # GGB200_DEVLIB: an A/B build of the same sources (scripts/ab_build.sh) for measurements; never set in product use
        path = os.environ.get("GGB200_DEVLIB") or os.path.join(_HERE, "libggb200.so")
        if not os.path.exists(path):
            raise ImportError("greengage_b200/libggb200.so is not built: run `python -c 'import __graft_entry__ as g; g.build()'`")
        L = C.CDLL(path)
        vp, u64, i32 = C.c_void_p, C.c_uint64, C.c_int
        L.gg_last_error.restype = C.c_char_p
        L.gg_strerror.restype = C.c_char_p
        L.gg_strerror.argtypes = [i32]
        L.gg_engine_create.argtypes = [i32, C.POINTER(vp)]
        L.gg_engine_free.argtypes = [vp]
        L.gg_engine_free.restype = None
        L.gg_engine_sm_count.argtypes = [vp]
        L.gg_engine_set_snapshot.argtypes = [vp, C.POINTER(gg_snapshot)]
        L.gg_engine_sync.argtypes = [vp]
        L.gg_engine_last_kernel_ms.argtypes = [vp, C.POINTER(C.c_float)]
        L.gg_engine_launch_count.argtypes = [vp]
        L.gg_engine_launch_count.restype = u64
        L.gg_engine_timer_start.argtypes = [vp]
        L.gg_engine_timer_stop.argtypes = [vp, C.POINTER(C.c_float)]
        L.gg_engine_stream.argtypes = [vp]
        L.gg_engine_stream.restype = vp
        L.gg_scanagg_scan_kernel_ms.argtypes = [vp, C.POINTER(C.c_float), C.POINTER(i32)]
        L.gg_scanagg_variant.argtypes = [vp]
        L.gg_relation_create.argtypes = [vp, u64, C.POINTER(vp)]
        L.gg_relation_attach.argtypes = [vp, vp, u64, C.POINTER(vp)]
        L.gg_relation_load.argtypes = [vp, u64, vp, u64]
        L.gg_relation_read.argtypes = [vp, u64, vp, u64]
        L.gg_relation_copy.argtypes = [vp, u64, vp, u64, u64]
        L.gg_relation_count_rows.argtypes = [vp, C.POINTER(u64)]
        L.gg_relation_nblocks.argtypes = [vp]
        L.gg_relation_nblocks.restype = u64
        L.gg_relation_device_ptr.argtypes = [vp]
        L.gg_relation_device_ptr.restype = vp
        L.gg_relation_free.argtypes = [vp]
        L.gg_relation_free.restype = None
        L.gg_host_alloc.argtypes = [u64, C.POINTER(vp)]
        L.gg_host_free.argtypes = [vp]
        L.gg_host_free.restype = None
        L.gg_scanagg_create.argtypes = [vp, C.POINTER(gg_scan), C.POINTER(gg_agg), C.POINTER(gg_exprpool), C.POINTER(vp)]
        L.gg_scanagg_run.argtypes = [vp, vp, u64, u64]
        L.gg_scanagg_run_host.argtypes = [vp, vp, u64]
        L.gg_scanagg_run_aocs.argtypes = [vp, vp, i32, u64, C.c_int32]
        L.gg_scanagg_fetch.argtypes = [vp, C.POINTER(gg_aggrow), i32, C.POINTER(i32), C.POINTER(u64), C.POINTER(u64)]
        L.gg_scanagg_reset.argtypes = [vp]
        L.gg_scanagg_free.argtypes = [vp]
        L.gg_scanagg_free.restype = None
        L.gg_agg_final.argtypes = [vp, C.POINTER(gg_agg), C.POINTER(gg_aggrow), i32, C.POINTER(gg_aggrow), i32, C.POINTER(i32)]
        L.gg_joinagg_create.argtypes = [vp, C.POINTER(gg_scan), C.POINTER(gg_scan), C.POINTER(gg_hashjoin), C.POINTER(gg_agg),
                                        C.POINTER(gg_exprpool), C.POINTER(vp)]
        L.gg_joinagg_build.argtypes = [vp, vp, u64, u64]
        L.gg_joinagg_probe.argtypes = [vp, vp, u64, u64]
        L.gg_joinagg_probe_host.argtypes = [vp, vp, u64]
        L.gg_joinagg_fetch.argtypes = [vp, C.POINTER(gg_aggrow), i32, C.POINTER(i32), C.POINTER(u64)]
        L.gg_joinagg_reset.argtypes = [vp]
        L.gg_joinagg_set_work_mem.argtypes = [vp, u64]
        L.gg_joinagg_run.argtypes = [vp, vp, vp]
        L.gg_joinagg_nbatch.argtypes = [vp]
        L.gg_joinagg_stats.argtypes = [vp, C.POINTER(u64), C.POINTER(u64), C.POINTER(C.c_float), C.POINTER(C.c_float)]
        L.gg_joinagg_free.argtypes = [vp]
        L.gg_joinagg_free.restype = None
        L.gg_joinrows_create.argtypes = [vp, C.POINTER(gg_scan), C.POINTER(gg_scan), C.POINTER(gg_hashjoin), C.POINTER(C.c_int32), i32,
                                         C.POINTER(gg_exprpool), C.POINTER(vp)]
        L.gg_joinagg_rows.argtypes = [vp, C.POINTER(vp), C.POINTER(u64), C.POINTER(u64)]
        L.gg_debug_disasm_joinrows.argtypes = [C.POINTER(gg_scan), C.POINTER(gg_scan), C.POINTER(gg_hashjoin), C.POINTER(C.c_int32), i32,
                                               C.POINTER(gg_exprpool), C.c_char_p, i32]
        L.gg_sort_rows.argtypes = [vp, C.POINTER(gg_sortkey), i32, i32, vp, vp, u64, vp]
        L.gg_sort_device.argtypes = [vp, C.POINTER(gg_sortkey), i32, i32, vp, vp, u64, vp, C.POINTER(i32)]
        L.gg_sort_datumrows.argtypes = [vp, C.POINTER(gg_sortkey), i32, i32, vp, u64, vp, C.POINTER(u64), C.POINTER(i32)]
        L.gg_sort_datumrows_bounded.argtypes = [vp, C.POINTER(gg_sortkey), i32, i32, vp, u64, u64, vp, C.POINTER(u64), C.POINTER(i32)]
        L.gg_sort_rows_bounded.argtypes = [vp, C.POINTER(gg_sortkey), i32, i32, vp, vp, u64, u64, vp, C.POINTER(u64)]
        L.gg_relation_attach_rows.argtypes = [vp, vp, u64, i32, C.POINTER(vp)]
        # device-resident aggregate rows and the NCCL interconnect
        L.gg_scanagg_groups.argtypes = [vp, C.POINTER(vp)]
        L.gg_joinagg_groups.argtypes = [vp, C.POINTER(vp)]
        L.gg_groups_final.argtypes = [vp, vp, C.POINTER(vp)]
        L.gg_groups_fetch.argtypes = [vp, C.POINTER(gg_aggrow), i32, C.POINTER(i32), C.POINTER(u64), C.POINTER(u64)]
        L.gg_groups_info.argtypes = [vp, C.POINTER(i32), C.POINTER(i32)]
        L.gg_groups_set_nonreceiver.argtypes = [vp]
        L.gg_groups_set_nonreceiver.restype = None
        L.gg_groups_free.argtypes = [vp]
        L.gg_groups_free.restype = None
        L.gg_scanagg_datumrows.argtypes = [vp, C.POINTER(vp), C.POINTER(u64)]
        L.gg_joinagg_datumrows.argtypes = [vp, C.POINTER(vp), C.POINTER(u64)]
        L.gg_groups_datumrows.argtypes = [vp, C.POINTER(vp), C.POINTER(u64)]
        L.gg_rowfilter_create.argtypes = [vp, C.POINTER(gg_tupdesc), C.c_int32, C.POINTER(gg_exprpool), C.POINTER(vp)]
        L.gg_rowfilter_run.argtypes = [vp, vp, u64, C.POINTER(vp), C.POINTER(u64)]
        L.gg_rowfilter_free.argtypes = [vp]
        L.gg_rowfilter_free.restype = None
        L.gg_window_create.argtypes = [vp, C.POINTER(gg_tupdesc), C.POINTER(gg_window), C.POINTER(gg_exprpool), C.POINTER(vp)]
        L.gg_window_run.argtypes = [vp, vp, u64, C.POINTER(vp), C.POINTER(u64)]
        L.gg_window_free.argtypes = [vp]
        L.gg_window_free.restype = None
        L.gg_ic_unique_id.argtypes = [vp, i32]
        L.gg_ic_create.argtypes = [vp, vp, i32, i32, C.POINTER(vp)]
        L.gg_ic_teardown.argtypes = [vp, i32]
        L.gg_ic_teardown.restype = None
        L.gg_ic_free.argtypes = [vp]
        L.gg_ic_free.restype = None
        L.gg_ic_nsegs.argtypes = [vp]
        L.gg_ic_segindex.argtypes = [vp]
        L.gg_ic_collective_count.argtypes = [vp]
        L.gg_ic_collective_count.restype = u64
        L.gg_ic_allgather_u64.argtypes = [vp, u64, C.POINTER(u64)]
        L.gg_ic_motion_groups.argtypes = [vp, i32, i32, i32, C.POINTER(C.c_int32), C.POINTER(C.c_int32), vp, i32, C.POINTER(vp)]
        L.gg_ic_exchange_rows.argtypes = [vp, vp, C.POINTER(u64), u64, i32, vp, u64, C.POINTER(u64)]
        L.gg_ic_exchange_host.argtypes = [vp, i32, C.c_int64, vp, vp, vp, i32, C.POINTER(C.c_int64), C.POINTER(vp), C.POINTER(vp)]
        L.gg_motion_partition.argtypes = [vp, C.POINTER(gg_scan), C.POINTER(gg_exprpool), C.POINTER(C.c_int32), i32,
                                          C.POINTER(C.c_int32), i32, i32, vp, u64, u64, vp, u64, C.POINTER(u64), C.POINTER(u64)]
        _dev = L
    return _dev


# ---------------------------------------------------------------------------
# numeric: text <-> (unscaled integer, display scale) <-> on-disk payload (utils/adt/numeric.c:95-190)
# ---------------------------------------------------------------------------

def numeric_parse(text):
    """'12.340' -> (12340, 3): the digits as an integer and the number of digits behind the point (numeric_in keeps them)"""
    t = str(text).strip()
    neg = t.startswith("-")
    t = t.lstrip("+-")
    ip, _, fp = t.partition(".")
    v = int((ip or "0") + fp)
    return (-v if neg else v), len(fp)


def numeric_text(unscaled, dscale):
    """(12340, 3) -> '12.340' (numeric_out: exactly dscale digits behind the point)"""
    neg = unscaled < 0
    d = str(abs(int(unscaled))).rjust(dscale + 1, "0")
    s = d if dscale == 0 else d[:-dscale] + "." + d[-dscale:]
    return ("-" if neg else "") + s


def numeric_payload(unscaled, dscale):
    """The bytes of a numeric datum behind its varlena header, as numeric_in -> make_result build them (numeric.c:5432 ff):
    base-10000 digits with leading and trailing zero digits stripped, the 2-byte short header when display scale and weight
    fit it (NUMERIC_CAN_BE_SHORT), else the 4-byte long one; zero has no digits and weight 0."""
    neg = unscaled < 0
    mag = abs(int(unscaled))
    d = str(mag).rjust(dscale + 1, "0")
    ip, fp = (d, "") if dscale == 0 else (d[:-dscale], d[-dscale:])
    ip = ip.lstrip("0")
    ip = ip.rjust((len(ip) + 3) // 4 * 4, "0")
    fp = fp.ljust((len(fp) + 3) // 4 * 4, "0")
    digits = [int(ip[i:i + 4]) for i in range(0, len(ip), 4)] + [int(fp[i:i + 4]) for i in range(0, len(fp), 4)]
    weight = len(ip) // 4 - 1
    while digits and digits[0] == 0:
        digits.pop(0)
        weight -= 1
    while digits and digits[-1] == 0:
        digits.pop()
    if not digits:
        weight, neg = 0, False
    import struct
    if dscale <= 0x3F and -64 <= weight <= 63:
        hdr = 0x8000 | (0x2000 if neg else 0) | (dscale << 7) | (0x40 if weight < 0 else 0) | (weight & 0x3F)
        out = struct.pack("<H", hdr)
    else:
        out = struct.pack("<Hh", (0x4000 if neg else 0) | (dscale & 0x3FFF), weight)
    return out + b"".join(struct.pack("<h", x) for x in digits)


def numeric_of_aggval(v):
    """a numeric sum / avg result (gg_aggval: i = low 64 bits, f[0] = bits of the high 64, f[1] = display scale) -> text"""
    import struct
    hi = struct.unpack("<q", struct.pack("<d", v.f[0]))[0]
    val = (hi << 64) | (v.i & 0xFFFFFFFFFFFFFFFF)
    return numeric_text(val, int(v.f[1]))


def check(rc):
    if rc != 0:
        raise GGError(rc, dev_lib().gg_last_error().decode("utf-8", "replace"))


# ---------------------------------------------------------------------------
# plan-building helpers (what a Postgres-side translator would emit from Plan/Expr trees)
# ---------------------------------------------------------------------------

def pack_str(s, bpchar=True):
    """<=8 bytes, trailing blanks stripped for bpchar, packed LSB-first (gg_plan.h GG_E_CONST)."""
    b = s.encode() if isinstance(s, str) else bytes(s)
    if bpchar:
        b = b.rstrip(b" ")
    assert len(b) <= 8
    return int.from_bytes(b.ljust(8, b"\0"), "little", signed=True), len(b)


def unpack_str(v, n):
    return (v & 0xFFFFFFFFFFFFFFFF).to_bytes(8, "little")[:n].decode("latin1")


class ExprPool:
    def __init__(self):
        self.pool = gg_exprpool()
        self.pool.nnodes = 0

    def _new(self):
        i = self.pool.nnodes
        assert i < GG_MAX_EXPR_NODES
        self.pool.nnodes += 1
        n = self.pool.nodes[i]
        n.args[0] = -1
        n.args[1] = -1
        return i, n

    def var(self, attno, typid, varno=0):
        i, n = self._new()
        n.kind, n.varno, n.varattno, n.rettype = E_VAR, varno, attno, typid
        return i

    def const(self, typid, value=None, isnull=False):
        i, n = self._new()
        n.kind, n.rettype = E_CONST, typid
        n.constisnull = 1 if isnull or value is None else 0
        if not n.constisnull:
            if typid == FLOAT8OID:
                n.constvalue = C.c_int64.from_buffer_copy(C.c_double(float(value))).value
            elif typid in (BPCHAROID, VARCHAROID, TEXTOID):
                n.constvalue, n.constlen = pack_str(value, typid == BPCHAROID)
            elif typid == NUMERICOID:
                n.constvalue, n.constlen = numeric_parse(value)      # unscaled integer + display scale (gg_plan.h "numeric")
            else:
                n.constvalue = int(value)
        return i

    def func(self, funcid, rettype, a, b=None):
        i, n = self._new()
        n.kind, n.funcid, n.rettype = E_FUNC, funcid, rettype
        n.args[0] = a
        n.nargs = 1
        if b is not None:
            n.args[1] = b
            n.nargs = 2
        return i

    def boolop(self, kind, a, b=None):
        i, n = self._new()
        n.kind, n.rettype = kind, BOOLOID
        n.args[0] = a
        n.nargs = 1
        if b is not None:
            n.args[1] = b
            n.nargs = 2
        return i


def make_scan(desc, qual=-1):
    s = gg_scan()
    C.memmove(C.byref(s.desc), C.byref(desc), C.sizeof(gg_tupdesc))
    s.qual = qual
    return s


AGGF_DEVICE_FINAL = 1      # gg_plan.h GG_AGGF_DEVICE_FINAL


def make_agg(stage, grpcols, aggs, num_groups=0, flags=0):
    a = gg_agg()
    a.aggstage = stage
    a.flags = flags
    a.numGroups = num_groups
    a.numCols = len(grpcols)
    for i, g in enumerate(grpcols):
        a.grpCol[i] = g
    a.numAggs = len(aggs)
    for i, (fn, arg) in enumerate(aggs):
        a.aggs[i].aggfnoid = fn
        a.aggs[i].arg = arg
    return a


def make_hashjoin(jointype, outerkeys, innerkeys, joinqual=-1):
    """HashJoin.hashclauses as (outer expr, inner expr) pairs + the residual join qual (plannodes.h HashJoin)."""
    h = gg_hashjoin()
    h.jointype = jointype
    h.nkeys = len(outerkeys)
    for i, (o, n) in enumerate(zip(outerkeys, innerkeys)):
        h.outerkey[i] = o
        h.innerkey[i] = n
    h.joinqual = joinqual
    return h


def make_sortkey(col, typid, desc=False, nulls_first=None):
    """Sort.sortColIdx / sortOperators / nullsFirst; PostgreSQL's default is NULLS LAST for ASC, NULLS FIRST for DESC."""
    k = gg_sortkey()
    k.col, k.typid, k.desc = col, typid, int(desc)
    k.nulls_first = int(desc if nulls_first is None else nulls_first)
    return k


FMT_HEAP, FMT_DATUMROWS = 0, 1


def rows_tupdesc(typids, notnull=None):
    """Descriptor of GG_FMT_DATUMROWS rows (what a receiving Motion delivers): one 64-bit word per column."""
    d = gg_tupdesc()
    d.natts = len(typids)
    d.format = FMT_DATUMROWS
    for i, t in enumerate(typids):
        a = d.attrs[i]
        a.atttypid, a.atttypmod, a.attlen, a.attalign, a.attbyval = t, -1, 8, ord("d"), 1
        a.attnotnull = int(bool(notnull[i])) if notnull is not None else 0
    return d


def synth_tupdesc(table):
    d = gg_tupdesc()
    assert host_lib().gg_synth_tupdesc(table, C.byref(d)) == 0
    return d
