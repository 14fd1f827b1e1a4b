"""ctypes binding of oracle/libggoracle.so — TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
legs may import this module.  It is the checker (and the timed CPU arm), never the product.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from greengage_b200 import capi

_HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None
_ref = None



class or_datum(C.Structure):
    _fields_ = [("v", C.c_int64), ("len", C.c_int32), ("isnull", C.c_int32), ("ptr", C.c_void_p),
                ("hi", C.c_int64), ("dscale", C.c_int32), ("pad", C.c_int32)]


XLIMBS = 68                     # OR_XLIMBS (gg_oracle.h)
EXACT_SCALE = 1074              # the exact sums are integers in units of 2^-EXACT_SCALE
XF_NAN, XF_PINF, XF_NINF, XF_ALL_NEGZERO, XF_POSZERO, XF_NEGZERO = 0x01, 0x02, 0x04, 0x08, 0x10, 0x20


class or_exact(C.Structure):
    _fields_ = [("n", C.c_int64), ("flags", C.c_int32), ("lowbit", C.c_int32), ("lowbit_sq", C.c_int32), ("pad", C.c_int32),
                ("sum", C.c_int64 * XLIMBS), ("abs", C.c_int64 * XLIMBS), ("sq", C.c_int64 * XLIMBS)]


class Exact:
    """What the float8 inputs of one aggregate in one group were, exactly (the oracle's exact mode, or_agg.c).
    s, a, q: the exact sum, sum of |x| and sum of fl(x*x) of the finite inputs, as integers in units of 2^-EXACT_SCALE;
    lowbit (lowbit_sq): exponent of the lowest set bit over the nonzero inputs (squares), None when there are none."""
    __slots__ = ("n", "flags", "lowbit", "lowbit_sq", "s", "a", "q")

    def __init__(self, r):
        self.n, self.flags = r.n, r.flags
        self.lowbit = None if r.lowbit == 0x7FFFFFFF else r.lowbit
        self.lowbit_sq = None if r.lowbit_sq == 0x7FFFFFFF else r.lowbit_sq
        self.s, self.a, self.q = (int.from_bytes(np.ctypeslib.as_array(getattr(r, f)).astype(np.uint32).tobytes(), "little", signed=True)
                                  for f in ("sum", "abs", "sq"))


def _exact_states(agg, nrows):
    """-> one list per emitted row: an Exact per aggregate (None for the non-float8 ones), in or_aggtable_emit's order"""
    f8 = {capi.AGG_SUM_FLOAT8, capi.AGG_AVG_FLOAT8, capi.AGG_MIN_FLOAT8, capi.AGG_MAX_FLOAT8}
    which = [agg.aggs[i].aggfnoid in f8 for i in range(agg.numAggs)]
    nf = sum(which)
    buf = (or_exact * max(nrows * nf, 1))()
    got = lib().or_exact_fetch(buf, nrows * nf)
    assert got == nrows * nf, (got, nrows, nf)
    out, k = [], 0
    for _ in range(nrows):
        row = []
        for w in which:
            row.append(Exact(buf[k]) if w else None)
            k += w
        out.append(row)
    return out


class exact_mode:
    """with po.exact_mode(): the operators record the exact inputs of every float8 aggregate (or_exact_mode)"""
    def __enter__(self):
        lib().or_exact_mode(1)

    def __exit__(self, *a):
        lib().or_exact_mode(0)


def build():
    subprocess.check_call(["make", "-s", "-C", _HERE])
    if os.path.isdir("/root/reference/src"):
        subprocess.check_call(["make", "-s", "-C", os.path.join(_HERE, "ref_build")])


def lib():
    global _lib
    if _lib is None:
        path = os.path.join(_HERE, "libggoracle.so")
        if not os.path.exists(path):
            build()
        L = C.CDLL(path)
        u32, i32, i64, u64, vp = C.c_uint32, C.c_int32, C.c_int64, C.c_uint64, C.c_void_p
        L.or_hash_any.restype = u32
        L.or_hash_any.argtypes = [C.c_char_p, i32]
        L.or_hash_uint32.restype = u32
        L.or_hash_uint32.argtypes = [u32]
        L.or_hashint4.restype = u32
        L.or_hashint4.argtypes = [i32]
        L.or_hashint8.restype = u32
        L.or_hashint8.argtypes = [i64]
        L.or_hashfloat8.restype = u32
        L.or_hashfloat8.argtypes = [C.c_double]
        L.or_hashbpchar.restype = u32
        L.or_hashbpchar.argtypes = [C.c_char_p, i32]
        L.or_bpchareq.argtypes = [C.c_char_p, i32, C.c_char_p, i32]
        L.or_bpcharcmp.argtypes = [C.c_char_p, i32, C.c_char_p, i32]
        L.or_cdbhash_add.restype = u32
        L.or_cdbhash_add.argtypes = [u32, u32, i32]
        L.or_jump_consistent_hash.argtypes = [u64, i32]
        L.or_cdbhash_reduce.argtypes = [u32, i32]
        L.or_route_datums.argtypes = [C.POINTER(i32), C.POINTER(i64), C.POINTER(i32), C.POINTER(i32), i32, i32]
        L.or_tuple_satisfies_mvcc.argtypes = [C.c_char_p, C.POINTER(capi.gg_snapshot)]
        L.or_set_snapshot.argtypes = [C.POINTER(capi.gg_snapshot)]
        L.or_heap_form_tuple.argtypes = [C.POINTER(capi.gg_tupdesc), C.POINTER(i64), C.POINTER(i32),
                                         C.POINTER(C.c_uint8), vp, i32]
        L.or_heap_deform.argtypes = [C.POINTER(capi.gg_tupdesc), vp, i32, C.POINTER(i64), C.POINTER(C.c_uint8)]
        L.or_page_init.argtypes = [vp]
        L.or_page_init.restype = None
        L.or_page_add_item.argtypes = [vp, vp, i32]
        L.or_page_nitems.argtypes = [vp]
        L.or_page_set_all_visible.argtypes = [vp]
        L.or_page_set_all_visible.restype = None
        L.or_seqscan_agg.argtypes = [C.POINTER(capi.gg_scan), C.POINTER(capi.gg_agg), C.POINTER(capi.gg_exprpool),
                                     vp, u64, C.POINTER(capi.gg_aggrow), i32, C.POINTER(i32),
                                     C.POINTER(u64), C.POINTER(u64)]
        L.or_agg_final.argtypes = [C.POINTER(capi.gg_agg), C.POINTER(capi.gg_aggrow), i32,
                                   C.POINTER(capi.gg_aggrow), i32, C.POINTER(i32)]
        L.or_hashjoin_agg.argtypes = [C.POINTER(capi.gg_scan), C.POINTER(capi.gg_scan), C.POINTER(capi.gg_hashjoin),
                                      C.POINTER(capi.gg_agg), C.POINTER(capi.gg_exprpool), vp, u64, vp, u64,
                                      C.POINTER(capi.gg_aggrow), i32, C.POINTER(i32), C.POINTER(u64)]
        L.or_hashjoin_tids.argtypes = [C.POINTER(capi.gg_scan), C.POINTER(capi.gg_scan), C.POINTER(capi.gg_hashjoin),
                                       C.POINTER(capi.gg_exprpool), vp, u64, vp, u64, vp, u64, C.POINTER(u64)]
        L.or_sort_perm.argtypes = [C.POINTER(capi.gg_sortkey), i32, i32, vp, vp, u64, vp]
        L.or_motion_route.argtypes = [C.POINTER(capi.gg_scan), C.POINTER(capi.gg_exprpool), C.POINTER(i32), i32, i32,
                                      vp, u64, vp, u64, C.POINTER(u64)]
        L.or_count_star_2stage.restype = i64
        L.or_count_star_2stage.argtypes = [C.POINTER(vp), C.POINTER(u64), i32]
        L.or_seqscan_agg_mt.argtypes = [C.POINTER(capi.gg_scan), C.POINTER(capi.gg_agg), C.POINTER(capi.gg_agg),
                                        C.POINTER(capi.gg_exprpool), vp, u64, i32,
                                        C.POINTER(capi.gg_aggrow), i32, C.POINTER(i32),
                                        C.POINTER(C.c_double), C.POINTER(u64)]
        L.or_eval.argtypes = [C.POINTER(capi.gg_exprpool), i32, vp, vp, C.POINTER(or_datum)]
        L.or_aocs_crc32c.restype = u32
        L.or_aocs_crc32c.argtypes = [vp, i64]
        L.or_aocs_write_column.restype = i64
        L.or_aocs_write_column.argtypes = [C.POINTER(capi.gg_attr), vp, vp, vp, i64, i32, i32, i64, vp, i64]
        L.or_aocs_read_column.restype = i64
        L.or_aocs_read_column.argtypes = [C.POINTER(capi.gg_attr), vp, i64, i32, vp, vp, i64, vp, vp, i32, C.POINTER(i32)]
        L.or_aocs_seqscan_agg.argtypes = [C.POINTER(capi.gg_scan), C.POINTER(capi.gg_agg), C.POINTER(capi.gg_exprpool),
                                          C.POINTER(vp), C.POINTER(i64), i32, i64, C.POINTER(capi.gg_aggrow), i32,
                                          C.POINTER(i32), C.POINTER(u64), C.POINTER(u64)]
        L.or_bctruelen.argtypes = [C.c_char_p, i32]
        L.or_exact_mode.argtypes = [i32]
        L.or_exact_mode.restype = None
        L.or_exact_fetch.argtypes = [C.POINTER(or_exact), C.c_long]
        L.or_exact_fetch.restype = C.c_long
        L.or_strerror.restype = C.c_char_p
        L.or_strerror.argtypes = [i32]
        _lib = L
    return _lib


def ref_lib():
    """The reference's own leaf objects (oracle/_ref/libggref.so), or None when not built."""
    global _ref
    if _ref is None:
        path = os.path.join(_HERE, "_ref", "libggref.so")
        if not os.path.exists(path):
            return None
        R = C.CDLL(path)
        u32, i32, i64 = C.c_uint32, C.c_int32, C.c_int64
        for name in ("ref_hash_any", "ref_hash_uint32", "ref_hashint4", "ref_hashint8", "ref_hashfloat8", "ref_hashbpchar"):
            getattr(R, name).restype = u32
        R.ref_hash_any.argtypes = [C.c_char_p, i32]
        R.ref_hash_uint32.argtypes = [u32]
        R.ref_hashint4.argtypes = [i32]
        R.ref_hashint8.argtypes = [i64]
        R.ref_hashfloat8.argtypes = [C.c_double]
        R.ref_hashbpchar.argtypes = [C.c_char_p, i32]
        R.ref_bpchareq.argtypes = [C.c_char_p, i32, C.c_char_p, i32]
        R.ref_cdbhash_route.argtypes = [C.POINTER(i32), C.POINTER(i64), C.POINTER(i32), C.POINTER(i32), i32, i32]
        R.ref_heap_form_tuple.argtypes = [i32, C.POINTER(capi.gg_attr), C.POINTER(i64), C.POINTER(i32),
                                          C.POINTER(C.c_uint8), C.c_void_p, i32]
        R.ref_heap_deform_tuple.argtypes = [i32, C.POINTER(capi.gg_attr), C.c_void_p, i32, C.POINTER(i64), C.POINTER(C.c_uint8)]
        for name in ("ref_float8pl", "ref_float8mi", "ref_float8mul", "ref_float8div"):
            getattr(R, name).restype = C.c_double
            getattr(R, name).argtypes = [C.c_double, C.c_double, C.POINTER(i32)]
        for name in ("ref_float8eq", "ref_float8lt", "ref_float8le", "ref_btfloat8cmp"):
            getattr(R, name).argtypes = [C.c_double, C.c_double]
        R.ref_float8_accum.argtypes = [C.POINTER(C.c_double), C.c_double, C.POINTER(i32)]
        R.ref_float8_accum.restype = None
        R.ref_float8_combine.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(i32)]
        R.ref_float8_combine.restype = None
        R.ref_float8_avg.argtypes = [C.POINTER(C.c_double), C.POINTER(i32)]
        R.ref_float8_avg.restype = C.c_double
        R.ref_int8inc.argtypes = [i64, C.POINTER(i32)]
        R.ref_int8inc.restype = i64
        R.ref_int8pl.argtypes = [i64, i64, C.POINTER(i32)]
        R.ref_int8pl.restype = i64
        R.ref_date_cmp_timestamp.argtypes = [i32, i32, i64, C.POINTER(i32)]
        if hasattr(R, "ref_aocs_write_column"):
            vp = C.c_void_p
            R.ref_aocs_write_column.restype = i64
            R.ref_aocs_write_column.argtypes = [i32, i32, i32, C.c_char, vp, vp, vp, i64, i32, i32, i64, vp, i64, C.POINTER(i32)]
            R.ref_aocs_read_column.restype = i64
            R.ref_aocs_read_column.argtypes = [i32, i32, i32, C.c_char, vp, i64, i32, vp, vp, i64, vp, vp, i32, C.POINTER(i32), C.POINTER(i32)]
            R.ref_aocs_crc32c.restype = u32
            R.ref_aocs_crc32c.argtypes = [vp, i64]
        _ref = R
    return _ref


def eval_expr(pool, root):
    """Evaluate a row-independent expression (constants only). Returns (rc, value_bits, isnull)."""
    d = or_datum()
    rc = lib().or_eval(C.byref(pool), root, None, None, C.byref(d))
    return rc, d.v, d.isnull


def eval_numeric(pool, root):
    """Evaluate a row-independent numeric expression: (rc, text or None when NULL)"""
    d = or_datum()
    rc = lib().or_eval(C.byref(pool), root, None, None, C.byref(d))
    if rc or d.isnull:
        return rc, None
    return rc, capi.numeric_text((d.hi << 64) | (d.v & 0xFFFFFFFFFFFFFFFF), d.dscale)


class OracleError(RuntimeError):
    def __init__(self, code):
        super().__init__("oracle error %d: %s" % (code, lib().or_strerror(code).decode()))
        self.code = code


def _chk(rc):
    if rc != 0:
        raise OracleError(rc)


def _exact(on):
    import contextlib
    return exact_mode() if on else contextlib.nullcontext()


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


# ---- page building from python rows (small fixtures) ----

def form_tuple(desc, values, isnull=None):
    """values: python list; strings/bytes for varlena attrs (payload, already blank-padded for bpchar)."""
    n = desc.natts
    vals = (C.c_int64 * n)()
    lens = (C.c_int32 * n)()
    nulls = (C.c_uint8 * n)()
    keep = []
    for i in range(n):
        a = desc.attrs[i]
        if isnull is not None and isnull[i]:
            nulls[i] = 1
            continue
        v = values[i]
        if a.attlen == -1:
            b = v.encode() if isinstance(v, str) else bytes(v)
            buf = C.create_string_buffer(b, len(b))
            keep.append(buf)
            vals[i] = C.addressof(buf)
            lens[i] = len(b)
        elif a.atttypid == capi.FLOAT8OID:
            vals[i] = C.c_int64.from_buffer_copy(C.c_double(float(v))).value
        else:
            vals[i] = int(v)
    out = (C.c_uint8 * 8192)()
    ln = lib().or_heap_form_tuple(C.byref(desc), vals, lens, nulls, out, 8192)
    assert ln > 0
    return bytes(out[:ln])


def build_pages(desc, rows, nulls=None, all_visible=True):
    """Greedy PageAddItem fill; returns a uint8 numpy array of whole pages."""
    L = lib()
    pages = []
    cur = None
    for r, row in enumerate(rows):
        t = form_tuple(desc, row, None if nulls is None else nulls[r])
        tb = C.create_string_buffer(t, len(t))
        if cur is None or L.or_page_add_item(_ptr(cur), tb, len(t)) == 0:
            cur = np.zeros(capi.GG_BLCKSZ, dtype=np.uint8)
            L.or_page_init(_ptr(cur))
            if all_visible:
                L.or_page_set_all_visible(_ptr(cur))
            pages.append(cur)
            assert L.or_page_add_item(_ptr(cur), tb, len(t)) > 0
    if not pages:
        return np.zeros(0, dtype=np.uint8)
    return np.concatenate(pages)


# ---- operators ----

def seqscan_agg(scan, agg, pool, pages, cap=4096, exact=False):
    """-> (rows, scanned, passed); exact=True: (rows, scanned, passed, [Exact per aggregate] per row)"""
    nb = pages.size // capi.GG_BLCKSZ
    out = (capi.gg_aggrow * cap)()
    n = C.c_int32(0)
    sc, ps = C.c_uint64(0), C.c_uint64(0)
    with _exact(exact):
        _chk(lib().or_seqscan_agg(C.byref(scan), C.byref(agg), C.byref(pool), _ptr(pages), nb, out, cap,
                                  C.byref(n), C.byref(sc), C.byref(ps)))
    rows = [out[i] for i in range(n.value)]
    return (rows, sc.value, ps.value) + ((_exact_states(agg, n.value),) if exact else ())


def agg_final(agg, rows, cap=4096):
    arr = (capi.gg_aggrow * max(len(rows), 1))()
    for i, r in enumerate(rows):
        C.memmove(C.byref(arr[i]), C.byref(r), C.sizeof(capi.gg_aggrow))
    out = (capi.gg_aggrow * cap)()
    n = C.c_int32(0)
    _chk(lib().or_agg_final(C.byref(agg), arr, len(rows), out, cap, C.byref(n)))
    return [out[i] for i in range(n.value)]


def seqscan_agg_mt(scan, partial, final, pool, pages, nthreads, cap=4096):
    nb = pages.size // capi.GG_BLCKSZ
    out = (capi.gg_aggrow * cap)()
    n = C.c_int32(0)
    secs = C.c_double(0)
    rows = C.c_uint64(0)
    _chk(lib().or_seqscan_agg_mt(C.byref(scan), C.byref(partial), C.byref(final), C.byref(pool), _ptr(pages), nb,
                                 nthreads, out, cap, C.byref(n), C.byref(secs), C.byref(rows)))
    return [out[i] for i in range(n.value)], secs.value, rows.value


def hashjoin_agg(outer, inner, hj, agg, pool, opages, ipages, cap=4096, exact=False):
    """-> (rows, joined); exact=True: (rows, joined, [Exact per aggregate] per row)"""
    out = (capi.gg_aggrow * cap)()
    n = C.c_int32(0)
    nj = C.c_uint64(0)
    with _exact(exact):
        _chk(lib().or_hashjoin_agg(C.byref(outer), C.byref(inner), C.byref(hj), C.byref(agg), C.byref(pool),
                                   _ptr(opages), opages.size // capi.GG_BLCKSZ, _ptr(ipages), ipages.size // capi.GG_BLCKSZ,
                                   out, cap, C.byref(n), C.byref(nj)))
    return ([out[i] for i in range(n.value)], nj.value) + ((_exact_states(agg, n.value),) if exact else ())


def hashjoin_tids(outer, inner, hj, pool, opages, ipages, cap=1 << 22):
    pairs = np.zeros(2 * cap, dtype=np.int64)
    n = C.c_uint64(0)
    _chk(lib().or_hashjoin_tids(C.byref(outer), C.byref(inner), C.byref(hj), C.byref(pool),
                                _ptr(opages), opages.size // capi.GG_BLCKSZ, _ptr(ipages), ipages.size // capi.GG_BLCKSZ,
                                _ptr(pairs), cap, C.byref(n)))
    return pairs[:2 * n.value].reshape(-1, 2)


def sort_perm(keys, ncols, rows, nulls=None):
    n = rows.shape[0]
    ka = (capi.gg_sortkey * len(keys))(*keys)
    perm = np.zeros(n, dtype=np.uint64)
    rows = np.ascontiguousarray(rows, dtype=np.int64)
    _chk(lib().or_sort_perm(ka, len(keys), ncols, _ptr(rows), _ptr(nulls) if nulls is not None else None, n, _ptr(perm)))
    return perm


def motion_route(scan, pool, hashkeys, nsegs, pages, cap=None):
    nb = pages.size // capi.GG_BLCKSZ
    cap = cap or nb * 1200
    dest = np.zeros(cap, dtype=np.int32)
    hk = (C.c_int32 * len(hashkeys))(*hashkeys)
    n = C.c_uint64(0)
    _chk(lib().or_motion_route(C.byref(scan), C.byref(pool), hk, len(hashkeys), nsegs, _ptr(pages), nb,
                               _ptr(dest), cap, C.byref(n)))
    return dest[:n.value]


def deform_page(desc, pages, blk):
    """All tuples of one page as lists of python values (strings as bytes)."""
    L = lib()
    pg = pages[blk * capi.GG_BLCKSZ:(blk + 1) * capi.GG_BLCKSZ]
    n = L.or_page_nitems(_ptr(pg))
    out = []
    vals = (C.c_int64 * desc.natts)()
    nulls = (C.c_uint8 * desc.natts)()
    for i in range(n):
        lp = int(pg[24 + 4 * i:28 + 4 * i].view(np.uint32)[0])
        off, ln = lp & 0x7FFF, lp >> 17
        tup = np.ascontiguousarray(pg[off:off + ln])
        L.or_heap_deform(C.byref(desc), _ptr(tup), desc.natts, vals, nulls)
        row = []
        for a in range(desc.natts):
            if nulls[a]:
                row.append(None)
            elif desc.attrs[a].attlen == -1:
                p = int(vals[a])
                h = int(tup[p])
                if h & 0x80:
                    row.append(bytes(tup[p + 1:p + (h & 0x7F)]))
                else:
                    l = int.from_bytes(bytes(tup[p:p + 4]), "big") & 0x3FFFFFFF
                    row.append(bytes(tup[p + 4:p + l]))
            elif desc.attrs[a].atttypid == capi.FLOAT8OID:
                row.append(C.c_double.from_buffer_copy(C.c_int64(vals[a])).value)
            else:
                row.append(int(vals[a]))
        out.append(row)
    return out


# ---- column-oriented append-only (AOCS) column files (or_aocs.c; SURVEY §8f rank 1) ----

def _aocs_inputs(att, values, nulls):
    """python values -> (int64 value array, int32 lens or None, uint8 nulls or None, keepalive)"""
    n = len(values)
    vals = np.zeros(n, dtype=np.int64)
    lens = np.zeros(n, dtype=np.int32) if att.attlen == -1 else None
    keep = []
    for i, v in enumerate(values):
        if nulls is not None and nulls[i]:
            continue
        if att.attlen == -1:
            b = v.encode() if isinstance(v, str) else bytes(v)
            buf = C.create_string_buffer(b, len(b))
            keep.append(buf)
            vals[i] = C.addressof(buf)
            lens[i] = len(b)
        elif att.atttypid == capi.FLOAT8OID:
            vals[i] = C.c_int64.from_buffer_copy(C.c_double(float(v))).value
        else:
            vals[i] = int(v)
    nl = None if nulls is None else np.ascontiguousarray(nulls, dtype=np.uint8)
    return vals, lens, nl, keep


def aocs_write_column(att, values, nulls=None, blocksize=32768, checksum=True, first_rownum=1, ref=False):
    """One column of an AOCS segment file as a uint8 array; ref=True has the REFERENCE'S OWN objects write it."""
    vals, lens, nl, keep = _aocs_inputs(att, values, nulls)
    n = len(values)
    out = np.zeros((n // 1000 + 2) * blocksize + (int(lens.sum()) if lens is not None else 8 * n) * 2, dtype=np.uint8)
    args = (_ptr(vals), _ptr(lens) if lens is not None else None, _ptr(nl) if nl is not None else None, n, blocksize,
            int(checksum), first_rownum, _ptr(out), out.size)
    if ref:
        err = C.c_int32(0)
        sz = ref_lib().ref_aocs_write_column(att.atttypid, att.attlen, att.attbyval, bytes([att.attalign]), *args, C.byref(err))
        if err.value:
            raise OracleError(-6)
    else:
        sz = lib().or_aocs_write_column(C.byref(att), *args)
        if sz < 0:
            raise OracleError(int(sz))
    return out[:sz].copy()


def aocs_read_column(att, file, nrows_cap, checksum=True, ref=False):
    """-> (values int64[n], nulls uint8[n], firstrows, rowcounts); varlena values are byte offsets into `file`."""
    vals = np.zeros(nrows_cap, dtype=np.int64)
    nl = np.zeros(nrows_cap, dtype=np.uint8)
    bcap = file.size // 24 + 1
    fr = np.zeros(bcap, dtype=np.int64)
    rc = np.zeros(bcap, dtype=np.int32)
    nb = C.c_int32(0)
    if ref:
        err = C.c_int32(0)
        n = ref_lib().ref_aocs_read_column(att.atttypid, att.attlen, att.attbyval, bytes([att.attalign]), _ptr(file), file.size,
                                           int(checksum), _ptr(vals), _ptr(nl), nrows_cap, _ptr(fr), _ptr(rc), bcap,
                                           C.byref(nb), C.byref(err))
        if err.value or n < 0:
            raise OracleError(-6)
    else:
        n = lib().or_aocs_read_column(C.byref(att), _ptr(file), file.size, int(checksum), _ptr(vals), _ptr(nl), nrows_cap,
                                      _ptr(fr), _ptr(rc), bcap, C.byref(nb))
        if n < 0:
            raise OracleError(int(n))
    return vals[:n], nl[:n], fr[:nb.value], rc[:nb.value]


def aocs_seqscan_agg(scan, agg, pool, colfiles, nrows, checksum=True, cap=4096, exact=False):
    """colfiles: one uint8 array per attribute of scan.desc, None for columns the plan does not read.
    -> (rows, scanned, passed); exact=True: (rows, scanned, passed, [Exact per aggregate] per row)"""
    natts = scan.desc.natts
    ptrs = (C.c_void_p * natts)(*[None if f is None else f.ctypes.data for f in colfiles])
    sizes = (C.c_int64 * natts)(*[0 if f is None else f.size for f in colfiles])
    out = (capi.gg_aggrow * cap)()
    n = C.c_int32(0)
    sc, ps = C.c_uint64(0), C.c_uint64(0)
    with _exact(exact):
        _chk(lib().or_aocs_seqscan_agg(C.byref(scan), C.byref(agg), C.byref(pool), ptrs, sizes, int(checksum), nrows, out, cap,
                                       C.byref(n), C.byref(sc), C.byref(ps)))
    rows = [out[i] for i in range(n.value)]
    return (rows, sc.value, ps.value) + ((_exact_states(agg, n.value),) if exact else ())


_snapshot_keep = None


def set_snapshot(snap):
    """the snapshot of the scans that follow (capi.make_snapshot), None: hint bits only"""
    global _snapshot_keep
    _snapshot_keep = snap
    lib().or_set_snapshot(C.byref(snap) if snap is not None else None)


def tuple_satisfies_mvcc(header, snap):
    """1 visible, 0 not, -1 undecidable without the server"""
    return lib().or_tuple_satisfies_mvcc(bytes(header), C.byref(snap))
