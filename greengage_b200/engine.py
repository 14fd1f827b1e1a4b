"""Thin object wrappers over the C-ABI (include/ggb200.h).  No operator logic lives here."""
import ctypes as C

import numpy as np

from . import capi
from .capi import check, dev_lib


class Engine:
    """One GPU segment (gg_engine).  Fails loudly when no CUDA device is usable: there is no CPU fallback."""

    def __init__(self, device=0):
        self.h = C.c_void_p()
        check(dev_lib().gg_engine_create(device, C.byref(self.h)))
        self.device = device

    def close(self):
        if self.h:
            dev_lib().gg_engine_free(self.h)
            self.h = C.c_void_p()

    def sync(self):
        check(dev_lib().gg_engine_sync(self.h))

    @property
    def sm_count(self):
        return dev_lib().gg_engine_sm_count(self.h)

    def set_snapshot(self, snap):
        """the snapshot every scan launched from now on decides visibility with (capi.make_snapshot); None: hint bits only"""
        check(dev_lib().gg_engine_set_snapshot(self.h, C.byref(snap) if snap is not None else None))
        self._snapshot = snap

    def last_kernel_ms(self):
        ms = C.c_float(0)
        check(dev_lib().gg_engine_last_kernel_ms(self.h, C.byref(ms)))
        return ms.value

    def launch_count(self):
        return dev_lib().gg_engine_launch_count(self.h)

    def timer_start(self):
        check(dev_lib().gg_engine_timer_start(self.h))

    def timer_stop(self):
        ms = C.c_float(0)
        check(dev_lib().gg_engine_timer_stop(self.h, C.byref(ms)))
        return ms.value


def host_alloc(nbytes):
    """Pinned host memory (cudaHostAlloc) as (address, numpy view)."""
    p = C.c_void_p()
    check(dev_lib().gg_host_alloc(nbytes, C.byref(p)))
    arr = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(nbytes,))
    return p.value, arr


def host_free(addr):
    dev_lib().gg_host_free(C.c_void_p(addr))


class Relation:
    """Heap pages resident in HBM (gg_relation)."""

    def __init__(self, eng, nblocks=None, host_pages=None, device_ptr=None):
        self.eng = eng
        self.h = C.c_void_p()
        L = dev_lib()
        if device_ptr is not None:
            check(L.gg_relation_attach(eng.h, C.c_void_p(device_ptr), nblocks, C.byref(self.h)))
        else:
            if host_pages is not None:
                nblocks = host_pages.size // capi.GG_BLCKSZ
            check(L.gg_relation_create(eng.h, nblocks, C.byref(self.h)))
            if host_pages is not None and nblocks:
                self.load(0, host_pages)
                eng.sync()
        self.nblocks = nblocks

    def load(self, first_block, host_pages):
        nb = host_pages.size // capi.GG_BLCKSZ
        check(dev_lib().gg_relation_load(self.h, first_block, host_pages.ctypes.data_as(C.c_void_p), nb))

    def read(self, first_block=0, nblocks=None):
        nblocks = self.nblocks - first_block if nblocks is None else nblocks
        out = np.empty(nblocks * capi.GG_BLCKSZ, dtype=np.uint8)
        check(dev_lib().gg_relation_read(self.h, first_block, out.ctypes.data_as(C.c_void_p), nblocks))
        return out

    def device_ptr(self):
        return dev_lib().gg_relation_device_ptr(self.h)

    def copy_from(self, src, dst_first=0, src_first=0, nblocks=None):
        """device -> device copy of pages (gg_relation_copy)"""
        nblocks = src.nblocks - src_first if nblocks is None else nblocks
        check(dev_lib().gg_relation_copy(self.h, dst_first, src.h, src_first, nblocks))

    def free(self):
        if self.h:
            dev_lib().gg_relation_free(self.h)
            self.h = C.c_void_p()


class RowRelation:
    """Datum rows (GG_FMT_DATUMROWS) in device memory, scanned like a heap relation (gg_relation_attach_rows)."""

    def __init__(self, eng, device_ptr, nrows, ncols):
        self.eng = eng
        self.h = C.c_void_p()
        self.nrows, self.ncols = nrows, ncols
        check(dev_lib().gg_relation_attach_rows(eng.h, C.c_void_p(device_ptr), nrows, ncols, C.byref(self.h)))
        self.nblocks = dev_lib().gg_relation_nblocks(self.h)

    def free(self):
        if self.h:
            dev_lib().gg_relation_free(self.h)
            self.h = C.c_void_p()


def motion_partition(eng, scan, pool, hashkeys, payload, nsegs, rel, out_ptr, out_cap_rows, first_block=0, nblocks=None):
    """Sending side of a Redistribute Motion on the device; returns (counts, offsets) in rows per destination."""
    nblocks = rel.nblocks - first_block if nblocks is None else nblocks
    hk = (C.c_int32 * len(hashkeys))(*hashkeys)
    pl = (C.c_int32 * len(payload))(*payload)
    counts = (C.c_uint64 * nsegs)()
    offs = (C.c_uint64 * nsegs)()
    check(dev_lib().gg_motion_partition(eng.h, C.byref(scan), C.byref(pool), hk, len(hashkeys), pl, len(payload), nsegs,
                                        rel.h, first_block, nblocks, C.c_void_p(out_ptr), out_cap_rows, counts, offs))
    return list(counts), list(offs)


def _datumrows(fn, h, ncols):
    """the datum rows an Agg's gg_*_datumrows hands out, read to the host: (values int64 [n][ncols], isnull bool [n][ncols])"""
    rel, n = C.c_void_p(), C.c_uint64(0)
    check(fn(h, C.byref(rel), C.byref(n)))
    n = n.value
    W = 1 + ncols
    nb = (n * W * 8 + capi.GG_BLCKSZ - 1) // capi.GG_BLCKSZ
    buf = np.zeros(nb * capi.GG_BLCKSZ // 8, dtype=np.uint64)
    if nb:
        check(dev_lib().gg_relation_read(rel, 0, buf.ctypes.data, nb))
    r = buf[:n * W].reshape(n, W)
    nulls = ((r[:, :1] >> np.arange(ncols, dtype=np.uint64)) & np.uint64(1)).astype(bool)
    return np.ascontiguousarray(r[:, 1:]).view(np.int64), nulls


class RowFilter:
    """An Agg's HAVING over datum rows (gg_rowfilter): the rows whose qual is TRUE, in input order."""

    def __init__(self, eng, rows_desc, qual, pool):
        self.eng = eng
        self.h = C.c_void_p()
        self.ncols = rows_desc.natts
        check(dev_lib().gg_rowfilter_create(eng.h, C.byref(rows_desc), qual, C.byref(pool), C.byref(self.h)))

    def run_raw(self, rows, nrows=None):
        """rows: a RowRelation of ncols columns; returns (view handle, number of rows), the view valid until the next run"""
        view, n = C.c_void_p(), C.c_uint64(0)
        check(dev_lib().gg_rowfilter_run(self.h, rows.h, rows.nrows if nrows is None else nrows, C.byref(view), C.byref(n)))
        return view, n.value

    def run(self, rows, nrows=None):
        """the surviving rows read to the host: their words as uint64 [n][1 + ncols] (NULL mask, then the columns)"""
        view, n = self.run_raw(rows, nrows)
        W = 1 + self.ncols
        nb = (n * W * 8 + capi.GG_BLCKSZ - 1) // capi.GG_BLCKSZ
        buf = np.zeros(nb * capi.GG_BLCKSZ // 8, dtype=np.uint64)
        if nb:
            check(dev_lib().gg_relation_read(view, 0, buf.ctypes.data, nb))
        return buf[:n * W].reshape(n, W).copy()

    def free(self):
        if self.h:
            dev_lib().gg_rowfilter_free(self.h)
            self.h = C.c_void_p()


class ScanAgg:
    """SeqScan -> qual -> Agg pipeline (gg_scanagg)."""

    def __init__(self, eng, scan, agg, pool):
        self.eng = eng
        self.h = C.c_void_p()
        self.agg = agg
        check(dev_lib().gg_scanagg_create(eng.h, C.byref(scan), C.byref(agg), C.byref(pool), C.byref(self.h)))

    def run(self, rel, first_block=0, nblocks=None):
        nblocks = rel.nblocks - first_block if nblocks is None else nblocks
        check(dev_lib().gg_scanagg_run(self.h, rel.h, first_block, nblocks))

    def run_host(self, host_ptr, nblocks):
        check(dev_lib().gg_scanagg_run_host(self.h, C.c_void_p(host_ptr), nblocks))

    def run_aocs(self, devcols):
        """fused scan over column files resident on the device (aocs.DeviceColumns); the plan's scan descriptor is
        devcols.rows_tupdesc()"""
        check(dev_lib().gg_scanagg_run_aocs(self.h, devcols.devcols, len(devcols.cols), devcols.nrows, devcols.tile_rows))

    def reset(self):
        check(dev_lib().gg_scanagg_reset(self.h))

    def fetch(self, cap=4096):
        out = (capi.gg_aggrow * cap)()
        n = C.c_int(0)
        sc, ps = C.c_uint64(0), C.c_uint64(0)
        check(dev_lib().gg_scanagg_fetch(self.h, out, cap, C.byref(n), C.byref(sc), C.byref(ps)))
        return [out[i] for i in range(n.value)], sc.value, ps.value

    def fetch_raw(self, cap=4096):
        """fetch() without building Python row objects: (numpy uint8 view of the gg_aggrow array, n, scanned, passed)"""
        if getattr(self, "_raw_cap", 0) < cap:
            self._raw = (capi.gg_aggrow * cap)()
            self._raw_cap = cap
        n = C.c_int(0)
        sc, ps = C.c_uint64(0), C.c_uint64(0)
        check(dev_lib().gg_scanagg_fetch(self.h, self._raw, cap, C.byref(n), C.byref(sc), C.byref(ps)))
        buf = np.frombuffer(self._raw, dtype=np.uint8, count=n.value * C.sizeof(capi.gg_aggrow))
        return buf, n.value, sc.value, ps.value

    def datumrows(self):
        """the groups finalised on the device (gg_scanagg_datumrows), in the order the device wrote them: (values, isnull)"""
        return _datumrows(dev_lib().gg_scanagg_datumrows, self.h, self.agg.numCols + self.agg.numAggs)

    def scan_kernel_ms(self):
        ms, n = C.c_float(0), C.c_int(0)
        check(dev_lib().gg_scanagg_scan_kernel_ms(self.h, C.byref(ms), C.byref(n)))
        return ms.value, n.value

    def variant(self):
        return dev_lib().gg_scanagg_variant(self.h)

    def free(self):
        if self.h:
            dev_lib().gg_scanagg_free(self.h)
            self.h = C.c_void_p()


class JoinAgg:
    """SeqScan(outer) ⋈ Hash(SeqScan(inner)) -> Agg pipeline (gg_joinagg)."""

    def __init__(self, eng, outer, inner, hj, agg, pool):
        self.eng = eng
        self.h = C.c_void_p()
        self.agg = agg
        check(dev_lib().gg_joinagg_create(eng.h, C.byref(outer), C.byref(inner), C.byref(hj), C.byref(agg), C.byref(pool),
                                          C.byref(self.h)))

    def build(self, rel, first_block=0, nblocks=None):
        nblocks = rel.nblocks - first_block if nblocks is None else nblocks
        check(dev_lib().gg_joinagg_build(self.h, rel.h, first_block, nblocks))

    def probe(self, rel, first_block=0, nblocks=None):
        nblocks = rel.nblocks - first_block if nblocks is None else nblocks
        check(dev_lib().gg_joinagg_probe(self.h, rel.h, first_block, nblocks))

    def probe_host(self, host_ptr, nblocks):
        check(dev_lib().gg_joinagg_probe_host(self.h, C.c_void_p(host_ptr), nblocks))

    def reset(self):
        check(dev_lib().gg_joinagg_reset(self.h))

    def set_work_mem(self, nbytes):
        """the operator's memory: a hash table larger than this makes run() join in batches (0 = no limit)"""
        check(dev_lib().gg_joinagg_set_work_mem(self.h, int(nbytes)))

    def run(self, inner, outer):
        """build + probe over whole relations, in batches when the hash table would exceed the work memory"""
        check(dev_lib().gg_joinagg_run(self.h, inner.h, outer.h))
        return dev_lib().gg_joinagg_nbatch(self.h)

    def fetch(self, cap=4096):
        out = (capi.gg_aggrow * cap)()
        n = C.c_int(0)
        nj = C.c_uint64(0)
        check(dev_lib().gg_joinagg_fetch(self.h, out, cap, C.byref(n), C.byref(nj)))
        return [out[i] for i in range(n.value)], nj.value

    def datumrows(self):
        """the joined-and-aggregated groups finalised on the device (gg_joinagg_datumrows): (values, isnull)"""
        return _datumrows(dev_lib().gg_joinagg_datumrows, self.h, self.agg.numCols + self.agg.numAggs)

    def stats(self):
        rb, tb = C.c_uint64(0), C.c_uint64(0)
        bms, pms = C.c_float(0), C.c_float(0)
        check(dev_lib().gg_joinagg_stats(self.h, C.byref(rb), C.byref(tb), C.byref(bms), C.byref(pms)))
        return {"rows_built": rb.value, "table_bytes": tb.value, "build_ms": bms.value, "probe_ms": pms.value}

    def free(self):
        if self.h:
            dev_lib().gg_joinagg_free(self.h)
            self.h = C.c_void_p()


class JoinRows(JoinAgg):
    """HashJoin with a target list (gg_joinrows_create): build / probe / run / reset / stats as JoinAgg; rows() instead of
    fetch()."""

    def __init__(self, eng, outer, inner, hj, targets, pool):
        self.eng = eng
        self.h = C.c_void_p()
        self.ncols = len(targets)
        t = (C.c_int32 * max(1, len(targets)))(*targets)
        check(dev_lib().gg_joinrows_create(eng.h, C.byref(outer), C.byref(inner), C.byref(hj), t, len(targets), C.byref(pool),
                                           C.byref(self.h)))

    def rows_raw(self):
        """(the output relation handle, slots, rows joined): gg_joinagg_rows"""
        rel, n, live = C.c_void_p(), C.c_uint64(0), C.c_uint64(0)
        check(dev_lib().gg_joinagg_rows(self.h, C.byref(rel), C.byref(n), C.byref(live)))
        return rel, n.value, live.value

    def rows(self):
        """the joined rows on the host, dead slots dropped: (values int64 [n][ncols], isnull bool [n][ncols], rows joined)"""
        rel, n, live = self.rows_raw()
        W = 1 + self.ncols
        nb = (n * W * 8 + capi.GG_BLCKSZ - 1) // capi.GG_BLCKSZ
        buf = np.zeros(nb * capi.GG_BLCKSZ // 8, dtype=np.uint64)
        if nb:
            check(dev_lib().gg_relation_read(rel, 0, buf.ctypes.data, nb))
        r = buf[:n * W].reshape(n, W)
        r = r[(r[:, 0] & np.uint64(1 << 63)) == 0]
        nulls = ((r[:, :1] >> np.arange(self.ncols, dtype=np.uint64)) & np.uint64(1)).astype(bool)
        return np.ascontiguousarray(r[:, 1:]).view(np.int64), nulls, live


def sort_rows(eng, keys, rows, nulls=None):
    """Sort n x ncols int64 Datum rows (host numpy) on the device; returns the sorted permutation (uint64)."""
    import numpy as np
    rows = np.ascontiguousarray(rows, dtype=np.int64)
    n, ncols = rows.shape
    ka = (capi.gg_sortkey * len(keys))(*keys)
    perm = np.zeros(n, dtype=np.uint64)
    if nulls is not None:
        nulls = np.ascontiguousarray(nulls, dtype=np.uint8)
    check(dev_lib().gg_sort_rows(eng.h, ka, len(keys), ncols, rows.ctypes.data,
                                 nulls.ctypes.data if nulls is not None else None, n, perm.ctypes.data))
    return perm


def agg_final_raw(eng, agg, buf, n, cap=4096):
    """gg_agg_final on a raw gg_aggrow buffer (numpy uint8); returns (buffer, n)"""
    out = np.zeros(cap * C.sizeof(capi.gg_aggrow), dtype=np.uint8)
    m = C.c_int(0)
    src = np.ascontiguousarray(buf)
    check(dev_lib().gg_agg_final(eng.h, C.byref(agg), C.cast(src.ctypes.data, C.POINTER(capi.gg_aggrow)), n,
                                 C.cast(out.ctypes.data, C.POINTER(capi.gg_aggrow)), cap, C.byref(m)))
    return out[:m.value * C.sizeof(capi.gg_aggrow)], m.value


def agg_final(eng, agg, rows, cap=4096):
    arr = (capi.gg_aggrow * max(len(rows), 1))()
    for i, r in enumerate(rows):
        C.memmove(C.byref(arr[i]), C.byref(r), C.sizeof(capi.gg_aggrow))
    out = (capi.gg_aggrow * cap)()
    n = C.c_int(0)
    check(dev_lib().gg_agg_final(eng.h, C.byref(agg), arr, len(rows), out, cap, C.byref(n)))
    return [out[i] for i in range(n.value)]


class Groups:
    """Aggregate rows left on the device as group records (gg_groups)."""

    def __init__(self, eng, h):
        self.eng, self.h = eng, h

    @classmethod
    def of(cls, pipeline):
        h = C.c_void_p()
        fn = dev_lib().gg_joinagg_groups if isinstance(pipeline, JoinAgg) else dev_lib().gg_scanagg_groups
        check(fn(pipeline.h, C.byref(h)))
        return cls(pipeline.eng, h)

    def final(self):
        """FINAL-stage combine on the device (gg_groups_final)"""
        h = C.c_void_p()
        check(dev_lib().gg_groups_final(self.eng.h, self.h, C.byref(h)))
        return Groups(self.eng, h)

    def datumrows(self, ncols):
        """the groups finalised on the device (gg_groups_datumrows): (values, isnull) of ncols = numCols + numAggs columns"""
        return _datumrows(dev_lib().gg_groups_datumrows, self.h, ncols)

    def fetch(self, cap=4096):
        out = (capi.gg_aggrow * cap)()
        n = C.c_int(0)
        sc, ps = C.c_uint64(0), C.c_uint64(0)
        check(dev_lib().gg_groups_fetch(self.h, out, cap, C.byref(n), C.byref(sc), C.byref(ps)))
        return [out[i] for i in range(n.value)], sc.value, ps.value

    def free(self):
        if self.h:
            dev_lib().gg_groups_free(self.h)
            self.h = C.c_void_p()


class Interconnect:
    """The Motion layer over NCCL (gg_interconnect): one communicator per query, rank = segment.  `unique_id` is the
    128 bytes one segment obtained from Interconnect.unique_id() and handed to the others (the dispatcher's job)."""

    @staticmethod
    def unique_id():
        buf = C.create_string_buffer(128)
        check(dev_lib().gg_ic_unique_id(buf, 128))
        return buf.raw

    def __init__(self, eng, nsegs=1, segindex=0, unique_id=None):
        self.eng, self.nsegs, self.segindex = eng, nsegs, segindex
        self.h = C.c_void_p()
        uid = C.create_string_buffer(unique_id, 128) if unique_id is not None else None
        check(dev_lib().gg_ic_create(eng.h, uid, nsegs, segindex, C.byref(self.h)))

    def allgather_u64(self, mine):
        out = (C.c_uint64 * self.nsegs)()
        check(dev_lib().gg_ic_allgather_u64(self.h, int(mine), out))
        return list(out)

    def collective_count(self):
        return dev_lib().gg_ic_collective_count(self.h)

    def motion_groups(self, groups, motion_type, hashcols=(), hashtypids=(), root=0):
        h = C.c_void_p()
        hc = (C.c_int32 * max(len(hashcols), 1))(*hashcols)
        ht = (C.c_int32 * max(len(hashtypids), 1))(*hashtypids)
        check(dev_lib().gg_ic_motion_groups(self.h, motion_type, root, len(hashcols), hc, ht, groups.h if groups is not None else None, 0, C.byref(h)))
        return Groups(self.eng, h)

    def exchange_rows(self, send_ptr, counts, region_cap, rowwords, recv_ptr, recv_cap):
        n = C.c_uint64(0)
        ca = (C.c_uint64 * len(counts))(*counts)
        check(dev_lib().gg_ic_exchange_rows(self.h, C.c_void_p(send_ptr), ca, region_cap, rowwords, C.c_void_p(recv_ptr), recv_cap, C.byref(n)))
        return n.value

    def close(self, has_errors=False):
        if self.h:
            dev_lib().gg_ic_teardown(self.h, 1 if has_errors else 0)
            self.h = C.c_void_p()
