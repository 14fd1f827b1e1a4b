"""GPU tests for the keys of every device key type — int4, int8, date, timestamp, bool, float8, bpchar, varchar, text — in
grouping, hash joins, Motion placement and Sort, against the oracle (oracle/: the reference's grouping, HashJoin, cdbhash and
sort comparator restated; cdbhash pinned to the reference's cdbhash.o by test_oracle_hash.py).

The key relation holds, per type, the values kernels get wrong: sign extension (INT32_MIN, -1), int8 pairs that collide in
hashint8 (0 / 2^32+1, -1 / 2^32-1), the int8 extremes, ±0 / ±inf / NaN / the smallest subnormal / DBL_MAX / 1.0 next to its
successor, bpchar values that are equal after blank stripping ('' = ' ', 'A' = 'A ') and 8-byte values padded past 8 bytes on
disk, varchar / text 'A' ≠ 'A ' and '' ≠ NULL, values that differ only in their last byte, and bytes >= 0x80.

Key rule: keys bit-exact, except that a NaN key matches any NaN and a float8 zero key is -0 when every zero input of its group
was -0 and +0 when every one was +0 (the reference keeps the first row's key); with both signs in the group either is right,
a parallel scan has no first row."""
import ctypes as C
import math

import numpy as np
import pytest

from _util import assert_aggrows_match, b2f, f2b, make_desc
from greengage_b200 import capi
from greengage_b200.capi import ExprPool
from oracle import pyoracle as po
from test_gpu_join import BOTH_SIDES, JOINTYPES, gpu_join_batched, gpu_joinagg
from test_gpu_scanagg import VARIANTS, gpu_scanagg
from test_gpu_sort import check_sorted

pytestmark = pytest.mark.gpu

INT4_MIN, INT4_MAX, INT8_MIN, INT8_MAX = -2**31, 2**31 - 1, -2**63, 2**63 - 1
NAN = b2f(0x7ff8000000000000)                             # the one NaN encoding of the relation
FLOATS = [0.0, math.inf, -math.inf, NAN, 5e-324, 1.7976931348623157e308, 1.0, math.nextafter(1.0, 2.0), -2.5]
STR_BP = [b"", b" ", b"A", b"A ", b"ABCDEFGH", b"ABCDEFGH  ", b"ABCDEFGI", b"\x80\xffA"]
STR_VT = [b"A", b"A ", b"", b"ABCDEFGH", b"ABCDEFGI", b"\x80\xff", b"ab "]
VALUES = {
    "int4": [0, 1, -1, INT4_MIN, INT4_MAX, -7, -65536, 123456],
    "int8": [0, 2**32 + 1, -1, 2**32 - 1, INT8_MIN, INT8_MAX, -5, 1],
    "date": [0, 1, -1, INT4_MIN, INT4_MAX, -730000, 36524],
    "timestamp": [0, 2**32 + 1, -1, 2**32 - 1, INT8_MIN, INT8_MAX, -86400000000],
    "bool": [0, 1],
    "float8": FLOATS,
    "bpchar": STR_BP,
    "varchar": STR_VT,
    "text": STR_VT,
}
# column layout of the key relation (attno = index + 1)
COLS = ["int4", "int8", "date", "timestamp", "bool", "float8", "bpchar", "varchar", "text", "z", "v", "w", "f0", "id"]
TYPID = {"int4": capi.INT4OID, "int8": capi.INT8OID, "date": capi.DATEOID, "timestamp": capi.TIMESTAMPOID, "bool": capi.BOOLOID,
         "float8": capi.FLOAT8OID, "bpchar": capi.BPCHAROID, "varchar": capi.VARCHAROID, "text": capi.TEXTOID,
         "z": capi.INT4OID, "v": capi.FLOAT8OID, "w": capi.INT8OID, "f0": capi.FLOAT8OID, "id": capi.INT4OID}
SPEC = {capi.INT4OID: (4, "i", 1), capi.INT8OID: (8, "d", 1), capi.DATEOID: (4, "i", 1), capi.TIMESTAMPOID: (8, "d", 1),
        capi.BOOLOID: (1, "c", 1), capi.FLOAT8OID: (8, "d", 1), capi.BPCHAROID: (-1, "i", 0), capi.VARCHAROID: (-1, "i", 0),
        capi.TEXTOID: (-1, "i", 0)}
KEYTYPES = list(VALUES) + ["f0"]
STRING = (capi.BPCHAROID, capi.VARCHAROID, capi.TEXTOID)


def col(name):
    return COLS.index(name) + 1


def key_relation(n, seed):
    """(desc, pages, rows, nulls): every key column nullable (8%); z in {0, 1, 2} sets the sign of a float8 zero key (-0, +0,
    either); f0 is float8 with every zero -0; v float8 / w int8 aggregate inputs; id the row number"""
    rng = np.random.default_rng(seed)
    desc = make_desc([(TYPID[c],) + SPEC[TYPID[c]] + (1 if c in ("z", "id") else 0,) for c in COLS])
    rows, nulls = [], []
    for i in range(n):
        r, nl = [], []
        z = int(rng.integers(0, 3))
        for c in COLS:
            if c == "z":
                r.append(z); nl.append(False); continue
            if c == "id":
                r.append(i); nl.append(False); continue
            if c == "v":
                r.append(float(rng.integers(-400, 400)) / 4); nl.append(bool(rng.random() < 0.1)); continue
            if c == "w":
                r.append(int(rng.choice([INT8_MIN, INT8_MAX, -1, 0, int(rng.integers(-2**40, 2**40))]))); nl.append(bool(rng.random() < 0.1)); continue
            vals = VALUES["float8" if c == "f0" else c]
            x = vals[int(rng.integers(0, len(vals)))]
            if c in ("float8", "f0") and x == 0:
                x = -0.0 if (c == "f0" or z == 0 or (z == 2 and rng.random() < 0.5)) else 0.0
            if c == "bpchar":
                x = x.ljust(10, b" ")                     # bpchar(10) on disk
            r.append(x)
            nl.append(bool(rng.random() < 0.08))
        rows.append(r)
        nulls.append(nl)
    return desc, po.build_pages(desc, rows, nulls), rows, nulls


_rel = {}


def rel(n=3000, seed=1):
    if (n, seed) not in _rel:
        _rel[(n, seed)] = key_relation(n, seed)
    return _rel[(n, seed)]


@pytest.fixture(scope="module")
def eng():
    from greengage_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


# ---- the key rule ----

def canon_value(name, x):
    """a python value of column `name` as the group it belongs to: ±0 one key, NaN one key, bpchar blank-stripped"""
    t = TYPID[name]
    if t == capi.FLOAT8OID:
        return "nan" if x != x else (0.0 if x == 0 else x)
    if t == capi.BPCHAROID:
        return bytes(x).rstrip(b" ")
    return x


def zero_signs(rows, nulls, keys, keep=None):
    """{canonical group: {key position: set of zero signs seen}} for the float8 keys, from the input rows"""
    out = {}
    for r, nl in zip(rows, nulls):
        if keep is not None and not keep(r):
            continue
        g = tuple(None if nl[col(k) - 1] else canon_value(k, r[col(k) - 1]) for k in keys)
        d = out.setdefault(g, {})
        for j, k in enumerate(keys):
            x = r[col(k) - 1]
            if TYPID[k] == capi.FLOAT8OID and not nl[col(k) - 1] and x == 0:
                d.setdefault(j, set()).add("-" if math.copysign(1, x) < 0 else "+")
    return out


def canon_row_key(r, keys):
    out = []
    for j, k in enumerate(keys):
        if r.keyisnull[j]:
            out.append(None)
        elif TYPID[k] == capi.FLOAT8OID:
            out.append(canon_value(k, b2f(r.key[j])))
        elif TYPID[k] in STRING:
            out.append(capi.unpack_str(r.key[j], r.keylen[j]).encode("latin1"))
        elif TYPID[k] in (capi.INT4OID, capi.DATEOID):
            out.append(int(np.uint32(r.key[j] & 0xFFFFFFFF).astype(np.int32)))
        else:
            out.append(int(r.key[j]))
    return tuple(out)


def canonical_copy(rows, keys):
    """copies of the rows with every float8 key normalised (±0 -> +0, NaN -> one encoding), for matching rows by key"""
    out = []
    for r in rows:
        c = capi.gg_aggrow()
        C.memmove(C.byref(c), C.byref(r), C.sizeof(capi.gg_aggrow))
        for j, k in enumerate(keys):
            if TYPID[k] == capi.FLOAT8OID and not c.keyisnull[j]:
                x = b2f(c.key[j])
                c.key[j] = f2b(NAN) if x != x else (0 if x == 0 else c.key[j])
        out.append(c)
    return out


def assert_keys_rule(got, want, agg, keys, signs, exact=None):
    """the key rule above, then the aggregates through assert_aggrows_match on canonical keys"""
    for who, rows in (("device", got), ("oracle", want)):
        for r in rows:
            g = canon_row_key(r, keys)
            assert g in signs, (who, g)
            for j, s in signs[g].items():
                if len(s) == 1 and not r.keyisnull[j]:
                    x = b2f(r.key[j])
                    assert x == 0 and (math.copysign(1, x) < 0) == (s == {"-"}), (who, g, j, s, hex(r.key[j] & (2**64 - 1)))
    assert_aggrows_match(canonical_copy(got, keys), canonical_copy(want, keys), agg, exact=exact)


# ---- grouping ----

KEYSETS = {k: [k] for k in KEYTYPES}
KEYSETS.update({"z,float8": ["z", "float8"], "float8,text": ["float8", "text"], "int8,bool": ["int8", "bool"],
                "int4,bpchar,float8": ["int4", "bpchar", "float8"], "bool,date,varchar,float8": ["bool", "date", "varchar", "float8"],
                "timestamp,f0,bpchar,int8": ["timestamp", "f0", "bpchar", "int8"]})
ALL_VARIANTS = ("f0", "float8", "z,float8", "bpchar", "float8,text", "int8,bool", "int4,bpchar,float8", "bool,date,varchar,float8")


def group_plan(keys, stage=capi.AGGSTAGE_NORMAL, num_groups=0, desc=None):
    """GROUP BY keys: count(*), count(v), sum(v), min(w), max(w)"""
    desc = desc or rel()[0]
    p = ExprPool()
    g = [p.var(col(k), TYPID[k]) for k in keys]
    v, w = p.var(col("v"), capi.FLOAT8OID), p.var(col("w"), capi.INT8OID)
    agg = capi.make_agg(stage, g, [(capi.AGG_COUNT_STAR, -1), (capi.AGG_COUNT_ANY, v), (capi.AGG_SUM_FLOAT8, v),
                                   (capi.AGG_MIN_INT8, w), (capi.AGG_MAX_INT8, w)], num_groups=num_groups)
    return capi.make_scan(desc, -1), agg, p.pool


@pytest.mark.parametrize("keyset", list(KEYSETS))
def test_group_keys_on_every_scan_agg_variant(eng, keyset):
    keys = KEYSETS[keyset]
    desc, pages, rows, nulls = rel()
    scan, agg, pool = group_plan(keys)
    want, wsc, wps, want_x = po.seqscan_agg(scan, agg, pool, pages, exact=True)
    signs = zero_signs(rows, nulls, keys)
    assert len(want) == len(signs)
    for variant in (VARIANTS if keyset in ALL_VARIANTS else ("interp-priv", "interp-tr")):
        got, sc, ps, var = gpu_scanagg(eng, scan, agg, pool, pages, variant)
        if variant.startswith(("specialised", "nvrtc")):
            assert var >= 16, (variant, var)
        else:
            assert var < 16, (variant, var)
        assert (sc, ps) == (wsc, wps)
        assert_keys_rule(got, want, agg, keys, signs, exact=want_x)


@pytest.mark.parametrize("keyset", list(KEYSETS))
def test_group_keys_on_the_general_hash_aggregate(eng, keyset):
    """the group table in HBM from a planner estimate of 500 groups, and grown from an estimate of 16"""
    keys = KEYSETS[keyset]
    desc, pages, rows, nulls = rel()
    signs = zero_signs(rows, nulls, keys)
    for est in (500, 16):
        scan, agg, pool = group_plan(keys, num_groups=est)
        want, _, _, want_x = po.seqscan_agg(scan, agg, pool, pages, exact=True)
        got, _, _, _ = gpu_scanagg(eng, scan, agg, pool, pages)
        assert_keys_rule(got, want, agg, keys, signs, exact=want_x)


def final_of(pagg, keys):
    fin = capi.gg_agg()
    C.memmove(C.byref(fin), C.byref(pagg), C.sizeof(capi.gg_agg))
    fin.aggstage = capi.AGGSTAGE_FINAL
    for j, k in enumerate(keys):
        fin.grpCol[j] = TYPID[k]                                  # a FINAL Agg's grpCol carries the key type OIDs
    return fin


@pytest.mark.parametrize("keyset", ["f0", "float8", "z,float8", "float8,text", "int4,bpchar,float8", "bool,date,varchar,float8",
                                    "timestamp,f0,bpchar,int8", "int4", "varchar", "bool"])
def test_group_keys_through_partial_and_final(eng, keyset):
    """PARTIAL over two halves -> agg_final on the host rows, and Groups.of(PARTIAL pipeline).final() on the device records"""
    from greengage_b200.engine import Groups, Relation, ScanAgg, agg_final
    keys = KEYSETS[keyset]
    desc, pages, rows, nulls = rel()
    signs = zero_signs(rows, nulls, keys)
    scan, pagg, pool = group_plan(keys, capi.AGGSTAGE_PARTIAL)
    fin = final_of(pagg, keys)
    nb = pages.size // capi.GG_BLCKSZ
    parts = []
    for a, b in ((0, nb // 2), (nb // 2, nb)):
        r, _, _, _ = gpu_scanagg(eng, scan, pagg, pool, pages, ranges=[(a, b)])
        parts += r
    got = agg_final(eng, fin, parts)
    want = po.agg_final(fin, parts)
    assert_keys_rule(got, want, fin, keys, signs)
    nscan, nagg, npool = group_plan(keys)
    one, _, _ = po.seqscan_agg(nscan, nagg, npool, pages)
    assert len(one) == len(got)
    r = Relation(eng, host_pages=pages)
    sa = ScanAgg(eng, scan, pagg, pool)
    try:
        for b in range(r.nblocks):
            sa.run(r, b, 1)
        part, _, _ = sa.fetch()
        try:
            g = Groups.of(sa)
        except capi.GGError as e:                                 # groups kept in the general hash table: rows only
            assert e.code == -6
            return
        f = g.final()
        try:
            got2, _, _ = f.fetch()
        finally:
            f.free()
            g.free()
        assert_keys_rule(got2, po.agg_final(fin, part), fin, keys, signs)
    finally:
        sa.free()
        r.free()


# ---- joins ----

JOINKEYS = {k: (k, k) for k in VALUES}
JOINKEYS["int4=int8"] = ("int4", "int8")
JOINKEYS["int8=int4"] = ("int8", "int4")


def join_plan(okey, ikey, jointype, nkeys):
    desc = rel()[0]
    p = ExprPool()
    ok, ik = [p.var(col(okey), TYPID[okey], 0)], [p.var(col(ikey), TYPID[ikey], 1)]
    if nkeys == 2:
        ok.append(p.var(col("z"), capi.INT4OID, 0))
        ik.append(p.var(col("z"), capi.INT4OID, 1))
    hj = capi.make_hashjoin(jointype, ok, ik)
    aggs = [(capi.AGG_COUNT_STAR, -1), (capi.AGG_SUM_FLOAT8, p.var(col("v"), capi.FLOAT8OID, 0))]
    if jointype in BOTH_SIDES:
        aggs += [(capi.AGG_COUNT_ANY, p.var(col("w"), capi.INT8OID, 1)), (capi.AGG_MAX_INT8, p.var(col("w"), capi.INT8OID, 1))]
    agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [p.var(col("z"), capi.INT4OID, 0)], aggs)
    return capi.make_scan(desc, -1), capi.make_scan(desc, -1), hj, agg, p.pool


@pytest.mark.parametrize("nkeys", [1, 2])
@pytest.mark.parametrize("pair", list(JOINKEYS))
def test_join_keys_of_every_type(eng, pair, nkeys):
    """every join type on the one-table path, and every type with a probe side batched (the batch bits come from each side's
    own hash type, so int4 and int8 keys of equal value land in the same batch)"""
    okey, ikey = JOINKEYS[pair]
    _, opages, _, _ = rel(1200, 11)
    _, ipages, _, _ = rel(250, 12)
    for jt in JOINTYPES:
        outer, inner, hj, agg, pool = join_plan(okey, ikey, jt, nkeys)
        want, nj_want, want_x = po.hashjoin_agg(outer, inner, hj, agg, pool, opages, ipages, exact=True)
        got, nj, _ = gpu_joinagg(eng, outer, inner, hj, agg, pool, opages, ipages)
        assert nj == nj_want, (pair, jt)
        assert_aggrows_match(got, want, agg, exact=want_x)
        if jt == capi.JOIN_LASJ_NOTIN:
            continue
        got, nj, nbatch, _ = gpu_join_batched(eng, outer, inner, hj, agg, pool, opages, ipages, work_mem=8192)
        assert nbatch >= 2 and nj == nj_want, (pair, jt, nbatch, nj, nj_want)
        assert_aggrows_match(got, want, agg, exact=want_x)


# ---- Motion ----

def route_one(typid, x):
    """the oracle's routing input for one python value: (datum, len)"""
    if typid == capi.FLOAT8OID:
        return f2b(x), 0
    if typid in STRING:
        return capi.pack_str(x, typid == capi.BPCHAROID)
    return int(x), 0


MOTIONKEYS = [[k] for k in KEYTYPES] + [["bool", "int8", "float8", "text"], ["int4", "bpchar", "timestamp"], ["date", "varchar"]]


@pytest.mark.parametrize("keys", MOTIONKEYS, ids=[",".join(k) for k in MOTIONKEYS])
def test_motion_placement_of_every_key_type(eng, keys):
    """each live row sits in the region of the segment the reference's cdbhash sends it to (po.motion_route), and a sample
    of rows routes there through or_route_datums from the input values"""
    from test_gpu_motion import partition
    desc, pages, rows, nulls = rel()
    p = ExprPool()
    hk = [p.var(col(k), TYPID[k]) for k in keys]
    payload = [p.var(col("id"), capi.INT4OID)]
    scan = capi.make_scan(desc, -1)
    DEAD = np.int64(-2**63)
    for nsegs in (1, 2, 3, 7, 8, 64, 1024):
        dest = po.motion_route(scan, p.pool, hk, nsegs, pages)
        assert len(dest) == len(rows)
        counts, offs, words, buf = partition(eng, scan, p, hk, payload, nsegs, pages, len(rows) * 2 + 4096 * nsegs)
        try:
            for d in range(nsegs):
                reg = words[offs[d]:offs[d] + counts[d]]
                reg = reg[(reg[:, 0] & DEAD) == 0]
                assert sorted(reg[:, 1].tolist()) == np.nonzero(dest == d)[0].tolist(), (keys, nsegs, d)
        finally:
            buf.free()
        for i in range(0, len(rows), 37):
            n = len(keys)
            dl = [route_one(TYPID[k], rows[i][col(k) - 1]) for k in keys]
            t = (C.c_int32 * n)(*[TYPID[k] for k in keys])
            v = (C.c_int64 * n)(*[x for x, _ in dl])
            ln = (C.c_int32 * n)(*[x for _, x in dl])
            nn = (C.c_int32 * n)(*[int(nulls[i][col(k) - 1]) for k in keys])
            assert po.lib().or_route_datums(t, v, ln, nn, n, nsegs) == dest[i], (keys, nsegs, i)


# ---- Sort ----

def datums(name, n, rng):
    t = TYPID[name]
    vals = VALUES["float8" if name == "f0" else name]
    xs = [vals[int(i)] for i in rng.integers(0, len(vals), n)]
    if t == capi.FLOAT8OID:
        return np.array([f2b(-0.0 if (x == 0 and rng.random() < 0.5) else x) for x in xs], dtype=np.int64)
    if t in STRING:
        return np.array([capi.pack_str(x, t == capi.BPCHAROID)[0] for x in xs], dtype=np.int64)
    return np.array(xs, dtype=np.int64)


@pytest.mark.parametrize("name", list(VALUES))
def test_sort_keys_of_every_type(eng, name):
    """ASC / DESC x NULLS FIRST / LAST over 50 000 rows (several tiles) of the type's edge values, then the type as the second
    key under an int8 key that varies only in its top byte (the radix passes that see no difference are skipped)"""
    from greengage_b200.engine import sort_rows
    rng = np.random.default_rng(len(name))
    n = 50_000
    k = datums(name, n, rng)
    rows = np.stack([k, np.arange(n)], axis=1)
    nulls = np.zeros_like(rows, dtype=np.uint8)
    nulls[:, 0] = rng.random(n) < 0.05
    for desc in (False, True):
        for nf in (False, True):
            keys = [capi.make_sortkey(0, TYPID[name], desc, nf)]
            check_sorted(keys, rows, nulls, sort_rows(eng, keys, rows, nulls))
    top = (rng.integers(-128, 128, n).astype(np.int64) << 56)
    rows2 = np.stack([top, k, np.arange(n)], axis=1)
    nulls2 = np.zeros_like(rows2, dtype=np.uint8)
    nulls2[:, 1] = nulls[:, 0]
    keys = [capi.make_sortkey(0, capi.INT8OID), capi.make_sortkey(1, TYPID[name], True, False)]
    check_sorted(keys, rows2, nulls2, sort_rows(eng, keys, rows2, nulls2))
    keys = [capi.make_sortkey(0, capi.INT8OID, True)]
    perm = sort_rows(eng, keys, rows2[:, :1])
    assert np.all(np.diff(top[perm.astype(np.int64)]) <= 0)


def test_sort_datumrows_drops_dead_slots_and_orders_the_live_rows(eng):
    """gg_sort_datumrows over GG_FMT_DATUMROWS rows with dead slots (mask bit 63) between them, as a windowed Motion leaves
    them: the output is exactly the live rows, in comparator order (float8 DESC NULLS LAST, then text, then bool)"""
    from greengage_b200.engine import Relation
    rng = np.random.default_rng(9)
    n = 30_000
    cols = [datums("float8", n, rng), datums("text", n, rng), datums("bool", n, rng), np.arange(n, dtype=np.int64)]
    mask = np.zeros(n, dtype=np.int64)
    for c in range(3):
        mask |= (rng.random(n) < 0.05).astype(np.int64) << c
    dead = rng.random(n) < 0.2
    mask[dead] = np.int64(-2**63)
    words = np.stack([mask] + cols, axis=1).astype(np.int64)
    keys = [capi.make_sortkey(0, capi.FLOAT8OID, True, False), capi.make_sortkey(1, capi.TEXTOID), capi.make_sortkey(2, capi.BOOLOID)]
    W = words.shape[1]
    nbytes = words.nbytes
    nbl = (nbytes + capi.GG_BLCKSZ - 1) // capi.GG_BLCKSZ
    host = np.zeros(nbl * capi.GG_BLCKSZ, dtype=np.uint8)
    host[:nbytes] = words.view(np.uint8).reshape(-1)
    src, dst = Relation(eng, host_pages=host), Relation(eng, nblocks=nbl)
    try:
        nlive, passes = C.c_uint64(0), C.c_int(0)
        ka = (capi.gg_sortkey * len(keys))(*keys)
        capi.check(capi.dev_lib().gg_sort_datumrows(eng.h, ka, len(keys), W - 1, C.c_void_p(src.device_ptr()), n,
                                                    C.c_void_p(dst.device_ptr()), C.byref(nlive), C.byref(passes)))
        out = dst.read().view(np.int64)[:nlive.value * W].reshape(-1, W)
    finally:
        src.free()
        dst.free()
    live = words[~dead]
    assert nlive.value == len(live)
    assert sorted(out[:, 4].tolist()) == sorted(live[:, 4].tolist())
    assert np.all(out[:, 0] >= 0)
    lrows = live[:, 1:]
    lnulls = np.stack([(live[:, 0] >> c) & 1 for c in range(4)], axis=1).astype(np.uint8)
    pos = {int(i): r for r, i in enumerate(live[:, 4])}
    perm = np.array([pos[int(i)] for i in out[:, 4]], dtype=np.uint64)
    check_sorted(keys, lrows, lnulls, perm)


# ---- refusals ----

def test_nine_byte_string_keys_are_refused_never_truncated(eng):
    """a 9-byte non-blank string as a grouping, join or Motion key: GG_ERR_UNSUPPORTED, never an answer on its first 8 bytes
    (the strings differ only in their ninth byte, so a truncated key would merge them)"""
    from test_gpu_motion import partition
    desc = make_desc([(capi.TEXTOID, -1, "i", 0), (capi.BPCHAROID, -1, "i", 0), (capi.INT4OID, 4, "i", 1)])
    rows = [[b"ABCDEFGH" + bytes([65 + i % 3]), b"ABCDEFGH" + bytes([65 + i % 3]), i] for i in range(600)]
    pages = po.build_pages(desc, rows)
    for c, t in ((1, capi.TEXTOID), (2, capi.BPCHAROID)):
        p = ExprPool()
        agg = capi.make_agg(capi.AGGSTAGE_NORMAL, [p.var(c, t)], [(capi.AGG_COUNT_STAR, -1)])
        for variant in ("interp-tr", "specialised-priv"):
            with pytest.raises(capi.GGError) as e:
                gpu_scanagg(eng, capi.make_scan(desc, -1), agg, p.pool, pages, variant)
            assert e.value.code == -6, (t, variant)
        hagg = capi.make_agg(capi.AGGSTAGE_NORMAL, [p.var(c, t)], [(capi.AGG_COUNT_STAR, -1)], num_groups=500)
        with pytest.raises(capi.GGError) as e:
            gpu_scanagg(eng, capi.make_scan(desc, -1), hagg, p.pool, pages)
        assert e.value.code == -6, t
        hj = capi.make_hashjoin(capi.JOIN_INNER, [p.var(c, t, 0)], [p.var(c, t, 1)])
        jagg = capi.make_agg(capi.AGGSTAGE_NORMAL, [], [(capi.AGG_COUNT_STAR, -1)])
        with pytest.raises(capi.GGError) as e:
            gpu_joinagg(eng, capi.make_scan(desc, -1), capi.make_scan(desc, -1), hj, jagg, p.pool, pages, pages)
        assert e.value.code == -6, t
        key = p.var(c, t)
        with pytest.raises(capi.GGError) as e:
            counts, offs, words, buf = partition(eng, capi.make_scan(desc, -1), p, [key], [p.var(3, capi.INT4OID)], 4, pages, 8192)
            buf.free()
        assert e.value.code == -6, t
