"""String dictionaries in program pipelines (LDB_OP_STRCODE, ldb_gpu_dict_*), multi-key ORDER BY and string gathers on the GPU,
checked against plain Python over the same bytes: Python's bytes order is the bytewise, unsigned, prefix-first order of LDB_OP_STRCMP
(tests/_progref.py pins it).  Codes are dense but which string gets which code is unspecified, so every check decodes them."""
import ctypes as C
import hashlib
import json
import os
import random
from collections import Counter

import numpy as np
import pytest

import _keyhash as K

from lingodb_b200 import capi, dbgen, program as P, runtime
from lingodb_b200.datagen import ColumnSpec

pytestmark = pytest.mark.gpu

col, const = (lambda n: ("col", n)), (lambda v: ("const", v))


def utf8(values):
    """bytes | None values → Arrow utf8 buffers (int32 offsets, bytes) and a validity bitmap"""
    offs = np.zeros(len(values) + 1, np.int32)
    offs[1:] = np.cumsum([len(v or b"") for v in values])
    data = np.frombuffer(b"".join(v or b"" for v in values) + b"\0", np.uint8).copy()
    valid = np.packbits(np.array([v is not None for v in values], bool), bitorder="little")
    return offs, data, valid


def make_table(ctx, name, columns, sizes=None, offset=0):
    """columns: {name: (phys, values)} with phys "utf8" (bytes | None) or "int32" / "int64"; sizes: rows per batch (one batch by
    default); offset: each batch is an Arrow slice that starts `offset` rows into its buffers"""
    n = len(next(iter(columns.values()))[1])
    sizes = sizes or [n]
    assert sum(sizes) == n
    t = runtime.Table(ctx, name, [ColumnSpec(c, phys) for c, (phys, _) in columns.items()])
    start = 0
    for m in sizes:
        chunk = {}
        for c, (phys, values) in columns.items():
            part = values[start:start + m]
            if phys == "utf8":
                offs, data, valid = utf8([b"pad%d" % i for i in range(offset)] + part)
                chunk[c] = (offs, data)
                if any(v is None for v in part):
                    chunk[c + "$valid"] = valid
            else:
                chunk[c] = np.array([0] * offset + part, dtype=np.int32 if phys == "int32" else np.int64)
        t.append_host(chunk, m, offset=offset)
        start += m
    return t


def codes_of(ctx, table, expr):
    """the value of `expr` for every row of `table`, in row order (None for NULL)"""
    mt = P.RawTable(ctx, P.materialize(ctx, table, [("rowid",), expr]))
    ids = list(range(mt.num_rows))
    rows = dict(zip(mt.gather("c0", ids), mt.gather("c1", ids)))
    mt.destroy()
    return [rows[i] for i in range(len(rows))]


def decode(ctx, d, codes):
    dt = P.dict_table(ctx, d)
    known = sorted({c for c in codes if c is not None})
    strs = dict(zip(known, dt.gather_strings("str", known, decode=False)))
    dt.destroy()
    return [None if c is None else strs[c] for c in codes]


def raises(code, fn, *a, **kw):
    with pytest.raises(capi.LdbRuntimeError) as e:
        fn(*a, **kw)
    assert e.value.code == code, str(e.value)
    return e.value


EDGE = ([b"", b"a", b"ab", b"ab\0", b"ab\0\0", b"\0", b"\0\0a", b"\x80", b"\xff\xfe", b"a\x80b", b"x" * 1000, b"x" * 999 + b"y"]
        + [bytes(range(65, 65 + n)) for n in range(1, 65)]
        + [b"PREFIX08" + s for s in (b"", b"1", b"2", b"PREFIX16", b"PREFIX16a", b"PREFIX16PREFIX24", b"PREFIX16PREFIX24z")]
        + [b"\xc3\xa9t\xc3\xa9", b"\x7f", b"\x80\x00", None])


def edge_values(n, seed):
    r = random.Random(seed)
    return [r.choice(EDGE) for _ in range(n)]


@pytest.mark.parametrize("layout", ["ragged", "offsets", "side"])
def test_round_trip(gpu_ctx, layout):
    vals = edge_values(4000, 1) + EDGE
    distinct = {v for v in vals if v is not None}
    d = P.dict_state(gpu_ctx, len(distinct), sum(map(len, distinct)))
    if layout == "ragged":
        t = make_table(gpu_ctx, "s", {"s": ("utf8", vals)}, sizes=[1, 31, 33, 3000, len(vals) - 3065])
        expr = lambda mode=(): ("strcode", d, "s") + mode
    elif layout == "offsets":
        t = None
        for off in range(1, 8):  # one table per Arrow slice offset, all encoded into the same dictionary
            tt = make_table(gpu_ctx, "s%d" % off, {"s": ("utf8", vals)}, sizes=[1000, 1000, 1000, len(vals) - 3000], offset=off)
            assert decode(gpu_ctx, d, codes_of(gpu_ctx, tt, ("strcode", d, "s"))) == vals
            t = t or tt
        expr = lambda mode=(): ("strcode", d, "s") + mode
    else:  # side column read through a ROWID join: row i of the probe table reads the build table's row at key (i * 7) % n
        n = len(vals)
        src = make_table(gpu_ctx, "src", {"k": ("int32", list(range(n))), "s": ("utf8", vals)}, sizes=[700, 1300, n - 2000])
        jt = runtime.join_table(gpu_ctx, n)
        P.build_join(gpu_ctx, src, jt, col("k"), payload=("rowid",))
        keys = [(i * 7) % n for i in range(n)]
        t = make_table(gpu_ctx, "probe", {"pk": ("int32", keys)}, sizes=[999, n - 999])
        fetched = ("fetch", src, ("probe", jt, col("pk")), "s")
        expr = lambda mode=(): ("strcode", d, fetched) + mode
        vals = [vals[k] for k in keys]
    codes = codes_of(gpu_ctx, t, expr())
    n_codes = P.dict_count(gpu_ctx, d)
    assert n_codes == len(distinct)
    assert sorted({c for c in codes if c is not None}) == list(range(n_codes))  # dense
    assert [c is None for c in codes] == [v is None for v in vals]  # NULL gives NULL
    assert decode(gpu_ctx, d, codes) == vals
    assert codes_of(gpu_ctx, t, expr()) == codes  # a second encode gives the same codes
    assert codes_of(gpu_ctx, t, expr(("lookup",))) == codes
    # lookup on another table: the same code for a known string, NULL for an absent one, and nothing is inserted
    probe = [b"absent", vals[5], b"ab\0\0\0", None, vals[17], b"x" * 1001]
    other = make_table(gpu_ctx, "other", {"s": ("utf8", probe)})
    want = [None if v is None or v not in distinct else codes[vals.index(v)] for v in probe]
    assert codes_of(gpu_ctx, other, ("strcode", d, "s", "lookup")) == want
    assert P.dict_count(gpu_ctx, d) == n_codes
    gpu_ctx.L.ldb_gpu_state_destroy(d)


def test_tag_collision_compares_the_whole_string(gpu_ctx):
    """Two strings that share their first 8 bytes and, in a 16-slot directory, their home slot and their 32-bit tag (found with the
    hash of tests/_keyhash.py, pinned to strHash in csrc/keyhash.cuh): the dictionary must still tell them apart."""
    h = K.str_hash
    a, b = b"COLLIDE#imldaaaa", b"COLLIDE#hzlbiaaa"
    assert h(a) >> 32 == h(b) >> 32 and h(a) & 15 == h(b) & 15  # still a collision for the current hash
    for vals in ([a, b] * 200, [b, a], [a] * 100 + [b] * 100):
        d = P.dict_state(gpu_ctx, 8, 64)
        t = make_table(gpu_ctx, "c", {"s": ("utf8", vals)})
        codes = codes_of(gpu_ctx, t, ("strcode", d, "s"))
        assert P.dict_count(gpu_ctx, d) == 2
        assert decode(gpu_ctx, d, codes) == vals
        gpu_ctx.L.ldb_gpu_state_destroy(d)


def test_contention_and_scale(gpu_ctx):
    three = [b"REGULAR AIR", b"REGULAR AIR FREIGHT", b"R"]
    idx = np.random.default_rng(3).integers(0, 3, 4 << 20)
    offs, data = dbgen._categorical_utf8(idx, [s.decode() for s in three])
    t = runtime.Table(gpu_ctx, "many", [ColumnSpec("s", "utf8")])
    t.append_host({"s": (offs.astype(np.int32), data)}, len(idx))
    d = P.dict_state(gpu_ctx, 3, 64)
    st = P.group_by(gpu_ctx, t, [("strcode", d, "s")], [("count_star", None)], expected_groups=16)
    assert P.dict_count(gpu_ctx, d) == 3
    got = P.decode_groups(P.read_groups(gpu_ctx, st, 16), 1, 1)
    strs = decode(gpu_ctx, d, [k for (k,) in got])
    assert {s: got[(k,)][0] for s, (k,) in zip(strs, got)} == {three[i]: int(c) for i, c in enumerate(np.bincount(idx, minlength=3))}
    gpu_ctx.L.ldb_gpu_state_destroy(st)
    gpu_ctx.L.ldb_gpu_state_destroy(d)
    # 2 M distinct strings of random lengths
    r = random.Random(4)
    n = 2 << 20
    vals = [b"%08x" % i + r.randbytes(r.randrange(0, 9)) * r.randrange(1, 5) for i in range(n)]
    r.shuffle(vals)
    d = P.dict_state(gpu_ctx, n, sum(map(len, vals)))
    t = make_table(gpu_ctx, "distinct", {"s": ("utf8", vals)}, sizes=[1 << 20, n - (1 << 20)])
    codes = codes_of(gpu_ctx, t, ("strcode", d, "s"))
    assert P.dict_count(gpu_ctx, d) == n and sorted(codes) == list(range(n))
    dt = P.dict_table(gpu_ctx, d)
    strs = dt.gather_strings("str", list(range(n)), decode=False)
    assert [strs[c] for c in codes] == vals
    ranks = dt.gather("rank", list(range(n)), cell_bytes=4)
    order = sorted(range(n), key=strs.__getitem__)
    assert [ranks[c] for c in order] == list(range(n))
    dt.destroy()
    gpu_ctx.L.ldb_gpu_state_destroy(d)


def test_ranks_are_the_bytewise_order(gpu_ctx):
    vals = EDGE + [bytes([b]) * k for b in (0, 1, 0x7f, 0x80, 0xff) for k in (1, 2, 8, 9, 17)]
    d = P.dict_state(gpu_ctx, len(vals), 8192)
    t = make_table(gpu_ctx, "r", {"s": ("utf8", vals)})
    codes_of(gpu_ctx, t, ("strcode", d, "s"))
    dt = P.dict_table(gpu_ctx, d)
    n = dt.num_rows
    strs = dt.gather_strings("str", list(range(n)), decode=False)
    want = sorted(set(v for v in vals if v is not None))
    assert sorted(strs) == want
    assert dt.gather("rank", list(range(n)), cell_bytes=4) == [want.index(s) for s in strs]
    dt.destroy()
    gpu_ctx.L.ldb_gpu_state_destroy(d)


def test_group_by_long_strings_whose_prefixes_collide(gpu_ctx):
    types = [b"STANDARD BRUSHED TIN", b"STANDARD BRUSHED COPPER", b"STANDARD BURNISHED NICKEL", b"STANDARD POLISHED TIN", None]
    conts = [b"MEDIUM POLISHED BOX", b"MEDIUM POLISHED BAG", b"MED BOX", b"\x80MEDIUM POLISHED BOX"]
    r = random.Random(5)
    n = 50_000
    a, b = [r.choice(types) for _ in range(n)], [r.choice(conts) for _ in range(n)]
    v = [r.randrange(-10**12, 10**12) for _ in range(n)]
    t = make_table(gpu_ctx, "g", {"a": ("utf8", a), "b": ("utf8", b), "v": ("int64", v)}, sizes=[20_000, n - 20_000])
    da, db = P.dict_state(gpu_ctx, 8, 256), P.dict_state(gpu_ctx, 8, 256)
    st = P.group_by(gpu_ctx, t, [("strcode", da, "a"), ("strcode", db, "b")], [("count_star", None), ("sum", col("v"))], expected_groups=64)
    got = P.decode_groups(P.read_groups(gpu_ctx, st, 64), 2, 2)
    keys = list(got)
    sa, sb = decode(gpu_ctx, da, [k[0] for k in keys]), decode(gpu_ctx, db, [k[1] for k in keys])
    want = {}
    for x, y, z in zip(a, b, v):
        c = want.setdefault((x, y), [0, 0])
        c[0] += 1
        c[1] += z
    assert {(x, y): got[k] for x, y, k in zip(sa, sb, keys)} == want
    assert len(want) == len(got) > 16  # STRKEY8 would merge the groups of each 8-byte prefix
    gpu_ctx.L.ldb_gpu_state_destroy(st)
    for s_ in (da, db):
        gpu_ctx.L.ldb_gpu_state_destroy(s_)


def test_string_equi_join(gpu_ctx):
    r = random.Random(6)
    pool = [b"k%03d-" % i + b"z" * r.randrange(0, 30) for i in range(40)] + [None]
    bs = [r.choice(pool) for _ in range(3000)]
    ps = [r.choice(pool + [b"unmatched", b"k000"]) for _ in range(5000)]
    bt = make_table(gpu_ctx, "build", {"bs": ("utf8", bs), "bid": ("int32", list(range(len(bs))))}, sizes=[1000, 2000])
    pt = make_table(gpu_ctx, "probe", {"ps": ("utf8", ps), "pid": ("int32", list(range(len(ps))))}, sizes=[2500, 2500])
    d = P.dict_state(gpu_ctx, 64, 4096)
    jt = runtime.join_table(gpu_ctx, len(bs), unique=False)
    P.build_join(gpu_ctx, bt, jt, ("strcode", d, "bs"), payload=("rowid",))
    n_codes = P.dict_count(gpu_ctx, d)
    m = ("probe_each", jt, ("strcode", d, "ps", "lookup"))
    mt = P.RawTable(gpu_ctx, P.materialize(gpu_ctx, pt, [col("pid"), ("fetch", bt, m, "bid")]))
    ids = list(range(mt.num_rows))
    got = Counter(zip(mt.gather("c0", ids), mt.gather("c1", ids)))
    want = Counter((i, j) for i, x in enumerate(ps) if x is not None for j, y in enumerate(bs) if y == x)
    assert got == want and len(want) > 1000
    assert P.dict_count(gpu_ctx, d) == n_codes  # the probe side only looked up
    mt.destroy()
    for s_ in (jt, d):
        gpu_ctx.L.ldb_gpu_state_destroy(s_)


def test_order_by_keys(gpu_ctx):
    r = random.Random(7)
    n = 3000
    strs = [b"ab\0", b"ab", b"ab\0\0", b"", b"\x80", b"\xff", b"a\x80", b"PREFIX08PREFIX16x", b"PREFIX08PREFIX16", b"PREFIX08Z", b"z" * 40]
    cols = {"i": ("int32", [r.randrange(-3, 4) for _ in range(n)]), "s": ("utf8", [r.choice(strs) for _ in range(n)]),
            "l": ("int64", [r.choice([-2**62, -1, 0, 5, 2**62]) for _ in range(n)]), "u": ("utf8", [r.choice(strs[:4]) for _ in range(n)]),
            "f": ("int32", list(range(n)))}
    t = P.RawTable(gpu_ctx, make_table(gpu_ctx, "o", cols).h)
    for keys in ([("s", False)], [("s", True)], [("u", False)], [("i", False), ("s", True)], [("s", False), ("l", True), ("i", False)],
                 [("u", True), ("i", True), ("s", False), ("l", False)], [("l", False), ("u", False)]):
        want = list(range(n))
        for c, desc in reversed(keys):  # stable sorts, the last key first
            want.sort(key=lambda i: cols[c][1][i], reverse=desc)
        assert t.order_by_keys(keys) == want, keys
        assert t.order_by_keys(keys, limit=17) == want[:17]
    assert t.order_by_keys([("s", False)], limit=0) == []
    raises(capi.LDB_ERR_INVALID, t.order_by_keys, [("nope", False)])
    ragged = P.RawTable(gpu_ctx, make_table(gpu_ctx, "two", {"s": ("utf8", [b"a", b"b", b"c"])}, sizes=[1, 2]).h)
    raises(capi.LDB_ERR_UNSUPPORTED, ragged.order_by_keys, [("s", False)])


def test_gather_strings(gpu_ctx):
    vals = edge_values(5000, 8)
    t = P.RawTable(gpu_ctx, make_table(gpu_ctx, "gs", {"s": ("utf8", vals)}).h)
    r = random.Random(9)
    ids = [r.randrange(5000) for _ in range(300)] + list(range(100, 400)) + list(range(4990, 5000)) + [0, 0, 1]
    assert t.gather_strings("s", ids, decode=False) == [vals[i] for i in ids]
    assert t.gather_strings("s", []) == []
    # a buffer one byte too small: LDB_ERR_CAPACITY, the bytes needed, nothing else written
    need = sum(len(vals[i] or b"") for i in ids)
    n = len(ids)
    arr, offs, valid = (C.c_int64 * n)(*ids), (C.c_int64 * (n + 1))(*([-7] * (n + 1))), (C.c_uint8 * n)(*([9] * n))
    buf, got, e = (C.c_uint8 * need)(*([0xAB] * need)), C.c_int64(), capi.Error()
    rc = gpu_ctx.L.ldb_gpu_table_gather_strings(t.h, b"s", arr, n, offs, buf, need - 1, C.byref(got), valid, C.byref(e))
    assert rc == capi.LDB_ERR_CAPACITY and got.value == need
    assert list(offs) == [-7] * (n + 1) and list(valid) == [9] * n and bytes(buf) == b"\xab" * need
    rc = gpu_ctx.L.ldb_gpu_table_gather_strings(t.h, b"s", arr, n, offs, buf, need, C.byref(got), valid, C.byref(e))
    assert rc == capi.LDB_OK and [bytes(buf)[offs[i]:offs[i + 1]] if valid[i] else None for i in range(n)] == [vals[i] for i in ids]
    raises(capi.LDB_ERR_INVALID, t.gather_strings, "s", [5000])
    raises(capi.LDB_ERR_INVALID, t.gather_strings, "nope", [0])


def test_documented_errors(gpu_ctx):
    vals = [b"string number %d" % i for i in range(100)]
    t = make_table(gpu_ctx, "e", {"s": ("utf8", vals), "k": ("int32", list(range(100)))})
    small = P.dict_state(gpu_ctx, 8, 1 << 16)  # 16 directory slots
    raises(capi.LDB_ERR_CAPACITY, codes_of, gpu_ctx, t, ("strcode", small, "s"))
    arena = P.dict_state(gpu_ctx, 1000, 40)
    raises(capi.LDB_ERR_CAPACITY, codes_of, gpu_ctx, t, ("strcode", arena, "s"))
    raises(capi.LDB_ERR_CAPACITY, P.dict_count, gpu_ctx, arena)
    raises(capi.LDB_ERR_CAPACITY, P.dict_table, gpu_ctx, arena)
    d = P.dict_state(gpu_ctx, 128, 4096)
    raises(capi.LDB_ERR_INVALID, codes_of, gpu_ctx, t, ("strcode", d, "k"))  # not a utf8 column
    jt = runtime.join_table(gpu_ctx, 128)
    raises(capi.LDB_ERR_INVALID, codes_of, gpu_ctx, t, ("strcode", jt, "s"))  # a join table is no dictionary
    raises(capi.LDB_ERR_INVALID, codes_of, gpu_ctx, t, ("probe", d, col("k")))  # a dictionary is no join table
    raises(capi.LDB_ERR_INVALID, codes_of, gpu_ctx, t, ("probe_each", d, col("k")))
    with runtime.Context(0) as other:
        foreign = P.dict_state(other, 128, 4096)
        raises(capi.LDB_ERR_INVALID, codes_of, gpu_ctx, t, ("strcode", foreign, "s"))
    # the dictionary that failed nothing still works
    assert decode(gpu_ctx, d, codes_of(gpu_ctx, t, ("strcode", d, "s"))) == vals
    for s_ in (small, arena, d, jt):
        gpu_ctx.L.ldb_gpu_state_destroy(s_)


def test_q16_sf1(gpu_ctx):
    """Q16: count(distinct ps_suppkey) per (p_brand, p_type, p_size) over parts that are not Brand#45, not MEDIUM POLISHED% and of
    eight sizes, without the suppliers with complaints (anti join) — string group keys through two dictionaries, count(distinct) as
    a group-by over the exported (brand, type, size, supplier) groups, ORDER BY count DESC, brand, type, size on the ranks."""
    GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "reference_kats.json")))["tpch_sf1"]["q16"]
    sf = dbgen.tpch(1.0, extended=True, attributes=True)
    pa, ps = gpu_ctx.table_from_host(sf["part"]), gpu_ctx.table_from_host(sf["partsupp"])
    bad = dbgen.complaint_suppliers(1.0)
    ct = runtime.Table(gpu_ctx, "complaints", [ColumnSpec("s_suppkey", "int32")])
    ct.append_host({"s_suppkey": bad}, len(bad))
    states = [runtime.join_table(gpu_ctx, 210_000), runtime.join_table(gpu_ctx, 1024), P.dict_state(gpu_ctx, 64, 1 << 12), P.dict_state(gpu_ctx, 256, 1 << 14)]
    part_rows, complaints, brands, types = states
    P.build_join(gpu_ctx, pa, part_rows, col("p_partkey"), payload=("rowid",))
    P.build_join(gpu_ctx, ct, complaints, col("s_suppkey"))
    prow = ("probe", part_rows, col("ps_partkey"))
    f = lambda c: ("fetch", pa, prow, c)
    size = f("p_size")
    sizes = ("cmp", "=", size, const(49))
    for s_ in (14, 23, 45, 19, 3, 36, 9):
        sizes = ("or", sizes, ("cmp", "=", size, const(s_)))
    where = ("and", ("and", ("strcmp", "!=", f("p_brand"), "Brand#45"), ("not", ("like", "prefix", f("p_type"), "MEDIUM POLISHED"))),
             ("and", sizes, ("isnull", ("probe", complaints, col("ps_suppkey")))))
    st1 = P.group_by(gpu_ctx, ps, [("strcode", brands, f("p_brand")), ("strcode", types, f("p_type")), size, col("ps_suppkey")], [("count_star", None)],
                     where=where, expected_groups=1 << 18)
    g1 = P.groups_table(gpu_ctx, st1)
    st2 = P.group_by(gpu_ctx, g1, [col("k0"), col("k1"), col("k2")], [("count_star", None)], expected_groups=1 << 15)  # count(distinct supplier)
    g2 = P.groups_table(gpu_ctx, st2)
    bt, tt = P.dict_table(gpu_ctx, brands), P.dict_table(gpu_ctx, types)
    mt = P.RawTable(gpu_ctx, P.materialize(gpu_ctx, g2, [col("a0"), ("fetch", bt, col("k0"), "rank"), ("fetch", tt, col("k1"), "rank"), col("k2"), col("k0"), col("k1")]))
    ids = mt.order_by_keys([("c0", True), ("c1", False), ("c2", False), ("c3", False)])
    counts, szs, bc, tc = (mt.gather(c, ids) for c in ("c0", "c3", "c4", "c5"))
    rows = [[b, t_, str(s_), str(n)] for b, t_, s_, n in zip(bt.gather_strings("str", bc), tt.gather_strings("str", tc), szs, counts)]
    assert len(rows) == GOLD["rows"] and rows[:3] == GOLD["first"] and rows[-3:] == GOLD["last"]
    assert hashlib.sha256("\n".join("\t".join(r) for r in rows).encode()).hexdigest() == GOLD["sha256"]
    for x in (mt, bt, tt, g2, g1):
        x.destroy()
    for s_ in states + [st1, st2]:
        gpu_ctx.L.ldb_gpu_state_destroy(s_)
