"""The repartition of table rows across ranks (ldb_gpu_table_exchange, parallel.Comm.table_exchange) against an exact model: every rank's
received table must be, cell for cell and validity for validity, the concatenation over source ranks (in rank order) of the rows it
owns, each source's rows in their source row order; with no keys, every source's rows on every rank.  The owner of a row is the rank
ldb_gpu_hashagg_exchange gives the group with the same key values; the numpy / Python keyTupleHash below restates it.  Also: capacity
(all ranks fail together and nothing is written), every documented error, back-to-back exchanges, and TPC-H Q12, Q4, Q3 and Q18 at SF1
with lineitem, orders and customer dealt to the ranks by batches, none replicated, against the reference's own answers.

Ranks are contexts of this process on device 0 wired by parallel.Comm.local_group.  The exchange waits for its peers on the host, so
each rank calls it from a thread of its own."""
import ctypes as C
import datetime
import os
import random
import re
import struct
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import _keyhash as K
import _progref as R
from _keyhash import mix64
from lingodb_b200 import capi, datagen

M64 = (1 << 64) - 1
# the nine fixed-width physical types, decimal128 at precision 38 and below 19, plus a utf8 column that is never shipped
COLUMNS = [("k", "int32", 0, 0), ("i8", "int8", 0, 0), ("i16", "int16", 0, 0), ("i32", "int32", 0, 0), ("i64", "int64", 0, 0),
           ("dw", "decimal128", 38, 2), ("dn", "decimal128", 18, 2), ("dt", "date32", 0, 0), ("fs", "fsb4", 0, 0),
           ("f4", "float32", 0, 0), ("f8", "float64", 0, 0), ("s", "utf8", 0, 0)]
PHYS = {n: p for n, p, _, _ in COLUMNS}
FIXED = [n for n, p, _, _ in COLUMNS if p != "utf8"]
WIDTH = {"int8": 1, "int16": 2, "int32": 4, "date32": 4, "fsb4": 4, "float32": 4, "int64": 8, "float64": 8, "decimal128": 16}
KEY_SETS = [[], ["i64"], ["dn", "dt"], ["i8", "fs", "dw"], ["k", "i16", "i32", "dn"]]
SUBSET = ["f8", "i8", "dw", "k"]


# ---------------------------------------------------------------------------------------------------- the model
def key_tuple_hash(keys: list) -> int:
    """keyTupleHash over key values (None = NULL: hashes as 0, sets bit k of the seed); a value is taken as int64 (its low 64 bits)"""
    return K.key_tuple_hash([0 if v is None else v for v in keys], sum(1 << k for k, v in enumerate(keys) if v is None))


def owner(keys: list, world: int) -> int:
    return ((key_tuple_hash(keys) >> 32) * world) >> 32


def test_model_hash_matches_known_values():
    """the restated hash is the splitmix-style fold of program.cu, pinned on values computed from its definition"""
    assert mix64(0) == 0
    h = key_tuple_hash([7])
    assert h == (mix64(0x9E3779B97F4A7C55 ^ 7) + 0x632BE59BD9B4E019) & M64
    assert key_tuple_hash([None]) == (mix64(0x9E3779B97F4A7C55 ^ 1) + 0x632BE59BD9B4E019) & M64
    assert key_tuple_hash([-1]) == key_tuple_hash([(1 << 64) - 1]) == key_tuple_hash([(5 << 64) - 1])  # only the low 64 bits count
    assert owner([], 5) == owner([], 5) and all(0 <= owner([i], 3) < 3 for i in range(100))
    shares = np.bincount([owner([i], 4) for i in range(20000)], minlength=4) / 20000
    assert (abs(shares - 0.25) < 0.02).all()


def raw_of(phys: str, v):
    """a cell as ldb_gpu_table_gather returns it: the signed little-endian integer of its bytes (floats by their bits)"""
    if v is None:
        return None
    if phys == "float32":
        return struct.unpack("<i", struct.pack("<f", v))[0]
    if phys == "float64":
        return struct.unpack("<q", struct.pack("<d", v))[0]
    return v


def expected(sources: list, keys: list, world: int) -> list:
    """sources[s] = rows (dicts column → raw cell / None) of rank s in row order; the rows every rank receives"""
    out = [[] for _ in range(world)]
    for rows in sources:
        for row in rows:
            if keys:
                out[owner([row[k] for k in keys], world)].append(row)
            else:
                for d in range(world):
                    out[d].append(row)
    return out


def read_table(t, columns: list, widths: dict) -> list:
    n = t.num_rows
    ids = list(range(n))
    cols = {c: t.gather(c, ids, cell_bytes=widths[c]) for c in columns}
    return [{c: cols[c][i] for c in columns} for i in range(n)]


def assert_received(got_tables: list, want: list, columns: list, widths: dict, what=""):
    for d, (t, rows) in enumerate(zip(got_tables, want)):
        assert t.num_rows == len(rows), (what, d, t.num_rows, len(rows))
        got = read_table(t, columns, widths)
        for i, (g, w) in enumerate(zip(got, rows)):
            assert g == {c: w[c] for c in columns}, (what, d, i, g, w)


# ---------------------------------------------------------------------------------------------------- ranks and staging
def ranks(world, user_bytes=16 << 20):
    from test_gpu_exchange import ranks as r
    return r(world, user_bytes=user_bytes)


def on_ranks(comms, fn):
    """fn(rank) on every rank, one thread each; returns (results, exceptions)"""
    def one(r):
        try:
            return fn(r), None
        except capi.LdbRuntimeError as e:
            return None, e
    with ThreadPoolExecutor(len(comms)) as ex:
        res = list(ex.map(one, range(len(comms))))
    return [a for a, _ in res], [b for _, b in res]


def all_ok(comms, fn):
    res, errs = on_ranks(comms, fn)
    assert errs == [None] * len(comms), [str(e) for e in errs]
    return res


def exchange(comms, tables, keys, columns=None, **kw):
    return all_ok(comms, lambda r: comms[r].table_exchange(tables[r], keys, columns=columns, **kw))


def stage(ctx, name: str, values: dict, how: str, seed: int):
    """values as a table of ctx, in ragged batches: "host" (HOST staging, whole-chunk bitmaps), "host_sliced" (HOST batches that are
    Arrow slices: bitmaps read from a bit offset), "device" (borrowed DEVICE batches, sliced bitmaps)"""
    import torch

    from lingodb_b200 import runtime
    n = len(values["k"])
    rng = random.Random(seed)
    cuts = sorted({rng.randrange(1, n) for _ in range(3)}) if n > 8 else []
    bounds = list(zip([0] + cuts, cuts + [n]))
    if how == "host":
        return ctx.table_from_host(R.to_table_data(name, values, COLUMNS, cuts))
    tab = runtime.Table(ctx, name, R.specs_of(COLUMNS))
    for lo, hi in bounds:
        off = rng.randrange(1, 12)
        ch = {}
        for cname, phys, _, _ in COLUMNS:
            buf, bm = R.column_buffers(phys, values[cname][lo:hi], offset=off)
            ch[cname] = buf
            if bm is not None:
                ch[cname + "$valid"] = bm
        if how == "host_sliced":
            tab.append_host(ch, hi - lo, offset=off)
        else:
            dev = {}
            for k, v in ch.items():
                if isinstance(v, tuple):
                    dev[k] = tuple(torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in v)
                else:
                    dev[k] = torch.from_numpy(np.ascontiguousarray(v)).cuda()
            tab.append_device(dev, hi - lo, offset=off)
    torch.cuda.synchronize()
    return tab


def shard_bounds(n: int, world: int, seed: int) -> list:
    """ragged row ranges [lo, hi) of `world` ranks; with more than one rank, one of them is empty"""
    rng = random.Random(seed)
    b = [0] + sorted(rng.randrange(n + 1) for _ in range(world - 1)) + [n]
    if world > 1:
        e = rng.randrange(world)
        if e + 1 < world:
            b[e + 1] = b[e]
        else:
            b[e] = n
    return list(zip(b, b[1:]))


def empty(ctx, name: str):
    """a table without batches"""
    from lingodb_b200 import runtime
    return runtime.Table(ctx, name, R.specs_of(COLUMNS))


def rows_of(values: dict, lo: int, hi: int) -> list:
    return [{c: raw_of(PHYS[c], values[c][i]) for c in FIXED} for i in range(lo, hi)]


# ---------------------------------------------------------------------------------------------------- 1. exact against the model
@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_exchange_matches_the_model(world):
    from lingodb_b200 import program as P
    n = 1600 if world < 8 else 2400
    v = R.gen_values(900 + world, n, COLUMNS, null_rate=0.12, key_domain=1 << 30)
    bounds = shard_bounds(n, world, 17 * world)
    assert world == 1 or any(hi == lo for lo, hi in bounds)
    widths = {c: WIDTH[PHYS[c]] for c in FIXED}
    with ranks(world) as (ctxs, comms):
        hows = ["host", "host_sliced", "device"]
        tabs = [stage(c, f"s{r}", {k: x[lo:hi] for k, x in v.items()}, hows[r % 3], 31 * world + r) if hi > lo else empty(c, f"s{r}")
                for r, (c, (lo, hi)) in enumerate(zip(ctxs, bounds))]
        sources = [rows_of(v, lo, hi) for lo, hi in bounds]
        for keys in KEY_SETS:
            for columns in (FIXED, SUBSET):
                got = exchange(comms, tabs, keys, columns=columns)
                assert_received(got, expected(sources, keys, world), columns, widths, (world, keys, len(columns)))
                if keys and world > 1:
                    assert sum(1 for t in got if t.num_rows) > 1, keys  # the rows really spread over the ranks
                if not keys:
                    assert all(t.num_rows == n for t in got)
                for t in got:
                    t.destroy()
        # library-made sources: materialized rows (16-byte cells, validity bytes) and exported groups (int64 keys)
        col, const = (lambda x: ("col", x)), (lambda x: ("const", x))
        mats = [P.RawTable(c, P.materialize(c, t, [col("i64"), col("dn"), ("add", col("i16"), const(1)), col("dt")],
                                            where=("not", ("isnull", col("i8"))))) for c, t in zip(ctxs, tabs)]
        groups = [P.groups_table(c, P.group_by(c, t, [col("i16"), col("dt")], [("count_star", None), ("sum", col("i64"))], expected_groups=4096))
                  for c, t in zip(ctxs, tabs)]
        for srcs, cols_, keysets in ((mats, ["c0", "c1", "c2", "c3"], [["c0"], ["c1", "c3"], []]), (groups, ["k0", "k1", "a0", "a1"], [["k0"], ["k1", "k0"]])):
            w = {c: 16 if c[0] in "ca" else 8 for c in cols_}
            src_rows = [read_table(t, cols_, w) for t in srcs]
            assert any(r[cols_[0]] is None for rows in src_rows for r in rows) or srcs is mats
            for keys in keysets:
                got = exchange(comms, srcs, keys)
                assert_received(got, expected(src_rows, keys, world), cols_, w, (world, "derived", keys))
                for t in got:
                    t.destroy()
        for t in mats + groups:
            t.destroy()


# ---------------------------------------------------------------------------------------------------- 2. owner agreement
@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_owner_depends_on_values_and_agrees_with_the_hash_aggregation_exchange(world):
    from lingodb_b200 import program as P
    col = lambda x: ("col", x)
    n = 3000
    keys = list(range(-200, n - 200))
    with ranks(world) as (ctxs, comms):
        cols = [datagen.ColumnSpec("okey", "int32", 0, 0), datagen.ColumnSpec("wide", "int64", 0, 0)]
        a, b = [], []
        for r, c in enumerate(ctxs):
            part = keys[r::world]
            td = datagen.TableData(f"a{r}", cols, [{"okey": np.array(part, np.int32), "wide": np.array(part, np.int64) * 3}], [len(part)])
            a.append(c.table_from_host(td))
            other = keys[(r + 1) % world::world]  # a different split of the same keys
            td = datagen.TableData(f"b{r}", cols, [{"okey": np.zeros(len(other), np.int32), "wide": np.array(other, np.int64)}], [len(other)])
            b.append(P.RawTable(c, P.materialize(c, c.table_from_host(td), [col("wide")])))  # the key as a decimal128 cell
        got_a = exchange(comms, a, ["okey"], columns=["okey"])
        got_b = exchange(comms, b, ["c0"])
        at_a = {k: d for d, t in enumerate(got_a) for k in t.gather("okey", list(range(t.num_rows)), cell_bytes=4)}
        at_b = {k: d for d, t in enumerate(got_b) for k in t.gather("c0", list(range(t.num_rows)))}
        assert set(at_a) == set(at_b) == set(keys)
        assert at_a == at_b
        assert at_a == {k: owner([k], world) for k in keys}
        locals_ = [P.group_by(c, t, [col("okey")], [("count_star", None)], expected_groups=4096) for c, t in zip(ctxs, a)]
        owneds = [P.hashagg_state(c, 1, ["count_star"], 4096) for c in ctxs]
        all_ok(comms, lambda r: comms[r].hashagg_exchange(locals_[r], owneds[r]))
        for d, (c, o) in enumerate(zip(ctxs, owneds)):
            held = P.decode_groups(P.read_groups(c, o, 4096), 1, 1)
            assert {k for (k,) in held} == {k for k, r in at_a.items() if r == d}
        for c, s1, s2 in zip(ctxs, locals_, owneds):
            c.L.ldb_gpu_state_destroy(s1)
            c.L.ldb_gpu_state_destroy(s2)
        for t in got_a + got_b + b:
            t.destroy()


# ---------------------------------------------------------------------------------------------------- 3. broadcast
@pytest.mark.gpu
def test_broadcast_gives_every_rank_the_same_concatenation():
    world = 4
    widths = {c: WIDTH[PHYS[c]] for c in FIXED}
    # one-tile shards; then shards of several 4 096-row tiles in ragged batches (staged with seeds 0..3) that end in partial tiles, a
    # middle batch's included, so most tiles start at a source row that is not a multiple of the tile
    for n, bounds in ((900, [(0, 100), (100, 100), (100, 650), (650, 900)]), (40000, [(0, 13000), (13000, 13000), (13000, 30000), (30000, 40000)])):
        v = R.gen_values(77, n, COLUMNS, null_rate=0.2, key_domain=1000)
        with ranks(world) as (ctxs, comms):
            tabs = [stage(c, f"s{r}", {k: x[lo:hi] for k, x in v.items()}, "host_sliced", r) if hi > lo else empty(c, f"s{r}") for r, (c, (lo, hi)) in enumerate(zip(ctxs, bounds))]
            got = exchange(comms, tabs, [], columns=FIXED, name=None)
            whole = rows_of(v, 0, n)
            assert_received(got, [whole] * world, FIXED, widths, f"broadcast of {n} rows")
            for t in got:
                t.destroy()


# ---------------------------------------------------------------------------------------------------- 4. capacity
SENTINEL = 0x5A5A5A5A


def region_bytes(n: int, widths: list) -> int:
    a16 = lambda x: (x + 15) // 16 * 16
    return sum(a16(n * w) for w in widths) + len(widths) * a16(n)


@pytest.mark.gpu
def test_capacity_fails_on_every_rank_writes_nothing_and_the_named_size_succeeds():
    from test_gpu_exchange import heap_fill, heap_read
    world, n, off = 3, 3000, 4096
    v = R.gen_values(55, n, COLUMNS, null_rate=0.1, key_domain=1 << 30)
    bounds = [(0, 1000), (1000, 1900), (1900, 3000)]
    widths = {c: WIDTH[PHYS[c]] for c in FIXED}
    with ranks(world) as (ctxs, comms):
        tabs = [stage(c, f"s{r}", {k: x[lo:hi] for k, x in v.items()}, "host", r) for r, (c, (lo, hi)) in enumerate(zip(ctxs, bounds))]
        want = expected([rows_of(v, lo, hi) for lo, hi in bounds], ["i64", "dt"], world)
        need = max(region_bytes(len(rows), [widths[c] for c in FIXED]) for rows in want)
        assert len({len(rows) for rows in want}) > 1  # one rank needs more than the others
        span = need + 8192
        for cm in comms:
            heap_fill(cm, off - 1024, span)
        _, errs = on_ranks(comms, lambda r: comms[r].table_exchange(tabs[r], ["i64", "dt"], columns=FIXED, recv_offset=off, recv_bytes=need - 16))
        assert all(e is not None and e.code == capi.LDB_ERR_CAPACITY for e in errs), errs
        named = {int(re.search(r"retry with recv_bytes (\d+)", str(e)).group(1)) for e in errs}
        assert named == {need}
        for cm in comms:  # nothing was written into any receive region
            raw = np.frombuffer(heap_read(cm, off - 1024, span), dtype=np.uint32)
            assert (raw == SENTINEL).all()
        got = all_ok(comms, lambda r: comms[r].table_exchange(tabs[r], ["i64", "dt"], columns=FIXED, recv_offset=off, recv_bytes=need))
        assert_received(got, want, FIXED, widths, "retry")
        for t in got:
            t.destroy()


# ---------------------------------------------------------------------------------------------------- 5. errors
@pytest.mark.gpu
def test_documented_errors():
    with ranks(2, user_bytes=1 << 20) as (ctxs, comms):
        c, cm = ctxs[0], comms[0]
        v = R.gen_values(3, 40, COLUMNS)
        t = c.table_from_host(R.to_table_data("t", v, COLUMNS))
        other = ctxs[1].table_from_host(R.to_table_data("o", v, COLUMNS))
        L, user = c.L, cm.heap()[1]

        def call(table=t, keys=("i64",), columns=("i32",), comm=cm, off=0, nbytes=4096, out=True, n_keys=None, n_columns=None):
            kn = [k.encode() if k is not None else None for k in keys]
            karr = (C.c_char_p * max(1, len(kn)))(*kn)
            carr = None
            if columns is not None:
                cn = [x.encode() if x is not None else None for x in columns]
                carr = (C.c_char_p * max(1, len(cn)))(*cn)
            res, e = C.c_void_p(), capi.Error()
            rc = L.ldb_gpu_table_exchange(table.h if table is not None else None, len(kn) if n_keys is None else n_keys, karr if keys is not None else None,
                                          (len(columns) if columns is not None else 0) if n_columns is None else n_columns, carr,
                                          comm.h if comm is not None else None, off, nbytes, b"x", C.byref(res) if out else None, C.byref(e))
            return rc, e.message.decode()
        INVALID, UNSUP = capi.LDB_ERR_INVALID, capi.LDB_ERR_UNSUPPORTED
        cases = [
            (dict(table=None), INVALID, "null argument"),
            (dict(comm=None), INVALID, "null argument"),
            (dict(out=False), INVALID, "null argument"),
            (dict(n_keys=5, keys=("i64",) * 5), INVALID, "0..4 key columns"),
            (dict(n_keys=-1), INVALID, "0..4 key columns"),
            (dict(keys=("nope",)), INVALID, "unknown key column"),
            (dict(columns=("i32", "nope")), INVALID, "unknown column"),
            (dict(columns=("i32",) * 17), INVALID, "up to 16 columns"),
            (dict(columns=("i32",), n_columns=0), INVALID, "1..16 columns"),
            (dict(table=other), INVALID, "different contexts"),
            (dict(off=8), INVALID, "16-byte aligned"),
            (dict(off=-16), INVALID, "outside"),
            (dict(off=user - 64, nbytes=128), INVALID, "outside"),
            (dict(nbytes=user + 16), INVALID, "outside"),
            (dict(columns=("i32", "s")), UNSUP, "fixed-width"),
            (dict(columns=None), UNSUP, "fixed-width"),  # all columns: the utf8 one among them
            (dict(keys=("s",)), UNSUP, "exchange keys"),
            (dict(keys=("f8",)), UNSUP, "exchange keys"),
            (dict(keys=("i64", "f4")), UNSUP, "exchange keys"),
        ]
        for kw, code, msg in cases:
            rc, m = call(**kw)
            assert rc == code and msg in m, (kw, rc, m)
        c.graph_begin()
        rc, m = call()
        c.graph_end().destroy()
        assert rc == UNSUP and "captured" in m, m
        # none of the refused calls started a collective: both ranks still exchange in step
        tabs = [t, ctxs[1].table_from_host(R.to_table_data("u", v, COLUMNS))]
        got = exchange(comms, tabs, ["i64"], columns=["i32"])
        assert sum(x.num_rows for x in got) == 80
        for x in got:
            x.destroy()


# ---------------------------------------------------------------------------------------------------- 6. back to back
@pytest.mark.gpu
def test_back_to_back_exchanges_over_the_same_region():
    world, n = 3, 2500
    v = R.gen_values(404, n, COLUMNS, null_rate=0.1, key_domain=1 << 30)
    bounds = [(0, 700), (700, 1500), (1500, 2500)]
    widths = {c: WIDTH[PHYS[c]] for c in FIXED}
    with ranks(world) as (ctxs, comms):
        tabs = [stage(c, f"s{r}", {k: x[lo:hi] for k, x in v.items()}, ["host", "device", "host_sliced"][r], r) for r, (c, (lo, hi)) in enumerate(zip(ctxs, bounds))]
        sources = [rows_of(v, lo, hi) for lo, hi in bounds]
        first = exchange(comms, tabs, ["k"], columns=FIXED)
        second = exchange(comms, tabs, ["dw", "i8"], columns=SUBSET)
        third = exchange(comms, second, ["k"], columns=SUBSET)  # an exchange of received tables
        assert_received(first, expected(sources, ["k"], world), FIXED, widths, "first")
        want2 = expected(sources, ["dw", "i8"], world)
        assert_received(second, want2, SUBSET, widths, "second")
        assert_received(third, expected(want2, ["k"], world), SUBSET, widths, "third")
        for cm in comms:
            cm.check()  # no peer timed out
        for t in first + second + third:
            t.destroy()


# ---------------------------------------------------------------------------------------------------- 6b. shards of many tiles
TILE_ROWS = 4096  # rows per CTA of the count and send kernels (kShipTile)


def owners_np(keys: list, world: int) -> np.ndarray:
    """the owner of every row: keys = [(int64 values, valid mask)] per key column, the same fold as key_tuple_hash, in numpy"""
    seed = np.zeros(len(keys[0][0]), np.uint64)
    for k, (_, valid) in enumerate(keys):
        seed |= (~valid).astype(np.uint64) << np.uint64(k)
    h = K.key_tuple_hash_np([np.where(valid, vals.astype(np.int64), 0) for vals, valid in keys], seed)
    return (((h >> np.uint64(32)) * np.uint64(world)) >> np.uint64(32)).astype(np.int64)


def test_numpy_owner_agrees_with_the_model():
    rng = np.random.default_rng(5)
    a, b = rng.integers(-2**63, 2**63 - 1, 3000, dtype=np.int64), rng.integers(-50, 50, 3000, dtype=np.int64)
    va, vb = rng.random(3000) > 0.2, rng.random(3000) > 0.1
    for world in (2, 3, 8):
        got = owners_np([(a, va), (b, vb)], world)
        want = [owner([int(x) if p else None, int(y) if q else None], world) for x, y, p, q in zip(a, b, va, vb)]
        assert got.tolist() == want


def gather_np(t, column: str, width: int):
    """a received column as (cells (n, width) uint8, validity bytes) in one gather"""
    n = t.num_rows
    ids = np.arange(n, dtype=np.int64)
    cells = np.zeros((max(n, 1), width), np.uint8)
    valid = np.zeros(max(n, 1), np.uint8)
    e = capi.Error()
    capi.check(t.ctx.L.ldb_gpu_table_gather(t.h, column.encode(), ids.ctypes.data_as(C.POINTER(C.c_int64)), n, cells.ctypes.data_as(C.c_void_p),
                                            valid.ctypes.data_as(C.POINTER(C.c_uint8)), C.byref(e)), e)
    return cells[:n], valid[:n].astype(bool)


WIDE_COLUMNS = [("i64", "int64", 0, 0), ("dn", "decimal128", 18, 2), ("dw", "decimal128", 38, 2), ("i8", "int8", 0, 0), ("dt", "date32", 0, 0),
                ("f4", "float32", 0, 0)]


def wide_values(rng, n: int) -> dict:
    """column → (cells (n, width) uint8 as the staged table holds them, valid mask); NULL cells hold 0"""
    lo = rng.integers(-2**63, 2**63 - 1, n, dtype=np.int64)
    vals = {"i64": rng.integers(-2**40, 2**40, n, dtype=np.int64), "dn": rng.integers(-10**17, 10**17, n, dtype=np.int64),
            "i8": rng.integers(-128, 128, n, dtype=np.int8), "dt": rng.integers(-10**6, 10**6, n, dtype=np.int32),
            "f4": rng.standard_normal(n).astype(np.float32)}
    out = {}
    for name, phys, _, _ in WIDE_COLUMNS:
        valid = rng.random(n) > 0.1
        if name == "dw":
            hi = rng.integers(-2**62, 2**62, n, dtype=np.int64)
            cells = np.stack([lo, hi], 1)
        elif phys == "decimal128":
            cells = np.stack([vals[name], vals[name] >> 63], 1)
        else:
            cells = vals[name]
        cells = np.where(valid.reshape((-1,) + (1,) * (cells.ndim - 1)), cells, 0)
        out[name] = (np.ascontiguousarray(cells).view(np.uint8).reshape(n, WIDTH[phys]), valid)
    return out


def stage_wide(ctx, name: str, parts: list, how: str):
    """batches of (cells, valid) columns: "host" (HOST staging; a batch of >= 65 536 rows is staged compressed), "sliced" (HOST
    batches that are Arrow slices at bit offset 5), "device" (borrowed DEVICE batches)"""
    import torch

    from lingodb_b200 import runtime
    tab = runtime.Table(ctx, name, R.specs_of(WIDE_COLUMNS))
    for part in parts:
        n = len(part["i64"][1])
        off = 5 if how == "sliced" else 0
        ch = {}
        for cname, phys, _, _ in WIDE_COLUMNS:
            cells, valid = part[cname]
            if off:
                cells = np.concatenate([np.zeros((off, cells.shape[1]), np.uint8), cells])
                valid = np.concatenate([np.zeros(off, bool), valid])
            ch[cname] = cells if phys == "decimal128" else np.ascontiguousarray(cells).view(R._NP[phys]).reshape(-1)
            ch[cname + "$valid"] = np.concatenate([np.packbits(valid, bitorder="little"), np.zeros(1, np.uint8)])
        if how == "device":
            tab.append_device({k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in ch.items()}, n)
        else:
            tab.append_host(ch, n, offset=off)
    torch.cuda.synchronize()
    return tab


@pytest.mark.gpu
def test_shards_of_many_tiles_and_a_compressed_batch_match_the_model():
    """several 4 096-row tiles per batch (the scanned per-CTA offsets), a HOST batch of 70 000 rows (compressed staging), sliced and
    DEVICE batches: every received cell and validity byte against the model"""
    world = 3
    rng = np.random.default_rng(11)
    layout = [("host", [70_000, 9_001]), ("device", [20_000, 13_333]), ("sliced", [30_017])]
    assert 70_000 >= 65_536 and all(sum(s) > 2 * TILE_ROWS for _, s in layout)
    names = [c for c, *_ in WIDE_COLUMNS]
    widths = {c: WIDTH[p] for c, p, _, _ in WIDE_COLUMNS}
    with ranks(world, user_bytes=64 << 20) as (ctxs, comms):
        tabs, sources = [], []
        for r, (how, sizes) in enumerate(layout):
            parts = [wide_values(rng, m) for m in sizes]
            tabs.append(stage_wide(ctxs[r], f"w{r}", parts, how))
            sources.append({c: (np.concatenate([p[c][0] for p in parts]), np.concatenate([p[c][1] for p in parts])) for c in names})
        for keys in (["i64", "dn"], ["dt"], []):
            got = exchange(comms, tabs, keys)
            for d, t in enumerate(got):
                picks = []
                for src in sources:
                    n = len(src["i64"][1])
                    if keys:
                        ks = [(src[k][0][:, :8].copy().view(np.int64).reshape(-1) if widths[k] >= 8 else src[k][0].view(np.int32).reshape(-1), src[k][1]) for k in keys]
                        picks.append((src, owners_np(ks, world) == d))
                    else:
                        picks.append((src, np.ones(n, bool)))
                want_n = sum(int(m.sum()) for _, m in picks)
                assert t.num_rows == want_n, (keys, d)
                for c in names:
                    cells, valid = gather_np(t, c, widths[c])
                    want_cells = np.concatenate([src[c][0][m] for src, m in picks])
                    want_valid = np.concatenate([src[c][1][m] for src, m in picks])
                    assert (valid == want_valid).all(), (keys, d, c)
                    assert (cells[valid] == want_cells[want_valid]).all(), (keys, d, c)
                t.destroy()


@pytest.mark.gpu
def test_more_than_1024_tiles_keep_source_order():
    """5 M rows on one rank: the per-destination scan runs over 1 221 CTA counts, past its 1 024-entry chunks"""
    import torch

    from lingodb_b200 import runtime
    world, sizes = 2, [5_000_000, 300_000]
    assert sizes[0] > 1024 * TILE_ROWS
    with ranks(world, user_bytes=128 << 20) as (ctxs, comms):
        tabs, vals = [], []
        for r, (c, n) in enumerate(zip(ctxs, sizes)):
            v = np.arange(n, dtype=np.int64) * 7919 + r * (1 << 40)
            t = runtime.Table(c, f"v{r}", [datagen.ColumnSpec("v", "int64", 0, 0)])
            t.append_device({"v": torch.from_numpy(v).cuda()}, n)
            tabs.append(t)
            vals.append(v)
        torch.cuda.synchronize()
        got = exchange(comms, tabs, ["v"])
        for d, t in enumerate(got):
            want = np.concatenate([v[owners_np([(v, np.ones(len(v), bool))], world) == d] for v in vals])
            cells, valid = gather_np(t, "v", 8)
            assert valid.all() and (cells.view(np.int64).reshape(-1) == want).all(), d
            t.destroy()


# ---------------------------------------------------------------------------------------------------- 7. distributed TPC-H at SF1
@pytest.fixture(scope="module")
def sf1():
    from lingodb_b200 import dbgen
    return dbgen.tpch(1.0, extended=True)


def _deal(td, world: int, rank: int, shift: int):
    """the batches i of td with (i + shift) % world == rank"""
    out = datagen.TableData(f"{td.name}{rank}", td.columns)
    for i in range(len(td.chunks)):
        if (i + shift) % world == rank:
            out.chunks.append(td.chunks[i])
            out.chunk_rows.append(td.chunk_rows[i])
    return out


def _union_groups(ctxs, states, n_keys, n_aggs):
    from lingodb_b200 import program as P
    out = {}
    for c, s in zip(ctxs, states):
        for k, a in P.decode_groups(P.read_groups(c, s, 1 << 12), n_keys, n_aggs).items():
            assert k not in out
            out[k] = a
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_distributed_tpch_q12_q4_q3_q18_reproduce_the_reference(sf1, world):
    from lingodb_b200 import dbgen, program as P, runtime
    from test_reference_answers_sf1 import GOLD, day, dec
    col, const = (lambda x: ("col", x)), (lambda x: ("const", x))
    d = lambda s: (datetime.date.fromisoformat(s) - datetime.date(1970, 1, 1)).days
    li_b, od_b = sf1["lineitem"], sf1["orders"]
    # the dealt batches do not line up by order key: an order's lines and the order itself sit on different ranks
    with ranks(world, user_bytes=512 << 20) as (ctxs, comms):
        lis = [c.table_from_host(_deal(li_b, world, r, 0)) for r, c in enumerate(ctxs)]
        ods = [c.table_from_host(_deal(od_b, world, r, 1)) for r, c in enumerate(ctxs)]
        cus = [c.table_from_host(_deal(sf1["customer"], world, r, 2)) for r, c in enumerate(ctxs)]
        assert sum(t.num_rows for t in lis) == li_b.num_rows and sum(t.num_rows for t in ods) == od_b.num_rows
        mat = lambda r, t, outs, where=None: P.RawTable(ctxs[r], P.materialize(ctxs[r], t, outs, where=where))
        drop = lambda ts: [t.destroy() for t in ts]
        # ---- Q12: lineitem(shipmode IN, dates) ⋈ orders on orderkey, high / low priority line counts per ship mode
        mode = ("case", ("strcmp", "=", "l_shipmode", "MAIL"), const(0), const(1))
        lwhere = ("and", ("and", ("or", ("strcmp", "=", "l_shipmode", "MAIL"), ("strcmp", "=", "l_shipmode", "SHIP")),
                          ("and", ("cmp", "<", col("l_commitdate"), col("l_receiptdate")), ("cmp", "<", col("l_shipdate"), col("l_commitdate")))),
                  ("and", ("cmp", ">=", col("l_receiptdate"), const(d("1994-01-01"))), ("cmp", "<", col("l_receiptdate"), const(d("1995-01-01")))))
        high = ("or", ("strcmp", "=", "o_orderpriority", "1-URGENT"), ("strcmp", "=", "o_orderpriority", "2-HIGH"))
        lm = [mat(r, lis[r], [col("l_orderkey"), mode], lwhere) for r in range(world)]
        om = [mat(r, ods[r], [col("o_orderkey"), ("case", high, const(1), const(0))]) for r in range(world)]
        lx, ox = exchange(comms, lm, ["c0"]), exchange(comms, om, ["c0"])
        locals_, owneds = [], []
        for r, c in enumerate(ctxs):
            j = runtime.join_table(c, 1_000_000, unique=True)
            P.build_join(c, ox[r], j, col("c0"), payload=col("c1"))
            pr = ("probe", j, col("c0"))
            aggs = [("sum", ("case", ("cmp", "=", pr, const(1)), const(1), const(0))), ("sum", ("case", ("cmp", "=", pr, const(0)), const(1), const(0)))]
            locals_.append(P.group_by(c, lx[r], [col("c1")], aggs, where=("not", ("isnull", pr)), expected_groups=16))
            owneds.append(P.hashagg_state(c, 1, ["sum", "sum"], 16))
            c.L.ldb_gpu_state_destroy(j)
        all_ok(comms, lambda r: comms[r].hashagg_exchange(locals_[r], owneds[r]))
        got = _union_groups(ctxs, owneds, 1, 2)
        assert [[m, str(got[(i,)][0]), str(got[(i,)][1])] for i, m in enumerate(("MAIL", "SHIP"))] == GOLD["q12_rows"]
        drop(lm + om + lx + ox)
        for c, a, b in zip(ctxs, locals_, owneds):
            c.L.ldb_gpu_state_destroy(a)
            c.L.ldb_gpu_state_destroy(b)
        # ---- Q4: orders(date range) with EXISTS lineitem(l_commitdate < l_receiptdate), order count per priority
        prio = ("case", ("strcmp", "=", "o_orderpriority", dbgen.ORDER_PRIORITIES[0]), const(0),
                ("case", ("strcmp", "=", "o_orderpriority", dbgen.ORDER_PRIORITIES[1]), const(1),
                 ("case", ("strcmp", "=", "o_orderpriority", dbgen.ORDER_PRIORITIES[2]), const(2),
                  ("case", ("strcmp", "=", "o_orderpriority", dbgen.ORDER_PRIORITIES[3]), const(3), const(4)))))
        owhere = ("and", ("cmp", ">=", col("o_orderdate"), const(d("1993-07-01"))), ("cmp", "<", col("o_orderdate"), const(d("1993-10-01"))))
        lm = [mat(r, lis[r], [col("l_orderkey")], ("cmp", "<", col("l_commitdate"), col("l_receiptdate"))) for r in range(world)]
        om = [mat(r, ods[r], [col("o_orderkey"), prio], owhere) for r in range(world)]
        lx, ox = exchange(comms, lm, ["c0"]), exchange(comms, om, ["c0"])
        locals_, owneds = [], []
        for r, c in enumerate(ctxs):
            late = runtime.join_table(c, 1_600_000, unique=True)
            P.build_join(c, lx[r], late, col("c0"))
            locals_.append(P.group_by(c, ox[r], [col("c1")], [("count_star", None)], where=("exists", late, col("c0"), None), expected_groups=16))
            owneds.append(P.hashagg_state(c, 1, ["count_star"], 16))
            c.L.ldb_gpu_state_destroy(late)
        all_ok(comms, lambda r: comms[r].hashagg_exchange(locals_[r], owneds[r]))
        got = _union_groups(ctxs, owneds, 1, 1)
        assert [[p, str(got[(i,)][0])] for i, p in enumerate(dbgen.ORDER_PRIORITIES)] == GOLD["q4_rows"]
        drop(lm + om + lx + ox)
        for c, a, b in zip(ctxs, locals_, owneds):
            c.L.ldb_gpu_state_destroy(a)
            c.L.ldb_gpu_state_destroy(b)
        # ---- Q3: BUILDING customers broadcast, orders probed locally and exchanged with lineitem on orderkey, local join + group-by,
        # top 10 over the ranks on the host
        cut = d("1995-03-15")
        cm_ = [mat(r, cus[r], [col("c_custkey")], ("strcmp", "=", "c_mktsegment", "BUILDING")) for r in range(world)]
        cx = exchange(comms, cm_, [])
        assert len({t.num_rows for t in cx}) == 1
        om, lm = [], []
        for r, c in enumerate(ctxs):
            cj = runtime.join_table(c, 400_000, unique=True)
            P.build_join(c, cx[r], cj, col("c0"))
            pc = ("probe", cj, col("o_custkey"))
            # payload: o_orderdate * 16 + o_shippriority (the priority is 0 in TPC-H data; 16 leaves room for it)
            om.append(mat(r, ods[r], [col("o_orderkey"), ("add", ("mul", col("o_orderdate"), const(16)), col("o_shippriority"))],
                          ("and", ("cmp", "<", col("o_orderdate"), const(cut)), ("not", ("isnull", pc)))))
            lm.append(mat(r, lis[r], [col("l_orderkey"), ("mul", col("l_extendedprice"), ("sub", const(100), col("l_discount")))],
                          ("cmp", ">", col("l_shipdate"), const(cut))))
            c.L.ldb_gpu_state_destroy(cj)
        ox, lx = exchange(comms, om, ["c0"]), exchange(comms, lm, ["c0"])
        rows = []
        for r, c in enumerate(ctxs):
            oj = runtime.join_table(c, 1_000_000, unique=True)
            P.build_join(c, ox[r], oj, col("c0"), payload=col("c1"))
            po = ("probe", oj, col("c0"))
            st = P.group_by(c, lx[r], [col("c0"), po], [("sum", col("c1"))], where=("not", ("isnull", po)), expected_groups=200_000)
            g = P.groups_table(c, st)
            ids = g.order_by("a0", descending=True, limit=64)
            rows += list(zip(g.gather("k0", ids, cell_bytes=8), g.gather("k1", ids, cell_bytes=8), g.gather("a0", ids)))
            g.destroy()
            c.L.ldb_gpu_state_destroy(st)
            c.L.ldb_gpu_state_destroy(oj)
        rows.sort(key=lambda x: (-x[2], x[1] // 16))
        assert [[str(k), dec(rev, 4), day(p // 16), str(p % 16)] for k, p, rev in rows[:10]] == GOLD["q3_rows"]
        drop(cm_ + cx + om + lm + ox + lx)
        # ---- Q18: lineitem sums per order merged on their owner ranks, then SHARDED orders exchanged on o_orderkey and semi-joined
        # against the owned groups: correct only if the exchange's owner is the hash aggregation exchange's
        locals_ = [P.group_by(c, t, [col("l_orderkey")], [("sum", col("l_quantity"))], expected_groups=1_600_000) for c, t in zip(ctxs, lis)]
        owneds = [P.hashagg_state(c, 1, ["sum"], 1_600_000) for c in ctxs]
        all_ok(comms, lambda r: comms[r].hashagg_exchange(locals_[r], owneds[r]))
        ox = exchange(comms, ods, ["o_orderkey"], columns=["o_custkey", "o_orderkey", "o_orderdate", "o_totalprice"])
        assert sum(t.num_rows for t in ox) == od_b.num_rows
        rows = []
        for r, c in enumerate(ctxs):
            groups = P.groups_table(c, owneds[r])
            big = runtime.join_table(c, 4096, unique=True)
            P.build_join(c, groups, big, col("k0"), payload=col("a0"), where=("cmp", ">", col("a0"), const(30000)))
            pb = ("probe", big, col("o_orderkey"))
            mt = mat(r, ox[r], [col("o_custkey"), col("o_orderkey"), col("o_orderdate"), col("o_totalprice"), pb], ("not", ("isnull", pb)))
            ids = mt.order_by("c3", descending=True)
            rows += list(zip(*[mt.gather(f"c{i}", ids) for i in range(5)]))
            mt.destroy()
            groups.destroy()
            c.L.ldb_gpu_state_destroy(big)
        rows.sort(key=lambda x: (-x[3], x[2]))
        got18 = [["Customer#%09d" % x[0], str(x[0]), str(x[1]), day(x[2]), dec(x[3], 2), dec(x[4], 2)] for x in rows[:100]]
        assert got18 == GOLD["q18_rows"]
        drop(ox)
        for c, a, b in zip(ctxs, locals_, owneds):
            c.L.ldb_gpu_state_destroy(a)
            c.L.ldb_gpu_state_destroy(b)


# ---------------------------------------------------------------------------------------------------- cross-process (two or more GPUs)
def _worker(rank: int, world: int, rendezvous: str):
    """one rank of test_across_processes_when_there_are_two_gpus: its shard → exchange → its received rows as JSON"""
    import json
    import sys
    import time

    from lingodb_b200 import parallel, runtime

    def swap(handle: bytes):
        with open(os.path.join(rendezvous, f"h{rank}.tmp"), "wb") as f:
            f.write(handle)
        os.replace(os.path.join(rendezvous, f"h{rank}.tmp"), os.path.join(rendezvous, f"h{rank}"))
        paths = [os.path.join(rendezvous, f"h{r}") for r in range(world)]
        deadline = time.monotonic() + 120
        while not all(os.path.exists(x) for x in paths):
            if time.monotonic() > deadline:  # a peer never started: give up rather than hold this GPU
                sys.exit(f"rank {rank}: the peers' handles did not arrive within 120 s")
            time.sleep(0.05)
        return [open(x, "rb").read() for x in paths]
    ctx = runtime.Context(rank)
    comm = parallel.Comm(ctx, rank, world, user_bytes=16 << 20, exchange=swap)
    v = R.gen_values(1234, 3000, COLUMNS, null_rate=0.1, key_domain=1 << 30)
    lo, hi = 3000 * rank // world, 3000 * (rank + 1) // world
    tab = stage(ctx, "s", {k: x[lo:hi] for k, x in v.items()}, "host", rank)
    widths = {c: WIDTH[PHYS[c]] for c in FIXED}
    res = {}
    for keys in (["i64", "dt"], []):
        t = comm.table_exchange(tab, keys, columns=FIXED)
        res[",".join(keys)] = read_table(t, FIXED, widths)
        t.destroy()
    comm.check()
    with open(os.path.join(rendezvous, f"out{rank}.json"), "w") as f:
        json.dump(res, f)
    comm.close()
    ctx.close()


@pytest.mark.gpu
def test_across_processes_when_there_are_two_gpus(tmp_path):
    import json
    import subprocess
    import sys

    import torch
    world = torch.cuda.device_count()
    if world < 2:
        pytest.skip("one GPU: the cross-process exchange needs two")
    world = min(world, 8)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([root] + [x for x in os.environ.get("PYTHONPATH", "").split(os.pathsep) if x]))
    procs = []
    try:
        for r in range(world):
            procs.append(subprocess.Popen([sys.executable, os.path.abspath(__file__), str(r), str(world), str(tmp_path)], env=env))
        codes = [p.wait(timeout=600) for p in procs]
    finally:  # no rank outlives the test, whatever ended it
        for p in procs:
            if p.poll() is None:
                p.kill()
            p.wait()
    assert codes == [0] * world
    v = R.gen_values(1234, 3000, COLUMNS, null_rate=0.1, key_domain=1 << 30)
    sources = [rows_of(v, 3000 * r // world, 3000 * (r + 1) // world) for r in range(world)]
    for keys in (["i64", "dt"], []):
        want = expected(sources, keys, world)
        for r in range(world):
            got = json.load(open(tmp_path / f"out{r}.json"))[",".join(keys)]
            assert got == [{c: w[c] for c in FIXED} for w in want[r]], (keys, r)


# ---------------------------------------------------------------------------------------------------- 8. host only
def test_entry_point_rejects_null_arguments_without_a_device():
    """Without a device no context, and so no table and no comm, can exist (ldb_gpu_context_create returns LDB_ERR_NO_DEVICE,
    test_cabi_symbols.py): what reaches the entry point on such a machine is null handles, refused before any CUDA call."""
    L = capi.lib()
    assert capi.SIGNATURES["ldb_gpu_table_exchange"][0] is C.c_int
    out, e = C.c_void_p(), capi.Error()
    for args in ((None, 1, None, 0, None, None, 0, 0, b"x", C.byref(out)), (None, 0, None, 0, None, None, 0, 0, None, None)):
        assert L.ldb_gpu_table_exchange(*args, C.byref(e)) == capi.LDB_ERR_INVALID
        assert b"null argument" in e.message and not out.value
        assert L.ldb_gpu_table_exchange(*args, None) == capi.LDB_ERR_INVALID


if __name__ == "__main__":  # a rank of the cross-process test
    import sys
    _worker(int(sys.argv[1]), int(sys.argv[2]), sys.argv[3])
