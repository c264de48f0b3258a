"""utf8 columns through the table exchange (ldb_gpu_table_exchange_varlen, parallel.Comm.table_exchange_varlen) against an exact model:
every rank's received table must be, cell for cell, validity for validity and string for string, the rows it owns from every source
rank in rank order, each source's rows in their source row order (every source's rows on every rank with no keys).  Also: without a utf8
column the new entry equals ldb_gpu_table_exchange byte for byte, received strings are ordinary utf8 columns for programs, ORDER BY and
gathers, capacity and the int32 offset limit fail on every rank with nothing written, every documented error, and TPC-H Q12, Q10 and
Q18 at SF1 with their string columns shipped as utf8 rather than materialized or coded.

Ranks are contexts of this process on device 0 wired by parallel.Comm.local_group; each rank calls the exchange from a thread of its own."""
import ctypes as C
import datetime
import os
import random
import re

import numpy as np
import pytest

import _progref as R
from lingodb_b200 import capi, datagen
from test_gpu_table_exchange import (KEY_SETS, WIDTH, _deal, _union_groups, all_ok, expected, on_ranks, owner, owners_np, ranks, raw_of,
                                     shard_bounds)

col, const = (lambda n: ("col", n)), (lambda v: ("const", v))
# 16 columns: every fixed-width type and five utf8 columns at different positions
COLUMNS = [("k", "int32", 0, 0), ("s", "utf8", 0, 0), ("i8", "int8", 0, 0), ("i16", "int16", 0, 0), ("t", "utf8", 0, 0), ("i32", "int32", 0, 0),
           ("i64", "int64", 0, 0), ("dw", "decimal128", 38, 2), ("u", "utf8", 0, 0), ("dn", "decimal128", 18, 2), ("dt", "date32", 0, 0),
           ("fs", "fsb4", 0, 0), ("v", "utf8", 0, 0), ("f4", "float32", 0, 0), ("f8", "float64", 0, 0), ("w", "utf8", 0, 0)]
PHYS = {n: p for n, p, _, _ in COLUMNS}
NAMES = [n for n, *_ in COLUMNS]
STRS = [n for n in NAMES if PHYS[n] == "utf8"]
FIXED = [n for n in NAMES if PHYS[n] != "utf8"]
SUBSETS = [NAMES, ["w", "k"], ["i8", "t", "dw", "s", "v"]]
EDGE = [b"", b"\0", b"\0\0", b"\x80", b"\xff", b"\xff\xfe", b"a\0b", b"x" * 300, b"PREFIX08PREFIX16"]


def rand_string(rng) -> bytes:
    n = rng.choice([0, 0, 1, 2, 7, 8, 9, 16, 31, 33, 64, 255, 300, rng.randrange(301)])
    alphabet = rng.choice([b"ab", b"abc\0", bytes(range(256))])
    return bytes(rng.choice(alphabet) for _ in range(n))


def gen(seed: int, n: int, big: int = 2) -> dict:
    """column values (None = NULL); utf8: edge strings first, NULLs, 0-300 bytes, and `big` strings of 4-64 KiB per column"""
    v = R.gen_values(seed, n, COLUMNS, null_rate=0.12, key_domain=1 << 30)
    rng = random.Random(seed)
    for s in STRS:
        vals = [EDGE[i] if i < len(EDGE) else (None if rng.random() < 0.12 else rand_string(rng)) for i in range(n)]
        for _ in range(big if n > 20 else 0):
            vals[rng.randrange(n)] = bytes(rng.randrange(256) for _ in range(rng.randrange(4096, 65537)))
        v[s] = vals
    return v


def rows_of(values: dict, lo: int, hi: int) -> list:
    return [{c: (values[c][i] if PHYS[c] == "utf8" else raw_of(PHYS[c], values[c][i])) for c in NAMES} for i in range(lo, hi)]


def stage(ctx, name: str, values: dict, how: str, seed: int):
    """values as a table of ctx in ragged batches: "host" (HOST staging), "host_sliced" (HOST Arrow slices: bitmaps from a bit offset,
    utf8 offsets not starting at 0), "device" (borrowed DEVICE batches, sliced the same way)"""
    import torch

    from lingodb_b200 import runtime
    n = len(values["k"])
    rng = random.Random(seed)
    cuts = sorted({rng.randrange(1, n) for _ in range(3)}) if n > 8 else []
    if how == "host":
        return ctx.table_from_host(R.to_table_data(name, values, COLUMNS, cuts))
    tab = runtime.Table(ctx, name, R.specs_of(COLUMNS))
    for lo, hi in zip([0] + cuts, cuts + [n]):
        off = rng.randrange(1, 12)
        ch = {}
        for cname, phys, _, _ in COLUMNS:
            part = values[cname][lo:hi]
            if phys == "utf8":  # filler strings in front: the slice's first offset is not 0
                filler = [b"pad%d" % i for i in range(off)]
                buf, bm = R.column_buffers(phys, filler + part)
                valid = np.array([True] * off + [x is not None for x in part], bool)
                bm = np.concatenate([np.packbits(valid, bitorder="little"), np.zeros(1, np.uint8)])
            else:
                buf, bm = R.column_buffers(phys, part, offset=off)
            ch[cname] = buf
            if bm is not None:
                ch[cname + "$valid"] = bm
        if how == "host_sliced":
            tab.append_host(ch, hi - lo, offset=off)
        else:
            dev = {k: tuple(torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in v) if isinstance(v, tuple) else torch.from_numpy(np.ascontiguousarray(v)).cuda()
                   for k, v in ch.items()}
            tab.append_device(dev, hi - lo, offset=off)
    torch.cuda.synchronize()
    return tab


def empty(ctx, name: str):
    from lingodb_b200 import runtime
    return runtime.Table(ctx, name, R.specs_of(COLUMNS))


def read_table(t, columns: list) -> list:
    ids = list(range(t.num_rows))
    cols = {c: (t.gather_strings(c, ids, decode=False) if PHYS[c] == "utf8" else t.gather(c, ids, cell_bytes=WIDTH[PHYS[c]])) for c in columns}
    return [{c: cols[c][i] for c in columns} for i in range(len(ids))]


def assert_received(got_tables: list, want: list, columns: list, what=""):
    for d, (t, rows) in enumerate(zip(got_tables, want)):
        assert t.num_rows == len(rows), (what, d, t.num_rows, len(rows))
        for i, (g, w) in enumerate(zip(read_table(t, columns), rows)):
            assert g == {c: w[c] for c in columns}, (what, d, i, c)


def xchg(comms, tables, keys, columns=None, **kw):
    return all_ok(comms, lambda r: comms[r].table_exchange_varlen(tables[r], keys, columns=columns, **kw))


def a16(x: int) -> int:
    return (x + 15) // 16 * 16


def region_layout(rows: list, columns: list) -> tuple:
    """the documented receive region of `rows`: (offset of every column's cells / offsets, of every utf8 column's bytes, of every
    validity array, total size)"""
    n, off, cells, chars, valid = len(rows), 0, {}, {}, {}
    for c in columns:
        cells[c] = off
        off += a16((n + 1) * 4 if PHYS[c] == "utf8" else n * WIDTH[PHYS[c]])
    for c in columns:
        if PHYS[c] == "utf8":
            chars[c] = off
            off += a16(sum(len(r[c] or b"") for r in rows))
    for c in columns:
        valid[c] = off
        off += a16(n)
    return cells, chars, valid, off


def run_isolated(args: list, env: dict, timeout: int = 900):
    """this file run as `python test_gpu_table_exchange_strings.py *args` with `env` added; the child is killed and reaped whatever ends
    the call"""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([root] + [x for x in os.environ.get("PYTHONPATH", "").split(os.pathsep) if x]), **env)
    p = subprocess.Popen([sys.executable, os.path.abspath(__file__)] + args, env=env)
    try:
        return p.wait(timeout=timeout)
    finally:
        if p.poll() is None:
            p.kill()
        p.wait()


# ---------------------------------------------------------------------------------------------------- 1. exact against the model
@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_exchange_with_strings_matches_the_model(world):
    if world == 8:  # eight in-process ranks on one GPU need more hardware work queues (as test_gpu_dict_unify.py)
        assert run_isolated(["model", str(world)], {"CUDA_DEVICE_MAX_CONNECTIONS": "32"}) == 0
        return
    check_model(world)


def check_model(world: int):
    from test_gpu_exchange import heap_read
    n = 1200 if world < 8 else 1600
    v = gen(700 + world, n, big=3)
    bounds = shard_bounds(n, world, 23 * world)
    with ranks(world, user_bytes=32 << 20) as (ctxs, comms):
        hows = ["host", "host_sliced", "device"]
        tabs = [stage(c, f"s{r}", {k: x[lo:hi] for k, x in v.items()}, hows[r % 3], 41 * world + r) if hi > lo else empty(c, f"s{r}")
                for r, (c, (lo, hi)) in enumerate(zip(ctxs, bounds))]
        sources = [rows_of(v, lo, hi) for lo, hi in bounds]
        for keys in KEY_SETS:
            for columns in SUBSETS:
                got = xchg(comms, tabs, keys, columns=columns)
                want = expected(sources, keys, world)
                assert_received(got, want, columns, (world, keys, columns))
                if keys and world > 1:
                    assert sum(1 for t in got if t.num_rows) > 1, keys
                # the receive region holds the documented layout (it is free again, but not cleared, after the call)
                for d, (cm, rows) in enumerate(zip(comms, want)):
                    cells, chars, valid, size = region_layout(rows, columns)
                    raw = heap_read(cm, 0, size)
                    for c in columns:
                        vb = np.frombuffer(raw, np.uint8, len(rows), valid[c])
                        assert vb.tolist() == [int(r[c] is not None) for r in rows], (world, keys, d, c)
                        if PHYS[c] == "utf8":
                            offs = np.frombuffer(raw, np.int32, len(rows) + 1, cells[c]).tolist()
                            data = raw[chars[c]:chars[c] + offs[-1]]
                            assert offs[0] == 0 and [data[a:b] for a, b in zip(offs, offs[1:])] == [r[c] or b"" for r in rows], (world, keys, d, c)
                for t in got:
                    t.destroy()
        # an exchange of received tables (validity bytes, offsets from 0), and of received strings next to their keys only
        first = xchg(comms, tabs, ["i64"], columns=NAMES)
        again = xchg(comms, first, ["dn", "dt"])
        assert_received(again, expected(expected(sources, ["i64"], world), ["dn", "dt"], world), NAMES, (world, "again"))
        for t in first + again:
            t.destroy()


# ---------------------------------------------------------------------------------------------------- 2. the same without strings
@pytest.mark.gpu
@pytest.mark.parametrize("keys", [["i64"], ["k", "i16", "i32", "dn"], []])
def test_without_strings_the_tables_and_regions_equal_the_fixed_width_exchange(keys):
    from lingodb_b200 import program as P
    from test_gpu_exchange import heap_read
    world, n = 3, 2000
    v = gen(31, n)
    bounds = [(0, 500), (500, 1300), (1300, 2000)]
    with ranks(world, user_bytes=8 << 20) as (ctxs, comms):
        tabs = [stage(c, f"s{r}", {k: x[lo:hi] for k, x in v.items()}, ["device", "host", "host_sliced"][r], r) for r, (c, (lo, hi)) in enumerate(zip(ctxs, bounds))]
        mats = [P.RawTable(c, P.materialize(c, t, [col("i64"), col("dn"), col("dt")], where=("not", ("isnull", col("i8"))))) for c, t in zip(ctxs, tabs)]
        for srcs, columns, ks in ((tabs, FIXED, keys), (mats, ["c0", "c1", "c2"], ["c0"] if keys else [])):
            span = 1 << 20
            for cm in comms:
                e = capi.Error()
                capi.check(cm.L.ldb_gpu_comm_heap_zero(cm.h, 0, span, C.byref(e)), e)
            old = all_ok(comms, lambda r: comms[r].table_exchange(srcs[r], ks, columns=columns))
            old_regions = [heap_read(cm, 0, span) for cm in comms]
            new = xchg(comms, srcs, ks, columns=columns)
            new_regions = [heap_read(cm, 0, span) for cm in comms]
            assert new_regions == old_regions, keys
            for a, b in zip(old, new):
                ids = list(range(a.num_rows))
                assert b.num_rows == a.num_rows
                for c in columns:
                    w = 16 if c.startswith("c") else WIDTH[PHYS[c]]
                    assert b.gather(c, ids, cell_bytes=w) == a.gather(c, ids, cell_bytes=w), (keys, c)
                a.destroy()
                b.destroy()
        for t in mats:
            t.destroy()


# ---------------------------------------------------------------------------------------------------- 3. source kinds
@pytest.mark.gpu
def test_compressed_batches_and_shards_of_many_tiles_keep_source_order_with_strings():
    """a 70 000-row HOST batch (compressed staging) and a 5 M-row DEVICE shard (1 221 tiles, past the scan's 1 024-entry chunks), each
    with a utf8 column whose strings name their row"""
    import torch

    from lingodb_b200 import runtime
    world = 2
    specs = [datagen.ColumnSpec("v", "int64", 0, 0), datagen.ColumnSpec("s", "utf8", 0, 0)]
    with ranks(world, user_bytes=512 << 20) as (ctxs, comms):
        vals, strs, tabs = [], [], []
        for r, (c, n) in enumerate(zip(ctxs, [70_000, 5_000_000])):
            v = np.arange(n, dtype=np.int64) * 7919 + r * (1 << 40)
            s = np.char.encode(np.char.add("r%d-" % r, (np.arange(n) * 13 % 100_003).astype(str)), "ascii")
            offs = np.zeros(n + 1, np.int32)
            offs[1:] = np.cumsum(np.char.str_len(s))
            data = np.frombuffer(b"".join(s.tolist()) + b"\0", np.uint8).copy()
            t = runtime.Table(c, f"v{r}", specs)
            if r == 0:
                t.append_host({"v": v, "s": (offs, data)}, n)
            else:
                t.append_device({"v": torch.from_numpy(v).cuda(), "s": (torch.from_numpy(offs).cuda(), torch.from_numpy(data).cuda())}, n)
            tabs.append(t)
            vals.append(v)
            strs.append(s)
        torch.cuda.synchronize()
        got = xchg(comms, tabs, ["v"])
        for d, t in enumerate(got):
            picks = [owners_np([(v, np.ones(len(v), bool))], world) == d for v in vals]
            want_v = np.concatenate([v[m] for v, m in zip(vals, picks)])
            want_s = np.concatenate([s[m] for s, m in zip(strs, picks)])
            assert t.num_rows == len(want_v)
            from test_gpu_table_exchange import gather_np
            cells, valid = gather_np(t, "v", 8)
            assert valid.all() and (cells.view(np.int64).reshape(-1) == want_v).all(), d
            step = max(1, len(want_v) // 20_000)  # a sample of the strings, spread over every tile
            ids = list(range(0, len(want_v), step)) + [len(want_v) - 1]
            assert t.gather_strings("s", ids, decode=False) == [bytes(want_s[i]) for i in ids], d
            t.destroy()


# ---------------------------------------------------------------------------------------------------- 4. capacity and the offset limit
@pytest.mark.gpu
def test_capacity_is_decided_by_the_bytes_and_the_named_size_succeeds():
    from test_gpu_exchange import SENTINEL, heap_fill, heap_read
    world, off = 3, 4096
    rng = random.Random(9)
    per = [[(i * world + r, bytes(rng.randrange(256) for _ in range(rng.randrange(2000, 9000)))) for i in range(6)] for r in range(world)]
    with ranks(world, user_bytes=4 << 20) as (ctxs, comms):
        from test_gpu_strings import make_table
        tabs = [make_table(c, f"c{r}", {"k": ("int64", [k for k, _ in per[r]]), "s": ("utf8", [s for _, s in per[r]])}) for r, c in enumerate(ctxs)]
        sources = [[{"k": k, "s": s} for k, s in p] for p in per]
        want = expected(sources, ["k"], world)
        need = max(a16(len(w) * 8) + a16((len(w) + 1) * 4) + a16(sum(len(x["s"]) for x in w)) + 2 * a16(len(w)) for w in want)
        assert need > 20 * max(a16(len(w) * 8) + a16((len(w) + 1) * 4) + 2 * a16(len(w)) for w in want)  # the bytes decide the size
        span = need + 8192
        for cm in comms:
            heap_fill(cm, off - 1024, span)
        _, errs = on_ranks(comms, lambda r: comms[r].table_exchange_varlen(tabs[r], ["k"], recv_offset=off, recv_bytes=need - 16))
        assert all(e is not None and e.code == capi.LDB_ERR_CAPACITY for e in errs), errs
        assert {int(re.search(r"retry with recv_bytes (\d+)", str(e)).group(1)) for e in errs} == {need}
        for cm in comms:
            assert (np.frombuffer(heap_read(cm, off - 1024, span), dtype=np.uint32) == SENTINEL).all()
        got = xchg(comms, tabs, ["k"], recv_offset=off, recv_bytes=need)
        for t, rows in zip(got, want):
            ids = list(range(t.num_rows))
            assert t.gather("k", ids, cell_bytes=8) == [x["k"] for x in rows]
            assert t.gather_strings("s", ids, decode=False) == [x["s"] for x in rows]
            t.destroy()


@pytest.mark.gpu
def test_more_than_int32_bytes_for_one_receiver_fails_on_every_rank():
    """rank 0 sends one receiver 2 200 000 000 bytes of one utf8 column (two DEVICE batches over one 1.1 GB buffer): every rank fails with
    LDB_ERR_UNSUPPORTED naming the column and the count, nothing is written, and the ranks stay in step"""
    import torch

    from lingodb_b200 import runtime
    from test_gpu_exchange import SENTINEL, heap_fill, heap_read
    world, half = 2, 1_100_000_000
    key = next(k for k in range(100) if owner([k], world) == 1)
    with ranks(world, user_bytes=1 << 20) as (ctxs, comms):
        specs = [datagen.ColumnSpec("k", "int64", 0, 0), datagen.ColumnSpec("s", "utf8", 0, 0)]
        data = torch.zeros(half, dtype=torch.uint8, device="cuda")
        offs = torch.tensor([0, half // 2, half], dtype=torch.int32, device="cuda")
        keys = torch.full((2,), key, dtype=torch.int64, device="cuda")
        big = runtime.Table(ctxs[0], "big", specs)
        for _ in range(2):
            big.append_device({"k": keys, "s": (offs, data)}, 2)
        small = runtime.Table(ctxs[1], "small", specs)
        small.append_device({"k": keys[:1], "s": (torch.zeros(2, dtype=torch.int32, device="cuda"), data[:16])}, 1)
        torch.cuda.synchronize()
        tabs = [big, small]
        for cm in comms:
            heap_fill(cm, 0, 1 << 16)
        _, errs = on_ranks(comms, lambda r: comms[r].table_exchange_varlen(tabs[r], ["k"]))
        assert all(e is not None and e.code == capi.LDB_ERR_UNSUPPORTED and "2200000000" in str(e) and "column s" in str(e) for e in errs), errs
        for cm in comms:
            assert (np.frombuffer(heap_read(cm, 0, 1 << 16), dtype=np.uint32) == SENTINEL).all()
        got = xchg(comms, tabs, ["k"], columns=["k"])  # still in step
        assert [t.num_rows for t in got] == [0, 5]
        for t in got:
            t.destroy()
        del data


# ---------------------------------------------------------------------------------------------------- 5. errors
@pytest.mark.gpu
def test_documented_errors():
    with ranks(2, user_bytes=1 << 20) as (ctxs, comms):
        c, cm = ctxs[0], comms[0]
        v = gen(3, 40, big=0)
        t = c.table_from_host(R.to_table_data("t", v, COLUMNS))
        other = ctxs[1].table_from_host(R.to_table_data("o", v, COLUMNS))
        L, user = c.L, cm.heap()[1]

        def call(table=t, keys=("i64",), columns=("s",), comm=cm, off=0, nbytes=1 << 16, out=True, n_keys=None, n_columns=None):
            kn = [k.encode() for k in keys]
            karr = (C.c_char_p * max(1, len(kn)))(*kn)
            carr = None
            if columns is not None:
                cn = [x.encode() for x in columns]
                carr = (C.c_char_p * max(1, len(cn)))(*cn)
            res, e = C.c_void_p(), capi.Error()
            rc = L.ldb_gpu_table_exchange_varlen(table.h if table is not None else None, len(kn) if n_keys is None else n_keys, karr,
                                                 (len(columns) if columns is not None else 0) if n_columns is None else n_columns, carr,
                                                 comm.h if comm is not None else None, off, nbytes, b"x", C.byref(res) if out else None, C.byref(e))
            return rc, e.message.decode()
        INVALID, UNSUP = capi.LDB_ERR_INVALID, capi.LDB_ERR_UNSUPPORTED
        cases = [(dict(table=None), INVALID, "null argument"), (dict(comm=None), INVALID, "null argument"), (dict(out=False), INVALID, "null argument"),
                 (dict(n_keys=5, keys=("i64",) * 5), INVALID, "0..4 key columns"), (dict(keys=("nope",)), INVALID, "unknown key column"),
                 (dict(columns=("s", "nope")), INVALID, "unknown column"), (dict(columns=("s",) * 17), INVALID, "up to 16 columns"),
                 (dict(columns=("s",), n_columns=0), INVALID, "1..16 columns"), (dict(table=other), INVALID, "different contexts"),
                 (dict(off=8), INVALID, "16-byte aligned"), (dict(nbytes=user + 16), INVALID, "outside"),
                 (dict(keys=("s",)), UNSUP, "exchange keys"), (dict(keys=("i64", "t")), UNSUP, "exchange keys"), (dict(keys=("f8",)), UNSUP, "exchange keys")]
        for kw, code, msg in cases:
            rc, m = call(**kw)
            assert rc == code and msg in m, (kw, rc, m)
        c.graph_begin()
        rc, m = call()
        c.graph_end().destroy()
        assert rc == UNSUP and "captured" in m, m
        # none of the refused calls started a collective; all 16 columns (five utf8) ship
        tabs = [t, ctxs[1].table_from_host(R.to_table_data("u", v, COLUMNS))]
        got = xchg(comms, tabs, ["i64"], columns=None)
        assert sum(x.num_rows for x in got) == 80
        sources = [rows_of(v, 0, 40)] * 2
        assert_received(got, expected(sources, ["i64"], 2), NAMES, "all columns")
        for x in got:
            x.destroy()


def test_entry_point_rejects_null_arguments_without_a_device():
    """Without a device no context, table or comm can exist: what reaches the entry point is null handles, refused before any CUDA call."""
    L = capi.lib()
    assert capi.SIGNATURES["ldb_gpu_table_exchange_varlen"] == capi.SIGNATURES["ldb_gpu_table_exchange"]
    out, e = C.c_void_p(), capi.Error()
    for args in ((None, 1, None, 0, None, None, 0, 0, b"x", C.byref(out)), (None, 0, None, 0, None, None, 0, 0, None, None)):
        assert L.ldb_gpu_table_exchange_varlen(*args, C.byref(e)) == capi.LDB_ERR_INVALID
        assert b"null argument" in e.message and not out.value
        assert L.ldb_gpu_table_exchange_varlen(*args, None) == capi.LDB_ERR_INVALID


# ---------------------------------------------------------------------------------------------------- 6. received strings are ordinary columns
M64 = (1 << 64) - 1


def per_row(ctx, table, expr) -> list:
    """the value of `expr` for every row of `table`, in row order (None for NULL)"""
    from lingodb_b200 import program as P
    mt = P.RawTable(ctx, P.materialize(ctx, table, [("rowid",), expr]))
    ids = list(range(mt.num_rows))
    res = dict(zip(mt.gather("c0", ids), mt.gather("c1", ids)))
    mt.destroy()
    return [res[i] for i in range(table.num_rows)]


@pytest.mark.gpu
def test_received_strings_work_in_programs_order_by_and_gathers():
    from lingodb_b200 import program as P
    world, n = 3, 900
    v = gen(66, n, big=1)
    rng = random.Random(4)
    v["s"] = [None if rng.random() < 0.1 else rng.choice([b"", b"ab", b"abc", b"abd", b"b", b"\xffz", b"PREFIX08-tail", b"ab\0"]) + rand_string(rng)[:5] for _ in range(n)]
    bounds = [(0, 200), (200, 650), (650, 900)]
    key8 = lambda s: int.from_bytes(s[:8].ljust(8, b"\0"), "big")
    with ranks(world, user_bytes=16 << 20) as (ctxs, comms):
        tabs = [stage(c, f"s{r}", {k: x[lo:hi] for k, x in v.items()}, ["host", "device", "host_sliced"][r], r) for r, (c, (lo, hi)) in enumerate(zip(ctxs, bounds))]
        got = xchg(comms, tabs, ["i32"], columns=["i32", "s", "w"])
        want = expected([rows_of(v, lo, hi) for lo, hi in bounds], ["i32"], world)
        for r, (c, t, rows) in enumerate(zip(ctxs, got, want)):
            S = [x["s"] for x in rows]
            exprs = [("strcmp", "<", "s", "abc"), ("strcmp", "=", "s", "ab"), ("like", "prefix", "s", "ab"), ("like", "suffix", "s", "z"),
                     ("like", "contains", "s", "b"), ("strkey8", "s")]
            models = [lambda s: int(s < b"abc"), lambda s: int(s == b"ab"), lambda s: int(s.startswith(b"ab")), lambda s: int(s.endswith(b"z")),
                      lambda s: int(b"b" in s), key8]
            for e, f in zip(exprs, models):
                got_e = [None if x is None else x & M64 for x in per_row(c, t, e)]
                assert got_e == [None if s is None else f(s) & M64 for s in S], (r, e)
            # STRCODE insert, then lookup: equal strings get equal codes, NULL none
            d = P.dict_state(c, 1024, 1 << 16)
            codes, look = per_row(c, t, ("strcode", d, "s")), per_row(c, t, ("strcode", d, "s", "lookup"))
            assert codes == look
            assert all((codes[i] is None) == (s is None) for i, s in enumerate(S))
            assert len({codes[i] for i, s in enumerate(S) if s is not None}) == len({s for s in S if s is not None})
            assert all(codes[i] == codes[j] for i in range(len(S)) for j in range(i) if S[i] is not None and S[i] == S[j])
            c.L.ldb_gpu_state_destroy(d)
            # a side-column fetch of the received utf8 column at the row after each row's
            fetched = per_row(c, t, ("strcmp", ">=", ("fetch", t, ("add", ("rowid",), const(1)), "w"), "PREFIX08PREFIX16"))
            assert fetched == [None if i + 1 >= len(rows) or rows[i + 1]["w"] is None else int(rows[i + 1]["w"] >= b"PREFIX08PREFIX16") for i in range(len(rows))]
            # ORDER BY the string (NULLs last, ties in row order) and gathers
            order = t.order_by_keys([("s", False)])
            assert order == sorted(range(len(S)), key=lambda i: (S[i] is None, S[i] or b"", i))
            assert t.gather_strings("w", order, decode=False) == [rows[i]["w"] for i in order]
            t.destroy()


# ---------------------------------------------------------------------------------------------------- 7. distributed TPC-H at SF1
@pytest.fixture(scope="module")
def sf1():
    from lingodb_b200 import dbgen
    return dbgen.tpch(1.0, extended=True)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_distributed_tpch_q12_q10_q18_ship_their_strings(sf1, world):
    from lingodb_b200 import program as P, runtime
    from test_reference_answers_sf1 import GOLD, day, dec
    d = lambda s: (datetime.date.fromisoformat(s) - datetime.date(1970, 1, 1)).days
    key8 = lambda s: int.from_bytes(s.encode()[:8].ljust(8, b"\0"), "big")
    with ranks(world, user_bytes=1 << 30) as (ctxs, comms):
        lis = [c.table_from_host(_deal(sf1["lineitem"], world, r, 0)) for r, c in enumerate(ctxs)]
        ods = [c.table_from_host(_deal(sf1["orders"], world, r, 1)) for r, c in enumerate(ctxs)]
        cus = [c.table_from_host(_deal(sf1["customer"], world, r, 2)) for r, c in enumerate(ctxs)]
        nat = [c.table_from_host(sf1["nation"]) if r == world - 1 else runtime.Table(c, "nation", sf1["nation"].columns) for r, c in enumerate(ctxs)]
        mat = lambda r, t, outs, where=None: P.RawTable(ctxs[r], P.materialize(ctxs[r], t, outs, where=where))
        drop = lambda ts: [t.destroy() for t in ts]

        def destroy(*lists):
            for xs in lists:
                for c, s in zip(ctxs, xs):
                    c.L.ldb_gpu_state_destroy(s)
        # ---- Q12: raw lineitem and orders rows exchanged on the order key; the string predicates and the STRKEY8 group key run on the
        # receiving rank
        lx = xchg(comms, lis, ["l_orderkey"], columns=["l_orderkey", "l_shipdate", "l_commitdate", "l_receiptdate", "l_shipmode"])
        ox = xchg(comms, ods, ["o_orderkey"], columns=["o_orderkey", "o_orderpriority"])
        assert sum(t.num_rows for t in lx) == sf1["lineitem"].num_rows
        locals_, owneds = [], []
        for r, c in enumerate(ctxs):
            j = runtime.join_table(c, 1_000_000, unique=True)
            high = ("or", ("strcmp", "=", "o_orderpriority", "1-URGENT"), ("strcmp", "=", "o_orderpriority", "2-HIGH"))
            P.build_join(c, ox[r], j, col("o_orderkey"), payload=("case", high, const(1), const(0)))
            pr = ("probe", j, col("l_orderkey"))
            where = ("and", ("and", ("or", ("strcmp", "=", "l_shipmode", "MAIL"), ("strcmp", "=", "l_shipmode", "SHIP")),
                             ("and", ("cmp", "<", col("l_commitdate"), col("l_receiptdate")), ("cmp", "<", col("l_shipdate"), col("l_commitdate")))),
                     ("and", ("and", ("cmp", ">=", col("l_receiptdate"), const(d("1994-01-01"))), ("cmp", "<", col("l_receiptdate"), const(d("1995-01-01")))),
                      ("not", ("isnull", pr))))
            aggs = [("sum", ("case", ("cmp", "=", pr, const(1)), const(1), const(0))), ("sum", ("case", ("cmp", "=", pr, const(0)), const(1), const(0)))]
            locals_.append(P.group_by(c, lx[r], [("strkey8", "l_shipmode")], aggs, where=where, expected_groups=16))
            owneds.append(P.hashagg_state(c, 1, ["sum", "sum"], 16))
            c.L.ldb_gpu_state_destroy(j)
        all_ok(comms, lambda r: comms[r].hashagg_exchange(locals_[r], owneds[r]))
        got = _union_groups(ctxs, owneds, 1, 2)
        assert [[m, str(got[(key8(m),)][0]), str(got[(key8(m),)][1])] for m in ("MAIL", "SHIP")] == GOLD["q12_rows"]
        drop(lx + ox)
        destroy(locals_, owneds)
        # ---- Q10: returned-item revenue per customer merged on the customer's owner rank, where the exchanged customer row (c_name as
        # utf8) lands too; nation broadcast with n_name; both names read from the received tables at row ids the programs materialized
        revenue = ("mul", col("l_extendedprice"), ("sub", const(100), col("l_discount")))
        om = [mat(r, ods[r], [col("o_orderkey"), col("o_custkey")], ("and", ("cmp", ">=", col("o_orderdate"), const(d("1993-10-01"))),
                                                                         ("cmp", "<", col("o_orderdate"), const(d("1994-01-01"))))) for r in range(world)]
        lm = [mat(r, lis[r], [col("l_orderkey"), revenue], ("cmp", "=", col("l_returnflag"), const(ord("R")))) for r in range(world)]
        ox, lx = xchg(comms, om, ["c0"]), xchg(comms, lm, ["c0"])
        cx = xchg(comms, cus, ["c_custkey"], columns=["c_custkey", "c_name", "c_nationkey"])
        nx = xchg(comms, nat, [], columns=["n_nationkey", "n_name"])
        locals_, owneds = [], []
        for r, c in enumerate(ctxs):
            oj = runtime.join_table(c, 200_000, unique=True)
            P.build_join(c, ox[r], oj, col("c0"), payload=col("c1"))
            ck = ("probe", oj, col("c0"))
            locals_.append(P.group_by(c, lx[r], [ck], [("sum", col("c1"))], where=("not", ("isnull", ck)), expected_groups=100_000))
            owneds.append(P.hashagg_state(c, 1, ["sum"], 100_000))
            c.L.ldb_gpu_state_destroy(oj)
        all_ok(comms, lambda r: comms[r].hashagg_exchange(locals_[r], owneds[r]))
        rows = []
        for r, c in enumerate(ctxs):
            g = P.groups_table(c, owneds[r])
            cj, nj = runtime.join_table(c, 200_000, unique=True), runtime.join_table(c, 64, unique=True)
            P.build_join(c, cx[r], cj, col("c_custkey"), payload=("rowid",))
            P.build_join(c, nx[r], nj, col("n_nationkey"), payload=("rowid",))
            crow = ("probe", cj, col("k0"))
            mt = mat(r, g, [col("k0"), col("a0"), crow, ("probe", nj, ("fetch", cx[r], crow, "c_nationkey"))])
            ids = mt.order_by("c1", descending=True, limit=20)
            top = list(zip(*[mt.gather(f"c{i}", ids) for i in range(4)]))
            assert all(x[2] is not None and x[3] is not None for x in top)  # every owned customer's row is on its owner rank
            cname = cx[r].gather_strings("c_name", [x[2] for x in top])
            nname = nx[r].gather_strings("n_name", [x[3] for x in top])
            rows += [(ck_, rev, cn, nn) for (ck_, rev, _, _), cn, nn in zip(top, cname, nname)]
            for x in (mt, g):
                x.destroy()
            c.L.ldb_gpu_state_destroy(cj)
            c.L.ldb_gpu_state_destroy(nj)
        assert {t.num_rows for t in nx} == {25}
        rows.sort(key=lambda x: -x[1])
        assert [[str(k), cn, dec(rev, 4), nn] for k, rev, cn, nn in rows[:20]] == [[g[0], g[1], g[2], g[4]] for g in GOLD["q10_rows"]]
        drop(om + lm + ox + lx + nx)
        destroy(locals_, owneds)
        # ---- Q18: lineitem sums merged on their owners, orders exchanged on o_orderkey, c_name shipped as utf8 with the customers
        locals_ = [P.group_by(c, t, [col("l_orderkey")], [("sum", col("l_quantity"))], expected_groups=1_600_000) for c, t in zip(ctxs, lis)]
        owneds = [P.hashagg_state(c, 1, ["sum"], 1_600_000) for c in ctxs]
        all_ok(comms, lambda r: comms[r].hashagg_exchange(locals_[r], owneds[r]))
        ox = xchg(comms, ods, ["o_orderkey"], columns=["o_custkey", "o_orderkey", "o_orderdate", "o_totalprice"])
        bx = xchg(comms, cx, [], columns=["c_custkey", "c_name"])  # every customer's name on every rank
        rows = []
        for r, c in enumerate(ctxs):
            groups = P.groups_table(c, owneds[r])
            big = runtime.join_table(c, 4096, unique=True)
            P.build_join(c, groups, big, col("k0"), payload=col("a0"), where=("cmp", ">", col("a0"), const(30000)))
            cj = runtime.join_table(c, 200_000, unique=True)
            P.build_join(c, bx[r], cj, col("c_custkey"), payload=("rowid",))
            pb = ("probe", big, col("o_orderkey"))
            mt = mat(r, ox[r], [("probe", cj, col("o_custkey")), col("o_custkey"), col("o_orderkey"), col("o_orderdate"), col("o_totalprice"), pb], ("not", ("isnull", pb)))
            ids = list(range(mt.num_rows))
            part = list(zip(*[mt.gather(f"c{i}", ids) for i in range(6)]))
            names = bx[r].gather_strings("c_name", [x[0] for x in part])
            rows += [(n_,) + x[1:] for n_, x in zip(names, part)]
            for x in (mt, groups):
                x.destroy()
            c.L.ldb_gpu_state_destroy(big)
            c.L.ldb_gpu_state_destroy(cj)
        rows.sort(key=lambda x: (-x[4], x[3]))
        got18 = [[x[0], str(x[1]), str(x[2]), day(x[3]), dec(x[4], 2), dec(x[5], 2)] for x in rows[:100]]
        assert got18 == GOLD["q18_rows"]
        drop(ox + bx + cx)
        destroy(locals_, owneds)


# ---------------------------------------------------------------------------------------------------- 8. cross-process (two or more GPUs)
def _worker(rank: int, world: int, rendezvous: str):
    """one rank of test_across_processes_when_there_are_two_gpus: its shard → exchange → its received rows as JSON (strings as hex)"""
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
    comm = parallel.Comm(ctx, rank, world, user_bytes=32 << 20, exchange=swap)
    v = gen(1234, 2000)
    lo, hi = 2000 * rank // world, 2000 * (rank + 1) // world
    tab = stage(ctx, "s", {k: x[lo:hi] for k, x in v.items()}, "host", rank)
    res = {}
    for keys in (["i64", "dt"], []):
        t = comm.table_exchange_varlen(tab, keys, columns=NAMES)
        res[",".join(keys)] = [{c: (x[c].hex() if isinstance(x[c], bytes) else x[c]) for c in NAMES} for x in read_table(t, NAMES)]
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
            procs.append(subprocess.Popen([sys.executable, os.path.abspath(__file__), "worker", str(r), str(world), str(tmp_path)], env=env))
        codes = [p.wait(timeout=600) for p in procs]
    finally:  # no rank outlives the test, whatever ended it
        for p in procs:
            if p.poll() is None:
                p.kill()
            p.wait()
    assert codes == [0] * world
    v = gen(1234, 2000)
    sources = [rows_of(v, 2000 * r // world, 2000 * (r + 1) // world) for r in range(world)]
    for keys in (["i64", "dt"], []):
        want = expected(sources, keys, world)
        for r in range(world):
            got = json.load(open(tmp_path / f"out{r}.json"))[",".join(keys)]
            assert got == [{c: (w[c].hex() if isinstance(w[c], bytes) else w[c]) for c in NAMES} for w in want[r]], (keys, r)


if __name__ == "__main__":  # an isolated case, or a rank of the cross-process test
    import sys
    if sys.argv[1] == "model":
        check_model(int(sys.argv[2]))
    else:
        _worker(int(sys.argv[2]), int(sys.argv[3]), sys.argv[4])
