"""ORDER BY across ranks (ldb_gpu_table_sort_exchange, parallel.Comm.sort_exchange) against an exact model: Python's `sorted` with the
order of ldb_gpu_table_order_by_keys (per key its NULL flag, then its value; DESC swaps both) and (source rank, source row) after the
keys.  Every rank's table must be its slice of that order cell for cell, first_row and total_rows must place it, the slices in rank
order must also equal order_by_keys over the concatenated shards, and with LIMIT rank 0 alone holds the first `limit` rows.  Also: the
balance the splitters reach at 1 M rows per rank over 8 ranks, a region sized for world * limit rows, capacity with sentinels, every
documented error, and the final ORDER BY of TPC-H Q16 (no LIMIT), Q18, Q3 and Q10 (LIMIT) at SF1 on the device.

Ranks are contexts of this process on device 0 wired by parallel.Comm.local_group; each rank calls the sort exchange from a thread of
its own."""
import ctypes as C
import os
import random
import sys

import numpy as np
import pytest

import _progref as R
from lingodb_b200 import capi
from test_gpu_table_exchange import all_ok, on_ranks, ranks, shard_bounds
from test_gpu_table_exchange_strings import COLUMNS, NAMES, PHYS, empty, gen, read_table, rows_of, stage

I128_MAX = (1 << 127) - 1
DW_EDGES = [(1 << 64) - 1, 1 << 64, -(1 << 64), -((1 << 64) - 1), -1, 0, I128_MAX, -I128_MAX, -(1 << 127), (1 << 63), -(1 << 63) - 1]
I32_EDGES = [-(1 << 31), (1 << 31) - 1, 0, -1]
# (column, descending) lists: 1-4 keys, mixed ASC / DESC, every accepted key type; "k" has few values (runs of ties)
KEY_SETS = [[("k", False)], [("dw", True)], [("dn", False), ("i32", True)], [("k", True), ("dt", False), ("fs", True)],
            [("i64", True), ("k", False), ("dn", True), ("dw", False)]]
SUBSETS = [NAMES, ["w", "s", "i8"]]  # every column (the keys among them), or strings and an int8 with the keys hidden
LIMITS = [None, 0, 1, 37, 10**9]


def model_key(row: dict, keys: list):
    out = []
    for c, desc in keys:
        v = row[c]
        flag, val = (1, 0) if v is None else (0, v)
        out += [-flag, -val] if desc else [flag, val]
    return out


def model(sources: list, keys: list, limit=None) -> list:
    """the global order of the rows of every source (rank order, then row order, breaks ties), cut at `limit`"""
    tagged = [(model_key(row, keys), s, i, row) for s, rows in enumerate(sources) for i, row in enumerate(rows)]
    out = [t[3] for t in sorted(tagged, key=lambda t: (t[0], t[1], t[2]))]
    return out if limit is None else out[:limit]


def order_by_keys(t, keys: list) -> list:
    """row ids of ldb_gpu_table_order_by_keys over the single-batch table t"""
    n = t.num_rows
    cols = (C.c_char_p * len(keys))(*[c.encode() for c, _ in keys])
    desc = (C.c_int32 * len(keys))(*[int(d) for _, d in keys])
    ids, m, e = (C.c_int64 * max(1, n))(), C.c_int64(), capi.Error()
    capi.check(t.ctx.L.ldb_gpu_table_order_by_keys(t.h, len(keys), cols, desc, -1, ids, C.byref(m), C.byref(e)), e)
    return list(ids[:m.value])


def sort_x(comms, tables, keys, **kw):
    return all_ok(comms, lambda r: comms[r].sort_exchange(tables[r], keys, **kw))


def check_slices(got: list, want: list, columns: list, limit, what=""):
    """every rank's table is its slice of `want`, in rank order, with first_row and total_rows placing it"""
    at = 0
    for d, (t, first, total) in enumerate(got):
        assert first == at and total == len(want), (what, d, first, at, total, len(want))
        if limit is not None and d > 0:
            assert t.num_rows == 0, (what, d, t.num_rows)
        rows = read_table(t, columns)
        assert rows == [{c: w[c] for c in columns} for w in want[at:at + t.num_rows]], (what, d)
        at += t.num_rows
    assert at == len(want), (what, at, len(want))


def gen_edges(seed: int, n: int) -> dict:
    v = gen(seed, n, big=1)
    rng = random.Random(seed)
    v["k"] = [rng.choice([None, -1, 0, 1, 2]) for _ in range(n)]
    for i in rng.sample(range(n), min(n, 60)):
        v["dw"][i] = rng.choice(DW_EDGES)
        v["i32"][i] = rng.choice(I32_EDGES)
    return v


# ---------------------------------------------------------------------------------------------------- 1. exact against the model
@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_sort_exchange_matches_the_model(world):
    if world == 8:  # eight in-process ranks on one GPU need more hardware work queues (as test_gpu_dict_unify.py)
        assert run_isolated(["model", str(world)], {"CUDA_DEVICE_MAX_CONNECTIONS": "32"}) == 0
        return
    check_model(world)


def check_model(world: int):
    n = 900 if world < 8 else 1400
    v = gen_edges(900 + world, n)
    bounds = shard_bounds(n, world, 31 * world)
    with ranks(world, user_bytes=32 << 20) as (ctxs, comms):
        # HOST staging narrows "dn" (decimal(18, 2)) to 8-byte cells, DEVICE batches hold it in 16 bytes: shards of both widths
        hows = ["host", "device", "host_sliced"]
        tabs = [stage(c, f"s{r}", {k: x[lo:hi] for k, x in v.items()}, hows[r % 3], 53 * world + r) if hi > lo else empty(c, f"s{r}")
                for r, (c, (lo, hi)) in enumerate(zip(ctxs, bounds))]
        sources = [rows_of(v, lo, hi) for lo, hi in bounds]
        # the second oracle: order_by_keys over the concatenation of the shards, one HOST batch
        whole = ctxs[0].table_from_host(R.to_table_data("whole", v, COLUMNS))
        flat = [row for rows in sources for row in rows]
        for keys in KEY_SETS:
            ref = [flat[i] for i in order_by_keys(whole, keys)]
            for columns in SUBSETS:
                for limit in LIMITS:
                    want = model(sources, keys, limit)
                    assert want == (ref if limit is None else ref[:limit]), (keys, limit)
                    got = sort_x(comms, tabs, keys, columns=columns, limit=limit)
                    check_slices(got, want, columns, limit, (world, keys, columns, limit))
                    if limit is None and world > 1 and len(want) > 100:
                        assert sum(1 for t, _, _ in got if t.num_rows) > 1, keys
                    for t, _, _ in got:
                        t.destroy()
        # received and exported tables are sources too: sort a sorted result again by other keys
        first = sort_x(comms, tabs, [("i64", False)], columns=NAMES)
        again = sort_x(comms, [t for t, _, _ in first], [("dn", True), ("dt", False)], columns=NAMES)
        flat1 = [r for t, _, _ in first for r in read_table(t, NAMES)]
        per_rank = []
        at = 0
        for t, _, _ in first:
            per_rank.append(flat1[at:at + t.num_rows])
            at += t.num_rows
        check_slices(again, model(per_rank, [("dn", True), ("dt", False)]), NAMES, None, (world, "again"))
        for t, _, _ in first + again:
            t.destroy()


# ---------------------------------------------------------------------------------------------------- 2. shapes of the shards
@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["one_rank_holds_all", "fewer_rows_than_ranks", "all_equal", "sorted", "reverse", "rank_correlated"])
def test_shard_shapes(shape):
    world = 3
    with ranks(world, user_bytes=16 << 20) as (ctxs, comms):
        n = {"fewer_rows_than_ranks": 2}.get(shape, 600)
        v = gen(77, n, big=0)
        keyvals = {"all_equal": [5] * n, "sorted": list(range(n)), "reverse": list(range(n, 0, -1)), "rank_correlated": list(range(n))}.get(shape)
        if keyvals is not None:
            v["i64"] = keyvals
        bounds = [(0, n), (n, n), (n, n)] if shape == "one_rank_holds_all" else shard_bounds(n, world, 5) if n > 2 else [(0, 1), (1, 1), (1, 2)]
        if shape == "rank_correlated":  # rank r holds the r-th third of the key range
            bounds = [(n * r // world, n * (r + 1) // world) for r in range(world)]
        tabs = [stage(c, f"s{r}", {k: x[lo:hi] for k, x in v.items()}, "host", r) if hi > lo else empty(c, f"s{r}")
                for r, (c, (lo, hi)) in enumerate(zip(ctxs, bounds))]
        sources = [rows_of(v, lo, hi) for lo, hi in bounds]
        for keys in ([("i64", False)], [("i64", True)], [("i64", False), ("k", True)]):
            for limit in (None, 3):
                got = sort_x(comms, tabs, keys, columns=["i64", "s", "k"], limit=limit)
                check_slices(got, model(sources, keys, limit), ["i64", "s", "k"], limit, (shape, keys, limit))
                for t, _, _ in got:
                    t.destroy()


# ---------------------------------------------------------------------------------------------------- 3. a compressed multi-batch shard
@pytest.mark.gpu
def test_compressed_multi_batch_shards_and_the_limit_path():
    from test_gpu_table_exchange import WIDE_COLUMNS, gather_np, stage_wide, wide_values
    world = 2
    rng = np.random.default_rng(3)
    with ranks(world, user_bytes=64 << 20) as (ctxs, comms):
        parts = [[wide_values(rng, 70_000), wide_values(rng, 1_000)], [wide_values(rng, 5_000), wide_values(rng, 66_000)]]
        tabs = [stage_wide(ctxs[0], "a", parts[0], "host"), stage_wide(ctxs[1], "b", parts[1], "sliced")]

        def column(p, c):
            cells, valid = p[c]
            w = cells.shape[1]
            vals = [int.from_bytes(bytes(x), "little", signed=True) for x in cells] if w == 16 else cells.view({8: np.int64, 4: np.int32, 1: np.int8}[w]).reshape(-1).tolist()
            return [x if ok else None for x, ok in zip(vals, valid.tolist())]
        sources = []
        for ps in parts:
            rows = []
            for p in ps:
                cols = {c: column(p, c) for c, *_ in WIDE_COLUMNS if c in ("i64", "dn", "dw", "dt")}
                rows += [{c: cols[c][i] for c in cols} for i in range(len(cols["i64"]))]
            sources.append(rows)
        keys = [("dn", True), ("dt", False), ("dw", False)]
        for limit in (None, 1000):
            got = sort_x(comms, tabs, keys, columns=["i64", "dw"], limit=limit)
            want = model(sources, keys, limit)
            at = 0
            for d, (t, first, total) in enumerate(got):
                assert first == at and total == len(want)
                cells, valid = gather_np(t, "i64", 8)
                vals = [x if ok else None for x, ok in zip(cells.view(np.int64).reshape(-1).tolist(), valid.tolist())]
                assert vals == [w["i64"] for w in want[at:at + t.num_rows]], (limit, d)
                at += t.num_rows
            assert at == len(want)
            for t, _, _ in got:
                t.destroy()


# ---------------------------------------------------------------------------------------------------- 4. balance
# S = 1024 samples per rank: a rank's range holds about S * world / world = S samples' worth of rows, with a relative spread of about
# 1 / sqrt(S) ~ 3 %; DESIGN §6 states the bound 1.25 x the mean (eight spreads) that this checks.
BALANCE_BOUND = 1.25


def balance_case(world: int, n: int, kind: str):
    import torch

    from lingodb_b200 import runtime
    rng = np.random.default_rng(17)
    with ranks(world, user_bytes=256 << 20) as (ctxs, comms):
        keys_np, tabs = [], []
        for r, c in enumerate(ctxs):
            if kind == "uniform":
                k = rng.integers(-(1 << 62), 1 << 62, n, dtype=np.int64)
            elif kind == "zipf":
                k = rng.zipf(1.3, n).astype(np.int64)
            elif kind == "all_equal":
                k = np.full(n, 7, np.int64)
            else:  # sorted over the ranks
                k = np.arange(r * n, (r + 1) * n, dtype=np.int64)
            keys_np.append(k)
            row = np.arange(n, dtype=np.int64) + r * n  # the global row: what breaks ties
            tab = runtime.Table(c, f"b{r}", R.specs_of([("key", "int64", 0, 0), ("row", "int64", 0, 0)]))
            tab.append_device({"key": torch.from_numpy(k).cuda(), "row": torch.from_numpy(row).cuda()}, n)
            tabs.append(tab)
        torch.cuda.synchronize()
        got = sort_x(comms, tabs, [("key", False)])
        counts = [t.num_rows for t, _, _ in got]
        assert sum(counts) == world * n
        assert max(counts) <= BALANCE_BOUND * world * n / world, (kind, counts)
        from test_gpu_table_exchange import gather_np
        k_all = np.concatenate(keys_np)
        order = np.lexsort((np.arange(world * n), k_all))
        key_out = np.concatenate([gather_np(t, "key", 8)[0].view(np.int64).reshape(-1) for t, _, _ in got])
        row_out = np.concatenate([gather_np(t, "row", 8)[0].view(np.int64).reshape(-1) for t, _, _ in got])
        assert np.array_equal(row_out, order) and np.array_equal(key_out, k_all[order]), kind
        for t, _, _ in got:
            t.destroy()
        return counts


@pytest.mark.gpu
def test_balance_over_eight_ranks_at_a_million_rows_each():
    assert run_isolated(["balance"], {"CUDA_DEVICE_MAX_CONNECTIONS": "32"}) == 0


# ---------------------------------------------------------------------------------------------------- 5. LIMIT needs world * limit rows
def a16(x: int) -> int:
    return (x + 15) // 16 * 16


@pytest.mark.gpu
def test_limit_succeeds_with_a_region_for_world_times_limit_rows():
    import torch

    from lingodb_b200 import runtime
    world, n, limit = 3, 100 * 50, 50
    need = a16(world * limit * 8) * 2 + a16(world * limit) * 2  # two int64 columns, their validity bytes
    rng = np.random.default_rng(5)
    with ranks(world, user_bytes=1 << 20) as (ctxs, comms):
        tabs, ks = [], []
        for r, c in enumerate(ctxs):
            k = rng.integers(0, 40, n, dtype=np.int64)  # runs of ties cut by the limit
            ks.append(k)
            tab = runtime.Table(c, f"l{r}", R.specs_of([("key", "int64", 0, 0), ("row", "int64", 0, 0)]))
            tab.append_device({"key": torch.from_numpy(k).cuda(), "row": torch.from_numpy(np.arange(n, dtype=np.int64) + r * n).cuda()}, n)
            tabs.append(tab)
        torch.cuda.synchronize()
        res, errs = on_ranks(comms, lambda r: comms[r].sort_exchange(tabs[r], [("key", True)], limit=limit, recv_bytes=need - 16))
        assert all(e is not None and e.code == capi.LDB_ERR_CAPACITY and f"retry with recv_bytes {need}" in str(e) for e in errs), [str(e) for e in errs]
        got = sort_x(comms, tabs, [("key", True)], limit=limit, recv_bytes=need)
        from test_gpu_table_exchange import gather_np
        k_all = np.concatenate(ks)
        order = np.lexsort((np.arange(world * n), -k_all))[:limit]
        assert [t.num_rows for t, _, _ in got] == [limit, 0, 0]
        assert gather_np(got[0][0], "row", 8)[0].view(np.int64).reshape(-1).tolist() == order.tolist()
        assert [(f, tot) for _, f, tot in got] == [(0, limit), (limit, limit), (limit, limit)]


# ---------------------------------------------------------------------------------------------------- 6. capacity
@pytest.mark.gpu
def test_capacity_fails_on_every_rank_writes_nothing_and_the_named_size_succeeds():
    from test_gpu_exchange import SENTINEL, heap_fill, heap_read
    world, n = 2, 700
    v = gen(11, n, big=0)
    with ranks(world, user_bytes=4 << 20) as (ctxs, comms):
        tabs = [stage(c, f"c{r}", {k: x[r * n // 2:(r + 1) * n // 2] for k, x in v.items()}, "host", r) for r, c in enumerate(ctxs)]
        for cm in comms:
            heap_fill(cm, 0, 4 << 20)
        res, errs = on_ranks(comms, lambda r: comms[r].sort_exchange(tabs[r], [("i64", False)], columns=["s", "dw"], recv_bytes=256))
        assert all(e is not None and e.code == capi.LDB_ERR_CAPACITY for e in errs), [str(e) for e in errs]
        msgs = {str(e) for e in errs}
        assert len(msgs) == 1, msgs
        need = int(msgs.pop().rsplit("retry with recv_bytes ", 1)[1].split()[0].rstrip(")"))
        for cm in comms:
            assert heap_read(cm, 0, 4 << 20) == SENTINEL.to_bytes(4, "little") * ((4 << 20) // 4)
        got = sort_x(comms, tabs, [("i64", False)], columns=["s", "dw"], recv_bytes=need)
        check_slices(got, model([rows_of(v, 0, n // 2), rows_of(v, n // 2, n)], [("i64", False)]), ["s", "dw"], None)


# ---------------------------------------------------------------------------------------------------- 7. errors
@pytest.mark.gpu
def test_documented_errors():
    with ranks(2, user_bytes=1 << 20) as (ctxs, comms):
        c, cm = ctxs[0], comms[0]
        v = R.gen_values(3, 40, COLUMNS)
        t = c.table_from_host(R.to_table_data("t", v, COLUMNS))
        other = ctxs[1].table_from_host(R.to_table_data("o", v, COLUMNS))
        L, user = c.L, cm.heap()[1]

        def call(table=t, keys=("i64",), columns=("i32",), comm=cm, off=0, nbytes=4096, n_keys=None, limit=-1):
            kn = [k.encode() for k in keys]
            karr = (C.c_char_p * max(1, len(kn)))(*kn)
            darr = (C.c_int32 * max(1, len(kn)))()
            carr = None
            if columns is not None:
                carr = (C.c_char_p * max(1, len(columns)))(*[x.encode() for x in columns])
            res, first, total, e = C.c_void_p(), C.c_int64(), C.c_int64(), capi.Error()
            rc = L.ldb_gpu_table_sort_exchange(table.h if table is not None else None, len(kn) if n_keys is None else n_keys, karr, darr,
                                               len(columns) if columns is not None else 0, carr, limit, comm.h if comm is not None else None, off, nbytes,
                                               b"x", C.byref(res), C.byref(first), C.byref(total), C.byref(e))
            return rc, e.message.decode()
        INVALID, UNSUP = capi.LDB_ERR_INVALID, capi.LDB_ERR_UNSUPPORTED
        cases = [
            (dict(table=None), INVALID, "null argument"),
            (dict(comm=None), INVALID, "null argument"),
            (dict(keys=(), n_keys=0), INVALID, "1..4 key columns"),
            (dict(keys=("i64",) * 5), INVALID, "1..4 key columns"),
            (dict(keys=("nope",)), INVALID, "unknown key column"),
            (dict(columns=("i32", "nope")), INVALID, "unknown column"),
            (dict(table=other), INVALID, "different contexts"),
            (dict(off=8), INVALID, "16-byte aligned"),
            (dict(nbytes=user + 16), INVALID, "outside"),
            (dict(keys=("s",)), UNSUP, "column s"),
            (dict(keys=("f8",)), UNSUP, "column f8"),
            (dict(keys=("i64", "f4")), UNSUP, "column f4"),
            (dict(keys=("i8",)), UNSUP, "column i8"),
            (dict(keys=("i16",), limit=3), UNSUP, "column i16"),
        ]
        for kw, code, msg in cases:
            rc, m = call(**kw)
            assert rc == code and msg in m, (kw, rc, m)
        c.graph_begin()
        rc, m = call()
        c.graph_end().destroy()
        assert rc == UNSUP and "captured" in m, m
        # none of the refused calls started a collective: both ranks still sort in step
        tabs = [t, ctxs[1].table_from_host(R.to_table_data("u", v, COLUMNS))]
        got = sort_x(comms, tabs, [("i64", False)], columns=["i32"])
        assert sum(x.num_rows for x, _, _ in got) == 80


@pytest.mark.skipif(os.path.exists("/dev/nvidiactl"), reason="a GPU is present")
def test_no_device_from_the_entry_point():
    L = capi.lib()
    out, first, total, e = C.c_void_p(), C.c_int64(), C.c_int64(), capi.Error()
    rc = L.ldb_gpu_table_sort_exchange(None, 1, None, None, 0, None, -1, None, 0, 0, None, C.byref(out), C.byref(first), C.byref(total), C.byref(e))
    assert rc == capi.LDB_ERR_NO_DEVICE and b"no CPU fallback" in e.message and not out.value


# ---------------------------------------------------------------------------------------------------- 8. TPC-H at SF1
@pytest.fixture(scope="module")
def sf1():
    from lingodb_b200 import dbgen
    return dbgen.tpch(1.0, chunk_rows=1 << 16, extended=True, attributes=True)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_distributed_tpch_q16_q18_q3_q10_end_with_the_sort_exchange(sf1, world):
    """Q16, Q18, Q3 and Q10 as test_gpu_dict_unify.py, test_gpu_table_exchange.py and test_gpu_table_exchange_strings.py run them, with
    the final ORDER BY on the device (Q16: all 18 314 rows by count DESC, brand code, type code, size; Q18: LIMIT 100 by o_totalprice
    DESC, o_orderdate; Q3: LIMIT 10 by revenue DESC, o_orderdate; Q10: LIMIT 20 by revenue DESC): the host only reads the ranks' tables
    in rank order."""
    import datetime
    import hashlib

    from lingodb_b200 import dbgen, program as P, runtime
    from lingodb_b200.datagen import ColumnSpec
    from test_gpu_dict_unify import destroy, dict_strings, drop, unified_column
    from test_gpu_table_exchange import _deal, exchange
    from test_gpu_table_exchange_strings import xchg
    from test_reference_answers_sf1 import GOLD, day, dec
    col, const = (lambda n: ("col", n)), (lambda v: ("const", v))

    def read_in_rank_order(got, columns, width):
        rows = []
        for t, first, total in got:
            assert first == len(rows)
            ids = list(range(t.num_rows))
            rows += list(zip(*[t.gather(c, ids, cell_bytes=width[c]) for c in columns])) if ids else []
        assert all(total == len(rows) for _, _, total in got)
        return rows
    with ranks(world, user_bytes=512 << 20) as (ctxs, comms):
        mat = lambda r, t, outs, where=None: P.RawTable(ctxs[r], P.materialize(ctxs[r], t, outs, where=where))
        # ---- Q16 (its pipeline as in test_gpu_dict_unify.py), ordered across ranks over the exported groups
        pas = [c.table_from_host(_deal(sf1["part"], world, r, 0)) for r, c in enumerate(ctxs)]
        pss = [c.table_from_host(_deal(sf1["partsupp"], world, r, 1)) for r, c in enumerate(ctxs)]
        brands = unified_column(ctxs, comms, pas, "p_brand", 64)
        types = unified_column(ctxs, comms, pas, "p_type", 256)
        bad = dbgen.complaint_suppliers(1.0)
        sizes = ("cmp", "=", col("p_size"), const(49))
        for s_ in (14, 23, 45, 19, 3, 36, 9):
            sizes = ("or", sizes, ("cmp", "=", col("p_size"), const(s_)))
        pm, sm = [], []
        for r, c in enumerate(ctxs):
            pwhere = ("and", ("and", ("strcmp", "!=", "p_brand", "Brand#45"), ("not", ("like", "prefix", "p_type", "MEDIUM POLISHED"))), sizes)
            pm.append(mat(r, pas[r], [col("p_partkey"), ("strcode", brands[r], "p_brand", "lookup"), ("strcode", types[r], "p_type", "lookup"), col("p_size")], pwhere))
            ct = runtime.Table(c, "complaints", [ColumnSpec("s_suppkey", "int32")])
            ct.append_host({"s_suppkey": bad}, len(bad))
            cj = runtime.join_table(c, 1024)
            P.build_join(c, ct, cj, col("s_suppkey"))
            sm.append(mat(r, pss[r], [col("ps_partkey"), col("ps_suppkey")], ("isnull", ("probe", cj, col("ps_suppkey")))))
            c.L.ldb_gpu_state_destroy(cj)
            ct.clear()
        px, sx = exchange(comms, pm, ["c0"]), exchange(comms, sm, ["c0"])
        l1, o1 = [], []
        for r, c in enumerate(ctxs):
            pj = runtime.join_table(c, 210_000, unique=True)
            P.build_join(c, px[r], pj, col("c0"), payload=("rowid",))
            prow = ("probe", pj, col("c0"))
            f = lambda x: ("fetch", px[r], prow, x)
            l1.append(P.group_by(c, sx[r], [f("c1"), f("c2"), f("c3"), col("c1")], [("count_star", None)], where=("not", ("isnull", prow)), expected_groups=1 << 18))
            o1.append(P.hashagg_state(c, 4, ["count_star"], 1 << 18))
            c.L.ldb_gpu_state_destroy(pj)
        all_ok(comms, lambda r: comms[r].hashagg_exchange(l1[r], o1[r]))
        g1 = [P.groups_table(c, s) for c, s in zip(ctxs, o1)]
        l2 = [P.group_by(c, g, [col("k0"), col("k1"), col("k2")], [("count_star", None)], expected_groups=1 << 15) for c, g in zip(ctxs, g1)]
        o2 = [P.hashagg_state(c, 3, ["count_star"], 1 << 15) for c in ctxs]
        all_ok(comms, lambda r: comms[r].hashagg_exchange(l2[r], o2[r]))
        g2 = [P.groups_table(c, s) for c, s in zip(ctxs, o2)]
        got = sort_x(comms, g2, [("a0", True), ("k0", False), ("k1", False), ("k2", False)])
        assert sum(1 for t, _, _ in got if t.num_rows) > 1
        bstr, tstr = dict_strings(ctxs[-1], brands[-1])[0], dict_strings(ctxs[-1], types[-1])[0]
        rows = [[bstr[b].decode(), tstr[t].decode(), str(s_), str(n_)]
                for b, t, s_, n_ in read_in_rank_order(got, ["k0", "k1", "k2", "a0"], {"k0": 8, "k1": 8, "k2": 8, "a0": 16})]
        want = GOLD["q16"]
        assert len(rows) == want["rows"] and rows[:3] == want["first"] and rows[-3:] == want["last"]
        assert hashlib.sha256("\n".join("\t".join(x) for x in rows).encode()).hexdigest() == want["sha256"]
        drop(pm + sm + px + sx + g1 + g2 + pas + pss + [t for t, _, _ in got])
        for x in (l1, o1, l2, o2, brands, types):
            destroy(ctxs, x)
        # ---- Q18 (its pipeline as in test_gpu_table_exchange_strings.py), LIMIT 100 on rank 0; c_name is broadcast, so its row ids
        # mean the same row on every rank
        lis = [c.table_from_host(_deal(sf1["lineitem"], world, r, 0)) for r, c in enumerate(ctxs)]
        ods = [c.table_from_host(_deal(sf1["orders"], world, r, 1)) for r, c in enumerate(ctxs)]
        cus = [c.table_from_host(_deal(sf1["customer"], world, r, 2)) for r, c in enumerate(ctxs)]
        locals_ = [P.group_by(c, t, [col("l_orderkey")], [("sum", col("l_quantity"))], expected_groups=1_600_000) for c, t in zip(ctxs, lis)]
        owneds = [P.hashagg_state(c, 1, ["sum"], 1_600_000) for c in ctxs]
        all_ok(comms, lambda r: comms[r].hashagg_exchange(locals_[r], owneds[r]))
        ox = xchg(comms, ods, ["o_orderkey"], columns=["o_custkey", "o_orderkey", "o_orderdate", "o_totalprice"])
        bx = xchg(comms, cus, [], columns=["c_custkey", "c_name", "c_nationkey"])  # every customer on every rank, in one order
        mts = []
        for r, c in enumerate(ctxs):
            groups = P.groups_table(c, owneds[r])
            big = runtime.join_table(c, 4096, unique=True)
            P.build_join(c, groups, big, col("k0"), payload=col("a0"), where=("cmp", ">", col("a0"), const(30000)))
            cj = runtime.join_table(c, 200_000, unique=True)
            P.build_join(c, bx[r], cj, col("c_custkey"), payload=("rowid",))
            pb = ("probe", big, col("o_orderkey"))
            mts.append(mat(r, ox[r], [("probe", cj, col("o_custkey")), col("o_custkey"), col("o_orderkey"), col("o_orderdate"), col("o_totalprice"), pb],
                           ("not", ("isnull", pb))))
            groups.destroy()
            c.L.ldb_gpu_state_destroy(big)
            c.L.ldb_gpu_state_destroy(cj)
        got = sort_x(comms, mts, [("c4", True), ("c3", False)], limit=100)
        assert [t.num_rows for t, _, _ in got] == [min(100, sum(t.num_rows for t in mts))] + [0] * (world - 1)
        part = read_in_rank_order(got, [f"c{i}" for i in range(6)], {f"c{i}": 16 for i in range(6)})
        names = bx[0].gather_strings("c_name", [x[0] for x in part])
        got18 = [[n_, str(x[1]), str(x[2]), day(x[3]), dec(x[4], 2), dec(x[5], 2)] for n_, x in zip(names, part)]
        assert got18 == GOLD["q18_rows"]
        drop(ox + mts + [t for t, _, _ in got])
        destroy(ctxs, locals_)
        destroy(ctxs, owneds)
        # ---- Q3 (its pipeline as in test_gpu_table_exchange.py), LIMIT 10 by revenue DESC, o_orderdate over the exported groups
        d = lambda s_: (datetime.date.fromisoformat(s_) - datetime.date(1970, 1, 1)).days
        cut = d("1995-03-15")
        cm_ = [mat(r, cus[r], [col("c_custkey")], ("strcmp", "=", "c_mktsegment", "BUILDING")) for r in range(world)]
        cx = exchange(comms, cm_, [])
        om, lm = [], []
        for r, c in enumerate(ctxs):
            cj = runtime.join_table(c, 400_000, unique=True)
            P.build_join(c, cx[r], cj, col("c0"))
            pc = ("probe", cj, col("o_custkey"))
            om.append(mat(r, ods[r], [col("o_orderkey"), ("add", ("mul", col("o_orderdate"), const(16)), col("o_shippriority"))],
                          ("and", ("cmp", "<", col("o_orderdate"), const(cut)), ("not", ("isnull", pc)))))
            lm.append(mat(r, lis[r], [col("l_orderkey"), ("mul", col("l_extendedprice"), ("sub", const(100), col("l_discount")))],
                          ("cmp", ">", col("l_shipdate"), const(cut))))
            c.L.ldb_gpu_state_destroy(cj)
        ox, lx = exchange(comms, om, ["c0"]), exchange(comms, lm, ["c0"])
        gs, sts = [], []
        for r, c in enumerate(ctxs):
            oj = runtime.join_table(c, 1_000_000, unique=True)
            P.build_join(c, ox[r], oj, col("c0"), payload=col("c1"))
            po = ("probe", oj, col("c0"))
            sts.append(P.group_by(c, lx[r], [col("c0"), po], [("sum", col("c1"))], where=("not", ("isnull", po)), expected_groups=200_000))
            gs.append(P.groups_table(c, sts[-1]))
            c.L.ldb_gpu_state_destroy(oj)
        got = sort_x(comms, gs, [("a0", True), ("k1", False)], limit=10)
        rows = read_in_rank_order(got, ["k0", "k1", "a0"], {"k0": 8, "k1": 8, "a0": 16})
        assert [[str(k), dec(rev, 4), day(p // 16), str(p % 16)] for k, p, rev in rows] == GOLD["q3_rows"]
        drop(cm_ + cx + om + lm + ox + lx + gs + [t for t, _, _ in got])
        destroy(ctxs, sts)
        # ---- Q10 (its pipeline as in test_gpu_table_exchange_strings.py), LIMIT 20 by revenue DESC; the customers and nations are
        # broadcast, so the row ids of c_name and n_name mean the same rows on every rank and rank 0 reads them
        revenue = ("mul", col("l_extendedprice"), ("sub", const(100), col("l_discount")))
        nat = [c.table_from_host(sf1["nation"]) if r == world - 1 else runtime.Table(c, "nation", sf1["nation"].columns) for r, c in enumerate(ctxs)]
        om = [mat(r, ods[r], [col("o_orderkey"), col("o_custkey")], ("and", ("cmp", ">=", col("o_orderdate"), const(d("1993-10-01"))),
                                                                         ("cmp", "<", col("o_orderdate"), const(d("1994-01-01"))))) for r in range(world)]
        lm = [mat(r, lis[r], [col("l_orderkey"), revenue], ("cmp", "=", col("l_returnflag"), const(ord("R")))) for r in range(world)]
        ox, lx = xchg(comms, om, ["c0"]), xchg(comms, lm, ["c0"])
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
        mts = []
        for r, c in enumerate(ctxs):
            g = P.groups_table(c, owneds[r])
            cj, nj = runtime.join_table(c, 200_000, unique=True), runtime.join_table(c, 64, unique=True)
            P.build_join(c, bx[r], cj, col("c_custkey"), payload=("rowid",))
            P.build_join(c, nx[r], nj, col("n_nationkey"), payload=("rowid",))
            crow = ("probe", cj, col("k0"))
            mts.append(mat(r, g, [col("k0"), col("a0"), crow, ("probe", nj, ("fetch", bx[r], crow, "c_nationkey"))]))
            for x in (cj, nj):
                c.L.ldb_gpu_state_destroy(x)
            g.destroy()
        got = sort_x(comms, mts, [("c1", True)], limit=20)
        part = read_in_rank_order(got, [f"c{i}" for i in range(4)], {f"c{i}": 16 for i in range(4)})
        cname = bx[0].gather_strings("c_name", [x[2] for x in part])
        nname = nx[0].gather_strings("n_name", [x[3] for x in part])
        assert [[str(k), cn_, dec(rev, 4), nn] for (k, rev, _, _), cn_, nn in zip(part, cname, nname)] == [[g[0], g[1], g[2], g[4]] for g in GOLD["q10_rows"]]
        drop(om + lm + ox + lx + nx + nat + mts + bx + lis + ods + cus + [t for t, _, _ in got])
        destroy(ctxs, locals_)
        destroy(ctxs, owneds)


def run_isolated(args: list, env: dict, timeout: int = 900):
    """this file run as `python test_gpu_sort_exchange.py *args` with `env` added; the child is killed and reaped whatever ends the call"""
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([root, here] + [x for x in os.environ.get("PYTHONPATH", "").split(os.pathsep) if x]), **env)
    p = subprocess.Popen([sys.executable, os.path.abspath(__file__)] + args, env=env)
    try:
        return p.wait(timeout=timeout)
    finally:
        if p.poll() is None:
            p.kill()
        p.wait()


if __name__ == "__main__":
    if sys.argv[1] == "model":
        check_model(int(sys.argv[2]))
    elif sys.argv[1] == "balance":
        for kind in ("uniform", "zipf", "all_equal", "sorted"):
            print(kind, balance_case(8, 1 << 20, kind), flush=True)
