"""Unified string dictionaries across ranks (ldb_gpu_dict_unify, parallel.Comm.dict_unify), checked against plain Python: every rank ends
up with the sorted union of all ranks' strings, the code of a string is its position in Python's bytes order (the bytewise, unsigned,
prefix-first order of LDB_OP_STRCMP), and those codes work as ordinary int32 keys in the hash-aggregation and table exchanges."""
import ctypes as C
import hashlib
import os
import random
import re

import numpy as np
import pytest

from lingodb_b200 import capi, dbgen, program as P, runtime
from lingodb_b200.datagen import ColumnSpec
from test_gpu_exchange import SENTINEL, heap_fill, heap_read
from test_gpu_strings import codes_of, make_table, utf8
from test_gpu_table_exchange import _deal, _union_groups, all_ok, exchange, on_ranks, ranks

col, const = (lambda n: ("col", n)), (lambda v: ("const", v))

EDGE = [b"", b"ab", b"abc", b"a", b"ab\0", b"\0", b"\0\0", b"\x80", b"\xff", b"\xff\xff\xfe", b"a\x80", b"x" * 300, b"x" * 299 + b"y",
        b"PREFIX08", b"PREFIX08PREFIX16", b"PREFIX08PREFIX16" + b"z" * 20, b"P" * 33]


def rand_string(rng) -> bytes:
    n = rng.choice([0, 1, 2, 3, 7, 8, 9, 15, 16, 17, 31, 32, 33, 64, 100, 255, 300, rng.randrange(301)])
    alphabet = rng.choice([b"ab", b"abc\0", bytes(range(256)), b"\x7f\x80\xff"])
    return bytes(rng.choice(alphabet) for _ in range(n))


def shared_pool(seed: int, n: int) -> list:
    rng = random.Random(seed)
    return EDGE + [rand_string(rng) for _ in range(n)]


def local_dict(ctx, values: list, name="loc"):
    """a dictionary of ctx holding the distinct non-NULL `values`, filled through an inserting STRCODE"""
    distinct = {v for v in values if v is not None}
    d = P.dict_state(ctx, max(len(distinct), 1), max(sum(map(len, distinct)), 1))
    if values:
        t = make_table(ctx, name, {"s": ("utf8", values)})
        P.run_effects(ctx, t, [("strcode", d, "s")])
        t.clear()
    return d


def dict_strings(ctx, d) -> list:
    """the strings of dictionary d in code order, and its rank column"""
    t = P.dict_table(ctx, d)
    ids = list(range(t.num_rows))
    out = (t.gather_strings("str", ids, decode=False), t.gather("rank", ids, cell_bytes=4))
    t.destroy()
    return out


def unify(comms, locals_, **kw):
    return all_ok(comms, lambda r: comms[r].dict_unify(locals_[r], **kw))


def drop(tables):
    """frees result tables (program.RawTable) and clears staged ones (runtime.Table)"""
    for t in tables:
        t.destroy() if isinstance(t, P.RawTable) else t.clear()


def destroy(ctxs, states):
    for c, s in zip(ctxs, states):
        c.L.ldb_gpu_state_destroy(s)


def shards_of(world: int, seed: int, n: int = 300) -> list:
    """per rank: a list of strings, overlapping across ranks; with more than one rank, rank 1 holds none"""
    pool = shared_pool(seed, n)
    rng = random.Random(seed + 1)
    out = []
    for r in range(world):
        own = [rand_string(rng) + b"#%d" % r for _ in range(rng.randrange(20, 80))]
        mine = [v for v in pool if rng.random() < 0.5] + own
        rng.shuffle(mine)
        out.append([] if world > 1 and r == 1 else mine + mine[:10])  # duplicates too
    return out


# ---------------------------------------------------------------------------------------------------- 1. exact against the model
def run_isolated(args: list, env: dict, timeout: int = 600):
    """this file run as `python test_gpu_dict_unify.py *args` with `env` added; the child is killed and reaped whatever ends the call"""
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


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_union_is_the_sorted_set_on_every_rank(world):
    if world == 8:
        # Eight ranks in one process on one GPU: with the default 8 hardware work queues their streams share queues, and a collective
        # kernel can then wait behind a peer's kernel that waits for it.  The case runs in a child process with 32 queues.
        assert run_isolated(["model", str(world)], {"CUDA_DEVICE_MAX_CONNECTIONS": "32"}) == 0
        return
    check_union(world)


def check_union(world: int):
    shards = shards_of(world, 10 + world)
    want = sorted(set(v for s in shards for v in s))
    with ranks(world, user_bytes=4 << 20) as (ctxs, comms):
        locs = [local_dict(c, s) for c, s in zip(ctxs, shards)]
        before = [dict_strings(c, d) for c, d in zip(ctxs, locs)]
        us = unify(comms, locs)
        for r, (c, u) in enumerate(zip(ctxs, us)):
            strs, rank = dict_strings(c, u)
            assert strs == want, r
            assert rank == list(range(len(want))), r
            assert P.dict_count(c, u) == len(want)
        assert [dict_strings(c, d) for c, d in zip(ctxs, locs)] == before  # the local dictionaries are only read
        destroy(ctxs, us)
        destroy(ctxs, locs)


# ---------------------------------------------------------------------------------------------------- 2. lookups on every kind of shard
def device_table(ctx, name, values: list):
    """one borrowed DEVICE batch, an Arrow slice 5 rows into its buffers (bitmap read from bit 5)"""
    import torch
    offs, data, valid = utf8([b"pad"] * 5 + values)
    t = runtime.Table(ctx, name, [ColumnSpec("s", "utf8")])
    t.append_device({"s": (torch.from_numpy(offs).cuda(), torch.from_numpy(data).cuda()), "s$valid": torch.from_numpy(valid).cuda()}, len(values), offset=5)
    torch.cuda.synchronize()
    return t


@pytest.mark.gpu
def test_lookups_give_the_index_in_the_sorted_union():
    world = 3
    shards = shards_of(world, 77)
    union = sorted(set(v for s in shards for v in s))
    code = {v: i for i, v in enumerate(union)}
    rng = random.Random(5)
    with ranks(world, user_bytes=4 << 20) as (ctxs, comms):
        locs = [local_dict(c, s) for c, s in zip(ctxs, shards)]
        us = unify(comms, locs)
        for r, (c, u) in enumerate(zip(ctxs, us)):
            # every rank probes strings of every rank, strings in no dictionary, and NULLs
            vals = [rng.choice(union) for _ in range(400)] + [b"absent", b"ab\0\0", b"x" * 301, None, None]
            rng.shuffle(vals)
            want = [None if v is None or v not in code else code[v] for v in vals]
            tables = {"host": make_table(c, "h", {"s": ("utf8", vals)}, sizes=[7, 190, len(vals) - 197]),
                      "host_sliced": make_table(c, "hs", {"s": ("utf8", vals)}, sizes=[100, len(vals) - 100], offset=3),
                      "device": device_table(c, "d", vals)}
            for how, t in tables.items():
                assert codes_of(c, t, ("strcode", u, "s", "lookup")) == want, (r, how)
            with pytest.raises(capi.LdbRuntimeError) as e:  # an inserting STRCODE against a unified dictionary
                codes_of(c, tables["host"], ("strcode", u, "s"))
            assert e.value.code == capi.LDB_ERR_INVALID and "unified" in str(e.value)
            assert P.dict_count(c, u) == len(union)
            drop(tables.values())
        destroy(ctxs, us)
        destroy(ctxs, locs)


# ---------------------------------------------------------------------------------------------------- 3. string GROUP BY and join across ranks
@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_string_group_by_and_join_across_ranks(world):
    rng = random.Random(world)
    keys = sorted(set(shared_pool(99, 60)))
    rows = [[(rng.choice(keys) if rng.random() > 0.05 else None, rng.randrange(-1000, 1000)) for _ in range(rng.randrange(200, 600))] for _ in range(world)]
    dim = [[(k, i * 7 + 1) for i, k in enumerate(keys) if i % world == r and i % 5] for r in range(world)]  # join build side, unique keys
    with ranks(world, user_bytes=16 << 20) as (ctxs, comms):
        facts = [make_table(c, f"f{r}", {"s": ("utf8", [s for s, _ in rows[r]]), "v": ("int64", [v for _, v in rows[r]])}) for r, c in enumerate(ctxs)]
        dims = [make_table(c, f"d{r}", {"s": ("utf8", [s for s, _ in dim[r]]), "w": ("int64", [w for _, w in dim[r]])}) for r, c in enumerate(ctxs)]
        locs = [local_dict(c, [s for s, _ in rows[r]] + [s for s, _ in dim[r]]) for r, c in enumerate(ctxs)]
        us = unify(comms, locs)
        union = dict_strings(ctxs[0], us[0])[0]
        # GROUP BY s: count(*), sum(v) by unified code, merged on the owner ranks
        key = lambda r: ("strcode", us[r], "s", "lookup")
        loc = [P.group_by(c, facts[r], [key(r)], [("count_star", None), ("sum", col("v"))], expected_groups=256) for r, c in enumerate(ctxs)]
        own = [P.hashagg_state(c, 1, ["count_star", "sum"], 256) for c in ctxs]
        all_ok(comms, lambda r: comms[r].hashagg_exchange(loc[r], own[r]))
        got = _union_groups(ctxs, own, 1, 2)
        want = {}
        for s, v in (x for rr in rows for x in rr):
            g = want.setdefault(s, [0, 0])
            g[0] += 1
            g[1] += v
        assert {(None if k[0] is None else union[k[0]]): list(a) for k, a in got.items()} == want
        coded = sorted(k[0] for k in got if k[0] is not None)
        assert [union[c] for c in coded] == sorted(k for k in want if k is not None)  # order by code = order by string
        # JOIN facts ⋈ dims ON s: both sides exchanged on the materialized code column, built and probed locally
        fm = [P.RawTable(c, P.materialize(c, facts[r], [key(r), col("v")], where=("not", ("isnull", key(r))))) for r, c in enumerate(ctxs)]
        dm = [P.RawTable(c, P.materialize(c, dims[r], [key(r), col("w")])) for r, c in enumerate(ctxs)]
        fx, dx = exchange(comms, fm, ["c0"]), exchange(comms, dm, ["c0"])
        joined = []
        for r, c in enumerate(ctxs):
            j = runtime.join_table(c, 4096, unique=True)
            P.build_join(c, dx[r], j, col("c0"), payload=col("c1"))
            pr = ("probe", j, col("c0"))
            mt = P.RawTable(c, P.materialize(c, fx[r], [col("c0"), col("c1"), pr], where=("not", ("isnull", pr))))
            ids = list(range(mt.num_rows))
            joined += [(union[k], v, w) for k, v, w in zip(*(mt.gather(x, ids) for x in ("c0", "c1", "c2")))]
            mt.destroy()
            c.L.ldb_gpu_state_destroy(j)
        wmap = {s: w for d in dim for s, w in d}
        assert sorted(joined) == sorted((s, v, wmap[s]) for rr in rows for s, v in rr if s is not None and s in wmap)
        drop(facts + dims + fm + dm + fx + dx)
        for x in (loc, own, us, locs):
            destroy(ctxs, x)


# ---------------------------------------------------------------------------------------------------- 4. scale
def random_strings(seed: int, n: int, max_len: int) -> list:
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, max_len + 1, n)
    raw = rng.integers(0, 256, int(lens.sum()), dtype=np.uint8).tobytes()
    ends = np.cumsum(lens)
    return [raw[e - l:e] for l, e in zip(lens.tolist(), ends.tolist())]


@pytest.mark.gpu
def test_a_million_strings_per_rank():
    world, n = 2, 1_000_000
    shared = random_strings(1, n // 2, 120)
    shards = [shared + random_strings(2 + r, n // 2, 120) for r in range(world)]
    want = sorted(set(shared) | set(shards[0][n // 2:]) | set(shards[1][n // 2:]))
    with ranks(world, user_bytes=256 << 20) as (ctxs, comms):
        locs = [local_dict(c, s) for c, s in zip(ctxs, shards)]
        assert [P.dict_count(c, d) for c, d in zip(ctxs, locs)] == [len(set(s)) for s in shards]
        us = unify(comms, locs)
        digests = []
        for c, u in zip(ctxs, us):
            strs, rank = dict_strings(c, u)
            assert len(strs) == len(want) and rank[:5] == [0, 1, 2, 3, 4] and rank[-1] == len(want) - 1
            digests.append(hashlib.sha256(b"\n".join(strs)).hexdigest())
        assert digests == [hashlib.sha256(b"\n".join(want)).hexdigest()] * world
        destroy(ctxs, us)
        destroy(ctxs, locs)


# ---------------------------------------------------------------------------------------------------- 5. capacity and errors
def region_bytes(shards: list) -> int:
    a16 = lambda x: (x + 15) // 16 * 16
    return sum(a16((len(set(s)) + 1) * 4) + a16(sum(map(len, set(s)))) for s in shards)


@pytest.mark.gpu
def test_capacity_fails_on_every_rank_writes_nothing_and_the_named_size_succeeds():
    world, off = 3, 4096
    shards = shards_of(world, 31)
    need = region_bytes(shards)
    with ranks(world, user_bytes=4 << 20) as (ctxs, comms):
        locs = [local_dict(c, s) for c, s in zip(ctxs, shards)]
        span = need + 8192
        for cm in comms:
            heap_fill(cm, off - 1024, span)
        _, errs = on_ranks(comms, lambda r: comms[r].dict_unify(locs[r], recv_offset=off, recv_bytes=need - 16))
        assert all(e is not None and e.code == capi.LDB_ERR_CAPACITY for e in errs), errs
        assert {int(re.search(r"retry with recv_bytes (\d+)", str(e)).group(1)) for e in errs} == {need}
        for cm in comms:
            assert (np.frombuffer(heap_read(cm, off - 1024, span), dtype=np.uint32) == SENTINEL).all()
        us = unify(comms, locs, recv_offset=off, recv_bytes=need)
        want = sorted(set(v for s in shards for v in s))
        assert all(dict_strings(c, u)[0] == want for c, u in zip(ctxs, us))
        destroy(ctxs, us)
        destroy(ctxs, locs)


@pytest.mark.gpu
def test_documented_errors_and_back_to_back_unifies():
    world = 2
    shards = shards_of(world, 3)
    with ranks(world, user_bytes=1 << 20) as (ctxs, comms):
        c, cm = ctxs[0], comms[0]
        locs = [local_dict(x, s) for x, s in zip(ctxs, shards)]
        L, user = c.L, cm.heap()[1]
        other = locs[1]  # a dictionary of the other context
        hashagg = P.hashagg_state(c, 1, ["count_star"], 16)

        def call(local=locs[0], comm=cm, off=0, nbytes=1 << 16, out=True):
            res, e = C.c_void_p(), capi.Error()
            rc = L.ldb_gpu_dict_unify(local, comm.h if comm is not None else None, off, nbytes, C.byref(res) if out else None, C.byref(e))
            return rc, e.message.decode()
        INVALID, UNSUP = capi.LDB_ERR_INVALID, capi.LDB_ERR_UNSUPPORTED
        cases = [(dict(local=None), INVALID, "null argument"), (dict(comm=None), INVALID, "null argument"), (dict(out=False), INVALID, "null argument"),
                 (dict(local=hashagg), INVALID, "not a string dictionary"), (dict(local=other), INVALID, "different contexts"),
                 (dict(off=8), INVALID, "16-byte aligned"), (dict(off=-16), INVALID, "outside"), (dict(off=user - 64, nbytes=128), INVALID, "outside"),
                 (dict(nbytes=user + 16), INVALID, "outside"), (dict(nbytes=-1), INVALID, "outside")]
        for kw, code, msg in cases:
            rc, m = call(**kw)
            assert rc == code and msg in m, (kw, rc, m)
        c.graph_begin()
        rc, m = call()
        c.graph_end().destroy()
        assert rc == UNSUP and "captured" in m, m
        # none of the refused calls started a collective: the ranks still unify in step, twice over the same region
        want = sorted(set(v for s in shards for v in s))
        first = unify(comms, locs)
        second = unify(comms, first)  # a unified dictionary unifies to itself
        for x, a, b in zip(ctxs, first, second):
            assert dict_strings(x, a)[0] == want and dict_strings(x, b)[0] == want
        # a local dictionary that overflowed: every rank fails with LDB_ERR_CAPACITY naming its rank, and the ranks stay in step
        small = P.dict_state(ctxs[1], 8, 4)
        t = make_table(ctxs[1], "big", {"s": ("utf8", [b"longer than four bytes"])})
        with pytest.raises(capi.LdbRuntimeError):
            P.run_effects(ctxs[1], t, [("strcode", small, "s")])
        t.clear()
        bad = [locs[0], small]
        _, errs = on_ranks(comms, lambda r: comms[r].dict_unify(bad[r]))
        assert all(e is not None and e.code == capi.LDB_ERR_CAPACITY and "rank 1" in str(e) for e in errs), errs
        third = unify(comms, locs)
        assert all(dict_strings(x, u)[0] == want for x, u in zip(ctxs, third))
        c.L.ldb_gpu_state_destroy(hashagg)
        ctxs[1].L.ldb_gpu_state_destroy(small)
        for x in (first, second, third, locs):
            destroy(ctxs, x)


def test_entry_point_rejects_null_arguments_without_a_device():
    """Without a device no context, and so no dictionary and no comm, can exist: what reaches the entry point on such a machine is null
    handles, refused before any CUDA call."""
    L = capi.lib()
    assert capi.SIGNATURES["ldb_gpu_dict_unify"][0] is C.c_int
    out, e = C.c_void_p(), capi.Error()
    for args in ((None, None, 0, 0, C.byref(out)), (None, None, 0, 1 << 20, None)):
        assert L.ldb_gpu_dict_unify(*args, C.byref(e)) == capi.LDB_ERR_INVALID
        assert b"null argument" in e.message and not out.value
        assert L.ldb_gpu_dict_unify(*args, None) == capi.LDB_ERR_INVALID


# ---------------------------------------------------------------------------------------------------- 6. TPC-H at SF1 over dealt batches
@pytest.fixture(scope="module")
def sf1():
    return dbgen.tpch(1.0, chunk_rows=1 << 16, extended=True, attributes=True)


def unified_column(ctxs, comms, tables, column: str, expected: int):
    """every rank's local dictionary of `column` over its shard, unified"""
    locs = []
    for c, t in zip(ctxs, tables):
        d = P.dict_state(c, expected, expected * 32)
        P.run_effects(c, t, [("strcode", d, column)])
        locs.append(d)
    us = unify(comms, locs)
    destroy(ctxs, locs)
    return us


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_distributed_tpch_q16_q4_q18_with_string_keys(sf1, world):
    import datetime

    from test_reference_answers_sf1 import GOLD, day, dec
    d = lambda s: (datetime.date.fromisoformat(s) - datetime.date(1970, 1, 1)).days
    with ranks(world, user_bytes=512 << 20) as (ctxs, comms):
        mat = lambda r, t, outs, where=None: P.RawTable(ctxs[r], P.materialize(ctxs[r], t, outs, where=where))
        pas = [c.table_from_host(_deal(sf1["part"], world, r, 0)) for r, c in enumerate(ctxs)]
        pss = [c.table_from_host(_deal(sf1["partsupp"], world, r, 1)) for r, c in enumerate(ctxs)]
        assert sum(t.num_rows for t in pas) == sf1["part"].num_rows and min(t.num_rows for t in pas) > 0
        # ---- Q16: brand and type as unified codes; part rows and partsupp rows exchanged on partkey, count(distinct supplier) as the
        # (brand, type, size, supplier) groups merged on their owners, then counted per (brand, type, size) and merged again
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
        got = {}
        for c, s in zip(ctxs, o2):  # Q16 has more groups than _union_groups reads
            part = P.decode_groups(P.read_groups(c, s, 1 << 16), 3, 1)
            assert not set(part) & set(got)
            got.update(part)
        bstr, tstr = dict_strings(ctxs[-1], brands[-1])[0], dict_strings(ctxs[-1], types[-1])[0]
        order = sorted(got, key=lambda k: (-got[k][0], k[0], k[1], k[2]))  # codes order like the strings
        rows = [[bstr[b].decode(), tstr[t].decode(), str(s_), str(got[(b, t, s_)][0])] for b, t, s_ in order]
        want = GOLD["q16"]
        assert len(rows) == want["rows"] and rows[:3] == want["first"] and rows[-3:] == want["last"]
        assert hashlib.sha256("\n".join("\t".join(x) for x in rows).encode()).hexdigest() == want["sha256"]
        drop(pm + sm + px + sx + g1 + pas + pss)
        for x in (l1, o1, l2, o2, brands, types):
            destroy(ctxs, x)
        # ---- Q4: orders grouped by the unified code of o_orderpriority, EXISTS lineitem(l_commitdate < l_receiptdate)
        lis = [c.table_from_host(_deal(sf1["lineitem"], world, r, 0)) for r, c in enumerate(ctxs)]
        ods = [c.table_from_host(_deal(sf1["orders"], world, r, 1)) for r, c in enumerate(ctxs)]
        prio = unified_column(ctxs, comms, ods, "o_orderpriority", 8)
        owhere = ("and", ("cmp", ">=", col("o_orderdate"), const(d("1993-07-01"))), ("cmp", "<", col("o_orderdate"), const(d("1993-10-01"))))
        lm = [mat(r, lis[r], [col("l_orderkey")], ("cmp", "<", col("l_commitdate"), col("l_receiptdate"))) for r in range(world)]
        om = [mat(r, ods[r], [col("o_orderkey"), ("strcode", prio[r], "o_orderpriority", "lookup")], owhere) for r in range(world)]
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
        pstr = dict_strings(ctxs[0], prio[0])[0]
        assert [[pstr[k[0]].decode(), str(got[k][0])] for k in sorted(got)] == GOLD["q4_rows"]
        drop(lm + om + lx + ox)
        for x in (locals_, owneds, prio):
            destroy(ctxs, x)
        # ---- Q18: big orders from the lineitem sums merged on their owners; c_name read from the customer shards through a unified
        # dictionary: (custkey, name code) broadcast, joined to the result rows on every rank
        cus = [c.table_from_host(_deal(sf1["customer"], world, r, 2)) for r, c in enumerate(ctxs)]
        names = unified_column(ctxs, comms, cus, "c_name", 160_000)
        locals_ = [P.group_by(c, t, [col("l_orderkey")], [("sum", col("l_quantity"))], expected_groups=1_600_000) for c, t in zip(ctxs, lis)]
        owneds = [P.hashagg_state(c, 1, ["sum"], 1_600_000) for c in ctxs]
        all_ok(comms, lambda r: comms[r].hashagg_exchange(locals_[r], owneds[r]))
        ox = exchange(comms, ods, ["o_orderkey"], columns=["o_custkey", "o_orderkey", "o_orderdate", "o_totalprice"])
        cm_ = [mat(r, cus[r], [col("c_custkey"), ("strcode", names[r], "c_name", "lookup")]) for r in range(world)]
        cx = exchange(comms, cm_, [])
        rows = []
        for r, c in enumerate(ctxs):
            groups = P.groups_table(c, owneds[r])
            big = runtime.join_table(c, 4096, unique=True)
            P.build_join(c, groups, big, col("k0"), payload=col("a0"), where=("cmp", ">", col("a0"), const(30000)))
            cj = runtime.join_table(c, 200_000, unique=True)
            P.build_join(c, cx[r], cj, col("c0"), payload=col("c1"))
            pb = ("probe", big, col("o_orderkey"))
            mt = mat(r, ox[r], [("probe", cj, col("o_custkey")), col("o_custkey"), col("o_orderkey"), col("o_orderdate"), col("o_totalprice"), pb], ("not", ("isnull", pb)))
            ids = list(range(mt.num_rows))
            rows += list(zip(*[mt.gather(f"c{i}", ids) for i in range(6)]))
            for x in (mt, groups):
                x.destroy()
            c.L.ldb_gpu_state_destroy(big)
            c.L.ldb_gpu_state_destroy(cj)
        rows.sort(key=lambda x: (-x[4], x[3]))
        nt = P.dict_table(ctxs[0], names[0])
        nstr = nt.gather_strings("str", [x[0] for x in rows[:100]])
        nt.destroy()
        got18 = [[n, str(x[1]), str(x[2]), day(x[3]), dec(x[4], 2), dec(x[5], 2)] for n, x in zip(nstr, rows[:100])]
        assert got18 == GOLD["q18_rows"]
        drop(ox + cm_ + cx + cus + lis + ods)
        for x in (locals_, owneds, names):
            destroy(ctxs, x)


# ---------------------------------------------------------------------------------------------------- 7. cross-process (two or more GPUs)
def _worker(rank: int, world: int, rendezvous: str):
    """one rank of test_across_processes_when_there_are_two_gpus: its dictionary → unify → the unified strings as hex"""
    import json
    import sys
    import time

    from lingodb_b200 import parallel

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
    comm = parallel.Comm(ctx, rank, world, user_bytes=4 << 20, exchange=swap)
    loc = local_dict(ctx, shards_of(world, 1234)[rank])
    u = comm.dict_unify(loc)
    strs, rank_col = dict_strings(ctx, u)
    comm.check()
    with open(os.path.join(rendezvous, f"out{rank}.json"), "w") as f:
        json.dump({"strs": [s.hex() for s in strs], "rank": rank_col}, f)
    ctx.L.ldb_gpu_state_destroy(u)
    ctx.L.ldb_gpu_state_destroy(loc)
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
        pytest.skip("one GPU: the cross-process unification needs two")
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
    want = sorted(set(v for s in shards_of(world, 1234) for v in s))
    for r in range(world):
        got = json.load(open(tmp_path / f"out{r}.json"))
        assert [bytes.fromhex(s) for s in got["strs"]] == want and got["rank"] == list(range(len(want))), r


if __name__ == "__main__":  # a rank of the cross-process test, or an isolated case
    import sys
    if sys.argv[1] == "model":
        check_union(int(sys.argv[2]))
    else:
        _worker(int(sys.argv[1]), int(sys.argv[2]), sys.argv[3])
