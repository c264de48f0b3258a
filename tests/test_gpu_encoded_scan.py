"""Scan-reduce / scan-group-by pipelines over the frame-of-reference copy of DEVICE batches (csrc/encode.cu,
`ldb_gpu_set_encoded_scan`): the same inputs with the copy and with Arrow cells, both against the exact reference of
tests/_piperef.py, bit for bit — every registered signature, every decimal mix (so every width 1/2/4/8), equal-valued blocks, partial
blocks and tail tiles, fsb4 / date32 keys and filters, DEVICE next to HOST batches, unaligned buffers, captured and replayed
queries, clear + re-append into reused buffers, the memory budget and the byte counter."""
import ctypes as C
import os

import numpy as np
import pytest

import _piperef as P
import _progref as R

pytestmark = pytest.mark.gpu
COLS = P.PIPE_COLUMNS + [("d", "decimal128", 18, 2), ("k2", "int32", 0, 0)]
SCHEMA = P.schema_of(COLS)
TILE_ROWS, BLOCK_ROWS, HEADER = 512, 65536, 16
Q1, Q6 = P.SIGNATURES[0], P.SIGNATURES[2]


def rt():
    from lingodb_b200 import runtime
    return runtime


def capi():
    from lingodb_b200 import capi as c
    return c


@pytest.fixture
def ctx():
    c = rt().Context(0)
    c.L.ldb_gpu_set_encoded_scan(1)
    yield c
    c.L.ldb_gpu_set_encoded_scan(1)
    c.close()


def encoded_bytes(ctx):
    return int(ctx.L.ldb_gpu_context_encoded_bytes(ctx.h))


def copy_bytes(n, width):
    """size of one column's encoded copy (kernels.h encodedColumnBytes)"""
    tiles = (n + TILE_ROWS - 1) // TILE_ROWS
    return (tiles * HEADER + n * width + 15) // 16 * 16


def values(seed, n, mix, key_domain=4):
    """seeded rows; decimals by `mix` as in test_gpu_pipelines.values: tpch, negative, wide (|v| up to 10^18) or mixed"""
    v = P.gen_table(seed, n, COLS, key_domain=key_domain)
    rng = np.random.default_rng(seed)
    v["k2"] = [int(x) for x in rng.integers(0, 3, n)]
    dec = {"tpch": lambda: (rng.integers(0, 10**7, n), rng.integers(0, 11, n), rng.integers(0, 9, n), rng.integers(0, 10**5, n)),
           "negative": lambda: tuple(rng.integers(-10**7, 10**7, n) for _ in range(4)),
           "wide": lambda: tuple(rng.integers(-10**18 + 1, 10**18, n) for _ in range(4))}
    if mix == "mixed":
        a, b, c, d = dec["tpch"]()
        for arr in (a, b, c, d):
            arr[7::32] = rng.integers(1 << 31, 1 << 32, len(arr[7::32]))
            arr[19::96] = (1 << 31) - 1 - arr[19::96] % 3
    else:
        a, b, c, d = dec[mix]()
    for name, arr in zip("abcd", (a, b, c, d)):
        v[name] = [int(x) for x in arr]
    return v


def width_of(xs):
    r = max(xs) - min(xs)
    return 1 if r < 1 << 8 else 2 if r < 1 << 16 else 4 if r < 1 << 32 else 8


def held_bytes(vals, batches, cols):
    """bytes of the copies of `cols` of the DEVICE batches (a, b): one width per (batch, column), the widest of its blocks"""
    total = 0
    for a, b in batches:
        for c in cols:
            total += copy_bytes(b - a, max(width_of(vals[c][lo:min(lo + BLOCK_ROWS, b)]) for lo in range(a, b, BLOCK_ROWS)))
    return total


def device_columns(ctx, vals, a, b, shift=0):
    """torch CUDA buffers of rows a..b; shift > 0 starts every fixed-width column `shift` cells into its allocation"""
    import torch
    ch = {}
    for cname, phys, _, _ in COLS:
        buf, _ = R.column_buffers(phys, vals[cname][a:b])
        if phys == "utf8":
            ch[cname] = (torch.from_numpy(buf[0]).cuda(ctx.device), torch.from_numpy(buf[1]).cuda(ctx.device))
            continue
        raw = np.ascontiguousarray(buf).view(np.uint8).ravel()
        pad = shift * (raw.nbytes // (b - a))
        t = torch.from_numpy(np.concatenate([np.zeros(pad, np.uint8), raw])).cuda(ctx.device)
        ch[cname] = t[pad:]
    return ch


def table(ctx, vals, cuts=(), host=(), shift=0):
    """a Table of `vals` cut into batches at `cuts`; batch i is a borrowed DEVICE batch unless i is in `host`"""
    t = rt().Table(ctx, "t", R.specs_of(COLS))
    n = len(next(iter(vals.values())))
    edges = [0] + list(cuts) + [n]
    for bi, (a, b) in enumerate(zip(edges, edges[1:])):
        if bi in host:
            t.append_host({cname: R.column_buffers(phys, vals[cname][a:b])[0] for cname, phys, _, _ in COLS}, b - a)
        else:
            t.append_device(device_columns(ctx, vals, a, b, shift), b - a)
    ctx.synchronize()
    return t


def read_groups(ctx, s, n_aggs):
    c = capi()
    rows = (c.GroupRow * 4096)()
    n, e = C.c_int32(), c.Error()
    c.check(ctx.L.ldb_gpu_groupby_read(s, rows, 4096, C.byref(n), C.byref(e)), e)
    return {(r.keys[0], r.keys[1]): [r.aggs[i].value() for i in range(n_aggs)] for r in rows[: n.value]}


def run(ctx, src, keys, aggs, filters=()):
    c, run_ = capi(), rt()
    if not keys:
        s, e = C.c_void_p(), c.Error()
        c.check(ctx.L.ldb_gpu_simple_state_create(ctx.h, len(aggs), C.byref(s), C.byref(e)), e)
        try:
            run_.run_pipeline(ctx, "scan_reduce", src, filters=filters, aggs=aggs, sink=s)
            out = (c.I128 * 8)()
            c.check(ctx.L.ldb_gpu_simple_state_read(s, out, C.byref(e)), e)
            return {(): [out[i].value() for i in range(len(aggs))]}
        finally:
            run_.state_destroy(ctx, s)
    s = run_.groupby_state(ctx, len(keys), len(aggs), 64)
    try:
        run_.run_pipeline(ctx, "scan_groupby", src, filters=filters, keys=keys, aggs=aggs, sink=s)
        return read_groups(ctx, s, len(aggs))
    finally:
        run_.state_destroy(ctx, s)


def sig_aggs(sig, keys=("k", "k2")):
    nk, aggs = sig
    return list(keys)[:nk], [(e, ["abcd"[p] for p in pos]) for e, pos in aggs]


def both(ctx, src, keys, aggs, filters=()):
    """(encoded, Arrow) results of one query"""
    ctx.L.ldb_gpu_set_encoded_scan(1)
    enc = run(ctx, src, keys, aggs, filters)
    ctx.L.ldb_gpu_set_encoded_scan(0)
    try:
        arrow = run(ctx, src, keys, aggs, filters)
    finally:
        ctx.L.ldb_gpu_set_encoded_scan(1)
    return enc, arrow


def check(ctx, src, vals, keys, aggs, filters=()):
    want = P.scan_groupby(vals, SCHEMA, list(filters), keys, aggs)
    enc, arrow = both(ctx, src, keys, aggs, filters)
    assert enc == want
    assert arrow == want


# ---------------------------------------------------------------------------------------------------- results
@pytest.mark.parametrize("mix", ["tpch", "negative", "wide", "mixed"])
def test_every_signature_with_and_without_the_copy(ctx, mix):
    """a batch of one full block + 1 row (partial block, 1-row tail tile) and a batch smaller than a tile"""
    vals = values(11, BLOCK_ROWS + 1 + 300, mix)
    src = table(ctx, vals, cuts=(BLOCK_ROWS + 1,))
    for sig in P.SIGNATURES:
        keys, aggs = sig_aggs(sig)
        check(ctx, src, vals, keys, aggs)
    assert encoded_bytes(ctx) > 0


def test_widths_and_held_bytes(ctx):
    """a: 1 byte, b: 2, c: 4, d: 8, keys 1 — the held bytes are exactly the copies of the columns Q1 stages"""
    n = 3 * BLOCK_ROWS + 1000
    vals = values(4, n, "tpch")
    rng = np.random.default_rng(4)
    vals["a"] = [int(x) for x in rng.integers(-100, 150, n)]
    vals["b"] = [int(x) for x in rng.integers(-1000, 60000, n)]
    vals["c"] = [int(x) for x in rng.integers(0, 1 << 31, n)]
    vals["d"] = [int(x) for x in rng.integers(-10**17, 10**17, n)]
    src = table(ctx, vals)
    assert encoded_bytes(ctx) == 0
    keys, aggs = sig_aggs(Q1)
    check(ctx, src, vals, keys, aggs)
    assert [width_of(vals[c]) for c in "abcd"] == [1, 2, 4, 8]
    assert encoded_bytes(ctx) == held_bytes(vals, [(0, n)], ["k", "k2", "a", "b", "c", "d"])


def test_blocks_of_equal_values(ctx):
    n = 2 * BLOCK_ROWS + 777
    vals = values(5, n, "mixed")
    for name, v in (("a", 5), ("b", -7), ("c", 0), ("d", (1 << 40) + 3), ("k", 2), ("k2", -1)):
        vals[name][:BLOCK_ROWS] = [v] * BLOCK_ROWS
    for name in "abcd":
        vals[name][BLOCK_ROWS:] = [vals[name][BLOCK_ROWS]] * (n - BLOCK_ROWS)  # every block constant
    src = table(ctx, vals, cuts=(BLOCK_ROWS + 5,))
    for sig in (Q1, Q6):
        keys, aggs = sig_aggs(sig)
        check(ctx, src, vals, keys, aggs)


FILTERS = [
    [("i", "=", 5)], [("i", "!=", 5)], [("i", "<", 0)], [("i", "<=", -1)], [("i", ">", 100)], [("i", ">=", P.I32_MIN)], [("i", "notnull", 0)],
    [("i", "in", [0, 1, -1, 2, 3, P.I32_MIN, P.I32_MAX, 99])], [("i", ">", -50), ("i", "<=", 50)], [("i", "<", 1 << 40)],
    [("dt", ">=", "1994-01-01"), ("dt", "<", "1995-01-01")], [("dt", "<", "1970-01-01")], [("dt", "=", "2000-02-29")], [("dt", ">", "1990-01-01")],
    [("dt", "in", ["1970-01-01", "2000-02-29"])],
    [("fs", "=", "A")], [("fs", "!=", "")], [("fs", ">", "B")], [("fs", "<=", "B")], [("fs", ">=", "A")], [("fs", "<", "\x7f")],
    [("a", ">=", "0.05"), ("a", "<=", "0.07")], [("a", "<", 0)], [("a", ">", "-1.5")], [("a", "!=", "0")],
    [("s", "contains", "a")],
    [("i", ">", -(1 << 30)), ("dt", ">", "1900-01-01"), ("a", "<", "1000000000"), ("s", "contains", "a")],
]


def test_every_filter_op_and_fsb4_date32_keys(ctx):
    """keyless over full-range int32 / date32 / fsb4 columns; keyed by (fs, dt) over small domains that still span int32"""
    vals = values(21, 9000, "negative")
    vals["i"] = [x if j % 3 else (j % 200) - 100 for j, x in enumerate(vals["i"])]
    vals["dt"] = [x if j % 5 else 11016 for j, x in enumerate(vals["dt"])]  # 2000-02-29
    keyed = dict(vals)
    keyed["fs"] = [[P.I32_MIN, ord("A"), P.I32_MAX][j % 3] for j in range(9000)]
    keyed["dt"] = [[-5, 8766, 9131, 11016][(j // 3) % 4] for j in range(9000)]
    src, ksrc = table(ctx, vals, cuts=(2049,)), table(ctx, keyed, cuts=(4000,))
    for f in FILTERS:
        keys, aggs = sig_aggs(Q6)
        check(ctx, src, vals, keys, aggs, f)
        keys, aggs = sig_aggs(Q1, keys=("fs", "dt"))
        check(ctx, ksrc, keyed, keys, aggs, f)


def test_device_next_to_host_batches(ctx):
    """HOST batches keep their staged layout; DEVICE batches of the same table read their copies"""
    vals = values(8, 70_000 + 3000, "mixed")
    cuts = (1000, 1700, 70_000)  # the >= 65 536-row HOST batch goes through compressed staging
    src = table(ctx, vals, cuts=cuts, host=(1, 2))
    for sig in (Q1, Q6, P.SIGNATURES[4]):
        keys, aggs = sig_aggs(sig)
        check(ctx, src, vals, keys, aggs)
    keys, aggs = sig_aggs(Q1)
    assert encoded_bytes(ctx) == held_bytes(vals, [(0, 1000), (70_000, 73_000)], ["k", "k2", "a", "b", "c", "d"])
    host_only = table(ctx, vals, cuts=(5000,), host=(0, 1))
    before = encoded_bytes(ctx)
    check(ctx, host_only, vals, keys, aggs)
    assert encoded_bytes(ctx) == before


def test_unaligned_device_buffers(ctx):
    """columns that start one cell into their allocation: the Arrow scan uses plain loads, the copy is aligned"""
    vals = values(6, 5000, "mixed")
    src = table(ctx, vals, cuts=(1234,), shift=1)
    for sig in (Q1, Q6, P.SIGNATURES[8]):
        keys, aggs = sig_aggs(sig)
        check(ctx, src, vals, keys, aggs)


# ---------------------------------------------------------------------------------------------------- lifetime
def test_captured_query_replays_without_re_encoding(ctx):
    vals = values(9, BLOCK_ROWS + 4321, "tpch")
    src = table(ctx, vals, cuts=(600,))
    keys, aggs = sig_aggs(Q1)
    want = P.scan_groupby(vals, SCHEMA, [], keys, aggs)
    ctx.graph_begin()
    s = rt().groupby_state(ctx, len(keys), len(aggs), 64)
    rt().run_pipeline(ctx, "scan_groupby", src, keys=keys, aggs=aggs, sink=s)
    g = ctx.graph_end()
    try:
        held = encoded_bytes(ctx)
        assert held > 0  # built during the capture, outside the graph
        counts = []
        for _ in range(4):
            n0 = ctx.launch_count()
            g.launch()
            assert read_groups(ctx, s, len(aggs)) == want
            counts.append(ctx.launch_count() - n0)
        assert len(set(counts)) == 1  # the encoder's kernels count as launches: none ran again
        assert encoded_bytes(ctx) == held
        assert run(ctx, src, keys, aggs) == want  # the eager run agrees
    finally:
        g.destroy()
        rt().state_destroy(ctx, s)


def test_clear_and_reappend_into_reused_buffers(ctx):
    import torch
    vals = values(12, 3000, "tpch")
    other = values(13, 3000, "negative")
    keys, aggs = sig_aggs(Q1)
    t = rt().Table(ctx, "t", R.specs_of(COLS))
    bufs = device_columns(ctx, vals, 0, 3000)
    t.append_device(bufs, 3000)
    assert run(ctx, t, keys, aggs) == P.scan_groupby(vals, SCHEMA, [], keys, aggs)
    assert encoded_bytes(ctx) > 0
    t.clear()
    assert encoded_bytes(ctx) == 0
    fresh = device_columns(ctx, other, 0, 3000)
    for name, phys, _, _ in COLS:
        if phys != "utf8":
            bufs[name].copy_(fresh[name])  # same device addresses, different contents
        else:
            bufs[name] = fresh[name]
    torch.cuda.synchronize()
    t.append_device(bufs, 3000)
    check(ctx, t, other, keys, aggs)


def test_budget_leaves_later_batches_in_arrow_layout():
    n_batch = 20_000
    budget = 6 * copy_bytes(n_batch, 4) + 100  # room for one batch's copies at most
    old = os.environ.get("LDB_ENCODED_SCAN_MAX_BYTES")
    os.environ["LDB_ENCODED_SCAN_MAX_BYTES"] = str(budget)  # read when a context is created
    try:
        c = rt().Context(0)
    finally:
        if old is None:
            del os.environ["LDB_ENCODED_SCAN_MAX_BYTES"]
        else:
            os.environ["LDB_ENCODED_SCAN_MAX_BYTES"] = old
    try:
        c.L.ldb_gpu_set_encoded_scan(1)
        vals = values(14, 3 * n_batch, "negative")
        src = table(c, vals, cuts=(n_batch, 2 * n_batch))
        keys, aggs = sig_aggs(Q1)
        check(c, src, vals, keys, aggs)
        held = encoded_bytes(c)
        assert 0 < held <= budget
        check(c, src, vals, keys, aggs)  # a batch that did not fit is not retried
        assert encoded_bytes(c) == held
    finally:
        c.close()


def test_held_bytes_follow_clear_and_destroy(ctx):
    vals = values(15, 7000, "tpch")
    keys, aggs = sig_aggs(Q6)
    src = table(ctx, vals, cuts=(3500,))
    assert encoded_bytes(ctx) == 0
    check(ctx, src, vals, keys, aggs)
    one = encoded_bytes(ctx)
    assert one > 0
    second = table(ctx, vals)
    check(ctx, second, vals, keys, aggs)
    assert encoded_bytes(ctx) > one
    second.clear()
    assert encoded_bytes(ctx) == one
    ctx.L.ldb_gpu_table_destroy(src.h)
    ctx._tables.remove(src)
    assert encoded_bytes(ctx) == 0
    ctx.L.ldb_gpu_set_encoded_scan(0)
    second.append_device(device_columns(ctx, vals, 0, 7000), 7000)
    assert run(ctx, second, keys, aggs) == P.scan_groupby(vals, SCHEMA, [], keys, aggs)
    assert encoded_bytes(ctx) == 0  # switched off: no copy is built
